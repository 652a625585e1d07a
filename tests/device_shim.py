"""The CPU test harness of the device commit: tests/host/device_shim.cpp runs the lattice kernel, the round commit, uniform
runs and binpacking fills as plain loops under the engine's own driver.  `load` compiles a shim of tests/host once per
process; `run` and `check` drive the device shim under the engine's commit knobs.  Not a test module (pytest does not
collect it): the test files import it."""
import ctypes as C
import functools
import os
import subprocess
import tempfile

import numpy as np
import pytest

from test_engine_host import run_engine_host

HERE = os.path.dirname(os.path.abspath(__file__))
INELIGIBLE = 100     # binpacking without the flag, negative weighted totals, duplicate NodeID ranks, mixed gangs
HOST_COMMIT = 101    # auto=True: the engine's choice starts the cycle on the host commit (nothing committed)
YK_ERR_RANGE = -5    # a NaN node score
# the device shim's counters, in its stats_out order
STATS = ("subruns", "fullscans", "sorts", "elems", "quick", "escalations", "handoffs", "batches", "uniform_attempts",
         "uniform_retries", "uniform_asks", "uniform_runs", "uniform_elements", "passes", "singles", "round_asks",
         "round_stretches", "parked", "device")


@functools.cache
def load(name):
    """tests/host/<name>.cpp as a loaded library, compiled once per process (the file is gone once it is loaded)"""
    with tempfile.TemporaryDirectory(prefix="yk_shim_") as d:
        out = os.path.join(d, name + ".so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-o", out,
                               os.path.join(HERE, "host", name + ".cpp")])
        return C.CDLL(out)


@pytest.fixture(scope="session")
def dshim():
    return load("device_shim")


def run(shim, s, rounds=1, binpacking=0, uniform=(0, 0), window=0, guard=-1, round_min=-1, auto=False, stats=None, **kw):
    """one cycle of snapshot s on the device shim -> run_engine_host's (rc, ask, node, state, avail).  The engine's knobs:
    auto is the engine's `auto` (its commit choice, first batch and routing; HOST_COMMIT when the cycle starts on the host
    commit); otherwise the forced `device` choice at `batch`, where rounds 1 is `auto`'s routing (round-eligible stretches
    on the round commit) and 0 forced `device`'s (the lattice kernel takes every stretch); binpacking 1 is
    YK_FLAG_BINPACKING_DEVICE; uniform = (shortest uniform run, first depth), 0 = off / the engine's rule; window, guard and
    round_min (YK_ROUND_MIN) of the round commit, 0 / < 0 / < 0 = the engine's.  `stats`, a list, gets the counters by
    name."""
    shim.host_set_device(C.c_int(rounds), C.c_int(binpacking), C.c_int(auto))
    shim.host_set_uniform(C.c_int(uniform[0]), C.c_int(uniform[1]))
    shim.host_set_rounds(C.c_int(window), C.c_int(guard), C.c_int(round_min))
    rows = []
    r = run_engine_host(shim, s, fn="device_host_run", rows=rows, **kw)
    if stats is not None:
        stats.append(dict(zip(STATS, rows[0])))
    return r


def check(shim, oracle, s, tag=None, **kw):
    """the shim's cycle equals the oracle's: bindings, node choices, final availability and (without a max_bindings cut)
    ask states -> (oracle result, counters).  (None, None) when the snapshot is not eligible for the device commit, or
    when it has a NaN node score: the oracle rejects it and the shim must report YK_ERR_RANGE."""
    try:
        want = oracle.run(s, max_bindings=kw.get("max_bindings") or -1)
    except RuntimeError:
        want = None
    st = []
    rc, ask, node, state, avail = run(shim, s, stats=st, **kw)
    if rc == INELIGIBLE:
        return None, None
    if want is None:
        assert rc == YK_ERR_RANGE, (tag, rc)
        return None, None
    assert rc == 0, (tag, rc)
    assert np.array_equal(ask, want["ask"]), tag
    assert np.array_equal(node, want["node"]), tag
    if kw.get("max_bindings") is None:
        assert np.array_equal(state, want["state"]), tag
    assert np.array_equal(avail, want["avail"]), tag
    return want, st[0]
