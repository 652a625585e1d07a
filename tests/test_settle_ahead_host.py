"""Settling a batch while it is being decided (yklt::settle_ahead, yklt::settle_back in csrc/yk_lattice_host.hpp), on the
CPU through tests/host/settle_shim.cpp: the device commit's batch loop over one placement-insensitive batch, decided by a
sequential first fit and settled a prefix at a time, the way the engine settles what the round kernel publishes.  Settled
in prefixes of any length, the cycle equals the oracle's; a batch that ends on a NaN after some prefixes were settled
binds nothing and leaves every ask in flight, its counters at zero and the orderer's application totals as they were."""
import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from device_shim import load
from test_engine_host import run_engine_host
from test_rounds_host import maskfree

YK_ERR_RANGE = -5
ST_ALLOCATED, ST_NOFIT = 1, 2


@pytest.fixture(scope="module")
def sshim():
    return load("settle_shim")


def snapshots():
    open_ = maskfree(synth.perf(60, 6, 40))      # 240 asks, all placed
    full = maskfree(synth.perf(60, 6, 40))
    full.node_total //= 40
    full.node_avail //= 40                       # some asks fail in place
    return {"open": open_, "full": full}


def _run(shim, s, chunk, nan_at=-1):
    shim.settle_set(chunk, nan_at)
    rows = []
    rc, ask, node, state, avail = run_engine_host(shim, s, fn="settle_host_run", rows=rows)
    allocations, nofit, ahead, app_back = rows[0][:4]
    return rc, ask, node, state, avail, dict(allocations=allocations, nofit=nofit, ahead=ahead, app_back=app_back)


@pytest.mark.parametrize("name", ["open", "full"])
@pytest.mark.parametrize("chunk", [1, 7, 64, 1 << 20])
def test_settled_in_prefixes_equals_the_oracle(sshim, oracle, name, chunk):
    s = snapshots()[name]
    want = oracle.run(s)
    rc, ask, node, state, avail, c = _run(sshim, s, chunk)
    assert rc == 0
    assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
    assert np.array_equal(state, want["state"]) and np.array_equal(avail, want["avail"])
    assert c["allocations"] == len(ask) and c["nofit"] == (want["state"] == ST_NOFIT).sum()
    assert c["ahead"] == s.n_asks // chunk
    if name == "full":
        assert c["nofit"] > 0


@pytest.mark.parametrize("name", ["open", "full"])
@pytest.mark.parametrize("chunk,nan_at", [(1, 0), (1, 1), (7, 50), (7, 239), (64, 200), (1 << 20, 100)])
def test_nan_takes_the_settled_prefix_back(sshim, name, chunk, nan_at):
    s = snapshots()[name]
    rc, ask, node, state, avail, c = _run(sshim, s, chunk, nan_at)
    assert rc == YK_ERR_RANGE
    assert len(ask) == 0
    assert not np.isin(state, [ST_ALLOCATED, ST_NOFIT]).any()
    assert np.array_equal(state, _run(sshim, s, 1 << 20, nan_at)[3])   # as if nothing had been settled ahead
    assert c["allocations"] == 0 and c["nofit"] == 0 and c["app_back"] == 1
    assert c["ahead"] == nan_at // chunk
