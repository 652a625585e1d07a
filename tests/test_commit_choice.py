"""Which commit a cycle starts on under the default `auto` commit (yklt::choose_commit, csrc/yk_lattice_host.hpp), on
snapshots scaled down with the engine's knobs (the shortest uniform run, YK_UNIFORM_MIN, and the fewest asks of a round
commit cycle, YK_ROUND_MIN).  On the CPU the device shim makes the engine's choice and cuts the engine's first batch;
every cycle it starts on the device must equal the oracle.  On the GPU the engine, under `auto` and forced `device`, must
count what the shim counts."""
import copy

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from device_shim import HOST_COMMIT, INELIGIBLE, check, dshim, run  # noqa: F401  (dshim: the shim fixture)
from test_rounds_host import maskfree

BP = synth.POLICY_BINPACKING
BATCH = 4096           # the engine's default batch
NO_UNIFORM = 1 << 30   # a shortest uniform run no run reaches


def duplicate_ranks(s):
    """two nodes share a NodeID rank"""
    r = s.node_rank()
    r[1] = r[0]
    s.node_rank = lambda: r
    return s


def negative_weight(s):
    s.weights = np.array(s.weights, dtype=np.float64)
    s.weights[0] = -1.0
    return s


def cases():
    """(name, snapshot, knobs, binpacking flag, starts on the device).  Knobs: the shortest uniform run and the round
    commit's fewest asks."""
    ref = synth.reference_shape(600, 40, 125)                          # one uniform run of 5 000 identical pods: long enough to
                                                                       # pay for the run's fixed cost
    fair = maskfree(synth.perf(200, 20, 30))                           # 600 mask-free asks of many shapes
    n = fair.n_asks
    runny = synth.runny(synth.perf(300, 10, 60, masks=True, policy=BP), 5)
    return [
        ("uniform run", ref, (64, -1), 0, True),
        ("mask-free at the round minimum", fair, (NO_UNIFORM, n), 0, True),
        ("mask-free below the round minimum", fair, (NO_UNIFORM, n + 1), 0, False),
        ("masked runs", synth.perf(200, 20, 30, masks=True), (16, 1), 0, False),
        ("runny binpacking", runny, (32, -1), 1, False),
        ("one binpacking run", synth.reference_shape(600, 30, 125, policy=BP), (64, -1), 1, True),
        ("binpacking without the flag", synth.reference_shape(100, 8, 50, policy=BP), (64, -1), 0, False),
        ("duplicate ranks", duplicate_ranks(copy.deepcopy(ref)), (64, -1), 0, False),
        ("negative weight", negative_weight(copy.deepcopy(ref)), (64, -1), 0, False),
        ("mixed-vector gangs", synth.poisoned_gangs(3), (16, 1), 0, False),
        ("quota'd order", maskfree(synth.hier(40, 2, 2, 2, 20)), (NO_UNIFORM, 1), 0, False),
    ]


CASES = cases()
IDS = [c[0] for c in CASES]


def knobs(k, guard=-1):
    return dict(uniform=(k[0], 0), round_min=k[1], guard=guard)


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_choice(dshim, oracle, case):
    name, s, k, flag, device = case
    if name == "quota'd order":
        assert (s.q_max >= 0).any()
    if device:
        want, st = check(dshim, oracle, s, tag=name, auto=True, binpacking=flag, batch=BATCH, **knobs(k))
        assert want is not None and st["device"] == 1, name
        assert st["uniform_asks"] + st["round_asks"] > 0, (name, st)
    else:
        assert run(dshim, s, auto=True, binpacking=flag, batch=BATCH, **knobs(k))[0] == HOST_COMMIT, name


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["auto", "device"])
@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_engine_counts_what_the_shim_counts(dshim, oracle, monkeypatch, case, commit):
    from yunikorn_k8shim_b200 import Engine
    name, s, k, flag, _ = case
    monkeypatch.setenv("YK_UNIFORM_MIN", str(k[0]))
    monkeypatch.setenv("YK_ROUND_MIN", str(k[1] if k[1] >= 0 else 10000))
    monkeypatch.setenv("YK_ROUND_GUARD", "0")
    c = []
    # forced: the engine decides a placement-insensitive order in one batch, the shim in `batch`-sized ones
    rc = run(dshim, s, auto=commit == "auto", rounds=0, binpacking=flag, batch=BATCH if commit == "auto" else max(BATCH, s.n_asks),
             stats=c, **knobs(k, guard=0))[0]
    c = c[0]
    want = oracle.run(s)
    with Engine.for_snapshot(s, batch=BATCH, commit=commit, binpacking_device=bool(flag)) as e:
        ask, node, _ = e.cycle(s.n_asks)
        st = e.stats()
    if name != "duplicate ranks":   # the oracle ranks NodeIDs itself
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"]), name
    if rc in (HOST_COMMIT, INELIGIBLE):
        assert st["lattice_cycles"] == 0, (name, st)
        return
    assert rc == 0, (name, rc)
    got = tuple(st[x] for x in ("lattice_cycles", "batches", "uniform_runs", "uniform_asks", "round_asks", "lattice_handoffs"))
    assert got == tuple(c[x] for x in ("device", "batches", "uniform_runs", "uniform_asks", "round_asks", "handoffs")), (name, c, st)
