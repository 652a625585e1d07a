"""Binpacking on the device commit (YK_FLAG_BINPACKING_DEVICE) on the GPU, through the C ABI: one ordered capacity fill per
uniform run (csrc/yk_uniform.cuh).  Bindings, node choices, final availability and ask states must equal the oracle's; the
fill counters must equal the CPU shim's (tests/host/binpack_shim.cpp) on the same snapshot; without the flag nothing
changes."""
import copy

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from test_binpack_host import (BP, bp, bshim, config_shapes, infinite_shares, mid_node, mixed_signature_gangs,  # noqa: F401
                               overcommitted, run as shim_run, shuffled_ranks)   # (bshim: the shim fixture)
from test_gpu_dims import ST_PENDING, YK_ERR_RANGE, nan_node, nan_repaired, widen
import test_sessions as ts

pytestmark = pytest.mark.gpu


def _run(s, want, **kw):
    from yunikorn_k8shim_b200 import Engine
    with Engine.for_snapshot(s, **kw) as e:
        ask, node, _ = e.cycle(s.n_asks)
        avail = e.nodes_available(np.arange(s.n_nodes))
        states = e.ask_states(np.arange(s.n_asks))
        st = e.stats()
    tag = (s.name, kw)
    assert np.array_equal(ask, want["ask"]), ("ask order differs", tag)
    assert np.array_equal(node, want["node"]), ("node choice differs", tag)
    assert np.array_equal(avail, want["avail"]), ("final availability differs", tag)
    assert np.array_equal(states, want["state"]), ("ask states differ", tag)
    return st


def _fill(s, want, commit="device", **kw):
    """the flag under `commit`: the cycle starts on the device and never takes a retry or a windowed / round stretch"""
    st = _run(s, want, commit=commit, binpacking_device=True, **kw)
    assert st["lattice_cycles"] == 1 and st["uniform_retries"] == 0 and st["lattice_subruns"] == 0, (s.name, st)
    assert st["round_asks"] == 0
    return st


def test_reference_shape(oracle):
    s = synth.reference_shape(5000, 400, 125, policy=BP)
    want = oracle.run(s)
    for commit in ("auto", "device"):
        st = _fill(s, want, commit=commit, batch=4096)
        assert st["uniform_asks"] == 50_000 and st["sweep_launches"] == 0 and st["uniform_runs"] == 1, commit
    st = _run(s, want, batch=4096)                          # no flag: the host commit, as before
    assert st["lattice_cycles"] == 0 and st["sweep_launches"] > 0
    st = _run(s, want, batch=4096, commit="host", binpacking_device=True)
    assert st["lattice_cycles"] == 0 and st["lattice_launches"] == 0


def test_runny_config_shapes(oracle):
    fills = 0
    for snap, batch in ((synth.runny(synth.perf(1500, 20, 100, policy=BP), 1), 4096),
                        (synth.runny(synth.perf(1500, 20, 100, masks=True, policy=BP), 2), 4096),
                        (synth.runny(synth.hier(400, 3, 3, 2, 40, policy=BP), 3), 512),
                        (synth.runny(synth.gangs(300, 60, 5, policy=BP), 4), 1000)):
        st = _fill(snap, oracle.run(snap), batch=batch)
        fills += st["uniform_runs"]
    assert fills > 500
    checked = 0
    for seed in range(40):
        s = config_shapes(seed)
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > 64:
            continue
        want = oracle.run(s)
        st = _run(s, want, commit="device", binpacking_device=True, batch=64)
        checked += st["lattice_cycles"]
    assert checked >= 30


@pytest.mark.parametrize("D", range(1, 9))
def test_every_dimension_count(oracle, D):
    s = bp(widen(synth.runny(synth.perf(1100, 20, 50, masks=True), D), D, D))
    st = _fill(s, oracle.run(s), batch=4096)
    assert st["uniform_asks"] > 0
    s = bp(widen(synth.reference_shape(600, 40, 125), D, D))
    st = _fill(s, oracle.run(s), commit="auto", batch=4096)
    assert st["uniform_asks"] == s.n_asks and st["sweep_launches"] == 0
    for seed in range(8):
        s = bp(synth.redim(synth.runny(synth.fuzz(seed), seed), D, seed))
        try:
            want = oracle.run(s)
        except RuntimeError:
            continue
        _run(s, want, commit="device", binpacking_device=True, batch=64)


@pytest.mark.parametrize("w", [[0, 0, 0, 0], [0, 1, 0, 0], [1, 0.5, 0, 0], [1e-3, 1e3, 0, 0], [1, 1, 1, 0], [0.1, 0.2, 0.3, 0.7]],
                         ids=["zero", "tw1_second", "tw1.5", "wide", "pods", "tenths"])
def test_configured_weights(oracle, w):
    for s in (synth.runny(synth.perf(600, 10, 60, masks=True, policy=BP, seed=3), 3), synth.kwok(600, 10, 250, variant="bare", policy=BP)):
        s = synth.reweigh(s, w)
        st = _fill(s, oracle.run(s), batch=4096)
        assert st["uniform_asks"] > 0


@pytest.mark.parametrize("D", [2, 4, 8])
def test_infinite_shares_and_rank_ties(oracle, D):
    s = infinite_shares(D)
    st = _fill(s, oracle.run(s), batch=1 << 16)
    assert st["uniform_asks"] == s.n_asks and st["uniform_runs"] == 1
    for seed in range(3):
        s = widen(shuffled_ranks(400, 40, 125, seed), D, D)
        st = _fill(s, oracle.run(s), batch=1 << 16)
        assert st["uniform_asks"] == s.n_asks


def test_edges(oracle):
    """capacity ending mid-node, over-committed clusters in both orders, gangs placed whole and handed off, max_bindings"""
    s = mid_node()
    _fill(s, oracle.run(s), batch=4096)
    for sensitive in (False, True):
        s = overcommitted(sensitive)
        st = _fill(s, oracle.run(s), batch=4096)
        assert st["allocations"] == 660 and st["uniform_asks"] == 900 and st["lattice_handoffs"] == 0
    handed = 0
    for seed in range(3):
        for fill in (0.5, 2.0):
            s = synth.gangs(300, 60, 5, seed=seed, fill=fill, policy=BP)
            s.ask_req[:] = s.ask_req[0]
            handed += _fill(s, oracle.run(s), batch=1000)["lattice_handoffs"]
        s = mixed_signature_gangs(seed)
        assert _fill(s, oracle.run(s), batch=1000)["lattice_handoffs"] == 1
    assert handed > 0
    from yunikorn_k8shim_b200 import Engine
    for seed in (1, 4, 9, 12):
        s = config_shapes(seed)
        k = max(1, len(oracle.run(s)["ask"]) // 2)
        want = oracle.run(s, max_bindings=k)
        with Engine.for_snapshot(s, batch=64, commit="device", binpacking_device=True) as e:
            ask, node, _ = e.cycle(k)
            assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
            assert np.array_equal(e.nodes_available(np.arange(s.n_nodes)), want["avail"])


@pytest.mark.parametrize("commit", ["device", "auto"])
def test_nan_score_is_a_clean_error(oracle, commit):
    from yunikorn_k8shim_b200 import Engine, YkError
    s = bp(nan_node())
    t = nan_repaired(s)
    want = oracle.run(t)
    A, N = np.arange(s.n_asks), np.arange(s.n_nodes)
    with Engine.for_snapshot(s, batch=4096, commit=commit, binpacking_device=True) as e:
        with pytest.raises(YkError) as ei:
            e.cycle(s.n_asks)
        assert ei.value.code == YK_ERR_RANGE
        st = e.stats()
        assert st["allocations"] == 0 and st["lattice_cycles"] == 1
        assert (e.ask_states(A) == ST_PENDING).all()
        assert np.array_equal(e.nodes_available(N), s.node_avail)
        e.nodes_upsert([5], t.node_total[[5]], t.node_avail[[5]], t.node_taint[[5]], t.node_label[[5]], s.node_rank()[[5]],
                       t.node_flags[[5]])
        ask, node, _ = e.cycle(s.n_asks)
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
        assert np.array_equal(e.nodes_available(N), want["avail"])
        assert e.stats()["lattice_cycles"] == 2


def test_counters_equal_the_shim(oracle, bshim):
    """uniform runs, fills (lattice launches: one per fill, no other kernel runs), uniform asks and hand-offs.  The batch
    holds every ask: in a placement-insensitive order the engine decides the whole order in one batch, the shim in
    `batch`-sized ones"""
    for s in (synth.reference_shape(600, 40, 125, policy=BP), overcommitted(True), mixed_signature_gangs(1),
              synth.runny(synth.perf(300, 10, 60, masks=True, policy=BP), 5), synth.runny(synth.hier(200, 2, 3, 2, 30, policy=BP), 6),
              synth.gangs(300, 60, 5, seed=1, fill=2.0, policy=BP)):
        batch = 8192
        if s.name.startswith("gangs"):
            s.ask_req[:] = s.ask_req[0]
        want = oracle.run(s)
        dev = _fill(s, want, batch=batch)
        c = []
        rc, ask, node, _, _ = shim_run(bshim, s, stats=c, batch=batch)
        assert rc == 0 and np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
        c = c[0]
        assert (dev["uniform_runs"], dev["uniform_asks"], dev["lattice_handoffs"], dev["lattice_launches"]) == \
            (c["uniform_runs"], c["uniform_asks"], c["handoffs"], c["uniform_attempts"]), s.name


# ---- sessions: releases, node upserts, removals, cordons between cycles ----
def _replay_two(m, batch, commit):
    """one host-commit engine and one flagged engine driven by the same script: both equal the model at every cycle"""
    from yunikorn_k8shim_b200 import Engine
    kw = dict(D=m.D, policy=m.policy, weights=m.weights, max_nodes=m.maxN, max_asks=m.maxA, max_apps=m.maxP,
              max_queues=m.maxQ, batch=batch)
    lattice = 0
    with Engine(commit="host", **kw) as h, Engine(commit=commit, binpacking_device=True, **kw) as d:
        for step in m.steps:
            if step[0] == "op":
                _, method, args, _ = step
                getattr(h, method)(**copy.deepcopy(args))
                getattr(d, method)(**copy.deepcopy(args))
                continue
            if step[0] != "cycle":
                continue
            c = step[1]
            mb = m.maxA if c.max_bindings is None else c.max_bindings
            before = d.stats()["lattice_cycles"]
            outs = []
            for e in (h, d):
                ask, node, _ = e.cycle(mb)
                outs.append((ask, node, e.nodes_available(c.present), e.ask_states(np.arange(m.maxA))))
            where = f"{m.name} [{commit}, batch {batch}] cycle {c.number}"
            for x, y in zip(outs[0], outs[1]):
                assert np.array_equal(x, y), where
            assert outs[1][0].tolist() == c.ask.tolist() and outs[1][1].tolist() == c.node.tolist(), where
            lattice += d.stats()["lattice_cycles"] - before
    return lattice


@pytest.mark.parametrize("seed", [104, 105, 106, 107])
def test_sessions_equal_the_host_commit(monkeypatch, seed):
    monkeypatch.setenv("YK_UNIFORM_MIN", str(ts.UNIFORM_MIN))
    m = ts.session(seed, 4, BP, 0)
    assert _replay_two(m, 64, "device") > 0
    _replay_two(m, 4096, "auto")
