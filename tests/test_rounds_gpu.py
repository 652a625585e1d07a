"""The round commit (csrc/yk_rounds.h) on the GPU, through the C ABI: the default (auto) commit takes big mask-free cycles
in a placement-insensitive order, and its bindings, ask states and node tables are bit-identical to the oracle's."""
import numpy as np
import pytest

from yunikorn_k8shim_b200 import Engine, synth

pytestmark = pytest.mark.gpu


def _run(snap, want, **kw):
    with Engine.for_snapshot(snap, **kw) as e:
        ask, node, _ = e.cycle(snap.n_asks)
        avail = e.nodes_available(np.arange(snap.n_nodes))
        states = e.ask_states(np.arange(snap.n_asks))
        st = e.stats()
    assert np.array_equal(ask, want["ask"]), ("ask order differs", kw)
    assert np.array_equal(node, want["node"]), ("node choice differs", kw)
    assert np.array_equal(avail, want["avail"]), kw
    assert np.array_equal(states, want["state"]), kw
    return st


def test_config2_takes_the_round_commit(oracle):
    snap = synth.perf()
    st = _run(snap, oracle.run(snap), batch=2048)
    assert st["lattice_cycles"] == 1 and st["round_asks"] == 50_000 and st["lattice_asks"] == 50_000
    assert st["sweep_launches"] == 0 and st["lattice_handoffs"] == 0 and st["lattice_subruns"] == 0
    assert st["round_passes"] < 1_000


def test_large_mask_free_cycle(oracle):
    snap = synth.perf(50_000, 2_000, 125)
    st = _run(snap, oracle.run(snap))
    assert st["lattice_cycles"] == 1 and st["round_asks"] == snap.n_asks and st["sweep_launches"] == 0


def test_masked_cycle_stays_on_the_host(oracle):
    snap = synth.perf(masks=True)
    st = _run(snap, oracle.run(snap), batch=2048)
    assert st["lattice_cycles"] == 0 and st["round_passes"] == 0 and st["sweep_launches"] > 0


def test_reference_shape_is_one_uniform_run(oracle):
    snap = synth.reference_shape()
    st = _run(snap, oracle.run(snap), batch=4096)
    assert st["uniform_runs"] == 1 and st["uniform_asks"] == 50_000 and st["round_passes"] == 0


def test_uniform_runs_and_round_stretches_in_one_batch(oracle, monkeypatch):
    """config 2 with two runs of 3 000 identical asks inside: uniform runs and round stretches alternate in one batch, on
    the same device-resident node state"""
    snap = synth.perf()
    for lo in (10_000, 30_000):
        snap.ask_req[lo:lo + 3_000] = snap.ask_req[lo]
    st = _run(snap, oracle.run(snap), batch=2048)
    assert st["lattice_cycles"] == 1 and st["uniform_runs"] == 2 and st["uniform_asks"] >= 6_000   # (a run may extend
    assert st["uniform_asks"] + st["round_asks"] == 50_000                                           # into its neighbours)
    assert st["lattice_subruns"] == 0 and st["sweep_launches"] == 0
    monkeypatch.setenv("YK_ROUND_MIN", "1")
    monkeypatch.setenv("YK_ROUND_GUARD", "0")
    monkeypatch.setenv("YK_ROUND_WINDOW", "2")   # rounds of at most two candidates
    snap = synth.perf(300, 10, 60)
    st = _run(snap, oracle.run(snap), batch=4096)
    assert st["round_asks"] == snap.n_asks and st["round_passes"] >= snap.n_asks // 2


def test_short_rounds_hand_over_to_the_host_commit(oracle, monkeypatch):
    """zero weights: every key is 0, the node just taken sorts first again and every round decides one ask"""
    monkeypatch.setenv("YK_ROUND_MIN", "1")
    snap = synth.reweigh(synth.perf(2_000, 40, 125), np.zeros(4))
    st = _run(snap, oracle.run(snap), batch=4096)
    assert st["lattice_cycles"] == 1 and st["lattice_handoffs"] == 1 and st["round_passes"] == 16
    assert st["round_asks"] == 16 and st["sweep_launches"] > 0


def test_full_cluster_single_steps_and_spent_nodes(oracle, monkeypatch):
    monkeypatch.setenv("YK_ROUND_MIN", "1")
    monkeypatch.setenv("YK_ROUND_GUARD", "0")
    snap = synth.perf(800, 40, 125)
    snap.node_total //= 12
    snap.node_avail //= 12
    want = oracle.run(snap)
    assert (want["state"] == 2).sum() > 0
    st = _run(snap, want, batch=4096)
    assert st["round_asks"] == snap.n_asks and st["round_single_steps"] > 0


def test_two_auto_cycles_with_releases(oracle, monkeypatch):
    """two consecutive cycles on one engine, some allocations released between them: the round commit and the host commit
    leave the same bindings and the same node tables, bit for bit"""
    monkeypatch.setenv("YK_ROUND_MIN", "1000")
    snap = synth.perf(3_000, 60, 125)
    want = oracle.run(snap)
    out = {}
    for commit in ("auto", "host"):
        with Engine.for_snapshot(snap, commit=commit, batch=2048) as e:
            ask, node, _ = e.cycle(snap.n_asks)
            assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"]), commit
            back = np.sort(ask[::3])
            e.release(back)   # released pods come back as new asks
            e.asks_upsert(back, snap.ask_req[back], snap.ask_app[back], snap.ask_create[back], snap.ask_tol[back],
                          snap.ask_need[back], snap.ask_deny[back], snap.ask_prio[back], snap.ask_node[back], snap.ask_flags[back],
                          snap.ask_gang[back])
            ask2, node2, _ = e.cycle(snap.n_asks)
            out[commit] = (ask2, node2, e.nodes_available(np.arange(snap.n_nodes)), e.ask_states(np.arange(snap.n_asks)), e.stats())
    a, h = out["auto"], out["host"]
    for x, y in zip(a[:4], h[:4]):
        assert np.array_equal(x, y)
    assert len(a[0]) > 0 and a[4]["lattice_cycles"] == 2 and a[4]["round_asks"] > snap.n_asks and h[4]["lattice_cycles"] == 0
