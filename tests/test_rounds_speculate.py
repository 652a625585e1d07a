"""The speculative round-commit launch (csrc/yk_spec.h, DESIGN.md §6.3) on the GPU: the device orders the cycle's asks and
starts yk_rounds_kernel before the host has set the cycle up, and the host adopts that launch only when its own first batch
and plan are exactly it.

Adopted: bindings, node choices, availability and ask states equal the oracle's, and passes, single steps, round asks and
hand-offs equal the CPU device shim's, as in test_rounds_parity.  Discarded or never started: everything equals the
oracle's, and a second cycle on the same engine (after releases) equals the host commit's.  A NaN node score: the adopted
kernel decides nothing and the cycle fails as before, with the tables unchanged."""
import numpy as np
import pytest

from yunikorn_k8shim_b200 import Engine, synth
from device_shim import dshim  # noqa: F401  (the shim fixture)
from test_gpu_dims import ST_PENDING, YK_ERR_RANGE, nan_node, nan_repaired
from test_rounds_parity import COUNTERS, GUARD, Run, _device, _knobs, _mb_base, _shim, guard_trip, insensitive, spent_many

pytestmark = pytest.mark.gpu


def _adopted(dshim, oracle, monkeypatch, r, cycles=1):
    want, shim = _shim(dshim, oracle, r)
    st = _device(monkeypatch, r, want)
    assert {k: st[k] for k in COUNTERS} == {k: shim[k] for k in COUNTERS}, (r, st, shim)
    assert st["spec_adopted"] == cycles and st["spec_discarded"] == 0, (r, st["spec_adopted"], st["spec_discarded"])
    return st


def _oracle_cycle(snap, want, **kw):
    with Engine.for_snapshot(snap, **kw) as e:
        ask, node, _ = e.cycle(snap.n_asks)
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
        assert np.array_equal(e.nodes_available(np.arange(snap.n_nodes)), want["avail"])
        assert np.array_equal(e.ask_states(np.arange(snap.n_asks)), want["state"])
        return e.stats()


def test_config2_is_adopted(oracle):
    snap = synth.perf()
    st = _oracle_cycle(snap, oracle.run(snap), batch=2048)
    assert st["spec_adopted"] == 1 and st["spec_discarded"] == 0 and st["round_asks"] == 50_000 and st["sweep_launches"] == 0


def test_250k_asks_are_adopted(oracle):
    snap = synth.perf(50_000, 2_000, 125)
    st = _oracle_cycle(snap, oracle.run(snap))
    assert st["spec_adopted"] == 1 and st["round_asks"] == snap.n_asks


@pytest.mark.parametrize("case", ["guard-handoff", "full-cluster", "max-bindings"])
def test_adopted_launch_matches_shim(dshim, oracle, monkeypatch, case):
    runs = {"guard-handoff": [Run(guard_trip(D), guard=GUARD) for D in (1, 8)],
            "full-cluster": [Run(spent_many())],
            "max-bindings": [Run(_mb_base(), mb=100), Run(_mb_base(40), mb=300)]}[case]
    for r in runs:
        st = _adopted(dshim, oracle, monkeypatch, r)
        if case == "guard-handoff":
            assert st["lattice_handoffs"] == 1


def _two_cycles(snap, commit, **kw):
    """a cycle, a third of its allocations released and upserted again, a second cycle"""
    with Engine.for_snapshot(snap, commit=commit, **kw) as e:
        ask, node, _ = e.cycle(snap.n_asks)
        back = np.sort(ask[::3])
        e.release(back)
        e.asks_upsert(back, snap.ask_req[back], snap.ask_app[back], snap.ask_create[back], snap.ask_tol[back], snap.ask_need[back],
                      snap.ask_deny[back], snap.ask_prio[back], snap.ask_node[back], snap.ask_flags[back], snap.ask_gang[back])
        ask2, node2, _ = e.cycle(snap.n_asks)
        return (ask, node, ask2, node2, e.nodes_available(np.arange(snap.n_nodes)), e.ask_states(np.arange(snap.n_asks))), e.stats()


def test_second_cycle_after_releases_is_adopted(oracle, monkeypatch):
    monkeypatch.setenv("YK_ROUND_MIN", "1000")
    snap = synth.perf(3_000, 60, 125)
    want = oracle.run(snap)
    a, sa = _two_cycles(snap, "auto", batch=2048)
    h, _ = _two_cycles(snap, "host", batch=2048)
    assert np.array_equal(a[0], want["ask"]) and np.array_equal(a[1], want["node"])
    for x, y in zip(a, h):
        assert np.array_equal(x, y)
    assert sa["spec_adopted"] == 2 and sa["spec_discarded"] == 0 and sa["lattice_cycles"] == 2


def _mixed_prio(s):
    s.ask_prio[::7] = 1
    return s


def _fair_leaf(s):
    s.q_sort[:] = 1
    return s


def _quota(s):
    s.q_max[:, 0] = 10 ** 15
    return s


def _gangs(s):
    s.ask_gang[:40] = 3
    s.ask_app[:40] = s.ask_app[0]
    return s


DISCARDED = {
    "reference-shape": lambda: synth.reference_shape(2_000, 100, 125),
    "config3-masks": lambda: synth.perf(2_000, 100, 125, masks=True),
    "gangs": lambda: _gangs(insensitive(synth.perf(2_000, 100, 125))),
    "mixed-priorities": lambda: _mixed_prio(insensitive(synth.perf(2_000, 100, 125))),
    "fair-leaf": lambda: _fair_leaf(insensitive(synth.perf(2_000, 100, 125))),
    "quota": lambda: _quota(insensitive(synth.perf(2_000, 100, 125))),
    "user-limit": lambda: synth.with_user_limits(insensitive(synth.perf(2_000, 100, 125))),
}


@pytest.mark.parametrize("name", list(DISCARDED))
def test_discarded_or_not_launched(oracle, monkeypatch, name):
    monkeypatch.setenv("YK_ROUND_MIN", "1000")
    snap = DISCARDED[name]()
    want = oracle.run(snap)
    a, sa = _two_cycles(snap, "auto", batch=2048)
    h, _ = _two_cycles(snap, "host", batch=2048)
    assert np.array_equal(a[0], want["ask"]) and np.array_equal(a[1], want["node"]), name
    for x, y in zip(a, h):
        assert np.array_equal(x, y), name
    assert sa["spec_adopted"] == 0, (name, sa["spec_adopted"], sa["spec_discarded"])


def test_nan_node_score_is_adopted_and_decides_nothing(dshim, oracle, monkeypatch):
    from yunikorn_k8shim_b200 import YkError
    s = nan_node()
    t = nan_repaired(s)
    r = Run(t)
    want, shim = _shim(dshim, oracle, r)
    A, N = np.arange(s.n_asks), np.arange(s.n_nodes)
    _knobs(monkeypatch, r)
    with Engine.for_snapshot(s, batch=4096) as e:
        with pytest.raises(YkError) as ei:
            e.cycle(s.n_asks)
        assert ei.value.code == YK_ERR_RANGE
        st = e.stats()
        assert st["allocations"] == 0 and st["round_asks"] == 0 and st["round_passes"] == 0 and st["spec_adopted"] == 1
        assert (e.ask_states(A) == ST_PENDING).all()
        assert np.array_equal(e.nodes_available(N), s.node_avail)
        e.nodes_upsert([5], t.node_total[[5]], t.node_avail[[5]], t.node_taint[[5]], t.node_label[[5]], s.node_rank()[[5]],
                       t.node_flags[[5]])
        ask, node, _ = e.cycle(s.n_asks)
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
        assert np.array_equal(e.nodes_available(N), want["avail"])
        st2 = e.stats()
    assert st2["spec_adopted"] == 2
    assert {k: st2[k] - st[k] for k in COUNTERS} == {k: shim[k] for k in COUNTERS}
