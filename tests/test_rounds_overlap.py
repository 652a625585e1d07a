"""The round commit settles each decided prefix of its stretch while the kernel is still running (yklt::settle_ahead,
csrc/yk_lattice_host.hpp). Every way a stretch can end must leave exactly what settling after the kernel leaves: the
guard's hand-off with re-keyed nodes still in the side list, a max_bindings cut, a full cluster whose asks fail in place,
and consecutive cycles with releases. Each case is checked against the oracle and against the CPU device shim, which
settles each stretch after it is decided."""
import numpy as np
import pytest

from yunikorn_k8shim_b200 import Engine, synth
from device_shim import check, dshim  # noqa: F401  (dshim: the shim fixture)
from test_rounds_host import maskfree

pytestmark = pytest.mark.gpu

ST_NOFIT = 2
BATCH = 4096
NO_UNIFORM = (1 << 30, 0)   # the shim's `auto` with a shortest uniform run no run reaches


def _engine_cycle(snap, max_bindings=None):
    with Engine.for_snapshot(snap, batch=BATCH) as e:
        ask, node, _ = e.cycle(snap.n_asks if max_bindings is None else max_bindings)
        out = dict(ask=ask, node=node, avail=e.nodes_available(np.arange(snap.n_nodes)), state=e.ask_states(np.arange(snap.n_asks)),
                   stats=e.stats())
    return out


def _same(got, want, states=True):
    assert np.array_equal(got["ask"], want["ask"]) and np.array_equal(got["node"], want["node"])
    assert np.array_equal(got["avail"], want["avail"])
    if states:
        assert np.array_equal(got["state"], want["state"])


def _knobs(monkeypatch, guard=None):
    monkeypatch.setenv("YK_ROUND_MIN", "1")
    if guard is not None:
        monkeypatch.setenv("YK_ROUND_GUARD", str(guard))


def test_guard_hand_off_with_a_side_list(dshim, oracle, monkeypatch):
    """zero weights: every round decides one ask and its node joins the side list; the guard hands the cycle to the host
    commit after 16 passes with 16 re-keyed nodes still in the side list"""
    s = maskfree(synth.reweigh(synth.perf(2_000, 40, 125), np.zeros(4)))
    want, shim = check(dshim, oracle, s, auto=True, uniform=NO_UNIFORM, round_min=1, batch=BATCH)
    assert shim["handoffs"] == 1 and shim["round_asks"] == 16
    _knobs(monkeypatch)
    got = _engine_cycle(s)
    _same(got, want)
    st = got["stats"]
    assert st["lattice_handoffs"] == 1 and st["round_passes"] == 16 and st["round_asks"] == 16 and st["sweep_launches"] > 0


def full_cluster():
    s = maskfree(synth.perf(800, 40, 125))
    s.node_total //= 12
    s.node_avail //= 12
    return s


def test_full_cluster_fails_in_place(dshim, oracle, monkeypatch):
    s = full_cluster()
    want, shim = check(dshim, oracle, s, auto=True, uniform=NO_UNIFORM, round_min=1, guard=0, batch=BATCH)
    assert (want["state"] == ST_NOFIT).sum() > 0 and shim["singles"] > 0
    _knobs(monkeypatch, guard=0)
    got = _engine_cycle(s)
    _same(got, want)
    st = got["stats"]
    assert st["round_asks"] == s.n_asks and st["round_single_steps"] == shim["singles"] and st["round_passes"] == shim["passes"]
    assert st["nofit"] == (want["state"] == ST_NOFIT).sum()


@pytest.mark.parametrize("cut", [1, 977, 3_001])
def test_max_bindings_cut(dshim, oracle, monkeypatch, cut):
    """a cut below what the cluster holds, on an open cluster and on a full one where some asks before the cut fail in place"""
    for s in (maskfree(synth.perf(3_000, 60, 125)), full_cluster()):
        want, shim = check(dshim, oracle, s, auto=True, uniform=NO_UNIFORM, round_min=1, guard=0, batch=BATCH, max_bindings=cut)
        assert len(want["ask"]) == cut
        _knobs(monkeypatch, guard=0)
        got = _engine_cycle(s, max_bindings=cut)
        _same(got, want, states=False)
        assert got["stats"]["allocations"] == cut and got["stats"]["batches"] == shim["batches"]


def test_two_cycles_with_releases(dshim, oracle, monkeypatch):
    """the second cycle starts from the first one's bindings less a third of them: the round commit and the host commit
    leave the same bindings, ask states and node tables"""
    snap = maskfree(synth.perf(3_000, 60, 125))
    want, _ = check(dshim, oracle, snap, auto=True, uniform=NO_UNIFORM, round_min=1, batch=BATCH)
    _knobs(monkeypatch)
    out = {}
    for commit in ("auto", "host"):
        with Engine.for_snapshot(snap, commit=commit, batch=BATCH) as e:
            ask, node, _ = e.cycle(snap.n_asks)
            assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"]), commit
            back = np.sort(ask[::3])
            e.release(back)
            e.asks_upsert(back, snap.ask_req[back], snap.ask_app[back], snap.ask_create[back], snap.ask_tol[back],
                          snap.ask_need[back], snap.ask_deny[back], snap.ask_prio[back], snap.ask_node[back], snap.ask_flags[back],
                          snap.ask_gang[back])
            ask2, node2, _ = e.cycle(snap.n_asks)
            out[commit] = (ask2, node2, e.nodes_available(np.arange(snap.n_nodes)), e.ask_states(np.arange(snap.n_asks)), e.stats())
    a, h = out["auto"], out["host"]
    for x, y in zip(a[:4], h[:4]):
        assert np.array_equal(x, y)
    assert len(a[0]) > 0 and a[4]["lattice_cycles"] == 2 and a[4]["round_asks"] > snap.n_asks and h[4]["lattice_cycles"] == 0
