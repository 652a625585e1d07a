"""The round commit (csrc/yk_rounds.h) on the CPU: the header is single-source, so tests/host/device_shim.cpp compiles the
very code of yk_rounds_kernel into plain loops and drives it with the engine's own batch loop, segment loop and stretch
routing (`auto`'s).  Bindings, ask states and node availability must equal the oracle's; after every stretch the shim also checks that
the node order is exactly "every node once, ascending by (current key, NodeID rank)" -- spent nodes included."""
import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from device_shim import check, dshim  # noqa: F401  (dshim: the shim fixture)

ALL = (1 << 64) - 1


def maskfree(s):
    """the same snapshot without masks or gangs: no required / forbidden labels, no node name, every taint tolerated"""
    s.ask_need[:] = 0
    s.ask_deny[:] = 0
    s.ask_node[:] = -1
    s.ask_tol[:] = ALL
    s.ask_gang[:] = -1
    return s


def infinite_shares(s):
    """nodes 1 and 3 have no vcore: one with some left (-Inf share), one over-committed (+Inf share); half the asks request
    no vcore and can land there"""
    s.node_total[[1, 3], 0] = 0
    s.node_avail[1, 0], s.node_avail[3, 0] = 500, -500
    s.ask_req[::2, 0] = 0
    return s


def shrunk(s, f):
    """every node 1/f of its size, same shares: the cluster fills up"""
    s.node_total //= f
    s.node_avail //= f
    return s


@pytest.mark.parametrize("D", range(1, 9))
def test_rounds_match_oracle_on_fuzz(dshim, oracle, D):
    rounds = 0
    for seed in range(16):
        s = maskfree(synth.redim(synth.fuzz(seed), D, seed))
        s.policy = synth.POLICY_FAIR
        if seed % 2:   # one fifo leaf, no limit, one priority: a placement-insensitive order, round-eligible
            s.q_max[:] = -1
            s.q_sort[:] = 0
            s.ask_prio[:] = 0
            s.app_queue[:] = s.app_queue[0]
        if seed % 3 == 1:
            s = synth.reweigh(s, np.linspace(0.25, 2.0, D))
        if seed % 4 == 2 and D >= 2:
            s = infinite_shares(s)
        _, st = check(dshim, oracle, s, tag=(D, seed), batch=1 << 16, guard=0 if seed % 4 == 1 else -1)
        rounds += st["round_asks"] if st else 0   # (not eligible, or a NaN score)
    assert rounds > 100
    s = maskfree(synth.redim(synth.perf(600, 12, 60), D, 3))
    _, st = check(dshim, oracle, s, batch=1 << 16, guard=0)
    assert st["round_asks"] == s.n_asks and st["handoffs"] == 0 and st["subruns"] == 0


def test_front_nodes_reject_by_capacity(dshim, oracle):
    """small nodes at the front of the order take the small requests and reject the large ones: single steps"""
    s = synth.perf(400, 10, 60, seed=4)
    small = np.arange(0, 400, 7)
    s.node_total[small] = s.ask_req.min(axis=0) * 3
    s.node_avail[small] = s.node_total[small]
    _, st = check(dshim, oracle, s, batch=1 << 16, guard=0)
    assert st["singles"] > 0 and st["round_asks"] == s.n_asks


def test_overcommitted_cluster_fails_in_place(dshim, oracle):
    s = shrunk(synth.perf(40, 10, 60, seed=5), 10)
    want, st = check(dshim, oracle, s, batch=1 << 16, guard=0)
    assert (want["state"] == 2).sum() > 0 and st["singles"] > 0 and st["parked"] > 0 and st["round_asks"] == s.n_asks


def test_spent_nodes_leave_and_return(dshim, oracle):
    """nodes fill up during the stretch and leave the order; uniform runs between the stretches read the order they left
    behind, so every spent node has to be back in place under its final key"""
    s = shrunk(synth.runny(synth.perf(60, 8, 40, seed=6), 6), 8)
    _, st = check(dshim, oracle, s, batch=1 << 16, uniform=(6, 0), guard=0)
    assert st["parked"] > 0 and st["round_stretches"] >= 2 and st["uniform_asks"] > 0


def test_flat_requests_end_in_a_handoff(dshim, oracle):
    """{pods: 1} moves no weighted resource: the node just taken sorts first again, every round decides one ask, and the
    guard hands the stretch over to the host commit after 16 passes"""
    s = synth.kwok(30, 3, 200, variant="bare")
    _, st = check(dshim, oracle, s, batch=1 << 16)
    assert st["handoffs"] == 1 and st["passes"] == 16 and st["round_asks"] == 16
    s = synth.reweigh(synth.perf(50, 4, 40), np.zeros(4))   # zero weights: every key is 0
    _, st = check(dshim, oracle, s, batch=1 << 16)
    assert st["handoffs"] == 1 and st["round_asks"] < s.n_asks


@pytest.mark.parametrize("window", [1, 2, 3, 64])
def test_narrow_windows(dshim, oracle, window):
    """the prefix-minimum boundaries: a round of at most 1, 2, ... candidates"""
    for seed in range(4):
        s = maskfree(synth.fuzz(seed))
        check(dshim, oracle, s, tag=(window, seed), batch=1 << 16, window=window, guard=0)
    s = synth.perf(300, 8, 50, seed=7)
    _, st = check(dshim, oracle, s, batch=1 << 16, window=window, guard=0)
    assert st["round_asks"] == s.n_asks and st["passes"] >= s.n_asks // window


def test_max_bindings(dshim, oracle):
    for seed in (1, 2, 3):
        s = synth.perf(200, 6, 50, seed=seed)
        k = s.n_asks // 3
        _, st = check(dshim, oracle, s, batch=1 << 16, max_bindings=k, guard=0)
        assert 0 < st["round_asks"] <= k


def test_uniform_runs_around_round_stretches(dshim, oracle):
    for seed in range(6):
        s = maskfree(synth.runny(synth.perf(300, 10, 60, seed=seed), seed))
        _, st = check(dshim, oracle, s, tag=seed, batch=1 << 16, uniform=(8, 0), guard=0)
        assert st["uniform_asks"] > 0 and st["round_asks"] > 0 and st["round_stretches"] >= 2
        assert st["uniform_asks"] + st["round_asks"] == s.n_asks


def test_masked_and_quota_stretches_keep_the_lattice(dshim, oracle):
    """a stretch with masks, or a placement-sensitive order, is not round-eligible: the lattice kernel decides it"""
    s = synth.perf(300, 10, 40, masks=True)
    _, st = check(dshim, oracle, s, batch=1 << 16)
    assert st["round_asks"] == 0 and st["subruns"] > 0
    s = synth.perf(300, 10, 40)
    s.q_max[-1, 0] = 1 << 60      # a max on the queue: placement-sensitive, even when it never binds
    _, st = check(dshim, oracle, s, batch=1 << 16)
    assert st["round_asks"] == 0 and st["subruns"] > 0


def test_side_list_fills_and_goes_back_into_the_order(dshim, oracle):
    """more re-keyed nodes than the side list holds (2 048): it is merged back into the order and starts again"""
    s = synth.perf(3_000, 60, 125, seed=8)
    _, st = check(dshim, oracle, s, batch=1 << 16, guard=0)
    assert st["round_asks"] == s.n_asks and st["singles"] == 0
