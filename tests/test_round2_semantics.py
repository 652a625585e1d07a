"""Semantics tightened in round 2, checked on the oracle, the independent Python restatement, the host engine shim (real
orderer + real host commit) and the device shim (real orderer + the device commit's code compiled for the CPU):
  * a weighted resource with total == 0: Go's float division gives +-Inf shares (0/0 = NaN is skipped), not "absent";
  * gangs are all-or-nothing whichever member is the bad one (ADVICE round 1: the first-reached member used to be dropped
    alone, the rest scheduled as a smaller gang);
  * slow-path members of a sunk gang are reported whether or not the order is placement-sensitive."""
import ctypes as C

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from oracle import py_oracle
import device_shim
from test_engine_host import run_engine_host


@pytest.fixture(scope="module")
def shims():
    return {"engine_shim": device_shim.load("engine_shim"), "device_shim": device_shim.load("device_shim")}


def everywhere(shims, oracle, s, batch=64):
    want = oracle.run(s)
    p = py_oracle.run(s)
    assert list(want["ask"]) == p["ask"] and list(want["node"]) == p["node"] and list(want["state"]) == p["state"]
    rc, ask, node, state, avail = run_engine_host(shims["engine_shim"], s, batch=batch)
    assert rc == 0 and np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"]) and np.array_equal(state, want["state"])
    rc, ask, node, state, avail = device_shim.run(shims["device_shim"], s, rounds=0, batch=batch)
    if rc != device_shim.INELIGIBLE:
        assert rc == 0 and np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"]) and np.array_equal(state, want["state"])
    return want


def test_zero_total_on_a_weighted_resource_is_an_infinite_share(shims, oracle):
    inf = float("inf")
    w = np.array([1.0, 1.0, 0.0, 0.0])
    tot = np.array([0, 64 << 30, 110, 0], dtype=np.int64)
    assert oracle.node_score(0, w, tot, np.array([-5, 32 << 30, 110, 0], dtype=np.int64)) == inf    # 1 - (-5/0) = +Inf
    assert oracle.node_score(0, w, tot, np.array([7, 32 << 30, 110, 0], dtype=np.int64)) == -inf     # 1 - (+7/0) = -Inf
    assert oracle.node_score(0, w, tot, np.array([0, 32 << 30, 110, 0], dtype=np.int64)) == 0.5      # 0/0 = NaN: skipped
    assert py_oracle.node_score(0, w, tot, np.array([-5, 32 << 30, 110, 0])) == inf
    assert py_oracle.node_score(0, w, tot, np.array([7, 32 << 30, 110, 0])) == -inf
    assert py_oracle.node_score(0, w, tot, np.array([0, 32 << 30, 110, 0])) == 0.5
    lib = shims["engine_shim"]
    lib.score_host.restype = C.c_double
    for av, exp in ((-5, inf), (7, -inf), (0, 0.5)):
        a = np.array([av, 32 << 30, 110, 0], dtype=np.int64)
        assert lib.score_host(C.c_int(4), C.c_uint32(0), w.ctypes.data_as(C.c_void_p), tot.ctypes.data_as(C.c_void_p),
                              a.ctypes.data_as(C.c_void_p)) == exp
    # in a cycle: the over-committed zero-CPU node sorts last under fair; asks that need no CPU still reach it last
    s = synth.perf(6, 1, 12)
    s.node_total[2, 0] = 0
    s.node_avail[2, 0] = -100
    s.ask_req[:, 0] = 0
    want = everywhere(shims, oracle, s)
    assert len(want["node"]) == 12 and 2 not in set(want["node"][:5].tolist())


def _gang_snapshot(bad_member, bad_kind):
    s = synth.perf(8, 2, 6)
    s.ask_gang[:] = -1
    s.ask_gang[0:4] = 7                      # application 0: a gang of four, then two plain asks
    if bad_kind == "slow":
        s.ask_flags[bad_member] = 1
    elif bad_kind == "invalid":
        s.ask_req[bad_member] = 0
    return s


@pytest.mark.parametrize("bad_kind,state", [("slow", 4), ("invalid", 5)])
def test_a_gang_sinks_whole_whichever_member_is_bad(shims, oracle, bad_kind, state):
    outs = []
    for bad in range(4):
        s = _gang_snapshot(bad, bad_kind)
        want = everywhere(shims, oracle, s, batch=16)
        assert list(want["state"][:4]) == [state] * 4, (bad, want["state"][:6])     # nobody of the gang is placed
        assert set(want["ask"].tolist()) == set(range(4, 12))
        outs.append((tuple(want["ask"]), tuple(want["node"])))
    assert len(set(outs)) == 1               # and the rest of the cycle does not depend on which member it was


def test_quota_sinks_a_gang_whole(shims, oracle):
    s = synth.hier(20, 1, 2, 1, 8, seed=3)
    s.ask_gang[:] = -1
    s.ask_gang[0:4] = 1
    leaf = int(s.app_queue[s.ask_app[0]])
    s.q_max[leaf] = -1
    s.q_max[leaf, 2] = 3                      # three pods fit the leaf's quota, the gang has four members
    want = everywhere(shims, oracle, s, batch=16)
    assert list(want["state"][:4]) == [3] * 4


def test_user_limits_through_orderer_and_commits(shims, oracle):
    """user / group resource limits (a14): per (queue, user) maxima fold into the headroom of the user's applications, on
    leaves and on their ancestors, in placement-sensitive orders with rewinds, gangs and fair leaves"""
    changed = 0
    for seed in range(40):
        s = synth.with_user_limits(synth.fuzz(seed), seed=seed)
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > 64:
            continue
        want = everywhere(shims, oracle, s, batch=64)
        changed += int(list(want["ask"]) != list(oracle.run(synth.fuzz(seed))["ask"]))
    assert changed > 10
    for s in (synth.with_user_limits(synth.hier(300, 3, 4, 2, 40, seed=21), n_users=4, seed=1, frac=0.3),
              synth.with_user_limits(synth.perf(200, 6, 50), n_users=2, seed=2, frac=0.4)):
        want = everywhere(shims, oracle, s, batch=128)
        assert (want["state"] == 3).sum() > 0          # some asks end SKIPPED on the user's headroom
