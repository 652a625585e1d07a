"""Binpacking on the device commit (YK_FLAG_BINPACKING_DEVICE), on the CPU.

Under the binpacking node sort a node's key never rises when it is allocated to, so a uniform run (consecutive asks with one
request vector and one predicate signature) fills the nodes in their ascending (key, NodeID rank) order, each one to its
capacity before the next: one sort, one 64-bit scan and one search per ask (csrc/yk_uniform.h, DESIGN.md §6.4).
tests/host/binpack_shim.cpp runs the fill's per-item bodies as plain loops under the engine's own driver
(csrc/yk_lattice_host.hpp).  Bindings, ask states and node availability must equal the oracle's; the shim also checks after
every fill that the node order is exactly "ascending by (current key, rank)"."""
import copy
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from test_engine_host import run_engine_host
from test_gpu_dims import _inf_nodes, widen

HERE = os.path.dirname(os.path.abspath(__file__))
BP = synth.POLICY_BINPACKING
INELIGIBLE = 100
# binpack_shim.cpp's counters (the layout of lattice_shim.cpp's)
STATS = ("subruns", "fullscans", "sorts", "elems", "quick", "escalations", "handoffs", "batches", "uniform_attempts",
         "uniform_retries", "uniform_asks", "uniform_runs", "uniform_elements")


@pytest.fixture(scope="module")
def bshim(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("binpack") / "binpack_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-fPIC", "-shared", "-w", "-o", out,
                           os.path.join(HERE, "host", "binpack_shim.cpp")])
    return C.CDLL(out)


def run(bshim, s, stats=None, **kw):
    rows = []
    r = run_engine_host(bshim, s, fn="binpack_host_run", rows=rows, **kw)
    if stats is not None:
        stats.append(dict(zip(STATS, rows[0])))
    return r


def check(bshim, oracle, s, tag=None, stats=None, **kw):
    """-> the oracle's result when the shim equals it, None when the snapshot is not eligible"""
    want = oracle.run(s, max_bindings=kw.get("max_bindings") or -1)
    rc, ask, node, state, avail = run(bshim, s, stats=stats, **kw)
    if rc == INELIGIBLE:
        return None
    assert rc == 0, (tag, rc)
    assert np.array_equal(ask, want["ask"]), tag
    assert np.array_equal(node, want["node"]), tag
    if kw.get("max_bindings") is None:
        assert np.array_equal(state, want["state"]), tag
    assert np.array_equal(avail, want["avail"]), tag
    return want


def bp(s):
    s = copy.deepcopy(s)
    s.policy = BP
    return s


def bcheck(bshim, oracle, s, tag=None, eligible=True, **kw):
    """-> (oracle result, shim counters); None when the snapshot is not eligible (only allowed with eligible=False)"""
    st = []
    want = check(bshim, oracle, s, tag=tag, stats=st, **kw)
    if want is None:
        assert not eligible, ("not eligible", tag)
        return None, None
    c = st[0]
    # never a retry; a fill that stands is one uniform run, one that falls back hands the cycle to the host commit
    assert c["uniform_retries"] == 0, (tag, c)
    assert c["uniform_runs"] + c["handoffs"] >= c["uniform_attempts"] >= c["uniform_runs"], (tag, c)
    return want, c


# ---- fixtures shared with tests/test_binpack_device.py ----
def config_shapes(seed):
    """small config-2 / config-3 / config-4 (with a quota) / gang snapshots whose asks come in runs, under binpacking"""
    k = seed % 4
    if k == 0:
        s = synth.perf(60, 6, 30, policy=BP, seed=seed)
    elif k == 1:
        s = synth.perf(60, 6, 30, masks=True, policy=BP, seed=seed)
    elif k == 2:
        s = synth.hier(40, 2, 2, 2, 20, policy=BP, seed=seed)
        assert (s.q_max >= 0).any()
    else:
        s = synth.gangs(40, 15, 4, seed=seed, policy=BP, fill=(0.5, 1.05, 2.0)[seed % 3])
    return synth.runny(s, seed)


def shuffled_ranks(n_nodes, apps, tasks, seed):
    """identical nodes whose NodeIDs sort in a shuffled order: every key ties, the rank decides"""
    s = synth.reference_shape(n_nodes, apps, tasks, policy=BP)
    perm = np.random.default_rng(seed).permutation(n_nodes)
    s.node_id = [f"kwok-node-{int(i):05d}" for i in perm]
    return s


def mid_node(n_nodes=7, tasks=250):
    """110 pods per node: the run's capacity ends 30 pods into its third node"""
    return synth.reference_shape(n_nodes, 1, tasks, policy=BP)


def overcommitted(sensitive):
    """900 identical pods, room for 660; with a max on the queue (never reached) the order is placement-sensitive and the
    batch stops at the first ask that finds no node"""
    s = synth.reference_shape(6, 3, 300, policy=BP)
    s.node_total[:, 2] = s.node_avail[:, 2] = 110
    if sensitive:
        s.q_max[-1, 0] = 1 << 60
    return s


def mixed_signature_gangs(seed):
    """one request per gang, but the last member of every gang tolerates one more taint: plan_segments cuts inside every
    gang, so the stretch goes to the host commit"""
    s = synth.gangs(60, 20, 4, seed=seed, policy=BP, fill=0.5)
    s.ask_req[:] = s.ask_req[0]
    for g in np.unique(s.ask_gang[s.ask_gang >= 0]):
        s.ask_tol[np.nonzero(s.ask_gang == g)[0][-1]] |= np.uint64(1 << 40)
    return s


def infinite_shares(D):
    """+Inf (node 3), -Inf (node 7) and skipped 0/0 (node 11) vcore shares; under binpacking the +Inf node sorts first"""
    s = bp(_inf_nodes(widen(synth.reference_shape(12, 12, 125), D, 1)))
    s.ask_req[:, 0] = 0
    return s


# ---- fuzz ----
@pytest.mark.parametrize("batch", [7, 64, 1024])
def test_fill_matches_oracle_on_config_shapes(bshim, oracle, batch):
    checked = fills = 0
    for seed in range(100):
        s = config_shapes(seed)
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > batch:
            continue
        want, c = bcheck(bshim, oracle, s, tag=(s.name, seed, batch), eligible=(seed % 4 != 3), batch=batch)
        if want is not None:   # (runny can give two gangs of one application different requests: not eligible)
            checked += 1
            fills += c["uniform_attempts"]
    assert checked >= 80 and fills > 1000


@pytest.mark.parametrize("batch", [7, 64, 1024])
def test_fill_matches_oracle_on_fuzz(bshim, oracle, batch):
    checked = asks = 0
    for seed in range(120):
        s = bp(synth.runny(synth.fuzz(seed), seed))
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > batch:
            continue
        try:
            oracle.run(s)
        except RuntimeError:   # a NaN score: the engine reports it (test_binpack_device)
            continue
        want, c = bcheck(bshim, oracle, s, tag=(seed, batch), eligible=False, batch=batch)
        if want is not None:
            checked += 1
            asks += c["uniform_asks"]
    assert checked > 20 and asks > 200


@pytest.mark.parametrize("D", range(1, 9))
def test_every_dimension_count(bshim, oracle, D):
    for seed in range(10):
        s = bp(synth.redim(synth.runny(synth.fuzz(seed), seed), D, seed))
        try:
            oracle.run(s)
        except RuntimeError:
            continue
        bcheck(bshim, oracle, s, tag=(seed, D), eligible=False, batch=64)
    want, c = bcheck(bshim, oracle, bp(widen(synth.runny(synth.perf(200, 8, 40, masks=True), D), D, D)), batch=512)
    assert c["uniform_asks"] > 0


@pytest.mark.parametrize("w", [[0, 0, 0, 0], [0, 1, 0, 0], [1, 0.5, 0, 0], [1e-3, 1e3, 0, 0], [1, 1, 1, 0], [0.1, 0.2, 0.3, 0.7]],
                         ids=["zero", "tw1_second", "tw1.5", "wide", "pods", "tenths"])
def test_configured_weights(bshim, oracle, w):
    for s in (synth.runny(synth.perf(300, 10, 60, masks=True, policy=BP, seed=3), 3), synth.kwok(200, 10, 50, variant="bare", policy=BP)):
        want, c = bcheck(bshim, oracle, synth.reweigh(s, w), tag=(s.name, w), batch=4096)
        assert c["uniform_asks"] > 0


@pytest.mark.parametrize("D", [2, 4, 8])
def test_infinite_shares(bshim, oracle, D):
    s = infinite_shares(D)
    want, c = bcheck(bshim, oracle, s, batch=1 << 20)
    assert c["uniform_asks"] == s.n_asks and c["uniform_attempts"] == 1
    assert want["node"][0] == 3   # +Inf usage share: binpacking score -Inf, first in the order


# ---- targeted cases ----
def test_flat_requests_fill_by_rank(bshim, oracle):
    """{pods: 1} moves no key: the nodes fill one after the other in rank order"""
    for nodes, apps, tasks in ((20, 4, 100), (50, 2, 100)):
        s = synth.kwok(nodes, apps, tasks, variant="bare", policy=BP)
        want, c = bcheck(bshim, oracle, s, batch=1 << 20)
        assert c["uniform_asks"] == s.n_asks and c["uniform_attempts"] == 1


@pytest.mark.parametrize("seed", range(4))
def test_identical_nodes_shuffled_ranks(bshim, oracle, seed):
    s = shuffled_ranks(40, 4, 125, seed)
    want, c = bcheck(bshim, oracle, s, batch=1 << 20)
    assert c["uniform_asks"] == s.n_asks == len(want["ask"]) and c["uniform_attempts"] == 1
    rank = s.node_rank()
    # every node takes its 110 pods in rank order (the run's keys fall as the node fills: it stays first)
    assert rank[want["node"][0]] == 0 and (np.diff(rank[want["node"]].astype(np.int64)) >= 0).all()


def test_capacity_ends_mid_node(bshim, oracle):
    s = mid_node()
    want, c = bcheck(bshim, oracle, s, batch=1 << 20)
    assert np.bincount(want["node"], minlength=s.n_nodes).tolist() == [110, 110, 30, 0, 0, 0, 0]
    assert c["uniform_asks"] == 250 and c["uniform_attempts"] == 1


@pytest.mark.parametrize("sensitive", [False, True])
def test_overcommitted_cluster(bshim, oracle, sensitive):
    s = overcommitted(sensitive)
    want, c = bcheck(bshim, oracle, s, batch=1 << 20)
    assert len(want["ask"]) == 660 and (want["state"] == 2).sum() == 240 and c["handoffs"] == 0 and c["uniform_asks"] == 900
    # insensitive: one fill decides all 900 asks; sensitive: a batch stops after its first NOFIT, the next one starts after it
    assert (c["uniform_attempts"] > 1) == sensitive


def test_gangs_whole_and_handed_off(bshim, oracle):
    whole = handed = 0
    for seed in range(6):
        for fill in (0.5, 1.05, 2.0):
            s = synth.gangs(60, 30, 5, seed=seed, fill=fill, policy=BP)
            s.ask_req[:] = s.ask_req[0]
            want, c = bcheck(bshim, oracle, s, tag=(seed, fill), batch=1000)
            assert c["uniform_attempts"] > 0
            whole += c["handoffs"] == 0 and c["uniform_asks"] == s.n_asks
            handed += c["handoffs"]
    assert whole > 0 and handed > 0
    for seed in range(3):   # a gang whose members differ in signature: the stretch is cut inside it and handed off
        want, c = bcheck(bshim, oracle, mixed_signature_gangs(seed), tag=seed, batch=1000)
        assert c["handoffs"] == 1 and c["uniform_asks"] == 0


def test_max_bindings(bshim, oracle):
    cut = 0
    for seed in (1, 4, 9, 12, 30, 41):
        s = config_shapes(seed)
        k = max(1, len(oracle.run(s)["ask"]) // 2)
        want = oracle.run(s, max_bindings=k)
        rc, ask, node, _, avail = run(bshim, s, batch=64, max_bindings=k)
        assert rc == 0, seed
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"]) and np.array_equal(avail, want["avail"])
        cut += len(ask) == k
    assert cut >= 4


def test_capacity_sum_is_clamped_and_64_bit(bshim, oracle):
    """a node's capacity for the run counts at most R: four nodes of 2^62 units would overflow even a 64-bit sum; 65 536
    nodes x 65 536 asks sum to 2^32, which a 32-bit scan wraps to 0"""
    s = synth.reference_shape(4, 1, 10, policy=BP)
    s.node_total[:, 0] = s.node_avail[:, 0] = 1 << 62
    s.ask_req[:] = [1, 0, 0, 0]
    want, c = bcheck(bshim, oracle, s, batch=1 << 20)
    assert len(want["ask"]) == 10 and c["uniform_asks"] == 10
    s = synth.reference_shape(1 << 16, 1, 1 << 16, policy=BP)
    s.node_total[:, 0] = s.node_avail[:, 0] = 1 << 40
    s.ask_req[:] = [1, 0, 0, 0]
    rc, ask, node, state, avail = run(bshim, s, batch=1 << 20)
    assert rc == 0 and len(ask) == s.n_asks and (state == 1).all()
    assert (node == np.argmin(s.node_rank())).all()   # one unit of 2^40 at a time: the first node keeps the lowest key
