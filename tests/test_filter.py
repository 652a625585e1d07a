"""yk_filter_nodes: every present node's first failing step for a list of asks, in the cycle's node order, on the device.

The expectation never comes from the engine: the order is the present nodes sorted by (oracle node score on the engine's
current availability, NodeID rank, index), and the slot of a pair is the oracle's predicate (reservation phase: its
reservation predicate), or 10 for a reserved node.  Every GPU test also checks that the engine launched kernels for it.
The CPU test at the end checks the expectation helper against the oracle's own scheduling run."""
import copy
import ctypes as C

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from test_gpu_dims import WEIGHT_CASES, infinite, nan_node, weighted, widen

YK_NONE = 0xFFFFFFFF
SLOTS, RESERVED, ABSENT = 11, 10, 9
YK_ERR_ARG, YK_ERR_RANGE = -1, -5


# ---- the expectation, from the oracle ----
def oracle_order(oracle, s, avail, present):
    """present nodes in ascending (oracle score on `avail`, NodeID rank, index)"""
    rank = s.node_rank()
    key = [(oracle.node_score(s.policy, s.weights, s.node_total[n], avail[n]), int(rank[n]), int(n)) for n in present]
    return [k[2] for k in sorted(key)]


def expect(oracle, s, asks, allocate=True, avail=None, present_nodes=None, present_asks=None):
    """-> (full list of passing nodes per ask, counts[n][11]) for snapshot `s` with the engine's availability `avail`"""
    avail = s.node_avail if avail is None else np.asarray(avail)
    present_nodes = np.arange(s.n_nodes) if present_nodes is None else present_nodes
    present_asks = set(range(s.n_asks) if present_asks is None else np.asarray(present_asks).tolist())
    t = copy.deepcopy(s)
    t.node_avail = np.ascontiguousarray(avail, dtype=np.int64)
    order = oracle_order(oracle, t, t.node_avail, present_nodes)
    st, keep = oracle._pack(t)
    fn = oracle.lib().yko_predicate if allocate else oracle.lib().yko_predicate_reserve
    fn.restype = C.c_int
    memo = {}                                  # asks with equal predicate inputs get equal answers
    lists, counts = [], np.zeros((len(asks), SLOTS), dtype=np.uint32)
    for i, a in enumerate(asks):
        a = int(a)
        if a not in present_asks:
            lists.append([])
            counts[i, ABSENT] = len(order)
            continue
        sig = (t.ask_req[a].tobytes(), int(t.ask_tol[a]), int(t.ask_need[a]), int(t.ask_deny[a]), int(t.ask_node[a]))
        if sig not in memo:
            slots = [RESERVED if t.node_flags[n] & synth.NODE_RESERVED else fn(C.byref(st), C.c_int32(a), C.c_int32(n))
                     for n in order]
            memo[sig] = ([n for n, x in zip(order, slots) if x == 0], np.bincount(slots, minlength=SLOTS))
        lists.append(memo[sig][0])
        counts[i] = memo[sig][1]
    return lists, counts


def window(full, skip, k):
    w = full[skip:skip + k]
    return w + [YK_NONE] * (k - len(w))


# ---- the GPU side ----
def _engine():
    from yunikorn_k8shim_b200 import Engine
    return Engine


def _check(e, oracle, s, asks=None, k=None, skip=0, phases=(True, False), **kw):
    asks = np.arange(s.n_asks) if asks is None else np.asarray(asks)
    k = s.n_nodes if k is None else k
    for allocate in phases:
        before = e.stats()["other_launches"]
        nodes, n_pass, counts = e.filter_nodes(asks, k=k, skip=skip, allocate=allocate)
        assert e.stats()["other_launches"] > before
        full, want_counts = expect(oracle, s, asks, allocate, **kw)
        assert np.array_equal(counts, want_counts), (s.name, allocate)
        assert n_pass.tolist() == [len(f) for f in full], (s.name, allocate)
        assert np.array_equal(n_pass, counts[:, 0])
        for i in range(len(asks)):
            assert nodes[i].tolist() == window(full[i], skip, k), (s.name, allocate, int(asks[i]))
    return full


def _nan_free(oracle, s):
    return not any(np.isnan(oracle.node_score(s.policy, s.weights, s.node_total[n], s.node_avail[n])) for n in range(s.n_nodes))


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(12))
def test_fuzz_snapshots(oracle, seed):
    """reserved and unschedulable nodes, slow-path asks, pod.Spec.NodeName, zero and negative requests, either policy"""
    s = synth.fuzz(seed)
    s.ask_req[::11, 1] = -5                                    # a negative request: step 3 in both phases
    with _engine().for_snapshot(s) as e:
        full = _check(e, oracle, s)
    assert any(full)


@pytest.mark.gpu
def test_masks_2000_nodes(oracle):
    s = synth.perf(2000, 6, 25, masks=True, seed=5)
    s.node_flags[::97] |= synth.NODE_RESERVED
    s.node_flags[5::89] = 0
    with _engine().for_snapshot(s) as e:
        full = _check(e, oracle, s)
    assert min(len(f) for f in full) > 0 and max(len(f) for f in full) < s.n_nodes


@pytest.mark.gpu
def test_binpacking(oracle):
    for s in (synth.binpacking_e2e(), synth.perf(700, 6, 20, masks=True, policy=synth.POLICY_BINPACKING, seed=8)):
        assert s.policy == synth.POLICY_BINPACKING
        with _engine().for_snapshot(s) as e:
            _check(e, oracle, s)


@pytest.mark.gpu
@pytest.mark.parametrize("D", range(1, 9))
def test_every_dimension_count(oracle, D):
    ran = 0
    for seed in range(4):
        s = synth.redim(synth.fuzz(seed), D, seed)
        if not _nan_free(oracle, s):
            continue
        with _engine().for_snapshot(s) as e:
            _check(e, oracle, s)
        ran += 1
    s = widen(synth.perf(600, 4, 20, masks=True, seed=D), D, D)   # over two node tiles
    with _engine().for_snapshot(s) as e:
        _check(e, oracle, s)
    assert ran >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("case", WEIGHT_CASES)
def test_configured_weights(oracle, case):
    s = weighted(case)
    with _engine().for_snapshot(s) as e:
        _check(e, oracle, s, asks=np.arange(0, s.n_asks, 3))


@pytest.mark.gpu
@pytest.mark.parametrize("D", [4, 8])
def test_infinite_shares(oracle, D):
    s = infinite(D)
    with _engine().for_snapshot(s) as e:
        full = _check(e, oracle, s)
    assert any(3 in f for f in full) and any(7 in f for f in full)


@pytest.mark.gpu
def test_paging(oracle):
    """windows of every size and start, also across node tiles (256 positions) and past the end; pages concatenate"""
    s = synth.perf(1100, 4, 10, masks=True, seed=17)
    asks = np.arange(s.n_asks)
    full, _ = expect(oracle, s, asks)
    npass = np.array([len(f) for f in full])
    assert npass.max() > 300                                    # long lists span several tiles
    mid = int(np.median(npass))
    with _engine().for_snapshot(s) as e:
        for k in (0, 1, 33, s.n_nodes):
            for skip in sorted({0, 31, 32, 255, 256, max(mid - 1, 0), mid, int(npass.max()) - 1, int(npass.max()), s.n_nodes + 7}):
                before = e.stats()["other_launches"]
                nodes, n_pass, counts = e.filter_nodes(asks, k=k, skip=skip)
                assert e.stats()["other_launches"] > before
                assert nodes.shape == (len(asks), k) and n_pass.tolist() == npass.tolist()
                for i in range(len(asks)):
                    assert nodes[i].tolist() == window(full[i], skip, k), (k, skip, i)
        pages = [e.filter_nodes(asks, k=64, skip=p)[0] for p in range(0, s.n_nodes, 64)]
        cat = np.concatenate(pages, axis=1)
        for i in range(len(asks)):
            assert cat[i].tolist() == window(full[i], 0, cat.shape[1])


@pytest.mark.gpu
def test_more_asks_than_one_chunk(oracle):
    """5 000 asks x 10 000 nodes in one call: the engine works in chunks of 4 096 asks"""
    s = synth.perf(10_000, 40, 125, seed=21)
    s.node_avail[::3, 0] = 500                                  # a third of the nodes fit only the smallest class
    asks = np.arange(s.n_asks)[::-1].copy()
    with _engine().for_snapshot(s) as e:
        full = _check(e, oracle, s, asks=asks, k=64, skip=100, phases=(True,))
        st = e.stats()
    assert len({len(f) for f in full}) > 1
    assert st["other_launches"] >= 11 + 4                        # order, then two chunks of filter + compaction


@pytest.mark.gpu
def test_after_cycles_and_removals(oracle):
    s = synth.fuzz(3, n_nodes=300, n_asks=400)
    rng = np.random.default_rng(1)
    with _engine().for_snapshot(s, batch=64) as e:
        ask, node, _ = e.cycle(s.n_asks)
        assert len(ask) > 0
        gone_n = np.sort(rng.choice(s.n_nodes, 40, replace=False))
        unbound = np.nonzero(e.ask_states(np.arange(s.n_asks)) != 1)[0]
        gone_a = np.sort(rng.choice(unbound, min(60, len(unbound) // 2), replace=False))   # bound asks are released instead
        e.release(ask[::3])                                    # gives the resources back and forgets the ask
        e.nodes_remove(gone_n)
        e.asks_remove(gone_a)
        avail = e.nodes_available(np.arange(s.n_nodes))
        assert not np.array_equal(avail, s.node_avail)
        keep_n = np.setdiff1d(np.arange(s.n_nodes), gone_n)
        keep_a = np.setdiff1d(np.arange(s.n_asks), np.concatenate([gone_a, ask[::3]]))
        _check(e, oracle, s, avail=avail, present_nodes=keep_n, present_asks=keep_a)
        nodes, n_pass, counts = e.filter_nodes(gone_a[:3], k=4)
        assert (nodes == YK_NONE).all() and (n_pass == 0).all() and (counts[:, ABSENT] == len(keep_n)).all()


def _sequence(s, commit, filter_first):
    from yunikorn_k8shim_b200 import Engine
    out = []
    with Engine.for_snapshot(s, batch=32, commit=commit) as e:
        launches = 0
        for step in range(4):
            if filter_first:
                before = e.stats()["other_launches"]
                e.filter_nodes(np.arange(s.n_asks), k=8, skip=step)
                e.filter_nodes(np.arange(0, s.n_asks, 2), allocate=False)
                launches += e.stats()["other_launches"] - before
            ask, node, _ = e.cycle(40)
            out.append((ask, node, e.ask_states(np.arange(s.n_asks)), e.nodes_available(np.arange(s.n_nodes))))
            if step == 1:
                e.release(ask[::2])
    return out, launches


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_no_interference_with_cycles(commit):
    for s in (synth.perf(300, 10, 20, masks=True, seed=12), synth.fuzz(4, n_nodes=200, n_asks=300)):
        plain, _ = _sequence(s, commit, False)
        filtered, launches = _sequence(s, commit, True)
        assert launches > 0
        for a, b in zip(plain, filtered):
            for x, y in zip(a, b):
                assert np.array_equal(x, y), (s.name, commit)


def single_ask(s, a):
    """the same snapshot with only ask `a` pending (every other ask is a slow-path ask, never bound) and no reserved node"""
    t = copy.deepcopy(s)
    t.node_flags &= ~np.uint32(synth.NODE_RESERVED)
    t.ask_flags[:] = 1
    t.ask_flags[a] = 0
    t.ask_gang[:] = -1
    return t


def _single_cases(oracle, seeds):
    for seed in seeds:
        s = synth.fuzz(seed)
        rng = np.random.default_rng(seed)
        for a in rng.choice(s.n_asks, min(4, s.n_asks), replace=False):
            t = single_ask(s, int(a))
            if not _nan_free(oracle, t):
                continue
            yield t, int(a), oracle.run(t)


@pytest.mark.gpu
def test_first_candidate_is_the_cycles_binding(oracle):
    bound = 0
    for t, a, want in _single_cases(oracle, range(10)):
        with _engine().for_snapshot(t) as e:
            before = e.stats()["other_launches"]
            nodes, n_pass, _ = e.filter_nodes([a], k=1)
            assert e.stats()["other_launches"] > before
            ask, node, _ = e.cycle(t.n_asks)
        if len(ask):
            assert ask.tolist() == [a] and nodes[0, 0] == node[0], (t.name, a)
            bound += 1
        elif want["state"][a] == 2:                            # no node fits
            assert n_pass[0] == 0 and nodes[0, 0] == YK_NONE
    assert bound >= 10


@pytest.mark.gpu
def test_errors(oracle):
    from yunikorn_k8shim_b200 import YkError
    s = nan_node()
    with _engine().for_snapshot(s) as e:
        nodes = np.full((3, 5), 7, dtype=np.uint32)
        n_pass = np.full(3, 7, dtype=np.uint32)
        counts = np.full((3, SLOTS), 7, dtype=np.uint32)
        asks = np.array([0, 1, 2], dtype=np.uint32)
        lib, h = e._lib, e._h
        p = lambda x: x.ctypes.data_as(C.c_void_p)            # noqa: E731
        before = e.stats()["other_launches"]
        rc = lib.yk_filter_nodes(h, 3, p(asks), 1, 0, 5, p(nodes), p(n_pass), p(counts))
        assert rc == YK_ERR_RANGE
        assert (nodes == 7).all() and (n_pass == 7).all() and (counts == 7).all()   # nothing written
        assert e.stats()["other_launches"] > before
        assert lib.yk_filter_nodes(h, 1, p(np.array([s.n_asks], dtype=np.uint32)), 1, 0, 0, None, None, None) == YK_ERR_ARG
        assert lib.yk_filter_nodes(h, 1, p(asks), 1, 0, 2, None, None, None) == YK_ERR_ARG
        assert lib.yk_filter_nodes(h, 1, None, 1, 0, 0, None, None, None) == YK_ERR_ARG
        assert lib.yk_filter_nodes(h, 0, None, 1, 0, 0, None, None, None) == 0
        with pytest.raises(YkError) as ei:
            e.filter_nodes([0])
        assert ei.value.code == YK_ERR_RANGE
        assert (e.ask_states(np.arange(s.n_asks)) == 0).all()


# ---- on the CPU ----
def test_expectation_helper_matches_oracle_run(oracle):
    """the helper's first candidate (oracle order + oracle predicate) is the node the oracle's own cycle binds"""
    bound = 0
    for t, a, want in _single_cases(oracle, range(10)):
        full, counts = expect(oracle, t, [a])
        assert counts.sum() == t.n_nodes
        if len(want["ask"]):
            assert want["ask"].tolist() == [a] and full[0][0] == want["node"][0], (t.name, a)
            bound += 1
        elif want["state"][a] == 2:
            assert full[0] == []
    assert bound >= 10
