"""yk_preemption_nodes: for a list of asks and one victim list each, every node those victims can free, in the cycle's node
order, on the device.

The expectation never comes from the engine.  Where each victim is bound and what every node has available come from the
oracle's own cycle (oracle_ctypes.run); the node order is test_filter.oracle_order; the answer of a (preemptor, node) pair
is oracle_ctypes' preemption index with start 0 over the list's victims bound to that node, in list order.  The CPU test at
the end checks the expectation helper against the reference's known answers (TestPreemptionPredicates)."""
import copy
import ctypes as C
import json
import os

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from test_filter import _nan_free, oracle_order, window
from test_gpu_dims import WEIGHT_CASES, infinite, nan_node, weighted, widen

YK_NONE = 0xFFFFFFFF
YK_ERR_ARG, YK_ERR_STATE, YK_ERR_RANGE = -1, -4, -5
ST_ALLOCATED, ST_NOFIT = 1, 2
CHUNK_ROWS, CHUNK_ENTRIES = 4096, 1 << 18        # a chunk of whole lists: at most this many lists / entries
GOLD = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "preemption_predicates.json")))


# ---- the expectation, from the oracle ----
def expect(oracle, t, bound, asks, lists, present_nodes=None, present_asks=None):
    """t: the snapshot as the engine holds it now (availability after the cycle, preemptors included); bound: {victim: node}.
    -> per ask, [(node, victims on it in list order, oracle answer)] for every present node holding one of its victims, in
    the cycle's node order"""
    present_nodes = np.arange(t.n_nodes) if present_nodes is None else present_nodes
    order = oracle_order(oracle, t, t.node_avail, present_nodes)
    pos = {n: i for i, n in enumerate(order)}
    st, keep = oracle._pack(t)
    fn = oracle.lib().yko_preemption_index
    fn.restype = C.c_int
    out = []
    for a, lst in zip(asks, lists):
        a = int(a)
        if present_asks is not None and a not in present_asks:
            out.append([])
            continue
        groups = {}
        for v in lst:
            n = bound.get(int(v))
            if n in pos:
                groups.setdefault(n, []).append(int(v))
        pairs = []
        for n in sorted(groups, key=pos.__getitem__):
            req = np.ascontiguousarray(t.ask_req[groups[n]], dtype=np.int64)
            ans = fn(C.byref(st), C.c_int32(a), C.c_int32(n), C.c_int32(len(req)), req.ctypes.data_as(C.c_void_p), C.c_int32(0))
            pairs.append((n, groups[n], ans))
        out.append(pairs)
    return out


def fits(pairs):
    return [(n, ans + 1) for n, _, ans in pairs if ans >= 0]


def best(pairs):
    f = fits(pairs)
    return min(f, key=lambda x: x[1]) if f else (YK_NONE, 0)     # min keeps the first of equal counts: the earlier node


def add_asks(e, t, req):
    """upsert new pending asks (application 0, tolerating every taint) behind the snapshot's, in the engine and in the
    expectation"""
    req = np.asarray(req, dtype=np.int64).reshape(-1, t.D)
    m, a0 = len(req), t.n_asks
    idx = np.arange(a0, a0 + m)
    create = np.arange(m, dtype=np.int64) + 10 ** 9
    tol = np.full(m, ~np.uint64(0), dtype=np.uint64)
    e.asks_upsert(idx, req, np.zeros(m, np.int32), create, tolerated_bits=tol)
    t.ask_req = np.vstack([t.ask_req, req])
    t.ask_tol = np.concatenate([t.ask_tol, tol])
    for f, v in (("ask_app", 0), ("ask_need", 0), ("ask_deny", 0), ("ask_prio", 0), ("ask_node", -1),
                 ("ask_flags", 0), ("ask_gang", -1)):
        x = getattr(t, f)
        setattr(t, f, np.concatenate([x, np.full(m, v, dtype=x.dtype)]))
    t.ask_create = np.concatenate([t.ask_create, create])
    return idx


# ---- the GPU side ----
def _engine_cls():
    from yunikorn_k8shim_b200 import Engine
    return Engine


def scenario(oracle, s, commit="auto", extra=4, batch=0):
    """one cycle on the engine and on the oracle (same bindings) -> (engine, t = the engine's state for the oracle, bound,
    oracle result)"""
    want = oracle.run(s)
    Engine = _engine_cls()
    e = Engine(D=s.D, policy=s.policy, weights=s.weights, max_nodes=s.n_nodes, max_asks=s.n_asks + extra,
               max_apps=max(s.n_apps, 1), max_queues=max(s.n_queues, 1), batch=batch, commit=commit)
    e.load_snapshot(s)
    ask, node, _ = e.cycle(s.n_asks)
    assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"]), (s.name, commit)
    t = copy.deepcopy(s)
    t.node_avail = np.ascontiguousarray(want["avail"], dtype=np.int64)
    bound = {int(a): int(n) for a, n in zip(want["ask"], want["node"])}
    return e, t, bound, want


def random_lists(rng, alloc, n, many=None):
    """n victim lists: random subsets of the allocated asks in random order, with 0, 1 and many entries"""
    lists = []
    for i in range(n):
        size = (0, 1, int(rng.integers(2, max(len(alloc), 2) + 1)) if many is None else many)[i % 3] if len(alloc) else 0
        lists.append(rng.permutation(alloc)[:size].astype(np.uint32))
    return lists


def preemptors(e, t, want, rng, n_new=3):
    """NOFIT asks, allocated asks and newly upserted asks larger than what any node has left"""
    nofit = np.nonzero(want["state"] == ST_NOFIT)[0]
    alloc = np.asarray(want["ask"])
    big = np.zeros((n_new, t.D), dtype=np.int64)
    big[:, :min(t.D, 2)] = (t.node_total[:, :min(t.D, 2)].max(axis=0) * rng.uniform(0.3, 0.8, (n_new, 1))).astype(np.int64)
    if t.D > 2:
        big[:, 2] = 1
    new = add_asks(e, t, big) if n_new else np.zeros(0, np.int64)
    return np.concatenate([rng.permutation(nofit)[:6], rng.permutation(alloc)[:4], new]).astype(np.uint32)


def check(e, t, want_pairs, asks, lists, k=None, skip=0):
    k = t.n_nodes if k is None else k
    before = e.stats()["other_launches"]
    nodes, need, n_fit, bn, bneed = e.preemption_nodes(asks, lists, k=k, skip=skip)
    assert e.stats()["other_launches"] > before
    assert nodes.shape == (len(asks), k) and need.shape == (len(asks), k)
    for i in range(len(asks)):
        f = fits(want_pairs[i])
        assert n_fit[i] == len(f), (t.name, i)
        assert nodes[i].tolist() == window([n for n, _ in f], skip, k), (t.name, i)
        w = f[skip:skip + k]
        assert need[i].tolist() == [c for _, c in w] + [0] * (k - len(w)), (t.name, i)
        assert (int(bn[i]), int(bneed[i])) == best(want_pairs[i]), (t.name, i)
    return nodes, need, n_fit


def run_case(oracle, s, commit, seed, many=None, n_new=3, search_check=True):
    rng = np.random.default_rng(seed)
    e, t, bound, want = scenario(oracle, s, commit, extra=n_new)
    with e:
        asks = preemptors(e, t, want, rng, n_new)
        lists = random_lists(rng, np.asarray(want["ask"]), len(asks), many)
        pairs = expect(oracle, t, bound, asks, lists)
        check(e, t, pairs, asks, lists)
        if search_check:   # every pair: the single-query search through the C ABI gives the same answer
            q = [(int(a), n, t.ask_req[vs]) for a, p in zip(asks, pairs) for n, vs, _ in p]
            if q:
                got = e.preemption_search([x[0] for x in q], [x[1] for x in q], [x[2] for x in q], [0] * len(q))
                assert got.tolist() == [ans for p in pairs for _, _, ans in p], s.name
    return pairs, lists


def _fuzz(seed):
    s = synth.fuzz(seed, n_asks=250 + 7 * seed)
    s.node_avail[:, :2] = s.node_avail[:, :2] * 2 // 3          # nearly full after the cycle: victims are needed
    return s


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(20))
def test_fuzz(oracle, seed):
    """masked snapshots with reserved, unschedulable and over-committed nodes, gangs, slow-path asks, either policy"""
    pairs, lists = run_case(oracle, _fuzz(seed), ("host", "device", "auto")[seed % 3], seed)
    assert any(len(x) == 0 for x in lists) and any(len(x) == 1 for x in lists) and any(len(x) > 1 for x in lists)


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_deep_and_wide_lists(oracle, commit):
    """over 32 victims of one list on one node (the search's warp step) and one list over more than 256 nodes"""
    deep = synth.kwok(3, 2, 150)
    deep.ask_req[:, 0] = 250                                     # 100 pods of 250 mCPU per node: 7 CPU left after the cycle
    pairs, _ = run_case(oracle, deep, commit, 1, many=10 ** 6, n_new=3)
    assert max(len(vs) for p in pairs for _, vs, _ in p) > 32
    assert any(ans >= 32 for p in pairs for _, _, ans in p)
    wide = synth.perf(600, 12, 50, masks=True, seed=4)
    wide.node_avail[:, :2] //= 8
    pairs, _ = run_case(oracle, wide, commit, 2, many=10 ** 6, n_new=3)
    assert max(len(p) for p in pairs) > 256
    assert max(len(fits(p)) for p in pairs) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("D", range(1, 9))
def test_every_dimension_count(oracle, D):
    ran = 0
    for seed in range(3):
        s = synth.redim(_fuzz(seed), D, seed)
        if not _nan_free(oracle, s):
            continue
        run_case(oracle, s, "auto", seed)
        ran += 1
    s = widen(synth.perf(400, 8, 40, masks=True, seed=D), D, D)
    s.node_avail[:, :min(D, 2)] //= 6
    run_case(oracle, s, "auto", D)
    assert ran >= 1


@pytest.mark.gpu
def test_binpacking(oracle):
    for i, s in enumerate((synth.binpacking_e2e(), synth.perf(500, 8, 40, masks=True, policy=synth.POLICY_BINPACKING, seed=8))):
        assert s.policy == synth.POLICY_BINPACKING
        run_case(oracle, s, "auto", i)


@pytest.mark.gpu
@pytest.mark.parametrize("case", WEIGHT_CASES)
def test_configured_weights(oracle, case):
    run_case(oracle, weighted(case), "auto", 3)


@pytest.mark.gpu
@pytest.mark.parametrize("D", [4, 8])
def test_infinite_shares(oracle, D):
    """nodes 3 (+Inf share) and 7 (-Inf) sort last and first: their victims' nodes come in that order"""
    pairs, _ = run_case(oracle, infinite(D), "auto", D, many=10 ** 6)
    assert any(n in (3, 7) for p in pairs for n, _, _ in p)


@pytest.mark.gpu
def test_node_changes_between_cycles(oracle):
    """after a cycle: a removed node still holding allocations (its entries are ignored), nodes re-upserted with new totals,
    cordoned (unschedulable: no fit) and reserved (not consulted); then a cycle with no binding left, and the same answers"""
    s = synth.perf(300, 10, 30, masks=True, seed=9)
    s.node_avail[:, :2] //= 4
    rng = np.random.default_rng(9)
    e, t, bound, want = scenario(oracle, s, "auto", extra=3)
    with e:
        asks = preemptors(e, t, want, rng)
        holding = np.unique(want["node"])
        pick = rng.permutation(holding)
        gone, cordon, reserve, resize = pick[:5], pick[5:10], pick[10:15], pick[15:25]
        e.nodes_remove(gone)
        t.node_flags[cordon] = 0
        t.node_flags[reserve] |= synth.NODE_RESERVED
        t.node_total[resize, 0] += 4000
        t.node_avail[resize, 0] += 4000
        ch = np.concatenate([cordon, reserve, resize])
        e.nodes_upsert(ch, t.node_total[ch], t.node_avail[ch], t.node_taint[ch], t.node_label[ch], s.node_rank()[ch], t.node_flags[ch])
        present = np.setdiff1d(np.arange(s.n_nodes), gone)
        lists = [rng.permutation(want["ask"]).astype(np.uint32) for _ in asks]
        pairs = expect(oracle, t, bound, asks, lists, present_nodes=present)
        check(e, t, pairs, asks, lists)
        assert not any(n in gone for p in pairs for n, _, _ in p)
        on_gone = np.array([a for a, n in bound.items() if n in gone], dtype=np.uint32)   # only victims on removed nodes
        _, _, n_fit, bn, _ = e.preemption_nodes(asks, [rng.permutation(on_gone) for _ in asks])
        assert len(on_gone) > 0 and (n_fit == 0).all() and (bn == YK_NONE).all()
        assert all(ans < 0 for p in pairs for n, _, ans in p if n in cordon)
        assert any(n in reserve for p in pairs for n, _, _ in p)
        ask, _, _ = e.cycle(0)                                   # a cycle that may bind nothing
        assert len(ask) == 0
        check(e, t, pairs, asks, lists)


@pytest.mark.gpu
def test_windows(oracle):
    """windows across the 32-group warp step and past the end, k = 0, and pages that concatenate"""
    s = synth.perf(1100, 12, 50, masks=True, seed=17)
    s.node_avail[:, :2] //= 10
    rng = np.random.default_rng(17)
    e, t, bound, want = scenario(oracle, s, "auto", extra=4)
    with e:
        asks = preemptors(e, t, want, rng, 4)
        lists = [rng.permutation(want["ask"]).astype(np.uint32) for _ in asks]
        pairs = expect(oracle, t, bound, asks, lists)
        nf = np.array([len(fits(p)) for p in pairs])
        assert nf.max() > 300
        mid = int(np.median(nf))
        for k in (0, 1, 33, s.n_nodes):
            for skip in sorted({0, 31, 32, 255, 256, max(mid - 1, 0), mid, int(nf.max()) - 1, int(nf.max()), s.n_nodes + 7}):
                check(e, t, pairs, asks, lists, k=k, skip=skip)
        pages = [e.preemption_nodes(asks, lists, k=64, skip=p) for p in range(0, s.n_nodes, 64)]
        cat_n = np.concatenate([p[0] for p in pages], axis=1)
        cat_c = np.concatenate([p[1] for p in pages], axis=1)
        for i in range(len(asks)):
            f = fits(pairs[i])
            assert cat_n[i].tolist() == window([n for n, _ in f], 0, cat_n.shape[1])
            assert cat_c[i].tolist()[:len(f)] == [c for _, c in f]


def chunks(off):
    """the documented chunk rule: whole lists, at most CHUNK_ROWS lists and CHUNK_ENTRIES entries unless one list is longer"""
    n, c0, out = len(off) - 1, 0, []
    while c0 < n:
        c1 = c0 + 1
        while c1 < n and c1 - c0 < CHUNK_ROWS and off[c1 + 1] - off[c0] <= CHUNK_ENTRIES:
            c1 += 1
        out.append((c0, c1))
        c0 = c1
    return out


@pytest.mark.gpu
def test_more_lists_and_entries_than_one_chunk(oracle):
    """10 000 nodes, 4 200 lists of 20 victims then 800 of 400 (404 000 entries): one chunk ends at the list bound, the next
    at the entry bound; the asks at both sides of every chunk end and a random sample are checked against the oracle"""
    s = synth.perf(10_000, 100, 125, masks=True, seed=2)
    rng = np.random.default_rng(21)
    e, t, bound, want = scenario(oracle, s, "auto", extra=1)
    with e:
        alloc = np.asarray(want["ask"])
        asks = rng.choice(s.n_asks, 5000).astype(np.uint32)
        lists = [rng.choice(alloc, 20 if i < 4200 else 400, replace=False).astype(np.uint32) for i in range(len(asks))]
        off = np.concatenate([[0], np.cumsum([len(x) for x in lists])])
        ch = chunks(off)
        assert ch[0] == (0, CHUNK_ROWS)                                                 # the list bound
        assert off[ch[1][1] + 1] - off[ch[1][0]] > CHUNK_ENTRIES and len(ch) == 3      # the entry bound
        nodes, need, n_fit, bn, bneed = e.preemption_nodes(asks, lists, k=8, skip=1)
        sample = sorted(set([c for c0, c1 in ch for c in (c0, c1 - 1)] + rng.choice(len(asks), 40).tolist()))
        pairs = expect(oracle, t, bound, asks[sample], [lists[i] for i in sample])
        for j, i in enumerate(sample):
            f = fits(pairs[j])
            assert n_fit[i] == len(f) and nodes[i].tolist() == window([n for n, _ in f], 1, 8), i
            assert need[i].tolist() == [c for _, c in f[1:9]] + [0] * (8 - len(f[1:9])), i
            assert (int(bn[i]), int(bneed[i])) == best(pairs[j]), i
        assert len(set(n_fit.tolist())) > 1


def _sequence(s, commit, call):
    Engine = _engine_cls()
    out, launches = [], 0
    with Engine.for_snapshot(s, batch=32, commit=commit) as e:
        for step in range(4):
            if call:
                alloc = np.nonzero(e.ask_states(np.arange(s.n_asks)) == ST_ALLOCATED)[0].astype(np.uint32)
                before = e.stats()["other_launches"]
                asks = np.arange(0, s.n_asks, 7)
                e.preemption_nodes(asks, [alloc[(i * 5) % max(len(alloc), 1):][:40] for i in range(len(asks))], k=4, skip=step)
                launches += e.stats()["other_launches"] - before
            ask, node, _ = e.cycle(40)
            out.append((ask, node, e.ask_states(np.arange(s.n_asks)), e.nodes_available(np.arange(s.n_nodes))))
            if step == 1:
                e.release(ask[::2])
    return out, launches


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_no_effect_on_later_cycles(commit):
    for s in (synth.perf(300, 10, 20, masks=True, seed=12), synth.fuzz(4, n_nodes=200, n_asks=300)):
        plain, _ = _sequence(s, commit, False)
        called, launches = _sequence(s, commit, True)
        assert launches > 0
        for a, b in zip(plain, called):
            for x, y in zip(a, b):
                assert np.array_equal(x, y), (s.name, commit)


@pytest.mark.gpu
def test_errors(oracle):
    from yunikorn_k8shim_b200 import YkError
    p = lambda x: None if x is None else x.ctypes.data_as(C.c_void_p)   # noqa: E731
    u32 = lambda x: np.asarray(x, dtype=np.uint32)                      # noqa: E731

    def outs(n, k):
        return [np.full((n, k), 7, np.uint32), np.full((n, k), 7, np.uint32)] + [np.full(n, 7, np.uint32) for _ in range(3)]

    # a NaN node score: YK_ERR_RANGE, nothing written
    s = nan_node()
    with _engine_cls().for_snapshot(s) as e:
        o = outs(1, 2)
        before = e.stats()["other_launches"]
        rc = e._lib.yk_preemption_nodes(e._h, 1, p(u32([0])), p(u32([0, 0])), None, 0, 2, *[p(x) for x in o])
        assert rc == YK_ERR_RANGE and all((x == 7).all() for x in o)
        assert e.stats()["other_launches"] > before
        with pytest.raises(YkError) as ei:
            e.preemption_nodes([0], [[]])
        assert ei.value.code == YK_ERR_RANGE

    s = synth.perf(40, 6, 30, masks=True, seed=5)
    s.node_avail[:, :2] //= 20                                   # some asks stay pending
    e, t, bound, want = scenario(oracle, s, "auto", extra=0)
    ref, _, _, _ = scenario(oracle, s, "auto", extra=0)
    with e, ref:
        alloc = u32(want["ask"])
        pend = u32(np.nonzero(want["state"] != ST_ALLOCATED)[0])
        assert len(alloc) >= 6 and len(pend) > 0
        A = s.n_asks
        lib, h = e._lib, e._h
        v = alloc[:6]
        cases = [  # (n, asks, off, victims, k, nodes_out given, expected code)
            (2, None, [0, 3, 6], v, 2, True, YK_ERR_ARG),                     # asks NULL
            (2, [0, 1], None, v, 2, True, YK_ERR_ARG),                        # victim_off NULL
            (2, [0, 1], [0, 3, 6], None, 2, True, YK_ERR_ARG),                # victims NULL with entries
            (2, [0, 1], [0, 3, 6], v, 2, False, YK_ERR_ARG),                  # nodes_out NULL with k > 0
            (2, [0, A], [0, 3, 6], v, 2, True, YK_ERR_ARG),                   # ask index >= max_asks
            (2, [0, 1], [0, 3, 6], list(v[:5]) + [A], 2, True, YK_ERR_ARG),  # victim index >= max_asks
            (2, [0, 1], [1, 3, 6], v, 2, True, YK_ERR_ARG),                   # victim_off[0] != 0
            (2, [0, 1], [0, 4, 3], v, 2, True, YK_ERR_ARG),                   # decreasing
            (2, [0, 1], [0, 3, 6], list(v[:5]) + [v[3]], 2, True, YK_ERR_ARG),   # the same victim twice in one list
            (2, [0, 1], [0, 3, 6], list(v[:5]) + [pend[0]], 2, True, YK_ERR_STATE),   # a victim that is not allocated
        ]
        for n, asks, off, vic, k, give, code in cases:
            o = outs(n, k)
            args = [p(None if asks is None else u32(asks)), p(None if off is None else u32(off)), p(None if vic is None else u32(vic))]
            rc = lib.yk_preemption_nodes(h, n, *args, 0, k, p(o[0]) if give else None, *[p(x) for x in o[1:]])
            assert rc == code, (asks, off, vic, k, give)
            assert all((x == 7).all() for x in o)
        # the same victim in two different lists is fine; n == 0 is YK_OK
        assert lib.yk_preemption_nodes(h, 2, p(u32([0, 1])), p(u32([0, 1, 2])), p(u32([v[0], v[0]])), 0, 0, None, None, None, None, None) == 0
        assert lib.yk_preemption_nodes(h, 0, None, None, None, 0, 0, None, None, None, None, None) == 0
        # a released victim
        e.release(v[:1])
        ref.release(v[:1])
        o = outs(1, 2)
        assert lib.yk_preemption_nodes(h, 1, p(u32([0])), p(u32([0, 2])), p(u32(v[:2])), 0, 2, *[p(x) for x in o]) == YK_ERR_STATE
        assert all((x == 7).all() for x in o)
        with pytest.raises(YkError) as ei:
            e.preemption_nodes([0], [v[:2]])
        assert ei.value.code == YK_ERR_STATE
        # the next cycle is the same as on an engine that saw none of these calls
        a1, n1, _ = e.cycle(A)
        a2, n2, _ = ref.cycle(A)
        assert np.array_equal(a1, a2) and np.array_equal(n1, n2) and len(a1) > 0
        assert np.array_equal(e.ask_states(np.arange(A)), ref.ask_states(np.arange(A)))
        assert np.array_equal(e.nodes_available(np.arange(s.n_nodes)), ref.nodes_available(np.arange(s.n_nodes)))


@pytest.mark.gpu
def test_counters(oracle):
    """per call: the node order (11 launches, 4 bytes back), the position scatter, and per chunk 5 kernels + the entry sort
    (2 + one pass per 8 key bits) + the group scan (2); H2D 4 bytes per list twice + 4, and 8 per kept entry; D2H 4 (2k + 3)
    per list"""
    s = synth.perf(300, 10, 20, masks=True, seed=3)
    rng = np.random.default_rng(3)
    e, t, bound, want = scenario(oracle, s, "auto", extra=0)
    with e:
        gone = np.unique(want["node"])[:3]
        e.nodes_remove(gone)
        alloc = np.asarray(want["ask"])
        asks = np.arange(0, 40, dtype=np.uint32)
        lists = [rng.permutation(alloc)[:int(rng.integers(0, 30))].astype(np.uint32) for _ in asks]
        k = 5
        e.preemption_nodes(asks, lists, k=k)                     # uploads the changed tables
        st0 = e.stats()
        e.preemption_nodes(asks, lists, k=k)
        st1 = e.stats()
        m = sum(1 for x in lists for v in x if bound[int(v)] not in gone)
        n, nlive = len(asks), s.n_nodes - len(gone)
        end_bit = max(1, (nlive - 1).bit_length()) + max(1, (n - 1).bit_length())
        assert st1["other_launches"] - st0["other_launches"] == 11 + 1 + 5 + 2 + (end_bit + 7) // 8 + 2
        assert st1["h2d_bytes"] - st0["h2d_bytes"] == 4 * (2 * n + 1) + 8 * m
        assert st1["d2h_bytes"] - st0["d2h_bytes"] == 4 + 4 * n * (2 * k + 3)
        assert st1["cycles"] == st0["cycles"] and st1["sweep_launches"] == st0["sweep_launches"]


# ---- the reference's known answers ----
def golden_snapshot():
    """one node; the four victims of TestPreemptionPredicates are asks that a cycle binds to it"""
    D = 3
    alloc = np.array([GOLD["node_alloc"]], dtype=np.int64)
    vic = np.array(GOLD["victims"], dtype=np.int64)
    z = np.zeros(1, dtype=np.uint64)
    z4 = np.zeros(len(vic), dtype=np.uint64)
    return synth._finish("preempt-nodes-golden", D, 0, alloc, alloc.copy(), z, z.copy(), ["node0"], synth._single_queue(D),
                         np.ones(1, np.int32), np.zeros(len(vic), np.int32), vic, z4, z4.copy(), z4.copy())


def golden_expect(oracle, c, e=None):
    """-> (t, bound, preemptor, list, pairs): after the cycle every victim is on node 0, then the preemptor is upserted"""
    s = golden_snapshot()
    want = oracle.run(s)
    t = copy.deepcopy(s)
    t.node_avail = np.ascontiguousarray(want["avail"], dtype=np.int64)
    bound = {int(a): int(n) for a, n in zip(want["ask"], want["node"])}
    if e is not None:
        ask, node, _ = e.cycle(s.n_asks)
        assert ask.tolist() == want["ask"].tolist() and node.tolist() == want["node"].tolist()
    pre = add_asks(e, t, [c["req"]]) if e is not None else _append_only(t, c["req"])
    lst = np.arange(len(GOLD["victims"]), dtype=np.uint32) if c["victims"] else np.zeros(0, np.uint32)
    return t, bound, int(pre[0]), lst, expect(oracle, t, bound, [int(pre[0])], [lst])[0]


def _append_only(t, req):
    class _NoEngine:
        def asks_upsert(self, *a, **kw):
            pass
    return add_asks(_NoEngine(), t, [req])


@pytest.mark.gpu
def test_reference_known_answers(oracle):
    for c in GOLD["cases"]:
        s = golden_snapshot()
        e = _engine_cls()(D=s.D, policy=s.policy, weights=s.weights, max_nodes=1, max_asks=8, max_apps=1, max_queues=2)
        with e:
            e.load_snapshot(s)
            t, bound, pre, lst, pairs = golden_expect(oracle, c, e)
            nodes, need, n_fit, bn, bneed = e.preemption_nodes([pre], [lst], k=2)
        if c["index"] >= 0:
            assert n_fit.tolist() == [1] and nodes[0].tolist() == [0, YK_NONE] and need[0].tolist() == [c["index"] + 1, 0], c["name"]
            assert (bn[0], bneed[0]) == (0, c["index"] + 1)
        else:
            assert n_fit.tolist() == [0] and nodes[0].tolist() == [YK_NONE] * 2 and bn[0] == YK_NONE and bneed[0] == 0, c["name"]


# ---- on the CPU ----
def test_expectation_helper_reproduces_known_answers(oracle):
    """the helper, from the oracle alone: the reference's answers (given at start 1) are the same at start 0; the empty list
    and the too-large pod do not fit"""
    assert len(GOLD["cases"]) == 3
    for c in GOLD["cases"]:
        t, bound, pre, lst, pairs = golden_expect(oracle, c)
        assert set(bound) == set(range(len(GOLD["victims"]))) and set(bound.values()) == {0}
        if c["victims"]:
            assert [(n, vs) for n, vs, _ in pairs] == [(0, lst.tolist())]
            assert pairs[0][2] == c["index"], c["name"]
        else:
            assert pairs == []
        assert fits(pairs) == ([(0, c["index"] + 1)] if c["index"] >= 0 else [])
