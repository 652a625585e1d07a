"""yk_node_sort_set: the node sort policy and resource weights switched on a live engine.

A partition's nodesortpolicy arrives with the scheduler configuration, after the engine exists, and can change with every
configuration update.  After a switch every path -- the sweep + host commit, uniform runs, rounds, the lattice kernel, the
binpacking fill, yk_filter_nodes, yk_preemption_nodes and yk_node_scores -- must order and score the nodes under the new
setting, and nothing derived from the old one may survive: the engine must be in the state an engine created with the new
setting and loaded with the same tables would be in.

The sessions are test_sessions' Model / Generator with one more operation between cycles: a switch of policy and weights
(default, all zero, configured, or weighting a resource on which some nodes have total 0 and so an infinite share).  The
model passes its current policy and weights to the oracle every cycle and the engine gets the same node_sort_set call, so
test_sessions.replay checks every cycle of a switched session exactly as it checks an unswitched one.  Sessions with a
seed of at least test_sessions.MIXED_FROM have fair leaves too.  The CPU tests check that both oracles agree on every switched cycle and that the sessions
switch in every direction and with every kind of weights."""
import copy
import ctypes as C
import functools

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
import test_sessions as ts
import test_preemption_nodes as tpn
from test_filter import expect as filter_expect, window

FAIR, BP = synth.POLICY_FAIR, synth.POLICY_BINPACKING
GI = synth.GI
YK_ERR_ARG, YK_ERR_RANGE = -1, -5
KINDS = ("default", "zero", "configured", "infinite")
NAMES = {FAIR: "fair", BP: "binpacking"}


# ---- the switch operation on the model ----
def switch(m, policy, weights, kind):
    """the model's node sort from now on, and the engine call that makes it the engine's"""
    m.note(f"switch_{NAMES[m.policy]}_to_{NAMES[policy]}")
    m.note(f"switch_{kind}")
    m.policy, m.weights = policy, np.asarray(weights, np.float64).copy()
    m._op("node_sort_set", "node_sort_set", policy=policy, weights=m.weights.copy())


def random_switch(m, rng):
    D = m.D
    policy = int(rng.integers(0, 2))
    kind = KINDS[int(rng.integers(0, len(KINDS)))]
    if kind == "default":
        w = ts._weights(D)
    elif kind == "zero":
        w = np.zeros(D)
    elif kind == "configured":
        w = rng.choice([0.0, 0.25, 0.5, 1.0, 2.0, 3.0], D)
        if not w.any():
            w[0] = 1.5
    else:
        # one or two idle nodes get total 0 on the last resource with something on it (a negative foreign occupancy gives
        # available > 0, share -Inf; a positive one available < 0, share +Inf), and the new weights count that resource.  One
        # infinite share per node, so no score is NaN.
        k = D - 1
        idle = [int(n) for n in m.present_nodes() if not m.n_used[n].any()]
        if idle:
            pick = sorted(rng.choice(idle, min(2, len(idle)), replace=False).tolist())
            for n in pick:
                m.n_total[n, k] = 0
                m.n_foreign[n, k] = int(rng.choice([-500, 500]))
            m.nodes_upsert(pick, "nodes_upsert(zero total)")
        w = ts._weights(D)
        w[k] = float(rng.choice([0.5, 1.0, 2.0]))
    switch(m, policy, w, kind)


def switched_session(oracle, seed, D=4, policy=FAIR):
    rng = np.random.default_rng([seed, D, policy, 17])
    m = ts.Model(oracle, f"switched(seed={seed}, D={D}, policy={policy})", D, policy, max_nodes=128, max_asks=1024,
                 seed=seed + 1000 * D)
    m.initial = (policy, m.weights.copy())
    g = ts.Generator(m, rng, leaves=ts.leaves(seed))
    g.start(int(rng.integers(12, 40)))
    for c in range(int(rng.integers(14, 27))):
        if c:
            g.step()
            if rng.random() < 0.55:
                random_switch(m, rng)
        m.check_conservation()
        m.cycle(*g.max_bindings())
        m.check_conservation()
    ts.finish(m)
    return m


SWITCHED = [(s, 4, FAIR) for s in range(5)] + [(s, 4, BP) for s in range(5, 10)] \
    + [(10, 1, FAIR), (11, 1, BP), (12, 8, FAIR), (13, 8, BP)] \
    + [(200, 4, FAIR), (201, 4, BP)]                                   # fair leaves (ts.MIXED_FROM)
SWITCHED_IDS = [f"seed{s}-D{d}-{NAMES[p]}" for s, d, p in SWITCHED]


@functools.lru_cache(maxsize=None)
def session(seed, D, policy):
    from oracle import oracle_ctypes
    oracle_ctypes.build()
    return switched_session(oracle_ctypes, seed, D, policy)


# ---- targeted scripts ----
def _start(oracle, name, first, n_nodes=12, **kw):
    m = ts._base(oracle, name, n_nodes, **kw)
    m.policy = first
    m.initial = (first, m.weights.copy())
    return m


def t_switch(oracle, first, then):
    """cycles under `first` with releases in between, leaving the nodes unevenly used; then a switch to `then` and cycles.
    m.after_switch: the cycles that follow the switch"""
    m = _start(oracle, f"switch-{NAMES[first]}-to-{NAMES[then]}", first)
    m.asks_upsert(list(range(40)), np.stack([ts._req(250 * (1 + i % 4)) for i in range(40)]), 0)
    ask, _, _ = m.cycle()
    m.release(ask[::3])
    m.asks_upsert(list(range(40, 60)), ts._req(500), 1)
    ask, _, _ = m.cycle()
    m.release(ask[::2])
    m.asks_upsert(list(range(60, 60 + 2 * ts.UNIFORM_MIN)), ts._req(300), 0)   # a run: the uniform path
    m.cycle()
    m.asks_upsert(list(range(100, 130)), np.stack([ts._req(100 * (1 + i % 5), GI * (1 + i % 3)) for i in range(30)]), 1)
    _, before, _ = m.preview()                          # where the old setting would put them
    switch(m, then, ts._weights(m.D), "default")
    m.after_switch = {m.cycles, m.cycles + 1}
    _, node, _ = m.cycle()
    assert len(node) == 30 and not np.array_equal(node, before), m.name
    m.asks_upsert(list(range(130, 130 + 2 * ts.UNIFORM_MIN)), ts._req(200), 0)
    m.cycle()
    ts.finish(m)
    return m


def t_binpacking_e2e(oracle):
    """The reference's bin packing scenario (test/e2e/bin_packing/bin_packing_test.go:46-200), on a live engine: the suite
    switches the partition to binpacking before it runs and back to fair after it.  Four identical nodes, each with one
    identity label bit; padding pods pinned by that label put nodeA at 20 % memory use and nodeB at 10 % (under fair).
    Then binpacking: job A (3 pods) lands on nodeA; job B (3 pods, node NotIn nodeA: a forbidden label bit) on nodeB.  Then
    fair again: the next pods go to the least used nodes."""
    mem = 64 * GI
    m = ts.Model(oracle, "binpacking-e2e-live", 4, FAIR, max_nodes=8, max_asks=64)
    m.initial = (FAIR, m.weights.copy())
    m.queues_set(np.full((m.maxQ, 4), -1), np.full((m.maxQ, 4), -1), np.zeros(m.maxQ))
    m.apps_upsert([0, 1, 2, 3], ts.LEAVES[0])
    for n in range(4):
        m.set_node(n, np.array([16000, mem, 110, 4000]), label=1 << n, num=100 + 10 * n)
        m.used_nums.add(100 + 10 * n)
    m.nodes_upsert(list(range(4)), "nodes_upsert(nodeA..nodeD)")
    m.asks_upsert([0], np.array([0, mem // 5, 1, 0]), 0, need=1)      # nodeA's padding (0 m CPU, 20 % memory)
    m.asks_upsert([1], np.array([0, mem // 10, 1, 0]), 1, need=2)     # nodeB's
    _, node, _ = m.cycle()
    assert node.tolist() == [0, 1], node
    switch(m, BP, ts._weights(4), "default")
    job = np.array([100, GI, 1, 0])
    m.asks_upsert([2, 3, 4], job, 2)
    _, node, _ = m.cycle()
    assert node.tolist() == [0, 0, 0], node                           # job A: the most used node
    m.asks_upsert([5, 6, 7], job, 3, deny=1)
    _, node, _ = m.cycle()
    assert node.tolist() == [1, 1, 1], node                           # job B: not nodeA, so the next most used
    switch(m, FAIR, ts._weights(4), "default")
    m.asks_upsert([8, 9, 10], job, 2)
    _, node, _ = m.cycle()
    assert node.tolist() == [2, 3, 2], node                           # fair: the least used nodes, NodeID order on ties
    ts.finish(m)
    return m


TARGETED = {"fair_to_binpacking": lambda o: t_switch(o, FAIR, BP), "binpacking_to_fair": lambda o: t_switch(o, BP, FAIR),
            "binpacking_e2e": t_binpacking_e2e}


# ---- replay on the engine ----
def _stats_ok(bp_device, m, c, commit, d, where):
    """test_sessions._stats_ok with the eligibility of the cycle's own setting: the device commit takes a cycle under fair
    (binpacking too with the flag) with non-negative weights and one request vector per gang"""
    s = c.snap
    assert d["cycles"] == 1 and d["allocations"] == len(c.ask), where
    eligible = (s.policy == FAIR or bp_device) and (s.weights >= 0).all() and ts._one_request_per_gang(s)
    lat = d["lattice_cycles"]
    if commit == "host" or not eligible:
        assert lat == 0 and d["lattice_launches"] == 0 and d["uniform_asks"] == 0 and d["round_asks"] == 0, (where, d)
    elif commit == "device":
        assert lat == 1, (where, d)
    else:
        assert lat in (0, 1) and (lat or d["uniform_asks"] == 0), (where, d)
    assert d["lattice_handoffs"] <= lat, (where, d)
    if s.policy == FAIR:
        assert d["lattice_handoffs"] == 0 or c.has_gang, (where, d)


def replay(monkeypatch, m, commit, batch, bp_device, **kw):
    """test_sessions.replay, on an engine created with the session's INITIAL setting (and the binpacking flag as given)"""
    from yunikorn_k8shim_b200 import Engine
    policy, weights = m.initial

    def engine(m, commit, batch):
        return Engine(D=m.D, policy=policy, weights=weights, max_nodes=m.maxN, max_asks=m.maxA, max_apps=m.maxP,
                      max_queues=m.maxQ, batch=batch, commit=commit, binpacking_device=bp_device)
    monkeypatch.setattr(ts, "_engine", engine)
    monkeypatch.setattr(ts, "_stats_ok", functools.partial(_stats_ok, bp_device))
    monkeypatch.setenv("YK_UNIFORM_MIN", str(ts.UNIFORM_MIN))
    return ts.replay(m, commit, batch, **kw)


# ---- GPU: 1. switched sessions ----
@pytest.mark.gpu
@pytest.mark.parametrize("bp_device", [False, True], ids=["noflag", "bpdevice"])
@pytest.mark.parametrize("batch", [64, 4096])
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
@pytest.mark.parametrize("seed,D,policy", SWITCHED, ids=SWITCHED_IDS)
def test_switched_session(monkeypatch, seed, D, policy, commit, batch, bp_device):
    """bindings, availability, device scores, ask states and commit counters against the model after every cycle; the host
    runs also check yk_filter_nodes before every cycle"""
    m = session(seed, D, policy)
    _, tot = replay(monkeypatch, m, commit, batch, bp_device, filter_k=9 if commit == "host" and batch == 64 else None)
    if commit == "device" and (bp_device or any(c.snap.policy == FAIR for c in ts._cycles(m))):
        assert tot["lattice_cycles"] > 0, m.name


# ---- GPU: 2. a switched engine equals a fresh one ----
@pytest.mark.gpu
@pytest.mark.parametrize("bp_device", [False, True], ids=["noflag", "bpdevice"])
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
@pytest.mark.parametrize("name", ["fair_to_binpacking", "binpacking_to_fair"])
def test_switched_engine_equals_a_fresh_one(oracle, monkeypatch, name, commit, bp_device):
    """every cycle after the switch: an engine created with the new setting and loaded with the model's state just before
    that cycle gives the same bindings, ask states, availability and device scores (and both give the oracle's)"""
    from yunikorn_k8shim_b200 import Engine
    m = TARGETED[name](oracle)
    seen = []

    def fresh(e, c, d):
        if c.number not in m.after_switch:
            return
        s = c.snap
        assert s.policy == m.policy
        with Engine.for_snapshot(s, batch=64, commit=commit, binpacking_device=bp_device) as f:
            ask, node, _ = f.cycle(max(s.n_asks, 1))
            assert c.amap[ask].tolist() == c.ask.tolist() and c.nmap[node].tolist() == c.node.tolist(), (name, c.number)
            assert np.array_equal(f.nodes_available(np.arange(s.n_nodes)), e.nodes_available(c.nmap)), (name, c.number)
            got, want = f.node_scores(np.arange(s.n_nodes)), e.node_scores(c.nmap)
            assert np.array_equal(got.view(np.int64), want.view(np.int64)), (name, c.number)
            assert np.array_equal(f.ask_states(np.arange(s.n_asks)), e.ask_states(c.amap)), (name, c.number)
            assert f.stats()["lattice_cycles"] == d["lattice_cycles"], (name, c.number)
        seen.append(c.number)
    replay(monkeypatch, m, commit, 64, bp_device, on_cycle=fresh)
    assert sorted(seen) == sorted(m.after_switch)


# ---- GPU: 3. the right path runs after a switch ----
def _live(s, first, batch, **kw):
    """an engine created under `first` (default weights) holding snapshot s, which has already ordered and scored the nodes
    under it (node scores, a filter query, a cycle cut at zero bindings)"""
    from yunikorn_k8shim_b200 import Engine
    e = Engine(D=s.D, policy=first, weights=None, max_nodes=s.n_nodes, max_asks=s.n_asks, max_apps=max(s.n_apps, 1),
               max_queues=max(s.n_queues, 1), batch=batch, **kw)
    e.load_snapshot(s)
    e.node_scores(np.arange(s.n_nodes))
    e.filter_nodes([0], k=4)
    ask, _, _ = e.cycle(0)
    assert len(ask) == 0
    return e


def _switched_cycle(oracle, s, first, batch, **kw):
    want = oracle.run(s)
    with _live(s, first, batch, **kw) as e:
        e.node_sort_set(s.policy, s.weights)
        before = e.stats()
        ask, node, _ = e.cycle(s.n_asks)
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"]), (s.name, kw)
        assert np.array_equal(e.nodes_available(np.arange(s.n_nodes)), want["avail"]), (s.name, kw)
        assert np.array_equal(e.ask_states(np.arange(s.n_asks)), want["state"]), (s.name, kw)
        st = e.stats()
    return {k: v - before[k] for k, v in st.items() if not isinstance(v, list)}


@pytest.mark.gpu
def test_fair_to_binpacking_takes_the_fill(oracle):
    s = synth.reference_shape(5000, 400, 125, policy=BP)
    for commit in ("auto", "device"):
        d = _switched_cycle(oracle, s, FAIR, 4096, commit=commit, binpacking_device=True)
        assert d["lattice_cycles"] == 1 and d["uniform_runs"] == 1 and d["uniform_asks"] == 50_000, (commit, d)
        assert d["sweep_launches"] == 0 and d["uniform_retries"] == 0 and d["round_asks"] == 0, (commit, d)


@pytest.mark.gpu
def test_fair_to_binpacking_without_the_flag_stays_on_the_host(oracle):
    s = synth.reference_shape(5000, 400, 125, policy=BP)
    for commit in ("auto", "device"):
        d = _switched_cycle(oracle, s, FAIR, 4096, commit=commit)
        for k in ("lattice_cycles", "lattice_launches", "lattice_asks", "uniform_runs", "uniform_asks", "round_passes", "round_asks"):
            assert d[k] == 0, (commit, k, d)
        assert d["sweep_launches"] > 0, (commit, d)


@pytest.mark.gpu
def test_binpacking_to_fair_takes_the_rounds(oracle):
    s = synth.perf()                                    # config 2: 10 000 nodes, 50 000 mask-free asks
    d = _switched_cycle(oracle, s, BP, 2048)
    assert d["lattice_cycles"] == 1 and d["round_passes"] > 0 and d["round_asks"] == 50_000, d


@pytest.mark.gpu
def test_binpacking_to_fair_takes_a_uniform_run(oracle):
    s = synth.reference_shape(5000, 400, 125)
    for bp_device in (False, True):
        d = _switched_cycle(oracle, s, BP, 4096, binpacking_device=bp_device)
        assert d["lattice_cycles"] == 1 and d["uniform_runs"] == 1 and d["uniform_asks"] == 50_000, (bp_device, d)


# ---- GPU: 4. the reference's bin packing scenario ----
@pytest.mark.gpu
@pytest.mark.parametrize("bp_device", [False, True], ids=["noflag", "bpdevice"])
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_reference_bin_packing_scenario(oracle, monkeypatch, commit, bp_device):
    replay(monkeypatch, t_binpacking_e2e(oracle), commit, 64, bp_device)


# ---- GPU: 5. the queries follow the switch ----
SWITCHES = [(FAIR, BP, None), (BP, FAIR, [0.5, 2.0, 1.0, 0.0]), (FAIR, FAIR, [0.0, 1.0, 0.0, 3.0])]


@pytest.mark.gpu
@pytest.mark.parametrize("first,then,w", SWITCHES, ids=["fair-binpacking", "binpacking-fair", "fair-weights"])
def test_queries_follow_the_switch(oracle, first, then, w):
    """yk_filter_nodes candidates and counts, yk_preemption_nodes windows and yk_node_scores under the new setting equal the
    oracle's; a cycle after them equals that of a twin engine that made the same switch and no query"""
    from yunikorn_k8shim_b200 import Engine
    rng = np.random.default_rng(5)
    s = synth.perf(800, 16, 40, masks=True, policy=first)
    e, t, bound, want = tpn.scenario(oracle, s, "auto", extra=3)
    twin = Engine(D=s.D, policy=first, weights=s.weights, max_nodes=s.n_nodes, max_asks=s.n_asks + 3, max_apps=s.n_apps,
                  max_queues=s.n_queues)
    twin.load_snapshot(s)
    twin.cycle(s.n_asks)
    with e, twin:
        weights = ts._weights(s.D) if w is None else np.asarray(w, np.float64)
        for x in (e, twin):
            x.node_sort_set(then, weights)
        t.policy, t.weights = then, weights
        N = np.arange(t.n_nodes)
        want_scores = np.array([oracle.node_score(then, weights, t.node_total[n], t.node_avail[n]) for n in N])
        assert np.array_equal(e.node_scores(N).view(np.int64), want_scores.view(np.int64))
        # yk_filter_nodes, both phases, a window in the middle of the order
        asks = np.arange(0, t.n_asks, 37)
        for allocate in (True, False):
            nodes, n_pass, counts = e.filter_nodes(asks, k=16, skip=5, allocate=allocate)
            full, want_counts = filter_expect(oracle, t, asks, allocate)
            assert np.array_equal(counts, want_counts), allocate
            for i in range(len(asks)):
                assert n_pass[i] == len(full[i]) and nodes[i].tolist() == window(full[i], 5, 16), (allocate, int(asks[i]))
        # yk_preemption_nodes: NOFIT, allocated and new big asks against random victim lists
        pre = tpn.preemptors(e, t, want, rng, n_new=3)
        new = pre[-3:]
        twin.asks_upsert(new, t.ask_req[new], np.zeros(3, np.int32), t.ask_create[new], tolerated_bits=t.ask_tol[new])
        lists = tpn.random_lists(rng, np.asarray(want["ask"]), len(pre))
        tpn.check(e, t, tpn.expect(oracle, t, bound, pre, lists), pre, lists, k=8, skip=1)
        outs = []
        for x in (e, twin):
            ask, node, _ = x.cycle(t.n_asks)
            outs.append((ask, node, x.nodes_available(N), x.ask_states(np.arange(t.n_asks)), x.node_scores(N).view(np.int64)))
        for a, b in zip(*outs):
            assert np.array_equal(a, b)


# ---- GPU: 6. errors ----
EXTRA_ASKS = 128


def _pair(s, extra_nodes=0, **kw):
    """two engines holding s: one receives the calls under test, the other never does"""
    from yunikorn_k8shim_b200 import Engine
    out = []
    for _ in range(2):
        e = Engine(D=s.D, policy=s.policy, weights=s.weights, max_nodes=s.n_nodes + extra_nodes, max_asks=s.n_asks + EXTRA_ASKS,
                   max_apps=s.n_apps, max_queues=s.n_queues, batch=256, **kw)
        e.load_snapshot(s)
        out.append(e)
    return out


def _same(a, b, s, n_nodes, tag):
    N, A = np.arange(n_nodes), np.arange(s.n_asks + EXTRA_ASKS)
    assert np.array_equal(a.node_scores(N).view(np.int64), b.node_scores(N).view(np.int64)), tag
    assert np.array_equal(a.ask_states(A), b.ask_states(A)), tag
    assert np.array_equal(a.nodes_available(N), b.nodes_available(N)), tag


def _more_asks(engines, s, k, j):
    """the same eight new pending asks in every engine (application j % n_apps)"""
    idx = np.arange(s.n_asks + 8 * k, s.n_asks + 8 * k + 8)
    req = np.tile(s.ask_req[0], (8, 1))
    for e in engines:
        e.asks_upsert(idx, req, np.full(8, j % s.n_apps, np.int32), 10 ** 9 + idx, tolerated_bits=np.full(8, ~np.uint64(0)))


def _cycle_same(a, b, tag):
    x, y = a.cycle(4096), b.cycle(4096)
    assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]), tag
    return x


def _counters(e):
    return {k: v for k, v in e.stats().items() if k not in ("other_launches", "h2d_bytes", "d2h_bytes")}


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_errors_leave_the_engine_as_it_was(oracle, commit):
    from yunikorn_k8shim_b200 import YkError
    s = synth.perf(300, 8, 40, masks=True)
    D = s.D
    a, b = _pair(s, extra_nodes=1, commit=commit)
    with a, b:
        # a node on which resources 0 and 3 have total 0: available +500 on 0 (share -Inf), -500 on 3 (share +Inf).  Under the
        # default weights only resource 0 counts (score -Inf); weighting resource 3 as well makes the score -Inf + Inf = NaN
        rank = int(s.node_rank().max()) + 1
        for e in (a, b):
            e.nodes_upsert([s.n_nodes], np.array([[0, 8 * GI, 110, 0]]), np.array([[500, 8 * GI, 110, -500]]),
                           np.zeros(1, np.uint64), np.zeros(1, np.uint64), [rank], [synth.NODE_SCHEDULABLE])
        n_nodes = s.n_nodes + 1
        _cycle_same(a, b, "first cycle")
        nan_w = ts._weights(D)
        nan_w[3] = 1.0
        bad = [("policy 2", 2, ts._weights(D), YK_ERR_ARG), ("policy ~0", 0xFFFFFFFF, ts._weights(D), YK_ERR_ARG),
               ("NaN weight", FAIR, [1.0, np.nan, 0, 0], YK_ERR_ARG), ("+Inf weight", BP, [np.inf, 1.0, 0, 0], YK_ERR_ARG),
               ("-Inf weight", FAIR, [1.0, 0, 0, -np.inf], YK_ERR_ARG), ("NaN score", FAIR, nan_w, YK_ERR_RANGE),
               ("NaN score, binpacking", BP, nan_w, YK_ERR_RANGE)]
        for k, (tag, policy, w, code) in enumerate(bad):
            before = _counters(a)
            with pytest.raises(YkError) as ei:
                a.node_sort_set(policy, w)
            assert ei.value.code == code, tag
            assert _counters(a) == before, tag
            _same(a, b, s, n_nodes, tag)
            _more_asks((a, b), s, k, k)
            _cycle_same(a, b, tag)
            _same(a, b, s, n_nodes, tag)
        # null weights and a null engine, through the library itself
        assert a._lib.yk_node_sort_set(a._h, C.c_uint32(FAIR), None) == YK_ERR_ARG
        assert a._lib.yk_node_sort_set(None, C.c_uint32(FAIR), ts._weights(D).ctypes.data_as(C.c_void_p)) == YK_ERR_ARG
        _same(a, b, s, n_nodes, "null")
        # the current setting again, and weights beyond D (ignored, NaN or not): YK_OK, one key launch and a 4-byte read-back,
        # nothing else moves and the next cycle is the same
        for k, w in enumerate((s.weights, list(s.weights) + [np.nan, np.inf, 7.0, 0])):
            before, launches, d2h = _counters(a), a.stats()["other_launches"], a.stats()["d2h_bytes"]
            a.node_sort_set(s.policy, w)
            assert a.stats()["other_launches"] == launches + 1 and a.stats()["d2h_bytes"] == d2h + 4
            assert _counters(a) == before
            _more_asks((a, b), s, len(bad) + k, k)
            _cycle_same(a, b, f"same setting {k}")
            _same(a, b, s, n_nodes, f"same setting {k}")


@pytest.mark.gpu
def test_no_node_launches_nothing_and_negative_weights_take_the_host_commit(oracle):
    from yunikorn_k8shim_b200 import Engine
    with Engine(D=4, commit="device") as e:
        before = e.stats()
        e.node_sort_set(BP, [2.0, 1.0, 0, 0])
        assert e.stats() == before                         # no present node: nothing launched, nothing read back
    # negative weights are accepted as yk_create accepts them; such cycles commit on the host, with the oracle's bindings
    s = synth.perf(300, 8, 40)
    t = copy.deepcopy(s)
    t.weights = np.array([-1.0, 2.0, 0.0, 0.5])
    want = oracle.run(t)
    with Engine.for_snapshot(s, commit="device", batch=4096) as e:
        e.node_sort_set(FAIR, t.weights)
        ask, node, _ = e.cycle(s.n_asks)
        st = e.stats()
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
        assert np.array_equal(e.nodes_available(np.arange(s.n_nodes)), want["avail"])
        assert st["lattice_cycles"] == 0 and st["sweep_launches"] > 0


# ---- CPU: 7. the switched sessions on their own ----
@pytest.mark.parametrize("seed,D,policy", SWITCHED, ids=SWITCHED_IDS)
def test_switched_sessions_oracles_agree(seed, D, policy):
    """every cycle's snapshot, under the setting of that cycle: the C++ and the Python oracle agree"""
    m = session(seed, D, policy)
    ts._oracles_agree(m)
    assert any(st[0] == "op" and st[1] == "node_sort_set" for st in m.steps), m.name


@pytest.mark.parametrize("name", sorted(TARGETED))
def test_targeted_switch_scripts(oracle, name):
    """each script has the shape it is meant to exercise (asserted inside), conserves its accounting and both oracles agree"""
    m = TARGETED[name](oracle)
    m.check_conservation()
    ts._oracles_agree(m)


def test_sessions_cover_every_switch():
    """the switched sessions switch in every direction and with every kind of weights a stated number of times, and each
    switch is an engine call in the script"""
    total, calls = {}, 0
    for args in SWITCHED:
        m = session(*args)
        for k, v in m.count.items():
            total[k] = total.get(k, 0) + v
        calls += sum(1 for st in m.steps if st[0] == "op" and st[1] == "node_sort_set")
    need = {"switch_fair_to_binpacking": 25, "switch_binpacking_to_fair": 25, "switch_fair_to_fair": 20,
            "switch_binpacking_to_binpacking": 20, "switch_default": 20, "switch_zero": 20, "switch_configured": 20,
            "switch_infinite": 20}
    short = {k: (total.get(k, 0), n) for k, n in need.items() if total.get(k, 0) < n}
    assert not short, short
    assert calls == sum(total[f"switch_{k}"] for k in KINDS)
    # the infinite shares are really there: some cycle snapshot holds a node with total 0 and available != 0 on a weighted
    # resource, under both policies
    inf = {p: 0 for p in (FAIR, BP)}
    for args in SWITCHED:
        for st in session(*args).steps:
            if st[0] == "cycle":
                s = st[1].snap
                hit = (s.node_total == 0) & (s.node_avail != 0) & (s.weights != 0)[None, :]
                inf[s.policy] += int(hit.any())
    assert inf[FAIR] >= 5 and inf[BP] >= 5, inf
