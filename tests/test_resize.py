"""yk_asks_resize: in-place pod resize (KEP-1287) of pending asks and of allocations.

The shim re-sends a task's allocation with the same AllocationKey whenever common.GetPodResource of its pod changes.  For a
bound pod the engine must move the bound node's available, the queue chain, the application and the user-limit held entries
by the change, with no fit, headroom or limit check (the kubelet has applied the resize); for a pending ask it must replace
the request, renumber the signature and recompute the cause, keeping everything else.  After a resize every path -- the
sweep + host commit, uniform runs, rounds, the lattice kernel, the binpacking fill, yk_filter_nodes and yk_preemption_nodes
-- must read the resized state, and yk_release must give back the new request.

The sessions are test_sessions' Model / Generator with one more operation between cycles: a batch of resizes (allocations up,
down, one resource to 0, unchanged, over-committing their node, pushing their queue over its max or their user over a limit,
on cordoned and on removed nodes; pending asks resized, made invalid and valid again, gang members resized apart and back to
one vector).  The model holds every allocation's request and derives node, queue and user accounting from it, so a resize on
the model is one assignment; test_node_sort_switch.replay then checks every cycle exactly as test_sessions checks it."""
import copy
import ctypes as C
import functools

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
import test_sessions as ts
import test_node_sort_switch as tns
import test_preemption_nodes as tpn
from test_filter import expect as filter_expect, window

FAIR, BP = synth.POLICY_FAIR, synth.POLICY_BINPACKING
GI, MI = synth.GI, 1 << 20
YK_ERR_ARG, YK_ERR_STATE, YK_ERR_RANGE = -1, -4, -5
ST_ALLOCATED, ST_NOFIT, ST_SKIPPED, ST_INVALID = 1, 2, 3, 5
INT64_MAX = np.iinfo(np.int64).max
KINDS = ("up", "down", "zero_dim", "unchanged", "overcommit", "queue_over_max", "user_over_limit", "on_cordoned", "on_removed",
         "pending", "invalid", "valid_again", "gang_apart", "gang_back")


# ---- the resize operation on the model ----
def resize(m, idx, req, text="asks_resize"):
    """new requests for present asks; an allocation's node, queues and user follow through the model's derived accounting"""
    idx = np.atleast_1d(np.asarray(idx, np.int64))
    req = np.broadcast_to(np.asarray(req, np.int64).reshape(-1, m.D), (len(idx), m.D)).copy()
    assert len(set(idx.tolist())) == len(idx)
    for a, r in zip(idx, req):
        assert m.a_state[a] != ts.ABSENT
        if m.a_state[a] == ts.ALLOCATED:
            assert (r >= 0).all()
            m.n_used[m.a_bound[a]] += r - m.a_req[a]
        m.a_req[a] = r
    m._op("asks_resize", text, idx=idx.copy(), req=req.copy())


def _valid(r):
    return (r >= 0).all() and (r > 0).any()


def _grow(rng, r, D):
    r = r.copy()
    r[0] += int(rng.choice([100, 250, 500]))
    if D > 1 and rng.random() < 0.5:
        r[1] += int(rng.choice([256 * MI, GI]))
    return r


def _shrink(rng, r, D):
    r = r.copy()
    r[0] //= 2
    if D > 1 and rng.random() < 0.5:
        r[1] //= 2
    return r


def random_resize(m, rng):
    """one asks_resize call of one to four resizes of random kinds (distinct asks)"""
    D = m.D
    chosen = {}
    alloc = lambda: [int(a) for a in np.nonzero(m.a_state == ts.ALLOCATED)[0] if a not in chosen]   # noqa: E731
    pending = lambda: [int(a) for a in np.nonzero(m.a_state == ts.PENDING)[0] if a not in chosen]   # noqa: E731

    def pick(c):
        return int(c[int(rng.integers(0, len(c)))])

    for _ in range(int(rng.integers(1, 5))):
        kind = KINDS[int(rng.integers(0, len(KINDS)))]
        al, pe = alloc(), pending()
        if kind in KINDS[:9] and not al:
            continue
        if kind in ("pending", "invalid") and not pe:
            continue
        if kind == "up":
            a = pick(al)
            chosen[a] = _grow(rng, m.a_req[a], D)
        elif kind == "down":
            a = pick(al)
            chosen[a] = _shrink(rng, m.a_req[a], D)
        elif kind == "zero_dim":
            a = pick(al)
            r = m.a_req[a].copy()
            r[int(rng.integers(0, D))] = 0
            chosen[a] = r
        elif kind == "unchanged":
            a = pick(al + pe)
            chosen[a] = m.a_req[a].copy()
        elif kind == "overcommit":
            live = [a for a in al if m.n_present[m.a_bound[a]]]
            if not live:
                continue
            a = pick(live)
            r = m.a_req[a].copy()
            r[0] += max(0, int(m.avail(m.a_bound[a])[0])) + int(rng.choice([1, 500]))
            chosen[a] = r
        elif kind == "queue_over_max":
            qa = m.q_alloc()
            cand = [(a, q) for a in al for q in m.chain(m.p_queue[m.a_app[a]]) if m.q_max[q, 0] >= 0]
            if not cand:
                continue
            a, q = cand[int(rng.integers(0, len(cand)))]
            r = m.a_req[a].copy()
            r[0] += max(0, int(m.q_max[q, 0] - qa[q, 0])) + 100
            chosen[a] = r
        elif kind == "user_over_limit":
            held = m.held()
            cand = [(a, i) for a in al for i, (q, u, mx) in enumerate(m.ul)
                    if m.p_user[m.a_app[a]] == u and q in set(m.chain(m.p_queue[m.a_app[a]])) and mx[0] >= 0]
            if not cand:
                continue
            a, i = cand[int(rng.integers(0, len(cand)))]
            r = m.a_req[a].copy()
            r[0] += max(0, int(m.ul[i][2][0] - held[i, 0])) + 100
            chosen[a] = r
        elif kind == "on_cordoned":
            on = [a for a in al if m.n_present[m.a_bound[a]] and not m.n_flags[m.a_bound[a]] & ts.SCHED]
            if not on:                                  # cordon the node of an allocation first
                live = [a for a in al if m.n_present[m.a_bound[a]]]
                if not live:
                    continue
                on = [pick(live)]
                n = int(m.a_bound[on[0]])
                m.n_flags[n] &= ~np.uint32(ts.SCHED)
                m.nodes_upsert([n], "nodes_upsert(cordon)")
            a = pick(on)
            chosen[a] = (_grow if rng.random() < 0.5 else _shrink)(rng, m.a_req[a], D)
        elif kind == "on_removed":
            on = [a for a in al if not m.n_present[m.a_bound[a]]]
            if not on:                                  # remove the node of an allocation first
                live = [a for a in al if m.n_present[m.a_bound[a]]]
                if not live or len(m.present_nodes()) <= 4:
                    continue
                on = [pick(live)]
                m.nodes_remove([int(m.a_bound[on[0]])])
            a = pick(on)
            chosen[a] = (_grow if rng.random() < 0.5 else _shrink)(rng, m.a_req[a], D)
        elif kind == "pending":
            a = pick(pe)
            chosen[a] = ts._ask_shape(rng, D) if rng.random() < 0.5 else _grow(rng, m.a_req[a], D)
        elif kind == "invalid":
            a = pick(pe)
            r = np.zeros(D, np.int64) if rng.random() < 0.5 else m.a_req[a].copy()
            if r.any():
                r[int(rng.integers(0, D))] = -100
            chosen[a] = r
        elif kind == "valid_again":
            bad = [a for a in pe if not _valid(m.a_req[a])]
            if not bad:
                continue
            a = pick(bad)
            chosen[a] = ts._ask_shape(rng, D)
            chosen[a][0] = max(chosen[a][0], 100)
        elif kind == "gang_apart":
            cand = [a for a in pe if m.a_gang[a] >= 0 and _gang_uniform(m, a)]
            if not cand:
                continue
            a = pick(cand)
            chosen[a] = _grow(rng, m.a_req[a], D)
        else:                                           # gang_back: every member of a split gang back to one vector
            cand = [a for a in pe if m.a_gang[a] >= 0 and not _gang_uniform(m, a)]
            if not cand:
                continue
            members = _gang(m, pick(cand))
            if any(x in chosen for x in members):
                continue
            for x in members:
                chosen[x] = m.a_req[members[0]].copy()
        m.note(f"resize_{kind}")
    if not chosen:
        return
    if len(chosen) > 1:
        m.note("resize_call_of_many")
    if any(m.a_state[a] == ts.ALLOCATED for a in chosen) and any(m.a_state[a] == ts.PENDING for a in chosen):
        m.note("resize_call_mixed")
    idx = sorted(chosen) if rng.random() < 0.5 else list(chosen)
    resize(m, idx, np.stack([chosen[a] for a in idx]))


def _gang(m, a):
    return [int(x) for x in np.nonzero((m.a_gang == m.a_gang[a]) & (m.a_app == m.a_app[a]) & (m.a_state != ts.ABSENT))[0]]


def _gang_uniform(m, a):
    g = _gang(m, a)
    return all(np.array_equal(m.a_req[x], m.a_req[g[0]]) for x in g)


def note_state(m):
    """what the state the next cycle starts from holds, counted once per cycle"""
    if any((m.avail(n) < 0).any() for n in m.present_nodes()):
        m.note("state_node_overcommitted")
    qa = m.q_alloc()
    if ((m.q_max >= 0) & (qa > m.q_max)).any():
        m.note("state_queue_over_max")
    if m.ul:
        mx = np.array([e[2] for e in m.ul])
        if ((mx >= 0) & (m.held() > mx)).any():
            m.note("state_user_over_limit")
    pend = m.pending()
    if len(pend) and any(not _valid(m.a_req[a]) for a in pend):
        m.note("state_pending_invalid")


def resized_session(oracle, seed, D=4, policy=FAIR):
    rng = np.random.default_rng([seed, D, policy, 23])
    m = ts.Model(oracle, f"resized(seed={seed}, D={D}, policy={policy})", D, policy, max_nodes=128, max_asks=1024,
                 seed=seed + 1000 * D)
    m.initial = (policy, m.weights.copy())
    g = ts.Generator(m, rng, leaves=ts.leaves(seed))
    g.start(int(rng.integers(12, 40)))
    for c in range(int(rng.integers(14, 27))):
        if c:
            g.step()
            for _ in range(int(rng.integers(1, 4))):
                random_resize(m, rng)
        note_state(m)
        m.check_conservation()
        m.cycle(*g.max_bindings())
        m.check_conservation()
    ts.finish(m)
    return m


RESIZED = [(s, 4, FAIR) for s in range(5)] + [(s, 4, BP) for s in range(5, 8)] \
    + [(8, 1, FAIR), (9, 1, BP), (10, 8, FAIR), (11, 8, BP)] \
    + [(200, 4, FAIR), (201, 4, BP), (202, 1, FAIR), (203, 8, FAIR)]   # fair leaves (ts.MIXED_FROM)
RESIZED_IDS = [f"seed{s}-D{d}-{tns.NAMES[p]}" for s, d, p in RESIZED]


@functools.lru_cache(maxsize=None)
def session(seed, D, policy):
    from oracle import oracle_ctypes
    oracle_ctypes.build()
    return resized_session(oracle_ctypes, seed, D, policy)


# ---- targeted scripts ----
def _start(oracle, name, n_nodes=12, policy=FAIR, **kw):
    m = ts._base(oracle, name, n_nodes, **kw)
    m.policy = policy
    m.initial = (policy, m.weights.copy())
    return m


def t_resize(oracle):
    """allocations resized up, down and to 0 on one resource, over their leaf's max and their user's limit, and over their
    node's capacity; pending asks resized and made invalid.  m.after_resize: the cycles that follow the first resize"""
    m = _start(oracle, "resize-then-cycles", 10)
    mx = np.full((m.maxQ, 4), -1)
    mx[3, 0] = 24000
    m.queues_set(np.full((m.maxQ, 4), -1), mx, np.zeros(m.maxQ))
    m.apps_upsert([0, 1], [3, 4], [0, 1])
    m.user_limits_set([(1, 1, np.array([16000, -1, -1, -1]))])
    m.asks_upsert(list(range(40)), np.stack([ts._req(250 * (1 + i % 4)) for i in range(40)]), 0)
    m.asks_upsert(list(range(40, 60)), ts._req(500), 1)
    ask, node, _ = m.cycle()
    a0, a1 = [int(a) for a in ask if m.a_app[a] == 0], [int(a) for a in ask if m.a_app[a] == 1]
    resize(m, a0[:4], np.stack([ts._req(2000, 2 * GI)] * 4))                        # leaf 3 over its max
    resize(m, a0[4:8], np.stack([ts._req(100, GI // 2)] * 4))
    resize(m, a1[:3], np.stack([ts._req(6000), ts._req(0), ts._req(2500, 0)]))      # user 1 over its limit
    pend = [int(a) for a in range(60) if m.a_state[a] == ts.PENDING][:3]
    if pend:
        resize(m, pend, np.stack([np.zeros(4, np.int64)] + [ts._req(150)] * (len(pend) - 1)))
    qa = m.q_alloc()
    assert qa[3, 0] > 24000 and m.held()[0, 0] > 16000, (qa[3], m.held())
    m.after_resize = {m.cycles, m.cycles + 1, m.cycles + 2}
    m.asks_upsert(list(range(60, 80)), np.stack([ts._req(100 * (1 + i % 5), GI) for i in range(20)]), 0)
    m.asks_upsert(list(range(80, 90)), ts._req(200), 1)
    m.cycle()
    n = int(m.a_bound[a0[8]])                                                         # its node over-committed
    r = m.a_req[a0[8]].copy()
    r[0] += int(m.avail(n)[0]) + 1500
    resize(m, [a0[8]], r)
    assert (m.avail(n) < 0).any()
    m.asks_upsert(list(range(90, 90 + 2 * ts.UNIFORM_MIN)), ts._req(300), 1)
    m.cycle()
    m.release(a0[:2])
    m.cycle()
    ts.finish(m)
    return m


def _front(m):
    """the present node the next ask would look at first (lowest oracle score, then NodeID)"""
    return min(m.present_nodes(), key=lambda n: (m.oracle.node_score(m.policy, m.weights, m.n_total[n], m.avail(n)), m.n_num[n]))


def t_overcommit(oracle, path):
    """a resize over-commits the node at the front of the order; then a cycle on the path under test fills the cluster: the
    uniform run (fair), rounds (fair, mixed requests, mask-free) or the binpacking fill (binpacking).  Under fair the node
    sorts last and every ask must pass it by; under binpacking it sorts first and the fill must skip it"""
    policy = BP if path == "fill" else FAIR
    m = _start(oracle, f"overcommit-{path}", 12, policy, shape=np.array([8000, 32 * GI, 110, 4000]))
    m.asks_upsert(list(range(12)), ts._req(1000), 0)
    m.cycle()
    n = int(_front(m))
    on = [int(a) for a in np.nonzero((m.a_state == ts.ALLOCATED) & (m.a_bound == n))[0]]
    assert on, (n, m.a_bound[:12])
    r = m.a_req[on[0]].copy()
    r[0] += int(m.avail(n)[0]) + 2000
    resize(m, [on[0]], r)
    assert m.avail(n)[0] == -2000
    m.overcommitted = n
    if path == "rounds":
        req = np.stack([ts._req(100 * (1 + i % 5), 256 * MI * (1 + i % 3)) for i in range(400)])
    else:
        req = ts._req(1000)
    k = 400 if path == "rounds" else 100
    m.asks_upsert(list(range(12, 12 + k)), req, 1)
    _, node, _ = m.cycle()
    assert n not in node.tolist() and (m.a_last[12:12 + k] == ts.NOFIT).any(), (path, n)
    ts.finish(m)
    return m


def t_fair_resize(oracle):
    """resizes decide a fair leaf's next order: applications 0, 1, 2 hold alike, so submit time orders them; 2's allocations
    grow and it goes last; then 0's shrink to zero on every resource (still held) and 1's grow past 2's: 0 goes first,
    then 2 before 1"""
    m = ts._fair_base(oracle, "fair-resize-order", 12, apps=(3, 3, 3))
    for p in range(3):
        m.asks_upsert(list(range(4 * p, 4 * p + 4)), ts._req(1000), p)
    m.cycle()
    resize(m, [8, 9], np.stack([ts._req(3000, 2 * GI)] * 2))
    for p in range(3):
        m.asks_upsert([20 + 2 * p, 21 + 2 * p], ts._req(200), p)
    ask, _, _ = m.cycle(5)
    assert [int(m.a_app[a]) for a in ask] == [0, 1, 0, 1, 2], ask
    resize(m, [0, 1, 2, 3], np.zeros((4, 4), np.int64))
    resize(m, [4, 5, 6, 7], np.stack([ts._req(4000, 4 * GI)] * 4))
    for p in range(3):
        m.asks_upsert([30 + 2 * p, 31 + 2 * p], ts._req(200), p)
    ask, _, _ = m.cycle(6)
    assert [int(m.a_app[a]) for a in ask][:4] == [0, 0, 2, 2] and ts.history_decided(m, ts._cycles(m)[-1]), ask
    ts.finish(m)
    return m


TARGETED = {"resize": t_resize, "overcommit_uniform": lambda o: t_overcommit(o, "uniform"),
            "overcommit_rounds": lambda o: t_overcommit(o, "rounds"), "overcommit_fill": lambda o: t_overcommit(o, "fill"),
            "fair_resize": t_fair_resize}


# ---- GPU: 1. resized sessions ----
@pytest.mark.gpu
@pytest.mark.parametrize("bp_device", [False, True], ids=["noflag", "bpdevice"])
@pytest.mark.parametrize("batch", [64, 4096])
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
@pytest.mark.parametrize("seed,D,policy", RESIZED, ids=RESIZED_IDS)
def test_resized_session(monkeypatch, seed, D, policy, commit, batch, bp_device):
    """bindings, availability, device scores, ask states and commit counters against the model after every cycle; the host
    runs also check yk_filter_nodes before every cycle"""
    m = session(seed, D, policy)
    _, tot = tns.replay(monkeypatch, m, commit, batch, bp_device, filter_k=9 if commit == "host" and batch == 64 else None)
    if commit == "device" and (policy == FAIR or bp_device):
        assert tot["lattice_cycles"] > 0, m.name


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_fair_resize_script(oracle, monkeypatch, commit):
    """resized holdings decide a fair leaf's order on every commit"""
    tns.replay(monkeypatch, t_fair_resize(oracle), commit, 64, False)


# ---- GPU: 2. a resized engine equals a fresh one ----
@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_resized_engine_equals_a_fresh_one(oracle, monkeypatch, commit):
    """every cycle after the first resize: an engine created and loaded with the model's state just before that cycle (node
    availability, queue allocated, user held, the pending asks) gives the same bindings, ask states, availability, device
    scores and commit"""
    from yunikorn_k8shim_b200 import Engine
    m = t_resize(oracle)
    seen = []

    def fresh(e, c, d):
        if c.number not in m.after_resize:
            return
        s = c.snap
        with Engine.for_snapshot(s, batch=64, commit=commit) as f:
            ask, node, _ = f.cycle(max(s.n_asks, 1))
            assert c.amap[ask].tolist() == c.ask.tolist() and c.nmap[node].tolist() == c.node.tolist(), c.number
            assert np.array_equal(f.nodes_available(np.arange(s.n_nodes)), e.nodes_available(c.nmap)), c.number
            got, want = f.node_scores(np.arange(s.n_nodes)), e.node_scores(c.nmap)
            assert np.array_equal(got.view(np.int64), want.view(np.int64)), c.number
            assert np.array_equal(f.ask_states(np.arange(s.n_asks)), e.ask_states(c.amap)), c.number
            assert f.stats()["lattice_cycles"] == d["lattice_cycles"], c.number
        seen.append(c.number)
    tns.replay(monkeypatch, m, commit, 64, False, on_cycle=fresh)
    assert sorted(seen) == sorted(m.after_resize)


# ---- GPU: 3. over-commit of the front node on the device paths ----
@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
@pytest.mark.parametrize("path", ["uniform", "rounds", "fill"])
def test_overcommitted_front_node(oracle, monkeypatch, path, commit):
    """the cycle after the resize runs on the path under test (from the counters) and matches the oracle"""
    if path == "rounds":
        monkeypatch.setenv("YK_ROUND_MIN", "1")
        monkeypatch.setenv("YK_ROUND_GUARD", "0")
    m = TARGETED[f"overcommit_{path}"](oracle)
    per = []
    tns.replay(monkeypatch, m, commit, 4096, path == "fill", on_cycle=lambda e, c, d: per.append(d))
    d = per[1]
    if commit == "host":
        assert d["lattice_cycles"] == 0 and d["sweep_launches"] > 0, d
    elif path == "rounds":
        assert d["lattice_cycles"] == 1 and (d["round_asks"] > 0 if commit == "auto" else d["lattice_asks"] > 0), d
    elif commit == "device":
        assert d["lattice_cycles"] == 1 and d["uniform_runs"] > 0 and d["uniform_asks"] > 0, d
    else:                                               # auto prices the run against the host commit
        assert d["lattice_cycles"] == 0 or d["uniform_asks"] > 0, d


# ---- GPU: 4. release, order, filter and preemption after a resize ----
@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_release_after_resize_restores_the_node(oracle, commit):
    """allocations resized up, down, to zero and back, some several times: releasing them all returns every node to what
    it had before the cycle, and the next cycle equals the oracle on the original snapshot"""
    from yunikorn_k8shim_b200 import Engine
    rng = np.random.default_rng(3)
    s = synth.perf(200, 8, 40, seed=5)
    want = oracle.run(s)
    with Engine.for_snapshot(s, commit=commit, batch=256) as e:
        ask, node, _ = e.cycle(s.n_asks)
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
        for step in range(3):
            pick = rng.permutation(ask)[:len(ask) // 2]
            req = s.ask_req[pick] * rng.integers(0, 4, (len(pick), 1))
            req[::5, 1] = 0
            e.asks_resize(pick, req)
        e.release(ask)
        assert np.array_equal(e.nodes_available(np.arange(s.n_nodes)), s.node_avail)
        e.asks_upsert(ask, s.ask_req[ask], s.ask_app[ask], s.ask_create[ask], s.ask_tol[ask], s.ask_need[ask], s.ask_deny[ask],
                      s.ask_prio[ask], s.ask_node[ask], s.ask_flags[ask], s.ask_gang[ask])
        ask2, node2, _ = e.cycle(s.n_asks)
        assert np.array_equal(ask2, want["ask"]) and np.array_equal(node2, want["node"])
        assert np.array_equal(e.nodes_available(np.arange(s.n_nodes)), want["avail"])


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_resized_pending_ask_keeps_its_place(oracle, commit):
    """pending asks of several priorities on a cluster too small for all of them: some are resized (smaller, larger, to an
    invalid request).  The cycle equals the oracle on the resized snapshot and an engine that re-upserted those asks with
    their other fields unchanged: priority and create_seq are kept"""
    from yunikorn_k8shim_b200 import Engine
    rng = np.random.default_rng(11)
    s = synth.perf(40, 6, 30, seed=7)
    s.ask_prio[:] = rng.integers(-1, 2, s.n_asks) * 10
    s.node_avail //= 16
    pick = np.sort(rng.permutation(s.n_asks)[:25])
    req = s.ask_req[pick].copy()
    req[:8, 0] //= 2
    req[8:16, 0] *= 2
    req[16, :] = 0
    req[17, 1] = -1
    t = copy.deepcopy(s)
    t.ask_req[pick] = req
    want = oracle.run(t)
    assert (want["state"] == ST_NOFIT).any() and want["state"][pick[16]] == ST_INVALID
    outs = []
    for how in ("resize", "upsert"):
        with Engine.for_snapshot(s, commit=commit, batch=64) as e:
            if how == "resize":
                e.asks_resize(pick, req)
            else:
                e.asks_upsert(pick, req, s.ask_app[pick], s.ask_create[pick], s.ask_tol[pick], s.ask_need[pick], s.ask_deny[pick],
                              s.ask_prio[pick], s.ask_node[pick], s.ask_flags[pick], s.ask_gang[pick])
            ask, node, _ = e.cycle(s.n_asks)
            assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"]), how
            outs.append((ask, node, e.nodes_available(np.arange(s.n_nodes)), e.ask_states(np.arange(s.n_asks))))
    for x, y in zip(*outs):
        assert np.array_equal(x, y)
    assert np.array_equal(outs[0][3], want["state"])


def _apply(t, bound, idx, req):
    """a resize on the expectation's snapshot: requests, and the bound node's available for allocations"""
    for a, r in zip(idx, req):
        a = int(a)
        if a in bound:
            t.node_avail[bound[a]] -= r - t.ask_req[a]
        t.ask_req[a] = r


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_filter_follows_a_resize(oracle, commit):
    """yk_filter_nodes after resizes of pending asks (larger, smaller, not positive) and of allocations (their nodes' room
    moves): candidates and counts equal the oracle's on the resized state, both phases"""
    rng = np.random.default_rng(13)
    s = synth.perf(300, 16, 40, masks=True, seed=3)
    s.node_avail[:, :2] //= 30                          # 74 of the 640 asks stay unplaced
    e, t, bound, want = tpn.scenario(oracle, s, commit, extra=0)
    with e:
        pend = np.sort(rng.permutation(np.nonzero(want["state"] != ST_ALLOCATED)[0])[:12])
        preq = t.ask_req[pend].copy()
        preq[:4, 0] *= 3
        preq[4:8, 0] //= 2
        preq[8] = 0
        preq[9, 0] = -5
        alloc = np.sort(rng.permutation(np.asarray(want["ask"]))[:30])
        areq = t.ask_req[alloc] * rng.integers(0, 4, (len(alloc), 1))
        idx, req = np.concatenate([pend, alloc]), np.vstack([preq, areq])
        e.asks_resize(idx, req)
        _apply(t, bound, idx, req)
        assert np.array_equal(e.nodes_available(np.arange(t.n_nodes)), t.node_avail)
        asks = np.concatenate([pend, alloc[:6], np.arange(0, t.n_asks, 41)])
        for allocate in (True, False):
            nodes, n_pass, counts = e.filter_nodes(asks, k=16, skip=2, allocate=allocate)
            full, want_counts = filter_expect(oracle, t, asks, allocate)
            assert np.array_equal(counts, want_counts), allocate
            for i in range(len(asks)):
                assert n_pass[i] == len(full[i]) and nodes[i].tolist() == window(full[i], 2, 16), (allocate, int(asks[i]))


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_preemption_nodes_after_victims_resize(oracle, commit):
    """victims resized up (some over their node's capacity), down and to zero on one resource: every victim frees its new
    request.  yk_preemption_nodes equals the oracle's expectation on the resized state and yk_preemption_search given the
    new requests"""
    rng = np.random.default_rng(17)
    s = tpn._fuzz(4)
    e, t, bound, want = tpn.scenario(oracle, s, commit, extra=3)
    with e:
        asks = tpn.preemptors(e, t, want, rng)
        alloc = np.asarray(want["ask"])
        vic = np.sort(rng.permutation(alloc)[:max(1, len(alloc) // 3)])
        req = t.ask_req[vic].copy()
        third = len(vic) // 3
        req[:third, 0] = req[:third, 0] * 2 + 1000
        req[third:2 * third] //= 2
        req[2 * third:, 1] = 0
        e.asks_resize(vic, req)
        _apply(t, bound, vic, req)
        lists = tpn.random_lists(rng, alloc, len(asks))
        lists[0] = vic[:min(len(vic), 40)].astype(np.uint32)
        pairs = tpn.expect(oracle, t, bound, asks, lists)
        tpn.check(e, t, pairs, asks, lists)
        q = [(int(a), n, t.ask_req[vs]) for a, p in zip(asks, pairs) for n, vs, _ in p]
        assert q
        got = e.preemption_search([x[0] for x in q], [x[1] for x in q], [x[2] for x in q], [0] * len(q))
        assert got.tolist() == [ans for p in pairs for _, _, ans in p]


# ---- GPU: 5. errors ----
@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_errors_leave_the_engine_as_it_was(oracle, commit):
    """every error: the same code, no counter moved, and scores, states, availability and the next cycle as on an engine that
    never got the call.  An unchanged vector and n == 0 are YK_OK and change nothing either"""
    from yunikorn_k8shim_b200 import YkError
    s = synth.perf(300, 8, 40, masks=True)
    a, b = tns._pair(s, commit=commit)
    with a, b:
        nofit, too_big = np.arange(s.n_asks + 120, s.n_asks + 123), s.node_total.max(axis=0) + 1   # they stay pending
        for e in (a, b):
            e.asks_upsert(nofit, np.tile(too_big, (3, 1)), np.zeros(3, np.int32), 10 ** 9 + nofit,
                          tolerated_bits=np.full(3, ~np.uint64(0)))
        ask = tns._cycle_same(a, b, "first cycle")[0]
        states = a.ask_states(np.arange(s.n_asks + tns.EXTRA_ASKS))
        pend = [int(x) for x in np.nonzero((states != ST_ALLOCATED) & (states != 255))[0]]
        big = int(ask[-1])                              # its leaf (and the root) hold other allocations: INT64_MAX overflows
        alloc = [int(x) for x in ask if x != big]
        assert sum(s.app_queue[s.ask_app[x]] == s.app_queue[s.ask_app[big]] for x in alloc) > 0 and len(pend) >= 2
        absent = s.n_asks + tns.EXTRA_ASKS - 1
        D = s.D
        r = lambda x: (s.ask_req[x] if x < s.n_asks else too_big).copy()   # noqa: E731
        neg = r(alloc[0])
        neg[1] = -1
        huge = r(big)
        huge[0] = INT64_MAX
        bad = [("index beyond max_asks", [s.n_asks + tns.EXTRA_ASKS], [r(0)], YK_ERR_ARG),
               ("same ask twice", [alloc[0], pend[0], alloc[0]], [r(0)] * 3, YK_ERR_ARG),
               ("negative for an allocation", [pend[0], alloc[0]], [r(pend[0]) * 2, neg], YK_ERR_ARG),
               ("absent ask", [alloc[1], absent], [r(alloc[1]) * 2, r(0)], YK_ERR_STATE),
               ("queue sum overflows", [big], [huge], YK_ERR_RANGE),
               ("overflow after an applied one", [alloc[2], pend[0], big], [r(alloc[2]) * 3, r(pend[0]) // 2, huge], YK_ERR_RANGE)]
        for k, (tag, idx, req, code) in enumerate(bad):
            before = a.stats()
            with pytest.raises(YkError) as ei:
                a.asks_resize(idx, np.stack(req))
            assert ei.value.code == code, tag
            assert a.stats() == before, tag
            tns._same(a, b, s, s.n_nodes, tag)
            tns._more_asks((a, b), s, k, k)
            tns._cycle_same(a, b, tag)
            tns._same(a, b, s, s.n_nodes, tag)
        # null arrays and a null engine, through the library itself
        one, vec = np.array([alloc[0]], np.uint32), np.ascontiguousarray(r(alloc[0]))
        assert a._lib.yk_asks_resize(a._h, C.c_uint32(1), None, vec.ctypes.data_as(C.c_void_p)) == YK_ERR_ARG
        assert a._lib.yk_asks_resize(a._h, C.c_uint32(1), one.ctypes.data_as(C.c_void_p), None) == YK_ERR_ARG
        assert a._lib.yk_asks_resize(None, C.c_uint32(1), one.ctypes.data_as(C.c_void_p), vec.ctypes.data_as(C.c_void_p)) == YK_ERR_ARG
        tns._same(a, b, s, s.n_nodes, "null")
        # n == 0, and the current vectors again (pending and allocated): YK_OK, nothing moves, the next cycle is the same
        for k, (idx, req) in enumerate((([], np.zeros((0, D), np.int64)),
                                         ([alloc[3], pend[1]], np.stack([r(alloc[3]), r(pend[1])])))):
            before = a.stats()
            a.asks_resize(idx, req)
            assert a.stats() == before
            tns._same(a, b, s, s.n_nodes, f"unchanged {k}")
            tns._more_asks((a, b), s, len(bad) + k, k)
            tns._cycle_same(a, b, f"unchanged {k}")
            tns._same(a, b, s, s.n_nodes, f"unchanged {k}")


# ---- GPU: 6. the reference's pod resource scaling scenario ----
def _pod(cpu, mem, status=None, infeasible=False):
    """one container requesting cpu / mem; status = the requests the kubelet reports as applied (None: as the spec)"""
    st = status or (cpu, mem)
    return {"containers": [{"name": "c", "requests": {"cpu": cpu, "memory": mem}}],
            "statuses": [{"name": "c", "allocated": None, "resources": {"cpu": st[0], "memory": st[1]}}],
            "resizeInfeasible": infeasible}


def _pod_vector(pod):
    """yk_podspec_vector of the pod on the dimensions vcore, memory: the request the adapter sends"""
    from yunikorn_k8shim_b200 import podres
    lib = podres._lib()
    h = C.c_void_p(lib.yk_podspec_new())
    try:
        c = pod["containers"][0]
        ci = podres._ck(lib, lib.yk_podspec_container(h, c["name"].encode(), C.c_uint32(podres.CONTAINER)))
        for res, q in c["requests"].items():
            podres._ck(lib, lib.yk_podspec_quantity(h, C.c_uint32(podres.LIST_REQUESTS), C.c_int32(ci), res.encode(), q.encode()))
        st = pod["statuses"][0]
        podres._ck(lib, lib.yk_podspec_status(h, st["name"].encode(), C.c_int32(1)))
        for res, q in st["resources"].items():
            podres._ck(lib, lib.yk_podspec_quantity(h, C.c_uint32(podres.LIST_STATUS_REQUESTS), C.c_int32(ci), res.encode(), q.encode()))
        podres._ck(lib, lib.yk_podspec_resize_infeasible(h, C.c_int32(1 if pod["resizeInfeasible"] else 0)))
        podres._ck(lib, lib.yk_podspec_compute(h))
        names = (C.c_char_p * 2)(b"vcore", b"memory")
        out, unmapped = np.zeros(2, np.int64), C.c_uint32(0)
        podres._ck(lib, lib.yk_podspec_vector(h, C.c_uint32(2), names, out.ctypes.data_as(C.c_void_p), C.byref(unmapped)))
        return out
    finally:
        lib.yk_podspec_free(h)


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_reference_pod_resource_scaling_scenario(commit):
    """test/e2e/pod_resource_scaling/pod_resource_scaling_test.go, restated on the engine: a 100m / 100Mi pod is bound; it
    is resized up (cpu, then memory), down, and then beyond what the node can give, which the kubelet marks infeasible.
    After each step the node's available, the leaf queue's allocation (probed against its max: an ask of exactly the
    headroom is placed, one unit more on either resource is SKIPPED) and the application's allocation (the fair leaf puts
    the application holding less first) follow the vector GetPodResource reports; the infeasible resize changes nothing"""
    from yunikorn_k8shim_b200 import Engine
    total = np.array([8000, 16 * GI])
    mx = np.array([4000, 4 * GI])
    other = np.array([150, 150 * MI])                        # application 1's pod, for the fair order
    with Engine(D=2, max_nodes=1, max_asks=16, max_apps=2, max_queues=2, commit=commit) as e:
        e.queues_set([-1, 0], max=np.stack([[-1, -1], mx]), sort=[0, 1])
        e.apps_upsert([0, 1], [1, 1], [1, 2])
        e.nodes_upsert([0], [total], [total], name_rank=[1], flags=[synth.NODE_SCHEDULABLE])
        seq = iter(range(10, 10 ** 6))
        v = _pod_vector(_pod("100m", "100Mi"))
        assert v.tolist() == [100, 100 * MI]
        e.asks_upsert([0, 1], np.stack([v, other]), [0, 1], [next(seq), next(seq)])
        ask, _, _ = e.cycle(16)
        assert sorted(ask.tolist()) == [0, 1]

        def probe(v):
            assert e.nodes_available([0]).tolist() == [(total - v - other).tolist()]
            h = mx - v - other
            e.asks_upsert([5], [h + [1, 0]], [1], [next(seq)])
            for over in (h + [1, 0], h + [0, 1], h):
                e.asks_resize([5], [over])
                e.cycle(16)
                assert e.ask_states([5])[0] == (ST_ALLOCATED if (over == h).all() else ST_SKIPPED), over
            e.release([5])
            e.asks_upsert([6, 7], np.stack([[10, MI]] * 2), [0, 1], [next(seq), next(seq)])
            ask, _, _ = e.cycle(16)
            e.release(ask)
            return ask.tolist()

        def step(pod, first_app):
            w = _pod_vector(pod)
            before = e.stats()
            e.asks_resize([0], [w])
            assert e.stats() == before
            assert probe(w) == ([6, 7] if first_app == 0 else [7, 6]), (pod, w)
            return w

        assert probe(v) == [6, 7]                                     # 100Mi < 150Mi: application 0 first
        v = step(_pod("200m", "100Mi"), 0)
        assert v.tolist() == [200, 100 * MI]
        v = step(_pod("200m", "200Mi"), 1)                            # 200Mi > 150Mi: application 1 first
        v = step(_pod("100m", "100Mi"), 0)
        w = step(_pod("100", "100Gi", status=("100m", "100Mi"), infeasible=True), 0)
        assert np.array_equal(w, v)                                    # the status requests: nothing changed
        e.release([0])
        assert e.nodes_available([0]).tolist() == [(total - other).tolist()]


# ---- CPU: 7. the resized sessions on their own ----
@pytest.mark.parametrize("seed,D,policy", RESIZED, ids=RESIZED_IDS)
def test_resized_sessions_oracles_agree(seed, D, policy):
    """every cycle's snapshot: the C++ and the Python oracle agree"""
    m = session(seed, D, policy)
    ts._oracles_agree(m)
    assert any(st[0] == "op" and st[1] == "asks_resize" for st in m.steps), m.name


@pytest.mark.parametrize("name", sorted(TARGETED))
def test_targeted_resize_scripts(oracle, name):
    """each script has the shape it is meant to exercise (asserted inside), conserves its accounting and both oracles agree"""
    m = TARGETED[name](oracle)
    m.check_conservation()
    ts._oracles_agree(m)


def test_resize_conserves_the_model():
    """the sessions check the model's accounting before and after every cycle, resizes included (resized_session), and
    end with a full release that brings every present node back to total - foreign (ts.finish)"""
    for args in RESIZED:
        m = session(*args)
        m.check_conservation()
        assert any(st[0] == "conserved" for st in m.steps), m.name


def test_sessions_cover_every_resize():
    """the resized sessions make every kind of resize, and reach every over-committed state, a stated number of times"""
    total, calls = {}, 0
    for args in RESIZED:
        m = session(*args)
        for k, v in m.count.items():
            total[k] = total.get(k, 0) + v
        calls += sum(1 for st in m.steps if st[0] == "op" and st[1] == "asks_resize")
    need = {f"resize_{k}": 40 for k in KINDS}
    need.update({"resize_user_over_limit": 30, "resize_gang_apart": 20, "resize_gang_back": 10, "resize_call_of_many": 200,
                 "resize_call_mixed": 100, "state_node_overcommitted": 100, "state_queue_over_max": 80,
                 "state_user_over_limit": 60, "state_pending_invalid": 80, "release_on_removed_node": 50})
    short = {k: (total.get(k, 0), n) for k, n in need.items() if total.get(k, 0) < n}
    assert not short, short
    assert calls >= 300, calls
