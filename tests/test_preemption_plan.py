"""yk_preemption_plan: preemption for queues below their guarantee (DESIGN.md §2 item 9).

The expectation comes from tests/preemption_oracle.py, a plain-Python restatement of the rules that never calls the engine.
The reference's end-to-end scenarios (test/e2e/preemption/preemption_test.go and deployments/examples/preemption) are written
here as data: queue trees, pod sizes and the pods running after each step.  The CPU tests run them on the oracle alone, with
a one-node cycle stand-in; the GPU tests run the same sessions through the engine's C ABI and check every plan against the
oracle and every count against the data."""
import copy

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
import preemption_oracle as po

YK_NONE = 0xFFFFFFFF
D4 = 4                         # vcore (milli), memory, pods, ephemeral storage
NO_SELF, NO_OTHER, ORIGINATOR = 2, 4, 8


# ---- scenarios as data: queues (name, parent, guaranteed {vcore, memory}, max, priority.offset, preemption fence) ----
def Q(name, parent, guar=None, mx=None, off=0, fence=False):
    return dict(name=name, parent=parent, guar=guar, max=mx, off=off, fence=fence)


M = 1000                       # one e2e sleep pod's memory
BASIC = dict(node=(100_000, 3 * M + M // 2), queues=[Q("root", None), Q("sandbox1", "root", (-1, M)), Q("sandbox2", "root", (-1, M))])
BELOW = dict(node=(100_000, 3 * M + M // 2), queues=[Q("root", None), Q("sandbox1", "root", (-1, 3 * M + M // 2)),
                                                      Q("sandbox2", "root", (-1, 3 * M + M // 2))])
FENCE = dict(node=(100_000, 3 * M + M // 2), queues=[Q("root", None), Q("sandbox1", "root", (-1, M)),
                                                      Q("sandbox2", "root", (-1, M), fence=True)])
PRIO = dict(node=(100_000, 10 * M), queues=[Q("root", None), Q("parent", "root", mx=(-1, 3 * M)),
                                            Q("high-priority", "parent", (-1, M), off=100), Q("sandbox1", "parent", (-1, M)),
                                            Q("low-priority", "parent", (-1, M), off=-100)])
ALLOW = dict(node=(100_000, 4 * M + M // 2), queues=[Q("root", None), Q("sandbox3", "root", (-1, M)), Q("sandbox4", "root", (-1, M)),
                                                      Q("sandbox5", "root", (-1, M))])
EXAMPLE = dict(node=(8000, 8000), queues=[
    Q("root", None), Q("sandbox", "root", mx=(1000, 1000)), Q("tenants", "sandbox", fence=True),
    Q("tenant-normal", "tenants", (300, 300), off=0), Q("tenant-high", "tenants", (300, 300), off=1000),
    Q("tenant-low", "tenants", off=-1000), Q("system", "sandbox"), Q("system-low", "system", off=-9999)])


class Session:
    """One scenario: the oracle's World, and with engine=True the engine driven through the same calls.  pods are declared
    up front ([(queue, vcore, memory, flags)]); `add` makes them present as pending asks in declaration order."""

    def __init__(self, sc, pods, engine=False, **ekw):
        self.names = [q["name"] for q in sc["queues"]]
        Qn = len(self.names)
        par = np.array([-1 if q["parent"] is None else self.names.index(q["parent"]) for q in sc["queues"]], dtype=np.int32)
        guar = np.full((Qn, D4), -1, dtype=np.int64)
        mx = np.full((Qn, D4), -1, dtype=np.int64)
        for i, q in enumerate(sc["queues"]):
            for k, v in enumerate(q["guar"] or ()):
                guar[i, k] = v
            for k, v in enumerate(q["max"] or ()):
                mx[i, k] = v
        req = np.array([[vc, mem, 1, 0] for (_, vc, mem, _) in pods], dtype=np.int64)
        app = np.array([self.names.index(q) for (q, _, _, _) in pods], dtype=np.int32)
        A = len(pods)
        node = np.array([[sc["node"][0], sc["node"][1], 110, 0]], dtype=np.int64)
        self.s = synth._finish("preempt", D4, 0, node, node.copy(), np.zeros(1, np.uint64), np.zeros(1, np.uint64), ["node-a"],
                               (par, guar, mx, np.zeros((Qn, D4), dtype=np.int64), np.zeros(Qn, dtype=np.uint8)),
                               np.arange(Qn, dtype=np.int32), app, req, np.zeros(A, np.uint64), np.zeros(A, np.uint64),
                               np.zeros(A, np.uint64), ask_flags=np.array([f for (_, _, _, f) in pods], dtype=np.uint32))
        self.s.q_prio_offset = np.array([q["off"] for q in sc["queues"]], dtype=np.int32)
        self.s.q_pp_fence = np.array([q["fence"] for q in sc["queues"]], dtype=np.uint8)
        self.w = po.World(self.s, {}, np.full(A, 255), self.s.node_avail)
        self.e = None
        if engine:
            from yunikorn_k8shim_b200 import Engine
            s = self.s
            self.e = Engine(D=D4, max_nodes=1, max_asks=A, max_apps=Qn, max_queues=Qn, **ekw)
            self.e.queues_set(s.q_parent, s.q_guaranteed, s.q_max, s.q_alloc, s.q_sort)
            self.e.queues_priority(s.q_prio_offset)
            self.e.queues_preemption(s.q_pp_fence)
            self.e.nodes_upsert([0], s.node_total, s.node_avail, name_rank=[0])
            self.e.apps_upsert(np.arange(Qn), np.arange(Qn), s.app_submit)

    def add(self, idx):
        idx = np.asarray(idx)
        if self.e is not None:
            s = self.s
            self.e.asks_upsert(idx, s.ask_req[idx], s.ask_app[idx], s.ask_create[idx], flags=s.ask_flags[idx])
        for a in idx:
            self.w.state[int(a)] = 0
            self.w.plans.pop(int(a), None)

    def cycle(self):
        w = self.w
        pend = sorted(a for a, st in w.state.items() if st not in (po.ST_ALLOCATED, 255))
        if self.e is not None:
            ask, node, _ = self.e.cycle(len(pend) + 1)
            for a, n in zip(ask, node):
                w.allocate(int(a), int(n))
            st = self.e.ask_states(pend) if pend else []
            for a, x in zip(pend, st):
                w.state[a] = int(x)
            return
        # one-node stand-in: planned preemptors first (the caller pins them there), then declaration order; headroom before fit
        for a in sorted(pend, key=lambda a: (a not in w.plans, a)):
            r, L = w.req[a], w.leaf(a)
            if any(w.qmax[q][k] >= 0 and w.alloc[q][k] + r[k] > w.qmax[q][k] for q in w.path(L) for k in range(D4)):
                w.state[a] = po.ST_SKIPPED
            elif any(r[k] > max(0, w.avail[0][k]) for k in range(D4)):
                w.state[a] = po.ST_NOFIT
            else:
                w.allocate(a, 0)

    def plan(self, idx, cap=None):
        want = po.plan(self.w, idx) if cap is None else None
        if self.e is not None:
            st, node, vic, done = self.e.preemption_plan(idx, victims_cap=cap)
            if want is not None:
                got = [(int(x), None if n == YK_NONE else int(n), [int(v) for v in vs]) for x, n, vs in zip(st, node, vic)]
                assert done == len(idx) and got == want, (got, want)
            return st, node, vic, done
        return want

    def release(self, idx):
        if self.e is not None:
            self.e.release(np.asarray(idx, dtype=np.uint32))
        self.w.release([int(a) for a in idx])

    def running(self):
        out = {}
        for a in self.w.bound:
            q = self.names[self.w.leaf(a)]
            out[q] = out.get(q, 0) + 1
        if self.e is not None:   # the engine agrees on what is allocated
            st = self.e.ask_states(np.arange(len(self.s.ask_app)))
            assert sorted(np.nonzero(st == po.ST_ALLOCATED)[0].tolist()) == sorted(self.w.bound)
        return out


def _plans(r):
    """(status, node, victims) per ask from either side"""
    if isinstance(r, list):
        return r
    st, node, vic, _ = r
    return [(int(x), None if n == YK_NONE else int(n), [int(v) for v in vs]) for x, n, vs in zip(st, node, vic)]


def run_basic(engine, **kw):
    pods = [("sandbox1", 100, M, 0)] * 3 + [("sandbox2", 100, M, 0)]
    ss = Session(BASIC, pods, engine, **kw)
    ss.add([0, 1, 2]); ss.cycle()
    ss.add([3]); ss.cycle()
    assert ss.w.state[3] == po.ST_NOFIT
    (st, node, vic), = _plans(ss.plan([3]))
    assert st == po.PLANNED and node == 0 and len(vic) == 1 and ss.w.leaf(vic[0]) == 1
    ss.release(vic); ss.cycle()
    assert ss.running() == {"sandbox1": 2, "sandbox2": 1}


def run_below_guarantee(engine, **kw):
    pods = [("sandbox1", 100, M, 0)] * 3 + [("sandbox2", 100, M, 0)]
    ss = Session(BELOW, pods, engine, **kw)
    ss.add([0, 1, 2]); ss.cycle(); ss.add([3]); ss.cycle()
    assert [p[0] for p in _plans(ss.plan([3]))] == [po.NO_VICTIMS]
    assert ss.running() == {"sandbox1": 3}


def run_fence(engine, **kw):
    pods = [("sandbox1", 100, M, 0)] * 3 + [("sandbox2", 100, M, 0)]
    ss = Session(FENCE, pods, engine, **kw)
    ss.add([0, 1, 2]); ss.cycle(); ss.add([3]); ss.cycle()
    assert [p[0] for p in _plans(ss.plan([3]))] == [po.NO_VICTIMS]


def run_priority_queue(engine, **kw):
    pods = [("sandbox1", 100, M, 0)] * 3 + [("low-priority", 100, M, 0), ("high-priority", 100, M, 0)]
    ss = Session(PRIO, pods, engine, **kw)
    ss.add([0, 1, 2]); ss.cycle(); ss.add([3, 4]); ss.cycle()
    assert ss.w.state[3] == ss.w.state[4] == po.ST_SKIPPED
    low, high = _plans(ss.plan([3, 4]))
    assert low == (po.NO_VICTIMS, None, [])
    assert high[0] == po.PLANNED and len(high[2]) == 1 and ss.names[ss.w.leaf(high[2][0])] == "sandbox1"   # headroom only
    ss.release(high[2]); ss.cycle()
    assert ss.running() == {"sandbox1": 2, "high-priority": 1}


def run_allow_preemption(engine, **kw):
    pods = [("sandbox3", 100, M, 0)] * 2 + [("sandbox4", 100, M, NO_SELF)] * 2 + [("sandbox5", 100, M, 0)]
    ss = Session(ALLOW, pods, engine, **kw)
    ss.add([0, 1, 2, 3]); ss.cycle(); ss.add([4]); ss.cycle()
    (st, _, vic), = _plans(ss.plan([4]))
    assert st == po.PLANNED and [ss.names[ss.w.leaf(v)] for v in vic] == ["sandbox3"]
    ss.release(vic); ss.cycle()
    assert ss.running() == {"sandbox3": 1, "sandbox4": 2, "sandbox5": 1}


def run_example(engine, **kw):
    pods = ([("system-low", 100, 100, 0)] * 5 + [("tenant-low", 100, 100, 0)] * 5 + [("tenant-normal", 100, 100, 0)] * 5
            + [("tenant-high", 100, 100, 0)] * 5)
    ss = Session(EXAMPLE, pods, engine, **kw)
    ss.add(range(10)); ss.cycle()
    assert ss.running() == {"system-low": 5, "tenant-low": 5}
    ss.add(range(10, 15)); ss.cycle()
    r = _plans(ss.plan(list(range(10, 15))))
    assert [x[0] for x in r] == [po.PLANNED] * 3 + [po.GUARANTEE] * 2
    assert all(ss.names[ss.w.leaf(v)] == "tenant-low" for x in r for v in x[2])
    ss.release([v for x in r for v in x[2]]); ss.cycle()
    assert ss.running() == {"system-low": 5, "tenant-low": 2, "tenant-normal": 3}
    ss.release([a for a in list(ss.w.bound) if ss.names[ss.w.leaf(a)] == "tenant-low"]); ss.cycle()
    assert ss.running() == {"system-low": 5, "tenant-normal": 5}
    ss.add(range(15, 20)); ss.cycle()
    r = _plans(ss.plan(list(range(15, 20))))
    assert [x[0] for x in r] == [po.PLANNED] * 2 + [po.NO_VICTIMS] * 3
    ss.release([v for x in r for v in x[2]]); ss.cycle()
    assert ss.running() == {"system-low": 5, "tenant-normal": 3, "tenant-high": 2}


SCENARIOS = [run_basic, run_below_guarantee, run_fence, run_priority_queue, run_allow_preemption, run_example]


@pytest.mark.parametrize("scenario", SCENARIOS, ids=lambda f: f.__name__[4:])
def test_reference_scenarios_on_the_oracle(scenario):
    scenario(False)


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["auto", "host", "device"])
@pytest.mark.parametrize("scenario", SCENARIOS, ids=lambda f: f.__name__[4:])
def test_reference_scenarios(scenario, commit):
    scenario(True, commit=commit)


# ---- fuzz against the oracle ----
# Queue tree of every fuzz cluster: root(0) -> p1(1) -> {pre1(3), v4(4), v5(5)}, root -> p2(2) -> {v6(6), pre2(7)}.  Victim leaves
# v4..v6 fill ~90 % of the cluster with guarantees well below what they hold; the preemptor leaves are far below their
# guarantee and ask more than any node has left, so most plans need victims on the node; p1 often has a max just above its
# load, so pre1's plans also need headroom victims under p1, which sit on other nodes.
PARENT = [-1, 0, 0, 1, 1, 1, 2, 2]
VICTIM_LEAVES, PRE_LEAVES = (4, 5, 6), (3, 7)


def fuzz_cluster(seed, D, policy):
    """-> (snapshot of every ask, n1): asks [0, n1) are the victims' pods (phase 1), the rest the preemptors (phase 2)"""
    rng = np.random.default_rng(seed)
    N = 4 + seed % 5
    Qn = len(PARENT)
    tot = np.tile([8000, 16000, 110, 0], (N, 1)).astype(np.int64)
    cap = tot[:, :2].sum(axis=0)
    vic_req, vic_app = [], []
    load = np.zeros(2, dtype=np.int64)
    while True:
        c = int(rng.choice([500, 1000, 1500]))
        r = np.array([c, 2 * c, 1, 0])
        if (load + r[:2] > 0.9 * cap).any():
            break
        load += r[:2]
        vic_req.append(r)
        vic_app.append(int(rng.choice(VICTIM_LEAVES)))
    n1 = len(vic_req)
    n2 = int(rng.integers(6, 14))
    pre_req = [np.array([c, 2 * c, 1, 0]) for c in rng.choice([1000, 2000, 3000], n2)]
    pre_app = [int(rng.choice(PRE_LEAVES)) for _ in range(n2)]
    req = np.array(vic_req + pre_req, dtype=np.int64)
    app = np.array(vic_app + pre_app, dtype=np.int32)   # application i lives in queue i
    A = n1 + n2
    guar = np.full((Qn, 4), -1, dtype=np.int64)
    mx = np.full((Qn, 4), -1, dtype=np.int64)
    for q in VICTIM_LEAVES:
        held = req[:n1][app[:n1] == q, :2].sum(axis=0)
        if rng.random() < 0.85:
            guar[q, :2] = (held * rng.uniform(0.05, 0.4)).astype(np.int64)
    for q in PRE_LEAVES:
        guar[q, :2] = (cap * rng.uniform(0.2, 0.4)).astype(np.int64)
    if rng.random() < 0.3:
        guar[1, :2] = (cap * 0.3).astype(np.int64)
    if rng.random() < 0.6:   # p1's max just above what its victim leaves hold: pre1 needs headroom victims
        held = req[:n1][(app[:n1] == 4) | (app[:n1] == 5), :2].sum(axis=0)
        mx[1, 0] = int(held[0] + rng.integers(0, 1500))
    prio = np.concatenate([rng.choice([-5, 0, 5], n1), rng.choice([0, 5, 10], n2)]).astype(np.int32)
    flags = np.concatenate([rng.choice([0, NO_SELF, ORIGINATOR, NO_SELF | ORIGINATOR], n1, p=[0.6, 0.15, 0.15, 0.1]),
                            rng.choice([0, NO_OTHER], n2, p=[0.9, 0.1])]).astype(np.uint32)
    create = rng.permutation(A).astype(np.int64)
    ids = [f"n{int(x):03d}" for x in rng.permutation(N)]
    Db = 8 if D == 8 else 4          # D = 8: four more small resources on every pod; D = 1: the first column of D = 4
    if Db == 8:
        tot = np.hstack([tot, np.full((N, 4), 4000, np.int64)])
        req = np.hstack([req, rng.integers(1, 4, (A, 4))]).astype(np.int64)
        guar = np.hstack([guar, np.full((Qn, 4), -1, np.int64)])
        mx = np.hstack([mx, np.full((Qn, 4), -1, np.int64)])

    def snap(sel, avail, qalloc):
        sel = np.asarray(sel)
        t = synth._finish(f"plan-fuzz-{seed}", Db, policy, tot, avail, np.zeros(N, np.uint64), np.zeros(N, np.uint64), ids,
                          (np.array(PARENT, dtype=np.int32), guar.copy(), mx.copy(), qalloc, np.zeros(Qn, np.uint8)),
                          np.arange(Qn, dtype=np.int32), app[sel], req[sel], np.zeros(len(sel), np.uint64),
                          np.zeros(len(sel), np.uint64), np.zeros(len(sel), np.uint64), ask_prio=prio[sel],
                          ask_flags=flags[sel], ask_create=create[sel])
        t.q_prio_offset = np.array([0, rng.choice([-10, 0, 10]), 0, 0, 0, 0, 0, 0], dtype=np.int32)
        t.q_prio_offset[3:] = rng.choice([-10, 0, 10], Qn - 3)
        t.q_pp_fence = (np.arange(Qn) == 2) & (rng.random() < 0.25)
        if D == 1:
            t = synth.redim(t, 1, seed)
        return t
    full = snap(np.arange(A), tot.copy(), np.zeros((Qn, Db), np.int64))
    return full, n1


def fuzz_world(seed, D, policy):
    """the cluster after phase 1 (victims) and phase 2 (preemptors, blocked), on the oracle alone -> (full, n1, want1, want2,
    World)"""
    from oracle import py_oracle
    full, n1 = fuzz_cluster(seed, D, policy)
    A = full.n_asks
    s1 = copy.deepcopy(full)
    for f in ("ask_app", "ask_req", "ask_tol", "ask_need", "ask_deny", "ask_prio", "ask_create", "ask_node", "ask_flags", "ask_gang"):
        setattr(s1, f, getattr(full, f)[:n1])
    want1 = py_oracle.run(s1)
    s2 = copy.deepcopy(full)
    for f in ("ask_app", "ask_req", "ask_tol", "ask_need", "ask_deny", "ask_prio", "ask_create", "ask_node", "ask_flags", "ask_gang"):
        setattr(s2, f, getattr(full, f)[n1:])
    s2.node_avail = np.ascontiguousarray(want1["avail"], dtype=np.int64)
    qa = np.zeros_like(full.q_alloc)
    for a in want1["ask"]:
        q = int(full.app_queue[int(full.ask_app[a])])
        while q >= 0:
            qa[q] += full.ask_req[a]
            q = int(full.q_parent[q]) if q else -1
    s2.q_alloc = qa
    want2 = py_oracle.run(s2)
    bound = {int(a): int(n) for a, n in zip(want1["ask"], want1["node"])}
    bound.update({int(a) + n1: int(n) for a, n in zip(want2["ask"], want2["node"])})
    state = np.full(A, 255)
    state[n1:] = want2["state"]
    state[list(bound)] = po.ST_ALLOCATED
    w = po.World(full, bound, state, want2["avail"])
    return full, n1, want1, want2, w


def fuzz_rounds(w, n1, A, plan_fn, on_release, on_remove, info=None):
    """round 1 plans the first half of the blocked preemptors, round 2 all of them (seeing round 1's marks and plans) after
    half of round 1's victims are released and one plan is removed.  plan_fn(order) -> [(status, node, victims)]"""
    blocked = [a for a in range(n1, A) if w.state[a] in (po.ST_NOFIT, po.ST_SKIPPED)]
    rounds = [blocked[: (len(blocked) + 1) // 2], blocked + [a for a in range(0, n1, 5)][:3]]
    out = []
    for rnd, order in enumerate(rounds):
        got = plan_fn(order, rnd)
        out.append(got)
        if rnd:
            break
        victims = [v for x in got for v in x[2]]
        if victims:
            on_release(victims[: (len(victims) + 1) // 2])
        planned = [a for a, x in zip(order, got) if x[0] == po.PLANNED]
        if len(planned) > 1:
            on_remove([planned[0]])
    return out


def oracle_rounds(w, n1, A):
    info = []

    def plan_fn(order, rnd):
        inf = []
        r = po.plan(w, order, inf)
        for x in inf:
            x["round"] = rnd
        info.extend(inf)
        return r
    fuzz_rounds(w, n1, A, plan_fn, w.release, w.remove)
    return info


def test_fuzz_coverage_floors():
    """the fuzz clusters reach every part of the plan: for each D and node sort over the 20 seeds, plans, plans that need
    victims on their node, headroom victims on other nodes, plans in the second call (after marks, releases and a removed
    plan) and plans that follow an earlier plan of the same call"""
    for D in (1, 4, 8):
        for policy in (0, 1):
            info = []
            for seed in range(20):
                full, n1, _, _, w = fuzz_world(seed, D, policy)
                info += oracle_rounds(w, n1, full.n_asks)
            counts = dict(planned=len(info), need=sum(1 for x in info if x["need"] > 0),
                          off_node=sum(1 for x in info if x["off_node"] > 0), round2=sum(1 for x in info if x["round"] == 1),
                          after_plan=sum(1 for x in info if x["after_plan"]))
            floors = dict(planned=60, need=40, off_node=3, round2=15, after_plan=30)
            assert all(counts[k] >= floors[k] for k in floors), (D, policy, counts)


def fuzz_session(seed, D, policy, commit, batch):
    """phase 1 and 2 on the engine (same bindings as the oracle), then the two plan calls: every answer equals the oracle's"""
    from yunikorn_k8shim_b200 import Engine
    full, n1, want1, want2, w = fuzz_world(seed, D, policy)
    A = full.n_asks
    e = Engine(D=full.D, policy=policy, weights=full.weights, max_nodes=full.n_nodes, max_asks=A, max_apps=full.n_apps,
               max_queues=full.n_queues, commit=commit, batch=batch)
    e.queues_set(full.q_parent, full.q_guaranteed, full.q_max, full.q_alloc, full.q_sort)
    e.queues_priority(full.q_prio_offset)
    e.queues_preemption(full.q_pp_fence)
    e.nodes_upsert(np.arange(full.n_nodes), full.node_total, full.node_avail, name_rank=full.node_rank())
    e.apps_upsert(np.arange(full.n_apps), full.app_queue, full.app_submit)

    def upsert(lo, hi):
        i = np.arange(lo, hi)
        e.asks_upsert(i, full.ask_req[i], full.ask_app[i], full.ask_create[i], priority=full.ask_prio[i], flags=full.ask_flags[i])
    upsert(0, n1)
    ask, node, _ = e.cycle(n1)
    assert ask.tolist() == list(want1["ask"]) and node.tolist() == list(want1["node"])
    left = sorted(set(range(n1)) - set(ask.tolist()))
    if left:
        e.asks_remove(left)
    upsert(n1, A)
    ask, node, _ = e.cycle(A - n1)
    assert (ask - n1).tolist() == list(want2["ask"]) and node.tolist() == list(want2["node"])
    for a in left:
        w.state[a] = 255

    def plan_fn(order, rnd):
        want = po.plan(w, order)
        st, nd, vic, done = e.preemption_plan(order)
        got = [(int(x), None if n == YK_NONE else int(n), [int(v) for v in vs]) for x, n, vs in zip(st, nd, vic)]
        assert done == len(order) and got == want, (full.name, D, policy, commit, batch, rnd)
        return got

    def release(v):
        e.release(v)
        w.release(v)

    def remove(a):
        e.asks_remove(a)
        w.remove(a)
    fuzz_rounds(w, n1, A, plan_fn, release, remove)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(20))
def test_fuzz(seed):
    for D in (1, 4, 8):
        for policy in (0, 1):
            for commit in ("host", "device", "auto"):
                for batch in (64, 4096):
                    fuzz_session(seed, D, policy, commit, batch)


# ---- edges ----
def wide_session(engine, n_nodes, per_node, big, **kw):
    """n_nodes full nodes holding per_node pods of queue a (guarantee 1 pod) each; preemptors in queue b (guaranteed big pods)"""
    names = ["root", "a", "b"]
    pods = [("a", 10, 10, 0)] * (n_nodes * per_node)
    sc = dict(node=(10 * per_node, 10 * per_node), queues=[Q("root", None), Q("a", "root", (10, 10)), Q("b", "root", (10 * big, 10 * big))])
    ss = Session(sc, pods + [("b", 10 * big, 10 * big, 0)], engine, **kw)
    assert ss.names == names
    return ss


@pytest.mark.gpu
def test_more_victims_than_a_warp_on_one_node():
    ss = wide_session(True, 1, 48, 40)
    ss.add(range(48)); ss.cycle(); ss.add([48]); ss.cycle()
    (st, node, vic), = _plans(ss.plan([48]))
    assert st == po.PLANNED and len(vic) == 40
    assert vic == sorted(vic, reverse=True)     # newest first


@pytest.mark.gpu
def test_more_than_2_16_eligible_allocations_and_ties():
    """70 000 bound pods on 700 equal nodes: every node needs one victim, the earliest node in the order wins and gives its
    newest pod"""
    from yunikorn_k8shim_b200 import Engine
    N, per = 700, 100
    A = N * per + 1
    e = Engine(D=4, max_nodes=N, max_asks=A, max_apps=3, max_queues=3)
    e.queues_set([-1, 0, 0], [[-1] * 4, [10, 10, -1, -1], [10, 10, -1, -1]])
    tot = np.tile([10 * per, 10 * per, 110, 0], (N, 1))
    e.nodes_upsert(np.arange(N), tot, tot, name_rank=np.arange(N))
    e.apps_upsert([0, 1], [1, 2], [1, 2])
    req = np.tile([10, 10, 1, 0], (A, 1))
    e.asks_upsert(np.arange(A - 1), req[:-1], np.zeros(A - 1, np.int32), np.arange(A - 1))
    ask, node, _ = e.cycle(A)
    assert len(ask) == A - 1
    e.asks_upsert([A - 1], req[-1:], [1], [10 ** 9])
    e.cycle(1)
    st, nd, vic, done = e.preemption_plan([A - 1])
    order = np.lexsort((np.arange(N), np.arange(N), e.node_scores(np.arange(N))))
    assert done == 1 and st[0] == po.PLANNED and nd[0] == order[0]
    on = ask[node == order[0]]
    assert vic[0].tolist() == [int(on.max())]


@pytest.mark.gpu
def test_fits_cap_clears_and_errors():
    import ctypes as C
    pods = [("sandbox1", 100, M, 0)] * 3 + [("sandbox2", 100, M, 0)] * 2
    ss = Session(BASIC, pods, True)
    ss.add([0, 1, 2]); ss.cycle(); ss.add([3, 4]); ss.cycle()
    e = ss.e
    # victims_cap: stops before the ask whose victims would pass it
    st, nd, vic, done = e.preemption_plan([3, 4], victims_cap=0)
    assert done == 0
    # errors: nothing marked, nothing planned
    for bad in ([3, 3], [3, 99]):
        with pytest.raises(Exception):
            e.preemption_plan(bad)
    rc = e._lib.yk_preemption_plan(e._h, C.c_uint32(1), None, None, None, None, None, C.c_uint32(0), None)
    assert rc == -1
    # plan ask 3 (one victim)
    assert _plans(ss.plan([3]))[0][0] == po.PLANNED
    # errors after a plan: the mark and the plan stay exactly as they were (ask 3 is still planned: not blocked; ask 4 sees
    # sandbox1 one pod lighter)
    for bad in ([4, 4], [4, 99]):
        with pytest.raises(Exception):
            e.preemption_plan(bad)
    assert _plans(e.preemption_plan([3, 4], victims_cap=0))[:1] == [(po.NOT_BLOCKED, None, [])]
    # a NaN node score is refused before anything is marked (node 0: a +Inf and a -Inf share)
    nan_total, nan_avail = ss.s.node_total.copy(), np.array([[-10, 5, 110, 0]], dtype=np.int64)
    nan_total[0, :2] = 0
    e.nodes_upsert([0], nan_total, nan_avail, name_rank=[0])
    with pytest.raises(Exception) as ei:
        e.preemption_plan([4])
    assert ei.value.code == -5
    e.nodes_upsert([0], ss.s.node_total, np.asarray([ss.w.avail[0]], dtype=np.int64), name_rank=[0])
    # a resize drops the plan: planning again takes a fresh victim, as the oracle says
    e.asks_resize([3], ss.s.ask_req[[3]]); ss.w.resize(3, ss.s.ask_req[3])
    ss.plan([3, 4])
    # remove drops the plan; release clears the marks
    e.asks_remove([4]); ss.w.remove([4])
    marked = sorted(ss.w.marked)
    ss.release(marked)
    ss.plan([3])                                 # as the oracle says
    ss.cycle()                                   # the allocation spends the plan
    assert 3 in ss.w.bound
    assert _plans(ss.plan([3])) == [(po.NOT_BLOCKED, None, [])]   # allocated: not blocked


@pytest.mark.gpu
def test_fits_when_room_was_freed_since_the_cycle():
    pods = [("sandbox1", 100, M, 0)] * 3 + [("sandbox2", 100, M, 0)]
    ss = Session(BASIC, pods, True)
    ss.add([0, 1, 2]); ss.cycle(); ss.add([3]); ss.cycle()
    assert ss.w.state[3] == po.ST_NOFIT
    ss.release([2])
    assert _plans(ss.plan([3])) == [(po.FITS, 0, [])]
    assert _plans(ss.plan([3])) == [(po.FITS, 0, [])]    # FITS marks and plans nothing


@pytest.mark.gpu
def test_step7_runs_out_and_marks_nothing():
    pods = [("sandbox1", 100, M, 0)] * 3 + [("low-priority", 100, M, 0), ("high-priority", 100, M, 0)]
    ss = Session(PRIO, pods, True)
    ss.add([0, 1, 2]); ss.cycle(); ss.add([3, 4]); ss.cycle()
    assert _plans(ss.plan([3])) == [(po.NO_VICTIMS, None, [])]
    assert not ss.w.marked
    assert _plans(ss.plan([4]))[0][0] == po.PLANNED   # the failed plan left nothing behind


# ---- no effect on existing behaviour ----
@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["auto", "host", "device"])
def test_plans_leave_the_next_cycle_alone(commit):
    from yunikorn_k8shim_b200 import Engine
    s = fuzz_cluster(3, 4, 0)[0]
    outs = []
    for plan in (False, True):
        e = Engine.for_snapshot(s, commit=commit)
        e.queues_preemption(s.q_pp_fence)
        e.cycle(s.n_asks)
        st = e.ask_states(np.arange(s.n_asks))
        if plan:
            blocked = np.nonzero((st == po.ST_NOFIT) | (st == po.ST_SKIPPED))[0]
            e.preemption_plan(blocked)
            with pytest.raises(Exception):
                e.preemption_plan([0, 0])
        e.release(np.nonzero(st == po.ST_ALLOCATED)[0][:5])
        ask, node, _ = e.cycle(s.n_asks)
        outs.append((ask.tolist(), node.tolist(), e.ask_states(np.arange(s.n_asks)).tolist(),
                     e.nodes_available(np.arange(s.n_nodes)).tolist(), e.node_scores(np.arange(s.n_nodes)).tolist()))
    assert outs[0] == outs[1]


@pytest.mark.gpu
def test_new_flag_bits_leave_cycles_and_rows_alone():
    from yunikorn_k8shim_b200 import Engine
    s = synth.fuzz(11, n_nodes=20, n_asks=150)
    t = copy.deepcopy(s)
    t.ask_flags = (t.ask_flags | np.random.default_rng(1).choice([0, 2, 4, 8, 14], t.n_asks)).astype(np.uint32)
    outs = []
    for snap in (s, t):
        e = Engine.for_snapshot(snap)
        ask, node, slow = e.cycle(snap.n_asks, slow_cap=snap.n_asks)
        outs.append((ask.tolist(), node.tolist(), slow.tolist(), e.ask_states(np.arange(snap.n_asks)).tolist(),
                     e.stats()["rows_swept"]))
    assert outs[0] == outs[1]
