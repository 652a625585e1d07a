"""yk_preemption_required_node: preemption for asks with a required node, DaemonSet pods (DESIGN.md §2 item 10).

The expectation comes from tests/required_node_oracle.py, a plain-Python restatement of the rules over
tests/preemption_oracle.World.  The reference's end-to-end scenarios (test/e2e/simple_preemptor/simple_preemptor_test.go) are
written here as data.  The CPU tests run every case on the oracle with a stand-in cycle; the GPU tests drive the engine through
the same calls and check every answer against the oracle."""
import copy

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
import preemption_oracle as po
import required_node_oracle as rno

YK_NONE = 0xFFFFFFFF
NO_SELF, NO_OTHER, ORIGINATOR, SLOWPATH = 2, 4, 8, 1
COMMITS = ["auto", "host", "device"]


def P(req, on=-1, node=-1, prio=0, flags=0, create=None, queue=1, app=None, tol=0):
    """one pod: on = the node a label pins it to (it may be a victim), node = its required node (a DaemonSet pod)"""
    return dict(req=list(req), on=on, node=node, prio=prio, flags=flags, create=create, queue=queue, app=app, tol=tol)


class Session:
    """The oracle's World for a small cluster, and with engine=True the engine driven through the same calls.  Node i carries
    label bit i, and a pod with on=i needs it, so that every placement is the same on both sides.  pods are declared up front;
    `add` makes them present as pending asks."""

    def __init__(self, totals, pods, engine=False, taint=None, flags=None, parent=(-1, 0), qmax=None, users=None, **ekw):
        N, A, D = len(totals), len(pods), len(totals[0])
        self.D = D
        parent = np.array(parent, dtype=np.int32)
        Qn = len(parent)
        mx = np.full((Qn, D), -1, dtype=np.int64)
        for q, row in (qmax or {}).items():
            mx[q] = row
        apps = [p["app"] if p["app"] is not None else i for i, p in enumerate(pods)]
        napp = max(apps) + 1
        app_queue = np.zeros(napp, dtype=np.int32)
        for p, ap in zip(pods, apps):
            app_queue[ap] = p["queue"]
        tot = np.array(totals, dtype=np.int64)
        self.s = synth._finish("required-node", D, 0, tot, tot.copy(),
                               np.array(taint or [0] * N, dtype=np.uint64), np.array([1 << i for i in range(N)], dtype=np.uint64),
                               [f"node-{i}" for i in range(N)],
                               (parent, np.full((Qn, D), -1, dtype=np.int64), mx, np.zeros((Qn, D), dtype=np.int64),
                                np.zeros(Qn, dtype=np.uint8)),
                               app_queue, np.array(apps, dtype=np.int32), np.array([p["req"] for p in pods], dtype=np.int64),
                               np.array([p["tol"] for p in pods], dtype=np.uint64),
                               np.array([(1 << p["on"]) if p["on"] >= 0 else 0 for p in pods], dtype=np.uint64),
                               np.zeros(A, np.uint64), ask_prio=np.array([p["prio"] for p in pods], dtype=np.int32),
                               ask_node=np.array([p["node"] for p in pods], dtype=np.int32),
                               ask_flags=np.array([p["flags"] for p in pods], dtype=np.uint32),
                               ask_create=np.array([i if p["create"] is None else p["create"] for i, p in enumerate(pods)]),
                               node_flags=None if flags is None else np.array(flags, dtype=np.uint32))
        if users:   # (app user per app, [(queue, user, max)])
            self.s.app_user = np.array(users[0], dtype=np.int32)
            self.s.ul_queue = np.array([x[0] for x in users[1]], dtype=np.int32)
            self.s.ul_user = np.array([x[1] for x in users[1]], dtype=np.int32)
            self.s.ul_max = np.array([x[2] for x in users[1]], dtype=np.int64)
            self.s.ul_alloc = np.zeros((len(users[1]), D), dtype=np.int64)
        self.w = po.World(self.s, {}, np.full(A, 255), self.s.node_avail)
        self.e = None
        if engine:
            from yunikorn_k8shim_b200 import Engine
            s = self.s
            self.e = Engine(D=D, max_nodes=N, max_asks=A, max_apps=napp, max_queues=Qn, **ekw)
            self.e.queues_set(s.q_parent, s.q_guaranteed, s.q_max, s.q_alloc, s.q_sort)
            self.e.nodes_upsert(np.arange(N), s.node_total, s.node_avail, s.node_taint, s.node_label, s.node_rank(), s.node_flags)
            self.e.apps_upsert(np.arange(napp), s.app_queue, s.app_submit)
            if users:
                self.e.apps_user(np.arange(napp), s.app_user)
                self.e.user_limits_set(s.ul_queue, s.ul_user, s.ul_max)

    def add(self, idx):
        idx = np.asarray(list(idx), dtype=np.int64)
        s = self.s
        if self.e is not None:
            self.e.asks_upsert(idx, s.ask_req[idx], s.ask_app[idx], s.ask_create[idx], s.ask_tol[idx], s.ask_need[idx],
                               s.ask_deny[idx], s.ask_prio[idx], s.ask_node[idx], s.ask_flags[idx])
        for a in idx:
            self.w.state[int(a)] = 0
            self.w.plans.pop(int(a), None)

    def cycle(self):
        w, s = self.w, self.s
        pend = sorted(a for a, st in w.state.items() if st not in (po.ST_ALLOCATED, 255))
        if self.e is not None:
            ask, node, _ = self.e.cycle(len(pend) + 1)
            for a, n in zip(ask, node):
                w.allocate(int(a), int(n))
            for a, x in zip(pend, self.e.ask_states(pend) if pend else []):
                w.state[a] = int(x)
            return
        # stand-in: each node is the only one a pinned pod can use, so the order of the nodes does not matter
        for a in pend:
            if any(w.qmax[q][k] >= 0 and w.alloc[q][k] + w.req[a][k] > w.qmax[q][k] for q in w.path(w.leaf(a)) for k in range(self.D)):
                w.state[a] = po.ST_SKIPPED
                continue
            if int(s.ask_flags[a]) & SLOWPATH:
                w.state[a] = 4                                   # YK_ST_SLOWPATH: left to the caller's predicates
                continue
            x = int(s.ask_node[a])
            for n in ([x] if x >= 0 else sorted(w.present_nodes)):
                if n in w.present_nodes and w.static_ok(a, n) and all(w.req[a][k] <= max(0, w.avail[n][k]) for k in range(self.D)):
                    w.allocate(a, n)
                    break
            else:
                w.state[a] = po.ST_NOFIT

    def plan(self, idx, cap=None):
        want = rno.plan_required(self.w, idx) if cap is None else None
        if self.e is not None:
            st, vic, done = self.e.preemption_required_node(idx, victims_cap=cap)
            got = [(int(x), [int(v) for v in vs]) for x, vs in zip(st, vic)]
            if want is not None:
                assert done == len(idx) and got == want, (got, want)
            return got
        return want

    def release(self, idx):
        if self.e is not None:
            self.e.release(np.asarray(idx, dtype=np.uint32))
        self.w.release([int(a) for a in idx])

    def running_on(self, n):
        got = sorted(a for a, x in self.w.bound.items() if x == n)
        if self.e is not None:
            st = self.e.ask_states(np.arange(self.s.n_asks))
            assert sorted(np.nonzero(st == po.ST_ALLOCATED)[0].tolist()) == sorted(self.w.bound)
        return got


# ---- the reference's scenarios as data (simple_preemptor_test.go): two workers, each pod's memory is allocatable / 3.5, every
# other node tainted; RequiredNode pods are DaemonSet pods ----
MEM = 7_000_000
LIM = MEM * 2 // 7
WORKERS = [[8000, MEM, 110, 0]] * 2 + [[8000, MEM, 110, 0]]
TAINTED = dict(taint=[0, 0, 1])


def run_basic(engine, **kw):
    # sleepjob (Worker1, DaemonSet), sleepjob2 (no node: lands on Worker2), sleepjob3 (Worker2, DaemonSet)
    pods = [P([100, 2 * LIM, 1, 0], node=0), P([100, 2 * LIM, 1, 0]), P([100, 2 * LIM, 1, 0], node=1)]
    for p in pods:
        p["flags"] = ORIGINATOR          # every pod is its own application
    ss = Session(WORKERS, pods, engine, **TAINTED, **kw)
    for a in range(3):
        ss.add([a]); ss.cycle()
    assert ss.w.bound == {0: 0, 1: 1} and ss.w.state[2] == po.ST_NOFIT
    (st, vic), = ss.plan([2])
    assert st == po.PLANNED and vic == [1]                       # sleepjob2 is killed
    ss.release(vic); ss.cycle()
    assert ss.running_on(1) == [2]


def run_simple(engine, **kw):
    # sleepjob, 2, 3 on Worker1 (3 is application test01's originator); sleepjob4 (test01, Allow), 5 and 6 (Deny) land on
    # Worker2; sleepjob7 is the Worker2 DaemonSet pod
    pods = [P([100, LIM, 1, 0], node=0, flags=ORIGINATOR, app=0), P([100, LIM, 1, 0], node=0, flags=ORIGINATOR, app=1),
            P([100, LIM, 1, 0], node=0, flags=ORIGINATOR, app=2), P([100, LIM, 1, 0], app=2),
            P([100, LIM, 1, 0], flags=NO_SELF | ORIGINATOR, app=3), P([100, LIM, 1, 0], flags=NO_SELF | ORIGINATOR, app=4),
            P([100, LIM, 1, 0], node=1, flags=ORIGINATOR, app=5)]
    ss = Session(WORKERS, pods, engine, **TAINTED, **kw)
    for a in range(7):
        ss.add([a]); ss.cycle()
    assert ss.running_on(1) == [3, 4, 5] and ss.w.state[6] == po.ST_NOFIT
    (st, vic), = ss.plan([6])
    assert st == po.PLANNED and vic == [3]                       # only sleepjob4; the opted-out pods stay
    ss.release(vic); ss.cycle()
    assert ss.running_on(1) == [4, 5, 6]


SCENARIOS = [run_basic, run_simple]


@pytest.mark.parametrize("scenario", SCENARIOS, ids=lambda f: f.__name__[4:])
def test_reference_scenarios_on_the_oracle(scenario):
    scenario(False)


@pytest.mark.gpu
@pytest.mark.parametrize("commit", COMMITS)
@pytest.mark.parametrize("scenario", SCENARIOS, ids=lambda f: f.__name__[4:])
def test_reference_scenarios(scenario, commit):
    scenario(True, commit=commit)


# ---- named cases: each runs on the oracle (CPU) and through the engine against the oracle (GPU) ----
NODE = [1000, 10, 110, 0]                # (vcore, memory, pods, ephemeral); the cases size pods in memory


def full_request_not_shortfall(engine):
    """room 1, request 4: the part room lacks (3) is one victim, the full request is two"""
    pods = [P([0, 3, 1, 0], on=0), P([0, 3, 1, 0], on=0), P([0, 3, 1, 0], on=0), P([0, 4, 1, 0], node=0)]
    ss = Session([NODE], pods, engine)
    ss.add(range(3)); ss.cycle(); ss.add([3]); ss.cycle()
    assert ss.plan([3]) == [(po.PLANNED, [2, 1])]               # newest first


def originator_dominates(engine):
    """a NO_PREEMPT_SELF non-originator goes before an originator here; the guarantee plan takes them the other way round"""
    pods = [P([0, 5, 1, 0], on=0, flags=ORIGINATOR, create=1), P([0, 5, 1, 0], on=0, flags=NO_SELF, create=0),
            P([0, 5, 1, 0], node=0, queue=2)]
    ss = Session([NODE], pods, engine, parent=(-1, 0, 0))
    ss.add([0, 1]); ss.cycle(); ss.add([2]); ss.cycle()
    assert ss.plan([2]) == [(po.PLANNED, [1])]
    # the same cluster through the guarantee plan: its preemptor has no required node and a guarantee
    twin = copy.deepcopy(ss.s)
    twin.ask_node[2] = -1
    twin.ask_need[2] = 1
    twin.q_guaranteed[2] = [-1, 100, -1, -1]
    w = po.World(twin, {0: 0, 1: 0}, [1, 1, po.ST_NOFIT], [[1000, 0, 108, 0]])
    assert po.plan(w, [2]) == [(po.PLANNED, 0, [0])]


def priorities(engine):
    """a higher priority is skipped, an equal one taken"""
    pods = [P([0, 5, 1, 0], on=0, prio=7), P([0, 5, 1, 0], on=0, prio=8), P([0, 5, 1, 0], node=0, prio=7)]
    ss = Session([NODE], pods, engine)
    ss.add([0, 1]); ss.cycle(); ss.add([2]); ss.cycle()
    assert ss.plan([2]) == [(po.PLANNED, [0])]


def skipped_allocations(engine):
    """a required-node allocation, a marked one and one without a shared resource are never victims"""
    pods = [P([0, 3, 1, 0], node=0), P([0, 3, 1, 0], on=0), P([0, 0, 1, 3], on=0), P([0, 3, 1, 0], on=0),
            P([0, 3, 0, 0], node=0), P([0, 3, 0, 0], node=0, create=-1)]
    ss = Session([[1000, 10, 110, 10]], pods, engine)
    ss.add(range(4)); ss.cycle(); ss.add([4, 5]); ss.cycle()
    assert ss.w.state[4] == ss.w.state[5] == po.ST_NOFIT
    # 4 takes 3 (newest); 5 cannot take 3 (marked), 2 (no memory, 5 asks no pods), 0 (a required node): it takes 1
    assert ss.plan([4, 5]) == [(po.PLANNED, [3]), (po.PLANNED, [1])]


def create_ties(engine):
    pods = [P([0, 4, 1, 0], on=0, create=5), P([0, 4, 1, 0], on=0, create=5), P([0, 4, 1, 0], node=0)]
    ss = Session([NODE], pods, engine)
    ss.add([0, 1]); ss.cycle(); ss.add([2]); ss.cycle()
    assert ss.plan([2]) == [(po.PLANNED, [0])]


def chains(engine):
    """two and three preemptors on one node in one call: each sees the victims and the requests of the earlier ones"""
    pods = [P([0, 2, 1, 0], on=0) for _ in range(5)] + [P([0, 3, 0, 0], node=0), P([0, 3, 0, 0], node=0),
                                                         P([0, 5, 0, 0], node=0)]
    ss = Session([NODE], pods, engine)
    ss.add(range(5)); ss.cycle(); ss.add([5, 6, 7]); ss.cycle()
    assert ss.plan([5, 6, 7]) == [(po.PLANNED, [4, 3]), (po.PLANNED, [2, 1]), (po.NO_VICTIMS, [])]
    pods2 = [P([0, 3, 1, 0], on=0) for _ in range(3)] + [P([0, 3, 0, 0], node=0), P([0, 2, 0, 0], node=0)]
    ss = Session([NODE], pods2, engine)
    ss.add(range(3)); ss.cycle(); ss.add([3, 4]); ss.cycle()
    # room 1: the first takes 2 (room 1 + 3 - 3 = 1), the second takes 1
    assert ss.plan([3, 4]) == [(po.PLANNED, [2]), (po.PLANNED, [1])]


def fits_through_marks(engine):
    pods = [P([0, 3, 1, 0], on=0), P([0, 6, 1, 0], on=0), P([0, 3, 0, 0], node=0), P([0, 2, 0, 0], node=0)]
    ss = Session([NODE], pods, engine)
    ss.add([0, 1]); ss.cycle(); ss.add([2, 3]); ss.cycle()
    assert ss.plan([2]) == [(po.PLANNED, [1])]                   # room 1 + 6 - 3 = 4 until the victim goes
    assert ss.plan([3]) == [(po.FITS, [])]
    assert ss.plan([3]) == [(po.FITS, [])]                       # FITS marks and plans nothing


def static_steps(engine):
    """cordoned, tainted, too small and absent nodes: NO_VICTIMS, and nothing is marked"""
    pods = [P([0, 8, 1, 0], on=n, tol=1) for n in range(4)] + [P([0, 5, 0, 0], node=n) for n in range(3)] + [P([0, 50, 0, 0], node=3)]
    ss = Session([NODE] * 4, pods, engine, taint=[0, 1, 0, 0])
    ss.add(range(4)); ss.cycle(); ss.add(range(4, 8)); ss.cycle()
    ss.w.node_remove(2)
    if ss.e is not None:
        ss.e.nodes_remove([2])
        ss.e.nodes_upsert([0], ss.s.node_total[[0]], [ss.w.avail[0]], label_bits=ss.s.node_label[[0]], name_rank=[0], flags=[0])
    ss.s.node_flags[0] = 0                                       # cordoned
    assert ss.plan([4, 5, 6, 7]) == [(po.NO_VICTIMS, [])] * 4
    assert not ss.w.marked


def headroom(engine):
    """a queue max and a user limit on the preemptor's path: NOT_ALLOWED, from what is allocated"""
    pods = [P([0, 8, 1, 0], on=0, queue=2), P([0, 5, 0, 0], node=0, queue=2), P([0, 5, 0, 0], node=0, queue=3),
            P([0, 5, 0, 0], node=0, queue=1)]
    ss = Session([NODE], pods, engine, parent=(-1, 0, 0, 0), qmax={2: [-1, 12, -1, -1]},
                 users=([0, 0, 1, 2], [(3, 1, [-1, 4, -1, -1])]))
    ss.add([0]); ss.cycle(); ss.add([1, 2, 3]); ss.cycle()
    assert ss.w.state[1] == po.ST_SKIPPED
    assert ss.plan([1, 2, 3]) == [(po.NOT_ALLOWED, []), (po.NOT_ALLOWED, []), (po.PLANNED, [0])]


def no_preempt_other_ignored(engine):
    pods = [P([0, 8, 1, 0], on=0), P([0, 5, 0, 0], node=0, flags=NO_OTHER)]
    ss = Session([NODE], pods, engine)
    ss.add([0]); ss.cycle(); ss.add([1]); ss.cycle()
    assert ss.plan([1]) == [(po.PLANNED, [0])]


def who_may_preempt(engine):
    """allocated, slow-path (never blocked) and absent asks are not blocked; a blocked ask without a required node is
    unsupported"""
    pods = [P([0, 8, 1, 0], on=0), P([0, 1, 0, 0], node=0), P([0, 5, 1, 0], on=0), P([0, 5, 0, 0], node=0, flags=SLOWPATH),
            P([0, 5, 0, 0], node=0), P([0, 5, 0, 0], node=0)]
    ss = Session([NODE], pods, engine)
    ss.add([0]); ss.cycle(); ss.add([1, 2, 3, 4]); ss.cycle()
    assert ss.plan([1, 2, 3, 5]) == [(po.NOT_BLOCKED, []), (po.UNSUPPORTED, []), (po.NOT_BLOCKED, []), (po.NOT_BLOCKED, [])]
    assert ss.plan([4]) == [(po.PLANNED, [0])]                   # 1 holds a required node: 0 is the only victim
    assert ss.plan([4]) == [(po.NOT_BLOCKED, [])]                # planned already


NAMED = [full_request_not_shortfall, originator_dominates, priorities, skipped_allocations, create_ties, chains,
         fits_through_marks, static_steps, headroom, no_preempt_other_ignored, who_may_preempt]


@pytest.mark.parametrize("case", NAMED, ids=lambda f: f.__name__)
def test_named_cases_on_the_oracle(case):
    case(False)


@pytest.mark.gpu
@pytest.mark.parametrize("case", NAMED, ids=lambda f: f.__name__)
def test_named_cases(case):
    case(True)


# ---- sessions on the engine: the cap, errors, what clears a plan, both plan calls, and no effect on cycles ----
def chain_session(engine, **kw):
    """three nodes, each full of 1-memory pods; per node two DaemonSet pods of 3"""
    pods = [P([0, 1, 1, 0], on=n) for n in range(3) for _ in range(10)]
    pods += [P([0, 3, 0, 0], node=n) for n in range(3) for _ in range(2)]
    ss = Session([NODE] * 3, pods, engine, **kw)
    ss.add(range(30)); ss.cycle(); ss.add(range(30, 36)); ss.cycle()
    return ss


@pytest.mark.gpu
def test_cap_cut_then_remainder_equals_one_call():
    order = [30, 32, 34, 31, 33, 35]
    whole = chain_session(True).plan(order)
    assert [x[0] for x in whole] == [po.PLANNED] * 6
    ss = chain_session(True)
    st, vic, done = ss.e.preemption_required_node(order, victims_cap=10)
    assert done == 3 and [v.tolist() for v in vic] == [x[1] for x in whole[:3]]   # the fourth would bring the victims to 12
    got = [(int(x), v.tolist()) for x, v in zip(st, vic)]
    ss.w.marked.update(v for x in whole[:3] for v in x[1])
    ss.w.plans.update({a: int(ss.s.ask_node[a]) for a in order[:3]})
    got += ss.plan(order[3:])
    assert got == whole


@pytest.mark.gpu
def test_argument_errors_change_nothing():
    import ctypes as C
    ss = chain_session(True)
    e = ss.e
    for bad in ([30, 30], [30, 10 ** 6]):
        with pytest.raises(Exception):
            e.preemption_required_node(bad)
    null = C.c_uint32(0)
    assert e._lib.yk_preemption_required_node(e._h, C.c_uint32(1), None, None, None, None, C.c_uint32(0), None) == -1
    off = (C.c_uint32 * 2)()
    ask, st = (C.c_uint32 * 1)(30), (C.c_uint32 * 1)()
    assert e._lib.yk_preemption_required_node(e._h, C.c_uint32(1), ask, st, off, None, C.c_uint32(5), C.byref(null)) == -1
    assert not ss.w.marked
    ss.plan([30, 31, 32])                                        # as if no error had happened


@pytest.mark.gpu
def test_plans_clear_on_allocation_removal_upsert_and_resize():
    ss = chain_session(True)
    e, s = ss.e, ss.s
    assert [x[0] for x in ss.plan([30, 32, 34, 35])] == [po.PLANNED] * 4
    e.asks_remove([32]); ss.w.remove([32])                        # removal
    ss.add([32])                                                 # upsert again: pending, not blocked until a cycle
    e.asks_resize([34], s.ask_req[[34]]); ss.w.resize(34, s.ask_req[34])
    ss.release([v for v in sorted(ss.w.marked) if ss.w.bound[v] < 10])
    ss.cycle()                                                   # allocates 30: its plan is spent
    assert 30 in ss.w.bound
    ss.plan([30, 31, 32, 33, 34, 35])


@pytest.mark.gpu
def test_both_plan_calls_in_one_session():
    """a guarantee plan's marks and plans are seen by the required-node call, and the other way round"""
    pods = [P([0, 2, 1, 0], on=n) for n in range(2) for _ in range(5)]
    pods += [P([0, 4, 0, 0], on=0, queue=2), P([0, 4, 0, 0], node=0), P([0, 4, 0, 0], node=1), P([0, 4, 0, 0], on=1, queue=2)]
    ss = Session([NODE] * 2, pods, True, parent=(-1, 0, 0))
    ss.s.q_guaranteed[2] = [-1, 100, -1, -1]
    ss.e.queues_set(ss.s.q_parent, ss.s.q_guaranteed, ss.s.q_max, ss.s.q_alloc, ss.s.q_sort)
    ss.w.guar[2] = [-1, 100, -1, -1]
    ss.add(range(10)); ss.cycle(); ss.add(range(10, 14)); ss.cycle()

    def gplan(idx):
        want = po.plan(ss.w, idx)
        st, nd, vic, done = ss.e.preemption_plan(idx)
        assert [(int(x), None if n == YK_NONE else int(n), v.tolist()) for x, n, v in zip(st, nd, vic)] == want
        return want
    assert gplan([10])[0][0] == po.PLANNED
    assert ss.plan([11, 12])[0][0] == po.PLANNED
    assert gplan([13])[0][0] == po.PLANNED
    assert ss.plan([11, 12]) == [(po.NOT_BLOCKED, [])] * 2


@pytest.mark.gpu
def test_nan_score_elsewhere_is_no_error():
    ss = chain_session(True)
    nan_total = ss.s.node_total[[2]].copy()
    nan_total[0, :2] = 0
    ss.e.nodes_upsert([2], nan_total, [[-10, 5, 110, 0]], label_bits=ss.s.node_label[[2]], name_rank=[2])
    st, vic, done = ss.e.preemption_required_node([30, 32])
    assert done == 2 and st.tolist() == [po.PLANNED] * 2


@pytest.mark.gpu
@pytest.mark.parametrize("commit", COMMITS)
def test_calls_leave_the_next_cycle_alone(commit):
    from yunikorn_k8shim_b200 import Engine
    s = rn_cluster(5, 4, 0)[0]
    outs = []
    for plan in (False, True):
        e = Engine.for_snapshot(s, commit=commit)
        e.cycle(s.n_asks)
        st = e.ask_states(np.arange(s.n_asks))
        if plan:
            blocked = np.nonzero((st == po.ST_NOFIT) | (st == po.ST_SKIPPED))[0]
            e.preemption_required_node(blocked)
            with pytest.raises(Exception):
                e.preemption_required_node([0, 0])
        e.release(np.nonzero(st == po.ST_ALLOCATED)[0][:5])
        r0 = e.stats()["rows_swept"]
        ask, node, _ = e.cycle(s.n_asks)
        outs.append((ask.tolist(), node.tolist(), e.ask_states(np.arange(s.n_asks)).tolist(),
                     e.nodes_available(np.arange(s.n_nodes)).tolist(), e.stats()["rows_swept"] - r0))
    assert outs[0] == outs[1]


# ---- fuzz against the oracle ----
# Queues: root(0) -> victims(1), daemons(2), capped(3) whose max is below what its pods ask.  Nodes are ~90 % full of random
# victims (tied priorities and create times, every flag mix, required-node allocations, zero resources); 0-3 DaemonSet pods
# per node, a few more on a node that is then cordoned, tainted or removed, and a few that are not DaemonSet pods.
def rn_cluster(seed, D, policy):
    """-> (snapshot of every ask, n1): asks [0, n1) are the victims (phase 1), the rest the preemptors (phase 2)"""
    rng = np.random.default_rng(seed + 1000)
    N = 6 + seed % 7
    tot = np.tile([8000, 16000, 110, 0], (N, 1)).astype(np.int64)
    cap = tot[:, :2].sum(axis=0)
    vreq, vnode = [], []
    load = np.zeros(2, dtype=np.int64)
    while True:
        c = int(rng.choice([250, 500, 1000, 1500]))
        r = np.array([c, 2 * c, 1, 0])
        if rng.random() < 0.15:
            r[0] = 0                                             # no vcore: shares only memory and pods
        if (load + r[:2] > 0.9 * cap).any():
            break
        load += r[:2]
        vreq.append(r)
        vnode.append(int(rng.integers(0, N)) if rng.random() < 0.08 else -1)
    n1 = len(vreq)
    preq, pnode, papp = [], [], []
    for n in range(N):
        for _ in range(int(rng.integers(0, 4))):
            c = int(rng.choice([500, 1500, 3000]))
            preq.append(np.array([c, 2 * c, int(rng.integers(0, 2)), 0]))
            pnode.append(n)
            papp.append(2 if rng.random() < 0.9 else 3)
    for _ in range(3):                                           # not DaemonSet pods: unsupported when blocked
        c = int(rng.choice([3000, 6000]))
        preq.append(np.array([c, 2 * c, 1, 0])); pnode.append(-1); papp.append(2)
    n2 = len(preq)
    A = n1 + n2
    req = np.array(vreq + preq, dtype=np.int64)
    app = np.array([1] * n1 + papp, dtype=np.int32)              # application i lives in queue i
    node = np.array(vnode + pnode, dtype=np.int32)
    prio = np.concatenate([rng.choice([-5, 0, 5], n1), rng.choice([0, 5], n2)]).astype(np.int32)
    flags = np.concatenate([rng.choice([0, NO_SELF, ORIGINATOR, NO_SELF | ORIGINATOR], n1, p=[0.4, 0.2, 0.2, 0.2]),
                            rng.choice([0, NO_OTHER], n2, p=[0.85, 0.15])]).astype(np.uint32)
    create = rng.integers(0, max(2, A // 3), A).astype(np.int64)
    Db = 8 if D == 8 else 4
    mx = np.full((4, Db), -1, dtype=np.int64)
    mx[3, 0] = 1000
    guar = np.full((4, Db), -1, dtype=np.int64)
    if Db == 8:
        tot = np.hstack([tot, np.full((N, 4), 4000, np.int64)])
        extra = rng.integers(0, 4, (A, 4))
        req = np.hstack([req, extra]).astype(np.int64)
    t = synth._finish(f"rn-fuzz-{seed}", Db, policy, tot, tot.copy(), np.zeros(N, np.uint64), np.zeros(N, np.uint64),
                      [f"n{int(x):03d}" for x in rng.permutation(N)],
                      (np.array([-1, 0, 0, 0], dtype=np.int32), guar, mx, np.zeros((4, Db), np.int64), np.zeros(4, np.uint8)),
                      np.arange(4, dtype=np.int32), app, req, np.zeros(A, np.uint64), np.zeros(A, np.uint64),
                      np.zeros(A, np.uint64), ask_prio=prio, ask_node=node, ask_flags=flags, ask_create=create)
    if D == 1:
        t = synth.redim(t, 1, seed)
    return t, n1


def rn_world(seed, D, policy):
    """phase 1 (victims) and phase 2 (preemptors) on the oracle's cycle -> (full, n1, want1, want2, World)"""
    from oracle import py_oracle
    full, n1 = rn_cluster(seed, D, policy)
    A = full.n_asks
    fields = ("ask_app", "ask_req", "ask_tol", "ask_need", "ask_deny", "ask_prio", "ask_create", "ask_node", "ask_flags", "ask_gang")
    s1 = copy.deepcopy(full)
    for f in fields:
        setattr(s1, f, getattr(full, f)[:n1])
    want1 = py_oracle.run(s1)
    s2 = copy.deepcopy(full)
    for f in fields:
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
    return full, n1, want1, want2, po.World(full, bound, state, want2["avail"])


def rn_session(w, n1, seed, ops, info=None):
    """node changes (cordon, taint, removal), two calls with releases, resizes and a cycle in between.  ops: the engine side
    (plan, release, resize, node_upsert, node_remove, cycle) or None for the oracle alone"""
    rng = np.random.default_rng(seed)
    s, A = w.s, w.s.n_asks
    N = s.n_nodes
    cord, taint, gone = int(rng.integers(0, N)), int(rng.integers(0, N)), int(rng.integers(0, N))
    for n, fl, tb in ((cord, 0, 0), (taint, 1, 1)):
        if n in w.present_nodes and n != gone:
            w.node_upsert(n, s.node_total[n].copy(), w.avail[n], taint=tb, label=0, flags=fl)
            if ops:
                ops["node_upsert"](n, fl, tb)
    w.node_remove(gone)
    if ops:
        ops["node_remove"](gone)

    def call(order):
        want = rno.plan_required(w, order, info)
        if ops:
            assert ops["plan"](order) == want, (s.name, order)
        return want
    daemons = [a for a in range(n1, A) if int(s.ask_node[a]) >= 0]
    blocked = [a for a in range(n1, A) if w.state[a] in (po.ST_NOFIT, po.ST_SKIPPED)]
    first = list(rng.permutation(sorted(set(blocked[: len(blocked) * 2 // 3] + daemons[:2] + [0]))))
    got = call([int(a) for a in first])
    victims = [v for _, vs in got for v in vs]
    if victims:
        rel = victims[: (len(victims) + 1) // 2]
        w.release(rel)
        if ops:
            ops["release"](rel)
    bound = sorted(a for a in w.bound if a < n1)
    for a in bound[:: max(1, len(bound) // 3)][:3]:              # resized victims, and one resized planned preemptor
        new = [int(x) for x in s.ask_req[a]]
        new[min(1, w.D - 1)] += 250
        w.resize(a, new)
        if ops:
            ops["resize"](a, new)
    planned = [a for a in first if a in w.plans]
    if planned:
        a = planned[-1]
        w.resize(a, [int(x) for x in s.ask_req[a]])
        if ops:
            ops["resize"](a, [int(x) for x in s.ask_req[a]])
    if ops:
        ops["cycle"]()
    second = [int(a) for a in rng.permutation(range(n1, A))]
    call(second)


def test_fuzz_coverage_floors():
    """the fuzz reaches every status at every D, plans of several victims, same-node chains, orders decided by the victim
    type and plans where the full request needs more victims than the part the room lacks"""
    for D in (1, 4, 8):
        info = []
        for seed in range(20):
            for policy in (0, 1):
                full, n1, _, _, w = rn_world(seed, D, policy)
                rn_session(w, n1, seed, None, info)
        st = {k: sum(1 for x in info if x["status"] == k) for k in range(7)}
        counts = dict(multi=sum(1 for x in info if x["victims"] > 1), chain=sum(1 for x in info if x["same_node_before"]),
                      typed=sum(1 for x in info if x["type_decides"]), shortfall=sum(1 for x in info if x["shortfall_differs"]))
        assert all(st[k] >= 5 for k in (po.PLANNED, po.FITS, po.NOT_BLOCKED, po.NOT_ALLOWED, po.UNSUPPORTED, po.NO_VICTIMS)), (D, st)
        assert st[po.GUARANTEE] == 0
        assert all(v >= 10 for v in counts.values()), (D, counts)


def rn_fuzz(seed, D, policy, commit, batch):
    from yunikorn_k8shim_b200 import Engine
    full, n1, want1, want2, w = rn_world(seed, D, policy)
    A = full.n_asks
    e = Engine(D=full.D, policy=policy, weights=full.weights, max_nodes=full.n_nodes, max_asks=A, max_apps=full.n_apps,
               max_queues=full.n_queues, commit=commit, batch=batch)
    e.queues_set(full.q_parent, full.q_guaranteed, full.q_max, full.q_alloc, full.q_sort)
    rank = full.node_rank()
    e.nodes_upsert(np.arange(full.n_nodes), full.node_total, full.node_avail, name_rank=rank)
    e.apps_upsert(np.arange(full.n_apps), full.app_queue, full.app_submit)

    def upsert(lo, hi):
        i = np.arange(lo, hi)
        e.asks_upsert(i, full.ask_req[i], full.ask_app[i], full.ask_create[i], priority=full.ask_prio[i],
                      required_node=full.ask_node[i], flags=full.ask_flags[i])
    upsert(0, n1)
    ask, node, _ = e.cycle(n1)
    assert ask.tolist() == list(want1["ask"]) and node.tolist() == list(want1["node"])
    left = sorted(set(range(n1)) - set(ask.tolist()))
    if left:
        e.asks_remove(left)
    for a in left:
        w.state[a] = 255
    upsert(n1, A)
    ask, node, _ = e.cycle(A - n1)
    assert (ask - n1).tolist() == list(want2["ask"]) and node.tolist() == list(want2["node"])

    def plan(order):
        st, vic, done = e.preemption_required_node(order)
        assert done == len(order)
        return [(int(x), [int(v) for v in vs]) for x, vs in zip(st, vic)]

    def cycle():
        pend = sorted(a for a, st in w.state.items() if st not in (po.ST_ALLOCATED, 255))
        ask, node, _ = e.cycle(len(pend) + 1)
        for a, n in zip(ask, node):
            w.allocate(int(a), int(n))
        for a, x in zip(pend, e.ask_states(pend)):
            w.state[a] = int(x)
        assert e.nodes_available(sorted(w.present_nodes)).tolist() == [w.avail[n] for n in sorted(w.present_nodes)]
    ops = dict(plan=plan, release=lambda v: e.release(v), resize=lambda a, r: e.asks_resize([a], [r]),
               node_upsert=lambda n, fl, tb: e.nodes_upsert([n], full.node_total[[n]], [w.avail[n]], taint_bits=[tb],
                                                            name_rank=[rank[n]], flags=[fl]),
               node_remove=lambda n: e.nodes_remove([n]), cycle=cycle)
    rn_session(w, n1, seed, ops)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(20))
def test_fuzz(seed):
    for D in (1, 4, 8):
        for policy in (0, 1):
            for commit in COMMITS:
                for batch in (64, 4096):
                    rn_fuzz(seed, D, policy, commit, batch)


# ---- scale ----
@pytest.mark.gpu
@pytest.mark.parametrize("per", [40, 100])
def test_more_eligible_victims_than_a_warp(per):
    """40 and 100 eligible victims on one node: the walk crosses 32-entry chunks, and the plan takes all but a few"""
    pods = [P([0, 1, 1, 0], on=0, create=i // 3) for i in range(per)] + [P([0, per - 3, 0, 0], node=0)]
    ss = Session([[1000, per, 200, 0]], pods, True)
    ss.add(range(per)); ss.cycle(); ss.add([per]); ss.cycle()
    (st, vic), = ss.plan([per])
    assert st == po.PLANNED and len(vic) == per - 3


def rollout(n_nodes, per=5, seed=0):
    """n_nodes nodes, each ~90 % full of `per` foreign-sized pods, and one DaemonSet pod per node"""
    rng = np.random.default_rng(seed)
    N = n_nodes
    tot = np.tile([8000, 16000, 110, 0], (N, 1)).astype(np.int64)
    vr = np.zeros((N * per, 4), dtype=np.int64)
    vr[:, 0] = rng.choice([1400, 1440], N * per)
    vr[:, 1] = 2 * vr[:, 0]
    vr[:, 2] = 1
    dr = np.tile([2000, 4000, 1, 0], (N, 1))
    A = N * per + N
    s = synth._finish("rollout", 4, 0, tot, tot.copy(), np.zeros(N, np.uint64), np.zeros(N, np.uint64),
                      [f"node-{i:05d}" for i in range(N)],
                      (np.array([-1, 0], dtype=np.int32), np.full((2, 4), -1, np.int64), np.full((2, 4), -1, np.int64),
                       np.zeros((2, 4), np.int64), np.zeros(2, np.uint8)),
                      np.array([1], dtype=np.int32), np.zeros(A, np.int32), np.vstack([vr, dr]), np.zeros(A, np.uint64),
                      np.zeros(A, np.uint64), np.zeros(A, np.uint64),
                      ask_prio=np.concatenate([rng.choice([0, 1], N * per), np.full(N, 1)]).astype(np.int32),
                      ask_node=np.concatenate([np.full(N * per, -1), np.arange(N)]).astype(np.int32),
                      ask_flags=rng.choice([0, NO_SELF, ORIGINATOR], A).astype(np.uint32),
                      ask_create=rng.integers(0, 1000, A))
    return s


@pytest.mark.gpu
def test_rollout_of_10000_nodes_in_one_call():
    N, per = 10_000, 5
    s = rollout(N, per)
    from yunikorn_k8shim_b200 import Engine
    e = Engine(D=4, max_nodes=N, max_asks=s.n_asks, max_apps=1, max_queues=2)
    e.queues_set(s.q_parent, s.q_guaranteed, s.q_max, s.q_alloc, s.q_sort)
    e.nodes_upsert(np.arange(N), s.node_total, s.node_avail, name_rank=np.arange(N))
    e.apps_upsert([0], [1], [1])
    bound = {}
    for lo, hi in ((0, N * per), (N * per, s.n_asks)):
        i = np.arange(lo, hi)
        e.asks_upsert(i, s.ask_req[i], s.ask_app[i], s.ask_create[i], priority=s.ask_prio[i], required_node=s.ask_node[i],
                      flags=s.ask_flags[i])
        ask, node, _ = e.cycle(hi - lo)
        bound.update({int(a): int(n) for a, n in zip(ask, node)})
    st = e.ask_states(np.arange(s.n_asks))
    w = po.World(s, bound, st, e.nodes_available(np.arange(N)).tolist())
    ds = list(range(N * per, s.n_asks))
    assert sum(1 for a in ds if w.state[a] == po.ST_NOFIT) > N // 2
    want = rno.plan_required(w, ds)
    got, vic, done = e.preemption_required_node(ds)
    assert done == N and [(int(x), v.tolist()) for x, v in zip(got, vic)] == want
    assert sum(1 for x in want if x[0] == po.PLANNED) > N // 2


@pytest.mark.gpu
def test_launches_do_not_grow_with_the_rollout():
    """the other_launches of one call is the same for 1 preemptor and for 10 000"""
    N, per = 10_000, 5
    s = rollout(N, per, seed=1)
    from yunikorn_k8shim_b200 import Engine
    deltas = []
    for n in (1, N):
        e = Engine(D=4, max_nodes=N, max_asks=s.n_asks, max_apps=1, max_queues=2)
        e.queues_set(s.q_parent, s.q_guaranteed, s.q_max, s.q_alloc, s.q_sort)
        e.nodes_upsert(np.arange(N), s.node_total, s.node_avail, name_rank=np.arange(N))
        e.apps_upsert([0], [1], [1])
        for lo, hi in ((0, N * per), (N * per, s.n_asks)):
            i = np.arange(lo, hi)
            e.asks_upsert(i, s.ask_req[i], s.ask_app[i], s.ask_create[i], priority=s.ask_prio[i],
                          required_node=s.ask_node[i], flags=s.ask_flags[i])
            e.cycle(hi - lo)
        st = e.ask_states(np.arange(N * per, s.n_asks))
        blocked = (np.nonzero(st == po.ST_NOFIT)[0] + N * per)[:n]
        assert len(blocked) >= min(n, N // 2)
        l0 = e.stats()["other_launches"]
        got, _, _ = e.preemption_required_node(blocked)
        deltas.append(e.stats()["other_launches"] - l0)
        assert (got == po.PLANNED).sum() > n // 2
    assert deltas[0] == deltas[1]
