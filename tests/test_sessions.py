"""Long scheduling sessions: one engine, many cycles, random state changes between them, every cycle checked against the oracle.

A real adapter never runs one cycle on a fresh snapshot.  It keeps one engine and, between cycles, adds, resizes, cordons,
renames and removes nodes, adds and removes pods and applications, releases allocations and replaces the queue and limit
tables.  The engine keeps device tables and caches across cycles (upload flags, the NodeID-rank order, signature numbers,
epoch rows, the device commit's node records); every one of them must be invalidated at the right moment.

`Model` holds the world as the adapter sees it.  Before each cycle it builds a compacted `synth.Snapshot` of the pending world
(present nodes, pending asks of present applications, in ascending engine index, with its own queue and user accounting),
runs the oracle on it and applies the ORACLE's bindings to itself.  It never reads the engine, so an error in one cycle
cannot leak into the expectation for the next.  Every operation is recorded in a script; the GPU tests replay a script on
an engine and compare, after every cycle, the bindings, every present node's availability (host table) and score (device
table), every ask's state and the counters.  The CPU tests check the model on its own: both oracles agree on every cycle's
snapshot, the accounting is conserved after every step, and the generated sessions cover every operation.

NodeIDs are zero-padded numbers (`n000123`) and the rank given to yk_nodes_upsert is that number: sparse and
order-preserving.  Create sequence numbers and submit times are unique, so compacting cannot reorder ties.
Removing an application that still holds allocations is not defined by include/ykgpu.h and is never generated."""
import functools

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from oracle import py_oracle

GI = synth.GI
ABSENT, PENDING, ALLOCATED, NOFIT = 255, 0, 1, 2
SCHED, RESERVED = synth.NODE_SCHEDULABLE, synth.NODE_RESERVED
# root -> two parents -> three leaves (leaves 3 and 4 under parent 1, leaf 5 under parent 2); applications live in leaves
Q_PARENT = np.array([-1, 0, 0, 1, 1, 2], dtype=np.int32)
LEAVES = (3, 4, 5)
UNIFORM_MIN = 8          # YK_UNIFORM_MIN of the session tests: runs of 8 identical asks take the uniform path


def _weights(D):
    w = np.zeros(D)
    w[0] = 1.0
    if D > 1:
        w[1] = 1.0
    return w


class Cycle:
    """one cycle of a script: the model's snapshot before it and everything the engine must show after it"""
    def __init__(self, **kw):
        self.__dict__.update(kw)


class Model:
    def __init__(self, oracle, name, D=4, policy=synth.POLICY_FAIR, max_nodes=128, max_asks=1024, max_apps=32, seed=0):
        self.oracle, self.name, self.D, self.policy = oracle, name, D, policy
        self.weights = _weights(D)
        self.maxN, self.maxA, self.maxP, self.maxQ = max_nodes, max_asks, max_apps, len(Q_PARENT)
        self.rng = np.random.default_rng(seed)
        N, A, P = max_nodes, max_asks, max_apps
        self.n_present = np.zeros(N, bool)
        self.n_total = np.zeros((N, D), np.int64)
        self.n_foreign = np.zeros((N, D), np.int64)      # occupied by pods the scheduler does not own
        self.n_used = np.zeros((N, D), np.int64)         # what this scheduler's allocations hold (per index)
        self.n_taint = np.zeros(N, np.uint64)
        self.n_label = np.zeros(N, np.uint64)
        self.n_num = np.zeros(N, np.int64)               # NodeID number = name rank
        self.n_flags = np.zeros(N, np.uint32)
        self.n_hi = 0
        self.used_nums = set()
        self.a_state = np.full(A, ABSENT, np.int64)      # ABSENT / PENDING / ALLOCATED
        self.a_req = np.zeros((A, D), np.int64)
        self.a_tol = np.zeros(A, np.uint64)
        self.a_need = np.zeros(A, np.uint64)
        self.a_deny = np.zeros(A, np.uint64)
        self.a_prio = np.zeros(A, np.int32)
        self.a_create = np.zeros(A, np.int64)
        self.a_app = np.zeros(A, np.int64)
        self.a_flags = np.zeros(A, np.uint32)
        self.a_gang = np.full(A, -1, np.int64)
        self.a_bound = np.full(A, -1, np.int64)
        self.a_last = np.full(A, ABSENT, np.int64)       # oracle state of the last uncut cycle
        self.a_hi = 0
        self.p_present = np.zeros(P, bool)
        self.p_queue = np.zeros(P, np.int64)
        self.p_submit = np.zeros(P, np.int64)
        self.p_user = np.full(P, -1, np.int64)
        self.q_guar = np.full((self.maxQ, D), -1, np.int64)
        self.q_max = np.full((self.maxQ, D), -1, np.int64)
        self.q_sort = np.zeros(self.maxQ, np.uint8)
        self.q_prio_offset = None
        self.q_prio_fence = None
        self.ul = []                                    # user-limit entries: (queue, user, max[D])
        self.seq = 0                                    # global counter: create_seq and submit times are unique
        self.gang_seq = 0
        self.steps = []                                 # ("op", method, kwargs, text) / ("cycle", Cycle)
        self.count = {}                                 # operations and interleavings generated
        self.cycles = 0
        self.since = []                                 # op texts since the last cycle
        self.removed_below_hi = False

    # ---- bookkeeping ----
    def note(self, key, n=1):
        self.count[key] = self.count.get(key, 0) + n

    def _op(self, method, text, **kw):
        self.steps.append(("op", method, kw, text))
        self.since.append(method)

    def _seq(self):
        self.seq += 1
        return self.seq

    def new_num(self):
        while True:
            x = int(self.rng.integers(1, 999_999))
            if x not in self.used_nums:
                self.used_nums.add(x)
                return x

    def avail(self, n):
        return self.n_total[n] - self.n_foreign[n] - self.n_used[n]

    def chain(self, q):
        while q >= 0:
            yield int(q)
            q = int(Q_PARENT[q])

    def q_alloc(self):
        qa = np.zeros((self.maxQ, self.D), np.int64)
        for a in np.nonzero(self.a_state == ALLOCATED)[0]:
            for q in self.chain(self.p_queue[self.a_app[a]]):
                qa[q] += self.a_req[a]
        return qa

    def held(self):
        h = np.zeros((len(self.ul), self.D), np.int64)
        for a in np.nonzero(self.a_state == ALLOCATED)[0]:
            p = self.a_app[a]
            for i, (q, u, _) in enumerate(self.ul):
                if self.p_user[p] == u and q in set(self.chain(self.p_queue[p])):
                    h[i] += self.a_req[a]
        return h

    def present_nodes(self):
        return np.nonzero(self.n_present)[0]

    def free_node_indices(self):
        """indices below n_hi no node occupies and no allocation points at (a new node may take them)"""
        bound = set(self.a_bound[self.a_state == ALLOCATED].tolist())
        return [n for n in range(self.n_hi) if not self.n_present[n] and n not in bound]

    def pending(self):
        """pending asks of present applications, ascending index"""
        return np.array([a for a in np.nonzero(self.a_state == PENDING)[0] if self.p_present[self.a_app[a]]], np.int64)

    # ---- operations (each mirrors the Engine method of the same name) ----
    def nodes_upsert(self, idx, text="nodes_upsert"):
        idx = np.asarray(idx, np.int64)
        for n in idx:
            self.n_present[n] = True
            self.n_hi = max(self.n_hi, int(n) + 1)
        contiguous = len(idx) == 1 or bool((np.diff(idx) == 1).all())
        self.note("upsert_contiguous" if contiguous else "upsert_scattered")
        self._op("nodes_upsert", text, idx=idx.copy(), total=self.n_total[idx].copy(),
                 avail=np.stack([self.avail(n) for n in idx]), taint_bits=self.n_taint[idx].copy(),
                 label_bits=self.n_label[idx].copy(), name_rank=self.n_num[idx].copy(), flags=self.n_flags[idx].copy())

    def set_node(self, n, total, foreign=None, taint=0, label=0, flags=SCHED, num=None):
        self.n_total[n] = total
        self.n_foreign[n] = 0 if foreign is None else foreign
        self.n_taint[n], self.n_label[n], self.n_flags[n] = taint, label, flags
        if num is None:
            num = self.new_num()
        self.n_num[n] = num

    def nodes_remove(self, idx):
        idx = np.asarray(idx, np.int64)
        if any(self.n_used[n].any() for n in idx):
            self.note("remove_with_allocations")
        if any(n < self.n_hi - 1 for n in idx):
            self.note("remove_below_hi")
            self.removed_below_hi = True
        self.n_present[idx] = False
        self._op("nodes_remove", "nodes_remove", idx=idx.copy())

    def rename(self, idx, nums):
        """give nodes new NodeIDs (new rank numbers); nothing else changes"""
        for n, x in zip(idx, nums):
            self.used_nums.add(int(x))
            self.n_num[n] = x
        self.nodes_upsert(idx, "rename")

    def apps_upsert(self, idx, queue, user=-1):
        idx = np.atleast_1d(np.asarray(idx, np.int64))
        queue = np.broadcast_to(np.asarray(queue, np.int64), idx.shape).copy()
        user = np.broadcast_to(np.asarray(user, np.int64), idx.shape).copy()
        submit = np.array([1_700_000_000 + self._seq() for _ in idx], np.int64)
        for p, q, u, s in zip(idx, queue, user, submit):
            self.p_present[p], self.p_queue[p], self.p_submit[p], self.p_user[p] = True, q, s, u
        self._op("apps_upsert", "apps_upsert", idx=idx, queue=queue, submit_time=submit)
        self._op("apps_user", "apps_user", idx=idx, user=user)

    def apps_remove(self, idx):
        idx = np.atleast_1d(np.asarray(idx, np.int64))
        for p in idx:
            assert not ((self.a_app == p) & (self.a_state == ALLOCATED)).any(), "an application with allocations"
            if ((self.a_app == p) & (self.a_state == PENDING)).any():
                self.note("app_removed_with_pending")
            self.p_present[p] = False
        self._op("apps_remove", "apps_remove", idx=idx)

    def asks_upsert(self, idx, req, app, tol=0, need=0, deny=0, prio=0, flags=0, gang=-1, text="asks_upsert"):
        idx = np.atleast_1d(np.asarray(idx, np.int64))
        k = len(idx)
        req = np.asarray(req, np.int64).reshape(-1, self.D)
        req = np.broadcast_to(req, (k, self.D)).copy()

        def col(x, dt):
            return np.broadcast_to(np.asarray(x, dt), (k,)).copy()
        app, tol, need, deny = col(app, np.int64), col(tol, np.uint64), col(need, np.uint64), col(deny, np.uint64)
        prio, flags, gang = col(prio, np.int32), col(flags, np.uint32), col(gang, np.int64)
        create = np.array([self._seq() for _ in idx], np.int64)
        for i, a in enumerate(idx):
            assert self.a_state[a] != ALLOCATED and self.p_present[app[i]]
            self.a_state[a] = PENDING
            self.a_req[a], self.a_tol[a], self.a_need[a], self.a_deny[a] = req[i], tol[i], need[i], deny[i]
            self.a_prio[a], self.a_create[a], self.a_app[a], self.a_flags[a], self.a_gang[a] = prio[i], create[i], app[i], flags[i], gang[i]
            self.a_bound[a] = -1
            self.a_last[a] = PENDING
            self.a_hi = max(self.a_hi, int(a) + 1)
        self._op("asks_upsert", text, idx=idx, req=req, app=app, create_seq=create, tolerated_bits=tol, required_bits=need,
                 forbidden_bits=deny, priority=prio, flags=flags, gang=gang)

    def asks_remove(self, idx):
        idx = np.atleast_1d(np.asarray(idx, np.int64))
        assert (self.a_state[idx] == PENDING).all()
        self.a_state[idx] = ABSENT
        self._op("asks_remove", "asks_remove", idx=idx)

    def release(self, idx, text="release"):
        idx = np.atleast_1d(np.asarray(idx, np.int64))
        assert (self.a_state[idx] == ALLOCATED).all()
        for a in idx:
            n = self.a_bound[a]
            if not self.n_present[n]:
                self.note("release_on_removed_node")
            self.n_used[n] -= self.a_req[a]                # the engine gives back only to a present node: a removed node's
            self.a_state[a], self.a_bound[a] = ABSENT, -1   # index is never reused while an allocation points at it
            if self.a_gang[a] >= 0:
                self.note("release_gang_member")
        self._op("release", text, ask_idx=idx)

    def queues_set(self, guar, mx, sort):
        self.q_guar, self.q_max, self.q_sort = np.asarray(guar, np.int64), np.asarray(mx, np.int64), np.asarray(sort, np.uint8)
        self.q_prio_offset = self.q_prio_fence = None     # yk_queues_set resets the priority properties
        self._op("queues_set", "queues_set", parent=Q_PARENT.copy(), guaranteed=self.q_guar.copy(), max=self.q_max.copy(),
                 allocated=None, sort=self.q_sort.copy())

    def queues_priority(self, offset, fence):
        self.q_prio_offset, self.q_prio_fence = np.asarray(offset, np.int32), np.asarray(fence, np.uint8)
        self._op("queues_priority", "queues_priority", offset=self.q_prio_offset.copy(), fence=self.q_prio_fence.astype(bool))

    def user_limits_set(self, entries):
        self.ul = [(int(q), int(u), np.asarray(m, np.int64)) for q, u, m in entries]
        n = len(self.ul)
        self._op("user_limits_set", "user_limits_set", queue=np.array([e[0] for e in self.ul], np.uint32),
                 user=np.array([e[1] for e in self.ul], np.uint32),
                 max=np.array([e[2] for e in self.ul], np.int64).reshape(n, self.D), held=self.held())

    # ---- the cycle ----
    def snapshot(self):
        """-> (compacted Snapshot of the pending world, engine ask index per snapshot ask, engine node index per snapshot node)"""
        D = self.D
        nodes = self.present_nodes()
        asks = self.pending()
        apps = np.nonzero(self.p_present)[0]
        app_pos = {int(p): i for i, p in enumerate(apps)}
        avail = np.stack([self.avail(n) for n in nodes]) if len(nodes) else np.zeros((0, D), np.int64)
        s = synth.Snapshot(
            D=D, policy=self.policy, weights=self.weights.copy(),
            node_total=self.n_total[nodes].copy(), node_avail=avail, node_taint=self.n_taint[nodes].copy(),
            node_label=self.n_label[nodes].copy(), node_flags=self.n_flags[nodes].copy(),
            node_id=[f"n{int(x):06d}" for x in self.n_num[nodes]],
            q_parent=Q_PARENT.copy(), q_guaranteed=self.q_guar.copy(), q_max=self.q_max.copy(), q_alloc=self.q_alloc(),
            q_sort=self.q_sort.copy(),
            app_queue=self.p_queue[apps].astype(np.int32), app_submit=self.p_submit[apps].copy(),
            ask_app=np.array([app_pos[int(p)] for p in self.a_app[asks]], np.int32), ask_req=self.a_req[asks].copy(),
            ask_tol=self.a_tol[asks].copy(), ask_need=self.a_need[asks].copy(), ask_deny=self.a_deny[asks].copy(),
            ask_prio=self.a_prio[asks].copy(), ask_create=self.a_create[asks].copy(),
            ask_node=np.full(len(asks), -1, np.int32), ask_flags=self.a_flags[asks].copy(),
            ask_gang=self.a_gang[asks].astype(np.int32), name=f"{self.name}-c{self.cycles}",
            q_prio_offset=None if self.q_prio_offset is None else self.q_prio_offset.copy(),
            q_prio_fence=None if self.q_prio_fence is None else self.q_prio_fence.copy())
        if self.ul:
            s.app_user = self.p_user[apps].astype(np.int32)
            s.ul_queue = np.array([e[0] for e in self.ul], np.int32)
            s.ul_user = np.array([e[1] for e in self.ul], np.int32)
            s.ul_max = np.array([e[2] for e in self.ul], np.int64).reshape(len(self.ul), D)
            s.ul_alloc = self.held()
        return s, asks, nodes

    def preview(self):
        """the oracle's uncut cycle on the current state, engine indices; the model does not change"""
        s, amap, nmap = self.snapshot()
        w = self.oracle.run(s)
        return amap[w["ask"]], nmap[w["node"]], w

    def cycle(self, max_bindings=None, kind=None):
        s, amap, nmap = self.snapshot()
        want = self.oracle.run(s, -1 if max_bindings is None else max_bindings)
        ask, node = amap[want["ask"]], nmap[want["node"]]
        cut = max_bindings is not None
        self.note("mb_" + (kind or ("unlimited" if not cut else "given")))
        if self.since == ["release"]:
            self.note("release_then_cycle")
        if self.removed_below_hi:
            self.note("cycle_after_removal_below_hi")
            self.removed_below_hi = False
        for a, n in zip(ask, node):
            if self.a_last[a] == NOFIT:
                self.note("nofit_then_fit")
            self.a_state[a], self.a_bound[a] = ALLOCATED, n
            self.n_used[n] += self.a_req[a]
        present = self.present_nodes()
        avail = np.stack([self.avail(n) for n in present]) if len(present) else np.zeros((0, self.D), np.int64)
        states = None
        if not cut:
            states = self.a_state.copy()                # ABSENT / ALLOCATED / PENDING (asks of removed applications)
            states[amap] = want["state"]
            self.a_last[amap] = want["state"]
        else:
            self.a_last[amap] = np.where(self.a_state[amap] == ALLOCATED, ALLOCATED, PENDING)
        scores = np.array([self.oracle.node_score(self.policy, self.weights, self.n_total[n], self.avail(n)) for n in present])
        runs = _longest_run(s)
        self.steps.append(("cycle", Cycle(number=self.cycles, snap=s, amap=amap, nmap=nmap, max_bindings=max_bindings,
                                          ask=ask, node=node, states=states, present=present, avail=avail, scores=scores,
                                          oracle_avail=nmap_avail(want["avail"], nmap, present), has_gang=bool((s.ask_gang >= 0).any()),
                                          eligible=self.policy == synth.POLICY_FAIR and _one_request_per_gang(s),
                                          pending=len(amap), longest_run=runs, recent=list(self.since[-6:]),
                                          absent=np.nonzero(self.a_state == ABSENT)[0][:2])))
        self.cycles += 1
        self.since = []
        return ask, node, want

    # ---- invariant ----
    def check_conservation(self):
        """what the model's allocations hold is exactly what the nodes, queues and users account for"""
        used = np.zeros_like(self.n_used)
        for a in np.nonzero(self.a_state == ALLOCATED)[0]:
            assert self.a_bound[a] >= 0 and self.p_present[self.a_app[a]], (self.name, int(a))
            used[self.a_bound[a]] += self.a_req[a]
        assert np.array_equal(used, self.n_used), self.name
        qa = self.q_alloc()
        assert (qa >= 0).all() and np.array_equal(qa[0], qa[1] + qa[2]), self.name
        assert np.array_equal(qa[1], qa[3] + qa[4]) and np.array_equal(qa[2], qa[5]), self.name
        assert (self.held() >= 0).all(), self.name
        assert (self.a_state[self.a_hi:] == ABSENT).all()


def _one_request_per_gang(s):
    first = {}
    for i in range(s.n_asks):
        if s.ask_gang[i] >= 0 and not np.array_equal(first.setdefault((int(s.ask_app[i]), int(s.ask_gang[i])), s.ask_req[i]), s.ask_req[i]):
            return False
    return True


def nmap_avail(avail, nmap, present):
    pos = {int(n): i for i, n in enumerate(nmap)}
    return np.stack([avail[pos[int(n)]] for n in present]) if len(present) else np.zeros((0, avail.shape[1]), np.int64)


def _longest_run(s):
    """longest run of consecutive pending asks of one application with one request and one predicate signature"""
    best = run = 0
    prev = None
    for i in range(s.n_asks):
        key = (int(s.ask_app[i]), s.ask_req[i].tobytes(), int(s.ask_tol[i]), int(s.ask_need[i]), int(s.ask_deny[i]),
               int(s.ask_prio[i]), int(s.ask_gang[i]))
        run = run + 1 if key == prev else 1
        prev = key
        best = max(best, run)
    return best


# ---- the seeded session generator ----
def _node_shape(rng, D):
    t = np.zeros(D, np.int64)
    t[0] = int(rng.integers(2, 9)) * 1000
    if D > 1:
        t[1] = int(rng.integers(4, 33)) * GI
    if D > 2:
        t[2] = int(rng.integers(6, 20))
    for k in range(3, D):
        t[k] = int(rng.integers(1, 5)) * 1000
    return t


def _ask_shape(rng, D):
    r = np.zeros(D, np.int64)
    r[0] = int(rng.choice([100, 250, 500, 1000, 2000]))
    if D > 1:
        r[1] = int(rng.choice([256 << 20, GI, 2 * GI, 4 * GI]))
    if D > 2:
        r[2] = 1
    for k in range(3, D):
        r[k] = int(rng.choice([0, 100, 400]))
    if rng.random() < 0.02:
        r[:] = 0                                       # nothing requested: INVALID
    return r


def _random_node(m, n, rng, tied_shape=None):
    if tied_shape is not None:
        m.set_node(n, tied_shape, taint=0, label=1)
        return
    t = _node_shape(rng, m.D)
    foreign = np.zeros(m.D, np.int64)
    if rng.random() < 0.3:
        foreign[0] = int(rng.integers(0, t[0] // 1000)) * 500
    taint = np.uint64(1 << int(rng.integers(0, 3))) if rng.random() < 0.2 else 0
    label = np.uint64((1 << int(rng.integers(0, 3))) | 8)
    flags = SCHED if rng.random() > 0.05 else 0
    m.set_node(n, t, foreign, taint, label, flags)


class Generator:
    def __init__(self, m, rng, big=0):
        self.m, self.rng, self.big = m, rng, big

    # nodes
    def add_nodes(self, k, tied=False):
        m, rng = self.m, self.rng
        free = m.free_node_indices()
        if free and rng.random() < 0.5:
            idx = sorted(rng.choice(free, min(k, len(free)), replace=False).tolist())
            m.note("nodes_new_reused_index")
        else:
            k = min(k, m.maxN - m.n_hi)
            if k <= 0:
                return
            idx = list(range(m.n_hi, m.n_hi + k))
            m.note("nodes_new_fresh_index")
        shape = _node_shape(rng, m.D) if tied else None
        for n in idx:
            _random_node(m, n, rng, shape)
        if tied:
            m.note("nodes_new_tied_group")
        m.nodes_upsert(idx, "nodes_upsert(new)")

    def change_nodes(self):
        m, rng = self.m, self.rng
        pres = m.present_nodes()
        if not len(pres):
            return
        idx = sorted(rng.choice(pres, min(len(pres), int(rng.integers(1, 5))), replace=False).tolist())
        for n in idx:
            what = rng.integers(0, 6)
            if what == 0:
                m.n_total[n, 0] = max(1000, m.n_total[n, 0] + int(rng.integers(-2, 3)) * 1000)
                m.note("node_resize")
            elif what == 1:
                m.n_foreign[n, 0] = int(rng.integers(0, 4)) * 500
                m.note("node_foreign_occupancy")
            elif what == 2:
                m.n_flags[n] ^= SCHED
                m.note("node_cordon" if not m.n_flags[n] & SCHED else "node_uncordon")
            elif what == 3:
                m.n_flags[n] ^= RESERVED
                m.note("node_reserved")
            elif what == 4:
                m.n_taint[n] = np.uint64(1 << int(rng.integers(0, 3))) if m.n_taint[n] == 0 else np.uint64(0)
                m.note("node_taint")
            else:
                m.n_label[n] = np.uint64(m.n_label[n] ^ np.uint64(1 << int(rng.integers(0, 3))))
                m.note("node_label")
        m.nodes_upsert(idx, "nodes_upsert(change)")

    def rename_tied(self):
        """nodes of one shape with nothing on them score the same: their order is their NodeID order.  Reverse it."""
        m = self.m
        groups = {}
        for n in m.present_nodes():
            if m.n_used[n].any() or m.n_foreign[n].any():
                continue
            key = (m.n_total[n].tobytes(), int(m.n_taint[n]), int(m.n_label[n]), int(m.n_flags[n]))
            groups.setdefault(key, []).append(int(n))
        groups = [g for g in groups.values() if len(g) >= 2]
        if not groups:
            return False
        g = groups[int(self.rng.integers(0, len(groups)))]
        first = min(g, key=lambda n: m.n_num[n])
        if self.rng.random() < 0.5:                   # the NodeID-first node goes last: one node, contiguous path
            mx = int(max(m.n_num[g]))
            cand = mx + 1 + int(self.rng.integers(0, 50))
            m.rename([first], [cand if cand < 999_999 and cand not in m.used_nums else m.new_num()])
        else:                                          # every member gets a new number, the order reversed
            nums = sorted(m.new_num() for _ in g)
            order = sorted(g, key=lambda n: m.n_num[n])
            m.rename(sorted(g), [nums[len(g) - 1 - order.index(n)] for n in sorted(g)])
        m.note("rename_tied")
        return True

    def rename_busy(self):
        m = self.m
        busy = [int(n) for n in m.present_nodes() if m.n_used[n].any()]
        if not busy:
            return
        n = busy[int(self.rng.integers(0, len(busy)))]
        m.rename([n], [m.new_num()])
        m.note("rename_with_allocations")

    def remove_nodes(self, k):
        m, rng = self.m, self.rng
        pres = m.present_nodes()
        if len(pres) <= 3:
            return
        m.nodes_remove(sorted(rng.choice(pres, min(k, len(pres) - 3), replace=False).tolist()))

    # asks
    def ask_indices(self, k):
        m, rng = self.m, self.rng
        free = [a for a in range(m.a_hi) if m.a_state[a] == ABSENT]
        if free and (rng.random() < 0.35 or m.a_hi + k > m.maxA):
            k = min(k, len(free))
            m.note("asks_reused_index")
            return sorted(rng.choice(free, k, replace=False).tolist())
        k = min(k, m.maxA - m.a_hi)
        return list(range(m.a_hi, m.a_hi + k))

    def new_asks(self):
        m, rng = self.m, self.rng
        apps = np.nonzero(m.p_present)[0]
        if not len(apps):
            return
        p = int(rng.choice(apps))
        kind = rng.random()
        tol = np.uint64(7) if rng.random() < 0.7 else np.uint64(int(rng.integers(0, 8)))
        need = np.uint64(1 << int(rng.integers(0, 3))) if rng.random() < 0.15 else 0
        deny = np.uint64(2) if rng.random() < 0.1 else 0
        prio = int(rng.integers(-1, 2)) * 10 if rng.random() < 0.3 else 0
        if kind < 0.25:                                # a run of identical asks: the uniform-run path
            idx = self.ask_indices(int(rng.integers(UNIFORM_MIN, 2 * UNIFORM_MIN + 5)))
            if idx:
                m.asks_upsert(idx, _ask_shape(rng, m.D), p, tol, need, deny, prio, text="asks_upsert(run)")
                m.note("asks_uniform_run")
        elif kind < 0.45:                              # a gang: identical members, all or nothing
            idx = self.ask_indices(int(rng.integers(2, 5)))
            if len(idx) >= 2:
                m.gang_seq += 1
                m.asks_upsert(idx, _ask_shape(rng, m.D), p, tol, need, deny, prio, gang=m.gang_seq, text="asks_upsert(gang)")
                m.note("asks_gang")
        else:
            idx = self.ask_indices(int(rng.integers(1, 10)))
            if idx:
                req = np.stack([_ask_shape(rng, m.D) for _ in idx])
                flags = (rng.random(len(idx)) < 0.03).astype(np.uint32)
                m.asks_upsert(idx, req, p, tol, need, deny, prio, flags=flags)
                m.note("asks_new")

    def reupsert_asks(self):
        m, rng = self.m, self.rng
        cand = [a for a in np.nonzero(m.a_state == PENDING)[0] if m.a_gang[a] < 0 and m.p_present[m.a_app[a]]]
        if not cand:
            return
        idx = sorted(rng.choice(cand, min(len(cand), int(rng.integers(1, 6))), replace=False).tolist())
        for a in idx:
            req, tol, need, deny = m.a_req[a].copy(), m.a_tol[a], m.a_need[a], m.a_deny[a]
            what = rng.integers(0, 3)
            if what == 0:
                req = _ask_shape(rng, m.D)
            elif what == 1:
                tol = np.uint64(int(rng.integers(0, 8)))
            else:
                need = np.uint64(1 << int(rng.integers(0, 3))) if need == 0 else np.uint64(0)
            m.asks_upsert([a], req, m.a_app[a], tol, need, deny, m.a_prio[a], m.a_flags[a], text="asks_upsert(re-upsert)")
        m.note("asks_reupsert")

    def remove_asks(self):
        m, rng = self.m, self.rng
        cand = np.nonzero(m.a_state == PENDING)[0]
        if len(cand):
            m.asks_remove(sorted(rng.choice(cand, min(len(cand), int(rng.integers(1, 6))), replace=False).tolist()))
            m.note("asks_remove")

    def release(self):
        m, rng = self.m, self.rng
        alloc = np.nonzero(m.a_state == ALLOCATED)[0]
        if len(alloc):
            frac = rng.random() * 0.5
            sel = [int(a) for a in alloc if rng.random() < frac] or [int(rng.choice(alloc))]
            gone = [int(a) for a in alloc if not m.n_present[m.a_bound[a]]]
            m.release(sorted(set(sel) | set(gone[:2])))
            m.note("release")

    # applications, queues, limits
    def new_app(self):
        m, rng = self.m, self.rng
        live = set(m.a_app[:m.a_hi][m.a_state[:m.a_hi] != ABSENT].tolist())
        free = [p for p in range(m.maxP) if not m.p_present[p] and p not in live]
        if free:
            m.apps_upsert([free[0]], int(rng.choice(LEAVES)), int(rng.integers(-1, 3)))
            m.note("apps_upsert")

    def remove_app(self):
        m, rng = self.m, self.rng
        cand = [p for p in np.nonzero(m.p_present)[0] if not ((m.a_app == p) & (m.a_state == ALLOCATED)).any()]
        if len(np.nonzero(m.p_present)[0]) <= 2 or not cand:
            return
        p = int(rng.choice(cand))
        pend = np.nonzero((m.a_app == p) & (m.a_state == PENDING))[0]
        if len(pend) and rng.random() < 0.75:          # what the shim does: the pods go first
            m.asks_remove(pend)
        m.apps_remove([p])
        m.note("apps_remove")

    def queues(self, first=False):
        m, rng = self.m, self.rng
        guar = np.full((m.maxQ, m.D), -1, np.int64)
        mx = np.full((m.maxQ, m.D), -1, np.int64)
        for q in range(1, m.maxQ):
            if rng.random() < 0.5:
                guar[q, 0] = int(rng.integers(1, 20)) * 1000
            if rng.random() < 0.35:
                mx[q, 0] = int(rng.integers(3, 40)) * 1000
            if m.D > 2 and rng.random() < 0.15:
                mx[q, 2] = int(rng.integers(5, 40))
        # fifo leaves only: a fair leaf orders its applications by what each has held since earlier cycles, and the oracle's
        # snapshot has no per-application allocation to start from (it would start every application at zero)
        m.queues_set(guar, mx, np.zeros(m.maxQ, np.uint8))
        if not first:
            m.note("queues_set")

    def priorities(self):
        m, rng = self.m, self.rng
        m.queues_priority(rng.integers(-1, 2, m.maxQ) * 50, rng.random(m.maxQ) < 0.2)
        m.note("queues_priority")

    def limits(self):
        m, rng = self.m, self.rng
        ent = []
        for q in (1, 3, 4, 5):
            for u in range(3):
                if rng.random() < 0.3:
                    mx = np.full(m.D, -1, np.int64)
                    mx[0] = int(rng.integers(1, 15)) * 1000
                    ent.append((q, u, mx))
        m.user_limits_set(ent)
        m.note("user_limits_set")

    def max_bindings(self):
        """unlimited, 1, a random value, a value inside a gang, or 0 -> (max_bindings, kind)"""
        m, rng = self.m, self.rng
        x = rng.random()
        if x < 0.5:
            return None, "unlimited"
        if x < 0.6:
            return 1, "one"
        if x < 0.65:
            return 0, "zero"
        ask, _, _ = m.preview()
        if x < 0.85:
            pos = [i for i in range(1, len(ask)) if m.a_gang[ask[i]] >= 0 and m.a_gang[ask[i]] == m.a_gang[ask[i - 1]]]
            if pos:
                return int(pos[int(rng.integers(0, len(pos)))]), "gang_cut"
        return int(rng.integers(1, max(2, len(ask) + 2))), "random"

    def step(self):
        m, rng, big = self.m, self.rng, self.big
        if big:                                        # live node count swings across a tile boundary (256 / 512 nodes)
            live = len(m.present_nodes())
            if live < big or (live < big + 30 and rng.random() < 0.5):
                self.add_nodes(int(rng.integers(20, 40)))
                if len(m.present_nodes()) > big >= live:
                    m.note("tile_crossed_up")
            else:
                self.remove_nodes(int(rng.integers(20, 40)))
                if len(m.present_nodes()) <= big < live:
                    m.note("tile_crossed_down")
        ops = [
            (0.25, lambda: self.add_nodes(int(rng.integers(1, 5)), tied=rng.random() < 0.4)),
            (0.35, self.change_nodes),
            (0.25, self.rename_tied),
            (0.10, self.rename_busy),
            (0.15, lambda: self.remove_nodes(int(rng.integers(1, 4)))),
            (0.70, self.new_asks),
            (0.35, self.new_asks),
            (0.15, self.reupsert_asks),
            (0.15, self.remove_asks),
            (0.40, self.release),
            (0.10, self.new_app),
            (0.08, self.remove_app),
            (0.08, self.queues),
            (0.05, self.priorities),
            (0.07, self.limits),
        ]
        if rng.random() < 0.12:                        # a release, and nothing else, before the cycle
            self.release()
            return
        for p, fn in ops:
            if rng.random() < p:
                fn()

    def start(self, n_nodes, n_apps=4):
        m, rng = self.m, self.rng
        self.queues(first=True)
        m.apps_upsert(list(range(n_apps)), [LEAVES[i % 3] for i in range(n_apps)], [i % 3 - (i == 3) for i in range(n_apps)])
        tied = int(rng.integers(3, 7))
        shape = _node_shape(rng, m.D)
        for n in range(n_nodes):
            _random_node(m, n, rng, shape if n < tied else None)
        m.nodes_upsert(list(range(n_nodes)), "nodes_upsert(initial)")
        for _ in range(3):
            self.new_asks()
        if rng.random() < 0.5:
            self.limits()


def random_session(oracle, seed, D=4, policy=synth.POLICY_FAIR, big=0):
    rng = np.random.default_rng([seed, D, policy, big])
    m = Model(oracle, f"session(seed={seed}, D={D}, policy={policy}, big={big})", D, policy,
              max_nodes=(big + 160) if big else 128, max_asks=1024, seed=seed + 1000 * D)
    g = Generator(m, rng, big)
    g.start(big - 10 if big else int(rng.integers(12, 40)))
    n_cycles = int(rng.integers(12, 31))
    for c in range(n_cycles):
        if c:
            g.step()
        m.check_conservation()
        m.cycle(*g.max_bindings())
        m.check_conservation()
    finish(m)
    return m


def finish(m):
    """release everything still allocated: every present node is back at its base value; a final uncut cycle"""
    alloc = np.nonzero(m.a_state == ALLOCATED)[0]
    if len(alloc):
        m.release(alloc, "release(all)")
    for n in m.present_nodes():
        assert np.array_equal(m.avail(n), m.n_total[n] - m.n_foreign[n]), (m.name, int(n))
    m.steps.append(("conserved", None))
    m.cycle(None, "final")
    m.check_conservation()


SEEDS = range(20)
EXTRA = [(s, 1, synth.POLICY_FAIR, 0) for s in (100, 101)] + [(s, 8, synth.POLICY_FAIR, 0) for s in (102, 103)] \
    + [(s, 4, synth.POLICY_BINPACKING, 0) for s in (104, 105, 106)]
BIG = [(110, 4, synth.POLICY_FAIR, 256), (111, 4, synth.POLICY_FAIR, 512)]
ALL = [(s, 4, synth.POLICY_FAIR, 0) for s in SEEDS] + EXTRA + BIG


@functools.lru_cache(maxsize=None)
def session(seed, D=4, policy=synth.POLICY_FAIR, big=0):
    from oracle import oracle_ctypes
    oracle_ctypes.build()
    return random_session(oracle_ctypes, seed, D, policy, big)


# ---- replay on the engine ----
def _engine(m, commit, batch):
    from yunikorn_k8shim_b200 import Engine
    return Engine(D=m.D, policy=m.policy, weights=m.weights, max_nodes=m.maxN, max_asks=m.maxA, max_apps=m.maxP,
                  max_queues=m.maxQ, batch=batch, commit=commit)


def _stats_ok(m, c, commit, d, where):
    assert d["cycles"] == 1 and d["allocations"] == len(c.ask), where
    lat = d["lattice_cycles"]
    if commit == "host" or not c.eligible:
        assert lat == 0 and d["lattice_launches"] == 0 and d["uniform_asks"] == 0, (where, d)
    elif commit == "device":
        assert lat == 1, (where, d)                    # fair sort, one request per gang: every such cycle starts on the device
    else:
        assert lat in (0, 1) and (lat or d["uniform_asks"] == 0), (where, d)
    assert d["lattice_handoffs"] <= lat and (d["lattice_handoffs"] == 0 or c.has_gang), (where, d)


def replay(m, commit="host", batch=64, filter_k=None, on_cycle=None):
    """drive an engine through the model's script; after every cycle compare with the model.  -> per-cycle outputs"""
    outs = []
    totals = {}
    with _engine(m, commit, batch) as e:
        for step in m.steps:
            if step[0] == "op":
                _, method, kw, _text = step
                getattr(e, method)(**kw)
                continue
            if step[0] == "conserved":
                pres = m.present_nodes()
                got = e.nodes_available(pres)
                assert np.array_equal(got, m.n_total[pres] - m.n_foreign[pres]), f"{m.name}: not back at base after release(all)"
                continue
            c = step[1]
            where = f"{m.name} [{commit}, batch {batch}] cycle {c.number} (max_bindings {c.max_bindings}; ops before: {c.recent})"
            if filter_k is not None:
                _filter_check(e, m, c, filter_k, where)
            before = e.stats()
            ask, node, _ = e.cycle(m.maxA if c.max_bindings is None else c.max_bindings)
            d = {k: v for k, v in e.stats().items() if not isinstance(v, list)}
            d = {k: v - before[k] for k, v in d.items()}
            assert ask.tolist() == c.ask.tolist(), f"{where}: ask order differs\n got {ask.tolist()}\nwant {c.ask.tolist()}"
            assert node.tolist() == c.node.tolist(), f"{where}: node choice differs\n got {node.tolist()}\nwant {c.node.tolist()}"
            avail = e.nodes_available(c.present)
            assert np.array_equal(avail, c.avail), f"{where}: nodes_available differs at {c.present[(avail != c.avail).any(1)].tolist()}"
            scores = e.node_scores(c.present)
            bad = np.nonzero(scores.view(np.int64) != c.scores.view(np.int64))[0]
            assert not len(bad), f"{where}: device node scores differ at {c.present[bad].tolist()}"
            states = e.ask_states(np.arange(m.maxA))
            if c.states is not None:
                wrong = np.nonzero(states != c.states)[0]
                assert not len(wrong), f"{where}: ask states differ at {wrong[:8].tolist()}: got {states[wrong[:8]].tolist()} want {c.states[wrong[:8]].tolist()}"
            _stats_ok(m, c, commit, d, where)
            for k in ("lattice_cycles", "uniform_asks", "lattice_handoffs", "uniform_retries", "sweep_launches"):
                totals[k] = totals.get(k, 0) + d[k]
            outs.append((ask, node, avail, scores, states if c.states is not None else None))
            if on_cycle:
                on_cycle(e, c, d)
    return outs, totals


def _filter_check(e, m, c, k, where):
    """yk_filter_nodes between ops and the cycle, against the oracle's order and predicates on the model's state"""
    from test_filter import expect, window
    from oracle import oracle_ctypes as oc
    s = c.snap
    pick = list(range(0, s.n_asks, max(1, s.n_asks // 12)))[:12]
    asks = np.array([int(c.amap[i]) for i in pick] + c.absent.tolist(), np.uint32)
    before = e.stats()["other_launches"]
    skip = int(c.number % 3) * 7
    nodes, n_pass, counts = e.filter_nodes(asks, k=k, skip=skip)
    assert e.stats()["other_launches"] > before, where
    full, want = expect(oc, s, pick) if pick else ([], np.zeros((0, 11), np.uint32))
    for i in range(len(pick)):
        eng = [int(c.nmap[x]) for x in full[i]]
        assert counts[i].tolist() == want[i].tolist(), f"{where}: filter counts of ask {int(asks[i])}"
        assert n_pass[i] == len(eng) and nodes[i].tolist() == window(eng, skip, k), f"{where}: filter candidates of ask {int(asks[i])}"
    for i in range(len(pick), len(asks)):
        assert counts[i, 9] == len(c.present) and n_pass[i] == 0, f"{where}: absent ask {int(asks[i])}"


# ---- GPU: session parity ----
@pytest.mark.gpu
@pytest.mark.parametrize("batch", [7, 64, 4096])
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
@pytest.mark.parametrize("seed", SEEDS)
def test_session_parity(monkeypatch, seed, commit, batch):
    monkeypatch.setenv("YK_UNIFORM_MIN", str(UNIFORM_MIN))
    replay(session(seed), commit, batch)


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device"])
@pytest.mark.parametrize("seed,D,policy,big", EXTRA, ids=[f"seed{s}-D{d}-policy{p}" for s, d, p, _ in EXTRA])
def test_session_parity_other_shapes(monkeypatch, seed, D, policy, big, commit):
    """D = 1 and D = 8, and binpacking (never eligible for the device commit: the device engine must stay on the host commit)"""
    monkeypatch.setenv("YK_UNIFORM_MIN", str(UNIFORM_MIN))
    replay(session(seed, D, policy, big), commit, 64)


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [0, 3, 7, 11])
def test_three_engines_in_lockstep(monkeypatch, seed):
    """host, device and auto engines driven by one session give identical outputs at every cycle"""
    monkeypatch.setenv("YK_UNIFORM_MIN", str(UNIFORM_MIN))
    m = session(seed)
    runs = {c: replay(m, c, 64)[0] for c in ("host", "device", "auto")}
    for i, (h, d, a) in enumerate(zip(runs["host"], runs["device"], runs["auto"])):
        for x, y, z in zip(h, d, a):
            if x is None:
                continue
            assert np.array_equal(x, y) and np.array_equal(x, z), f"{m.name} cycle {i}: host / device / auto outputs differ"


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device"])
@pytest.mark.parametrize("seed,D,policy,big", BIG + [(4, 4, synth.POLICY_FAIR, 0)],
                         ids=["tile256", "tile512", "small"])
def test_filter_mid_session(monkeypatch, seed, D, policy, big, commit):
    """yk_filter_nodes between cycles equals the oracle's candidates on the model's state, and it changes nothing: the
    session stays bit-identical.  The big sessions' live node count crosses a 256- / 512-node tile boundary both ways."""
    monkeypatch.setenv("YK_UNIFORM_MIN", str(UNIFORM_MIN))
    m = session(seed, D, policy, big)
    replay(m, commit, 64, filter_k=9)
    if big:
        assert m.count.get("tile_crossed_up", 0) and m.count.get("tile_crossed_down", 0), m.count


# ---- GPU: targeted sessions ----
def _base(oracle, name, n_nodes=12, D=4, shape=None, apps=2, max_asks=2048):
    m = Model(oracle, name, D, max_nodes=64, max_asks=max_asks)
    m.queues_set(np.full((m.maxQ, D), -1), np.full((m.maxQ, D), -1), np.zeros(m.maxQ))
    if apps:
        m.apps_upsert(list(range(apps)), [LEAVES[i % 3] for i in range(apps)])
    shape = np.array([8000, 32 * GI, 20, 4000][:D]) if shape is None else np.asarray(shape)
    for n in range(n_nodes):
        m.set_node(n, shape, label=1, num=100 + 10 * n)
        m.used_nums.add(100 + 10 * n)
    m.nodes_upsert(list(range(n_nodes)), "nodes_upsert(initial)")
    return m


def _req(cpu, mem=GI):
    return np.array([cpu, mem, 1, 0], np.int64)


def _cycles(m):
    return [st[1] for st in m.steps if st[0] == "cycle"]


def t_release_then_cycle(oracle):
    """(a) release -> cycle with nothing in between: only yk_release marks the node tables for upload"""
    m = _base(oracle, "release-then-cycle", 6)
    m.asks_upsert(list(range(60)), _req(2000), 0)
    ask, _, _ = m.cycle()
    assert (m.a_last[:60] == NOFIT).sum() == 36
    m.release(ask[:20])
    ask, _, _ = m.cycle()
    assert len(ask) == 20
    m.release(ask[:5])
    m.cycle()
    finish(m)
    return m


def t_removed_below_hi(oracle):
    """(b) nodes below the highest index removed, then cycles: the device commit's export must cover every index up to
    n_hi, not just as many as there are live nodes"""
    m = _base(oracle, "removed-below-hi", 40)
    m.asks_upsert(list(range(100)), _req(500), 0)
    m.cycle(30)
    m.nodes_remove([1, 2, 3, 10, 20])                  # the highest index (39) stays: fewer live nodes than n_hi
    ask, node, _ = m.cycle()
    assert (node >= 35).sum() > 0
    m.asks_upsert(list(range(100, 110)), np.stack([_req(100 * (i + 1)) for i in range(10)]), 1)
    m.cycle()
    finish(m)
    return m


def t_rename_tied(oracle):
    """(c) renames of tied empty nodes decide where the next ask goes: the tie order is the NodeID order (both upsert paths)"""
    m = _base(oracle, "rename-tied", 8)
    m.asks_upsert([0], _req(100), 0)
    m.cycle()                                          # node 0 (NodeID first) takes it
    m.rename([7], [50])                                # contiguous path: node 7 becomes NodeID-first
    m.asks_upsert([1], _req(100), 0)
    m.cycle()
    m.rename([2, 4, 6], [20, 30, 40])                  # scattered path
    m.asks_upsert([2, 3], _req(100), 0)
    m.cycle()
    m.rename([5], [10])
    m.asks_upsert(list(range(4, 4 + UNIFORM_MIN)), _req(100), 1)
    m.cycle()
    m.rename(list(range(8)), [900 - 10 * n for n in range(8)])   # every node, order reversed
    m.asks_upsert(list(range(20, 26)), _req(100), 1)
    m.cycle()
    finish(m)
    firsts = [c.node[0] for c in _cycles(m) if len(c.node)]
    assert firsts[:4] == [0, 7, 2, 5], firsts
    return m


def t_nofit_then_fit(oracle):
    """(d) NOFIT in cycle k, room made, placed in cycle k + 1 (every cycle starts unallocated asks as pending again)"""
    shape = np.array([4000, 16 * GI, 20, 4000])
    m = _base(oracle, "nofit-then-fit", 3, shape=shape)
    m.asks_upsert(list(range(6)), _req(3000), 0)
    ask, _, _ = m.cycle()
    m.asks_upsert([6], _req(3000), 1)
    m.cycle()
    assert (m.a_last[:7] == NOFIT).sum() == 4
    m.release(ask[:1])
    m.cycle()
    assert m.count.get("nofit_then_fit") == 1
    m.set_node(1, shape + np.array([8000, 0, 0, 0]), num=m.n_num[1], label=1)   # a node grows: room for the other three
    m.nodes_upsert([1], "nodes_upsert(grow)")
    m.cycle()
    assert m.count.get("nofit_then_fit") == 4
    finish(m)
    return m


def t_epoch_rows(oracle):
    """(e) epoch rows on -> off -> on: a few signatures, then more than 1 024, then few again"""
    m = _base(oracle, "epoch-rows", 40, shape=np.array([64000, 256 * GI, 110, 64000]))
    m.asks_upsert(list(range(200)), np.stack([_req(100 * (1 + i % 3)) for i in range(200)]), 0)
    m.cycle(50)
    many = list(range(200, 1300))
    m.asks_upsert(many, np.stack([_req(10 + i) for i in range(len(many))]), 1)
    m.cycle(200)
    m.asks_remove([a for a in many if m.a_state[a] == PENDING])
    m.cycle(60)
    m.cycle()
    finish(m)
    return m


def t_uniform_uneven(oracle):
    """(f) uniform-run cycle -> release of half its asks -> another uniform-run cycle on the now uneven cluster"""
    m = _base(oracle, "uniform-uneven", 24)
    m.asks_upsert(list(range(120)), _req(500), 0)
    ask, _, _ = m.cycle()
    m.release(ask[::2])
    m.asks_upsert(list(range(120, 240)), _req(700), 1)
    m.cycle()
    m.asks_upsert(list(range(240, 300)), _req(300), 0)
    m.cycle()
    finish(m)
    return m


def t_gang_handoff(oracle):
    """(g) device commit with a gang hand-off, then a cycle the device commit cannot take (a gang of mixed requests: host
    commit), then a device cycle again"""
    m = _base(oracle, "gang-handoff", 3, shape=np.array([4000, 16 * GI, 20, 4000]))
    m.gang_seq += 1
    m.asks_upsert(list(range(4)), _req(3000), 0, gang=m.gang_seq)   # three members fit, the fourth does not: rolled back
    m.asks_upsert(list(range(4, 8)), _req(200), 1)
    m.cycle()
    assert (m.a_last[:4] == NOFIT).all() and (m.a_state[4:8] == ALLOCATED).all()
    m.asks_remove(list(range(4)))
    m.gang_seq += 1
    m.asks_upsert([8, 9], np.stack([_req(1500), _req(1000)]), 1, gang=m.gang_seq)
    m.cycle()
    assert not _cycles(m)[-1].eligible
    m.asks_upsert(list(range(10, 16)), np.stack([_req(100 * (i + 1)) for i in range(6)]), 0)
    m.cycle()
    finish(m)
    return m


def t_quota_from_history(oracle):
    """(h) a queue max that binds only because of earlier cycles' allocations, and a user limit that binds only because of
    what the user already holds"""
    m = _base(oracle, "quota-from-history", 10, apps=0)
    m.apps_upsert([0, 1, 2], [3, 4, 5], [0, 1, 1])
    m.asks_upsert(list(range(10)), _req(1000), 0)
    m.asks_upsert(list(range(10, 20)), _req(1000), 1)
    m.cycle()
    mx = np.full((m.maxQ, 4), -1)
    mx[3, 0] = 12000                                   # leaf 3 already holds 10 000: two more fit, not ten
    m.queues_set(np.full((m.maxQ, 4), -1), mx, np.zeros(m.maxQ))
    m.user_limits_set([(1, 1, np.array([13000, -1, -1, -1]))])   # user 1 holds 10 000 below parent 1: three more
    m.asks_upsert(list(range(20, 30)), _req(1000), 0)
    m.asks_upsert(list(range(30, 40)), _req(1000), 1)
    m.asks_upsert(list(range(40, 45)), _req(1000), 2)   # user 1 too, but in leaf 5: the entry does not apply
    m.cycle()
    st = _cycles(m)[-1].states
    assert (st[20:30] == 3).sum() == 8 and (st[30:40] == 3).sum() == 7 and (st[40:45] == 1).all(), st[20:45]
    m.release(list(range(0, 4)))
    m.cycle()
    finish(m)
    return m


@pytest.mark.parametrize("name", sorted(["a_release_then_cycle", "b_removed_below_hi", "c_rename_tied", "d_nofit_then_fit",
                                         "e_epoch_rows", "f_uniform_uneven", "g_gang_handoff", "h_quota_from_history"]))
def test_targeted_script(oracle, name):
    """each targeted script on the CPU: it has the shape it is meant to exercise (asserted inside), the model's accounting is
    conserved, and both oracles agree on every cycle"""
    m = TARGETED[name](oracle)
    m.check_conservation()
    _oracles_agree(m, every=1 if name != "e_epoch_rows" else 0)


TARGETED = {"a_release_then_cycle": t_release_then_cycle, "b_removed_below_hi": t_removed_below_hi,
            "c_rename_tied": t_rename_tied, "d_nofit_then_fit": t_nofit_then_fit, "e_epoch_rows": t_epoch_rows,
            "f_uniform_uneven": t_uniform_uneven, "g_gang_handoff": t_gang_handoff, "h_quota_from_history": t_quota_from_history}


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device"])
@pytest.mark.parametrize("name", sorted(TARGETED))
def test_targeted_session(oracle, monkeypatch, name, commit):
    monkeypatch.setenv("YK_UNIFORM_MIN", str(UNIFORM_MIN))
    m = TARGETED[name](oracle)
    per = []
    _, tot = replay(m, commit, 64, on_cycle=lambda e, c, d: per.append(d))
    cyc = _cycles(m)
    if commit == "device":
        assert [d["lattice_cycles"] for d in per] == [int(c.eligible) for c in cyc], name
    else:
        assert all(d["lattice_cycles"] == 0 for d in per) and tot["sweep_launches"] > 0, name
    if name == "e_epoch_rows" and commit == "host":
        # epoch rows: one row per signature per epoch sweep (3 signatures); without them a row per distinct ask of a batch
        assert 0 < per[0]["rows_swept"] <= 3 * per[0]["sweep_launches"], per[0]
        assert per[1]["rows_swept"] > 8 * per[1]["sweep_launches"], per[1]
        assert 0 < per[2]["rows_swept"] <= 3 * per[2]["sweep_launches"], per[2]
    if name == "g_gang_handoff":
        assert [d["lattice_handoffs"] for d in per[:3]] == ([1, 0, 0] if commit == "device" else [0, 0, 0]), per
    if name == "f_uniform_uneven" and commit == "device":
        assert per[0]["uniform_asks"] > 0 and per[1]["uniform_asks"] > 0, per
    if name == "g_gang_handoff" and commit == "device":
        assert per[0]["lattice_handoffs"] == 1, per[0]


@pytest.mark.gpu
def test_uniform_retry_on_uneven_cluster(oracle, monkeypatch):
    """(f) with YK_UNIFORM_DEPTH=1 a uniform run's first attempt is too shallow on a cluster earlier cycles left uneven:
    the retry path runs, the bindings stay the oracle's"""
    monkeypatch.setenv("YK_UNIFORM_MIN", str(UNIFORM_MIN))
    monkeypatch.setenv("YK_UNIFORM_DEPTH", "1")
    m = t_uniform_uneven(oracle)
    per = []
    _, tot = replay(m, "device", 4096, on_cycle=lambda e, c, d: per.append(d))
    assert per[1]["uniform_asks"] > 0 and per[1]["uniform_retries"] > 0, per[1]


@pytest.mark.gpu
def test_device_then_host_after_removal(oracle, monkeypatch):
    """(b) on ONE engine: a device-committed cycle after removals below n_hi, then host-committed cycles (a binpacking-free
    auto engine picks the device commit only for long uniform runs, so the long run goes first)"""
    monkeypatch.setenv("YK_UNIFORM_MIN", "16")
    m = _base(oracle, "removed-below-hi-auto", 40, shape=np.array([64000, 256 * GI, 110, 64000]), max_asks=5200)
    m.asks_upsert(list(range(20)), np.stack([_req(100 * (i + 1)) for i in range(20)]), 0)
    m.cycle()
    m.nodes_remove([0, 5, 6, 7, 30])
    m.asks_upsert(list(range(20, 5020)), _req(10, 1 << 20), 1)   # 5 000 identical asks: auto takes the device commit
    m.cycle()
    m.asks_upsert(list(range(5020, 5040)), np.stack([_req(100 * (i + 1)) for i in range(20)]), 0)
    m.cycle()
    finish(m)
    per = []
    replay(m, "auto", 4096, on_cycle=lambda e, c, d: per.append(d))
    assert [d["lattice_cycles"] for d in per[:3]] == [0, 1, 0], per


# ---- CPU: the model on its own ----
@pytest.mark.parametrize("seed,D,policy,big", ALL, ids=[f"seed{s}-D{d}-p{p}-big{b}" for s, d, p, b in ALL])
def test_model_sessions_oracles_agree(seed, D, policy, big):
    """every cycle's snapshot: the C++ oracle and the Python oracle agree; the model applied exactly the oracle's bindings"""
    _oracles_agree(session(seed, D, policy, big), every=4 if big else 1)


def _oracles_agree(m, every=1):
    """every cycle: the model's availability is the oracle's; on every `every`-th cycle (0: none) the Python oracle agrees"""
    for c in _cycles(m):
        where = f"{m.name} cycle {c.number}"
        assert np.array_equal(c.avail, c.oracle_avail), where
        if not every or c.number % every:
            continue
        p = py_oracle.run(c.snap, -1 if c.max_bindings is None else c.max_bindings)
        assert c.amap[p["ask"]].tolist() == c.ask.tolist(), where
        assert c.nmap[p["node"]].tolist() == c.node.tolist(), where
        if c.states is not None:
            assert np.array_equal(np.asarray(p["state"]), c.states[c.amap]), where


def test_sessions_cover_every_operation():
    """the generator still produces every operation and interleaving, a stated number of times over the session set"""
    total = {}
    for args in ALL:
        for k, v in session(*args).count.items():
            total[k] = total.get(k, 0) + v
    need = {"upsert_contiguous": 40, "upsert_scattered": 20, "nodes_new_fresh_index": 10, "nodes_new_reused_index": 5,
            "nodes_new_tied_group": 5, "node_resize": 10, "node_foreign_occupancy": 10, "node_cordon": 5, "node_uncordon": 2,
            "node_reserved": 5, "node_taint": 5, "node_label": 5, "rename_tied": 20, "rename_with_allocations": 5,
            "remove_with_allocations": 5, "remove_below_hi": 10, "asks_new": 50, "asks_uniform_run": 20, "asks_gang": 20,
            "asks_reupsert": 10, "asks_reused_index": 10, "asks_remove": 10, "release": 40, "release_gang_member": 10,
            "release_on_removed_node": 3, "apps_upsert": 5, "apps_remove": 5, "app_removed_with_pending": 1,
            "queues_set": 5, "queues_priority": 3, "user_limits_set": 10, "mb_unlimited": 50, "mb_one": 10,
            "mb_zero": 5, "mb_random": 10, "mb_gang_cut": 5, "mb_final": len(ALL), "release_then_cycle": 10,
            "cycle_after_removal_below_hi": 10, "nofit_then_fit": 3, "tile_crossed_up": 2, "tile_crossed_down": 2}
    short = {k: (total.get(k, 0), n) for k, n in need.items() if total.get(k, 0) < n}
    assert not short, short
    # the uniform path has long runs to take, and NOFIT / SKIPPED states occur
    runs = sum(1 for a in ALL for st in session(*a).steps if st[0] == "cycle" and st[1].longest_run >= UNIFORM_MIN)
    states = np.concatenate([st[1].states for a in ALL for st in session(*a).steps if st[0] == "cycle" and st[1].states is not None])
    assert runs >= 30 and (states == 2).sum() > 50 and (states == 3).sum() > 10, (runs, np.bincount(states[states < 8]))
