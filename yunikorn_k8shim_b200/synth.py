"""Seeded synthetic cluster snapshots for the BASELINE.json configs (SURVEY.md section 8d).

A Snapshot is plain numpy: it is the *input* both the engine (through the C ABI) and the
test oracle consume.  Nothing here computes a scheduling decision.

Shapes follow the reference's own perf inputs:
  * kwok nodes 32 CPU / 256 Gi / 110 pods, taint kwok.x-k8s.io/node=fake:NoSchedule, label type=kwok
    (deployments/kwok-perf-test/kwok-setup.sh:30-62)
  * sleep deployments, one application per deployment, toleration Exists
    (deployments/kwok-perf-test/deploy-tool.sh:34-67)
  * 400 apps x 125 tasks, 10 mCPU / 1 MB asks
    (pkg/shim/scheduler_perf_test.go:151-171,283-328)
Resource vectors are the shim's: cpu in milli-units, everything else integer Value(), "pods": 1 per ask
(pkg/common/resource.go:56-59,273-285).
"""
from __future__ import annotations

from dataclasses import dataclass, field
import numpy as np

RESOURCES = ("vcore", "memory", "pods", "ephemeral-storage")
GI = 1 << 30
MI = 1 << 20

NODE_SCHEDULABLE = 1
NODE_RESERVED = 2
ASK_SLOWPATH = 1
POLICY_FAIR = 0
POLICY_BINPACKING = 1
SORT_FIFO = 0
SORT_FAIR = 1

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def splitmix64(seed: int, n: int) -> np.ndarray:
    """n 64-bit values of the splitmix64 stream started at `seed` (vectorised, wraps mod 2^64)."""
    with np.errstate(over="ignore"):
        i = np.arange(1, n + 1, dtype=np.uint64)
        z = (np.uint64(seed & 0xFFFFFFFFFFFFFFFF) + i * np.uint64(0x9E3779B97F4A7C15)) & _M64
        z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & _M64
        z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & _M64
        return z ^ (z >> np.uint64(31))


class _Rng:
    def __init__(self, seed: int):
        self.seed = seed
        self.ctr = 0

    def u64(self, n: int) -> np.ndarray:
        out = splitmix64(self.seed * 0x1000003 + self.ctr, n)
        self.ctr += 0x10000019
        return out

    def below(self, n: int, hi: int) -> np.ndarray:
        return (self.u64(n) % np.uint64(hi)).astype(np.int64)

    def uniform(self, n: int) -> np.ndarray:
        return (self.u64(n) >> np.uint64(11)).astype(np.float64) / float(1 << 53)


@dataclass
class Snapshot:
    D: int
    policy: int
    weights: np.ndarray          # [D] f64
    node_total: np.ndarray       # [N][D] i64
    node_avail: np.ndarray       # [N][D] i64
    node_taint: np.ndarray       # [N] u64
    node_label: np.ndarray       # [N] u64
    node_flags: np.ndarray       # [N] u32
    node_id: list                # [N] str
    q_parent: np.ndarray         # [Q] i32
    q_guaranteed: np.ndarray     # [Q][D] i64 (-1 unset)
    q_max: np.ndarray            # [Q][D] i64 (-1 unset)
    q_alloc: np.ndarray          # [Q][D] i64
    q_sort: np.ndarray           # [Q] u8
    app_queue: np.ndarray        # [P] i32
    app_submit: np.ndarray       # [P] i64
    ask_app: np.ndarray          # [A] i32
    ask_req: np.ndarray          # [A][D] i64
    ask_tol: np.ndarray          # [A] u64
    ask_need: np.ndarray         # [A] u64
    ask_deny: np.ndarray         # [A] u64
    ask_prio: np.ndarray         # [A] i32
    ask_create: np.ndarray       # [A] i64
    ask_node: np.ndarray         # [A] i32
    ask_flags: np.ndarray        # [A] u32
    ask_gang: np.ndarray         # [A] i32
    name: str = ""
    meta: dict = field(default_factory=dict)
    q_prio_offset: np.ndarray = None   # [Q] i32 queue property priority.offset (None = all 0)
    q_prio_fence: np.ndarray = None    # [Q] u8  queue property priority.policy == fence (None = none)
    # user / group resource limits (the core's queue `limits:`): entry l = user ul_user[l] may hold at most ul_max[l] below
    # queue ul_queue[l]; app_user = the application's user (pkg/cache/application.go:430 sends it), -1 = none
    app_user: np.ndarray = None        # [P] i32
    ul_queue: np.ndarray = None        # [L] i32
    ul_user: np.ndarray = None         # [L] i32
    ul_max: np.ndarray = None          # [L][D] i64 (-1 unset)
    ul_alloc: np.ndarray = None        # [L][D] i64 held at cycle start (None = 0)

    @property
    def n_nodes(self): return len(self.node_id)
    @property
    def n_asks(self): return len(self.ask_app)
    @property
    def n_apps(self): return len(self.app_queue)
    @property
    def n_queues(self): return len(self.q_parent)

    def node_rank(self) -> np.ndarray:
        """rank of each NodeID in Go string order (bytewise) -- what the Go side would pass as name_rank."""
        enc = [s.encode() for s in self.node_id]
        order = sorted(range(len(enc)), key=lambda i: enc[i])
        rank = np.empty(len(enc), dtype=np.uint32)
        rank[np.asarray(order, dtype=np.int64)] = np.arange(len(enc), dtype=np.uint32)
        return rank


def _single_queue(D: int):
    # root -> root.default ; no quotas (deployments/scheduler/yunikorn-configs.yaml:23-32)
    qp = np.array([-1, 0], dtype=np.int32)
    unset = np.full((2, D), -1, dtype=np.int64)
    return qp, unset.copy(), unset.copy(), np.zeros((2, D), dtype=np.int64), np.zeros(2, dtype=np.uint8)


def _finish(name, D, policy, node_total, node_avail, node_taint, node_label, node_id, queues, app_queue,
            ask_app, ask_req, ask_tol, ask_need, ask_deny, ask_prio=None, ask_node=None, ask_flags=None,
            ask_gang=None, node_flags=None, app_submit=None, ask_create=None, meta=None) -> Snapshot:
    N, A, P = len(node_id), len(ask_app), len(app_queue)
    w = np.zeros(D, dtype=np.float64)
    w[0] = 1.0
    w[1] = 1.0   # default node-sort weights vcore=1, memory=1 (SURVEY A.3)
    qp, qg, qm, qa, qs = queues
    return Snapshot(
        D=D, policy=policy, weights=w,
        node_total=np.ascontiguousarray(node_total, dtype=np.int64),
        node_avail=np.ascontiguousarray(node_avail, dtype=np.int64),
        node_taint=np.ascontiguousarray(node_taint, dtype=np.uint64),
        node_label=np.ascontiguousarray(node_label, dtype=np.uint64),
        node_flags=(np.full(N, NODE_SCHEDULABLE, dtype=np.uint32) if node_flags is None
                    else np.ascontiguousarray(node_flags, dtype=np.uint32)),
        node_id=list(node_id),
        q_parent=qp, q_guaranteed=qg, q_max=qm, q_alloc=qa, q_sort=qs,
        app_queue=np.ascontiguousarray(app_queue, dtype=np.int32),
        app_submit=(np.arange(P, dtype=np.int64) + 1_700_000_000 if app_submit is None
                    else np.ascontiguousarray(app_submit, dtype=np.int64)),
        ask_app=np.ascontiguousarray(ask_app, dtype=np.int32),
        ask_req=np.ascontiguousarray(ask_req, dtype=np.int64),
        ask_tol=np.ascontiguousarray(ask_tol, dtype=np.uint64),
        ask_need=np.ascontiguousarray(ask_need, dtype=np.uint64),
        ask_deny=np.ascontiguousarray(ask_deny, dtype=np.uint64),
        ask_prio=(np.zeros(A, dtype=np.int32) if ask_prio is None else np.ascontiguousarray(ask_prio, dtype=np.int32)),
        ask_create=(np.arange(A, dtype=np.int64) if ask_create is None
                    else np.ascontiguousarray(ask_create, dtype=np.int64)),
        ask_node=(np.full(A, -1, dtype=np.int32) if ask_node is None else np.ascontiguousarray(ask_node, dtype=np.int32)),
        ask_flags=(np.zeros(A, dtype=np.uint32) if ask_flags is None else np.ascontiguousarray(ask_flags, dtype=np.uint32)),
        ask_gang=(np.full(A, -1, dtype=np.int32) if ask_gang is None else np.ascontiguousarray(ask_gang, dtype=np.int32)),
        name=name, meta=meta or {})


def kwok(n_nodes=100, n_apps=10, replicas=50, variant="sized", policy=POLICY_FAIR, seed=1) -> Snapshot:
    """BASELINE config 1: kwok-perf-test shape. variant "bare" = {pods:1} asks exactly as the script
    (container without resources), "sized" = {100 mCPU, 128 Mi, 1 pod} so the fit test is not trivial."""
    D = 4
    tot = np.tile(np.array([32_000, 256 * GI, 110, 0], dtype=np.int64), (n_nodes, 1))
    ids = [f"kwok-node-{i}" for i in range(n_nodes)]
    taint = np.full(n_nodes, 1, dtype=np.uint64)          # bit0: kwok.x-k8s.io/node=fake:NoSchedule
    label = np.full(n_nodes, 1, dtype=np.uint64)          # bit0: type=kwok
    A = n_apps * replicas
    app = np.repeat(np.arange(n_apps, dtype=np.int32), replicas)
    req = np.zeros((A, D), dtype=np.int64)
    req[:, 2] = 1
    if variant == "sized":
        req[:, 0] = 100
        req[:, 1] = 128 * MI
    tol = np.full(A, 1, dtype=np.uint64)
    z = np.zeros(A, dtype=np.uint64)
    return _finish(f"kwok-{n_nodes}x{A}-{variant}", D, policy, tot, tot.copy(), taint, label, ids,
                   _single_queue(D), np.ones(n_apps, dtype=np.int32), app, req, tol, z, z.copy(),
                   meta={"config": 1, "seed": seed})


_CLASSES = np.array([[10, 1_000_000], [100, 128 * MI], [500, 1 * GI], [2000, 8 * GI]], dtype=np.int64)
_CLASS_CUM = np.array([40, 70, 90, 100], dtype=np.int64)


def perf(n_nodes=10_000, n_apps=400, tasks=125, masks=False, policy=POLICY_FAIR, seed=2) -> Snapshot:
    """BASELINE config 2 (masks=False) / 3 (masks=True): jittered kwok-sized nodes, 10% pre-loaded,
    asks drawn from four request classes (40/30/20/10 %), single leaf queue, distinct create keys."""
    D = 4
    r = _Rng(seed)
    cpu = (32 + r.below(n_nodes, 17) - 8) * 1000                 # 24..40 CPU in 1-CPU steps
    mem = (256 + r.below(n_nodes, 129) - 64) * GI                # 192..320 Gi in 1-Gi steps
    tot = np.stack([cpu, mem, np.full(n_nodes, 110, dtype=np.int64), np.zeros(n_nodes, dtype=np.int64)], axis=1)
    avail = tot.copy()
    loaded = r.uniform(n_nodes) < 0.10
    frac = r.uniform(n_nodes) * 0.8
    used_cpu = (tot[:, 0] * frac).astype(np.int64) // 10 * 10
    used_mem = (tot[:, 1] * frac).astype(np.int64) // MI * MI
    used_pods = (frac * 60).astype(np.int64)
    avail[:, 0] -= np.where(loaded, used_cpu, 0)
    avail[:, 1] -= np.where(loaded, used_mem, 0)
    avail[:, 2] -= np.where(loaded, used_pods, 0)
    ids = [f"kwok-node-{i}" for i in range(n_nodes)]
    A = n_apps * tasks
    app = np.repeat(np.arange(n_apps, dtype=np.int32), tasks)
    cls = np.searchsorted(_CLASS_CUM, r.below(A, 100), side="right")
    req = np.zeros((A, D), dtype=np.int64)
    req[:, 0] = _CLASSES[cls, 0]
    req[:, 1] = _CLASSES[cls, 1]
    req[:, 2] = 1
    taint = np.zeros(n_nodes, dtype=np.uint64)
    label = np.zeros(n_nodes, dtype=np.uint64)
    tol = np.zeros(A, dtype=np.uint64)
    need = np.zeros(A, dtype=np.uint64)
    deny = np.zeros(A, dtype=np.uint64)
    if masks:
        # 16 taint bits, each on a node with p=0.05; asks tolerate each with p=0.5
        tb = r.uniform(n_nodes * 16).reshape(n_nodes, 16) < 0.05
        taint = (tb.astype(np.uint64) << np.arange(16, dtype=np.uint64)).sum(axis=1).astype(np.uint64)
        ab = r.uniform(A * 16).reshape(A, 16) < 0.5
        tol = (ab.astype(np.uint64) << np.arange(16, dtype=np.uint64)).sum(axis=1).astype(np.uint64)
        # 48 label bits: zone x8 [0,8), instance-type x16 [8,24), arch x2 [24,26), pool x22 [26,48)
        zone = r.below(n_nodes, 8)
        itype = r.below(n_nodes, 16)
        arch = r.below(n_nodes, 2)
        pool = r.below(n_nodes, 22)
        one = np.uint64(1)
        label = ((one << zone.astype(np.uint64)) | (one << (8 + itype).astype(np.uint64))
                 | (one << (24 + arch).astype(np.uint64)) | (one << (26 + pool).astype(np.uint64)))
        nsel = r.below(A, 3)                                      # nodeSelector on 0..2 label bits
        szone = r.below(A, 8)
        sarch = r.below(A, 2)
        need = np.where(nsel >= 1, one << szone.astype(np.uint64), np.uint64(0))
        need = need | np.where(nsel >= 2, one << (24 + sarch).astype(np.uint64), np.uint64(0))
        dn = r.uniform(A) < 0.10                                  # 10% carry a NotIn / DoesNotExist bit
        dpool = r.below(A, 22)
        deny = np.where(dn, one << (26 + dpool).astype(np.uint64), np.uint64(0))
        # every ask must have >=1 feasible node: asks keep at least the untainted nodes of their
        # zone/arch that are not in the denied pool; with 10k nodes that set is never empty, and the
        # generator verifies it for small N by falling back to "tolerate everything"
        if n_nodes < 2000:
            ok = np.array([bool(np.any(((taint & ~tol[a]) == 0) & ((label & need[a]) == need[a])
                                       & ((label & deny[a]) == 0))) for a in range(A)])
            tol = np.where(ok, tol, np.uint64(0xFFFF))
            need = np.where(ok, need, np.uint64(0))
            deny = np.where(ok, deny, np.uint64(0))
    return _finish(f"perf-{n_nodes}x{A}-{'masks' if masks else 'plain'}", D, policy, tot, avail, taint, label, ids,
                   _single_queue(D), np.ones(n_apps, dtype=np.int32), app, req, tol, need, deny,
                   meta={"config": 3 if masks else 2, "seed": seed})


def reference_shape(n_nodes=5_000, n_apps=400, tasks=125, policy=POLICY_FAIR) -> Snapshot:
    """The reference's own in-process benchmark (BenchmarkSchedulingThroughPut): identical kwok-sized nodes, 400 applications
    x 125 tasks = 50 000 pods, every pod requesting 10 mCPU / 1 MB
    (pkg/shim/scheduler_perf_test.go:62-63 nodes and pods, :151-171 apps x tasks, :283-288 the request)."""
    D = 4
    tot = np.tile(np.array([32_000, 256 * GI, 110, 0], dtype=np.int64), (n_nodes, 1))
    ids = [f"kwok-node-{i}" for i in range(n_nodes)]
    z_n = np.zeros(n_nodes, dtype=np.uint64)
    A = n_apps * tasks
    app = np.repeat(np.arange(n_apps, dtype=np.int32), tasks)
    req = np.zeros((A, D), dtype=np.int64)
    req[:, 0], req[:, 1], req[:, 2] = 10, 1_000_000, 1
    z = np.zeros(A, dtype=np.uint64)
    return _finish(f"reference-shape-{n_nodes}x{A}", D, policy, tot, tot.copy(), z_n, z_n.copy(), ids,
                   _single_queue(D), np.ones(n_apps, dtype=np.int32), app, req, z, z.copy(), z.copy(),
                   meta={"config": "reference", "seed": 0})


def hier(n_nodes=50_000, n_parents=8, leaves_per_parent=8, apps_per_leaf=5, tasks=625, masks=False,
         policy=POLICY_FAIR, seed=4, quota_frac=1.2, priorities=False, big_nodes=False, leaf_sort=SORT_FIFO) -> Snapshot:
    """BASELINE config 4: 3-level queue tree (root -> parents -> leaves), guaranteed + max per leaf, fifo apps
    in the leaves, fair (DRF) parents; demand is `quota_frac` x some leaf maxima so the headroom checks bite.
    Default sizes: 50k nodes, 64 leaves x 5 apps x 625 tasks = 200k asks."""
    base = perf(n_nodes, n_parents * leaves_per_parent * apps_per_leaf, tasks, masks=masks, policy=policy, seed=seed)
    D = base.D
    r = _Rng(seed * 7919 + 13)
    L = n_parents * leaves_per_parent
    Q = 1 + n_parents + L
    qp = np.empty(Q, dtype=np.int32)
    qp[0] = -1
    qp[1:1 + n_parents] = 0
    qp[1 + n_parents:] = 1 + np.repeat(np.arange(n_parents, dtype=np.int32), leaves_per_parent)
    guar = np.full((Q, D), -1, dtype=np.int64)
    mx = np.full((Q, D), -1, dtype=np.int64)
    app_leaf = np.repeat(np.arange(L, dtype=np.int32), apps_per_leaf)
    app_queue = 1 + n_parents + app_leaf
    ask_leaf = app_leaf[base.ask_app]
    demand = np.zeros((L, D), dtype=np.int64)
    np.add.at(demand, ask_leaf, base.ask_req)
    # guaranteed: a random 20..60 % of the leaf's demand on cpu/memory; max on every third leaf at demand/quota_frac
    gfrac = 0.2 + 0.4 * r.uniform(L)
    for li in range(L):
        q = 1 + n_parents + li
        guar[q, 0] = max(1000, int(demand[li, 0] * gfrac[li]) // 1000 * 1000)
        guar[q, 1] = max(GI, int(demand[li, 1] * gfrac[li]) // GI * GI)
        if li % 3 == 0:
            mx[q, 0] = max(1000, int(demand[li, 0] / quota_frac) // 1000 * 1000)
            mx[q, 1] = max(GI, int(demand[li, 1] / quota_frac) // GI * GI)
    for pi in range(n_parents):
        q = 1 + pi
        kids = np.nonzero(qp == q)[0]
        guar[q, 0] = guar[kids, 0].sum()
        guar[q, 1] = guar[kids, 1].sum()
    prio = None
    if priorities:
        prio = (r.below(base.n_asks, 3) - 1).astype(np.int32) * 100
    if big_nodes:   # every node can hold everything: isolates the ordering logic
        base.node_total[:, 0] = 1 << 40
        base.node_total[:, 1] = 1 << 50
        base.node_total[:, 2] = 1 << 30
        base.node_avail[:] = base.node_total
    queues = (qp, guar, mx, np.zeros((Q, D), dtype=np.int64), np.full(Q, leaf_sort, dtype=np.uint8))
    s = _finish(f"hier-{n_nodes}x{base.n_asks}-q{Q}", D, policy, base.node_total, base.node_avail, base.node_taint,
                base.node_label, base.node_id, queues, app_queue, base.ask_app, base.ask_req, base.ask_tol,
                base.ask_need, base.ask_deny, ask_prio=prio, meta={"config": 4, "seed": seed})
    return s


def gangs(n_nodes=10_000, n_gangs=2000, members=10, seed=5, policy=POLICY_FAIR, fill=1.11) -> Snapshot:
    """BASELINE config 5: n_gangs gangs of `members` identical members (task-group semantics,
    pkg/cache/amprotocol.go:47-57), one application per gang, one leaf queue; total demand is
    `fill` x the cluster's CPU so that roughly the last tenth of the gangs cannot be placed whole."""
    D = 4
    base = perf(n_nodes, 1, 1, seed=seed, policy=policy)
    r = _Rng(seed * 31 + 7)
    cls = r.below(n_gangs, 4)
    cpu_cls = np.array([2000, 4000, 8000, 12000], dtype=np.int64)
    mem_cls = np.array([8, 16, 32, 64], dtype=np.int64) * GI
    cap = int(base.node_avail[:, 0].sum())
    demand = int((cpu_cls[cls] * members).sum())
    scale = fill * cap / demand
    cpu = np.maximum(100, (cpu_cls[cls] * scale).astype(np.int64) // 100 * 100)
    A = n_gangs * members
    app = np.repeat(np.arange(n_gangs, dtype=np.int32), members)
    req = np.zeros((A, D), dtype=np.int64)
    req[:, 0] = np.repeat(cpu, members)
    req[:, 1] = np.repeat(mem_cls[cls], members)
    req[:, 2] = 1
    z = np.zeros(A, dtype=np.uint64)
    return _finish(f"gangs-{n_nodes}x{n_gangs}x{members}", D, policy, base.node_total, base.node_avail, base.node_taint,
                   base.node_label, base.node_id, _single_queue(D), np.ones(n_gangs, dtype=np.int32), app, req, z,
                   z.copy(), z.copy(), ask_gang=app.copy(), meta={"config": 5, "seed": seed})


def poisoned_gangs(seed: int, n_nodes=64, n_gangs=80, members=4, policy=POLICY_FAIR) -> Snapshot:
    """Roll-back stress: an under-committed gangs() cluster where ~30% of the gangs have a LAST member no node can
    hold (so the gang is placed, then undone) and half of the healthy gangs are dissolved into plain asks, so single
    asks keep landing on nodes that roll-backs have just handed back."""
    s = gangs(n_nodes, n_gangs, members, seed=seed, fill=0.7, policy=policy)
    rng = np.random.default_rng(seed)
    bad = rng.random(n_gangs) < 0.3
    last = np.arange(n_gangs) * members + members - 1
    s.ask_req[last[bad], 2] = 1 << 31
    plain = (~bad) & (rng.random(n_gangs) < 0.5)
    for g in np.nonzero(plain)[0]:
        s.ask_gang[g * members:(g + 1) * members] = -1
    s.name = f"poisoned-gangs-{seed}"
    return s


def runny(s: Snapshot, seed: int) -> Snapshot:
    """Make the snapshot's asks come in runs (in place): blocks of consecutive asks of one application copy everything the
    commit looks at (request, masks, node name, priority, flags) from the block's first ask -- the replicas of one
    deployment / the executors of one job."""
    r = np.random.default_rng(seed)
    i = 0
    while i < s.n_asks:
        ln = int(r.integers(1, 14))
        j = i + 1
        while j < s.n_asks and j - i < ln and s.ask_app[j] == s.ask_app[i]:
            for col in (s.ask_req, s.ask_tol, s.ask_need, s.ask_deny, s.ask_node, s.ask_prio, s.ask_flags):
                col[j] = col[i]
            j += 1
        i = j
    return s


def fuzz(seed: int, n_nodes=None, n_asks=None) -> Snapshot:
    """Small snapshot mixing every feature of the path at once (used by the randomized parity tests): random queue
    tree with guarantees and quotas, fifo and fair leaves, priorities, gangs, taints / selectors, pod.Spec.NodeName,
    slow-path asks, zero requests, unschedulable / reserved / over-committed nodes, either node-sort policy."""
    r = _Rng(seed * 2654435761 + 17)
    D = 4
    N = int(n_nodes or (3 + r.below(1, 40)[0]))
    n_par = int(1 + r.below(1, 3)[0])
    n_leaf_per = int(1 + r.below(1, 3)[0])
    L = n_par * n_leaf_per
    Q = 1 + n_par + L
    qp = np.empty(Q, dtype=np.int32)
    qp[0] = -1
    qp[1:1 + n_par] = 0
    qp[1 + n_par:] = 1 + np.repeat(np.arange(n_par, dtype=np.int32), n_leaf_per)
    apps_per_leaf = int(1 + r.below(1, 3)[0])
    P = L * apps_per_leaf
    app_queue = 1 + n_par + np.repeat(np.arange(L, dtype=np.int32), apps_per_leaf)
    A = int(n_asks or (5 + r.below(1, 150)[0]))
    ask_app = np.sort(r.below(A, P)).astype(np.int32)
    cpu = (16 + r.below(N, 25)) * 1000
    mem = (64 + r.below(N, 129)) * GI
    tot = np.stack([cpu, mem, 8 + r.below(N, 30), np.zeros(N, dtype=np.int64)], axis=1)
    avail = tot.copy()
    frac = r.uniform(N) * 0.9 * (r.uniform(N) < 0.4)
    avail[:, 0] -= (tot[:, 0] * frac).astype(np.int64) // 10 * 10
    avail[:, 1] -= (tot[:, 1] * frac).astype(np.int64) // MI * MI
    avail[:, 2] -= (tot[:, 2] * frac * 0.5).astype(np.int64)
    over = r.uniform(N) < 0.05
    avail[over, 0] = -3000                                  # over-committed: FitIn clamps at 0
    flags = np.full(N, NODE_SCHEDULABLE, dtype=np.uint32)
    flags[r.uniform(N) < 0.07] = 0
    flags[r.uniform(N) < 0.05] |= NODE_RESERVED
    ids = [f"n{int(x)}" for x in (r.below(N, 1000) * 1000 + np.arange(N))]   # unique, not in index order
    taint = np.where(r.uniform(N) < 0.3, np.uint64(1) << r.below(N, 4).astype(np.uint64), np.uint64(0)).astype(np.uint64)
    label = (np.uint64(1) << r.below(N, 3).astype(np.uint64)) | (np.uint64(1) << (3 + r.below(N, 2)).astype(np.uint64))
    cls = r.below(A, 5)
    cpus = np.array([10, 250, 1000, 4000, 0], dtype=np.int64)
    mems = np.array([1_000_000, 256 * MI, 2 * GI, 16 * GI, 0], dtype=np.int64)
    req = np.zeros((A, D), dtype=np.int64)
    req[:, 0] = cpus[cls]
    req[:, 1] = mems[cls]
    req[:, 2] = (cls != 4).astype(np.int64)                  # class 4 = nothing requested at all: invalid
    tol = np.where(r.uniform(A) < 0.6, np.uint64(0xF), (np.uint64(1) << r.below(A, 4).astype(np.uint64))).astype(np.uint64)
    need = np.where(r.uniform(A) < 0.3, np.uint64(1) << r.below(A, 3).astype(np.uint64), np.uint64(0)).astype(np.uint64)
    deny = np.where(r.uniform(A) < 0.15, np.uint64(1) << (3 + r.below(A, 2)).astype(np.uint64), np.uint64(0)).astype(np.uint64)
    prio = (r.below(A, 3) - 1).astype(np.int32) * 10 * (r.uniform(1)[0] < 0.5)
    ask_node = np.where(r.uniform(A) < 0.04, r.below(A, N), -1).astype(np.int32)
    aflags = (r.uniform(A) < 0.04).astype(np.uint32)
    gang = np.full(A, -1, dtype=np.int32)
    if r.uniform(1)[0] < 0.6:                               # gangs: runs of 2..4 consecutive asks of one application
        i = 0
        g = 0
        while i < A:
            ln = int(2 + r.below(1, 3)[0])
            j = i
            while j < A and j - i < ln and ask_app[j] == ask_app[i]:
                j += 1
            if j - i >= 2 and r.uniform(1)[0] < 0.35:
                gang[i:j] = g
                g += 1
            i = max(j, i + 1)
    guar = np.full((Q, D), -1, dtype=np.int64)
    mx = np.full((Q, D), -1, dtype=np.int64)
    for q in range(1, Q):
        if r.uniform(1)[0] < 0.7:
            guar[q, 0] = int(1000 * (1 + r.below(1, 40)[0]))
            guar[q, 1] = int(GI * (1 + r.below(1, 200)[0]))
        if r.uniform(1)[0] < 0.35:
            mx[q, 0] = int(1000 * (1 + r.below(1, 60)[0]))
        if r.uniform(1)[0] < 0.2:
            mx[q, 2] = int(1 + r.below(1, 40)[0])
    qsort = np.zeros(Q, dtype=np.uint8)
    qsort[1 + n_par:] = (r.uniform(L) < 0.3).astype(np.uint8)
    policy = int(r.below(1, 2)[0])
    return _finish(f"fuzz-{seed}", D, policy, tot, avail, taint, label, ids,
                   (qp, guar, mx, np.zeros((Q, D), dtype=np.int64), qsort), app_queue, ask_app, req, tol, need, deny,
                   ask_prio=prio, ask_node=ask_node, ask_flags=aflags, ask_gang=gang, node_flags=flags,
                   meta={"seed": seed})


def priority_fence(quota_pods: int = 1, done=()) -> Snapshot:
    """The scenario of test/e2e/priority_scheduling/priority_scheduling_test.go:70-133
    (Verify_Static_Queue_App_Scheduling_Order): root -> fence (max = `quota_pods` pods) -> child1, child2; applications
    low (child1, priority -100), normal (child2, 0), high (child1, +100) submitted in that order, one pod each.  The
    reference serves them high, normal, low.  `done` lists applications ("high", ...) already finished."""
    D = 4
    base = perf(4, 1, 1)
    qp = np.array([-1, 0, 1, 1], dtype=np.int32)
    unset = np.full((4, D), -1, dtype=np.int64)
    qmax = unset.copy()
    req = np.array([100, 100 * 1000 * 1000, 1, 0], dtype=np.int64)            # rr: one pod's request
    qmax[1, :3] = req[:3] * quota_pods
    queues = (qp, unset.copy(), qmax, np.zeros((4, D), dtype=np.int64), np.zeros(4, dtype=np.uint8))
    apps = [("low", 2, -100), ("normal", 3, 0), ("high", 2, 100)]
    apps = [a for a in apps if a[0] not in done]
    z = np.zeros(len(apps), dtype=np.uint64)
    s = _finish("priority-fence", D, POLICY_FAIR, base.node_total, base.node_avail, base.node_taint, base.node_label, base.node_id,
                queues, np.array([a[1] for a in apps], dtype=np.int32), np.arange(len(apps), dtype=np.int32),
                np.tile(req, (len(apps), 1)), z, z.copy(), z.copy(), ask_prio=np.array([a[2] for a in apps], dtype=np.int32))
    s.meta["apps"] = [a[0] for a in apps]
    return s


def binpacking_e2e() -> Snapshot:
    """The scenario of test/e2e/bin_packing/bin_packing_test.go:46-200: binpacking node sort; nodeA is the
    most utilised node, nodeB the second; job A (3 pods) must land on nodeA, job B (3 pods that may not run on nodeA --
    pod anti-affinity in the reference, a forbidden label bit here) on nodeB."""
    D = 4
    total = np.tile(np.array([16000, 64 * GI, 110, 0], dtype=np.int64), (4, 1))
    avail = total.copy()
    avail[0, 1] -= 40 * GI            # nodeA: least available memory
    avail[1, 1] -= 30 * GI            # nodeB
    avail[2, 1] -= 10 * GI
    label = np.array([1, 2, 4, 8], dtype=np.uint64)                         # one identity bit per node
    req = np.tile(np.array([100, 1 * GI, 1, 0], dtype=np.int64), (6, 1))
    z = np.zeros(6, dtype=np.uint64)
    deny = z.copy()
    deny[3:] = 1                                                            # job B: not on nodeA
    return _finish("binpacking-e2e", D, POLICY_BINPACKING, total, avail, np.zeros(4, dtype=np.uint64), label,
                   ["nodeA", "nodeB", "nodeC", "nodeD"], _single_queue(D), np.array([1, 1], dtype=np.int32),
                   np.array([0, 0, 0, 1, 1, 1], dtype=np.int32), req, z, z.copy(), deny)


def priority_offsets(quota_pods: int = 1, done=()) -> Snapshot:
    """The scenario of priority_scheduling_test.go:179-251 (Verify_Priority_Offset_Queue_App_Scheduling_Order):
    root -> priority (fence, max = `quota_pods` pods) -> high (priority.offset +100), normal (0), low (-100); one pod
    without a priority class in each, submitted low, normal, high.  The reference serves them high, normal, low."""
    D = 4
    base = perf(4, 1, 1)
    qp = np.array([-1, 0, 1, 1, 1], dtype=np.int32)                          # root, priority, high, normal, low
    unset = np.full((5, D), -1, dtype=np.int64)
    qmax = unset.copy()
    req = np.array([100, 100 * 1000 * 1000, 1, 0], dtype=np.int64)
    qmax[1, :3] = req[:3] * quota_pods
    queues = (qp, unset.copy(), qmax, np.zeros((5, D), dtype=np.int64), np.zeros(5, dtype=np.uint8))
    apps = [("low", 4), ("normal", 3), ("high", 2)]
    apps = [a for a in apps if a[0] not in done]
    z = np.zeros(len(apps), dtype=np.uint64)
    s = _finish("priority-offsets", D, POLICY_FAIR, base.node_total, base.node_avail, base.node_taint, base.node_label, base.node_id,
                queues, np.array([a[1] for a in apps], dtype=np.int32), np.arange(len(apps), dtype=np.int32),
                np.tile(req, (len(apps), 1)), z, z.copy(), z.copy())
    s.q_prio_offset = np.array([0, 0, 100, 0, -100], dtype=np.int32)
    s.q_prio_fence = np.array([0, 1, 0, 0, 0], dtype=np.uint8)
    s.meta["apps"] = [a[0] for a in apps]
    return s


def with_user_limits(s: Snapshot, n_users: int = 3, seed: int = 0, frac: float = 0.5) -> Snapshot:
    """the same snapshot with `n_users` users owning the applications round-robin and a resource limit for some
    (queue, user) pairs -- on leaves and on their parents -- at about `frac` of what the user's asks there add up to"""
    import copy
    s = copy.deepcopy(s)
    rng = np.random.default_rng(seed)
    P, D = s.n_apps, s.D
    s.app_user = (np.arange(P) % n_users).astype(np.int32)
    if rng.random() < 0.3:
        s.app_user[rng.integers(0, P)] = -1
    demand = {}
    for a in range(s.n_asks):
        p = int(s.ask_app[a])
        u = int(s.app_user[p])
        if u < 0:
            continue
        q = int(s.app_queue[p])
        while q >= 0:
            demand.setdefault((q, u), np.zeros(D, dtype=np.int64))
            demand[(q, u)] += s.ask_req[a]
            q = int(s.q_parent[q])
    uq, uu, um = [], [], []
    for (q, u), d in sorted(demand.items()):
        if rng.random() < 0.5:
            continue
        mx = np.full(D, -1, dtype=np.int64)
        for k in rng.choice(D, size=int(rng.integers(1, 3)), replace=False):
            if d[k] > 0:
                mx[k] = max(1, int(d[k] * frac * (0.5 + rng.random())))
        uq.append(q); uu.append(u); um.append(mx)
    s.ul_queue, s.ul_user = np.array(uq, dtype=np.int32), np.array(uu, dtype=np.int32)
    s.ul_max = np.array(um, dtype=np.int64).reshape(len(uq), D)
    s.ul_alloc = np.zeros((len(uq), D), dtype=np.int64)
    s.name = f"{s.name}-userlimits"
    return s


def redim(s: Snapshot, D2: int, seed: int = 0) -> Snapshot:
    """The same snapshot with D2 resource dimensions (1..8): the first dimensions are kept, extra ones copy random existing
    columns (quotas: unset), weights are extended with 0 / 0.5 / 1 -- for tests of the code paths that depend on D."""
    import copy
    import random
    rng = random.Random(seed)
    s = copy.deepcopy(s)
    D = s.D

    def cols(x, fill):
        x = np.asarray(x)
        if D2 <= D:
            return np.ascontiguousarray(x[:, :D2])
        extra = np.stack([x[:, rng.randrange(D)] if fill is None else np.full(x.shape[0], fill, dtype=x.dtype)
                          for _ in range(D2 - D)], axis=1)
        return np.ascontiguousarray(np.concatenate([x, extra], axis=1))
    s.node_total, s.node_avail, s.ask_req = cols(s.node_total, None), cols(s.node_avail, None), cols(s.ask_req, None)
    s.q_guaranteed, s.q_max, s.q_alloc = cols(s.q_guaranteed, -1), cols(s.q_max, -1), cols(s.q_alloc, 0)
    if s.ul_max is not None and len(s.ul_max):
        s.ul_max, s.ul_alloc = cols(s.ul_max, -1), cols(s.ul_alloc, 0)
    w = np.zeros(D2)
    w[:min(D, D2)] = s.weights[:min(D, D2)]
    if D2 > D and rng.random() < 0.5:
        w[D:] = rng.choice([0.0, 1.0, 0.5])
    if w.sum() == 0:
        w[0] = 1.0
    s.weights, s.D = w, D2
    s.name = f"{s.name}-D{D2}"
    return s


def reweigh(s: Snapshot, w) -> Snapshot:
    """The same snapshot with node-sort weights `w` (one per resource dimension, >= 0) -- the scheduler's configured
    resource weights instead of the default vcore = memory = 1."""
    import copy
    w = np.asarray(w, dtype=np.float64)
    if w.shape != (s.D,):
        raise ValueError(f"expected {s.D} weights, got shape {w.shape}")
    if (w < 0).any() or not np.isfinite(w).all():
        raise ValueError("weights must be finite and >= 0")
    s = copy.deepcopy(s)
    s.weights = w.copy()
    s.name = f"{s.name}-w{'_'.join(f'{x:g}' for x in w)}"
    return s
