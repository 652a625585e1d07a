"""yk_preemption_plan (DESIGN.md §2 item 9) at the edges the first fuzz never reaches, against tests/preemption_oracle.py.

Every cluster here is played as one script: phase 1 places the victims' pods, phase 2 blocks the preemptors, then four plan
calls with random changes between them (releases, a removed or resized preemptor, resized victims, cordoned, uncordoned,
shrunk, re-tainted, re-labelled and removed nodes, and cycles that spend plans while marks stay).  The oracle writes the
script once, with the C++ oracle's cycles on a compacted snapshot of its own state; every engine configuration replays it and
must give the same status, node and victim list for every preemptor, and the same bindings, states and availability after
every cycle.

The clusters (`edge_cluster`): random queue trees of 10-40 queues up to depth 6 with guarantees, maxima, fences and
priority offsets at every level; priorities at INT32_MIN / INT32_MAX and offsets near +-2^31, so that the int32 clamp of
the adjusted priority decides orders; create times with ties and near +-2^63; required-node victims; slow-path, gang and
required-node preemptors; users with limits, on and off the preemptor's chain; 16-300 nodes with taints, labels, cordons and
reservations; clusters with more than 256 bound allocations, so that the victim kernel runs over several CTAs and the
node kernel over several blocks; and totals near 2^62 in the first resource."""
import copy
import functools

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
import preemption_oracle as po
from test_preemption_plan import YK_NONE, NO_SELF, NO_OTHER, ORIGINATOR

I32MIN, I32MAX = po.I32
I64MIN, I64MAX = -(1 << 63), (1 << 63) - 1
FAMILIES = ("masks", "wide", "offsets", "huge")
ASK_COLS = ("ask_app", "ask_req", "ask_tol", "ask_need", "ask_deny", "ask_prio", "ask_create", "ask_node", "ask_flags", "ask_gang")
SLOWPATH = 1
# every D three times, under both node sorts, and every family at most D
CASES = [(seed, D, (seed // 3 + D) % 2) for seed in range(9) for D in range(1, 9) if (seed + D) % 3 == 0]


def _tree(rng):
    """parent, depth, leaves: 10-40 queues, depth up to 6, leaves at different depths"""
    while True:
        Qn = int(rng.integers(10, 41))
        parent, depth = [-1], [0]
        for q in range(1, Qn):
            cand = [p for p in range(q) if depth[p] < 6]
            p = cand[int(len(cand) * rng.random() ** 0.5)]          # leans toward later queues: deep paths
            parent.append(p)
            depth.append(depth[p] + 1)
        leaves = [q for q in range(1, Qn) if q not in parent]
        if len(leaves) >= 4 and len({depth[q] for q in leaves}) >= 2:
            return parent, depth, leaves


def _chain(parent, q):
    out = []
    while q >= 0:
        out.append(q)
        q = parent[q]
    return out


def edge_cluster(seed, D, policy):
    """-> (snapshot of every ask, n1): asks [0, n1) are the victims' pods (phase 1), the rest the preemptors (phase 2)"""
    rng = np.random.default_rng(7919 * seed + 3)
    fam = FAMILIES[seed % 4]
    parent, depth, leaves = _tree(rng)
    hot = None
    if fam == "wide":   # Y under the root with a preemptor leaf and a victim leaf whose pods sort after the others
        Y = len(parent)
        parent += [0, Y, Y]
        depth += [1, 2, 2]
        hot = (Y, Y + 1, Y + 2)
        leaves = leaves + [Y + 1, Y + 2]
    G = len(parent)          # a preemptors' leaf over its guarantee from the start: GUARANTEE
    parent += [0]
    depth += [1]
    Qn = len(parent)
    perm = [leaves[i] for i in rng.permutation(len(leaves))]
    npre = max(1, len(leaves) // 3)
    pre_leaves, vic_leaves = perm[:npre], perm[npre:]
    if hot:
        pre_leaves = [q for q in pre_leaves if q != hot[2]] + ([hot[1]] if hot[1] not in pre_leaves else [])
        vic_leaves = [q for q in vic_leaves if q != hot[1]] + ([hot[2]] if hot[2] not in vic_leaves else [])
    pre_leaves = pre_leaves + [G]
    leaves = leaves + [G]
    P = len(leaves)
    app_of = {q: i for i, q in enumerate(leaves)}

    # nodes
    N = int({"masks": rng.integers(16, 41), "wide": rng.integers(200, 301), "offsets": rng.integers(16, 33),
             "huge": rng.integers(16, 25)}[fam])
    unit = [2000, 4000, 110, 100_000] if fam == "wide" else [8000, 16000, 110, 100_000]
    S = (1 << 62) // (N * (unit[0] + 1000)) if fam == "huge" else 1          # first resource's scale: sums near 2^62
    tot = np.tile(np.array(unit, np.int64), (N, 1))
    if S > 1:
        tot[:, 0] = tot[:, 0] * S + rng.integers(0, S, N)
    taint = np.where(rng.random(N) < 0.35, np.uint64(1) << rng.integers(0, 4, N).astype(np.uint64), np.uint64(0)).astype(np.uint64)
    label = ((np.uint64(1) << rng.integers(0, 3, N).astype(np.uint64)) | (np.uint64(1) << (3 + rng.integers(0, 3, N)).astype(np.uint64)))
    nflags = np.where(rng.random(N) < 0.08, 3, 1).astype(np.uint32)              # reserved nodes: the cycle skips them
    usable = np.nonzero(nflags == 1)[0]

    def vec(c):
        return [c * S + (int(rng.integers(0, 1000)) if S > 1 else 0), 2 * c, 1, int(rng.integers(1, 100))]

    # phase 1: victims until the usable nodes are ~90 % full
    cap = tot[usable, :2].sum(axis=0)
    sizes = [250, 500, 1000] if fam == "wide" else [500, 1000, 1500]
    load = np.zeros(2, dtype=np.int64)
    vreq, vleaf = [], []
    while True:
        r = vec(int(rng.choice(sizes)))
        if (load + np.array(r[:2]) > 0.9 * cap).any():
            break
        load += np.array(r[:2])
        vreq.append(r)
        vleaf.append(hot[2] if hot and rng.random() < 0.12 else int(rng.choice(vic_leaves)))
    n1 = len(vreq)
    v_prio = rng.choice([-5, 0, 5, I32MIN, I32MAX], n1, p=[0.3, 0.3, 0.3, 0.05, 0.05])
    if fam == "offsets":   # with an offset near -2^31 above them, these leave int32 at different depths
        v_prio = rng.choice([-50, -5, 0, I32MIN], n1, p=[0.3, 0.3, 0.2, 0.2])
    if hot:
        v_prio = np.where(np.array(vleaf) == hot[2], 100, rng.choice([-5, 0, 5], n1))
    v_flags = rng.choice([0, NO_SELF, ORIGINATOR, NO_SELF | ORIGINATOR], n1, p=[0.6, 0.15, 0.15, 0.1])
    if hot:   # the hot leaf's pods sort after every other victim: the headroom step reaches past position 256
        v_flags = np.where(np.array(vleaf) == hot[2], NO_SELF | ORIGINATOR, rng.choice([0, ORIGINATOR], n1, p=[0.8, 0.2]))
    v_node = np.where(rng.random(n1) < 0.2, rng.choice(usable, n1), -1)

    # phase 2: preemptors
    n2 = int(rng.integers(16, 24) if fam == "wide" else rng.integers(24, 40))
    psizes = [1000, 1500, 2000] if fam == "wide" else [2000, 3000, 4000]
    preq = [vec(int(c)) for c in rng.choice(psizes, n2)]
    pleaf = [hot[1] if hot and rng.random() < 0.5 else G if rng.random() < 0.08 else int(rng.choice(pre_leaves[:-1]))
             for _ in range(n2)]
    p_prio = rng.choice([5, 10, 20, I32MAX, I32MIN], n2, p=[0.3, 0.3, 0.3, 0.05, 0.05])
    if hot:
        p_prio = np.where(np.array(pleaf) == hot[1], 1000, p_prio)
    p_flags = rng.choice([0, NO_OTHER, SLOWPATH], n2, p=[0.93, 0.05, 0.02])
    p_node = np.where(rng.random(n2) < 0.04, rng.choice(usable, n2), -1)
    p_gang = np.full(n2, -1)
    for i in range(0, n2 - 1):
        if p_gang[i] < 0 and rng.random() < 0.04:         # a pair in one application
            p_gang[i] = p_gang[i + 1] = i
            pleaf[i + 1] = pleaf[i]
    # one preemptor leaf keeps three pods and gets a user limit they rarely pass (below)
    others = [q for q in pre_leaves if q != G and (not hot or q != hot[1])]
    tight_leaf = int(rng.choice(others)) if len(others) > 1 else None
    if tight_leaf is not None:
        rest = [q for q in pre_leaves if q not in (tight_leaf, G)]
        mine = [i for i in range(n2) if pleaf[i] == tight_leaf and p_gang[i] < 0]
        for i in mine[3:]:
            pleaf[i] = int(rng.choice(rest))
    p_tol = rng.integers(0, 16, n2).astype(np.uint64)
    p_need = np.where(rng.random(n2) < 0.3, np.uint64(1) << rng.integers(0, 6, n2).astype(np.uint64), np.uint64(0)).astype(np.uint64)
    p_need[rng.random(n2) < 0.05] = np.uint64(1 << 6)                             # a label no node has: no node at all
    p_deny = np.where(rng.random(n2) < 0.15, np.uint64(1) << rng.integers(0, 6, n2).astype(np.uint64), np.uint64(0)).astype(np.uint64)
    p_deny &= ~p_need

    A = n1 + n2
    req = np.array(vreq + preq, dtype=np.int64)
    app = np.array([app_of[q] for q in vleaf + pleaf], dtype=np.int32)
    prio = np.concatenate([v_prio, p_prio]).astype(np.int32)
    flags = np.concatenate([v_flags, p_flags]).astype(np.uint32)
    anode = np.concatenate([v_node, p_node]).astype(np.int32)
    gang = np.concatenate([np.full(n1, -1), p_gang]).astype(np.int32)
    tol = np.concatenate([np.full(n1, 0xF, np.uint64), p_tol]).astype(np.uint64)
    need = np.concatenate([np.zeros(n1, np.uint64), p_need]).astype(np.uint64)
    deny = np.concatenate([np.zeros(n1, np.uint64), p_deny]).astype(np.uint64)
    create = rng.integers(0, max(2, A // 8), A).astype(np.int64)                  # ties
    if fam in ("offsets", "huge"):
        far = rng.random(A) < 0.3
        create[far] = np.where(rng.random(A) < 0.5, I64MIN + rng.integers(0, 4, A), I64MAX - rng.integers(0, 4, A))[far]

    # queues: guarantees at every level, maxima above the preemptors' leaves, offsets, fences
    demand = np.zeros((Qn, 4), dtype=np.int64)
    for r, q in zip(vreq, vleaf):
        for x in _chain(parent, q):
            demand[x] += r
    above_pre = {x for q in pre_leaves for x in _chain(parent, q)}
    guar = np.full((Qn, 4), -1, dtype=np.int64)
    mx = np.full((Qn, 4), -1, dtype=np.int64)
    for q in range(1, Qn):
        dims = [0] + [1] * (rng.random() < 0.8)
        if q in pre_leaves:
            for k in dims:
                guar[q, k] = int(int(cap[k]) * rng.uniform(0.2, 0.4))
            if q == G:
                guar[q] = -1
                guar[q, 0] = 1
        elif q in vic_leaves:
            if rng.random() < 0.85:
                for k in dims:
                    guar[q, k] = int(int(demand[q, k]) * rng.uniform(0.05, 0.5))
        elif q in above_pre:
            u = rng.random()
            if u < 0.25:
                for k in dims:
                    guar[q, k] = int(demand[q, k]) + int(cap[k])
            elif u < 0.32:
                guar[q, 0] = int(demand[q, 0] // 2)
            if rng.random() < 0.25:
                mx[q, 0] = int(demand[q, 0]) + int(rng.integers(0, 3000)) * S
        elif rng.random() < 0.3:
            for k in dims:
                guar[q, k] = int(int(demand[q, k]) * rng.uniform(0.2, 0.7))
    if hot:
        guar[hot[2]] = -1
        guar[hot[0]] = -1
        mx[hot[0], 0] = int(demand[hot[0], 0]) + int(rng.integers(0, 400)) * S
    off = np.where(rng.random(Qn) < 0.25, rng.choice([-10, 10], Qn), 0).astype(np.int64)
    if fam == "offsets":   # near -2^31 above victims (two on one path leave int32), near +2^31 on preemptors' leaves
        low = (rng.random(Qn) < 0.5) & ~np.isin(np.arange(Qn), list(above_pre))
        off[low] = (I32MIN + rng.integers(0, 50, Qn))[low]
        high = (rng.random(Qn) < 0.3) & np.isin(np.arange(Qn), pre_leaves)
        off[high] = (I32MAX - rng.integers(0, 50, Qn))[high]
    if hot:
        off[list(hot)] = 0
    fence = rng.random(Qn) < 0.06
    if hot:
        fence[list(hot)] = False
    qsort = np.where(rng.random(Qn) < 0.3, synth.SORT_FAIR, synth.SORT_FIFO).astype(np.uint8)

    ids = [f"n{int(x):04d}" for x in rng.permutation(N)]
    t = synth._finish(f"plan-edge-{fam}-{seed}", 4, policy, tot, tot.copy(), taint, label, ids,
                      (np.array(parent, dtype=np.int32), guar, mx, np.zeros((Qn, 4), np.int64), qsort),
                      np.array(leaves, dtype=np.int32), app, req, tol, need, deny, ask_prio=prio, ask_node=anode,
                      ask_flags=flags, ask_gang=gang, node_flags=nflags, ask_create=create)
    t.q_prio_offset = off.astype(np.int32)
    t.q_pp_fence = fence.astype(np.uint8)
    # users: limits on the preemptors' chains (some preemptors are over them) and limits off every chain of their user
    t.app_user = rng.integers(-1, 3, P).astype(np.int32)
    uq, uu, um = [], [], []
    # that leaf's limit (one only: a limit the cycle fills binds every later pod of its user below it)
    if tight_leaf is not None and int(t.app_user[app_of[tight_leaf]]) < 0:
        t.app_user[app_of[tight_leaf]] = int(rng.integers(0, 3))
    for q in [tight_leaf] if tight_leaf is not None else []:
        u = int(t.app_user[app_of[q]])
        x = q
        held = sum((np.array(r) for r, l in zip(vreq, vleaf) if x in _chain(parent, l) and int(t.app_user[app_of[l]]) == u),
                   np.zeros(4, np.int64))
        m = np.full(4, -1, np.int64)
        m[0] = int(held[0]) + int(rng.integers(0, 2000)) * S
        uq.append(x); uu.append(u); um.append(m)
        break
    for _ in range(2):
        u = int(rng.integers(0, 3))
        mine = {x for p in range(P) if int(t.app_user[p]) == u for x in _chain(parent, leaves[p])}
        off_chain = [q for q in range(1, Qn) if q not in mine and not any(x in mine for x in range(Qn) if q in _chain(parent, x))]
        qq = int(rng.choice(off_chain)) if off_chain else None
        if qq is not None and (qq, u) not in zip(uq, uu):
            m = np.full(4, -1, np.int64)
            m[0] = 0
            uq.append(qq); uu.append(u); um.append(m)
    t.ul_queue, t.ul_user = np.array(uq, dtype=np.int32), np.array(uu, dtype=np.int32)
    t.ul_max = np.array(um, dtype=np.int64).reshape(len(uq), 4)
    t.ul_alloc = np.zeros((len(uq), 4), dtype=np.int64)
    t.meta = dict(family=fam, hot=hot)
    return _dims(t, D), n1


def _dims(t, D):
    """t with D resources: the first D, or the four and then copies of memory, storage and pods (the same column for
    totals, availability and requests, so that every pod still fits an empty node; quotas unset, weight 0.5)"""
    if D == 4:
        return t
    t = copy.deepcopy(t)
    src = list(range(min(D, 4))) + [(1, 3, 2)[k % 3] for k in range(max(0, D - 4))]
    for f in ("node_total", "node_avail", "ask_req", "q_alloc", "ul_alloc"):
        setattr(t, f, np.ascontiguousarray(getattr(t, f)[:, src]))
    for f in ("q_guaranteed", "q_max", "ul_max"):
        x = np.ascontiguousarray(getattr(t, f)[:, src])
        x[:, 4:] = -1
        setattr(t, f, x)
    t.weights = np.array([1.0, 1.0, 0.0, 0.0, 0.5, 0.5, 0.5, 0.5][:D])
    t.D = D
    t.name = f"{t.name}-D{D}"
    return t


# ---- the script: the oracle's run, which every engine configuration replays ----
def oracle_cycle(w, oracle):
    """a cycle of the C++ oracle on a compacted snapshot of w's pending world; w follows its bindings and states"""
    s = w.s
    pend = [a for a in range(s.n_asks) if w.state[a] not in (po.ST_ALLOCATED, 255)]
    nodes = sorted(w.present_nodes)
    pos = {n: i for i, n in enumerate(nodes)}
    t = copy.copy(s)
    t.node_total, t.node_taint, t.node_label, t.node_flags = (s.node_total[nodes], s.node_taint[nodes], s.node_label[nodes],
                                                              s.node_flags[nodes])
    t.node_avail = np.array([w.avail[n] for n in nodes], dtype=np.int64).reshape(len(nodes), w.D)
    t.node_id = [s.node_id[n] for n in nodes]
    t.q_alloc = np.array(w.alloc, dtype=np.int64)
    for f in ASK_COLS:
        setattr(t, f, getattr(s, f)[pend])
    t.ask_req = np.array([w.req[a] for a in pend], dtype=np.int64).reshape(len(pend), w.D)
    t.ask_node = np.array([pos[int(x)] if x >= 0 else -1 for x in s.ask_node[pend]], dtype=np.int32)
    if w.ul:
        t.ul_alloc = np.array([held for (_, _, _, held) in w.ul], dtype=np.int64).reshape(len(w.ul), w.D)
    want = oracle.run(t)
    ask = [pend[int(i)] for i in want["ask"]]
    node = [nodes[int(i)] for i in want["node"]]
    for a, n in zip(ask, node):
        w.allocate(a, n)
    for a, st in zip(pend, want["state"]):
        w.state[a] = int(st)
    return ("cycle", ask, node, pend, [w.state[a] for a in pend], nodes, [list(w.avail[n]) for n in nodes])


class Script:
    """the oracle's World driven through engine-shaped steps; `steps` is what an engine replays"""

    def __init__(self, full, oracle):
        self.full, self.oracle = full, oracle
        self.w = po.World(copy.deepcopy(full), {}, np.full(full.n_asks, 255), full.node_avail)
        self.steps, self.info, self.since = [], [], set()

    def upsert(self, idx):
        idx = [int(a) for a in idx]
        self.steps.append(("asks_upsert", idx))
        for a in idx:
            self.w.state[a] = 0
            self.w.plans.pop(a, None)

    def remove(self, idx):
        self.steps.append(("asks_remove", list(idx)))
        self.w.remove(idx)

    def release(self, idx):
        self.steps.append(("release", list(idx)))
        self.w.release(idx)

    def resize(self, a, new):
        self.steps.append(("resize", a, [int(x) for x in new]))
        self.w.resize(a, new)
        self.since.add("resize")

    def node_upsert(self, n, total=None, avail=None, taint=None, label=None, flags=None):
        s = self.w.s
        total = [int(x) for x in (s.node_total[n] if total is None else total)]
        avail = list(self.w.avail[n]) if avail is None else [int(x) for x in avail]
        taint = int(s.node_taint[n]) if taint is None else int(taint)
        label = int(s.node_label[n]) if label is None else int(label)
        flags = int(s.node_flags[n]) if flags is None else int(flags)
        self.steps.append(("nodes_upsert", n, total, avail, taint, label, flags))
        self.w.node_upsert(n, total, avail, taint, label, flags)

    def node_remove(self, n):
        self.steps.append(("nodes_remove", n))
        self.w.node_remove(n)
        self.since.add("node_remove")

    def cycle(self):
        self.steps.append(oracle_cycle(self.w, self.oracle))

    def plan(self, order, call):
        inf = []
        got = po.plan(self.w, order, inf)
        for x in inf:
            x.update(call=call, since=set(self.since))
        self.info += inf
        self.steps.append(("plan", [int(a) for a in order], got))
        return got


def _session(sc, rng, n1, calls=4):
    """plan calls with random changes between them (DESIGN §2 item 9: marks clear on release, plans on allocation, removal and
    resize; removed nodes hold no victims)"""
    w, full = sc.w, sc.full
    A = full.n_asks
    cordoned = {}
    for call in range(calls):
        blocked = [a for a in range(n1, A) if w.state[a] in (po.ST_NOFIT, po.ST_SKIPPED)]
        others = [int(a) for a in rng.choice(A, 3, replace=False) if a not in blocked]
        order = [int(a) for a in rng.permutation(blocked)] + others
        got = sc.plan(order, call)
        if call == calls - 1:
            break
        planned = [a for a, x in zip(order, got) if x[0] == po.PLANNED]
        victims = [v for x in got for v in x[2]]
        ops = ["release_planned", "release_other", "remove_planned", "resize_victim", "resize_preemptor", "cordon", "uncordon",
               "shrink", "masks", "remove_node", "cycle"]
        drawn = list(rng.permutation(ops)[:int(rng.integers(3, 7))])
        drawn += [op for op in (["resize_victim"] if call == 0 else ["remove_node"] if call == 1 else []) if op not in drawn]
        for op in drawn:
            bound = sorted(w.bound)
            present = sorted(w.present_nodes)
            if op == "release_planned" and victims:
                sc.release([v for v in victims[::2] if v in w.bound])
            elif op == "release_other" and bound:
                sc.release([int(v) for v in rng.choice(bound, min(3, len(bound)), replace=False)])
            elif op == "remove_planned":
                live = [a for a in planned if a in w.plans]
                if live:
                    sc.remove([live[0]])
            elif op == "resize_victim" and bound:
                marked = sorted(w.marked)
                for v in ([int(rng.choice(marked))] if marked else []) + [int(rng.choice(bound))]:
                    if v in w.bound:
                        r = np.array(w.req[v], dtype=np.int64)
                        sc.resize(v, r + r // 2 if rng.random() < 0.5 else r - r // 2)
            elif op == "resize_preemptor":
                live = [a for a in planned if a in w.plans]
                if live:
                    r = np.array(w.req[live[-1]], dtype=np.int64)
                    sc.resize(live[-1], r - r // 3 if rng.random() < 0.5 else r + r // 3)
            elif op == "cordon" and present:
                busy = [n for n in present if any(w.bound[v] == n for v in w.marked)] or present
                n = int(rng.choice(busy))
                cordoned[n] = int(w.s.node_flags[n])
                sc.node_upsert(n, flags=0)
            elif op == "uncordon" and cordoned:
                n, f = cordoned.popitem()
                if n in w.present_nodes:
                    sc.node_upsert(n, flags=f or 1)
            elif op == "shrink" and present:
                n = int(rng.choice(present))
                tot = np.array(w.s.node_total[n], dtype=np.int64)
                cut = tot // 4
                sc.node_upsert(n, total=tot - cut, avail=np.array(w.avail[n], dtype=np.int64) - cut)
            elif op == "masks" and present:
                n = int(rng.choice(present))
                sc.node_upsert(n, taint=int(1 << int(rng.integers(0, 4))) if rng.random() < 0.5 else 0,
                               label=int((1 << int(rng.integers(0, 3))) | (1 << int(rng.integers(3, 6)))))
            elif op == "remove_node":   # never the required node of a pending ask: its cycle would need the node
                pinned = {int(full.ask_node[a]) for a in range(A) if w.state[a] not in (po.ST_ALLOCATED, 255)}
                cand = [n for n in present if n not in pinned and any(w.bound[v] == n for v in bound)]
                marked_on = [n for n in cand if any(w.bound[v] == n for v in w.marked)]
                if cand and len(present) > 2:
                    sc.node_remove(int(rng.choice(marked_on or cand)))
            elif op == "cycle":
                sc.cycle()


@functools.lru_cache(maxsize=None)
def edge_script(seed, D, policy):
    """-> (full snapshot, Script) of one cluster: both phases and the session, on the oracle alone"""
    from oracle import oracle_ctypes
    oracle_ctypes.build()
    full, n1 = edge_cluster(seed, D, policy)
    sc = Script(full, oracle_ctypes)
    rng = np.random.default_rng(seed * 131 + D * 7 + policy)
    sc.upsert(range(n1))
    sc.cycle()
    left = [a for a in range(n1) if sc.w.state[a] != po.ST_ALLOCATED]
    if left:
        sc.remove(left)
    # between the phases: some nodes holding victims are cordoned or reserved (the plan reads neither the reservation nor
    # the cycle's skipping of reserved nodes)
    busy = sorted({n for n in sc.w.bound.values()})
    for n in rng.permutation(busy)[:max(1, len(busy) // 8)]:
        sc.node_upsert(int(n), flags=int(rng.choice([0, 3])))
    sc.upsert(range(n1, full.n_asks))
    sc.cycle()
    # before the first plan call: a node holding victims is removed (its pods stay allocated but are no victims) and one
    # victim is resized
    pinned = {int(full.ask_node[a]) for a in range(full.n_asks) if sc.w.state[a] not in (po.ST_ALLOCATED, 255)}
    busy = sorted({n for n in sc.w.bound.values() if n in sc.w.present_nodes and n not in pinned})
    if busy:
        sc.node_remove(int(rng.choice(busy)))
    v = int(rng.choice(sorted(sc.w.bound)))
    r = np.array(sc.w.req[v], dtype=np.int64)
    sc.resize(v, r + r // 2 if rng.random() < 0.5 else r - r // 2)
    _session(sc, rng, n1)
    return full, sc


def _engine(full, commit, batch, binpacking_device=False):
    from yunikorn_k8shim_b200 import Engine
    e = Engine(D=full.D, policy=full.policy, weights=full.weights, max_nodes=full.n_nodes, max_asks=full.n_asks,
               max_apps=full.n_apps, max_queues=full.n_queues, commit=commit, batch=batch, binpacking_device=binpacking_device)
    e.queues_set(full.q_parent, full.q_guaranteed, full.q_max, full.q_alloc, full.q_sort)
    e.queues_priority(full.q_prio_offset)
    e.queues_preemption(full.q_pp_fence)
    e.nodes_upsert(np.arange(full.n_nodes), full.node_total, full.node_avail, full.node_taint, full.node_label, full.node_rank(),
                   full.node_flags)
    e.apps_upsert(np.arange(full.n_apps), full.app_queue, full.app_submit)
    if getattr(full, "ul_queue", None) is not None and len(full.ul_queue):
        e.apps_user(np.arange(full.n_apps), full.app_user)
        e.user_limits_set(full.ul_queue, full.ul_user, full.ul_max, full.ul_alloc)
    return e


def replay(full, steps, commit, batch, binpacking_device=False, on_cycle=None):
    """drive an engine through the script; every cycle and every plan must equal the oracle's"""
    rank = full.node_rank()
    where = f"{full.name} [{commit}, batch {batch}]"
    with _engine(full, commit, batch, binpacking_device) as e:
        for i, step in enumerate(steps):
            op = step[0]
            if op == "asks_upsert":
                a = np.asarray(step[1], dtype=np.int64)
                e.asks_upsert(a, full.ask_req[a], full.ask_app[a], full.ask_create[a], full.ask_tol[a], full.ask_need[a],
                              full.ask_deny[a], full.ask_prio[a], full.ask_node[a], full.ask_flags[a], full.ask_gang[a])
            elif op == "asks_remove":
                e.asks_remove(step[1])
            elif op == "release":
                if step[1]:
                    e.release(step[1])
            elif op == "resize":
                e.asks_resize([step[1]], np.array([step[2]], dtype=np.int64))
            elif op == "nodes_upsert":
                _, n, total, avail, taint, label, flags = step
                e.nodes_upsert([n], np.array([total], dtype=np.int64), np.array([avail], dtype=np.int64), [taint], [label],
                               [rank[n]], [flags])
            elif op == "nodes_remove":
                e.nodes_remove([step[1]])
            elif op == "cycle":
                _, ask, node, pend, states, nodes, avail = step
                before = e.stats()
                got_a, got_n, _ = e.cycle(len(pend) + 1)
                assert got_a.tolist() == ask and got_n.tolist() == node, f"{where} step {i}: bindings differ"
                assert e.ask_states(pend).tolist() == states if pend else True, f"{where} step {i}: ask states differ"
                assert e.nodes_available(nodes).tolist() == avail, f"{where} step {i}: availability differs"
                if on_cycle:
                    after = e.stats()
                    on_cycle(i, {k: v - before[k] for k, v in after.items() if not isinstance(v, list)})
            elif op == "plan":
                _, order, want = step
                st, nd, vic, done = e.preemption_plan(order)
                got = [(int(x), None if n == YK_NONE else int(n), [int(v) for v in vs]) for x, n, vs in zip(st, nd, vic)]
                assert done == len(order), f"{where} step {i}: {done} of {len(order)} planned"
                bad = [(a, g, x) for a, g, x in zip(order, got, want) if g != x]
                assert not bad, f"{where} step {i}: plans differ (ask, engine, oracle): {bad[:3]}"


# ---- 1 and 2: the edge fuzz, every D, both node sorts, every commit, two batch sizes ----
@pytest.mark.gpu
@pytest.mark.parametrize("seed,D,policy", CASES, ids=[f"s{s}-D{d}-{'bp' if p else 'fair'}" for s, d, p in CASES])
def test_edge_fuzz(seed, D, policy):
    full, sc = edge_script(seed, D, policy)
    for commit in ("host", "device", "auto"):
        for batch in (64, 4096):
            replay(full, sc.steps, commit, batch)


def _facts(sc):
    """coverage counts of one script: statuses (NOT_ALLOWED split by cause) and the edges each plan went through"""
    w, s = sc.w, sc.full
    c = {}

    def add(k, n=1):
        c[k] = c.get(k, 0) + n
    for step in sc.steps:
        if step[0] != "plan":
            continue
        for a, (st, _, vs) in zip(step[1], step[2]):
            name = ["planned", "fits", "not_blocked", "not_allowed", "unsupported", "guarantee", "no_victims"][st]
            if st == po.NOT_ALLOWED:
                name = "not_allowed_flag" if int(s.ask_flags[a]) & NO_OTHER else "not_allowed_user"
            add(name)
    for x in sc.info:
        add("masked", x["masked"])
        add("required_skipped", x["required_skipped"] > 0)
        add("clamp_decides", x["clamp_decides"])
        add("rule7_past_256", x["pos7"] >= 256)
        add("after_node_remove", "node_remove" in x["since"])
        add("after_resize", "resize" in x["since"])
        add("create_ties", x["create_ties"])
    return c


def test_edge_coverage_floors(oracle):
    """for every D: every status (NOT_ALLOWED by flag and by user limit), plans, plans whose fewest-victims node is cordoned
    or masked, plans after a node removal and after a resize, victim lists with create-time ties; over all D, plans next to
    required-node allocations.  Per family where only that family draws the edge: in every "wide" cluster, plans whose headroom
    victims lie past position 256 of the victim order (more than one CTA of the victim kernel); over the "offsets"
    clusters, plans whose victims an int32 wrap of the adjusted priority would reorder (`test_clamp_decides_the_order`
    holds one such plan by construction)"""
    per_d = dict(planned=10, fits=3, not_blocked=30, not_allowed_flag=3, not_allowed_user=10, unsupported=10, guarantee=10,
                 no_victims=10, masked=2, after_node_remove=10, after_resize=10, create_ties=2)
    fam = {}
    for D in range(1, 9):
        c = {}
        for seed, d, policy in CASES:
            if d != D:
                continue
            full, sc = edge_script(seed, d, policy)
            f = _facts(sc)
            if full.meta["family"] == "wide":
                assert f.get("rule7_past_256", 0) >= 5, (full.name, f)
            for k, v in f.items():
                c[k] = c.get(k, 0) + v
                fam[(full.meta["family"], k)] = fam.get((full.meta["family"], k), 0) + v
        short = {k: (c.get(k, 0), f) for k, f in per_d.items() if c.get(k, 0) < f}
        assert not short, (D, short, c)
    assert fam.get(("offsets", "clamp_decides"), 0) >= 3, fam
    # required-node allocations on the chosen node: drawn at random, so over all D
    assert sum(v for (f, k), v in fam.items() if k == "required_skipped") >= 10, fam


# ---- a removed node that holds the first victim in order ----
def removed_node_script(oracle):
    """root -> Y (max 4 pods' vcore) -> {V, P}: four pods of V fill Y on two nodes; P's pod fits a node but not Y's max, so
    the headroom step takes the first victim in order, the newest pod.  Its node is removed before the plan: the removed
    node's allocations are no victims, so the plan takes the newest pod on the node left"""
    D = 4
    tot = np.tile(np.array([3000, 3000, 110, 100], np.int64), (2, 1))
    guar = np.full((4, D), -1, np.int64)
    mx = np.full((4, D), -1, np.int64)
    guar[3, :2] = 10_000
    mx[1, 0] = 4000
    req = np.tile(np.array([1000, 1000, 1, 1], np.int64), (5, 1))
    z = np.zeros(5, np.uint64)
    full = synth._finish("plan-removed-node", D, synth.POLICY_FAIR, tot, tot.copy(), np.zeros(2, np.uint64), np.zeros(2, np.uint64),
                         ["node-a", "node-b"], (np.array([-1, 0, 1, 1], np.int32), guar, mx, np.zeros((4, D), np.int64),
                                                np.zeros(4, np.uint8)),
                         np.array([2, 3], np.int32), np.array([0, 0, 0, 0, 1], np.int32), req, z, z.copy(), z.copy(),
                         ask_create=np.arange(5, dtype=np.int64))
    full.q_prio_offset = np.zeros(4, np.int32)
    full.q_pp_fence = np.zeros(4, np.uint8)
    sc = Script(full, oracle)
    sc.upsert(range(4))
    sc.cycle()
    sc.upsert([4])
    sc.cycle()
    assert sc.w.state[4] == po.ST_SKIPPED and len(sc.w.bound) == 4
    newest = max(sc.w.bound, key=lambda a: int(full.ask_create[a]))
    gone = sc.w.bound[newest]
    sc.node_remove(gone)
    (st, node, vic), = sc.plan([4], 0)
    assert st == po.PLANNED and node != gone and len(vic) == 1 and sc.w.bound[vic[0]] != gone, (st, node, vic)
    return full, sc


def test_removed_node_script(oracle):
    removed_node_script(oracle)


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_removed_node_holds_the_first_victim(oracle, commit):
    full, sc = removed_node_script(oracle)
    replay(full, sc.steps, commit, 64)


# ---- an order the int32 clamp decides ----
def clamp_script(oracle):
    """root -> A (offset -2^31) -> V (offset -2^31), root -> P: V's three pods fill the node and their adjusted priorities
    (their own plus 2 * -2^31) all leave int32.  Clamped they tie at INT32_MIN and the newest goes first; an int32 wrap would
    order them by their own priorities and give the oldest, lowest one instead"""
    D = 4
    tot = np.array([[3000, 3000, 110, 100]], np.int64)
    guar = np.full((4, D), -1, np.int64)
    guar[3, :2] = 10_000
    req = np.tile(np.array([1000, 1000, 1, 1], np.int64), (4, 1))
    z = np.zeros(4, np.uint64)
    full = synth._finish("plan-clamp", D, synth.POLICY_FAIR, tot, tot.copy(), np.zeros(1, np.uint64), np.zeros(1, np.uint64),
                         ["node-a"], (np.array([-1, 0, 1, 0], np.int32), guar, np.full((4, D), -1, np.int64),
                                      np.zeros((4, D), np.int64), np.zeros(4, np.uint8)),
                         np.array([2, 3], np.int32), np.array([0, 0, 0, 1], np.int32), req, z, z.copy(), z.copy(),
                         ask_prio=np.array([0, -100, -50, 0], np.int32), ask_create=np.array([1, 0, -1, 5], np.int64))
    full.q_prio_offset = np.array([0, I32MIN, I32MIN, 0], np.int32)
    full.q_pp_fence = np.zeros(4, np.uint8)
    sc = Script(full, oracle)
    sc.upsert(range(3))
    sc.cycle()
    sc.upsert([3])
    sc.cycle()
    assert len(sc.w.bound) == 3 and sc.w.state[3] == po.ST_NOFIT
    (st, node, vic), = sc.plan([3], 0)
    assert (st, node, vic) == (po.PLANNED, 0, [0]) and sc.info[-1]["clamp_decides"], (st, node, vic, sc.info)
    return full, sc


def test_clamp_script(oracle):
    clamp_script(oracle)


@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_clamp_decides_the_order(oracle, commit):
    full, sc = clamp_script(oracle)
    replay(full, sc.steps, commit, 64)


# ---- 3: the plan after each commit path of the cycle that placed the victims ----
PATHS = ("host", "uniform", "rounds", "fill", "lattice")


def path_script(oracle, path):
    """12 nodes filled by one fifo leaf's pods in a cycle on the path under test; then six preemptors of a guaranteed leaf
    that the next cycle blocks, and one plan call for all of them.  The plan reads the allocations, states, availability and
    queue usage that path left on the host"""
    D = 4
    N = 12
    tot = np.tile(np.array([8000, 16000, 110, 4000], np.int64), (N, 1))
    if path == "rounds":
        vreq = [[100 * (1 + i % 5), 200 * (1 + i % 3), 1, 1] for i in range(400)]
    elif path == "lattice":
        vreq = [[(500, 1000, 1500)[i % 3], (1000, 2000, 3000)[i % 3], 1, 1] for i in range(150)]
    else:
        vreq = [[1000, 2000, 1, 10]] * 100
    n1 = len(vreq)
    req = np.array(vreq + [[3000, 6000, 1, 10]] * 6, np.int64)
    A = len(req)
    guar = np.full((3, D), -1, np.int64)
    guar[2, :2] = [40_000, 80_000]
    z = np.zeros(A, np.uint64)
    policy = synth.POLICY_BINPACKING if path == "fill" else synth.POLICY_FAIR
    full = synth._finish(f"plan-after-{path}", D, policy, tot, tot.copy(), np.zeros(N, np.uint64), np.zeros(N, np.uint64),
                         [f"n{i:02d}" for i in range(N)], (np.array([-1, 0, 0], np.int32), guar, np.full((3, D), -1, np.int64),
                                                            np.zeros((3, D), np.int64), np.zeros(3, np.uint8)),
                         np.array([1, 2], np.int32), np.array([0] * n1 + [1] * 6, np.int32), req, z, z.copy(), z.copy(),
                         ask_prio=np.array([0] * n1 + [10] * 6, np.int32),
                         ask_flags=np.array([(0, NO_SELF, ORIGINATOR, 0, 0)[i % 5] for i in range(n1)] + [0] * 6, np.uint32))
    full.q_prio_offset = np.zeros(3, np.int32)
    full.q_pp_fence = np.zeros(3, np.uint8)
    sc = Script(full, oracle)
    sc.upsert(range(n1))
    sc.cycle()
    left = [a for a in range(n1) if sc.w.state[a] != po.ST_ALLOCATED]
    if left:
        sc.remove(left)
    sc.upsert(range(n1, A))
    sc.cycle()
    got = sc.plan(list(range(n1, A)), 0)
    assert sum(1 for x in got if x[0] == po.PLANNED) >= 3, got
    return full, sc


def path_engine(path, monkeypatch):
    """(commit, binpacking_device) of the path, and its environment"""
    monkeypatch.setenv("YK_UNIFORM_MIN", "8")
    if path == "rounds":
        monkeypatch.setenv("YK_ROUND_MIN", "1")
        monkeypatch.setenv("YK_ROUND_GUARD", "0")
    return {"host": ("host", False), "uniform": ("device", False), "rounds": ("auto", False), "fill": ("device", True),
            "lattice": ("device", False)}[path]


@pytest.mark.parametrize("path", PATHS)
def test_path_script(oracle, path):
    path_script(oracle, path)


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS)
def test_plan_after_each_commit_path(oracle, monkeypatch, path):
    """the victims' cycle ran on the path under test (from the counters), and the plan equals the oracle's"""
    full, sc = path_script(oracle, path)
    commit, bp = path_engine(path, monkeypatch)
    per = {}
    replay(full, sc.steps, commit, 4096, bp, on_cycle=lambda i, d: per.setdefault("first", d))
    d = per["first"]
    if path == "host":
        assert d["lattice_cycles"] == 0 and d["sweep_launches"] > 0, d
    elif path == "rounds":
        assert d["lattice_cycles"] == 1 and d["round_asks"] > 0, d
    elif path == "lattice":
        assert d["lattice_cycles"] == 1 and d["lattice_asks"] > 0 and d["uniform_asks"] == 0, d
    else:   # uniform run; the binpacking fill is a uniform run under the binpacking sort
        assert d["lattice_cycles"] == 1 and d["uniform_runs"] > 0 and d["uniform_asks"] > 0, d
