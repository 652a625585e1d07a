"""Preemption for queues below their guarantee (DESIGN.md §2 item 9), restated in plain Python -- TEST INFRASTRUCTURE ONLY.

Written from the rules, not from the engine: no engine code, no preorder intervals, no sort keys.  Every eligible victim of a
node is re-tested with explicit sums over the queue paths, and the node choice is a plain loop over the node order.  The state
is the oracle's own: a `World` built from a snapshot and the bindings of the oracle's cycle, changed by `release`, `remove`,
`allocate` and `resize` as the engine's calls change it.
"""
from __future__ import annotations

import math

import numpy as np

from oracle.py_oracle import node_score

PLANNED, FITS, NOT_BLOCKED, NOT_ALLOWED, UNSUPPORTED, GUARANTEE, NO_VICTIMS = range(7)
ST_ALLOCATED, ST_NOFIT, ST_SKIPPED = 1, 2, 3
NO_SELF, NO_OTHER, ORIGINATOR = 2, 4, 8
I32 = (-(1 << 31), (1 << 31) - 1)


class World:
    """s: a synth.Snapshot (plus q_pp_fence, [Q] bool, optional); bound: {ask: node} of the asks allocated; state: per-ask
    state after the cycle; avail: [N][D] node availability after the cycle"""

    def __init__(self, s, bound, state, avail):
        self.s, self.D = s, s.D
        self.parent = [int(x) for x in s.q_parent]
        self.parent[0] = -1
        self.Q = len(self.parent)
        self.guar = [[int(x) for x in row] for row in s.q_guaranteed]
        self.qmax = [[int(x) for x in row] for row in s.q_max]
        self.off = [int(x) for x in s.q_prio_offset] if getattr(s, "q_prio_offset", None) is not None else [0] * self.Q
        self.fence = [bool(x) for x in s.q_pp_fence] if getattr(s, "q_pp_fence", None) is not None else [False] * self.Q
        self.req = {a: [int(x) for x in s.ask_req[a]] for a in range(s.n_asks)}
        self.state = {a: int(state[a]) for a in range(s.n_asks)}
        self.bound = dict(bound)
        self.avail = [[int(x) for x in row] for row in avail]
        self.alloc = [[int(x) for x in row] for row in s.q_alloc]
        for a in self.bound:
            for q in self.path(self.leaf(a)):
                for k in range(self.D):
                    self.alloc[q][k] += self.req[a][k]
        self.present_nodes = set(range(s.n_nodes))
        self.ul = []   # (user, queue, max, held)
        if getattr(s, "ul_queue", None) is not None:
            for l in range(len(s.ul_queue)):
                held = [int(x) for x in s.ul_alloc[l]] if getattr(s, "ul_alloc", None) is not None else [0] * self.D
                self.ul.append((int(s.ul_user[l]), int(s.ul_queue[l]), [int(x) for x in s.ul_max[l]], held))
            for a in self.bound:
                for (u, q, _, held) in self.ul_of(a):
                    for k in range(self.D):
                        held[k] += self.req[a][k]
        self.marked = set()
        self.plans = {}

    # ---- tree ----
    def leaf(self, a):
        return int(self.s.app_queue[int(self.s.ask_app[a])])

    def path(self, q):
        out = []
        while q >= 0:
            out.append(q)
            q = self.parent[q]
        return out

    def lca(self, x, y):
        px = self.path(x)
        for q in self.path(y):
            if q in px:
                return q
        return 0

    def below(self, x, c):
        """queues on x's path strictly below c"""
        out = []
        for q in self.path(x):
            if q == c:
                break
            out.append(q)
        return out

    def ul_of(self, a):
        p = int(self.s.ask_app[a])
        user = int(self.s.app_user[p]) if getattr(self.s, "app_user", None) is not None else -1
        if user < 0:
            return []
        chain = self.path(self.leaf(a))
        return [e for e in self.ul if e[0] == user and e[1] in chain]

    # ---- engine calls ----
    def release(self, asks):
        for a in asks:
            n = self.bound.pop(a)
            for k in range(self.D):
                if n in self.present_nodes:
                    self.avail[n][k] += self.req[a][k]
            for q in self.path(self.leaf(a)):
                for k in range(self.D):
                    self.alloc[q][k] -= self.req[a][k]
            for (_, _, _, held) in self.ul_of(a):
                for k in range(self.D):
                    held[k] -= self.req[a][k]
            self.state[a] = 255
            self.marked.discard(a)

    def remove(self, asks):
        for a in asks:
            self.state[a] = 255
            self.plans.pop(a, None)

    def allocate(self, a, n):
        """what a cycle binding does"""
        self.bound[a] = n
        self.state[a] = ST_ALLOCATED
        for k in range(self.D):
            self.avail[n][k] -= self.req[a][k]
        for q in self.path(self.leaf(a)):
            for k in range(self.D):
                self.alloc[q][k] += self.req[a][k]
        for (_, _, _, held) in self.ul_of(a):
            for k in range(self.D):
                held[k] += self.req[a][k]
        self.plans.pop(a, None)

    def resize(self, a, new):
        self.req[a] = [int(x) for x in new]
        self.plans.pop(a, None)

    # ---- plan-call views ----
    def usage(self, q):
        u = list(self.alloc[q])
        for v in self.marked:
            if q in self.path(self.leaf(v)):
                u = [u[k] - self.req[v][k] for k in range(self.D)]
        for p in self.plans:
            if q in self.path(self.leaf(p)):
                u = [u[k] + self.req[p][k] for k in range(self.D)]
        return u

    def room(self, n):
        r = list(self.avail[n])
        for v in self.marked:
            if self.bound[v] == n:
                r = [r[k] + self.req[v][k] for k in range(self.D)]
        for p, pn in self.plans.items():
            if pn == n:
                r = [r[k] - self.req[p][k] for k in range(self.D)]
        return r

    def node_order(self):
        s = self.s
        w = [float(x) for x in s.weights]
        ranks = s.node_rank()
        nodes = sorted(self.present_nodes)
        sc = {n: node_score(s.policy, w, [int(x) for x in s.node_total[n]], self.avail[n]) for n in nodes}
        if any(math.isnan(v) for v in sc.values()):
            raise ValueError("NaN node score")
        return sorted(nodes, key=lambda n: (sc[n], int(ranks[n]), n))

    def static_ok(self, a, n):
        s = self.s
        if not (int(s.node_flags[n]) & 1):
            return False
        if int(s.node_taint[n]) & ~int(s.ask_tol[a]) & 0xFFFFFFFFFFFFFFFF:
            return False
        lab, need, deny = int(s.node_label[n]), int(s.ask_need[a]), int(s.ask_deny[a])
        if (lab & need) != need or (lab & deny):
            return False
        return all(self.req[a][k] <= max(0, int(s.node_total[n][k])) for k in range(self.D))


def _has_guarantee(w, q):
    return any(g >= 0 for g in w.guar[q])


def plan(w, asks, info=None):
    """-> [(status, node or None, [victims])] per ask handled, marking and planning in w as the engine does.  info (a list):
    one dict per plan made -- victims needed on the node, headroom victims bound elsewhere, whether an earlier ask of the
    same call was planned -- for the tests' coverage counts"""
    out = []
    order = w.node_order() if w.present_nodes else []
    for a in asks:
        a = int(a)
        s = w.s
        st = w.state.get(a, 255)
        fl = int(s.ask_flags[a])
        if st not in (ST_NOFIT, ST_SKIPPED) or a in w.plans:
            out.append((NOT_BLOCKED, None, []))
            continue
        if fl & NO_OTHER:
            out.append((NOT_ALLOWED, None, []))
            continue
        if (fl & 1) or int(s.ask_gang[a]) >= 0 or int(s.ask_node[a]) >= 0:
            out.append((UNSUPPORTED, None, []))
            continue
        if any(held[k] + w.req[a][k] > mx[k] for (_, _, mx, held) in w.ul_of(a) for k in range(w.D) if mx[k] >= 0):
            out.append((NOT_ALLOWED, None, []))
            continue
        L = w.leaf(a)
        use = {q: w.usage(q) for q in range(w.Q)}
        if not _has_guarantee(w, L) or any(w.guar[q][k] >= 0 and use[q][k] + w.req[a][k] > w.guar[q][k]
                                           for q in w.path(L) for k in range(w.D)):
            out.append((GUARANTEE, None, []))
            continue
        fence = next((q for q in w.path(L) if w.fence[q]), 0)

        def adjusted(x, prio, c):
            return prio + sum(w.off[q] for q in w.below(x, c))

        victims = []
        for v in sorted(w.bound):
            if w.state.get(v) != ST_ALLOCATED or v in w.marked or int(s.ask_node[v]) >= 0 or w.bound[v] not in w.present_nodes:
                continue
            x = w.leaf(v)
            if x == L or fence not in w.path(x):
                continue
            c = w.lca(x, L)
            pv, pa = adjusted(x, int(s.ask_prio[v]), c), adjusted(L, int(s.ask_prio[a]), c)
            if pv > pa:
                continue
            fv = int(s.ask_flags[v])
            victims.append(((1 if fv & NO_SELF else 0, 1 if fv & ORIGINATOR else 0, min(max(pv, I32[0]), I32[1]),
                             -int(s.ask_create[v]), v), v))
        victims = [v for _, v in sorted(victims)]

        def allowed(v, taken):
            """rule 5: v may go once `taken` are gone"""
            x = w.leaf(v)
            for q in w.below(x, w.lca(x, L)):
                if not _has_guarantee(w, q):
                    continue
                gone = [sum(w.req[t][k] for t in taken + [v] if q in w.path(w.leaf(t))) for k in range(w.D)]
                if any(w.guar[q][k] >= 0 and use[q][k] - gone[k] < w.guar[q][k] for k in range(w.D)):
                    return False
            return True

        def fits(r):
            return all(w.req[a][k] <= max(0, r[k]) for k in range(w.D))

        best = None
        for n in order:
            if not w.static_ok(a, n):
                continue
            r = w.room(n)
            taken = []
            if not fits(r):
                for v in victims:
                    if w.bound[v] != n or not allowed(v, taken):
                        continue
                    taken.append(v)
                    r = [r[k] + w.req[v][k] for k in range(w.D)]
                    if fits(r):
                        break
                if not fits(r):
                    continue
            if best is None or len(taken) < len(best[1]):
                best = (n, taken)
        if best is None:
            out.append((NO_VICTIMS, None, []))
            continue
        node, v6 = best
        taken = list(v6)

        def over(q):
            gone = [sum(w.req[t][k] for t in taken if q in w.path(w.leaf(t))) for k in range(w.D)]
            return any(w.qmax[q][k] >= 0 and use[q][k] - gone[k] + w.req[a][k] > w.qmax[q][k] for k in range(w.D))

        v7 = []
        for v in victims:
            deficit = [q for q in w.path(L) if over(q)]
            if not deficit:
                break
            if v in taken or not any(q in w.path(w.leaf(v)) for q in deficit) or not allowed(v, taken):
                continue
            taken.append(v)
            v7.append(v)
        if any(over(q) for q in w.path(L)):
            out.append((NO_VICTIMS, None, []))
            continue
        if not taken:
            out.append((FITS, node, []))
            continue
        if info is not None:
            info.append(dict(need=len(v6), off_node=sum(1 for v in v7 if w.bound[v] != node),
                             after_plan=any(x[0] == PLANNED for x in out)))
        out.append((PLANNED, node, taken))
        w.marked.update(taken)
        w.plans[a] = node
    return out


def world_from_cycle(s, want):
    """the World after the oracle's cycle `want` (py_oracle.run / oracle_ctypes.run) on snapshot s"""
    bound = {int(a): int(n) for a, n in zip(want["ask"], want["node"])}
    return World(s, bound, np.asarray(want["state"]), want["avail"])
