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
        """an allocation moves by new - old in its node (while present), queues and user entries; a pending ask's plan goes"""
        new = [int(x) for x in new]
        if a in self.bound:
            n = self.bound[a]
            d = [new[k] - self.req[a][k] for k in range(self.D)]
            for k in range(self.D):
                if n in self.present_nodes:
                    self.avail[n][k] -= d[k]
            for q in self.path(self.leaf(a)):
                for k in range(self.D):
                    self.alloc[q][k] += d[k]
            for (_, _, _, held) in self.ul_of(a):
                for k in range(self.D):
                    held[k] += d[k]
        self.req[a] = new
        self.plans.pop(a, None)

    def node_upsert(self, n, total, avail, taint=0, label=0, flags=1):
        """yk_nodes_upsert of one node: its tables are what is given (a removed node comes back with them)"""
        s = self.s
        s.node_total[n] = total
        s.node_taint[n], s.node_label[n], s.node_flags[n] = taint, label, flags
        self.avail[n] = [int(x) for x in avail]
        self.present_nodes.add(n)

    def node_remove(self, n):
        """yk_nodes_remove: allocations bound there stay allocated, but are no victims and give nothing back on release"""
        self.present_nodes.discard(n)
        self.s.node_flags[n] = 0

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

    def usages(self):
        """usage(q) of every queue, in one pass"""
        u = [list(row) for row in self.alloc]
        for v, sign in [(v, -1) for v in self.marked] + [(p, 1) for p in self.plans]:
            for q in self.path(self.leaf(v)):
                for k in range(self.D):
                    u[q][k] += sign * self.req[v][k]
        return dict(enumerate(u))

    def room(self, n):
        r = list(self.avail[n])
        for v in self.marked:
            if self.bound[v] == n:
                r = [r[k] + self.req[v][k] for k in range(self.D)]
        for p, pn in self.plans.items():
            if pn == n:
                r = [r[k] - self.req[p][k] for k in range(self.D)]
        return r

    def rooms(self):
        """room(n) of every present node, in one pass"""
        r = {n: list(self.avail[n]) for n in self.present_nodes}
        for v, n, sign in [(v, self.bound[v], 1) for v in self.marked] + [(p, n, -1) for p, n in self.plans.items()]:
            if n in r:
                for k in range(self.D):
                    r[n][k] += sign * self.req[v][k]
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
    one dict per plan made, for the tests' coverage counts: victims needed on the node, headroom victims bound elsewhere,
    whether an earlier ask of the same call was planned, whether a node that fails only the cordon / taint / label steps
    would have needed fewer victims (or as few, earlier in the order), how many allocations on the node would be victims but for
    their required node, whether an int32 wrap instead of the clamp would reorder the node's victims, the victim-order
    position of the last headroom victim, and whether two victims share a create time"""
    out = []
    order = w.node_order() if w.present_nodes else []
    s = w.s
    D = w.D
    for a in asks:
        a = int(a)
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
        if any(held[k] + w.req[a][k] > mx[k] for (_, _, mx, held) in w.ul_of(a) for k in range(D) if mx[k] >= 0):
            out.append((NOT_ALLOWED, None, []))
            continue
        L = w.leaf(a)
        use = w.usages()
        if not _has_guarantee(w, L) or any(w.guar[q][k] >= 0 and use[q][k] + w.req[a][k] > w.guar[q][k]
                                           for q in w.path(L) for k in range(D)):
            out.append((GUARANTEE, None, []))
            continue
        fence = next((q for q in w.path(L) if w.fence[q]), 0)

        def adjusted(x, prio, c):
            return prio + sum(w.off[q] for q in w.below(x, c))

        def candidate(v):
            """rule 3 apart from the required node: v's adjusted priority, or None"""
            if w.state.get(v) != ST_ALLOCATED or v in w.marked or w.bound[v] not in w.present_nodes:
                return None
            x = w.leaf(v)
            if x == L or fence not in w.path(x):
                return None
            c = w.lca(x, L)
            pv, pa = adjusted(x, int(s.ask_prio[v]), c), adjusted(L, int(s.ask_prio[a]), c)
            return None if pv > pa else pv

        victims, required = [], []
        for v in sorted(w.bound):
            pv = candidate(v)
            if pv is None:
                continue
            if int(s.ask_node[v]) >= 0:
                required.append((v, pv))
                continue
            fv = int(s.ask_flags[v])
            victims.append(((1 if fv & NO_SELF else 0, 1 if fv & ORIGINATOR else 0, min(max(pv, I32[0]), I32[1]),
                             -int(s.ask_create[v]), v), v, pv))
        victims.sort()
        adj = {v: pv for _, v, pv in victims}
        victims = [v for _, v, _ in victims]

        def allowed(v, taken):
            """rule 5: v may go once `taken` are gone"""
            x = w.leaf(v)
            for q in w.below(x, w.lca(x, L)):
                if not _has_guarantee(w, q):
                    continue
                gone = [sum(w.req[t][k] for t in taken + [v] if q in w.path(w.leaf(t))) for k in range(D)]
                if any(w.guar[q][k] >= 0 and use[q][k] - gone[k] < w.guar[q][k] for k in range(D)):
                    return False
            return True

        def fits(r):
            return all(w.req[a][k] <= max(0, r[k]) for k in range(D))

        rooms = w.rooms()
        on_node = {}
        for v in victims:
            on_node.setdefault(w.bound[v], []).append(v)

        def walk(n):
            """rule 6 on node n: the fewest victims in order after which the ask fits, or None"""
            r = list(rooms[n])
            taken = []
            if not fits(r):
                for v in on_node.get(n, []):
                    if not allowed(v, taken):
                        continue
                    taken.append(v)
                    r = [r[k] + w.req[v][k] for k in range(D)]
                    if fits(r):
                        break
                if not fits(r):
                    return None
            return taken

        def masks_ok(n):
            return w.static_ok(a, n)

        def total_ok(n):
            return all(w.req[a][k] <= max(0, int(s.node_total[n][k])) for k in range(D))

        best, masked = None, None
        for n in order:
            if not total_ok(n):
                continue
            ok = masks_ok(n)
            if not ok and info is None:
                continue
            taken = walk(n)
            if taken is None:
                continue
            if ok and (best is None or len(taken) < len(best[1])):
                best = (n, taken)
            if masked is None or len(taken) < len(masked[1]):
                masked = (n, taken, ok)
        if best is None:
            out.append((NO_VICTIMS, None, []))
            continue
        node, v6 = best
        taken = list(v6)

        def over(q):
            gone = [sum(w.req[t][k] for t in taken if q in w.path(w.leaf(t))) for k in range(D)]
            return any(w.qmax[q][k] >= 0 and use[q][k] - gone[k] + w.req[a][k] > w.qmax[q][k] for k in range(D))

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
            mine = on_node.get(node, [])
            last = mine.index(v6[-1]) if v6 else -1
            walked_key = {v: (min(max(adj[v], I32[0]), I32[1]), -int(s.ask_create[v]), v) for v in mine}
            wrapped_key = {v: ((adj[v] + (1 << 31)) % (1 << 32) - (1 << 31), -int(s.ask_create[v]), v) for v in mine}
            flags = {v: (int(s.ask_flags[v]) & NO_SELF, int(s.ask_flags[v]) & ORIGINATOR) for v in mine}
            creates = [int(s.ask_create[v]) for v in taken]
            info.append(dict(
                need=len(v6), off_node=sum(1 for v in v7 if w.bound[v] != node),
                after_plan=any(x[0] == PLANNED for x in out),
                masked=masked[2] is False,
                required_skipped=sum(1 for v, _ in required if w.bound[v] == node) if v6 else 0,
                clamp_decides=bool(v6) and sorted(mine, key=lambda v: (flags[v], walked_key[v]))[:last + 1]
                != sorted(mine, key=lambda v: (flags[v], wrapped_key[v]))[:last + 1],
                pos7=max((victims.index(v) for v in v7), default=-1),
                create_ties=len(set(creates)) < len(creates)))
        out.append((PLANNED, node, taken))
        w.marked.update(taken)
        w.plans[a] = node
    return out


def world_from_cycle(s, want):
    """the World after the oracle's cycle `want` (py_oracle.run / oracle_ctypes.run) on snapshot s"""
    bound = {int(a): int(n) for a, n in zip(want["ask"], want["node"])}
    return World(s, bound, np.asarray(want["state"]), want["avail"])
