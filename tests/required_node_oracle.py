"""Preemption for asks with a required node (DaemonSet pods, DESIGN.md §2 item 10), restated in plain Python -- TEST
INFRASTRUCTURE ONLY.

Written from the rules, not from the engine: no groups, no segments, no sort keys.  The victims of a preemptor are found by
looping over the allocations on its node and taking, again and again, the first remaining one by an explicit pairwise
comparison.  The state is preemption_oracle.World, so marks and plans are shared with the guarantee oracle and every World
call (release, remove, allocate, resize) changes both the same way.
"""
from __future__ import annotations

import preemption_oracle as po
from preemption_oracle import PLANNED, FITS, NOT_BLOCKED, NOT_ALLOWED, UNSUPPORTED, NO_VICTIMS  # noqa: F401

NO_SELF, ORIGINATOR = po.NO_SELF, po.ORIGINATOR


def victim_type(w, v):
    """0: neither flag, 1: NO_PREEMPT_SELF and not an originator, 2: an originator"""
    f = int(w.s.ask_flags[v])
    if f & ORIGINATOR:
        return 2
    return 1 if f & NO_SELF else 0


def before(w, u, v):
    """u comes before v in victim order: type, then priority ascending, then create_seq descending, then index"""
    s = w.s
    if victim_type(w, u) != victim_type(w, v):
        return victim_type(w, u) < victim_type(w, v)
    if int(s.ask_prio[u]) != int(s.ask_prio[v]):
        return int(s.ask_prio[u]) < int(s.ask_prio[v])
    if int(s.ask_create[u]) != int(s.ask_create[v]):
        return int(s.ask_create[u]) > int(s.ask_create[v])
    return u < v


def over_headroom(w, a):
    """a queue max on a's path or a user / group limit that applies to a would go over with a's request, from what is
    allocated"""
    D = w.D
    for q in w.path(w.leaf(a)):
        for k in range(D):
            if w.qmax[q][k] >= 0 and w.alloc[q][k] + w.req[a][k] > w.qmax[q][k]:
                return True
    for (_, _, mx, held) in w.ul_of(a):
        for k in range(D):
            if mx[k] >= 0 and held[k] + w.req[a][k] > mx[k]:
                return True
    return False


def plan_required(w, asks, info=None):
    """-> [(status, [victims])] per ask, marking and planning in w as the engine does.  info (a list): one dict per ask, for
    the tests' coverage counts"""
    s, D = w.s, w.D
    # room and the allocations of each node, once per call (the plans and marks of this call are folded in as they happen)
    rooms = w.rooms()
    on_node = {}
    for v in sorted(w.bound):
        on_node.setdefault(w.bound[v], []).append(v)
    out, planned_here = [], set()
    for a in asks:
        a = int(a)
        x = int(s.ask_node[a])
        note = dict(status=None, victims=0, same_node_before=False, type_decides=False, shortfall_differs=False)
        if w.state.get(a, 255) not in (po.ST_NOFIT, po.ST_SKIPPED) or a in w.plans:
            st, victims = NOT_BLOCKED, []
        elif x < 0 or int(s.ask_flags[a]) & 1 or int(s.ask_gang[a]) >= 0:
            st, victims = UNSUPPORTED, []
        elif over_headroom(w, a):
            st, victims = NOT_ALLOWED, []
        elif x not in w.present_nodes or not w.static_ok(a, x):
            st, victims = NO_VICTIMS, []
        elif all(w.req[a][k] <= max(0, rooms[x][k]) for k in range(D)):
            st, victims = FITS, []
        else:
            cands = []
            for v in on_node.get(x, []):
                if w.state.get(v) != po.ST_ALLOCATED or v in w.marked or int(s.ask_node[v]) >= 0:
                    continue
                if int(s.ask_prio[v]) > int(s.ask_prio[a]):
                    continue
                if not any(w.req[v][k] != 0 and w.req[a][k] != 0 for k in range(D)):
                    continue
                cands.append(v)
            left = list(cands)
            victims, total = [], [0] * D
            while left and not all(total[k] >= w.req[a][k] for k in range(D)):
                first = left[0]
                for v in left:
                    if before(w, v, first):
                        first = v
                left.remove(first)
                victims.append(first)
                total = [total[k] + w.req[first][k] for k in range(D)]
            if all(total[k] >= w.req[a][k] for k in range(D)):
                st = PLANNED
                # coverage facts: would the part room(x) lacks have needed fewer victims; did the type decide the order
                lack = [max(0, w.req[a][k] - max(0, rooms[x][k])) for k in range(D)]
                part, need = [0] * D, 0
                for v in victims:
                    if all(part[k] >= lack[k] for k in range(D)):
                        break
                    part = [part[k] + w.req[v][k] for k in range(D)]
                    need += 1
                note["shortfall_differs"] = need < len(victims)
                types = {victim_type(w, v) for v in cands}
                note["type_decides"] = len(types) > 1
                note["same_node_before"] = x in planned_here
                note["type_decides"] = note["type_decides"] and len(victims) < len(cands)
            else:
                st, victims = NO_VICTIMS, []
        note["status"], note["victims"] = st, len(victims)
        if info is not None:
            info.append(note)
        if st == PLANNED:
            w.marked.update(victims)
            w.plans[a] = x
            planned_here.add(x)
            for v in victims:
                for k in range(D):
                    rooms[x][k] += w.req[v][k]
            for k in range(D):
                rooms[x][k] -= w.req[a][k]
        out.append((st, victims))
    return out
