"""Second, independent restatement of the cycle in plain Python -- TEST INFRASTRUCTURE ONLY.

Written from SURVEY.md Appendix A, not from yk_oracle.cpp, and structured differently on purpose:
instead of walking a (score, NodeID)-sorted tree with early exit, each ask takes the *minimum*
(score, NodeID bytes) over all nodes that pass -- the exhaustive formulation the GPU uses.  Agreement of
the two on small snapshots is the only protection available while the Go reference cannot run here.
Only small cases: pure-Python loops.
"""
from __future__ import annotations

import math

UNSET = -1
ST_PENDING, ST_ALLOCATED, ST_NOFIT, ST_SKIPPED, ST_SLOWPATH, ST_INVALID = range(6)


def fit_in(larger, smaller):
    return all(sm <= max(0, lg) for lg, sm in zip(larger, smaller))


def strictly_gt_zero(r):
    return all(v >= 0 for v in r) and any(v > 0 for v in r)


def node_score(policy, w, total, avail):
    usage = 0.0
    tw = 0.0
    for k in range(len(w)):
        if w[k] == 0.0:
            continue
        t, v = float(total[k]), float(avail[k])
        if t == 0.0:        # Go float division: x/0 = +-Inf, 0/0 = NaN (the NaN share is skipped, the infinite one counts)
            if v == 0.0:
                continue
            share = 1.0 - math.copysign(math.inf, v)
        else:
            share = 1.0 - v / t
        if math.isnan(share):
            continue
        usage += share * w[k]
        tw += w[k]
    a = 0.0 if tw == 0.0 else usage / tw
    return ((1.0 - a) if policy == 1 else a) + 0.0


def shares(res, total):
    out = []
    for k, v in enumerate(res):
        if v == 0:
            out.append(0.0)
        elif total is None or total[k] <= 0:
            out.append(float(v))
        else:
            out.append(float(v) / float(total[k]))
    return sorted(out)


def compare_shares(l, r):
    l = list(reversed(l))
    r = list(reversed(r))
    for x, y in zip(l, r):
        if x > y:
            return 1
        if x < y:
            return -1
    if len(l) > len(r):
        return 1 if any(v > 0 for v in l[len(r):]) else 0
    if len(r) > len(l):
        return -1 if any(v > 0 for v in r[len(l):]) else 0
    return 0


def run(s, max_bindings=-1):
    D, N, A = s.D, s.n_nodes, s.n_asks
    w = [float(x) for x in s.weights]
    total = [[int(x) for x in row] for row in s.node_total]
    avail = [[int(x) for x in row] for row in s.node_avail]
    ids = [i.encode() for i in s.node_id]
    for n in range(N):   # a +Inf and a -Inf share: the score is NaN, rejected up front like the C++ oracle and the library
        if math.isnan(node_score(s.policy, w, total[n], avail[n])):
            raise ValueError(f"node {n} scores NaN")
    req = [[int(x) for x in row] for row in s.ask_req]
    Q = s.n_queues
    children = [[] for _ in range(Q)]
    for q in range(1, Q):
        children[int(s.q_parent[q])].append(q)
    q_alloc = [[int(x) for x in row] for row in s.q_alloc]
    q_pending = [[0] * D for _ in range(Q)]
    q_npend = [0] * Q
    q_apps = [[] for _ in range(Q)]
    for p in range(s.n_apps):
        q_apps[int(s.app_queue[p])].append(p)
    app_asks = [[] for _ in range(s.n_apps)]
    for a in range(A):
        app_asks[int(s.ask_app[a])].append(a)
    for p in range(s.n_apps):
        app_asks[p].sort(key=lambda a: (-int(s.ask_prio[a]), int(s.ask_create[a]), a))
    state = [ST_PENDING] * A
    dead = [False] * A
    held = getattr(s, "app_alloc", None)      # what each application holds from earlier cycles (None = nothing)
    app_alloc = [[int(x) for x in held[p]] if held is not None else [0] * D for p in range(s.n_apps)]

    def chain(q):
        while q >= 0:
            yield q
            q = int(s.q_parent[q])

    for a in range(A):
        for q in chain(int(s.app_queue[int(s.ask_app[a])])):
            q_npend[q] += 1
            for k in range(D):
                q_pending[q][k] += req[a][k]

    has_limits = getattr(s, "ul_queue", None) is not None and len(s.ul_queue) > 0
    ualloc = [[int(x) for x in (s.ul_alloc[l] if getattr(s, "ul_alloc", None) is not None else [0] * D)] for l in range(len(s.ul_queue))] if has_limits else []
    app_limits = {}

    def limits_of(p):
        """the user-limit entries that apply to the application: its user, a queue on its chain"""
        if p not in app_limits:
            out = []
            if has_limits and int(s.app_user[p]) >= 0:
                ch = set(chain(int(s.app_queue[p])))
                out = [l for l in range(len(s.ul_queue)) if int(s.ul_user[l]) == int(s.app_user[p]) and int(s.ul_queue[l]) in ch]
            app_limits[p] = out
        return app_limits[p]

    def with_user_headroom(p, hr):
        hr = list(hr)
        for l in limits_of(p):
            for k in range(D):
                mx = int(s.ul_max[l][k])
                if mx == UNSET:
                    continue
                own = max(0, mx - ualloc[l][k])
                hr[k] = own if hr[k] == UNSET else min(hr[k], own)
        return hr

    def headroom(q):
        hr = [UNSET] * D
        for qq in reversed(list(chain(q))):
            for k in range(D):
                mx = int(s.q_max[qq][k])
                if mx == UNSET:
                    continue
                own = max(0, mx - q_alloc[qq][k])
                hr[k] = own if hr[k] == UNSET else min(hr[k], own)
        return hr

    def passes_node(a, n):
        if not (int(s.node_flags[n]) & 1) or (int(s.node_flags[n]) & 2):
            return False
        if not fit_in(total[n], req[a]) or not fit_in(avail[n], req[a]):
            return False
        if int(s.ask_node[a]) >= 0 and int(s.ask_node[a]) != n:
            return False
        if int(s.node_taint[n]) & ~int(s.ask_tol[a]) & 0xFFFFFFFFFFFFFFFF:
            return False
        lab, need, deny = int(s.node_label[n]), int(s.ask_need[a]), int(s.ask_deny[a])
        return (lab & need) == need and (lab & deny) == 0

    def pick_node(a):
        best = None
        for n in range(N):
            if passes_node(a, n):
                key = (node_score(s.policy, w, total[n], avail[n]), ids[n])
                if best is None or key < best[0]:
                    best = (key, n)
        return None if best is None else best[1]

    def app_prio(p):
        pr = [int(s.ask_prio[a]) for a in app_asks[p] if state[a] != ST_ALLOCATED]
        return max(pr) if pr else -(1 << 31)

    def app_npend(p):
        return sum(1 for a in app_asks[p] if state[a] != ST_ALLOCATED)

    def apply(a, n, sign):
        for k in range(D):
            avail[n][k] -= sign * req[a][k]
        p = int(s.ask_app[a])
        for k in range(D):
            app_alloc[p][k] += sign * req[a][k]
        for l in limits_of(p):
            for k in range(D):
                ualloc[l][k] += sign * req[a][k]
        for qq in chain(int(s.app_queue[p])):
            q_npend[qq] -= sign
            for k in range(D):
                q_alloc[qq][k] += sign * req[a][k]
                q_pending[qq][k] -= sign * req[a][k]
        state[a] = ST_ALLOCATED if sign > 0 else ST_PENDING

    stop = [False]
    room = None

    def try_queue(q):
        nonlocal room
        if not children[q]:
            hr = headroom(q)
            cand = [p for p in q_apps[q] if app_npend(p) > 0]
            if int(s.q_sort[q]) == 1:
                import functools
                base = [int(x) for x in s.q_guaranteed[q]]

                def cmp(l, r):
                    pl, pr = app_prio(l), app_prio(r)
                    if pl != pr:
                        return -1 if pl > pr else 1
                    c = compare_shares(shares(app_alloc[l], base), shares(app_alloc[r], base))
                    if c:
                        return c
                    kl = (int(s.app_submit[l]), l)
                    kr = (int(s.app_submit[r]), r)
                    return -1 if kl < kr else (1 if kl > kr else 0)
                cand.sort(key=functools.cmp_to_key(cmp))
            else:
                cand.sort(key=lambda p: (-app_prio(p), int(s.app_submit[p]), p))
            hr_queue = hr
            for p in cand:
                if stop[0]:
                    return None
                hr = with_user_headroom(p, hr_queue)
                for a in app_asks[p]:
                    if stop[0]:
                        return None
                    if state[a] == ST_ALLOCATED or dead[a]:
                        continue
                    g = int(s.ask_gang[a])
                    if g < 0:
                        if int(s.ask_flags[a]) & 1:
                            state[a], dead[a] = ST_SLOWPATH, True
                            continue
                        if any(hr[k] != UNSET and req[a][k] > hr[k] for k in range(D)):
                            state[a], dead[a] = ST_SKIPPED, True
                            continue
                        if not strictly_gt_zero(req[a]):
                            state[a], dead[a] = ST_INVALID, True
                            continue
                    if g >= 0:      # a gang member: the gang-wide checks below decide for every member (all or nothing)
                        members = [m for m in app_asks[p] if int(s.ask_gang[m]) == g and state[m] != ST_ALLOCATED and not dead[m]]
                        placed, cause = [], 0
                        hrm = with_user_headroom(p, headroom(q))   # queue-side checks of all members first, headroom shrinking
                        for m in members:
                            if int(s.ask_flags[m]) & 1:
                                cause = ST_SLOWPATH
                            elif any(hrm[k] != UNSET and req[m][k] > hrm[k] for k in range(D)):
                                cause = ST_SKIPPED
                            elif not strictly_gt_zero(req[m]):
                                cause = ST_INVALID
                            if cause:
                                break
                            hrm = [hrm[k] if hrm[k] == UNSET else hrm[k] - req[m][k] for k in range(D)]
                        if not cause and room is not None and len(members) > room:
                            stop[0] = True          # passed the queue-side checks but does not fit in max_bindings: the
                            return None             # cycle ends (a gang sunk above needs no room and does not end it)
                        for m in members:           # then the node walks
                            if cause:
                                break
                            nm = pick_node(m)
                            if nm is None:
                                cause = ST_NOFIT
                                break
                            apply(m, nm, +1)
                            placed.append((m, nm))
                        if cause:
                            for m, nm in reversed(placed):
                                apply(m, nm, -1)
                            for m in members:
                                state[m], dead[m] = cause, True
                            continue
                        return placed
                    n = pick_node(a)
                    if n is not None:
                        apply(a, n, +1)
                        return [(a, n)]
                    state[a], dead[a] = ST_NOFIT, True
            return None
        import functools
        cand = [c for c in children[q] if q_npend[c] > 0]

        def queue_prio(x):            # highest priority among the asks still pending below queue x
            if not children[x]:
                pr = [app_prio(p) for p in q_apps[x] if app_npend(p) > 0]
            else:
                pr = [queue_prio(c) for c in children[x] if q_npend[c] > 0]
            best = max(pr) if pr else -(1 << 31)
            off = int(s.q_prio_offset[x]) if getattr(s, "q_prio_offset", None) is not None else 0
            fence = bool(s.q_prio_fence[x]) if getattr(s, "q_prio_fence", None) is not None else False
            return max(-(1 << 31), min((1 << 31) - 1, off + (0 if fence else best)))   # priorityValueByPolicy
        qp = {c: queue_prio(c) for c in cand}

        def qcmp(l, r):
            if qp[l] != qp[r]:            # priority first (sortQueuesByPriorityAndFairness), then the shares
                return -1 if qp[l] > qp[r] else 1
            c = compare_shares(shares(q_alloc[l], [int(x) for x in s.q_guaranteed[l]]),
                               shares(q_alloc[r], [int(x) for x in s.q_guaranteed[r]]))
            if c:
                return c
            d = [q_pending[l][k] - q_pending[r][k] for k in range(D)]
            if strictly_gt_zero(d):
                return -1
            if strictly_gt_zero([-x for x in d]):
                return 1
            return -1 if l < r else (1 if l > r else 0)
        cand.sort(key=functools.cmp_to_key(qcmp))
        for c in cand:
            r = try_queue(c)
            if r is not None or stop[0]:
                return r
        return None

    out = []
    while max_bindings < 0 or len(out) < max_bindings:
        room = None if max_bindings < 0 else max_bindings - len(out)
        r = try_queue(0)
        if r is None:
            break
        out.extend(r)
    return {"ask": [a for a, _ in out], "node": [n for _, n in out], "state": state, "avail": avail}
