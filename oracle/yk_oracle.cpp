// yk_oracle.cpp -- TEST INFRASTRUCTURE ONLY (see yk_oracle.h header comment).
//
// Sequential CPU restatement of the reference's scheduling cycle.  It keeps the
// reference's *structure* on purpose: one allocation per schedule() pass, queues
// and applications re-sorted on every pass, nodes walked in ascending
// (score, NodeID) order with early exit at the first node that passes, one
// predicate call per (ask,node) visited, re-key of the committed node.
//
// What each function follows:
//   fit_in / strictly_gt_zero  yunikorn-core pkg/common/resources/resources.go (FitIn,
//                              StrictlyGreaterThanZero)              [EXT, SURVEY A.2]
//   yko_node_score             yunikorn-core objects/node.go GetResourceUsageShares +
//                              objects/nodesorting.go absResourceUsage/ScoreNode [EXT, A.3]
//   NodeLess                   yunikorn-core objects/node_collection.go nodeRef.Less [EXT, A.3]
//   shim_predicates            pkg/plugin/predicates/predicate_manager.go:202-283
//                              (podFitsNode: prefilter then filters, first failure wins) with the
//                              k8s plugins restated as mask ops (SURVEY A.4); entry through
//                              pkg/cache/scheduler_callback.go:196-198 -> pkg/cache/context.go:683-703
//   try_node / try_nodes       yunikorn-core objects/application.go tryNodes/tryNode,
//                              objects/node.go preAllocateCheck/TryAddAllocation [EXT, A.2]
//   get_shares/compare_shares  yunikorn-core resources.go getShares/compareShares  [EXT]
//   headroom                   yunikorn-core objects/queue.go getHeadRoom/internalHeadRoom [EXT]
//   try_queue                  yunikorn-core objects/queue.go TryAllocate/sortQueues/sortApplications [EXT]
//   request vectors (inputs)   pkg/common/resource.go:56-109,188-195,273-285
//
// Build: g++ -O2 -std=c++17 -ffp-contract=off -fPIC -shared (oracle/Makefile).
#include "yk_oracle.h"

#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <set>
#include <string>
#include <vector>

namespace {

constexpr int64_t UNSET = -1;

inline int64_t clamp0(int64_t v) { return v < 0 ? 0 : v; }

// FitIn(larger, smaller): for every type in smaller: smaller <= max(0, larger or 0)
inline bool fit_in(int D, const int64_t* larger, const int64_t* smaller) {
    for (int k = 0; k < D; ++k)
        if (smaller[k] > clamp0(larger[k])) return false;
    return true;
}
// no negative quantity and at least one positive one
inline bool strictly_gt_zero(int D, const int64_t* r) {
    bool pos = false;
    for (int k = 0; k < D; ++k) {
        if (r[k] < 0) return false;
        if (r[k] > 0) pos = true;
    }
    return pos;
}

double node_score(int D, int policy, const double* w, const int64_t* total, const int64_t* avail) {
    double usage = 0.0, tw = 0.0;
    for (int k = 0; k < D; ++k) {
        if (w[k] == 0.0) continue;       // unweighted types do not count
        // Go float division: x/0 = +-Inf (the infinite share counts), 0/0 = NaN (skipped below)
        double share = 1.0 - (double)avail[k] / (double)total[k];
        if (std::isnan(share)) continue;
        usage += share * w[k];
        tw += w[k];
    }
    double abs_usage = (tw == 0.0) ? 0.0 : usage / tw;
    double s = (policy == YKO_POLICY_BINPACKING) ? 1.0 - abs_usage : abs_usage;
    return s + 0.0;  // -0.0 -> +0.0 (Go compares them equal; keeps the order total)
}

struct NodeRef {
    double score;
    int32_t rank;   // rank of NodeID in bytewise string order
    int32_t node;
};
struct NodeLess {
    bool operator()(const NodeRef& a, const NodeRef& b) const {
        if (a.score < b.score) return true;
        if (b.score < a.score) return false;
        return a.rank < b.rank;
    }
};

std::vector<double> get_shares(int D, const int64_t* res, const int64_t* total) {
    std::vector<double> sh((size_t)D, 0.0);
    for (int k = 0; k < D; ++k) {
        int64_t v = res[k];
        if (v == 0) continue;
        if (total == nullptr || total[k] <= 0) sh[(size_t)k] = (double)v;   // unset (-1) or 0 total
        else sh[(size_t)k] = (double)v / (double)total[k];
    }
    std::sort(sh.begin(), sh.end());
    return sh;
}
int compare_shares(const std::vector<double>& l, const std::vector<double>& r) {
    int li = (int)l.size() - 1, ri = (int)r.size() - 1;
    while (ri >= 0 && li >= 0) {
        if (l[(size_t)li] > r[(size_t)ri]) return 1;
        if (l[(size_t)li] < r[(size_t)ri]) return -1;
        --li; --ri;
    }
    if (li == -1 && ri == -1) return 0;
    for (; li >= 0; --li) if (l[(size_t)li] > 0) return 1;
    for (; ri >= 0; --ri) if (r[(size_t)ri] > 0) return -1;
    return 0;
}

struct Engine {
    const yko_snapshot* s;
    int D;
    uint32_t mode;
    std::vector<int64_t> avail;          // [n][D] working copy
    std::vector<int32_t> rank;           // node -> string rank
    std::vector<double> score;           // node -> current score
    std::set<NodeRef, NodeLess> order;   // the btree of SURVEY A.3

    struct Queue {
        int parent = -1;
        std::vector<int> children;
        std::vector<int> apps;
        std::vector<int64_t> alloc, pending;
        int64_t pending_asks = 0;
        int prio = INT32_MIN;     // cached current priority (the core keeps it up to date incrementally, too)
        bool prio_ok = false;
    };
    std::vector<Queue> queues;
    bool uniform_prio = false;    // every ask has the same priority and no queue shifts / fences: priorities cannot matter
    struct App {
        std::vector<int> asks;   // sorted (priority desc, create asc, index asc)
        int64_t pending_asks = 0;
        size_t head = 0;          // first ask not yet allocated (asks are in priority order)
        std::vector<int64_t> alloc;
        std::vector<int> limits;  // user-limit entries that apply: the app's user, a queue on the app's chain
    };
    std::vector<int64_t> ualloc;  // [l][D] what each user-limit entry's user holds below its queue

    // the application's user headroom folded into the queue headroom [EXT ugm Headroom]: hr = min(hr, max - held)
    void user_headroom(int p, int64_t* hr) {
        for (int l : apps[(size_t)p].limits)
            for (int k = 0; k < D; ++k) {
                const int64_t mx = s->ul_max[(size_t)l * D + k];
                if (mx == UNSET) continue;
                const int64_t own = clamp0(mx - ualloc[(size_t)l * D + k]);
                hr[k] = (hr[k] == UNSET) ? own : std::min(hr[k], own);
            }
    }
    std::vector<App> apps;
    std::vector<uint8_t> state;
    std::vector<uint8_t> done;   // allocated, or known-unplaceable (shortcut)
    yko_stats st{};

    const int64_t* total(int n) const { return s->node_total + (size_t)n * D; }
    int64_t* av(int n) { return avail.data() + (size_t)n * D; }
    const int64_t* req(int a) const { return s->ask_req + (size_t)a * D; }

    // ---- shim side: predicate_manager.go podFitsNode for the bitmaskable plugin set ----
    int shim_predicates(int a, int n) {
        ++st.evaluations;
        // Filter order: NodeUnschedulable, NodeName, TaintToleration, NodeAffinity, (NodePorts n/a),
        // NodeResourcesFit (predicate_manager.go:339-351)
        if (s->ask_node[a] >= 0 && s->ask_node[a] != n) return YKO_FAIL_NODENAME;
        if (s->node_taint[n] & ~s->ask_tol[a]) return YKO_FAIL_TAINT;
        if ((s->node_label[n] & s->ask_need[a]) != s->ask_need[a]) return YKO_FAIL_AFFINITY;
        if (s->node_label[n] & s->ask_deny[a]) return YKO_FAIL_AFFINITY;
        // NodeResourcesFit on the shim's NodeInfo: allocatable - requested is the same column as
        // the core's available in this model (DESIGN.md "one availability column")
        if (!fit_in(D, av(n), req(a))) return YKO_FAIL_RESOURCES;
        return 0;
    }

    // Predicates(Allocate = false): the reservation phase runs the same plugins without NodeResourcesFit ("during reservation,
    // node resources are not enough", predicate_manager.go:353-368) and the core does not ask for available resources either
    int evaluate_reserve(int a, int n) {
        if (!(s->node_flags[n] & YKO_NODE_SCHEDULABLE)) return YKO_FAIL_NODE_NOT_SCHEDULABLE;
        if (!fit_in(D, total(n), req(a))) return YKO_FAIL_TOTAL;
        if (!strictly_gt_zero(D, req(a))) return YKO_FAIL_REQUEST_NOT_POSITIVE;
        if (s->ask_node[a] >= 0 && s->ask_node[a] != n) return YKO_FAIL_NODENAME;
        if (s->node_taint[n] & ~s->ask_tol[a]) return YKO_FAIL_TAINT;
        if ((s->node_label[n] & s->ask_need[a]) != s->ask_need[a]) return YKO_FAIL_AFFINITY;
        if (s->node_label[n] & s->ask_deny[a]) return YKO_FAIL_AFFINITY;
        return 0;
    }

    int evaluate(int a, int n) {  // core tryNodes filter + tryNode + shim predicates
        if (!(s->node_flags[n] & YKO_NODE_SCHEDULABLE)) return YKO_FAIL_NODE_NOT_SCHEDULABLE;
        if (!fit_in(D, total(n), req(a))) return YKO_FAIL_TOTAL;
        if (!strictly_gt_zero(D, req(a))) return YKO_FAIL_REQUEST_NOT_POSITIVE;
        if (!fit_in(D, av(n), req(a))) return YKO_FAIL_AVAILABLE;
        return shim_predicates(a, n);
    }

    void rekey(int n) {
        double ns = node_score(D, s->policy, s->weights, total(n), av(n));
        if (ns != score[(size_t)n]) {
            order.erase(NodeRef{score[(size_t)n], rank[(size_t)n], n});
            score[(size_t)n] = ns;
            order.insert(NodeRef{ns, rank[(size_t)n], n});
        }
    }

    int try_nodes(int a) {
        for (const NodeRef& nr : order) {
            int n = nr.node;
            ++st.node_visits;
            if (s->node_flags[n] & YKO_NODE_RESERVED) continue;
            if (evaluate(a, n) == 0) return n;
        }
        return -1;
    }

    void headroom(int q, int64_t* hr) {   // hr[k] = UNSET if unlimited
        if (queues[(size_t)q].parent >= 0) headroom(queues[(size_t)q].parent, hr);
        else for (int k = 0; k < D; ++k) hr[k] = UNSET;
        const int64_t* mx = s->q_max + (size_t)q * D;
        for (int k = 0; k < D; ++k) {
            if (mx[k] == UNSET) continue;
            int64_t own = mx[k] - queues[(size_t)q].alloc[(size_t)k];
            // stored clamped at 0: UNSET is -1, and FitInMaxUndef clamps negatives to 0 anyway
            own = clamp0(own);
            hr[k] = (hr[k] == UNSET) ? own : std::min(hr[k], own);
        }
    }
    bool fit_in_max_undef(const int64_t* hr, const int64_t* r) const {
        for (int k = 0; k < D; ++k) {
            if (hr[k] == UNSET) continue;
            if (r[k] > hr[k]) return false;
        }
        return true;
    }

    void commit(int a, int n) {
        int64_t* v = av(n);
        const int64_t* r = req(a);
        for (int k = 0; k < D; ++k) v[k] -= r[k];
        rekey(n);
        int p = s->ask_app[a];
        App& ap = apps[(size_t)p];
        ap.pending_asks--;
        for (int k = 0; k < D; ++k) ap.alloc[(size_t)k] += r[k];
        for (int l : ap.limits) for (int k = 0; k < D; ++k) ualloc[(size_t)l * D + k] += r[k];
        for (int q = s->app_queue[p]; q >= 0; q = queues[(size_t)q].parent) {
            Queue& Q = queues[(size_t)q];
            Q.pending_asks--;
            Q.prio_ok = false;
            for (int k = 0; k < D; ++k) { Q.alloc[(size_t)k] += r[k]; Q.pending[(size_t)k] -= r[k]; }
        }
        state[(size_t)a] = YKO_ST_ALLOCATED;
        done[(size_t)a] = 1;
        ++st.allocations;
    }

    void uncommit(int a, int n) {   // exact inverse of commit (all-or-nothing gangs)
        int64_t* v = av(n);
        const int64_t* r = req(a);
        for (int k = 0; k < D; ++k) v[k] += r[k];
        rekey(n);
        int p = s->ask_app[a];
        App& ap = apps[(size_t)p];
        ap.pending_asks++;
        for (int k = 0; k < D; ++k) ap.alloc[(size_t)k] -= r[k];
        for (int l : ap.limits) for (int k = 0; k < D; ++k) ualloc[(size_t)l * D + k] -= r[k];
        for (int q = s->app_queue[p]; q >= 0; q = queues[(size_t)q].parent) {
            Queue& Q = queues[(size_t)q];
            Q.pending_asks++;
            Q.prio_ok = false;
            for (int k = 0; k < D; ++k) { Q.alloc[(size_t)k] -= r[k]; Q.pending[(size_t)k] += r[k]; }
        }
        state[(size_t)a] = YKO_ST_PENDING;
        done[(size_t)a] = 0;
        --st.allocations;
    }

    int gang_of(int a) const { return s->ask_gang ? s->ask_gang[a] : -1; }

    // All-or-nothing placement of the gang that ask `first` belongs to (DESIGN.md "gangs", SURVEY A.7):
    // members are placed one after the other in the application's ask order, each exactly like an ordinary
    // ask (headroom re-read after every member, ordered node walk, commit + re-score); if any member cannot
    // be placed every earlier member is rolled back and the whole gang is marked with that member's cause.
    bool stop = false;
    bool try_gang(int p, int first, std::vector<std::pair<int, int>>& out, int room) {
        const int g = gang_of(first);
        App& ap = apps[(size_t)p];
        std::vector<int> members;
        for (size_t i = ap.head; i < ap.asks.size(); ++i) {
            int a = ap.asks[i];
            if (gang_of(a) == g && state[(size_t)a] != YKO_ST_ALLOCATED && !done[(size_t)a]) members.push_back(a);
        }
        std::vector<std::pair<int, int>> placed;
        uint8_t cause = 0;
        // queue-side checks of every member first (headroom shrinking as if the earlier members were placed) ...
        {
            int64_t hr[YKO_MAX_D];
            headroom(s->app_queue[p], hr);
            user_headroom(p, hr);
            for (int a : members) {
                if (s->ask_flags[a] & YKO_ASK_SLOWPATH) { cause = YKO_ST_SLOWPATH; break; }
                if (!fit_in_max_undef(hr, req(a))) { cause = YKO_ST_SKIPPED; break; }
                if (!strictly_gt_zero(D, req(a))) { cause = YKO_ST_INVALID; break; }
                for (int k = 0; k < D; ++k) if (hr[k] != UNSET) hr[k] -= req(a)[k];
            }
        }
        // a gang that passed them but has more members than max_bindings leaves room for ends the cycle (one that was
        // sunk above needs no room and does not)
        if (!cause && room >= 0 && (int)members.size() > room) { stop = true; return false; }
        // ... then the node walks, member by member
        for (int a : members) {
            if (cause) break;
            int n = try_nodes(a);
            if (n < 0) { cause = YKO_ST_NOFIT; break; }
            commit(a, n);
            placed.emplace_back(a, n);
        }
        if (cause) {
            for (auto it = placed.rbegin(); it != placed.rend(); ++it) uncommit(it->first, it->second);
            for (int a : members) { state[(size_t)a] = cause; done[(size_t)a] = 1; }
            return false;
        }
        out.insert(out.end(), placed.begin(), placed.end());
        return true;
    }

    int app_priority(int p) {   // max priority over pending asks = priority of the first pending one
        App& ap = apps[(size_t)p];
        while (ap.head < ap.asks.size() && state[(size_t)ap.asks[ap.head]] == YKO_ST_ALLOCATED) ++ap.head;
        return ap.head < ap.asks.size() ? s->ask_prio[ap.asks[ap.head]] : INT32_MIN;
    }

    // Queue.GetCurrentPriority with default offsets / policies [EXT]: leaf = max over its applications that still have
    // pending asks; parent = max over its children
    int queue_priority(int q) {
        Queue& Q = queues[(size_t)q];
        if (Q.prio_ok) return Q.prio;
        int best = INT32_MIN;
        if (Q.children.empty()) {
            for (int p : Q.apps) if (apps[(size_t)p].pending_asks > 0) best = std::max(best, app_priority(p));
        } else {
            for (int c : Q.children) if (queues[(size_t)c].pending_asks > 0) best = std::max(best, queue_priority(c));
        }
        // priorityValueByPolicy [EXT]: offset, plus what is pending below unless the queue is a fence; clamped to int32
        const int64_t off = s->q_prio_offset ? s->q_prio_offset[q] : 0;
        const bool fence = s->q_prio_fence && s->q_prio_fence[q];
        const int64_t v = off + (fence ? 0 : (int64_t)best);
        Q.prio = (int)std::min<int64_t>(INT32_MAX, std::max<int64_t>(INT32_MIN, v));
        Q.prio_ok = true;
        return Q.prio;
    }

    // appends the pass's allocation(s) to out (one ask, or a whole gang); returns true if anything was allocated
    bool try_app(int p, const int64_t* hr_queue, std::vector<std::pair<int, int>>& out, int room) {
        bool retry = (mode & YKO_MODE_RETRY_FAILED) != 0;
        App& ap = apps[(size_t)p];
        int64_t hr[YKO_MAX_D];
        for (int k = 0; k < D; ++k) hr[k] = hr_queue[k];
        user_headroom(p, hr);
        for (size_t i = ap.head; i < ap.asks.size(); ++i) {
            int a = ap.asks[i];
            if (state[(size_t)a] == YKO_ST_ALLOCATED) continue;
            if (done[(size_t)a] && !retry) continue;
            if (gang_of(a) >= 0) {   // a gang member: the gang-wide checks decide for every member (all or nothing)
                if (try_gang(p, a, out, room)) return true;
                if (stop) return false;   // the gang does not fit in max_bindings: end of the cycle
                continue;
            }
            if (s->ask_flags[a] & YKO_ASK_SLOWPATH) { state[(size_t)a] = YKO_ST_SLOWPATH; done[(size_t)a] = 1; continue; }
            if (!fit_in_max_undef(hr, req(a))) { state[(size_t)a] = YKO_ST_SKIPPED; done[(size_t)a] = 1; continue; }
            if (!strictly_gt_zero(D, req(a))) { state[(size_t)a] = YKO_ST_INVALID; done[(size_t)a] = 1; continue; }
            int n = try_nodes(a);
            if (n >= 0) { commit(a, n); out.emplace_back(a, n); return true; }
            state[(size_t)a] = YKO_ST_NOFIT;
            done[(size_t)a] = 1;
        }
        return false;
    }

    bool try_queue(int q, std::vector<std::pair<int, int>>& out, int room) {
        Queue& Q = queues[(size_t)q];
        if (Q.children.empty()) {
            int64_t hr[YKO_MAX_D];
            headroom(q, hr);
            ++st.app_sorts;
            std::vector<int> sorted;
            for (int p : Q.apps) if (apps[(size_t)p].pending_asks > 0) sorted.push_back(p);
            if (s->q_sort[q] == YKO_SORT_FAIR) {
                // fair: max pending priority first (application.sort.priority is enabled by default), then ascending
                // dominant share of the application's allocation against the queue's guaranteed resource
                const int64_t* base = s->q_guaranteed + (size_t)q * D;
                std::vector<int> prio((size_t)s->n_apps, 0);
                for (int p : sorted) prio[(size_t)p] = app_priority(p);
                std::stable_sort(sorted.begin(), sorted.end(), [&](int l, int r) {
                    if (prio[(size_t)l] != prio[(size_t)r]) return prio[(size_t)l] > prio[(size_t)r];
                    int c = compare_shares(get_shares(D, apps[(size_t)l].alloc.data(), base),
                                           get_shares(D, apps[(size_t)r].alloc.data(), base));
                    if (c != 0) return c < 0;
                    if (s->app_submit[l] != s->app_submit[r]) return s->app_submit[l] < s->app_submit[r];
                    return l < r;
                });
            } else {
                std::vector<int> prio((size_t)s->n_apps, 0);
                for (int p : sorted) prio[(size_t)p] = app_priority(p);
                std::stable_sort(sorted.begin(), sorted.end(), [&](int l, int r) {
                    if (prio[(size_t)l] != prio[(size_t)r]) return prio[(size_t)l] > prio[(size_t)r];
                    if (s->app_submit[l] != s->app_submit[r]) return s->app_submit[l] < s->app_submit[r];
                    return l < r;
                });
            }
            for (int p : sorted) {
                if (try_app(p, hr, out, room)) return true;
                if (stop) return false;
            }
            return false;
        }
        ++st.queue_sorts;
        std::vector<int> sorted;
        for (int c : Q.children) if (queues[(size_t)c].pending_asks > 0) sorted.push_back(c);
        // sortQueuesByPriorityAndFairness [EXT yunikorn-core objects/sorters.go; priority sorting is on by default]: the
        // queue's current priority (highest priority among the asks still pending below it) first, then the shares.
        // Behaviour pinned by test/e2e/priority_scheduling/priority_scheduling_test.go:70-133.
        auto child_less = [&](int l, int r) {
            if (!uniform_prio) {
                const int pl = queue_priority(l), pr = queue_priority(r);
                if (pl != pr) return pl > pr;
            }
            int c = yko_comp_usage_ratio_separately(D, queues[(size_t)l].alloc.data(), s->q_guaranteed + (size_t)l * D,
                                                    queues[(size_t)r].alloc.data(), s->q_guaranteed + (size_t)r * D);
            if (c != 0) return c < 0;
            // equal shares: larger pending first (StrictlyGreaterThan(lPending - rPending, 0))
            int64_t diff[YKO_MAX_D];
            for (int k = 0; k < D; ++k) diff[k] = queues[(size_t)l].pending[(size_t)k] - queues[(size_t)r].pending[(size_t)k];
            if (strictly_gt_zero(D, diff)) return true;
            for (int k = 0; k < D; ++k) diff[k] = -diff[k];
            if (strictly_gt_zero(D, diff)) return false;
            return l < r;
        };
        // stable insertion sort from index order: what Go's sort.SliceStable does for n <= 20 [EXT]; written out so
        // that the engine's orderer can use the very same algorithm (the tie-break on pending is only a partial order)
        for (size_t a = 1; a < sorted.size(); ++a)
            for (size_t b = a; b > 0 && child_less(sorted[b], sorted[b - 1]); --b) std::swap(sorted[b], sorted[b - 1]);
        for (int c : sorted) {
            if (try_queue(c, out, room)) return true;
            if (stop) return false;
        }
        return false;
    }
};

}  // namespace

extern "C" {

double yko_node_score(int32_t D, int32_t policy, const double* weights, const int64_t* total, const int64_t* avail) {
    return node_score(D, policy, weights, total, avail);
}

int yko_comp_usage_ratio_separately(int32_t D, const int64_t* lalloc, const int64_t* lguar,
                                    const int64_t* ralloc, const int64_t* rguar) {
    return compare_shares(get_shares(D, lalloc, lguar), get_shares(D, ralloc, rguar));
}

static int check(const yko_snapshot* s) {
    if (!s || s->D < 1 || s->D > YKO_MAX_D) return -1;
    if (s->n_nodes < 0 || s->n_asks < 0 || s->n_apps < 0 || s->n_queues < 1) return -2;
    if (s->policy != YKO_POLICY_FAIR && s->policy != YKO_POLICY_BINPACKING) return -3;
    for (int q = 0; q < s->n_queues; ++q) {
        if (q == 0 ? s->q_parent[q] != -1 : (s->q_parent[q] < 0 || s->q_parent[q] >= q)) return -4;
    }
    for (int p = 0; p < s->n_apps; ++p)
        if (s->app_queue[p] < 0 || s->app_queue[p] >= s->n_queues) return -5;
    for (int a = 0; a < s->n_asks; ++a) {
        if (s->ask_app[a] < 0 || s->ask_app[a] >= s->n_apps) return -6;
        if (s->ask_node[a] < -1 || s->ask_node[a] >= s->n_nodes) return -7;
    }
    return 0;
}

int yko_predicate(const yko_snapshot* s, int32_t ask, int32_t node) {
    if (!s || ask < 0 || ask >= s->n_asks || node < 0 || node >= s->n_nodes) return -1;
    Engine e;
    e.s = s; e.D = s->D; e.mode = 0;
    e.avail.assign(s->node_avail, s->node_avail + (size_t)s->n_nodes * s->D);
    return e.evaluate(ask, node);
}

int yko_predicate_reserve(const yko_snapshot* s, int32_t ask, int32_t node) {
    if (!s || ask < 0 || ask >= s->n_asks || node < 0 || node >= s->n_nodes) return -1;
    Engine e;
    e.s = s; e.D = s->D; e.mode = 0;
    e.avail.assign(s->node_avail, s->node_avail + (size_t)s->n_nodes * s->D);
    return e.evaluate_reserve(ask, node);
}

int yko_preemption_index(const yko_snapshot* s, int32_t ask, int32_t node, int32_t n_victims,
                         const int64_t* victim_req, int32_t start) {
    if (!s || ask < 0 || ask >= s->n_asks || node < 0 || node >= s->n_nodes) return -2;
    const int D = s->D;
    // clone the node, then remove victims one at a time (predicate_manager.go:153-168): the loop body only runs
    // for i >= start, so with no victims (or start past the end) the answer is -1 even if the pod would fit
    std::vector<int64_t> avail(s->node_avail + (size_t)node * D, s->node_avail + (size_t)(node + 1) * D);
    for (int i = 0; i < n_victims; ++i) {
        for (int k = 0; k < D; ++k) avail[(size_t)k] += victim_req[(size_t)i * D + k];
        if (i < start) continue;
        yko_snapshot t = *s;
        std::vector<int64_t> all(s->node_avail, s->node_avail + (size_t)s->n_nodes * D);
        std::copy(avail.begin(), avail.end(), all.begin() + (size_t)node * D);
        t.node_avail = all.data();
        if (yko_predicate(&t, ask, node) == 0) return i;
    }
    return -1;
}

int yko_run(const yko_snapshot* s, uint32_t mode, int32_t max_bindings, int32_t* out_ask, int32_t* out_node,
            int32_t* n_out, uint8_t* ask_state, int64_t* node_avail_out, yko_stats* stats) {
    int rc = check(s);
    if (rc) return rc;
    Engine e;
    e.s = s; e.D = s->D; e.mode = mode;
    const int D = s->D, N = s->n_nodes;
    e.avail.assign(s->node_avail, s->node_avail + (size_t)N * D);

    // NodeID string ranks (Go string compare = bytewise unsigned)
    std::vector<int32_t> idx((size_t)N);
    for (int i = 0; i < N; ++i) idx[(size_t)i] = i;
    std::sort(idx.begin(), idx.end(), [&](int a, int b) { return strcmp(s->node_id[a], s->node_id[b]) < 0; });
    e.rank.assign((size_t)N, 0);
    for (int r = 0; r < N; ++r) {
        if (r > 0 && strcmp(s->node_id[idx[(size_t)r - 1]], s->node_id[idx[(size_t)r]]) == 0) return -8;  // duplicate NodeID
        e.rank[(size_t)idx[(size_t)r]] = r;
    }
    e.score.assign((size_t)N, 0.0);
    for (int n = 0; n < N; ++n) {
        double sc = node_score(D, s->policy, s->weights, e.total(n), e.av(n));
        if (std::isnan(sc)) return -9;
        e.score[(size_t)n] = sc;
        e.order.insert(NodeRef{sc, e.rank[(size_t)n], n});
    }

    e.uniform_prio = true;
    for (int a = 1; a < s->n_asks; ++a) if (s->ask_prio[a] != s->ask_prio[0]) { e.uniform_prio = false; break; }
    for (int q = 0; q < s->n_queues && e.uniform_prio; ++q)
        if ((s->q_prio_offset && s->q_prio_offset[q] != 0) || (s->q_prio_fence && s->q_prio_fence[q])) e.uniform_prio = false;
    e.queues.resize((size_t)s->n_queues);
    for (int q = 0; q < s->n_queues; ++q) {
        auto& Q = e.queues[(size_t)q];
        Q.parent = s->q_parent[q];
        if (Q.parent >= 0) e.queues[(size_t)Q.parent].children.push_back(q);
        Q.alloc.assign(s->q_alloc + (size_t)q * D, s->q_alloc + (size_t)(q + 1) * D);
        Q.pending.assign((size_t)D, 0);
    }
    e.apps.resize((size_t)s->n_apps);
    for (int p = 0; p < s->n_apps; ++p) {
        if (!e.queues[(size_t)s->app_queue[p]].children.empty()) return -10;  // apps live in leaves
        e.queues[(size_t)s->app_queue[p]].apps.push_back(p);
        if (s->app_alloc) e.apps[(size_t)p].alloc.assign(s->app_alloc + (size_t)p * D, s->app_alloc + (size_t)(p + 1) * D);
        else e.apps[(size_t)p].alloc.assign((size_t)D, 0);
        if (s->app_user && s->n_limits > 0 && s->app_user[p] >= 0)
            for (int l = 0; l < s->n_limits; ++l) {
                if (s->ul_user[l] != s->app_user[p]) continue;
                for (int q = s->app_queue[p]; q >= 0; q = e.queues[(size_t)q].parent)
                    if (q == s->ul_queue[l]) { e.apps[(size_t)p].limits.push_back(l); break; }
            }
    }
    e.ualloc.assign((size_t)std::max(s->n_limits, 0) * D, 0);
    if (s->ul_alloc) e.ualloc.assign(s->ul_alloc, s->ul_alloc + (size_t)s->n_limits * D);
    e.state.assign((size_t)s->n_asks, YKO_ST_PENDING);
    e.done.assign((size_t)s->n_asks, 0);
    for (int a = 0; a < s->n_asks; ++a) {
        int p = s->ask_app[a];
        e.apps[(size_t)p].asks.push_back(a);
        e.apps[(size_t)p].pending_asks++;
        for (int q = s->app_queue[p]; q >= 0; q = e.queues[(size_t)q].parent) {
            e.queues[(size_t)q].pending_asks++;
            for (int k = 0; k < D; ++k) e.queues[(size_t)q].pending[(size_t)k] += s->ask_req[(size_t)a * D + k];
        }
    }
    for (auto& ap : e.apps)
        std::stable_sort(ap.asks.begin(), ap.asks.end(), [&](int l, int r) {
            if (s->ask_prio[l] != s->ask_prio[r]) return s->ask_prio[l] > s->ask_prio[r];
            if (s->ask_create[l] != s->ask_create[r]) return s->ask_create[l] < s->ask_create[r];
            return l < r;
        });

    int32_t n = 0;
    std::vector<std::pair<int, int>> got;
    while (max_bindings < 0 || n < max_bindings) {
        ++e.st.passes;
        got.clear();
        if (!e.try_queue(0, got, max_bindings < 0 ? -1 : max_bindings - n)) break;
        for (auto& b : got) { out_ask[n] = b.first; out_node[n] = b.second; ++n; }
    }
    *n_out = n;
    if (ask_state) memcpy(ask_state, e.state.data(), (size_t)s->n_asks);
    if (node_avail_out) memcpy(node_avail_out, e.avail.data(), sizeof(int64_t) * (size_t)N * D);
    if (stats) *stats = e.st;
    return 0;
}

}  // extern "C"
