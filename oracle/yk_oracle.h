/*
 * yk_oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement of the YuniKorn pod->node allocation cycle (the path named by
 * BASELINE.json north_star; SURVEY.md section 8).  Nothing in the product
 * (yunikorn_k8shim_b200/, include/ykgpu.h) may include, link or call this.
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
 * legs load it, and only as the checker / the timed CPU arm.
 *
 * PARITY STATUS: the per-(ask,node) predicate semantics are pinned against the
 * reference's own known-answer tables (tests/golden/ (JSON), transcribed from
 * pkg/plugin/predicates/predicate_manager_test.go and
 * pkg/common/resource_test.go).  The node scoring / ordering / queue ordering
 * steps live in third-party modules that are NOT in the reference repository
 * (github.com/apache/yunikorn-core v0.0.0-20260325023719-8ae738dc14e9,
 * go.mod:24) and no test in the reference pins a pod->node map, so for those
 * steps this oracle is "parity unpinned": it restates the published algorithm
 * (SURVEY.md Appendix A) and is cross-checked only by an independent second
 * restatement (oracle/py_oracle.py).
 */
#ifndef YK_ORACLE_H
#define YK_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YKO_MAX_D 8

/* node flags */
#define YKO_NODE_SCHEDULABLE 1u
#define YKO_NODE_RESERVED    2u   /* hidden from the normal iterator (SURVEY A.2) */
/* ask flags */
#define YKO_ASK_SLOWPATH     1u   /* needs a non-bitmask predicate: not handled by the fast path */
/* queue app-sort policy (leaf) */
#define YKO_SORT_FIFO 0
#define YKO_SORT_FAIR 1
/* node sort policy */
#define YKO_POLICY_FAIR       0
#define YKO_POLICY_BINPACKING 1
/* per-ask result state */
#define YKO_ST_PENDING   0  /* never reached (max_bindings hit) */
#define YKO_ST_ALLOCATED 1
#define YKO_ST_NOFIT     2  /* tried, no node passed (shim would get SchedulingState FAILED) */
#define YKO_ST_SKIPPED   3  /* queue headroom exceeded (SchedulingState SKIPPED) */
#define YKO_ST_SLOWPATH  4  /* flagged slow-path, left to the Go PredicateManager */
#define YKO_ST_INVALID   5  /* request not strictly greater than zero */

typedef struct {
    int32_t D;                   /* resource dimensions, <= YKO_MAX_D */
    int32_t policy;              /* YKO_POLICY_* */
    const double* weights;       /* [D] node-sort resource weights */

    int32_t n_nodes;
    const int64_t* node_total;   /* [n][D] row-major */
    const int64_t* node_avail;   /* [n][D] */
    const uint64_t* node_taint;  /* [n] */
    const uint64_t* node_label;  /* [n] */
    const uint32_t* node_flags;  /* [n] */
    const char* const* node_id;  /* [n] NodeID strings (tie-break is bytewise string order) */

    int32_t n_queues;            /* queue 0 is root; q_parent[i] < i */
    const int32_t* q_parent;     /* [q], -1 for root */
    const int64_t* q_guaranteed; /* [q][D], -1 = not set */
    const int64_t* q_max;        /* [q][D], -1 = not set */
    const int64_t* q_alloc;      /* [q][D] allocated at cycle start (every level) */
    const uint8_t* q_sort;       /* [q] leaf application sort policy */

    int32_t n_apps;
    const int32_t* app_queue;    /* [p] leaf queue index */
    const int64_t* app_submit;   /* [p] submission time, unique per queue */

    int32_t n_asks;
    const int32_t* ask_app;      /* [a] */
    const int64_t* ask_req;      /* [a][D] */
    const uint64_t* ask_tol;     /* [a] tolerated taint bits */
    const uint64_t* ask_need;    /* [a] label bits that must all be set */
    const uint64_t* ask_deny;    /* [a] label bits that must all be clear */
    const int32_t* ask_prio;     /* [a] */
    const int64_t* ask_create;   /* [a] creation order key (unique within an app) */
    const int32_t* ask_node;     /* [a] required node index or -1 (pod.Spec.NodeName) */
    const uint32_t* ask_flags;   /* [a] */
    const int32_t* ask_gang;     /* [a] gang id or -1; may be NULL */
    /* queue priority properties (priority.offset, priority.policy = fence) [EXT yunikorn-core configs]; may be NULL = 0 */
    const int32_t* q_prio_offset;   /* [q] */
    const uint8_t* q_prio_fence;    /* [q] 1 = fence: the queue shows its parent only its offset */
    /* user / group resource limits (the core's queue `limits:` entries, [EXT yunikorn-core ugm]; the shim sends the
     * user with every application, pkg/cache/application.go:430): entry l = "user ul_user[l] may hold at most ul_max[l]
     * below queue ul_queue[l]" (summed over the user's applications in that queue's subtree).  The group / wildcard entry
     * that applies to a user is resolved by the caller.  All may be NULL / 0 = no limits. */
    const int32_t* app_user;        /* [p] user index or -1 */
    int32_t n_limits;
    const int32_t* ul_queue;        /* [l] */
    const int32_t* ul_user;         /* [l] */
    const int64_t* ul_max;          /* [l][D], -1 = not set */
    const int64_t* ul_alloc;        /* [l][D] held at cycle start; may be NULL = 0 */
    /* what each application holds from earlier cycles: a fair leaf orders its applications by these shares */
    const int64_t* app_alloc;       /* [p][D] held at cycle start; may be NULL = 0 */
} yko_snapshot;

typedef struct {
    int64_t passes;         /* schedule() passes executed */
    int64_t node_visits;    /* nodes stepped over by the ordered walk */
    int64_t evaluations;    /* (ask,node) predicate evaluations (PredicateManager calls) */
    int64_t allocations;
    int64_t app_sorts;      /* sortApplications invocations */
    int64_t queue_sorts;    /* sortQueues invocations */
} yko_stats;

/* mode bits for yko_run */
#define YKO_MODE_RETRY_FAILED 1u  /* literally re-try asks that already failed on every pass
                                     (what the reference does; result-identical, slower) */

/* Runs the cycle to exhaustion (or max_bindings). out_ask/out_node receive the
 * bindings in commit order; ask_state[a] one of YKO_ST_*; node_avail_out (may be
 * NULL) gets the final [n][D] available.  Returns 0, or <0 on malformed input. */
int yko_run(const yko_snapshot* s, uint32_t mode, int32_t max_bindings,
            int32_t* out_ask, int32_t* out_node, int32_t* n_out,
            uint8_t* ask_state, int64_t* node_avail_out, yko_stats* stats);

/* One (ask,node) evaluation against the snapshot as given, in the reference's
 * plugin order.  Returns 0 if the pod fits, else a YKO_FAIL_* code naming the
 * first failing step (the reference returns that plugin's name, context.go:698-701). */
#define YKO_FAIL_NODE_NOT_SCHEDULABLE 1  /* core: node.IsSchedulable() */
#define YKO_FAIL_TOTAL                2  /* core: node.FitInNode(total) */
#define YKO_FAIL_REQUEST_NOT_POSITIVE 3  /* core: preAllocateCheck */
#define YKO_FAIL_AVAILABLE            4  /* core: preAllocateCheck available.FitIn */
#define YKO_FAIL_NODENAME             5  /* k8s NodeName */
#define YKO_FAIL_TAINT                6  /* k8s NodeUnschedulable / TaintToleration */
#define YKO_FAIL_AFFINITY             7  /* k8s NodeAffinity (nodeSelector + required terms) */
#define YKO_FAIL_RESOURCES            8  /* k8s NodeResourcesFit */
int yko_predicate(const yko_snapshot* s, int32_t ask, int32_t node);
/* the same for the reservation phase, Predicates(Allocate = false): no NodeResourcesFit, no available check
 * (pkg/plugin/predicates/predicate_manager.go:130-135,353-368) */
int yko_predicate_reserve(const yko_snapshot* s, int32_t ask, int32_t node);

/* Preemption victim search for one (ask,node): pkg/plugin/predicates/predicate_manager.go:137-175.
 * victim_req is [n][D] (what removing each victim gives back).  Returns the first index >= start that fits, or -1. */
int yko_preemption_index(const yko_snapshot* s, int32_t ask, int32_t node, int32_t n_victims,
                         const int64_t* victim_req, int32_t start);

/* float64 node score exactly as SURVEY A.3 (exposed for known-answer tests) */
double yko_node_score(int32_t D, int32_t policy, const double* weights,
                      const int64_t* total, const int64_t* avail);

/* DRF comparison of two (allocated, guaranteed) pairs: -1, 0, 1 (exposed for the
 * resource_fairness known-answer vector) */
int yko_comp_usage_ratio_separately(int32_t D, const int64_t* lalloc, const int64_t* lguar,
                                    const int64_t* ralloc, const int64_t* rguar);

#ifdef __cplusplus
}
#endif
#endif
