/*
 * ykgpu.h -- C ABI of the H100 scheduling-cycle engine (libykgpu.so).
 *
 * This is the drop-in boundary for YuniKorn's pod->node allocation hot path.  A thin Go type
 * implementing api.SchedulerAPI (method set: pkg/common/test/schedulerapi_mock.go:88-146)
 * binds these entry points through cgo and drives api.ResourceManagerCallback
 * (pkg/cache/scheduler_callback.go:42-43) with what yk_cycle returns; pkg/shim,
 * pkg/plugin and cache.Context stay unchanged.  INTEGRATION.md shows the cgo side.
 *
 * What each entry point replaces in the reference:
 *   yk_nodes_upsert / yk_nodes_remove   SchedulerAPI.UpdateNode(*si.NodeRequest) -- call sites
 *                                       pkg/cache/context.go:256,1610,1630,1635,1656; node vector
 *                                       = common.GetNodeResource, pkg/common/resource.go:188-195
 *   yk_queues_set                       the queues.yaml half of RegisterResourceManager /
 *                                       UpdateConfiguration (pkg/shim/scheduler.go:147-167)
 *   yk_node_sort_set                    the partition's nodesortpolicy (type, resourceweights) of the same configuration
 *   yk_apps_upsert / yk_apps_remove     SchedulerAPI.UpdateApplication (pkg/cache/application.go:423)
 *   yk_asks_upsert / yk_asks_remove     SchedulerAPI.UpdateAllocation(*si.AllocationRequest) with
 *                                       Allocations without NodeID = asks (pkg/cache/task.go:311-334,
 *                                       pkg/common/si_helper.go:75-115); ask vector = common.GetPodResource,
 *                                       pkg/common/resource.go:56-109
 *   yk_release                          AllocationRequest.Releases (pkg/cache/task.go:518, context.go:459)
 *   yk_asks_resize                      UpdateAllocation re-sending a known AllocationKey with a new resource vector: an
 *                                       in-place pod resize (Task.SetTaskPod, pkg/cache/task.go:633-647)
 *   yk_cycle                            yunikorn-core partition.tryAllocate loop [EXT, SURVEY 3.3] INCLUDING
 *                                       the per-(ask,node) callback ResourceManagerCallback.Predicates
 *                                       (pkg/cache/scheduler_callback.go:196-198 -> pkg/cache/context.go:683-703
 *                                       -> pkg/plugin/predicates/predicate_manager.go:130-283) for the
 *                                       bitmaskable plugin set, and the node sorter/scorer.  Its output is the
 *                                       payload of ResourceManagerCallback.UpdateAllocation(New: ...)
 *                                       (pkg/cache/scheduler_callback.go:49-91).
 *   yk_ask_states                       UpdateContainerSchedulingState FAILED / SKIPPED
 *                                       (pkg/cache/scheduler_callback.go:218-222, context.go:1232-1272)
 *   yk_evaluate                         one ResourceManagerCallback.Predicates(ask,node) answer, for the
 *                                       slow-path bridge and for known-answer tests
 *   yk_filter_nodes                     the same answers for every node and a list of asks at once: the candidates a
 *                                       slow-path pod is walked through Predicates in, and the per-cause counts of the
 *                                       FAILED reason of an unplaceable pod
 *   yk_preemption_search                ResourceManagerCallback.PreemptionPredicates for one (ask, node, victims) query
 *   yk_preemption_nodes                 the same search on every node for a list of asks, from the allocations the
 *                                       engine made: the search half of a preemptor (its policy stays with the caller)
 *   yk_preemption_plan                  the core's preemption for queues below their guarantee: victims, node and marks
 *   yk_preemption_required_node         the core's preemption for asks with a required node (DaemonSet pods): victims on
 *                                       that node and marks, for a whole rollout in one device pass
 *
 * Conventions: every call returns YK_OK (0) or a negative yk_status; no exceptions or aborts cross the
 * boundary.  Inputs are caller-owned host memory, fully consumed before return (cgo: no Go pointer is
 * retained).  Outputs are caller-allocated.  All resource matrices are COLUMN-MAJOR: element (k, i) of a
 * [D][count] matrix is at m[k*count + i].  Strings never cross: nodes, asks, apps and queues are dense
 * uint32 indices below the capacities given at yk_create (the Go side already owns the name->index maps,
 * pkg/cache/external/scheduler_cache.go:53-54).  One writer at a time per engine (internal mutex).
 * A missing CUDA device or kernel image is an error (YK_ERR_CUDA), never a CPU fallback.
 */
#ifndef YKGPU_H
#define YKGPU_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YK_ABI_VERSION 3
#define YK_MAX_D 8
#define YK_NONE 0xFFFFFFFFu          /* "no node" / "no gang" index */

typedef enum {
    YK_OK = 0,
    YK_ERR_ARG = -1,        /* null pointer, index out of capacity, bad enum */
    YK_ERR_CUDA = -2,       /* no device, no sm_90a image, launch or copy failed */
    YK_ERR_NOMEM = -3,
    YK_ERR_STATE = -4,      /* e.g. release of an ask that holds no allocation */
    YK_ERR_RANGE = -5,      /* NaN node score (zero total on a weighted resource with non-zero available) */
    YK_ERR_COMM = -6        /* multi-GPU exchange failed */
} yk_status;

/* node sort policy (core NodeSortingPolicy, SURVEY A.3 / A.8) */
#define YK_POLICY_FAIR 0u
#define YK_POLICY_BINPACKING 1u
/* leaf application sort policy */
#define YK_SORT_FIFO 0u
#define YK_SORT_FAIR 1u
/* node flags */
#define YK_NODE_SCHEDULABLE 1u   /* cleared by DRAIN_NODE / cordon (pkg/cache/context.go:247-257) */
#define YK_NODE_RESERVED 2u      /* hidden from the normal node iterator */
/* ask flags */
#define YK_ASK_SLOWPATH 1u       /* carries a predicate that does not reduce to the masks (ports, volumes,
                                    pod (anti-)affinity, topology spread): never bound by yk_cycle, returned
                                    in its slow-path list for the unchanged Go PredicateManager */
/* preemption policy of the pod (si.PreemptionPolicy, pkg/cache/task.go:233-258): read only by yk_preemption_plan, never by
   yk_cycle (they are not part of the sweep's row signature) */
#define YK_ASK_NO_PREEMPT_SELF 2u   /* not AllowPreemptSelf: taken as a victim only after every allocation without it */
#define YK_ASK_NO_PREEMPT_OTHER 4u  /* not AllowPreemptOther (preemptionPolicy: Never): never preempts */
#define YK_ASK_ORIGINATOR 8u        /* the pod that originated its application: taken as a victim after the others */
/* per-ask state reported by yk_ask_states */
#define YK_ST_PENDING 0u
#define YK_ST_ALLOCATED 1u
#define YK_ST_NOFIT 2u           /* -> UpdateContainerSchedulingState FAILED */
#define YK_ST_SKIPPED 3u         /* queue headroom; -> SchedulingState SKIPPED */
#define YK_ST_SLOWPATH 4u
#define YK_ST_INVALID 5u         /* request not strictly greater than zero */
#define YK_ST_ABSENT 255u

/* yk_evaluate answers: 0 = fits, else first failing step in the reference's order */
#define YK_FAIL_NODE_NOT_SCHEDULABLE 1
#define YK_FAIL_TOTAL 2
#define YK_FAIL_REQUEST_NOT_POSITIVE 3
#define YK_FAIL_AVAILABLE 4
#define YK_FAIL_NODENAME 5
#define YK_FAIL_TAINT 6
#define YK_FAIL_AFFINITY 7
#define YK_FAIL_RESOURCES 8
#define YK_FAIL_ABSENT 9         /* pod or node not in the cache (context.go:686-694) */

/* yk_config.flags */
#define YK_FLAG_NO_ROW_SHARING 1u   /* sweep one row per ask even when asks of a batch have identical predicate inputs
                                      (requests, tolerations, label masks, node name); default: one row per distinct set */
/* Where the ordered commit runs.  Default (neither flag): automatic -- a cycle whose order consists of long UNIFORM RUNS
   (>= 2048 consecutive asks with one request vector and one predicate signature: the replicas of a deployment, the executors of
   a job, the reference's own benchmark) and that is eligible (fair node sort, non-negative weights and weighted totals, unique
   NodeID ranks, every gang's members requesting one vector) is decided on the device by a grid-wide sort (csrc/yk_uniform.cuh);
   so is an eligible cycle of at least 10 000 pending asks without masks (no required / forbidden labels, no node name, every
   node taint tolerated, no gangs) in a placement-insensitive order, by rounds at the front of the node order
   (csrc/yk_rounds.cuh); every other cycle takes the sweep + host commit path.  The bindings are the same either way. */
#define YK_FLAG_HOST_COMMIT 2u      /* never commit on the device */
#define YK_FLAG_DEVICE_COMMIT 4u    /* commit on the device whenever the cycle is eligible, also where the order is not made of
                                      uniform runs (yk_lattice_kernel: exact, no bitmap read-back, no host work per ask, but
                                      measured slower than the host commit there) */
#define YK_FLAG_BINPACKING_DEVICE 8u /* also take eligible cycles under the binpacking node sort, in auto and device commit: every
                                      maximal uniform run is decided by one ordered capacity fill on the device (a node's key never
                                      rises under binpacking, so the front node fills to its capacity before the next one: one sort,
                                      one 64-bit scan, one search per ask, csrc/yk_uniform.h); gangs that may need a roll-back and
                                      stretches cut inside a gang go to the host commit.  auto prices a fill at its measured cost
                                      against the host commit's per-ask cost (DESIGN.md §6.4).  Unset: binpacking cycles always take
                                      the sweep + host commit path.  Same bindings either way. */

typedef struct yk_engine yk_engine;

typedef struct {
    uint32_t abi_version;        /* YK_ABI_VERSION */
    uint32_t D;                  /* resource dimensions 1..YK_MAX_D; by convention 0 vcore(milli) 1 memory 2 pods 3 ephemeral-storage */
    uint32_t policy;             /* YK_POLICY_*: the initial node sort policy (yk_node_sort_set replaces it) */
    uint32_t batch;              /* asks per sweep batch; 0 = default */
    double weights[YK_MAX_D];    /* initial node-sort resource weights (yk_node_sort_set replaces them); core default
                                    vcore=1, memory=1 */
    uint32_t max_nodes, max_asks, max_apps, max_queues;
    int32_t device;              /* CUDA ordinal, -1 = current device */
    uint32_t flags;              /* YK_FLAG_* (0 = defaults) */
    /* multi-GPU (one process per GPU): asks of every batch are split in `world` contiguous shards, this
       engine sweeps shard `rank`; the caller wires the exchange with yk_set_exchange.  world<=1: single GPU */
    uint32_t rank, world;
} yk_config;

typedef struct { uint32_t ask; uint32_t node; } yk_binding;

typedef struct {
    uint64_t cycles, batches, allocations, nofit, skipped;
    uint64_t evaluations;        /* (ask,node) pairs swept by the kernel */
    uint64_t sweep_launches, other_launches;   /* kernels launched by this library */
    uint64_t h2d_bytes, d2h_bytes;
    double sweep_ms, sort_ms, commit_ms, total_ms;   /* CUDA-event / wall accumulations */
    double last_sweep_ms;
    uint64_t last_sweep_pairs;
    /* host wall-clock split of yk_cycle: 0 table upload + initial device sort, 1 orderer begin_cycle,
       2 orderer fill/rewind, 3 waiting for device results, 4 ordered commit, 5 order merge + state push, 6 launch,
       7 orderer + launch time spent on the helper thread (overlapped with the commit) */
    double host_ms[8];
    /* commit counters: 0 bitmap words scanned, 1 re-scored candidates examined, 2 asks won by a re-scored node,
       3 re-keys of an already re-scored node */
    uint64_t dbg[4];
    /* with YK_PROFILE_COMMIT set: TSC cycles in the commit loop -- 0 clean scan, 1 re-scored walk, 2 choose + undo log
       + erase, 3 subtract + float64 re-score, 4 re-insert + bookkeeping, 5 asks counted */
    uint64_t prof[6];
    /* row sharing: asks that went through a sweep batch, and the rows (distinct predicate signatures) actually swept */
    uint64_t asks_swept, rows_swept;
    /* device-resident ordered commit (yk_lattice_kernel): launches, sub-runs (scan + lattice + chain + patch rounds), asks it
       decided, lattice elements evaluated, sorts, full-order scans (an ask with no candidate near the front), asks decided by
       the capacity bound alone, cycles handed over to the host commit (a gang that has to be rolled back), CUDA-event time */
    uint64_t lattice_launches, lattice_subruns, lattice_asks, lattice_elements, lattice_sorts, lattice_fullscans,
             lattice_quick, lattice_handoffs;
    double lattice_ms;
    uint64_t lattice_cycles;     /* cycles that started on the device commit */
    /* uniform runs of the device commit (consecutive asks with one request vector and one predicate signature, decided by a
       grid-wide sort instead of the sequential chain): runs, asks they decided, elements generated, deeper retries */
    uint64_t uniform_runs, uniform_asks, uniform_elements, uniform_retries;
    /* round commit of the device commit (mask-free stretches decided in rounds at the front of the node order): passes
       (rounds and single steps), asks it decided, single steps (the front node rejected the ask) */
    uint64_t round_passes, round_asks, round_single_steps;
    /* speculative round-commit launches (started on the device's own order of the cycle's asks before the host has set the
       cycle up): adopted (the host's first batch and plan were exactly that launch), discarded (stopped; nothing it wrote read) */
    uint64_t spec_adopted, spec_discarded;
} yk_stats_t;

int yk_create(const yk_config* cfg, yk_engine** out);
void yk_destroy(yk_engine* e);

/* nodes: total/avail are [D][n]; name_rank = rank of the NodeID in Go string (bytewise) order among all
 * nodes -- it must be order-preserving, not dense.  avail = total - allocated - occupied as the core
 * tracks it (SURVEY A.5). */
int yk_nodes_upsert(yk_engine* e, uint32_t n, const uint32_t* idx, const int64_t* total, const int64_t* avail,
                    const uint64_t* taint_bits, const uint64_t* label_bits, const uint32_t* name_rank,
                    const uint32_t* flags);
int yk_nodes_remove(yk_engine* e, uint32_t n, const uint32_t* idx);

/* queues: whole tree at once.  parent[0] = YK_NONE (root), parent[i] < i.  guaranteed/max/allocated are
 * [D][q] with -1 = not set (allocated: 0).  sort = leaf application sort policy. */
int yk_queues_set(yk_engine* e, uint32_t q, const uint32_t* parent, const int64_t* guaranteed,
                  const int64_t* max, const int64_t* allocated, const uint8_t* sort);

/* optional queue priority properties of the core's queue configuration [EXT yunikorn-core configs: properties
 * priority.offset, priority.policy]: a parent sorts its children by their current priority first (highest priority among the
 * asks pending below the child, plus the child's offset; a child with policy "fence" shows only its offset), then by share.
 * Both arrays are [q] in yk_queues_set order and may be NULL (= 0 / no fence); yk_queues_set resets them.  Behaviour
 * checked by the reference in test/e2e/priority_scheduling/priority_scheduling_test.go:70-251. */
int yk_queues_priority(yk_engine* e, uint32_t q, const int32_t* offset, const uint8_t* fence);

/* optional queue property preemption.policy of the core's queue configuration: fence[i] != 0 = "fence" (a preemptor below queue
 * i takes victims only inside i's subtree).  [q] in yk_queues_set order, NULL = no fence; yk_queues_set resets it.  Read only by
 * yk_preemption_plan. */
int yk_queues_preemption(yk_engine* e, uint32_t q, const uint8_t* fence);

/* applications live in LEAF queues (as in the core: placement into a parent queue is rejected there; here an application
 * whose queue has children is accepted but never scheduled -- the adapter must not produce one).
 * An application's allocations stay accounted to its index and its queue chain until each is released, even after
 * yk_apps_remove; a removed application's index must not come back while any ask of it is still allocated.  So
 * yk_apps_upsert returns YK_ERR_STATE and changes nothing when one of its entries
 *   - names an index that is not present while an allocated ask still belongs to it (release those first), or
 *   - moves a present application to another queue while an allocated ask belongs to it (its holdings would stay on
 *     the old queue chain).
 * An allocated ask counts as held whatever its request, zero included. */
int yk_apps_upsert(yk_engine* e, uint32_t n, const uint32_t* idx, const uint32_t* queue,
                   const int64_t* submit_time);
int yk_apps_remove(yk_engine* e, uint32_t n, const uint32_t* idx);

/* User / group resource limits: the core's queue `limits:` entries [EXT yunikorn-core ugm]; the shim sends the user and its
 * groups with every application (si.AddApplicationRequest.Ugi, pkg/cache/application.go:430).  yk_apps_user names the user
 * of each application (dense index, YK_NONE = none).  yk_user_limits_set replaces the whole table: entry l says "user
 * user[l] may hold at most max[.][l] ([D][n], -1 = not limited in that dimension) below queue queue[l]", summed over the
 * user's applications in that queue's subtree; an ask that exceeds what is left is SKIPPED for the cycle exactly like one
 * that exceeds the queue headroom.  The adapter resolves which entry applies to a user (its own, its group's, the
 * wildcard).  held[.][l] = what the user holds there now ([D][n], NULL = 0); the engine keeps it current afterwards
 * (cycle, yk_release).  maxapplications is not modelled (it gates application acceptance, not this path). */
int yk_apps_user(yk_engine* e, uint32_t n, const uint32_t* idx, const uint32_t* user);
int yk_user_limits_set(yk_engine* e, uint32_t n, const uint32_t* queue, const uint32_t* user, const int64_t* max,
                       const int64_t* held);

/* asks: req is [D][a].  create_seq is the total-order key within an application (ties pre-broken by the
 * caller: the reference's CreationTime is second-granular, pkg/common/si_helper.go:109).
 * required_node = YK_NONE or the node index pod.Spec.NodeName names.  gang = YK_NONE or a gang id
 * (all-or-nothing group).  Any of tolerated/required/forbidden/priority/required_node/flags/gang may be
 * NULL = all zero / YK_NONE. */
int yk_asks_upsert(yk_engine* e, uint32_t a, const uint32_t* idx, const int64_t* req,
                   const uint64_t* tolerated_bits, const uint64_t* required_bits, const uint64_t* forbidden_bits,
                   const int32_t* priority, const int64_t* create_seq, const uint32_t* app,
                   const uint32_t* required_node, const uint32_t* flags, const uint32_t* gang);
int yk_asks_remove(yk_engine* e, uint32_t a, const uint32_t* idx);

/* give the resources of allocated asks back to their nodes and queues, and forget the asks */
int yk_release(yk_engine* e, uint32_t n, const uint32_t* ask_idx);

/* Replace the request of present asks, pending or allocated: an in-place pod resize (KEP-1287).  The shim re-sends a task's
 * allocation with the same AllocationKey whenever common.GetPodResource of its pod changes (Task.SetTaskPod,
 * pkg/cache/task.go:633-647, from Context.updateYuniKornPod, context.go:341-349); req is the new vector, [D][n].
 *   Allocated ask (YK_ST_ALLOCATED), delta = new - old: its bound node's available goes down by delta (a node that is no longer
 *     present is left alone, as yk_release leaves it), and every queue on its application's chain, the application's
 *     allocation and the user-limit held entries that apply go up by delta; yk_release later gives back the new request.
 *     Nothing is checked against fit, headroom or limits: the kubelet has applied the resize already (an infeasible one never
 *     arrives: GetPodResource then reports the status requests).  A node may so end up with negative available (every path
 *     treats it as 0), a queue over its max or a user over a limit (their later asks are SKIPPED).
 *   Any other present ask (pending, NOFIT, SKIPPED, INVALID, SLOWPATH): the request is replaced, the ask is signed again and
 *     its cause follows the new request (not strictly greater than zero: INVALID from the next cycle, and valid again after a
 *     later resize).  Priority, create_seq, application, masks, required node, flags and gang stay, and so does its place in
 *     the order; the next cycle is the one yk_asks_upsert with the same other fields would give.  Its state stays what the
 *     last cycle left until the next cycle.
 *   Errors, all checked before anything changes; nothing changes on an error:
 *     YK_ERR_ARG   idx / req NULL with n > 0, an index >= max_asks, the same index twice, a negative entry for an allocated ask;
 *     YK_ERR_STATE an ask that is not present;
 *     YK_ERR_RANGE a sum that would overflow int64 (a node's available, a queue's, application's or user's allocation).
 *   n == 0 and an unchanged vector are YK_OK, and the next cycle is unchanged.  No counter moves and nothing is launched; the
 *   node and ask tables are uploaded by the next call that reads them.  Multi-GPU split sweep (world > 1): every rank makes
 *   the same call between the same two cycles. */
int yk_asks_resize(yk_engine* e, uint32_t n, const uint32_t* idx, const int64_t* req /* [D][n] column-major */);

/* One scheduling cycle: runs schedule() passes until no pending ask can be placed or max_bindings is
 * reached.  out[0..*n_out) are the bindings in the reference's commit order.  slow_path_asks (may be NULL)
 * receives up to slow_cap asks flagged YK_ASK_SLOWPATH that were reached in order.
 * max_bindings ends the cycle at the first placement it cannot hold (an ask, or a gang that passed its queue-side checks
 * and has more members than bindings are left); the bindings are a prefix of the uncut cycle's.
 * The engine looks one batch ahead, so a few asks just behind the cut may already carry a cause (INVALID / SLOWPATH /
 * SKIPPED / NOFIT) that the uncut order would have given them later; every cycle starts all unallocated asks as pending
 * again, so this never changes a later binding. */
int yk_cycle(yk_engine* e, uint32_t max_bindings, yk_binding* out, uint32_t* n_out,
             uint32_t* slow_path_asks, uint32_t slow_cap, uint32_t* n_slow);

int yk_ask_states(yk_engine* e, uint32_t n, const uint32_t* idx, uint8_t* state_out);
/* current node available, [D][n] */
int yk_nodes_available(yk_engine* e, uint32_t n, const uint32_t* idx, int64_t* avail_out);
/* one (ask,node) answer on the current state, evaluated on the device: 0 fits / YK_FAIL_* / <0 error */
int yk_evaluate(yk_engine* e, uint32_t ask, uint32_t node);
/* the same answer for the reservation phase, Predicates(Allocate = false): the reference then runs the same plugins WITHOUT
 * NodeResourcesFit (pkg/plugin/predicates/predicate_manager.go:130-135, reservation filter set :353-368) and the core does
 * not ask for available resources: YK_FAIL_AVAILABLE / YK_FAIL_RESOURCES cannot come back.  (Reservations themselves --
 * an old unplaceable ask pinning a node -- are not made by yk_cycle: SURVEY A.1, DESIGN.md.) */
int yk_evaluate_reserve(yk_engine* e, uint32_t ask, uint32_t node);
/* node sort keys as the device computes them (float64 score bits), for known-answer tests */
int yk_node_scores(yk_engine* e, uint32_t n, const uint32_t* idx, double* score_out);

/* Replace the node sort policy and resource weights of a live engine: the partition's nodesortpolicy (type, resourceweights)
 * of the core's configuration, which the shim hands over in RegisterResourceManager / UpdateConfiguration, after the engine
 * exists.  weights is [YK_MAX_D]; entries at or beyond D are ignored, exactly as in yk_create.  Takes effect from the next
 * call that orders or scores nodes (yk_cycle, yk_filter_nodes, yk_preemption_nodes, yk_node_scores).
 *   Errors: YK_ERR_ARG for a null engine or weights, a policy other than YK_POLICY_FAIR / YK_POLICY_BINPACKING, or a NaN or
 *     infinite weight among the first D.  Negative weights are accepted, as yk_create accepts them (cycles under them take the
 *     sweep + host commit).
 *   All or nothing: before anything changes, every present node is scored on the device under the new setting; if one scores
 *     NaN (as yk_cycle refuses: e.g. weighted resources with total 0 and non-zero available whose infinite shares cancel), the
 *     call returns YK_ERR_RANGE and the old setting stays.  With no present node nothing is launched.
 *   What stays: node tables, ask states, queue / application / user accounting and every counter but other_launches /
 *     h2d_bytes / d2h_bytes.  Setting the current values again is YK_OK, and the next yk_cycle is the one it would have been.
 *     The engine keeps no order or key across calls, so the next call behaves exactly as on an engine created with the new
 *     setting and the same tables.
 *   Creation-time, not switched: YK_FLAG_BINPACKING_DEVICE, YK_FLAG_HOST_COMMIT / YK_FLAG_DEVICE_COMMIT, D and the capacities.
 *     An engine created without YK_FLAG_BINPACKING_DEVICE commits binpacking cycles on the host after a switch.
 *   Multi-GPU split sweep (world > 1): every rank orders the nodes itself, so every rank must make the same call between the
 *     same two cycles. */
int yk_node_sort_set(yk_engine* e, uint32_t policy, const double* weights);

/* Every present node's first failing step for a list of asks, in the cycle's node order, evaluated on the device in one
 * grid-wide pass (csrc/yk_filter.cuh).  For the slow-path bridge (walk only the nodes that pass the engine's own steps, in
 * the engine's order, through the Go PredicateManager) and for the per-cause FAILED reason of an unplaceable pod.  Read-only.
 *   Nodes considered: every present node, ordered exactly as yk_cycle would order them now -- ascending float64 score under
 *     the engine's policy and weights (yk_score.h), ties by name_rank, then by node index.
 *   Slot of a pair: YK_FILTER_RESERVED if the node is flagged YK_NODE_RESERVED (hidden from the core's node iterator, never
 *     evaluated); otherwise exactly what yk_evaluate(ask, node) returns -- yk_evaluate_reserve(ask, node) when allocate == 0 --
 *     on the current tables; slot 0 = passes.  An ask that is not present counts every node in slot YK_FAIL_ABSENT and has
 *     no candidates.  counts[i*YK_FILTER_SLOTS + slot] (may be NULL) sums to the number of present nodes.
 *   Candidates: nodes_out[i*k + j] = the passing node of rank skip + j in that order (j < k), YK_NONE past the last one;
 *     n_pass[i] (may be NULL) = the number of passing nodes = counts[i*YK_FILTER_SLOTS].  With allocate == 1 and no reserved
 *     node, candidate 0 (skip = 0) is the node the frozen-snapshot sweep of a cycle picks for that ask.
 *   Node side only: queue headroom, user limits, gangs and YK_ASK_SLOWPATH play no part, as in yk_evaluate.
 *   Errors: YK_ERR_ARG for an ask index >= max_asks, k > 0 with nodes_out == NULL, or n > 0 with asks == NULL;
 *     YK_ERR_RANGE when a present node scores NaN (as yk_cycle), and then nothing is written.  n == 0 is YK_OK.
 *   No state changes: stale tables are uploaded and the nodes sorted in the filter's own device buffers, so the next yk_cycle
 *     is the same whether or not this ran.  Counted in other_launches / h2d_bytes / d2h_bytes; local to this engine
 *     whatever rank / world are. */
#define YK_FILTER_SLOTS 11      /* slot 0 = passes, 1..9 = the YK_FAIL_* answer of yk_evaluate, 10 = reserved */
#define YK_FILTER_RESERVED 10   /* YK_NODE_RESERVED: hidden from the core's node iterator, never evaluated */
int yk_filter_nodes(yk_engine* e, uint32_t n, const uint32_t* asks, int allocate, uint32_t skip, uint32_t k,
                    uint32_t* nodes_out /* [n][k] row-major, YK_NONE padded, may be NULL iff k == 0 */,
                    uint32_t* n_pass /* [n], may be NULL */, uint32_t* counts /* [n][YK_FILTER_SLOTS] row-major, may be NULL */);

/* Preemption victim search, batched (ResourceManagerCallback.PreemptionPredicates,
 * pkg/cache/scheduler_callback.go:200-209 -> context.go:705-729 -> predicate_manager.go:137-175).  Query q: the
 * smallest index i >= start[q] such that ask[q] passes every predicate on node[q] once the victims
 * victim_off[q] .. victim_off[q]+i (in the given order) are removed, or -1.  victim_req is [D][victim_off[n]]: what
 * each victim gives back to the node.  Known answers: TestPreemptionPredicates(+Empty), predicate_manager_test.go:67-134. */
int yk_preemption_search(yk_engine* e, uint32_t n_queries, const uint32_t* ask, const uint32_t* node,
                         const uint32_t* victim_off, const int64_t* victim_req, const uint32_t* start, int32_t* index_out);

/* The same victim search over every node at once, for allocations this engine made: for each ask a victim list (the
 * caller's policy picks the victims and their order), and back the nodes those victims can free, in the cycle's node order,
 * evaluated on the device (csrc/yk_preempt_nodes.cuh).  The engine knows where each victim is bound and what it holds, so
 * the caller sends only ask indices.  Read-only.
 *   Victims of ask i on node p: V(i,p) = the entries of victims[victim_off[i] .. victim_off[i+1]) bound to p, in list order.
 *     answer(i,p) is exactly what yk_preemption_search(asks[i], p, <requests of V(i,p)>, start = 0) returns on the current
 *     tables.  p FITS when answer >= 0 and then needs answer + 1 victims.  A node with no victim in the list does not fit (the
 *     reference's loop never runs for it).  Reservation flags are not consulted (PreemptionPredicates does not look at
 *     them); an unschedulable node fails the static part.
 *   Nodes considered: every present node, ordered as yk_filter_nodes orders them (ascending float64 score, then name_rank,
 *     then index).  An entry whose victim is bound to a node that is no longer present is ignored.
 *   Per ask: n_fit[i] = the number of fitting nodes; nodes_out[i*k + j] / need_out[i*k + j] = the fitting node of fit rank
 *     skip + j and its victim count (YK_NONE / 0 past the last one); best_node[i] / best_need[i] = the fitting node with the
 *     fewest victims, ties to the earlier node in the order (YK_NONE / 0 when nothing fits).  An ask that is not present has
 *     no fitting node.
 *   Errors, all checked before any device work; nothing is written on an error:
 *     YK_ERR_ARG   asks / victim_off NULL with n > 0, victims NULL with victim_off[n] > 0, nodes_out NULL with k > 0, an ask
 *                  or victim index >= max_asks, victim_off[0] != 0 or decreasing, the same victim twice in one list;
 *     YK_ERR_STATE a victim that is not YK_ST_ALLOCATED;
 *     YK_ERR_RANGE a present node scores NaN (as yk_cycle).
 *     n == 0 is YK_OK.
 *   No state changes: the next yk_cycle is the same whether or not this ran.  Counted in other_launches / h2d_bytes /
 *     d2h_bytes; local to this engine whatever rank / world are.  Lists are processed in chunks of whole lists: a chunk ends
 *     before the list that would take it past 4096 lists or 2^18 entries (a longer list is a chunk of its own). */
int yk_preemption_nodes(yk_engine* e, uint32_t n, const uint32_t* asks,
                        const uint32_t* victim_off /* [n+1], victim_off[0] = 0, non-decreasing */,
                        const uint32_t* victims /* [victim_off[n]] ask indices, per ask in the caller's victim order */,
                        uint32_t skip, uint32_t k,
                        uint32_t* nodes_out /* [n][k] row-major, YK_NONE padded; may be NULL iff k == 0 */,
                        uint32_t* need_out /* [n][k] victims needed on that node, 0 padded; may be NULL */,
                        uint32_t* n_fit /* [n], may be NULL */,
                        uint32_t* best_node /* [n], may be NULL */, uint32_t* best_need /* [n], may be NULL */);

/* Preemption for queues below their guarantee: for each preemptor, in the order given, the victims and the node that let it run
 * (the core's guarantee preemption, DESIGN.md §2 item 9), evaluated on the device (csrc/yk_preempt_plan.cuh).  A plan MARKS
 * its victims and records the preemptor as planned on its node; the caller releases the victims (yk_release) and pins the
 * preemptor (required_node), and the next yk_cycle places it.  yk_cycle never reads marks or plans.
 *   For plan calls, usage(q) = allocated(q) - marked victims below q + requests of planned preemptors below q, and
 *   room(node) = available + marked victims on it - requests of planned preemptors on it.  Later preemptors of one call see the
 *   marks and plans of the earlier ones.
 *   Status per ask (status_out[i]):
 *     YK_PP_NOT_BLOCKED  not present, state not YK_ST_NOFIT / YK_ST_SKIPPED, or already planned by an earlier call;
 *     YK_PP_NOT_ALLOWED  YK_ASK_NO_PREEMPT_OTHER, or over the headroom of a user limit that applies to it;
 *     YK_PP_UNSUPPORTED  slow path, gang member or required node;
 *     YK_PP_GUARANTEE    its leaf has no guarantee, or some queue on its path with a guarantee would go over it;
 *     YK_PP_NO_VICTIMS   no node fits it with victims, or the queue headroom cannot be freed;
 *     YK_PP_FITS         a node fits it and no victim is needed (the next cycle places it): nothing is marked;
 *     YK_PP_PLANNED      victims marked, the ask planned on node_out[i].
 *   Victims: an allocation bound by this engine to a present node, not marked, without a required node, outside the
 *     preemptor's leaf, inside the fence root's subtree (the nearest queue on the preemptor's path with preemption fence, or
 *     root), whose priority plus the priority.offset of its queues strictly below the lowest common ancestor is at most the
 *     preemptor's computed the same way.  Order: without YK_ASK_NO_PREEMPT_SELF first, non-originators first, adjusted
 *     priority ascending (saturated to int32), create_seq descending, index.  A victim is taken only if every queue with a
 *     guarantee on its path strictly below the lowest common ancestor stays at or above it with every victim taken so far.
 *   Node: of the present nodes that pass the preemptor's static steps (schedulable, taints, labels, total), the one needing the
 *     fewest of its own victims (in order) until request <= max(0, room); ties to the earlier node in the cycle's order.
 *   Headroom: while a queue on the preemptor's path with a max is over it (usage + request > max), further victims in order from
 *     any node below a queue still over its max are taken; if they run out the status is YK_PP_NO_VICTIMS and nothing is marked.
 *   Output: node_out[i] = the node (PLANNED / FITS) or YK_NONE; the victims of ask i are
 *     victims_out[victim_off_out[i] .. victim_off_out[i+1]), node victims first, each group in victim order.  Planning stops
 *     before the first ask whose victims would pass victims_cap; *n_done = the asks handled, and only status_out / node_out
 *     [0, n_done) and victim_off_out [0, n_done] are written.
 *   Marks clear when the allocation is released (yk_release); plans when the preemptor is allocated by a cycle, removed,
 *     upserted again or resized.
 *   Errors, all checked before anything is marked; nothing changes on an error:
 *     YK_ERR_ARG   asks / status_out / node_out / victim_off_out / n_done NULL with n > 0, victims_out NULL with victims_cap > 0,
 *                  an index >= max_asks, the same ask twice;
 *     YK_ERR_RANGE a present node scores NaN (as yk_cycle).
 *   A YK_ERR_CUDA rolls every mark and plan of the call back.  n == 0 is YK_OK.  Counted in other_launches / h2d_bytes /
 *   d2h_bytes.  Multi-GPU split sweep (world > 1): every rank makes the same call between the same two cycles. */
#define YK_PP_PLANNED 0u
#define YK_PP_FITS 1u
#define YK_PP_NOT_BLOCKED 2u
#define YK_PP_NOT_ALLOWED 3u
#define YK_PP_UNSUPPORTED 4u
#define YK_PP_GUARANTEE 5u
#define YK_PP_NO_VICTIMS 6u
int yk_preemption_plan(yk_engine* e, uint32_t n, const uint32_t* asks, uint32_t* status_out, uint32_t* node_out,
                       uint32_t* victim_off_out /* [n+1] */, uint32_t* victims_out /* [victims_cap] */, uint32_t victims_cap,
                       uint32_t* n_done);

/* Preemption for asks with a required node (DaemonSet pods): for each preemptor a, in the order given, the victims on its node
 * X = required_node(a) that let it run (the core's required-node preemption, DESIGN.md §2 item 10), evaluated for every
 * preemptor of the call in one pass on the device (csrc/yk_preempt_required.cuh).  Marks and plans are those of
 * yk_preemption_plan, and each call sees the other's; room(X) is as documented there.
 *   Status per ask (status_out[i], the YK_PP_* values; YK_PP_GUARANTEE is never returned):
 *     YK_PP_NOT_BLOCKED  not present, state not YK_ST_NOFIT / YK_ST_SKIPPED, or already planned by either plan call;
 *     YK_PP_UNSUPPORTED  no required node, slow path or gang member;
 *     YK_PP_NOT_ALLOWED  over the headroom of a queue max on its path or of a user / group limit that applies to it, from what
 *                        is allocated (marks and plans play no part); YK_ASK_NO_PREEMPT_OTHER is not read;
 *     YK_PP_NO_VICTIMS   X not present, X fails its static steps (schedulable, taints, labels, request <= max(0, total)), or
 *                        the eligible victims never add up to the request;
 *     YK_PP_FITS         request <= max(0, room(X)) in every resource: nothing is marked;
 *     YK_PP_PLANNED      victims marked, the ask planned on X, room(X) moved by + victims - request for later preemptors.
 *   Victims: allocations bound to X, not marked, without a required node, with priority <= the preemptor's (no queue offsets),
 *     and a non-zero request on some resource the preemptor asks for.  Order: neither YK_ASK_NO_PREEMPT_SELF nor
 *     YK_ASK_ORIGINATOR first, then YK_ASK_NO_PREEMPT_SELF non-originators, then originators; priority ascending; create_seq
 *     descending; index.  The victims are the shortest prefix of that order whose sum covers the preemptor's full request in
 *     every resource (not the part room(X) lacks).
 *   Output: the victims of ask i are victims_out[victim_off_out[i] .. victim_off_out[i+1]), in victim order.  Planning stops
 *     before the first ask, in the order given, whose victims would pass victims_cap; *n_done = the asks handled, and only
 *     status_out [0, n_done) and victim_off_out [0, n_done] are written.  Nothing past the stop is marked or planned.
 *   No node order is used: node scores are not computed and a NaN score elsewhere is no error.
 *   Errors, all checked before anything is marked; nothing changes on an error:
 *     YK_ERR_ARG   asks / status_out / victim_off_out / n_done NULL with n > 0, victims_out NULL with victims_cap > 0, an index
 *                  >= max_asks, the same ask twice.
 *   A YK_ERR_CUDA rolls every mark and plan of the call back.  n == 0 is YK_OK.  Counted in other_launches / h2d_bytes /
 *   d2h_bytes.  Multi-GPU split sweep (world > 1): every rank makes the same call between the same two cycles. */
int yk_preemption_required_node(yk_engine* e, uint32_t n, const uint32_t* asks, uint32_t* status_out,
                                uint32_t* victim_off_out /* [n+1] */, uint32_t* victims_out /* [victims_cap] */,
                                uint32_t victims_cap, uint32_t* n_done);

/* multi-GPU exchange hook: called once per batch on every rank, after the local shard's rows of `buf`
 * (device pointer, row-major, `row_bytes` per ask, rows [first_row, first_row+n_rows) are this rank's)
 * have been written on `stream`; must make all `total_rows` rows valid on every rank (an all-gather). */
typedef int (*yk_allgather_fn)(void* ctx, void* device_buf, uint64_t row_bytes, uint32_t first_row,
                               uint32_t n_rows, uint32_t total_rows, void* cuda_stream);
int yk_set_exchange(yk_engine* e, yk_allgather_fn fn, void* ctx);

/* Peer-to-peer exchange (preferred over yk_set_exchange when all ranks sit on one NVLink / NVSwitch node): every
 * rank exports its fit buffers and sync block as CUDA IPC handles, imports every other rank's, and from then on the
 * sweep kernel stores its rows straight into all ranks' buffers -- the all-gather is fused into the sweep, ordered by
 * sequence flags in peer memory, with no collective launch and no host involvement.  Call yk_peer_export on every
 * rank, exchange the blobs (any transport), call yk_peer_import once per other rank, then yk_peer_enable. */
typedef struct { unsigned char blob[3][64]; } yk_peer_handles;   /* cudaIpcMemHandle_t x {slot 0, slot 1, sync} */
int yk_peer_export(yk_engine* e, yk_peer_handles* out);
int yk_peer_import(yk_engine* e, uint32_t peer_rank, const yk_peer_handles* in);
int yk_peer_enable(yk_engine* e);

int yk_stats(yk_engine* e, yk_stats_t* out);
int yk_stats_reset(yk_engine* e);
const char* yk_strerror(int status);
const char* yk_last_error(yk_engine* e);
uint32_t yk_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif
