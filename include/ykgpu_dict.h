/*
 * ykgpu_dict.h -- C ABI of the label / taint dictionary encoder (part of libykgpu.so).
 *
 * Turns the string-level Kubernetes predicates of a pod and a node into the 64-bit sets the engine sweeps
 * (SURVEY.md Appendix A.4).  This is the "snapshot builder" half of the boundary: the Go adapter calls it
 * when cache.Context sees a node or pod change (pkg/cache/context.go:127-171 handlers), then passes the
 * masks to yk_nodes_upsert / yk_asks_upsert.  What it restates [EXT k8s.io/kubernetes v1.34.6, go.mod:46,
 * k8s.io/component-helpers/scheduling/corev1/nodeaffinity, k8s.io/api core/v1 toleration.go]:
 *   NodeAffinity      pod.Spec.NodeSelector AND required node affinity (terms ORed; a term = matchExpressions
 *                     AND matchFields; empty or unparsable term matches nothing; nil/empty term list matches
 *                     nothing); operators In, NotIn, Exists, DoesNotExist, Gt, Lt; matchFields metadata.name
 *   TaintToleration   a node taint with effect NoSchedule / NoExecute must be tolerated
 *                     (Toleration.ToleratesTaint: effect, key, operator Equal|Exists)
 *   NodeUnschedulable node.Spec.Unschedulable acts as taint node.kubernetes.io/unschedulable:NoSchedule
 *   NodeName          pod.Spec.NodeName must name the node
 * pinned by the reference's tables: TestPodFitsSelector (27 cases) predicate_manager_test.go:366-1061,
 * TestReserveAlloc / TestReserveNodeSelector :2152-2242, TestPodFitsHost :162-222 (tests/golden/).
 *
 * Encoding: one label bit per distinct positive requirement (key In {values} | key Exists | key Gt v | key Lt v)
 * referenced by some pod, or per whole selector when it has several terms or matchFields; NotIn / DoesNotExist use
 * the same bit on the forbidden side.  Label bit 63 is reserved "impossible" (set on no node).  One taint bit per
 * distinct (key, value, effect in {NoSchedule, NoExecute}).  When the dictionary is full the pod is flagged
 * YK_ASK_SLOWPATH -- never approximated.
 */
#ifndef YKGPU_DICT_H
#define YKGPU_DICT_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define YK_OP_IN 0u
#define YK_OP_NOT_IN 1u
#define YK_OP_EXISTS 2u
#define YK_OP_DOES_NOT_EXIST 3u
#define YK_OP_GT 4u
#define YK_OP_LT 5u

#define YK_EFFECT_ALL 0u              /* toleration only: empty effect tolerates every effect */
#define YK_EFFECT_NO_SCHEDULE 1u
#define YK_EFFECT_PREFER_NO_SCHEDULE 2u
#define YK_EFFECT_NO_EXECUTE 3u

#define YK_TOL_EQUAL 0u               /* "" or Equal */
#define YK_TOL_EXISTS 1u

typedef struct { const char* key; uint32_t op; uint32_t n_values; const char* const* values; } yk_requirement;
typedef struct { uint32_t n_expressions; const yk_requirement* expressions;
                 uint32_t n_fields; const yk_requirement* fields; } yk_selector_term;
typedef struct { const char* key; const char* value; uint32_t effect; } yk_taint;
typedef struct { const char* key; uint32_t op; const char* value; uint32_t effect; } yk_toleration;

typedef struct {
    uint32_t n_selector; const char* const* selector_keys; const char* const* selector_values;  /* pod.Spec.NodeSelector */
    int32_t has_required_affinity;          /* Affinity.NodeAffinity.RequiredDuringSchedulingIgnoredDuringExecution != nil */
    uint32_t n_terms; const yk_selector_term* terms;
    uint32_t n_tolerations; const yk_toleration* tolerations;
    const char* node_name;                  /* pod.Spec.NodeName or NULL/"" */
} yk_pod_spec;

typedef struct {
    uint64_t tolerated_bits, required_bits, forbidden_bits;
    uint32_t required_node;                 /* node index or YK_NONE */
    uint32_t flags;                         /* YK_ASK_SLOWPATH when the dictionary has no bit left */
} yk_pod_masks;

typedef struct yk_dict yk_dict;

yk_dict* yk_dict_create(void);
void yk_dict_destroy(yk_dict* d);
/* (re)register a node under a dense index; writes its current bit sets */
int yk_dict_node(yk_dict* d, uint32_t node_idx, const char* name, uint32_t n_labels, const char* const* label_keys,
                 const char* const* label_values, uint32_t n_taints, const yk_taint* taints, int32_t unschedulable,
                 uint64_t* label_bits, uint64_t* taint_bits);
int yk_dict_node_remove(yk_dict* d, uint32_t node_idx);
/* compile a pod; may allocate new bits, which changes node bit sets: compare yk_dict_generation before/after
 * and re-read the nodes with yk_dict_node_bits when it moved */
int yk_dict_pod(yk_dict* d, const yk_pod_spec* pod, yk_pod_masks* out);
/* a pod whose node is fixed before it is scheduled (a DaemonSet pod: the node its required affinity names through matchFields
 * metadata.name): encoded as yk_dict_pod does, with required_node = the index of node_name.  An unknown node_name, or a
 * pod->node_name that differs from it, sets the impossible bit.  The required-affinity terms are resolved against node_name
 * first: a term whose matchFields reject it is dropped, a term whose fields accept it keeps only its expressions, and a term
 * left without expressions matches unconditionally, so the affinity adds no bit (an originally empty term still matches
 * nothing).  The rest is encoded as yk_dict_pod encodes a term list.  Exact for the only node the ask can use; the usual
 * DaemonSet pod takes no label bit. */
int yk_dict_pod_required_node(yk_dict* d, const yk_pod_spec* pod, const char* node_name, yk_pod_masks* out);
uint64_t yk_dict_generation(const yk_dict* d);
int yk_dict_node_bits(const yk_dict* d, uint32_t node_idx, uint64_t* label_bits, uint64_t* taint_bits);

#ifdef __cplusplus
}
#endif
#endif
