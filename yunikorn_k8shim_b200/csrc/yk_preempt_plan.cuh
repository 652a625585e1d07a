// yk_preempt_plan.cuh -- sm_90a device code of yk_preemption_plan: the victims a preemptor may take (DESIGN.md §2 item 9,
// rules 3-6) and the node that needs the fewest of them.
//
// Per call the host lists the bound allocations (a "slot" each) and sorts them once by (create_seq descending, index): the
// position t of a slot in that order is the last part of the victim-order key, so one 64-bit key carries the whole order.
// Then per preemptor:
//   yk_pp_victim_kernel   one thread per position t: eligibility (fence subtree, own queue, LCA-relative priorities) and the
//                         key (no-preempt-self, originator, adjusted priority, t); ineligible: YK_PP_INELIGIBLE
//   cub radix sort        by that key: the global victim order (eligible first)
//   yk_pp_nodekey_kernel  the node position of each entry in victim order (ineligible: nlive)
//   cub radix sort        stable, by node position: per-node segments, still in victim order
//   yk_pp_node_kernel     one warp per node: the static steps, then the victims in order under the guarantee rule; the fewest
//                         that make the ask fit, folded into one (need, position) minimum with atomicMin
// Queue ancestry is an interval test on a preorder numbering (tin / tout); priority offsets are prefix sums from the root.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "yk_kernels.cuh"

#define YK_PP_INELIGIBLE 0xFFFFFFFFFFFFFFFFull
#define YK_PPF_NO_SELF 1u       // slot flags: the allocation's YK_ASK_NO_PREEMPT_SELF
#define YK_PPF_ORIGINATOR 2u    // YK_ASK_ORIGINATOR
#define YK_PPF_OUT 4u           // never a victim: a required node, or already marked

struct YkPPArgs {
    int D;
    // queue tables [nq]; q_guar / q_use are [D][nq] (q_guar -1 = not set)
    const uint32_t* q_parent; const uint32_t* q_depth; const uint32_t* q_tin; const uint32_t* q_tout;
    const int64_t* q_poff; const int64_t* q_guar; const int64_t* q_use; const uint8_t* q_hasg; int nq;
    // bound allocations: per slot the ask, its leaf queue, priority, YK_PPF_* flags and node; perm[t] = slot of position t
    const uint32_t* v_ask; const uint32_t* v_leaf; const int32_t* v_prio; const uint32_t* v_flag; const uint32_t* v_node;
    const uint32_t* perm; int m;
    // node side: position of each node in the cycle's order, the order itself, room [D][ldn] for plan calls
    const uint32_t* pos; const uint32_t* sorted; int nlive; const int64_t* room;
    const int64_t* total; size_t ldn; const uint64_t* taint; const uint64_t* label; const uint32_t* flags;
    const int64_t* a_req; const uint64_t* a_tol; const uint64_t* a_need; const uint64_t* a_deny; size_t lda;
    // the preemptor: ask, leaf queue, fence root, priority
    uint32_t ask, leaf, fence; int32_t prio;
};

__device__ __host__ inline bool yk_pp_inside(const uint32_t* tin, const uint32_t* tout, uint32_t q, uint32_t x) {
    return tin[q] <= tin[x] && tin[x] < tout[q];
}
__device__ __host__ inline uint32_t yk_pp_lca(const uint32_t* parent, const uint32_t* depth, uint32_t a, uint32_t b) {
    while (depth[a] > depth[b]) a = parent[a];
    while (depth[b] > depth[a]) b = parent[b];
    while (a != b) { a = parent[a]; b = parent[b]; }
    return a;
}
// rule 3's priority test and rule 4's key for the allocation of leaf x and priority pv; YK_PP_INELIGIBLE when it is not a victim
__device__ __host__ inline uint64_t yk_pp_key(const YkPPArgs& a, uint32_t x, int32_t pv, uint32_t f, uint32_t t) {
    if ((f & YK_PPF_OUT) || x == a.leaf || !yk_pp_inside(a.q_tin, a.q_tout, a.fence, x)) return YK_PP_INELIGIBLE;
    const uint32_t c = yk_pp_lca(a.q_parent, a.q_depth, x, a.leaf);
    const int64_t adj_v = (int64_t)pv + a.q_poff[x] - a.q_poff[c];
    const int64_t adj_a = (int64_t)a.prio + a.q_poff[a.leaf] - a.q_poff[c];
    if (adj_v > adj_a) return YK_PP_INELIGIBLE;
    const int64_t sat = adj_v < INT32_MIN ? INT32_MIN : (adj_v > INT32_MAX ? INT32_MAX : adj_v);
    const uint64_t biased = (uint64_t)((uint32_t)(int32_t)sat ^ 0x80000000u);
    return ((uint64_t)(f & YK_PPF_NO_SELF) << 63) | ((uint64_t)((f & YK_PPF_ORIGINATOR) ? 1 : 0) << 62) | (biased << 30) | t;
}

__global__ void yk_pp_victim_kernel(YkPPArgs a, uint64_t* __restrict__ key, uint32_t* __restrict__ val, uint32_t* __restrict__ n_elig) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    uint64_t k = YK_PP_INELIGIBLE;
    if (t < a.m) {
        const uint32_t s = a.perm[t];
        k = yk_pp_key(a, a.v_leaf[s], a.v_prio[s], a.v_flag[s], (uint32_t)t);
        key[t] = k;
        val[t] = (uint32_t)t;
    }
    const int c = __syncthreads_count(k != YK_PP_INELIGIBLE);
    if (threadIdx.x == 0 && c) atomicAdd(n_elig, (uint32_t)c);
}

// entry i of the victim order: its node's position (nlive past the eligible ones), value = its position t
__global__ void yk_pp_nodekey_kernel(YkPPArgs a, const uint64_t* __restrict__ key, const uint32_t* __restrict__ tv,
                                     uint32_t* __restrict__ nkey, uint32_t* __restrict__ nval) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.m) return;
    const uint32_t t = tv[i];
    nkey[i] = key[i] == YK_PP_INELIGIBLE ? (uint32_t)a.nlive : a.pos[a.v_node[a.perm[t]]];
    nval[i] = t;
}

// one warp per node position p.  Segment [lo, hi) of the node-sorted entries; taken[j] = whether entry j was taken (written for
// every entry walked, so no reset is needed).  need = 0 when the ask fits the room already, else the fewest taken victims after
// which it fits; best = min over nodes of need << 32 | p.  seg[2p], seg[2p+1] = the segment, for the host's read-back.
__global__ void yk_pp_node_kernel(YkPPArgs a, const uint32_t* __restrict__ nkey, const uint32_t* __restrict__ nval,
                                  uint8_t* __restrict__ taken, uint32_t* __restrict__ seg, unsigned long long* __restrict__ best) {
    const int p = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (p >= a.nlive) return;
    auto lower = [&](uint32_t x) {
        int lo = 0, hi = a.m;
        while (lo < hi) { const int mid = (lo + hi) >> 1; if (nkey[mid] < x) lo = mid + 1; else hi = mid; }
        return lo;
    };
    const int lo = lower((uint32_t)p), hi = lower((uint32_t)p + 1);
    if (lane == 0) { seg[2 * p] = (uint32_t)lo; seg[2 * p + 1] = (uint32_t)hi; }
    const uint32_t node = a.sorted[p], ask = a.ask;
    const int D = a.D;
    bool stat = (a.flags[node] & 1u) != 0;
    stat = stat && !(a.taint[node] & ~a.a_tol[ask]);
    stat = stat && (a.label[node] & a.a_need[ask]) == a.a_need[ask] && !(a.label[node] & a.a_deny[ask]);
    int64_t rq[8], room[8];
    bool fit = true;
    for (int k = 0; k < D; ++k) {
        rq[k] = a.a_req[(size_t)k * a.lda + ask];
        const int64_t t = a.total[(size_t)k * a.ldn + node];
        room[k] = a.room[(size_t)k * a.ldn + node];
        if (rq[k] > (t < 0 ? 0 : t)) stat = false;
        if (rq[k] > (room[k] < 0 ? 0 : room[k])) fit = false;
    }
    if (!stat) return;
    uint32_t need = fit ? 0u : 0xFFFFFFFFu, cnt = 0;
    for (int j = lo; j < hi && need == 0xFFFFFFFFu; ++j) {
        const uint32_t s = a.perm[nval[j]], x = a.v_leaf[s], va = a.v_ask[s];
        const uint32_t c = yk_pp_lca(a.q_parent, a.q_depth, x, a.leaf);
        int64_t vr[8];
        for (int k = 0; k < D; ++k) vr[k] = a.a_req[(size_t)k * a.lda + va];
        // rule 5: every guaranteed queue on x's path strictly below the LCA stays at or above its guarantee once the victims
        // already taken on this node and this one are removed
        bool ok = true;
        for (uint32_t q = x; q != c && ok; q = a.q_parent[q]) {
            if (!a.q_hasg[q]) continue;
            int64_t rem[8];
            for (int k = 0; k < D; ++k) rem[k] = 0;
            for (int i = lo + lane; i < j; i += 32) {
                if (!taken[i]) continue;
                const uint32_t si = a.perm[nval[i]];
                if (!yk_pp_inside(a.q_tin, a.q_tout, q, a.v_leaf[si])) continue;
                for (int k = 0; k < D; ++k) rem[k] += a.a_req[(size_t)k * a.lda + a.v_ask[si]];
            }
            for (int k = 0; k < D; ++k) {
#pragma unroll
                for (int o = 16; o; o >>= 1) rem[k] += __shfl_xor_sync(0xFFFFFFFFu, rem[k], o);
                const int64_t g = a.q_guar[(size_t)k * a.nq + q];
                if (g >= 0 && a.q_use[(size_t)k * a.nq + q] - rem[k] - vr[k] < g) ok = false;
            }
        }
        __syncwarp();
        if (lane == 0) taken[j] = ok ? 1 : 0;
        __syncwarp();
        if (!ok) continue;
        ++cnt;
        bool f2 = true;
        for (int k = 0; k < D; ++k) { room[k] += vr[k]; if (rq[k] > (room[k] < 0 ? 0 : room[k])) f2 = false; }
        if (f2) need = cnt;
    }
    if (lane == 0 && need != 0xFFFFFFFFu) atomicMin(best, ((unsigned long long)need << 32) | (uint32_t)p);
}
