// yk_preempt_required.cuh -- sm_90a device code of yk_preemption_required_node: preemption for asks with a required node
// (DaemonSet pods, DESIGN.md §2 item 10), for every preemptor of a call in a fixed number of launches.
//
// Victims come only from the preemptor's own node and their order does not depend on the preemptor, so one order serves the
// whole call.  The host lists the allocations that may ever be victims (a "slot" each: bound to a node some preemptor of the
// call requires, not marked, without a required node) and groups the preemptors by node, in call order.  Then:
//   cub radix sort         slots by (create_seq descending, index): the position t in that order, once per call
//   yk_prn_key_kernel      per position: key = group | type | biased priority; stable, so equal keys stay in create order
//   cub radix sort         stable, by that key: per-group segments, each in victim order
//   yk_prn_node_kernel     one warp per group: its preemptors in call order against the group's running room; a walk over the
//                          segment 32 entries at a time (inclusive shuffle scan of the request sums, ballot for the first
//                          lane that covers the request), taken bits per entry
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/ykgpu.h"

#define YK_PRN_TYPE_REGULAR 0u      // neither YK_ASK_NO_PREEMPT_SELF nor YK_ASK_ORIGINATOR
#define YK_PRN_TYPE_NO_SELF 1u      // YK_ASK_NO_PREEMPT_SELF, not an originator
#define YK_PRN_TYPE_ORIGINATOR 2u   // YK_ASK_ORIGINATOR: taken after every other type

struct YkPRNArgs {
    int D;
    // slots: ask, priority, (type << 30 | group)
    const uint32_t* s_ask; const int32_t* s_prio; const uint32_t* s_tg; int m;
    // groups [G]: node, segment [seg[g], seg[g+1]) of the sorted entries, preemptors [p_off[g], p_off[g+1]), room [D][G]
    const uint32_t* g_node; const uint32_t* g_seg; const uint32_t* g_poff; const int64_t* g_room; int G;
    const uint32_t* p_ask; const int32_t* p_prio;
    // node and ask tables of the engine
    const int64_t* total; size_t ldn; const uint64_t* taint; const uint64_t* label; const uint32_t* flags;
    const int64_t* a_req; const uint64_t* a_tol; const uint64_t* a_need; const uint64_t* a_deny; size_t lda;
};

// position t of the create order -> key of slot perm[t]: group (bits 34..63) | type (32..33) | priority biased to unsigned
__global__ void yk_prn_key_kernel(YkPRNArgs a, const uint32_t* __restrict__ perm, uint64_t* __restrict__ key,
                                  uint32_t* __restrict__ val) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.m) return;
    const uint32_t s = perm[t], tg = a.s_tg[s];
    key[t] = ((uint64_t)(tg & 0x3FFFFFFFu) << 34) | ((uint64_t)(tg >> 30) << 32) | (uint32_t)(a.s_prio[s] ^ (int32_t)0x80000000);
    val[t] = s;
}

// entry j may be taken: not taken yet, priority at most the preemptor's, and a non-zero request on some resource the preemptor
// asks for; v = its request when it may (zero otherwise, and past D)
__device__ __forceinline__ bool yk_prn_eligible(const YkPRNArgs& a, const uint32_t* __restrict__ ent, const uint8_t* taken,
                                                uint32_t j, int32_t prio, const int64_t (&rq)[8], int64_t (&v)[8]) {
    const uint32_t s = ent[j];
    bool el = !taken[j] && a.s_prio[s] <= prio, shared = false;
    const uint32_t va = a.s_ask[s];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        v[k] = k < a.D ? a.a_req[(size_t)k * a.lda + va] : 0;
        shared = shared || (v[k] != 0 && rq[k] != 0);
    }
    el = el && shared;
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = el ? v[k] : 0;
    return el;
}

// One warp per group g; ent[j] = the slot of sorted entry j.  taken[j] is owned by the warp of the segment holding j.  Per
// preemptor pi: status[pi], count[pi] and voff[pi] (its victims are vout[voff .. voff + count), in victim order).
__global__ void __launch_bounds__(128) yk_prn_node_kernel(YkPRNArgs a, const uint32_t* __restrict__ ent,
                                                          uint8_t* __restrict__ taken, uint32_t* __restrict__ status,
                                                          uint32_t* __restrict__ count, uint32_t* __restrict__ voff,
                                                          uint32_t* __restrict__ vout) {
    const int g = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (g >= a.G) return;
    const int D = a.D;
    const uint32_t lo = a.g_seg[g], hi = a.g_seg[g + 1], node = a.g_node[g];
    for (uint32_t j = lo + lane; j < hi; j += 32) taken[j] = 0;
    __syncwarp();
    int64_t room[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) room[k] = k < D ? a.g_room[(size_t)k * a.G + g] : 0;
    uint32_t wout = lo;   // a group never takes more victims than its segment holds
    for (uint32_t pi = a.g_poff[g]; pi < a.g_poff[g + 1]; ++pi) {
        const uint32_t ask = a.p_ask[pi];
        const int32_t prio = a.p_prio[pi];
        // the static steps: preemption cannot make the ask fit a node that fails them
        bool stat = (a.flags[node] & 1u) != 0;
        stat = stat && !(a.taint[node] & ~a.a_tol[ask]);
        stat = stat && (a.label[node] & a.a_need[ask]) == a.a_need[ask] && !(a.label[node] & a.a_deny[ask]);
        int64_t rq[8];
        bool fit = true;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            rq[k] = k < D ? a.a_req[(size_t)k * a.lda + ask] : 0;
            if (k < D) {
                const int64_t t = a.total[(size_t)k * a.ldn + node];
                if (rq[k] > (t < 0 ? 0 : t)) stat = false;
                if (rq[k] > (room[k] < 0 ? 0 : room[k])) fit = false;
            }
        }
        uint32_t st = YK_PP_NO_VICTIMS, cnt = 0;
        if (stat && fit) st = YK_PP_FITS;
        else if (stat) {
            // the shortest prefix of the eligible entries whose request sum covers the full request: find its last entry
            int64_t carry[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) carry[k] = 0;
            uint32_t last = hi;
            for (uint32_t j0 = lo; j0 < hi && last == hi; j0 += 32) {
                const uint32_t j = j0 + lane;
                int64_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};   // stays zero past the segment
                const bool el = j < hi && yk_prn_eligible(a, ent, taken, j, prio, rq, v);
                bool reach = el;
#pragma unroll
                for (int k = 0; k < 8; ++k) {
                    if (k >= D) break;   // D is the same on every lane
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
                        const int64_t x = __shfl_up_sync(0xFFFFFFFFu, v[k], o);
                        if (lane >= o) v[k] += x;
                    }
                    if (carry[k] + v[k] < rq[k]) reach = false;
                    carry[k] += __shfl_sync(0xFFFFFFFFu, v[k], 31);
                }
                const unsigned b = __ballot_sync(0xFFFFFFFFu, reach);
                if (b) last = j0 + (uint32_t)(__ffs(b) - 1);
            }
            if (last != hi) {
                // take every eligible entry up to `last`, in order
                for (uint32_t j0 = lo; j0 <= last; j0 += 32) {
                    const uint32_t j = j0 + lane;
                    int64_t v[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                    const bool el = j <= last && yk_prn_eligible(a, ent, taken, j, prio, rq, v);
                    const unsigned b = __ballot_sync(0xFFFFFFFFu, el);
                    if (el) {
                        vout[wout + cnt + __popc(b & ((1u << lane) - 1u))] = a.s_ask[ent[j]];
                        taken[j] = 1;
                    }
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        if (k >= D) break;
#pragma unroll
                        for (int o = 16; o; o >>= 1) v[k] += __shfl_xor_sync(0xFFFFFFFFu, v[k], o);
                        room[k] += v[k];
                    }
                    cnt += (uint32_t)__popc(b);
                }
                __syncwarp();
#pragma unroll
                for (int k = 0; k < 8; ++k) room[k] -= rq[k];
                st = YK_PP_PLANNED;
            }
        }
        if (lane == 0) { status[pi] = st; count[pi] = cnt; voff[pi] = wout; }
        wout += cnt;
    }
}
