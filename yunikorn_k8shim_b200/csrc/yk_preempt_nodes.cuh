// yk_preempt_nodes.cuh -- sm_90a device code of yk_preemption_nodes: for a list of asks and one victim list per ask, every
// node those victims can free, in the cycle's node order.
//
// Node order: the filter's (yk_filter_nodes): yk_key_kernel + radix sort, then yk_pn_pos_kernel scatters each node's
// position.  Then per chunk of whole victim lists (an entry = one victim of one list, its node looked up on the host):
//   yk_pn_key_kernel     key = (list, position of the victim's node), value = entry; a STABLE radix sort by key keeps the
//                        entries of one (list, node) group in list order -- the order the victims are removed in
//   yk_pn_head_kernel    1 where a group starts; an inclusive scan numbers the groups
//   yk_pn_group_kernel   one query of yk_preempt_kernel per group (ask, node, victim range, start 0) and the victims'
//                        requests gathered into a [D][entries] column block
//   yk_preempt_kernel    (yk_kernels.cuh, unchanged) answers every group: the answer yk_preemption_search gives
//   yk_pn_rank_kernel    one warp per list over its groups, already in node order: fit ranks, the [skip, skip + k)
//                        window, and the fitting node with the fewest victims
// Only [rows][2k + 3] words are read back.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "yk_kernels.cuh"

// pos[sorted[i]] = i: a node's position in the cycle's order
__global__ void yk_pn_pos_kernel(const uint32_t* __restrict__ sorted, int nlive, uint32_t* __restrict__ pos) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nlive) pos[sorted[i]] = (uint32_t)i;
}

// entry j of list r (off[r] <= j < off[r+1]) on node enode[j]: key = r << pbits | pos[node], value = j
__global__ void yk_pn_key_kernel(const uint32_t* __restrict__ off, int rows, const uint32_t* __restrict__ enode,
                                 const uint32_t* __restrict__ pos, int m, int pbits, uint64_t* __restrict__ key,
                                 uint32_t* __restrict__ val) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    int lo = 0, hi = rows;                     // the largest r with off[r] <= j (off[rows] = m > j)
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (off[mid] <= (uint32_t)j) lo = mid; else hi = mid - 1;
    }
    key[j] = ((uint64_t)lo << pbits) | pos[enode[j]];
    val[j] = (uint32_t)j;
}

__global__ void yk_pn_head_kernel(const uint64_t* __restrict__ key, int m, uint32_t* __restrict__ head) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < m) head[j] = (j == 0 || key[j] != key[j - 1]) ? 1u : 0u;
}

// incl = inclusive scan of the heads, G = incl[m-1] groups.  Group g = incl[j] - 1 of head j: query (asks[r], node at
// position p, victims g_off[g] .. g_off[g+1]).  The launch of yk_preempt_kernel covers m queries; those past G get no
// victims (answer -1, never read).
__global__ void yk_pn_group_kernel(int D, const uint64_t* __restrict__ key, const uint32_t* __restrict__ val,
                                   const uint32_t* __restrict__ incl, int m, int pbits, const uint32_t* __restrict__ asks,
                                   const uint32_t* __restrict__ victim, const uint32_t* __restrict__ sorted,
                                   const int64_t* __restrict__ a_req, size_t lda, uint32_t* __restrict__ g_ask,
                                   uint32_t* __restrict__ g_node, uint32_t* __restrict__ g_off, int64_t* __restrict__ vreq) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= m) return;
    const uint32_t G = incl[m - 1];
    const uint64_t kj = key[j];
    if (j == 0 || kj != key[j - 1]) {
        const uint32_t g = incl[j] - 1;
        g_ask[g] = asks[kj >> pbits];
        g_node[g] = sorted[kj & ((1ull << pbits) - 1)];
        g_off[g] = (uint32_t)j;
    }
    const uint32_t v = victim[val[j]];
    for (int k = 0; k < D; ++k) vreq[(size_t)k * m + j] = a_req[(size_t)k * lda + v];
    if ((uint32_t)j >= G) { g_ask[j] = 0; g_node[j] = 0; g_off[j + 1] = (uint32_t)m; }
    if (j == m - 1) g_off[G] = (uint32_t)m;
}

// one warp per list r: its groups are [incl[off[r]] - 1, incl[off[r+1] - 1]), in node order.  out row r (2k + 3 words):
// [0, k) nodes of fit rank skip + j (YK_NONE past the end), [k, 2k) their victim counts (0 past the end), then the number of
// fitting nodes, the fitting node with the fewest victims (ties: the earlier node) and its count (YK_NONE / 0: none fits).
__global__ void yk_pn_rank_kernel(const uint32_t* __restrict__ off, const uint32_t* __restrict__ incl,
                                  const int32_t* __restrict__ res, const uint32_t* __restrict__ g_node, int rows,
                                  uint32_t skip, uint32_t k, uint32_t* __restrict__ out) {
    const int r = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;
    const uint32_t e0 = off[r], e1 = off[r + 1];
    const uint32_t g0 = e0 < e1 ? incl[e0] - 1 : 0, g1 = e0 < e1 ? incl[e1 - 1] : 0;
    uint32_t* o = out + (size_t)r * (2 * (size_t)k + 3);
    const uint64_t lo = skip, hi = (uint64_t)skip + k;
    uint64_t nfit = 0;
    unsigned long long best = ~0ull;           // need << 32 | group: the fewest victims, then the earliest node
    for (uint32_t b = g0; b < g1; b += 32) {
        const uint32_t g = b + (uint32_t)lane;
        const int32_t ans = g < g1 ? res[g] : -1;
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, ans >= 0);
        if (ans >= 0) {
            const uint64_t rank = nfit + (uint64_t)__popc(m & ((1u << lane) - 1u));
            const uint32_t need = (uint32_t)ans + 1u;
            if (rank >= lo && rank < hi) { o[rank - lo] = g_node[g]; o[k + (rank - lo)] = need; }
            best = min(best, ((unsigned long long)need << 32) | g);
        }
        nfit += (uint64_t)__popc(m);
    }
#pragma unroll
    for (int x = 16; x; x >>= 1) best = min(best, __shfl_xor_sync(0xFFFFFFFFu, best, x));
    for (uint64_t j = lane; j < k; j += 32)
        if (lo + j >= nfit) { o[j] = YK_NONE_U32; o[k + j] = 0; }
    if (lane == 0) {
        o[2 * (size_t)k] = (uint32_t)nfit;
        o[2 * (size_t)k + 1] = best == ~0ull ? YK_NONE_U32 : g_node[(uint32_t)best];
        o[2 * (size_t)k + 2] = best == ~0ull ? 0u : (uint32_t)(best >> 32);
    }
}
