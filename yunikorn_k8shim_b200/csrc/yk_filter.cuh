// yk_filter.cuh -- sm_90a device code of yk_filter_nodes: every (ask, node) pair of a list of asks, in the cycle's node order.
//
// Node order: yk_key_kernel + radix sort over live nodes by NodeID rank (the cycle's device_order), kept in the filter's own
// buffers.  Then two kernels per chunk of asks:
//   yk_filter_kernel<D>        grid.x = node tiles of YK_FILTER_THREADS sorted positions, grid.y = ask splits.  A thread holds
//                              one node's columns in registers, the CTA stages AC asks at a time in shared memory.  Per pair:
//                              its slot (0 = passes, YK_FAIL_* of yk_evaluate, 9 = ask absent, 10 = node reserved), by
//                              yk_first_fail, the step order yk_evaluate_kernel uses.  Per (ask, warp): one ballot = one pass
//                              bitmap word.  Per (ask, CTA): the slot histogram, reduced in shared memory (warp-aggregated by
//                              __match_any_sync), added to the ask's global counts once per non-zero slot; its slot-0 entry is
//                              the tile's pass count.
//   yk_filter_compact_kernel   one warp per ask: exclusive scan over the tile pass counts, then only the tiles that hold pass
//                              ranks [skip, skip + k) are opened and their set bits turned into node indices.
// Only the counts [rows][11] and the window [rows][k] are read back.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "yk_kernels.cuh"

#define YK_FILTER_THREADS 256
#define YK_FILTER_NSLOT 11        // YK_FILTER_SLOTS
#define YK_FILTER_ABSENT 9        // YK_FAIL_ABSENT
#define YK_FILTER_RES 10          // YK_FILTER_RESERVED
#define YK_FILTER_TW (YK_FILTER_THREADS / 32)   // bitmap words per node tile

struct YkFilterArgs {
    const int64_t* total;     // [D][ldn] node table (node-index space)
    const int64_t* avail;
    size_t ldn;
    const uint64_t* taint;
    const uint64_t* label;
    const uint32_t* flags;
    const uint32_t* sorted;   // [nlive]: node index at each position of the cycle's order
    int nlive;
    const int64_t* a_req;     // [D][lda] ask table
    const uint64_t* a_tol;
    const uint64_t* a_need;
    const uint64_t* a_deny;
    const uint32_t* a_node;
    size_t lda;
    const uint32_t* asks;     // [rows]: ask index, YK_NONE_U32 = not present
    int rows, per;            // this launch's asks; asks per CTA along grid.y
    int allocate;             // 1: Predicates(Allocate = true), 0: the reservation phase
    uint32_t* bits;           // [rows][W]: bit p of row i = ask i passes the node at position p
    uint32_t* tilecnt;        // [rows][tiles]: passing nodes per tile
    uint32_t* counts;         // [rows][YK_FILTER_NSLOT], zeroed before the launch
    int W, tiles;             // W = tiles * YK_FILTER_TW
};

template <int D, int AC>
__global__ void __launch_bounds__(YK_FILTER_THREADS) yk_filter_kernel(const YkFilterArgs p) {
    __shared__ int64_t sh_req[AC][D];
    __shared__ uint64_t sh_mask[AC][3];
    __shared__ uint32_t sh_want[AC];
    __shared__ uint32_t sh_kind[AC];          // bit 0: ask present, bit 1: requests valid (none < 0, one > 0)
    __shared__ uint32_t sh_hist[AC][YK_FILTER_NSLOT];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int pos = blockIdx.x * YK_FILTER_THREADS + tid;
    const bool live = pos < p.nlive;

    // this thread's node -> registers, clamped at zero as FitIn does
    int64_t tot[D], av[D];
    uint64_t taint = 0, label = 0;
    uint32_t node = YK_NONE_U32, fl = 0;
    if (live) {
        node = __ldg(p.sorted + pos);
        taint = __ldg(p.taint + node);
        label = __ldg(p.label + node);
        fl = __ldg(p.flags + node);
    }
#pragma unroll
    for (int k = 0; k < D; ++k) {
        const int64_t t = live ? __ldg(p.total + (size_t)k * p.ldn + node) : 0;
        const int64_t a = live ? __ldg(p.avail + (size_t)k * p.ldn + node) : 0;
        tot[k] = t < 0 ? 0 : t;
        av[k] = a < 0 ? 0 : a;
    }
    const bool schedulable = (fl & 1u) != 0, reserved = (fl & 2u) != 0;

    const int r_begin = (int)blockIdx.y * p.per;
    const int r_end = min(p.rows, r_begin + p.per);
    for (int a0 = r_begin; a0 < r_end; a0 += AC) {
        const int na = min(AC, r_end - a0);
        __syncthreads();   // previous sub-chunk's histogram flushed
        for (int i = tid; i < na; i += YK_FILTER_THREADS) {
            const uint32_t a = p.asks[a0 + i];
            uint32_t kind = 0;
            if (a != YK_NONE_U32) {
                bool neg = false, any = false;
#pragma unroll
                for (int k = 0; k < D; ++k) {
                    const int64_t q = p.a_req[(size_t)k * p.lda + a];
                    sh_req[i][k] = q;
                    neg = neg || q < 0;
                    any = any || q > 0;
                }
                sh_mask[i][0] = p.a_tol[a]; sh_mask[i][1] = p.a_need[a]; sh_mask[i][2] = p.a_deny[a];
                sh_want[i] = p.a_node[a];
                kind = 1u | ((any && !neg) ? 2u : 0u);
            }
            sh_kind[i] = kind;
        }
        for (int t = tid; t < na * YK_FILTER_NSLOT; t += YK_FILTER_THREADS) (&sh_hist[0][0])[t] = 0;
        __syncthreads();

        for (int i = 0; i < na; ++i) {
            const uint32_t kind = sh_kind[i];
            int slot;
            if (!(kind & 1u)) {
                slot = YK_FILTER_ABSENT;
            } else if (reserved) {
                slot = YK_FILTER_RES;
            } else {
                bool fit_total = true, fit_avail = true;
#pragma unroll
                for (int k = 0; k < D; ++k) {
                    const int64_t q = sh_req[i][k];
                    fit_total = fit_total && q <= tot[k];
                    fit_avail = fit_avail && q <= av[k];
                }
                slot = yk_first_fail(schedulable, fit_total, (kind & 2u) != 0, fit_avail, sh_want[i], node, taint, label,
                                     sh_mask[i][0], sh_mask[i][1], sh_mask[i][2], p.allocate);
            }
            const uint32_t pass = __ballot_sync(0xFFFFFFFFu, live && slot == 0);
            if (lane == 0) p.bits[(size_t)(a0 + i) * p.W + (size_t)blockIdx.x * YK_FILTER_TW + warp] = pass;
            // one shared atomic per distinct slot in the warp, by the lowest lane holding it
            const uint32_t same = __match_any_sync(0xFFFFFFFFu, live ? slot : -1);
            if (live && lane == __ffs((int)same) - 1) atomicAdd(&sh_hist[i][slot], (uint32_t)__popc(same));
        }
        __syncthreads();
        for (int t = tid; t < na * YK_FILTER_NSLOT; t += YK_FILTER_THREADS) {
            const int i = t / YK_FILTER_NSLOT, s = t % YK_FILTER_NSLOT;
            const uint32_t v = sh_hist[i][s];
            if (s == 0) p.tilecnt[(size_t)(a0 + i) * p.tiles + blockIdx.x] = v;
            if (v) atomicAdd(&p.counts[(size_t)(a0 + i) * YK_FILTER_NSLOT + s], v);
        }
    }
}

// one warp per ask: out[r][j] = node of pass rank skip + j, YK_NONE_U32 past the last passing node
__global__ void yk_filter_compact_kernel(const uint32_t* __restrict__ bits, const uint32_t* __restrict__ tilecnt,
                                         const uint32_t* __restrict__ counts, const uint32_t* __restrict__ sorted, int rows,
                                         int W, int tiles, uint32_t skip, uint32_t k, uint32_t* __restrict__ out) {
    const int r = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (r >= rows) return;
    const uint32_t* tc = tilecnt + (size_t)r * tiles;
    const uint32_t* bw = bits + (size_t)r * W;
    uint32_t* o = out + (size_t)r * k;
    const uint64_t lo = skip, hi = (uint64_t)skip + k;
    const uint64_t npass = counts[(size_t)r * YK_FILTER_NSLOT];
    for (uint64_t j = lane; j < k; j += 32)
        if (lo + j >= npass) o[j] = YK_NONE_U32;
    uint64_t base = 0;   // pass ranks before tile t0
    for (int t0 = 0; t0 < tiles && base < hi && base < npass; t0 += 32) {
        const int t = t0 + lane;
        const uint32_t c = t < tiles ? tc[t] : 0u;
        uint32_t incl = c;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, off);
            if (lane >= off) incl += y;
        }
        const uint64_t first = base + incl - c;   // pass rank of tile t's first passing node
        uint32_t m = __ballot_sync(0xFFFFFFFFu, c != 0 && first < hi && first + c > lo);
        while (m) {
            const int src = __ffs((int)m) - 1;
            m &= m - 1;
            uint64_t rb = __shfl_sync(0xFFFFFFFFu, first, src);
            const int tile = t0 + src;
            for (int w = 0; w < YK_FILTER_TW && rb < hi; ++w) {
                const int wi = tile * YK_FILTER_TW + w;
                const uint32_t word = bw[wi];
                const uint64_t rank = rb + (uint64_t)__popc(word & ((1u << lane) - 1u));
                if (((word >> lane) & 1u) && rank >= lo && rank < hi) o[rank - lo] = sorted[(size_t)wi * 32 + lane];
                rb += (uint64_t)__popc(word);
            }
        }
        base += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
}
