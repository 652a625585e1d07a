// yk_kernels.cuh -- sm_90a device code of the scheduling-cycle engine.
//
// Data layout in HBM (DESIGN.md "layout"): everything is structure-of-arrays, column-major.
//   node table (node-index space, resident):  total[D][ldn] i64, avail[D][ldn] i64, taint[ldn] u64,
//                                             label[ldn] u64, flags[ldn] u32
//   ask table  (ask-index space, resident):   req[D][lda] i64, tol/need/deny[lda] u64, node[lda] u32
//   sorted view (rebuilt per batch):          cap[D][Np] i64, taint/label[Np] u64, node[Np] u32, key[Np] u64
//                                             position p = p-th node in ascending (score, NodeID) order
//   outputs per batch:                        fit[B][W+1] u32: W bitmap words (bit p of row i = ask i fits sorted node p)
//                                             + 1 word = lowest set position = the frozen-snapshot argmin
//
// The sweep is integer compare + reduce: no tensor cores (not a contraction).  The node tile lives in
// registers and is reused across the whole ask chunk; the ask chunk is staged once in shared memory and
// read back as warp-wide broadcasts.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "yk_score.h"

#define YK_NONE_U32 0xFFFFFFFFu
#define YK_SWEEP_THREADS 256

struct YkWeights { double w[8]; };

// ---- per-node sort key --------------------------------------------------------------------------------
// key_in[i] / val_in[i] for the i-th live node in NodeID-rank order; a stable sort by key then yields
// ascending (score, NodeID) -- the order of the core's node btree (SURVEY A.3).
__global__ void yk_key_kernel(int D, uint32_t policy, YkWeights w, const int64_t* __restrict__ total,
                              const int64_t* __restrict__ avail, size_t ldn, const uint32_t* __restrict__ by_rank,
                              int nlive, uint64_t* __restrict__ key_in, uint32_t* __restrict__ val_in,
                              int* __restrict__ nan_flag) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nlive) return;
    uint32_t n = by_rank[i];
    double s = yk_node_score(D, policy, w.w, total + n, avail + n, ldn);
    uint64_t k = yk_key_bits(s);
    if (k == YK_KEY_NAN) atomicExch(nan_flag, 1);
    key_in[i] = k;
    val_in[i] = n;
}

__global__ void yk_score_kernel(int D, uint32_t policy, YkWeights w, const int64_t* __restrict__ total,
                                const int64_t* __restrict__ avail, size_t ldn, const uint32_t* __restrict__ idx,
                                int n, double* __restrict__ out) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t node = idx[i];
    out[i] = yk_node_score(D, policy, w.w, total + node, avail + node, ldn);
}

// ---- sorted view ---------------------------------------------------------------------------------------
// cap_k = min(max(0,total_k), max(0,avail_k)) folds the core's FitInNode(total) and preAllocateCheck
// available.FitIn (FitIn clamps negatives to 0, SURVEY A.2) and the shim's NodeResourcesFit into ONE
// compare per dimension; cap = -1 on every dimension for nodes that are unschedulable, reserved or padding,
// so no request (requests are >= 0 by the time they reach the sweep) can fit them.
__global__ void yk_gather_kernel(int D, const int64_t* __restrict__ total, const int64_t* __restrict__ avail,
                                 size_t ldn, const uint64_t* __restrict__ taint, const uint64_t* __restrict__ label,
                                 const uint32_t* __restrict__ flags, const uint32_t* __restrict__ sorted_node,
                                 int nlive, int Np, int64_t* __restrict__ s_cap, uint64_t* __restrict__ s_taint,
                                 uint64_t* __restrict__ s_label, uint32_t* __restrict__ s_node) {
    int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= Np) return;
    if (p < nlive) {
        uint32_t n = sorted_node[p];
        bool usable = (flags[n] & 1u) && !(flags[n] & 2u);
        for (int k = 0; k < D; ++k) {
            int64_t t = total[(size_t)k * ldn + n], a = avail[(size_t)k * ldn + n];
            t = t < 0 ? 0 : t;
            a = a < 0 ? 0 : a;
            s_cap[(size_t)k * Np + p] = usable ? (a < t ? a : t) : -1;
        }
        s_taint[p] = taint[n];
        s_label[p] = label[n];
        s_node[p] = n;
    } else {
        for (int k = 0; k < D; ++k) s_cap[(size_t)k * Np + p] = -1;
        s_taint[p] = ~0ull;
        s_label[p] = 0;
        s_node[p] = YK_NONE_U32;
    }
}

// ---- the fused sweep: resource fit + taint/affinity masks + node name + first-fit argmin ---------------
struct YkSweepArgs {
    // sorted node view
    const int64_t* s_cap;     // [D][Np]
    const uint64_t* s_taint;  // [Np]
    const uint64_t* s_label;  // [Np]
    const uint32_t* s_node;   // [Np]
    int Np;                   // multiple of YK_SWEEP_THREADS * NPT
    // ask table + batch order
    const int64_t* a_req;     // [D][lda]
    const uint64_t* a_tol;
    const uint64_t* a_need;
    const uint64_t* a_deny;
    const uint32_t* a_node;
    size_t lda;
    const uint32_t* batch;    // [B] ask indices in commit order
    int row0, rows;           // this launch handles batch rows [row0, row0+rows)
    int per;                  // rows per CTA along grid.y (multiple of 32)
    // outputs
    uint32_t* fit;            // [B][WS]: W bitmap words, then word W = first fit position (pre-set to YK_NONE_U32)
    int W;                    // bitmap words per row = Np/32
    int WS;                   // row stride in words (W + 1): one row = one exchange / read-back unit
    // multi-GPU, peer-to-peer: every rank's fit buffer for this slot (IPC-mapped over NVLink, own pointer included).
    // n_peer == 0: single GPU (or NCCL exchange): write `fit` only.  Otherwise the kernel stores its rows straight into
    // every rank's buffer -- the all-gather is fused into the sweep, tile by tile, no separate collective launch.
    uint32_t* fit_peer[8];
    int n_peer;
};

struct YkPeerFit { uint32_t* fit[8]; };

// One (ask, 32 x NPT nodes) step.  MASKS / WANT are warp-uniform properties of the ask (staged in shared
// memory as `kind`): an ask without tolerations, selectors or a node name needs no mask work at all -- a node
// passes its mask test iff it carries no taint, which is a per-node constant hoisted out of the loop.
template <int D, int NPT, bool MASKS, bool WANT>
__device__ __forceinline__ void yk_pair_step(const int64_t (&cap)[NPT][D], const uint64_t (&ntaint)[NPT],
                                             const uint64_t (&nlabel)[NPT], const uint32_t (&nidx)[NPT],
                                             const bool (&taintfree)[NPT], const int64_t (&rq)[D], uint64_t tol,
                                             uint64_t need, uint64_t deny, uint32_t want, uint32_t (&word)[NPT]) {
#pragma unroll
    for (int j = 0; j < NPT; ++j) {
        bool ok = true;
#pragma unroll
        for (int k = 0; k < D; ++k) ok = ok && (rq[k] <= cap[j][k]);
        if (MASKS) {
            const uint64_t bad = (ntaint[j] & ~tol) | (~nlabel[j] & need) | (nlabel[j] & deny);
            ok = ok && (bad == 0ull);
        } else {
            ok = ok && taintfree[j];
        }
        if (WANT) ok = ok && (want == nidx[j]);
        word[j] = __ballot_sync(0xFFFFFFFFu, ok);
    }
}

// grid.x = node tiles of YK_SWEEP_THREADS*NPT sorted positions; grid.y = ask splits.  A CTA keeps its node tile
// in registers and walks its share of the batch rows in sub-chunks of AC asks staged in shared memory, so the
// host can size grid.y to fill the machine exactly once (no tail wave) whatever the batch size.
template <int D, int NPT, int AC>
__global__ void __launch_bounds__(YK_SWEEP_THREADS, NPT <= 2 ? 4 : 2) yk_sweep_kernel(const YkSweepArgs p) {
    __shared__ int64_t sh_req[AC][D];
    __shared__ uint64_t sh_mask[AC][3];
    __shared__ uint32_t sh_node[AC];
    __shared__ uint32_t sh_kind[AC];
    constexpr int TW = YK_SWEEP_THREADS / 32 * NPT;   // bitmap words this CTA produces per ask (its node tile / 32)
    __shared__ uint32_t sh_word[32][TW];              // [ask in group][word in tile]: a row's words sit together

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    // node tile -> registers (coalesced column reads: consecutive lanes = consecutive positions)
    int64_t cap[NPT][D];
    uint64_t ntaint[NPT], nlabel[NPT];
    uint32_t nidx[NPT];
    bool taintfree[NPT];
    const int pos0 = blockIdx.x * (YK_SWEEP_THREADS * NPT) + tid;
#pragma unroll
    for (int j = 0; j < NPT; ++j) {
        const int pos = pos0 + j * YK_SWEEP_THREADS;
#pragma unroll
        for (int k = 0; k < D; ++k) cap[j][k] = __ldg(p.s_cap + (size_t)k * p.Np + pos);
        ntaint[j] = __ldg(p.s_taint + pos);
        nlabel[j] = __ldg(p.s_label + pos);
        nidx[j] = __ldg(p.s_node + pos);
        taintfree[j] = ntaint[j] == 0ull;
    }
    const int tile_word0 = blockIdx.x * TW;   // first bitmap word of this CTA's tile

    // this CTA's rows: [r_begin, r_end)
    const int r_begin = p.row0 + (int)blockIdx.y * p.per;
    const int r_end = min(p.row0 + p.rows, r_begin + p.per);

    for (int a0 = r_begin; a0 < r_end; a0 += AC) {
        const int na = min(AC, r_end - a0);
        __syncthreads();   // previous sub-chunk fully consumed
        for (int i = tid; i < AC; i += YK_SWEEP_THREADS) {
            uint32_t kind = 0;
            if (i < na) {
                const uint32_t a = p.batch[a0 + i];
#pragma unroll
                for (int k = 0; k < D; ++k) sh_req[i][k] = p.a_req[(size_t)k * p.lda + a];
                const uint64_t tol = p.a_tol[a], need = p.a_need[a], deny = p.a_deny[a];
                const uint32_t want = p.a_node[a];
                sh_mask[i][0] = tol; sh_mask[i][1] = need; sh_mask[i][2] = deny;
                sh_node[i] = want;
                kind = ((tol | need | deny) != 0ull ? 1u : 0u) | (want != YK_NONE_U32 ? 2u : 0u);
            } else {   // rows past the end can never fit
#pragma unroll
                for (int k = 0; k < D; ++k) sh_req[i][k] = INT64_MAX;
                sh_mask[i][0] = 0; sh_mask[i][1] = ~0ull; sh_mask[i][2] = ~0ull; sh_node[i] = YK_NONE_U32;
                kind = 1u;
            }
            sh_kind[i] = kind;
        }
        __syncthreads();

        for (int ab = 0; ab < na; ab += 32) {
            const int nl = min(32, na - ab);
#pragma unroll 4
            for (int l = 0; l < nl; ++l) {
                const int i = ab + l;
                int64_t rq[D];
#pragma unroll
                for (int k = 0; k < D; ++k) rq[k] = sh_req[i][k];
                const uint32_t kind = sh_kind[i];
                uint32_t word[NPT];
                if (kind == 0u) {
                    yk_pair_step<D, NPT, false, false>(cap, ntaint, nlabel, nidx, taintfree, rq, 0, 0, 0, 0, word);
                } else {
                    const uint64_t tol = sh_mask[i][0], need = sh_mask[i][1], deny = sh_mask[i][2];
                    const uint32_t want = sh_node[i];
                    if (kind & 2u) yk_pair_step<D, NPT, true, true>(cap, ntaint, nlabel, nidx, taintfree, rq, tol, need, deny, want, word);
                    else yk_pair_step<D, NPT, true, false>(cap, ntaint, nlabel, nidx, taintfree, rq, tol, need, deny, want, word);
                }
                // park the ballot words in shared memory (LSU pipe) instead of select-chains on the ALU pipe; word
                // j of warp w is tile word w + j*8, so the TW words of one ask end up contiguous
                if (lane == 0) {
#pragma unroll
                    for (int j = 0; j < NPT; ++j) sh_word[l][warp + j * (YK_SWEEP_THREADS / 32)] = word[j];
                }
            }
            __syncthreads();
            // cooperative store: TW consecutive threads write the TW consecutive words of one row (64-byte segments
            // at TW = 16) -- to the local buffer, or straight into every rank's buffer over NVLink
            for (int t = tid; t < nl * TW; t += YK_SWEEP_THREADS) {
                const int l = t / TW, wv = t % TW;
                const uint32_t w = sh_word[l][wv];
                const size_t off = (size_t)(a0 + ab + l) * p.WS + (size_t)(tile_word0 + wv);
                if (p.n_peer == 0) p.fit[off] = w;
                else for (int g = 0; g < p.n_peer; ++g) p.fit_peer[g][off] = w;
                if (wv == 0) {   // one thread per row: first fit position inside this tile, folded into the row's last word
                    uint32_t best = YK_NONE_U32;
                    for (int x = 0; x < TW; ++x) {
                        const uint32_t wx = sh_word[l][x];
                        if (wx) { best = (uint32_t)(tile_word0 + x) * 32u + (uint32_t)(__ffs((int)wx) - 1); break; }
                    }
                    // always the LOCAL buffer: the owner of the rows publishes the final value to the peers afterwards
                    if (best != YK_NONE_U32) atomicMin(&p.fit[(size_t)(a0 + ab + l) * p.WS + p.W], best);
                }
            }
            __syncthreads();
        }
    }
}

// multi-GPU, peer-to-peer: after the sweep the first-fit words of this rank's rows are final in the local buffer;
// copy them into every other rank's buffer (the bitmap words went there directly from the sweep)
__global__ void yk_p2p_first_kernel(const uint32_t* __restrict__ local, YkPeerFit pf, int n_peer, int self, int row0,
                                    int rows, int W, int WS) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows) return;
    const size_t off = (size_t)(row0 + i) * WS + W;
    const uint32_t v = local[off];
    for (int g = 0; g < n_peer; ++g) if (g != self) pf.fit[g][off] = v;
}

// ---- one (ask,node) answer in the reference's step order, on the device --------------------------------
// order: core tryNodes (schedulable, FitInNode total) -> tryNode preAllocateCheck (request > 0, available)
// -> shim Predicates: NodeName, TaintToleration/NodeUnschedulable, NodeAffinity, NodeResourcesFit
// (predicate_manager.go:339-351 filter order).  The one place that order is written down: yk_evaluate_kernel and
// yk_filter_kernel (yk_filter.cuh) both call it.  fit_total / fit_avail: request <= max(0, total / available) in every
// dimension; req_ok: no request below zero and at least one above.  Returns 0 (fits) or YK_FAIL_NODE_NOT_SCHEDULABLE ..
// YK_FAIL_AFFINITY.
__host__ __device__ __forceinline__ int yk_first_fail(bool schedulable, bool fit_total, bool req_ok, bool fit_avail,
                                                      uint32_t want, uint32_t node, uint64_t taint, uint64_t label,
                                                      uint64_t tol, uint64_t need, uint64_t deny, int allocate) {
    if (!schedulable) return 1;
    if (!fit_total) return 2;
    if (!req_ok) return 3;
    if (allocate && !fit_avail) return 4;   // reservation phase (Allocate = false): no NodeResourcesFit, no available check
    if (want != YK_NONE_U32 && want != node) return 5;
    if (taint & ~tol) return 6;
    if ((label & need) != need || (label & deny)) return 7;
    return 0;
}

__global__ void yk_evaluate_kernel(int D, const int64_t* __restrict__ total, const int64_t* __restrict__ avail,
                                   size_t ldn, const uint64_t* __restrict__ taint, const uint64_t* __restrict__ label,
                                   const uint32_t* __restrict__ flags, const int64_t* __restrict__ a_req,
                                   const uint64_t* __restrict__ a_tol, const uint64_t* __restrict__ a_need,
                                   const uint64_t* __restrict__ a_deny, const uint32_t* __restrict__ a_node, size_t lda,
                                   uint32_t ask, uint32_t node, int allocate, int* __restrict__ out) {
    if (threadIdx.x || blockIdx.x) return;
    bool pos = false, neg = false, fit_total = true, fit_avail = true;
    for (int k = 0; k < D; ++k) {
        int64_t q = a_req[(size_t)k * lda + ask];
        int64_t t = total[(size_t)k * ldn + node], a = avail[(size_t)k * ldn + node];
        if (q < 0) neg = true;
        if (q > 0) pos = true;
        if (q > (t < 0 ? 0 : t)) fit_total = false;
        if (q > (a < 0 ? 0 : a)) fit_avail = false;
    }
    *out = yk_first_fail((flags[node] & 1u) != 0, fit_total, pos && !neg, fit_avail, a_node[ask], node, taint[node],
                         label[node], a_tol[ask], a_need[ask], a_deny[ask], allocate);
}

// ---- preemption victim search (predicate_manager.go:137-175), one warp per query ---------------------
// Query q: does ask[q] fit node[q] once victims voff[q]..voff[q+1] are removed in order up to index i, for the
// smallest i >= start[q]?  The victims before start are always removed.  Static predicates (the reference's
// PreFilter + non-resource Filters) do not depend on the victims: if they fail the answer is -1.  The resource
// part is a prefix sum of what the victims give back: warp-wide inclusive scan per dimension, 32 victims a step.
__global__ void yk_preempt_kernel(int D, const int64_t* __restrict__ total, const int64_t* __restrict__ avail, size_t ldn,
                                  const uint64_t* __restrict__ taint, const uint64_t* __restrict__ label,
                                  const uint32_t* __restrict__ flags, const int64_t* __restrict__ a_req,
                                  const uint64_t* __restrict__ a_tol, const uint64_t* __restrict__ a_need,
                                  const uint64_t* __restrict__ a_deny, const uint32_t* __restrict__ a_node, size_t lda,
                                  int nq, const uint32_t* __restrict__ q_ask, const uint32_t* __restrict__ q_node,
                                  const uint32_t* __restrict__ voff, const int64_t* __restrict__ vreq, size_t ldv,
                                  const uint32_t* __restrict__ start, int32_t* __restrict__ out) {
    const int q = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= nq) return;
    const uint32_t ask = q_ask[q], node = q_node[q];
    bool stat = (flags[node] & 1u) != 0;
    stat = stat && !(a_node[ask] != YK_NONE_U32 && a_node[ask] != node);
    stat = stat && !(taint[node] & ~a_tol[ask]);
    stat = stat && (label[node] & a_need[ask]) == a_need[ask] && !(label[node] & a_deny[ask]);
    int64_t rq[8], carry[8];
    bool pos = false;
    for (int k = 0; k < D; ++k) {
        rq[k] = a_req[(size_t)k * lda + ask];
        const int64_t t = total[(size_t)k * ldn + node];
        carry[k] = avail[(size_t)k * ldn + node];
        if (rq[k] < 0 || rq[k] > (t < 0 ? 0 : t)) stat = false;
        if (rq[k] > 0) pos = true;
    }
    stat = stat && pos;
    const uint32_t v0 = voff[q], v1 = voff[q + 1], st = start[q];
    int32_t answer = -1;
    for (uint32_t base = v0; stat && base < v1 && answer < 0; base += 32) {
        const uint32_t v = base + (uint32_t)lane;
        bool fit = v < v1;
        for (int k = 0; k < D; ++k) {
            int64_t x = (v < v1) ? vreq[(size_t)k * ldv + v] : 0;
#pragma unroll
            for (int off = 1; off < 32; off <<= 1) {   // inclusive scan
                const int64_t y = __shfl_up_sync(0xFFFFFFFFu, x, off);
                if (lane >= off) x += y;
            }
            const int64_t have = carry[k] + x;
            fit = fit && rq[k] <= (have < 0 ? 0 : have);
            carry[k] += __shfl_sync(0xFFFFFFFFu, x, 31);
        }
        fit = fit && (v - v0) >= st;
        const uint32_t m = __ballot_sync(0xFFFFFFFFu, fit);
        if (m) answer = (int32_t)(base - v0) + (__ffs((int)m) - 1);
    }
    if (lane == 0) out[q] = answer;
}

// ---- peer-to-peer flags (multi-GPU): "rows ready" / "slot consumed" sequence numbers in every rank's sync block ----
struct YkPeerSync { uint32_t* sync[8]; };

// one thread per rank: publish `value` at word `offset` of every rank's sync block (after all earlier writes of this
// stream -- the sweep's peer stores -- are visible system-wide)
__global__ void yk_p2p_signal_kernel(YkPeerSync ps, int world, int offset, uint32_t value) {
    const int g = threadIdx.x;
    if (g >= world) return;
    __threadfence_system();
    volatile uint32_t* q = ps.sync[g] + offset;
    *q = value;
}
// one thread per rank: spin until word base+g of MY sync block has reached `value` (sequence compare), bounded
__global__ void yk_p2p_wait_kernel(volatile uint32_t* my_sync, int world, int base, uint32_t value, int* err,
                                   long long max_cycles) {
    const int g = threadIdx.x;
    if (g >= world) return;
    const long long t0 = clock64();
    while ((int32_t)(my_sync[base + g] - value) < 0) {
        if (clock64() - t0 > max_cycles) { atomicExch(err, 2); break; }
        __nanosleep(200);
    }
    __threadfence_system();
}

// scatter new availability for a list of nodes (after the ordered commit)
__global__ void yk_apply_avail_kernel(int D, int64_t* __restrict__ avail, size_t ldn, const uint32_t* __restrict__ nodes,
                                      const int64_t* __restrict__ vals /*[D][n]*/, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t node = nodes[i];
    for (int k = 0; k < D; ++k) avail[(size_t)k * ldn + node] = vals[(size_t)k * n + i];
}

__global__ void yk_fill_u32_kernel(uint32_t* __restrict__ p, uint32_t v, int n) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) p[i] = v;
}
