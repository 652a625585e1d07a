// yk_uniform.cuh -- sm_90a kernels of the uniform-run commit (algorithm and per-item bodies: yk_uniform.h).  Grid-wide,
// one thread per node / per ask; the two sorts between them are cub::DeviceRadixSort (stable).  Integer compares, one
// 64-bit divide per node and dimension, float64 re-scores: no tensor cores, a few hundred KB of traffic per run.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "yk_uniform.h"

namespace ykun {

__device__ __forceinline__ unsigned long long warp_min64(unsigned long long v) {
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long x = __shfl_xor_sync(0xFFFFFFFFu, v, o); v = x < v ? x : v; }
    return v;
}

__global__ void un_reset_kernel(Globals* g) {
    g->bkey = KEY_INF; g->brank = KEY_INF; g->last_key = 0; g->last_rank = 0; g->valid = 0; g->nan = 0; g->status = U_RETRY; g->consumed = 0;
}

template <int D>
__global__ void __launch_bounds__(256) un_depth_kernel(const Args a) {
    const long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one thread per (node, depth) element
    DepthOut o; o.valid = 0; o.bk = KEY_INF; o.nan = 0;
    if (x < (long long)a.nlive * a.L) o = element_item<D>(a, x);
    const unsigned v = __reduce_add_sync(0xFFFFFFFFu, o.valid);
    const unsigned long long b = warp_min64(o.bk);
    const unsigned nn = __ballot_sync(0xFFFFFFFFu, o.nan != 0);
    if ((threadIdx.x & 31) == 0) {
        if (v) atomicAdd(&a.g->valid, v);
        if (b != KEY_INF) atomicMin(&a.g->bkey, b);
        if (nn) a.g->nan = 1;
    }
}

template <int D>
__global__ void __launch_bounds__(256) un_brank_kernel(const Args a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned long long bkey = a.g->bkey;
    if (bkey == KEY_INF) return;   // uniform: whole grid
    unsigned long long r = i < a.nlive ? brank_item<D>(a, i, bkey) : KEY_INF;
    r = warp_min64(r);
    if ((threadIdx.x & 31) == 0 && r != KEY_INF) atomicMin(&a.g->brank, r);
}

template <int D>
__global__ void __launch_bounds__(256) un_select_kernel(const Args a) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < a.R) select_item<D>(a, q, a.g->valid);
}

__global__ void un_decide_kernel(const Args a) { decide(a); }

template <int D>
__global__ void __launch_bounds__(256) un_apply_rekey_kernel(const Args a) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.nlive) return;
    apply_item<D>(a, i, a.g->status);
    if (rekey_item<D>(a, i)) a.g->nan = 2;   // a NaN score AFTER the commit (status stays: the host reports it)
}

// the binpacking fill (yk_uniform.h): un_depth_kernel at L = 1, a radix sort, then these three around a cub inclusive scan
template <int D>
__global__ void __launch_bounds__(256) un_fill_cap_kernel(const Args a) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < a.nlive) fill_cap_item<D>(a, p);
}

__global__ void un_fill_decide_kernel(const Args a) { fill_decide(a); }

__global__ void __launch_bounds__(256) un_fill_select_kernel(const Args a) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < a.R) fill_select_item(a, q, a.g->valid);
}

__global__ void un_order_kernel(const Args a) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= a.nlive) return;
    yklt::Ent e; e.key = a.okey[p]; e.rn = a.orn[p];
    a.ord[*a.cur & 1][p] = e;
}

}  // namespace ykun
