// yk_spec.cuh -- sm_90a kernels of the speculative static order (rules: yk_spec.h).  The radix sorts between them are
// cub's; csrc/yk_engine.cu (spec_launch) strings them together on the engine's stream.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "yk_spec.h"

// One thread per ask, live node and application (grid over the largest of the three): the first sort's keys and values,
// the reductions of the screen (kept count, non-plain asks, untolerated bits, priority range, live taints), and the
// application sort's keys and values.  w[] holds its initial words (spec_launch).
__global__ void yk_spec_scan_kernel(uint32_t a_hi, const uint8_t* state, const uint32_t* app, const int64_t* create,
                                    const int32_t* prio, const uint32_t* gang, const uint8_t* cause, const uint64_t* tol,
                                    const uint64_t* need, const uint64_t* deny, const uint32_t* node, const uint8_t* present,
                                    uint32_t maxP, const int64_t* submit, uint32_t nlive, const uint32_t* by_rank,
                                    const uint64_t* taint, uint64_t* ckey, uint32_t* cval, uint64_t* pkey, uint32_t* pval,
                                    uint32_t* w) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned full = 0xFFFFFFFFu;
    const bool lane0 = (threadIdx.x & 31) == 0;
    bool k = false, bad = false;
    uint64_t nt = 0, tn = 0;
    uint32_t pmin = 0xFFFFFFFFu, pmax = 0;
    if (i < a_hi) {
        const uint32_t p = app[i];
        k = ykspec::kept(state[i], p < maxP ? present[p] : 0, cause[i]);
        ckey[i] = ykspec::time_key(create[i]);
        cval[i] = i;
        if (k) {
            bad = !ykspec::plain(gang[i], need[i], deny[i], node[i]);
            nt = ~tol[i];
            pmin = pmax = ykspec::prio_word(prio[i]);
        }
    }
    if (i < nlive) tn = taint[by_rank[i]];
    if (i < maxP) { pkey[i] = ykspec::time_key(submit[i]); pval[i] = i; }
    const uint32_t kb = __ballot_sync(full, k), bb = __ballot_sync(full, bad);
    const uint32_t ntl = __reduce_or_sync(full, (uint32_t)nt), nth = __reduce_or_sync(full, (uint32_t)(nt >> 32));
    const uint32_t tnl = __reduce_or_sync(full, (uint32_t)tn), tnh = __reduce_or_sync(full, (uint32_t)(tn >> 32));
    pmin = __reduce_min_sync(full, pmin); pmax = __reduce_max_sync(full, pmax);
    if (lane0) {
        if (kb) {
            atomicAdd(&w[ykspec::W_KEPT], (uint32_t)__popc(kb));
            atomicMin(&w[ykspec::W_PRIO_MIN], pmin); atomicMax(&w[ykspec::W_PRIO_MAX], pmax);
            if (ntl) atomicOr(&w[ykspec::W_NOTTOL_LO], ntl);
            if (nth) atomicOr(&w[ykspec::W_NOTTOL_HI], nth);
        }
        if (bb) atomicOr(&w[ykspec::W_BAD], 1u);
        if (tnl) atomicOr(&w[ykspec::W_TAINT_LO], tnl);
        if (tnh) atomicOr(&w[ykspec::W_TAINT_HI], tnh);
    }
}

// pos[app] = the application's position in the sorted order of the applications
__global__ void yk_spec_pos_kernel(uint32_t maxP, const uint32_t* sorted_apps, uint32_t* pos) {
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < maxP) pos[sorted_apps[j]] = j;
}

// the second sort's keys, for the asks in create order
__global__ void yk_spec_appkey_kernel(uint32_t a_hi, const uint32_t* by_create, const uint8_t* state, const uint32_t* app,
                                      const uint8_t* cause, const uint8_t* present, const uint32_t* pos, uint32_t maxP,
                                      uint32_t* key) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a_hi) return;
    const uint32_t a = by_create[i], p = app[a];
    const bool k = ykspec::kept(state[a], p < maxP ? present[p] : 0, cause[a]);
    key[i] = ykspec::app_key(k, k ? pos[p] : 0, maxP);
}

// over the stretch (its length from w): run breaks for the run test, and the order into mapped host memory for the host's
// element-for-element compare; zero breaks past the stretch
__global__ void yk_spec_break_kernel(uint32_t a_hi, const uint32_t* order, const uint32_t* sigid, const uint32_t* w,
                                     uint32_t max_bindings, uint32_t* brk, uint32_t* order_host) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a_hi) return;
    const uint32_t n = ykspec::stretch_len(w[ykspec::W_KEPT], max_bindings);
    if (i < n) { brk[i] = ykspec::run_break(order, sigid, (int)i); order_host[i] = order[i]; }
    else brk[i] = 0;
}

// run test over the inclusive sums of the breaks
__global__ void yk_spec_run_kernel(uint32_t a_hi, const uint32_t* brk, int un_min, uint32_t max_bindings, uint32_t* w) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a_hi) return;
    const uint32_t n = ykspec::stretch_len(w[ykspec::W_KEPT], max_bindings);
    if (ykspec::long_run_at(brk, (int)i, (int)n, un_min)) w[ykspec::W_RUN] = 1;
}

// one thread: the status word and the stretch length, on the device and in mapped host memory
__global__ void yk_spec_decide_kernel(uint32_t* w, uint32_t rd_min, uint32_t max_bindings, uint32_t* w_host) {
    ykspec::decide(w, rd_min, max_bindings);
    for (int k = 0; k < ykspec::W_N; ++k) w_host[k] = w[k];
}
