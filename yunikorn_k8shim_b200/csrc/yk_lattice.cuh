// yk_lattice.cuh -- sm_90a kernels of the device-resident ordered commit.  The algorithm is in yk_lattice.h (single
// source with the CPU test emulation); this file wraps it into a persistent one-CTA kernel and adds the two small
// kernels that move the engine's column-major node tables into / out of the lattice's per-node records.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "yk_lattice.h"

// One CTA of 1024 threads owns the batch: the commit is a chain of sub-runs whose phases are separated by CTA barriers
// (a grid-wide barrier would cost more than the work between two of them); everything the phases share lives in the
// ~200 KB of dynamic shared memory this kernel asks for.  Integer compare / bit arithmetic + float64 re-scores: no
// tensor cores.
template <int D>
__global__ void __launch_bounds__(yklt::THREADS, 1) yk_lattice_kernel(const yklt::Args a) {
    extern __shared__ __align__(16) unsigned char yk_lt_smem[];
    yklt::Shared<D>& s = *reinterpret_cast<yklt::Shared<D>*>(yk_lt_smem);
    yklt::lattice_batch<D>(a, s);
}

// node records + the cycle's initial order from what the key kernel and the stable radix sort produced (yklt::init_node)
__global__ void yk_lt_init_kernel(int D, const int64_t* __restrict__ total, const int64_t* __restrict__ avail, size_t ldn,
                                  const uint64_t* __restrict__ taint, const uint64_t* __restrict__ label,
                                  const uint32_t* __restrict__ flags, const uint32_t* __restrict__ rank,
                                  const uint64_t* __restrict__ sorted_key, const uint32_t* __restrict__ sorted_node, int nlive,
                                  int64_t* __restrict__ rec, int RS, yklt::Ent* __restrict__ ord) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= nlive) return;
    yklt::init_node(D, p, total, avail, ldn, taint, label, flags, rank, sorted_key, sorted_node, rec, RS, ord);
}

// available of every live node back into the column-major table (position order = any order: each node once)
__global__ void yk_lt_export_kernel(int D, const int64_t* __restrict__ rec, int RS, const yklt::Ent* __restrict__ ord, int nlive,
                                    int64_t* __restrict__ avail, size_t ldn) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= nlive) return;
    const uint32_t n = (uint32_t)ord[p].rn;
    const int64_t* r = rec + (size_t)n * RS;
    for (int k = 0; k < D; ++k) avail[(size_t)k * ldn + n] = r[k];
}
