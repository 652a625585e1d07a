// yk_rounds.cuh -- sm_90a kernel of the round commit (algorithm and per-item bodies: yk_rounds.h).  One persistent CTA
// of 1024 threads decides a whole stretch, round after round, with CTA barriers only: a round is a few dozen barriers
// apart, and the node order and records it reads and rewrites (~1 MB at 10 000 nodes) stay in L2.  Integer compares and
// float64 re-scores: no tensor cores.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "yk_rounds.h"

template <int D>
__global__ void __launch_bounds__(yklt::THREADS, 1) yk_rounds_kernel(const ykrd::Args a) {
    extern __shared__ __align__(16) unsigned char yk_rd_smem[];
    ykrd::Shared& s = *reinterpret_cast<ykrd::Shared*>(yk_rd_smem);
    ykrd::rounds_stretch<D>(a, s);
}
