"""Build libykgpu.so in-tree for sm_90a, H100 (nvcc cross-compiles without a GPU)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libykgpu.so")
SOURCES = ["yk_engine.cu", "yk_dict.cpp", "yk_podres.cpp"]
DEPS = ["yk_engine.cu", "yk_dict.cpp", "yk_podres.cpp", "../../include/ykgpu_pod.h", "yk_kernels.cuh", "yk_filter.cuh", "yk_preempt_nodes.cuh", "yk_preempt_plan.cuh", "yk_preempt_required.cuh", "yk_lattice.cuh", "yk_lattice.h", "yk_uniform.cuh", "yk_uniform.h", "yk_rounds.cuh", "yk_rounds.h", "yk_spec.cuh", "yk_spec.h", "yk_lattice_host.hpp", "yk_orderer.hpp", "yk_dirty.hpp", "yk_commit.hpp", "yk_score.h", "../../include/ykgpu.h",
        "../../include/ykgpu_dict.h"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "--fmad=false",                 # float64 node score must not be contracted (SURVEY A.3)
] + (["-DYK_LT_THREADS=" + os.environ["YK_LT_THREADS"]] if os.environ.get("YK_LT_THREADS") else []) + \
    (["-DYK_NPT=" + os.environ["YK_NPT"]] if os.environ.get("YK_NPT") else []) + [
    "-Xcompiler", "-fPIC,-ffp-contract=off,-O2,-Wall,-pthread",
    "-shared",
]


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(os.path.join(CSRC, d)) > t for d in DEPS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
          ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed building libykgpu.so")
    if verbose:
        sys.stderr.write(r.stdout + r.stderr)
    return LIB


if __name__ == "__main__":
    print(build(force=True, verbose="-v" in sys.argv))
