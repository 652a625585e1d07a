"""Time yk_filter_nodes on config 3 (10 000 nodes, taint / affinity mask asks) with k = 64 candidates per ask.

Prints one JSON line: time per call for 1, 64 and 4 096 asks, (ask, node) pairs per second, bytes copied each way and
launches per call, the mean share of nodes that pass an ask, and the GPU's name and power limit.  The call returns after a
synchronise of the engine's stream, so a host clock around it is the call's time.  Writes nothing.

    python scripts/filter_bench.py [--k 64]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.dont_write_bytecode = True
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
from yunikorn_k8shim_b200 import Engine, synth  # noqa: E402


def gpu_name_and_power_limit():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, timeout=10).stdout.strip()
    name, limit = [x.strip() for x in out.splitlines()[0].split(",")]
    return name, float(limit)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=64)
    args = ap.parse_args()
    s = synth.perf(10_000, 400, 125, masks=True, seed=2)      # BASELINE config 3
    name, limit = gpu_name_and_power_limit()
    out = {"workload": "config3: 10k nodes / 50k pods + taints + nodeAffinity bitmasks", "k": args.k, "n_nodes": s.n_nodes,
           "gpu": name, "power_limit_w": limit,
           "time": "host clock around the call (it returns after its stream synchronise), mean over the repetitions"}
    with Engine.for_snapshot(s) as e:
        for n, reps in ((1, 200), (64, 100), (4096, 20)):
            asks = np.linspace(0, s.n_asks - 1, n).astype(np.uint32)
            for _ in range(3):
                e.filter_nodes(asks, k=args.k)
            st0 = e.stats()
            t0 = time.perf_counter()
            for _ in range(reps):
                e.filter_nodes(asks, k=args.k)
            dt = (time.perf_counter() - t0) / reps
            st1 = e.stats()
            out[f"asks_{n}"] = {"ms_per_call": dt * 1e3, "pairs_per_s": n * s.n_nodes / dt,
                                "d2h_bytes_per_call": (st1["d2h_bytes"] - st0["d2h_bytes"]) // reps,
                                "h2d_bytes_per_call": (st1["h2d_bytes"] - st0["h2d_bytes"]) // reps,
                                "launches_per_call": (st1["other_launches"] - st0["other_launches"]) // reps}
        _, n_pass, _ = e.filter_nodes(np.arange(s.n_asks), k=0)
    out["mean_pass_fraction"] = float(n_pass.mean()) / s.n_nodes
    print(json.dumps(out))


if __name__ == "__main__":
    main()
