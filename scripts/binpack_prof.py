#!/usr/bin/env python
"""What the binpacking fill (csrc/yk_uniform.h, YK_FLAG_BINPACKING_DEVICE) costs against the sweep + host commit: ms per
cycle of binpacking cycles under the host commit (no flag) and under the flag with the device commit forced, in
alternating pairs on one engine each, with the kernel time, the number of fills and whether the bindings are equal.  The
`auto` arm (flag, default commit) shows what the cost rule chooses.  The cost rule's constants (csrc/yk_engine.cu BP_*) are
set from these runs: a fill's fixed cost from the runny snapshot (thousands of short runs), the host commit's per-ask cost
from the reference shapes.

  python scripts/binpack_prof.py [--steps 5] [--shapes ref,ref10,runny] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

import numpy as np  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        q = f"nvidia-smi unavailable: {ex}"
    return q


def shapes(names):
    from yunikorn_k8shim_b200 import synth
    bp = synth.POLICY_BINPACKING
    make = {"ref": lambda: synth.reference_shape(5_000, 400, 125, policy=bp),          # 50 000 identical pods
            "ref10": lambda: synth.reference_shape(50_000, 4_000, 125, policy=bp),     # 500 000
            "runny": lambda: synth.runny(synth.perf(10_000, 400, 125, policy=bp), 1)}  # config 2 in runs of 1..13
    return [(n, make[n]()) for n in names]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--shapes", default="ref,ref10,runny")
    ap.add_argument("--out")
    args = ap.parse_args()
    from yunikorn_k8shim_b200 import Engine, build
    build.build()
    rows = {"card": card(), "shapes": []}
    print(rows["card"], flush=True)
    arms = {"host": dict(commit="auto"), "fill": dict(commit="device", binpacking_device=True),
            "auto": dict(commit="auto", binpacking_device=True)}
    for name, snap in shapes(args.shapes.split(",")):
        N, A = np.arange(snap.n_nodes), np.arange(snap.n_asks)
        engines = {k: Engine.for_snapshot(snap, batch=4096, **kw) for k, kw in arms.items()}
        times = {k: [] for k in arms}
        out = {}
        try:
            for i in range(args.steps + 1):   # step 0 warms every arm up; then the arms alternate
                for k, e in engines.items():
                    e.nodes_upsert(N, snap.node_total, snap.node_avail, snap.node_taint, snap.node_label, snap.node_rank(), snap.node_flags)
                    e.asks_upsert(A, snap.ask_req, snap.ask_app, snap.ask_create, snap.ask_tol, snap.ask_need, snap.ask_deny,
                                  snap.ask_prio, snap.ask_node, snap.ask_flags, snap.ask_gang)
                    if i == 1:
                        e.stats_reset()
                    t0 = time.perf_counter()
                    ask, node, _ = e.cycle(snap.n_asks)
                    if i >= 1:
                        times[k].append((time.perf_counter() - t0) * 1e3)
                    out[k] = (ask, node)
                    e.release(ask)
            st = {k: e.stats() for k, e in engines.items()}
        finally:
            for e in engines.values():
                e.close()
        n = args.steps
        r = {"shape": name, "nodes": snap.n_nodes, "asks": snap.n_asks, "bound": int(len(out["host"][0])),
             "identical": all(np.array_equal(out["host"][j], out[k][j]) for k in ("fill", "auto") for j in (0, 1))}
        for k in arms:
            r[k] = {"ms": sorted(round(t, 3) for t in times[k]), "device_cycles": st[k]["lattice_cycles"] / n,
                    "fills": st[k]["uniform_runs"] / n, "kernel_ms": round(st[k]["lattice_ms"] / n, 3),
                    "handoffs": st[k]["lattice_handoffs"] / n, "sweep_launches": st[k]["sweep_launches"] / n}
        med = {k: float(np.median(times[k])) for k in arms}
        r["host_us_per_ask"] = round(1e3 * med["host"] / snap.n_asks, 4)
        r["fill_us_per_fill"] = round(1e3 * med["fill"] / max(r["fill"]["fills"], 1), 2)
        r["speedup_fill_vs_host"] = round(med["host"] / med["fill"], 3)
        rows["shapes"].append(r)
        print(json.dumps(r), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
