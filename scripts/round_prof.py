#!/usr/bin/env python
"""Where the round commit (csrc/yk_rounds.h) pays off: ms per cycle of mask-free fair cycles (synth.perf, 5 000 to 250 000
pending asks) under the host commit and under the round commit, with the rounds, asks per round, single steps and
the kernel time of each.  The round arm lowers YK_ROUND_MIN to 1 so that it runs at every size; the crossover with the
host arm is what YK_ROUND_MIN, the guard and the cost rule's per-ask constant (csrc/yk_engine.cu) are set from.

  python scripts/round_prof.py [--steps 5] [--sizes 5000,10000,20000,50000,250000] [--out FILE] [--phases]
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

# asks -> (nodes, apps); 125 tasks per app, 5 pending asks per node as in config 2
SHAPES = {5_000: (2_000, 40), 10_000: (4_000, 80), 20_000: (8_000, 160), 50_000: (10_000, 400), 250_000: (50_000, 2_000)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        q = f"nvidia-smi unavailable: {ex}"
    return q


def arm(snap, commit, steps, phases=False):
    from yunikorn_k8shim_b200 import Engine
    os.environ["YK_ROUND_MIN"] = "1"
    if phases:   # the round kernel's SM clocks per phase, printed to stderr when the engine is destroyed
        os.environ["YK_PROFILE_LATTICE"] = "1"
    else:
        os.environ.pop("YK_PROFILE_LATTICE", None)
    times, st = [], None
    with Engine.for_snapshot(snap, commit=commit) as e:
        N, A = np.arange(snap.n_nodes), np.arange(snap.n_asks)
        for i in range(steps + 1):
            e.nodes_upsert(N, snap.node_total, snap.node_avail, snap.node_taint, snap.node_label, snap.node_rank(), snap.node_flags)
            e.asks_upsert(A, snap.ask_req, snap.ask_app, snap.ask_create, snap.ask_tol, snap.ask_need, snap.ask_deny,
                          snap.ask_prio, snap.ask_node, snap.ask_flags, snap.ask_gang)
            if i == 1:
                e.stats_reset()
            t0 = time.perf_counter()
            ask, node, _ = e.cycle(snap.n_asks)
            if i >= 1:
                times.append((time.perf_counter() - t0) * 1e3)
            e.release(ask)
        st = e.stats()
    return times, st, (ask, node)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--sizes", default=",".join(str(k) for k in SHAPES))
    ap.add_argument("--out")
    ap.add_argument("--phases", action="store_true", help="also print the round kernel's clocks per phase (round arm)")
    args = ap.parse_args()
    from yunikorn_k8shim_b200 import build, synth
    build.build()
    rows = {"card": card(), "sizes": []}
    print(rows["card"], flush=True)
    for n_asks in (int(x) for x in args.sizes.split(",")):
        nodes, apps = SHAPES[n_asks]
        snap = synth.perf(nodes, apps, 125)
        th, sh, bh = arm(snap, "host", args.steps)
        ta, sa, ba = arm(snap, "auto", args.steps, args.phases)
        k = args.steps
        r = {"asks": n_asks, "nodes": nodes, "identical": bool(np.array_equal(bh[0], ba[0]) and np.array_equal(bh[1], ba[1])),
             "host_ms": sorted(th), "rounds_ms": sorted(ta),
             "rounds_on_device": sa["round_asks"] // k == n_asks,
             "passes": sa["round_passes"] / k, "asks_per_pass": sa["round_asks"] / max(sa["round_passes"], 1),
             "single_steps": sa["round_single_steps"] / k, "lattice_ms": sa["lattice_ms"] / k,
             "handoffs": sa["lattice_handoffs"] / k}
        r["kernel_us_per_pass"] = 1e3 * r["lattice_ms"] / max(r["passes"], 1)
        r["kernel_us_per_ask"] = 1e3 * r["lattice_ms"] / n_asks
        rows["sizes"].append(r)
        print(json.dumps(r), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
