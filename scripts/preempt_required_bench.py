"""Time one yk_preemption_required_node call for a DaemonSet rollout: config 3 after one cycle (10 000 nodes, ~50 000 bound
allocations), with 1, 100 and 10 000 DaemonSet preemptors, one per node.

Foreign pods hold 90 % of every node's vcore, so the cycle packs the allocations into the last 10 %.  Each DaemonSet pod is
a new ask pinned to its node (required_node), asking one vcore-milli more than its node has left after the cycle and a
little memory: none fits without victims, and every plan takes pods off its own node.  Each timed call runs on a fresh copy
of the state (the marks of one call would change the next): the engine is rebuilt from the snapshot and cycled before each
call, and only the call is timed (host clock; the call ends in a stream synchronise).  Every shape is warmed up once.
Prints one JSON line with the GPU's name and power limit.  Writes nothing.

    python scripts/preempt_required_bench.py
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.dont_write_bytecode = True
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
from yunikorn_k8shim_b200 import Engine, synth  # noqa: E402


def gpu_name_and_power_limit():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                         capture_output=True, text=True, timeout=10).stdout.strip()
    name, limit = [x.strip() for x in out.splitlines()[0].split(",")]
    return name, float(limit)


def fresh(s, n_pre):
    e = Engine(D=s.D, policy=s.policy, weights=s.weights, max_nodes=s.n_nodes, max_asks=s.n_asks + s.n_nodes,
               max_apps=s.n_apps, max_queues=s.n_queues)
    e.load_snapshot(s)
    e.cycle(s.n_asks)
    left = e.nodes_available(np.arange(s.n_nodes))
    nodes = np.arange(n_pre) * (s.n_nodes // n_pre)
    req = np.zeros((n_pre, s.D), dtype=np.int64)
    req[:, 0] = np.maximum(left[nodes, 0], 0) + 1
    req[:, 1], req[:, 2] = 1 << 20, 1
    idx = np.arange(s.n_asks, s.n_asks + n_pre)
    e.asks_upsert(idx, req, np.zeros(n_pre), np.arange(n_pre) + 10 ** 9,
                  tolerated_bits=np.full(n_pre, ~np.uint64(0), dtype=np.uint64), required_node=nodes)
    e.cycle(n_pre)
    return e, idx


def main():
    argparse.ArgumentParser(description=__doc__).parse_args()
    name, limit = gpu_name_and_power_limit()
    s = synth.perf(masks=True)
    s.node_avail[:, 0] = s.node_total[:, 0] // 10
    res = {"gpu": name, "power_limit_w": limit, "nodes": s.n_nodes}
    for n_pre in (1, 100, 10_000):
        times = []
        for rep in range(4):                   # the first is the warm-up
            e, idx = fresh(s, n_pre)
            bound = int(np.sum(e.ask_states(np.arange(s.n_asks)) == 1))
            l0 = e.stats()["other_launches"]
            t0 = time.perf_counter()
            st, vic, done = e.preemption_required_node(idx)
            dt = time.perf_counter() - t0
            launches = e.stats()["other_launches"] - l0
            if rep:
                times.append(dt * 1e3)
            e.close()
        res[f"call_ms_{n_pre}"] = round(float(np.median(times)), 3)
        res[f"bound_{n_pre}"] = bound
        res[f"launches_{n_pre}"] = int(launches)
        names = ["planned", "fits", "not_blocked", "not_allowed", "unsupported", "guarantee", "no_victims"]
        res[f"status_{n_pre}"] = {names[k]: int(np.sum(st == k)) for k in range(7) if np.sum(st == k)}
        res[f"victims_{n_pre}"] = int(sum(len(v) for v in vic))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
