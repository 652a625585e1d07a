"""Time one yk_preemption_plan call at 10 000 nodes and ~50 000 bound allocations (config 3 after one cycle), for 1, 16 and
256 preemptors.  (The plain-Python restatement in tests/preemption_oracle.py loops over every allocation per node and is
far too slow at this size to be a timing baseline; the tests compare answers at small sizes.)

Queues: the snapshot's tree with a guarantee on every leaf of a tenth of its allocation, so every leaf sits above its
guarantee.  Foreign pods hold 90 % of every node's vcore, so the cycle packs the allocations into the last 10 %.  The
preemptors are new asks in an extra leaf with a large guarantee, each asking one vcore-milli more than the most any node has
left after the cycle (and a little memory): none fits anywhere without victims, and each plan takes pods off one node.
Each timed call runs on a fresh copy of the state (the plans of one call would change the next): the engine is rebuilt from
the snapshot and cycled before each call, and only the call is timed (host clock; the call ends in a stream synchronise).
Every shape is warmed up once.  Prints one JSON line with the GPU's name and power limit.  Writes nothing.

    python scripts/preempt_plan_bench.py
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


def snapshot(n_pre):
    s = synth.perf(masks=True)
    s.node_avail[:, 0] = s.node_total[:, 0] // 10
    Q = s.n_queues
    s.q_parent = np.append(s.q_parent, 0).astype(np.int32)
    alloc = np.zeros((Q + 1, s.D), dtype=np.int64)
    for a in range(s.n_asks):
        alloc[int(s.app_queue[int(s.ask_app[a])])] += s.ask_req[a]
    s.q_guaranteed = np.vstack([np.where(alloc[:Q] > 0, alloc[:Q] // 10, -1), np.full((1, s.D), -1)]).astype(np.int64)
    s.q_guaranteed[Q, :2] = np.maximum(s.node_total[:, :2].max(axis=0), 1) * (n_pre + 1)
    s.q_max = np.vstack([s.q_max, np.full((1, s.D), -1)]).astype(np.int64)
    s.q_alloc = np.zeros((Q + 1, s.D), dtype=np.int64)
    s.q_sort = np.append(s.q_sort, 0).astype(np.uint8)
    s.app_queue = np.append(s.app_queue, Q).astype(np.int32)
    s.app_submit = np.append(s.app_submit, s.app_submit.max() + 1)
    return s


def fresh(s, n_pre):
    e = Engine(D=s.D, policy=s.policy, weights=s.weights, max_nodes=s.n_nodes, max_asks=s.n_asks + n_pre, max_apps=s.n_apps,
               max_queues=s.n_queues)
    e.load_snapshot(s)
    e.cycle(s.n_asks)
    left = e.nodes_available(np.arange(s.n_nodes))
    one = np.zeros(s.D, dtype=np.int64)
    one[0], one[1], one[2] = max(int(left[:, 0].max()), 0) + 1, 1 << 20, 1
    req = np.tile(one, (n_pre, 1))
    idx = np.arange(s.n_asks, s.n_asks + n_pre)
    e.asks_upsert(idx, req, np.full(n_pre, s.n_apps - 1), np.arange(n_pre) + 10 ** 9,
                  tolerated_bits=np.full(n_pre, ~np.uint64(0), dtype=np.uint64))
    e.cycle(n_pre)
    return e, idx


def main():
    argparse.ArgumentParser(description=__doc__).parse_args()
    name, limit = gpu_name_and_power_limit()
    res = {"gpu": name, "power_limit_w": limit, "nodes": 10_000}
    for n_pre in (1, 16, 256):
        s = snapshot(n_pre)
        times = []
        for rep in range(3):                   # the first is the warm-up
            e, idx = fresh(s, n_pre)
            bound = int(np.sum(e.ask_states(np.arange(s.n_asks)) == 1))
            t0 = time.perf_counter()
            st, node, vic, done = e.preemption_plan(idx)
            dt = time.perf_counter() - t0
            if rep:
                times.append(dt * 1e3)
            e.close()
        res[f"plan_ms_{n_pre}"] = round(float(np.median(times)), 3)
        res[f"bound_{n_pre}"] = bound
        names = ["planned", "fits", "not_blocked", "not_allowed", "unsupported", "guarantee", "no_victims"]
        res[f"status_{n_pre}"] = {names[k]: int(np.sum(st == k)) for k in range(7) if np.sum(st == k)}
        res[f"victims_{n_pre}"] = int(sum(len(v) for v in vic))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
