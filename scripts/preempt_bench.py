"""Time yk_preemption_nodes on config 3 (10 000 nodes, taint / affinity mask asks) after one cycle, against the caller's only
alternative without it: one yk_preemption_search query per (ask, node holding victims), built on the host.

Victim list: the lowest-priority half of the allocated asks, in a seeded order (ties in priority broken by that order).
For 1, 64 and 1 024 preemptors (pending and allocated asks, spread over the snapshot) each ask gets its own seeded
permutation of that list.  Both calls end in a synchronise of the engine's stream, so a host clock around a call is its
time; every shape is warmed up first.  The batch of the alternative is built on the host once per shape (vectorised numpy;
its build time is reported apart from the call).  The answers of both are compared: fit counts, best node and count, and
the first k fitting nodes.  Prints one JSON line with the GPU's name and power limit.  Writes nothing.

    python scripts/preempt_bench.py [--k 16]
"""
import argparse
import ctypes as C
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


def p(x):
    return x.ctypes.data_as(C.c_void_p)


def host_batch(asks, lists, bound, pos, req):
    """queries of yk_preemption_search: per ask, one per node holding its victims, in node order; victims in list order"""
    n = len(asks)
    lens = np.array([len(x) for x in lists])
    owner = np.repeat(np.arange(n), lens)
    vic = np.concatenate(lists)
    node = bound[vic]
    o = np.lexsort((pos[node], owner))                  # stable: list order inside each (ask, node)
    owner, vic, node = owner[o], vic[o], node[o]
    head = np.ones(len(vic), bool)
    head[1:] = (owner[1:] != owner[:-1]) | (node[1:] != node[:-1])
    starts = np.nonzero(head)[0]
    q_ask = asks[owner[starts]].astype(np.uint32)
    q_node = node[starts].astype(np.uint32)
    off = np.append(starts, len(vic)).astype(np.uint32)
    vreq = np.ascontiguousarray(req[vic].T)             # [D][entries]
    return q_ask, q_node, off, vreq, owner[starts]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=16)
    args = ap.parse_args()
    k = args.k
    s = synth.perf(10_000, 400, 125, masks=True, seed=2)      # BASELINE config 3
    name, limit = gpu_name_and_power_limit()
    out = {"workload": "config3 after one cycle: 10k nodes / 50k pods + taints + nodeAffinity bitmasks", "k": k,
           "n_nodes": s.n_nodes, "gpu": name, "power_limit_w": limit,
           "time": "host clock around the call (it returns after its stream synchronise), mean over the repetitions"}
    rng = np.random.default_rng(7)
    with Engine.for_snapshot(s) as e:
        ask, node, _ = e.cycle(s.n_asks)
        bound = np.full(s.n_asks, -1, np.int64)
        bound[ask] = node
        seeded = rng.permutation(ask)
        victims = seeded[np.argsort(s.ask_prio[seeded], kind="stable")][:len(ask) // 2].astype(np.uint32)
        scores = e.node_scores(np.arange(s.n_nodes))
        order = np.lexsort((np.arange(s.n_nodes), s.node_rank(), scores))
        pos = np.empty(s.n_nodes, np.int64)
        pos[order] = np.arange(s.n_nodes)
        out["allocated"], out["victims_per_list"] = int(len(ask)), int(len(victims))
        lib, h = e._lib, e._h
        for n, reps in ((1, 50), (64, 10), (1024, 3)):
            asks = np.linspace(0, s.n_asks - 1, n).astype(np.uint32)
            lists = [rng.permutation(victims) for _ in range(n)]
            res = e.preemption_nodes(asks, lists, k=k)
            v_off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.uint32)
            v_all = np.concatenate(lists).astype(np.uint32)
            o = [np.zeros((n, k), np.uint32), np.zeros((n, k), np.uint32)] + [np.zeros(n, np.uint32) for _ in range(3)]

            def nodes_call():                               # the C call alone, on arrays built once
                rc = lib.yk_preemption_nodes(h, C.c_uint32(n), p(asks), p(v_off), p(v_all), C.c_uint32(0), C.c_uint32(k),
                                             *[p(x) for x in o])
                assert rc == 0, rc
            nodes_call()
            st0 = e.stats()
            t0 = time.perf_counter()
            for _ in range(reps):
                nodes_call()
            dt = (time.perf_counter() - t0) / reps
            st1 = e.stats()
            assert all(np.array_equal(x, y) for x, y in zip(o, res))
            t0 = time.perf_counter()
            q_ask, q_node, off, vreq, q_row = host_batch(asks, lists, bound, pos, s.ask_req)
            build_s = time.perf_counter() - t0
            start = np.zeros(len(q_ask), np.uint32)
            ans = np.zeros(len(q_ask), np.int32)

            def search():
                rc = lib.yk_preemption_search(h, C.c_uint32(len(q_ask)), p(q_ask), p(q_node), p(off), p(vreq), p(start), p(ans))
                assert rc == 0, rc
            search()
            t0 = time.perf_counter()
            for _ in range(reps):
                search()
            dt_alt = (time.perf_counter() - t0) / reps
            nodes, need, n_fit, best_node, best_need = res
            bounds = np.searchsorted(q_row, np.arange(n + 1))
            for i in range(n):                              # the same answers
                a, qn = ans[bounds[i]:bounds[i + 1]], q_node[bounds[i]:bounds[i + 1]]
                fit = a >= 0
                assert n_fit[i] == fit.sum(), i
                assert nodes[i, :min(k, fit.sum())].tolist() == qn[fit][:k].tolist(), i
                assert need[i, :min(k, fit.sum())].tolist() == (a[fit][:k] + 1).tolist(), i
                if fit.any():
                    j = int(np.argmin(np.where(fit, a, np.iinfo(np.int32).max)))
                    assert (best_node[i], best_need[i]) == (qn[j], a[j] + 1), i
                else:
                    assert best_node[i] == 0xFFFFFFFF and best_need[i] == 0, i
            out[f"asks_{n}"] = {
                "entries": int(n * len(victims)), "queries": int(len(q_ask)), "mean_fitting_nodes": float(n_fit.mean()),
                "preemption_nodes_ms": dt * 1e3,
                "h2d_bytes_per_call": (st1["h2d_bytes"] - st0["h2d_bytes"]) // reps,
                "d2h_bytes_per_call": (st1["d2h_bytes"] - st0["d2h_bytes"]) // reps,
                "launches_per_call": (st1["other_launches"] - st0["other_launches"]) // reps,
                "host_built_search_ms": dt_alt * 1e3, "host_build_ms": build_s * 1e3,
                "host_built_h2d_bytes": int(4 * (3 * len(q_ask) + 1) + vreq.nbytes),
                "host_built_d2h_bytes": int(4 * len(q_ask)),
                "answers_equal": True}
            del q_ask, q_node, off, vreq, q_row, v_all
    print(json.dumps(out))


if __name__ == "__main__":
    main()
