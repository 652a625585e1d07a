"""ctypes access to oracle/_build/libykoracle.so -- TEST INFRASTRUCTURE ONLY.

Imported only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "_build", "libykoracle.so")


class _Snap(C.Structure):
    _fields_ = [
        ("D", C.c_int32), ("policy", C.c_int32), ("weights", C.c_void_p),
        ("n_nodes", C.c_int32), ("node_total", C.c_void_p), ("node_avail", C.c_void_p),
        ("node_taint", C.c_void_p), ("node_label", C.c_void_p), ("node_flags", C.c_void_p),
        ("node_id", C.POINTER(C.c_char_p)),
        ("n_queues", C.c_int32), ("q_parent", C.c_void_p), ("q_guaranteed", C.c_void_p),
        ("q_max", C.c_void_p), ("q_alloc", C.c_void_p), ("q_sort", C.c_void_p),
        ("n_apps", C.c_int32), ("app_queue", C.c_void_p), ("app_submit", C.c_void_p),
        ("n_asks", C.c_int32), ("ask_app", C.c_void_p), ("ask_req", C.c_void_p),
        ("ask_tol", C.c_void_p), ("ask_need", C.c_void_p), ("ask_deny", C.c_void_p),
        ("ask_prio", C.c_void_p), ("ask_create", C.c_void_p), ("ask_node", C.c_void_p),
        ("ask_flags", C.c_void_p), ("ask_gang", C.c_void_p),
        ("q_prio_offset", C.c_void_p), ("q_prio_fence", C.c_void_p),
        ("app_user", C.c_void_p), ("n_limits", C.c_int32), ("ul_queue", C.c_void_p), ("ul_user", C.c_void_p),
        ("ul_max", C.c_void_p), ("ul_alloc", C.c_void_p), ("app_alloc", C.c_void_p),
    ]


class Stats(C.Structure):
    _fields_ = [("passes", C.c_int64), ("node_visits", C.c_int64), ("evaluations", C.c_int64),
                ("allocations", C.c_int64), ("app_sorts", C.c_int64), ("queue_sorts", C.c_int64)]


def build(force: bool = False) -> str:
    if force or not os.path.exists(_LIB_PATH) or \
            os.path.getmtime(_LIB_PATH) < os.path.getmtime(os.path.join(_HERE, "yk_oracle.cpp")):
        subprocess.check_call(["make", "-C", _HERE, "-B", "_build/libykoracle.so"],
                              stdout=subprocess.DEVNULL)
    return _LIB_PATH


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = C.CDLL(build())
        _lib.yko_run.restype = C.c_int
        _lib.yko_predicate.restype = C.c_int
        _lib.yko_node_score.restype = C.c_double
        _lib.yko_comp_usage_ratio_separately.restype = C.c_int
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _pack(s):
    """-> (struct, keepalive list)"""
    keep = []

    def arr(x, dt):
        a = np.ascontiguousarray(x, dtype=dt)
        keep.append(a)
        return _p(a)
    ids = (C.c_char_p * s.n_nodes)(*[i.encode() for i in s.node_id])
    keep.append(ids)
    st = _Snap(
        D=s.D, policy=s.policy, weights=arr(s.weights, np.float64),
        n_nodes=s.n_nodes, node_total=arr(s.node_total, np.int64), node_avail=arr(s.node_avail, np.int64),
        node_taint=arr(s.node_taint, np.uint64), node_label=arr(s.node_label, np.uint64),
        node_flags=arr(s.node_flags, np.uint32), node_id=C.cast(ids, C.POINTER(C.c_char_p)),
        n_queues=s.n_queues, q_parent=arr(s.q_parent, np.int32), q_guaranteed=arr(s.q_guaranteed, np.int64),
        q_max=arr(s.q_max, np.int64), q_alloc=arr(s.q_alloc, np.int64), q_sort=arr(s.q_sort, np.uint8),
        n_apps=s.n_apps, app_queue=arr(s.app_queue, np.int32), app_submit=arr(s.app_submit, np.int64),
        n_asks=s.n_asks, ask_app=arr(s.ask_app, np.int32), ask_req=arr(s.ask_req, np.int64),
        ask_tol=arr(s.ask_tol, np.uint64), ask_need=arr(s.ask_need, np.uint64), ask_deny=arr(s.ask_deny, np.uint64),
        ask_prio=arr(s.ask_prio, np.int32), ask_create=arr(s.ask_create, np.int64), ask_node=arr(s.ask_node, np.int32),
        ask_flags=arr(s.ask_flags, np.uint32), ask_gang=arr(s.ask_gang, np.int32),
        q_prio_offset=(arr(s.q_prio_offset, np.int32) if getattr(s, "q_prio_offset", None) is not None else None),
        q_prio_fence=(arr(s.q_prio_fence, np.uint8) if getattr(s, "q_prio_fence", None) is not None else None))
    if getattr(s, "ul_queue", None) is not None and len(s.ul_queue):
        st.app_user = arr(s.app_user, np.int32)
        st.n_limits = len(s.ul_queue)
        st.ul_queue, st.ul_user = arr(s.ul_queue, np.int32), arr(s.ul_user, np.int32)
        st.ul_max = arr(s.ul_max, np.int64)
        st.ul_alloc = arr(s.ul_alloc, np.int64) if getattr(s, "ul_alloc", None) is not None else None
    if getattr(s, "app_alloc", None) is not None:
        st.app_alloc = arr(np.asarray(s.app_alloc, np.int64).reshape(s.n_apps, s.D), np.int64)
    return st, keep


def run(s, max_bindings: int = -1, retry_failed: bool = False):
    """-> dict(ask=[...], node=[...], state=[A], avail=[N][D], stats=Stats)"""
    st, keep = _pack(s)
    A = max(s.n_asks, 1)
    out_ask = np.zeros(A, dtype=np.int32)
    out_node = np.zeros(A, dtype=np.int32)
    n_out = C.c_int32(0)
    state = np.zeros(A, dtype=np.uint8)
    avail = np.zeros((s.n_nodes, s.D), dtype=np.int64)
    stats = Stats()
    rc = lib().yko_run(C.byref(st), C.c_uint32(1 if retry_failed else 0), C.c_int32(max_bindings),
                       _p(out_ask), _p(out_node), C.byref(n_out), _p(state), _p(avail), C.byref(stats))
    if rc != 0:
        raise RuntimeError(f"yko_run failed: {rc}")
    n = n_out.value
    return {"ask": out_ask[:n].copy(), "node": out_node[:n].copy(), "state": state[:s.n_asks].copy(),
            "avail": avail, "stats": stats}


def predicate(s, ask: int, node: int) -> int:
    st, keep = _pack(s)
    return lib().yko_predicate(C.byref(st), C.c_int32(ask), C.c_int32(node))


def predicate_reserve(s, ask: int, node: int) -> int:
    st, keep = _pack(s)
    lib().yko_predicate_reserve.restype = C.c_int
    return lib().yko_predicate_reserve(C.byref(st), C.c_int32(ask), C.c_int32(node))


def preemption_index(s, ask: int, node: int, victim_req, start: int) -> int:
    st, keep = _pack(s)
    v = np.ascontiguousarray(victim_req, dtype=np.int64).reshape(-1, s.D)
    lib().yko_preemption_index.restype = C.c_int
    return lib().yko_preemption_index(C.byref(st), C.c_int32(ask), C.c_int32(node), C.c_int32(len(v)), _p(v), C.c_int32(start))


def node_score(policy, weights, total, avail) -> float:
    w = np.ascontiguousarray(weights, dtype=np.float64)
    t = np.ascontiguousarray(total, dtype=np.int64)
    a = np.ascontiguousarray(avail, dtype=np.int64)
    return lib().yko_node_score(C.c_int32(len(w)), C.c_int32(policy), _p(w), _p(t), _p(a))


def comp_usage_ratio_separately(lalloc, lguar, ralloc, rguar) -> int:
    arrs = [np.ascontiguousarray(x, dtype=np.int64) for x in (lalloc, lguar, ralloc, rguar)]
    return lib().yko_comp_usage_ratio_separately(C.c_int32(len(arrs[0])), *[_p(a) for a in arrs])


def bindings_hash(ask, node) -> int:
    """FNV-1a 64 over (ask_id, node_id) little-endian u32 pairs in commit order (BASELINE.md section 3)."""
    h = 0xCBF29CE484222325
    data = np.stack([np.asarray(ask, dtype=np.uint32), np.asarray(node, dtype=np.uint32)], axis=1).tobytes()
    for b in data:
        h = ((h ^ b) * 0x100000001B3) & 0xFFFFFFFFFFFFFFFF
    return h
