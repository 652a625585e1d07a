"""ctypes binding of libykgpu.so (include/ykgpu.h) -- the same stub a cgo / JNI binding would be.

No scheduling logic lives here: every method marshals numpy arrays into the C ABI call of the same name.
There is no CPU path: if the library is missing, or the machine has no CUDA device, construction raises.
"""
from __future__ import annotations

import ctypes as C
import os
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libykgpu.so")

YK_NONE = 0xFFFFFFFF
ST_PENDING, ST_ALLOCATED, ST_NOFIT, ST_SKIPPED, ST_SLOWPATH, ST_INVALID = range(6)
ST_ABSENT = 255
YK_ERR_CUDA = -2
FILTER_SLOTS = 11          # yk_filter_nodes counts: 0 passes, 1..9 YK_FAIL_*, 10 node reserved
FILTER_RESERVED = 10
ASK_SLOWPATH = 1
ASK_NO_PREEMPT_SELF = 2    # not AllowPreemptSelf
ASK_NO_PREEMPT_OTHER = 4   # not AllowPreemptOther (preemptionPolicy: Never)
ASK_ORIGINATOR = 8
# yk_preemption_plan and yk_preemption_required_node statuses
PP_PLANNED, PP_FITS, PP_NOT_BLOCKED, PP_NOT_ALLOWED, PP_UNSUPPORTED, PP_GUARANTEE, PP_NO_VICTIMS = range(7)

EXPORTS = [
    "yk_abi_version", "yk_create", "yk_destroy", "yk_nodes_upsert", "yk_nodes_remove", "yk_queues_set", "yk_queues_priority",
    "yk_queues_preemption", "yk_apps_upsert", "yk_apps_remove", "yk_apps_user", "yk_user_limits_set", "yk_asks_upsert",
    "yk_asks_remove", "yk_release",
    "yk_asks_resize", "yk_cycle",
    "yk_ask_states", "yk_nodes_available", "yk_evaluate", "yk_evaluate_reserve", "yk_node_scores", "yk_node_sort_set", "yk_filter_nodes",
    "yk_preemption_search", "yk_preemption_nodes", "yk_preemption_plan", "yk_preemption_required_node",
    "yk_set_exchange",
    "yk_peer_export", "yk_peer_import", "yk_peer_enable", "yk_stats",
    "yk_stats_reset", "yk_strerror", "yk_last_error",
]


class Config(C.Structure):
    _fields_ = [("abi_version", C.c_uint32), ("D", C.c_uint32), ("policy", C.c_uint32), ("batch", C.c_uint32),
                ("weights", C.c_double * 8),
                ("max_nodes", C.c_uint32), ("max_asks", C.c_uint32), ("max_apps", C.c_uint32), ("max_queues", C.c_uint32),
                ("device", C.c_int32), ("flags", C.c_uint32), ("rank", C.c_uint32), ("world", C.c_uint32)]


FLAG_NO_ROW_SHARING = 1
FLAG_HOST_COMMIT = 2
FLAG_DEVICE_COMMIT = 4
FLAG_BINPACKING_DEVICE = 8


class Stats(C.Structure):
    _fields_ = [("cycles", C.c_uint64), ("batches", C.c_uint64), ("allocations", C.c_uint64), ("nofit", C.c_uint64),
                ("skipped", C.c_uint64), ("evaluations", C.c_uint64), ("sweep_launches", C.c_uint64),
                ("other_launches", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64),
                ("sweep_ms", C.c_double), ("sort_ms", C.c_double), ("commit_ms", C.c_double), ("total_ms", C.c_double),
                ("last_sweep_ms", C.c_double), ("last_sweep_pairs", C.c_uint64),
                ("host_ms", C.c_double * 8), ("dbg", C.c_uint64 * 4), ("prof", C.c_uint64 * 6),
                ("asks_swept", C.c_uint64), ("rows_swept", C.c_uint64),
                ("lattice_launches", C.c_uint64), ("lattice_subruns", C.c_uint64), ("lattice_asks", C.c_uint64),
                ("lattice_elements", C.c_uint64), ("lattice_sorts", C.c_uint64), ("lattice_fullscans", C.c_uint64),
                ("lattice_quick", C.c_uint64), ("lattice_handoffs", C.c_uint64), ("lattice_ms", C.c_double),
                ("lattice_cycles", C.c_uint64),
                ("uniform_runs", C.c_uint64), ("uniform_asks", C.c_uint64), ("uniform_elements", C.c_uint64),
                ("uniform_retries", C.c_uint64),
                ("round_passes", C.c_uint64), ("round_asks", C.c_uint64), ("round_single_steps", C.c_uint64),
                ("spec_adopted", C.c_uint64), ("spec_discarded", C.c_uint64)]

    def as_dict(self):
        d = {f: getattr(self, f) for f, _ in self._fields_}
        d["host_ms"] = list(d["host_ms"])
        d["dbg"] = list(d["dbg"])
        d["prof"] = list(d["prof"])
        return d


ALLGATHER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p)

_lib = None


class YkError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"ykgpu error {code}: {msg}")
        self.code = code


def load_library():
    """dlopen libykgpu.so; fails loudly when it has not been built (python -m yunikorn_k8shim_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} not built: run `python __graft_entry__.py build` "
                                    "(nvcc, sm_90a). There is no CPU fallback.")
        lib = C.CDLL(LIB_PATH)
        lib.yk_abi_version.restype = C.c_uint32
        lib.yk_strerror.restype = C.c_char_p
        lib.yk_last_error.restype = C.c_char_p
        lib.yk_last_error.argtypes = [C.c_void_p]
        lib.yk_destroy.restype = None
        lib.yk_destroy.argtypes = [C.c_void_p]
        for name in EXPORTS:
            fn = getattr(lib, name)
            if name not in ("yk_abi_version", "yk_strerror", "yk_last_error", "yk_destroy"):
                fn.restype = C.c_int
        _lib = lib
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _arr(x, dt, n=None):
    if x is None:
        return None
    a = np.ascontiguousarray(x, dtype=dt)
    if n is not None and a.size != n:
        raise ValueError(f"expected {n} elements, got {a.size}")
    return a


def _colmajor(x, D, n):
    """[n][D] row-major (or already [D][n]) -> contiguous [D][n] int64"""
    a = np.asarray(x, dtype=np.int64)
    if a.shape == (n, D):
        a = a.T
    elif a.shape != (D, n):
        raise ValueError(f"expected shape ({n},{D}) or ({D},{n}), got {a.shape}")
    return np.ascontiguousarray(a)


def _node_sort_weights(D, weights):
    """[8] float64 node-sort weights: None = the core default, vcore = memory = 1 (as far as D reaches)"""
    w = np.zeros(8)
    if weights is None:
        w[0] = 1.0
        if D > 1:
            w[1] = 1.0
    else:
        w[:len(weights)] = weights
    return w


class Engine:
    """One yk_engine.  Method names and arguments mirror include/ykgpu.h one to one.

    commit: where the ordered commit runs -- "auto" (the library's default: on the device for cycles made of long uniform runs,
    sweep + host commit otherwise), "host" (YK_FLAG_HOST_COMMIT), "device" (YK_FLAG_DEVICE_COMMIT: every eligible cycle).
    binpacking_device: under the binpacking node sort, let "auto" and "device" commit eligible cycles on the device too, one
    ordered capacity fill per uniform run (YK_FLAG_BINPACKING_DEVICE); off, binpacking cycles stay on the host commit."""

    def __init__(self, D=4, policy=0, weights=None, max_nodes=1024, max_asks=4096, max_apps=64, max_queues=8,
                 batch=0, device=-1, rank=0, world=1, share_rows=True, commit="auto", binpacking_device=False):
        self._lib = load_library()
        cfg = Config()
        cfg.abi_version = self._lib.yk_abi_version()
        cfg.D, cfg.policy, cfg.batch = D, policy, batch
        w = _node_sort_weights(D, weights)
        for i in range(8):
            cfg.weights[i] = float(w[i])
        cfg.max_nodes, cfg.max_asks, cfg.max_apps, cfg.max_queues = max_nodes, max_asks, max_apps, max_queues
        cfg.device, cfg.rank, cfg.world = device, rank, world
        cfg.flags = (0 if share_rows else FLAG_NO_ROW_SHARING) | {"auto": 0, "host": FLAG_HOST_COMMIT, "device": FLAG_DEVICE_COMMIT}[commit]
        if binpacking_device:
            cfg.flags |= FLAG_BINPACKING_DEVICE
        self.D = D
        self.max_asks = max_asks
        self._h = C.c_void_p()
        rc = self._lib.yk_create(C.byref(cfg), C.byref(self._h))
        if rc != 0:
            raise YkError(rc, self._lib.yk_strerror(rc).decode())
        self._keep = []

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.yk_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _ck(self, rc):
        if rc < 0:
            raise YkError(rc, (self._lib.yk_last_error(self._h) or b"").decode() or self._lib.yk_strerror(rc).decode())
        return rc

    # ---- state ----
    def nodes_upsert(self, idx, total, avail, taint_bits=None, label_bits=None, name_rank=None, flags=None):
        idx = _arr(idx, np.uint32)
        n = idx.size
        self._ck(self._lib.yk_nodes_upsert(self._h, C.c_uint32(n), _p(idx), _p(_colmajor(total, self.D, n)),
                                           _p(_colmajor(avail, self.D, n)), _p(_arr(taint_bits, np.uint64, n)),
                                           _p(_arr(label_bits, np.uint64, n)), _p(_arr(name_rank, np.uint32, n)),
                                           _p(_arr(flags, np.uint32, n))))

    def nodes_remove(self, idx):
        idx = _arr(idx, np.uint32)
        self._ck(self._lib.yk_nodes_remove(self._h, C.c_uint32(idx.size), _p(idx)))

    def queues_set(self, parent, guaranteed=None, max=None, allocated=None, sort=None):
        par = np.asarray(parent, dtype=np.int64).copy()
        par[par < 0] = YK_NONE
        par = par.astype(np.uint32)
        q = par.size
        self.n_queues = q
        g = None if guaranteed is None else _colmajor(guaranteed, self.D, q)
        m = None if max is None else _colmajor(max, self.D, q)
        al = None if allocated is None else _colmajor(allocated, self.D, q)
        self._ck(self._lib.yk_queues_set(self._h, C.c_uint32(q), _p(par), _p(g), _p(m), _p(al), _p(_arr(sort, np.uint8, q))))

    def queues_priority(self, offset=None, fence=None):
        """queue properties priority.offset ([Q] int32) / priority.policy == fence ([Q] bool); call after queues_set"""
        off = _arr(offset, np.int32) if offset is not None else None
        fen = _arr(np.asarray(fence).astype(np.uint8), np.uint8) if fence is not None else None
        q = off.size if off is not None else (fen.size if fen is not None else 0)
        self._ck(self._lib.yk_queues_priority(self._h, C.c_uint32(q), _p(off), _p(fen)))

    def queues_preemption(self, fence=None):
        """queue property preemption.policy == fence ([Q] bool, None = no fence); call after queues_set"""
        fen = _arr(np.asarray(fence).astype(np.uint8), np.uint8) if fence is not None else None
        q = fen.size if fen is not None else getattr(self, "n_queues", 0)
        self._ck(self._lib.yk_queues_preemption(self._h, C.c_uint32(q), _p(fen)))

    def apps_upsert(self, idx, queue, submit_time):
        idx = _arr(idx, np.uint32)
        n = idx.size
        self._ck(self._lib.yk_apps_upsert(self._h, C.c_uint32(n), _p(idx), _p(_arr(queue, np.uint32, n)),
                                          _p(_arr(submit_time, np.int64, n))))

    def apps_user(self, idx, user):
        idx = _arr(idx, np.uint32)
        u = np.asarray(user, dtype=np.int64).copy()
        u[u < 0] = YK_NONE
        u = _arr(u.astype(np.uint32), np.uint32, idx.size)
        self._ck(self._lib.yk_apps_user(self._h, C.c_uint32(idx.size), _p(idx), _p(u)))

    def user_limits_set(self, queue, user, max, held=None):
        q, u = _arr(queue, np.uint32), _arr(user, np.uint32)
        n = q.size
        mx = _colmajor(np.asarray(max, dtype=np.int64).reshape(n, self.D), self.D, n) if n else np.zeros(0, dtype=np.int64)
        hd = None if held is None or not n else _colmajor(np.asarray(held, dtype=np.int64).reshape(n, self.D), self.D, n)
        self._ck(self._lib.yk_user_limits_set(self._h, C.c_uint32(n), _p(q), _p(u), _p(mx), _p(hd)))

    def apps_remove(self, idx):
        idx = _arr(idx, np.uint32)
        self._ck(self._lib.yk_apps_remove(self._h, C.c_uint32(idx.size), _p(idx)))

    def asks_upsert(self, idx, req, app, create_seq, tolerated_bits=None, required_bits=None, forbidden_bits=None,
                    priority=None, required_node=None, flags=None, gang=None):
        idx = _arr(idx, np.uint32)
        n = idx.size

        def u32none(x):
            if x is None:
                return None
            if isinstance(x, np.ndarray) and x.dtype == np.uint32:   # already in the ABI's encoding (YK_NONE = 0xFFFFFFFF)
                return _arr(x, np.uint32, n)
            a = np.asarray(x, dtype=np.int64).copy()
            a[a < 0] = YK_NONE
            return _arr(a, np.uint32, n)
        self._ck(self._lib.yk_asks_upsert(
            self._h, C.c_uint32(n), _p(idx), _p(_colmajor(req, self.D, n)), _p(_arr(tolerated_bits, np.uint64, n)),
            _p(_arr(required_bits, np.uint64, n)), _p(_arr(forbidden_bits, np.uint64, n)), _p(_arr(priority, np.int32, n)),
            _p(_arr(create_seq, np.int64, n)), _p(_arr(app, np.uint32, n)), _p(u32none(required_node)),
            _p(_arr(flags, np.uint32, n)), _p(u32none(gang))))

    def asks_remove(self, idx):
        idx = _arr(idx, np.uint32)
        self._ck(self._lib.yk_asks_remove(self._h, C.c_uint32(idx.size), _p(idx)))

    def release(self, ask_idx):
        idx = _arr(ask_idx, np.uint32)
        self._ck(self._lib.yk_release(self._h, C.c_uint32(idx.size), _p(idx)))

    def asks_resize(self, idx, req):
        """new requests for present asks, pending or allocated (an in-place pod resize); req as in asks_upsert"""
        idx = _arr(idx, np.uint32)
        n = idx.size
        self._ck(self._lib.yk_asks_resize(self._h, C.c_uint32(n), _p(idx), _p(_colmajor(req, self.D, n))))

    # ---- the cycle ----
    def cycle(self, max_bindings, slow_cap=0):
        """-> (ask[n], node[n]) in commit order, slow_path_asks"""
        out = np.zeros((max(max_bindings, 1), 2), dtype=np.uint32)
        n_out = C.c_uint32(0)
        slow = np.zeros(max(slow_cap, 1), dtype=np.uint32)
        n_slow = C.c_uint32(0)
        self._ck(self._lib.yk_cycle(self._h, C.c_uint32(max_bindings), _p(out), C.byref(n_out), _p(slow),
                                    C.c_uint32(slow_cap), C.byref(n_slow)))
        n = n_out.value
        return out[:n, 0].copy(), out[:n, 1].copy(), slow[:n_slow.value].copy()

    def ask_states(self, idx):
        idx = _arr(idx, np.uint32)
        out = np.zeros(idx.size, dtype=np.uint8)
        self._ck(self._lib.yk_ask_states(self._h, C.c_uint32(idx.size), _p(idx), _p(out)))
        return out

    def nodes_available(self, idx):
        idx = _arr(idx, np.uint32)
        out = np.zeros((self.D, idx.size), dtype=np.int64)
        self._ck(self._lib.yk_nodes_available(self._h, C.c_uint32(idx.size), _p(idx), _p(out)))
        return out.T.copy()

    def evaluate(self, ask, node):
        return self._ck(self._lib.yk_evaluate(self._h, C.c_uint32(ask), C.c_uint32(node)))

    def evaluate_reserve(self, ask, node):
        return self._ck(self._lib.yk_evaluate_reserve(self._h, C.c_uint32(ask), C.c_uint32(node)))

    def node_scores(self, idx):
        idx = _arr(idx, np.uint32)
        out = np.zeros(idx.size, dtype=np.float64)
        self._ck(self._lib.yk_node_scores(self._h, C.c_uint32(idx.size), _p(idx), _p(out)))
        return out

    def node_sort_set(self, policy, weights=None):
        """replace the node sort policy and weights of this engine from the next call on; weights=None as in the constructor"""
        w = _node_sort_weights(self.D, weights)
        self._ck(self._lib.yk_node_sort_set(self._h, C.c_uint32(policy), w.ctypes.data_as(C.c_void_p)))

    def filter_nodes(self, asks, k=0, skip=0, allocate=True):
        """-> (nodes[n][k], n_pass[n], counts[n][FILTER_SLOTS]) uint32: per ask, the passing nodes of pass rank skip .. skip+k-1
        in the cycle's node order (YK_NONE past the end), how many pass, and every present node's first failing step"""
        asks = _arr(asks, np.uint32)
        n = asks.size
        nodes = np.zeros((n, k), dtype=np.uint32)
        n_pass = np.zeros(n, dtype=np.uint32)
        counts = np.zeros((n, FILTER_SLOTS), dtype=np.uint32)
        self._ck(self._lib.yk_filter_nodes(self._h, C.c_uint32(n), _p(asks), C.c_int(1 if allocate else 0), C.c_uint32(skip),
                                           C.c_uint32(k), _p(nodes) if k else None, _p(n_pass), _p(counts)))
        return nodes, n_pass, counts

    def preemption_search(self, ask, node, victim_req_lists, start):
        """victim_req_lists: per query an [n_victims][D] array of what each victim gives back -> index per query"""
        ask, node, start = _arr(ask, np.uint32), _arr(node, np.uint32), _arr(start, np.uint32)
        off = np.zeros(len(ask) + 1, dtype=np.uint32)
        off[1:] = np.cumsum([len(v) for v in victim_req_lists])
        flat = np.zeros((self.D, max(int(off[-1]), 1)), dtype=np.int64)
        pos = 0
        for v in victim_req_lists:
            v = np.asarray(v, dtype=np.int64).reshape(-1, self.D)
            flat[:, pos:pos + len(v)] = v.T
            pos += len(v)
        flat = np.ascontiguousarray(flat[:, :max(int(off[-1]), 1)])
        out = np.zeros(len(ask), dtype=np.int32)
        self._ck(self._lib.yk_preemption_search(self._h, C.c_uint32(len(ask)), _p(ask), _p(node), _p(off), _p(flat), _p(start), _p(out)))
        return out

    def preemption_nodes(self, asks, victim_lists, k=0, skip=0):
        """victim_lists: per ask the allocated asks that may be preempted for it, in victim order -> (nodes[n][k], need[n][k],
        n_fit[n], best_node[n], best_need[n]) uint32: per ask, the fitting nodes of fit rank skip .. skip+k-1 in the cycle's node
        order with the victims each needs (YK_NONE / 0 past the end), how many nodes fit, and the one needing the fewest"""
        asks = _arr(asks, np.uint32)
        n = asks.size
        if len(victim_lists) != n:
            raise ValueError(f"expected {n} victim lists, got {len(victim_lists)}")
        off = np.zeros(n + 1, dtype=np.uint32)
        off[1:] = np.cumsum([len(v) for v in victim_lists])
        victims = np.concatenate([np.asarray(v, dtype=np.uint32).ravel() for v in victim_lists]) if n else np.zeros(0, np.uint32)
        victims = _arr(victims, np.uint32)
        nodes = np.zeros((n, k), dtype=np.uint32)
        need = np.zeros((n, k), dtype=np.uint32)
        n_fit, best_node, best_need = (np.zeros(n, dtype=np.uint32) for _ in range(3))
        self._ck(self._lib.yk_preemption_nodes(self._h, C.c_uint32(n), _p(asks), _p(off), _p(victims) if victims.size else None,
                                               C.c_uint32(skip), C.c_uint32(k), _p(nodes) if k else None, _p(need) if k else None,
                                               _p(n_fit), _p(best_node), _p(best_need)))
        return nodes, need, n_fit, best_node, best_need

    def preemption_plan(self, asks, victims_cap=None):
        """plan preemption for the preemptors in order -> (status[d], node[d], victims: d arrays of ask indices, d = n_done);
        victims_cap (default max_asks) bounds the victims of the whole call: planning stops before the ask that would pass it"""
        asks = _arr(asks, np.uint32)
        n = asks.size
        cap = self.max_asks if victims_cap is None else int(victims_cap)
        status = np.zeros(max(n, 1), dtype=np.uint32)
        node = np.zeros(max(n, 1), dtype=np.uint32)
        off = np.zeros(n + 1, dtype=np.uint32)
        vic = np.zeros(max(cap, 1), dtype=np.uint32)
        done = C.c_uint32(0)
        self._ck(self._lib.yk_preemption_plan(self._h, C.c_uint32(n), _p(asks), _p(status), _p(node), _p(off),
                                              _p(vic) if cap else None, C.c_uint32(cap), C.byref(done)))
        d = done.value
        return status[:d].copy(), node[:d].copy(), [vic[off[i]:off[i + 1]].copy() for i in range(d)], d

    def preemption_required_node(self, asks, victims_cap=None):
        """preemption for required-node (DaemonSet) asks on their own node, in order -> (status[d], victims: d arrays of ask
        indices, d = n_done); victims_cap (default max_asks) bounds the victims of the whole call: planning stops before the
        ask that would pass it"""
        asks = _arr(asks, np.uint32)
        n = asks.size
        cap = self.max_asks if victims_cap is None else int(victims_cap)
        status = np.zeros(max(n, 1), dtype=np.uint32)
        off = np.zeros(n + 1, dtype=np.uint32)
        vic = np.zeros(max(cap, 1), dtype=np.uint32)
        done = C.c_uint32(0)
        self._ck(self._lib.yk_preemption_required_node(self._h, C.c_uint32(n), _p(asks), _p(status), _p(off),
                                                       _p(vic) if cap else None, C.c_uint32(cap), C.byref(done)))
        d = done.value
        return status[:d].copy(), [vic[off[i]:off[i + 1]].copy() for i in range(d)], d

    def set_exchange(self, fn):
        cb = ALLGATHER_FN(fn) if fn is not None else C.cast(None, ALLGATHER_FN)
        self._keep.append(cb)
        self._ck(self._lib.yk_set_exchange(self._h, cb, None))

    def peer_export(self) -> bytes:
        buf = (C.c_ubyte * 192)()
        self._ck(self._lib.yk_peer_export(self._h, buf))
        return bytes(buf)

    def peer_import(self, peer_rank: int, blob: bytes):
        buf = (C.c_ubyte * 192).from_buffer_copy(blob)
        self._ck(self._lib.yk_peer_import(self._h, C.c_uint32(peer_rank), buf))

    def peer_enable(self):
        self._ck(self._lib.yk_peer_enable(self._h))

    def stats(self) -> dict:
        s = Stats()
        self._ck(self._lib.yk_stats(self._h, C.byref(s)))
        return s.as_dict()

    def stats_reset(self):
        self._ck(self._lib.yk_stats_reset(self._h))

    # ---- convenience: push a synth.Snapshot through the ABI (what the Go SchedulerAPI adapter does) ----
    def load_snapshot(self, s):
        N, A, P = s.n_nodes, s.n_asks, s.n_apps
        if getattr(s, "app_alloc", None) is not None and np.any(s.app_alloc):
            # the ABI has no call that loads what applications already hold: a fair leaf would order them from zero
            raise ValueError("load_snapshot: the snapshot's applications hold allocations (app_alloc), which an engine "
                             "cannot load")
        self.queues_set(s.q_parent, s.q_guaranteed, s.q_max, s.q_alloc, s.q_sort)
        if getattr(s, "q_prio_offset", None) is not None or getattr(s, "q_prio_fence", None) is not None:
            self.queues_priority(s.q_prio_offset, s.q_prio_fence)
        self.nodes_upsert(np.arange(N), s.node_total, s.node_avail, s.node_taint, s.node_label, s.node_rank(), s.node_flags)
        self.apps_upsert(np.arange(P), s.app_queue, s.app_submit)
        if getattr(s, "ul_queue", None) is not None and len(s.ul_queue):
            self.apps_user(np.arange(P), s.app_user)
            self.user_limits_set(s.ul_queue, s.ul_user, s.ul_max, s.ul_alloc)
        self.asks_upsert(np.arange(A), s.ask_req, s.ask_app, s.ask_create, s.ask_tol, s.ask_need, s.ask_deny,
                         s.ask_prio, s.ask_node, s.ask_flags, s.ask_gang)

    @classmethod
    def for_snapshot(cls, s, **kw):
        e = cls(D=s.D, policy=s.policy, weights=s.weights, max_nodes=max(s.n_nodes, 1), max_asks=max(s.n_asks, 1),
                max_apps=max(s.n_apps, 1), max_queues=max(s.n_queues, 1), **kw)
        e.load_snapshot(s)
        return e
