"""ctypes stub of the label / taint dictionary encoder (include/ykgpu_dict.h, csrc/yk_dict.cpp)."""
from __future__ import annotations

import ctypes as C

from .engine import load_library, YkError

OPS = {"In": 0, "NotIn": 1, "Exists": 2, "DoesNotExist": 3, "Gt": 4, "Lt": 5}
EFFECTS = {"": 0, "NoSchedule": 1, "PreferNoSchedule": 2, "NoExecute": 3}
TOL_OPS = {"": 0, "Equal": 0, "Exists": 1}
DICT_EXPORTS = ["yk_dict_create", "yk_dict_destroy", "yk_dict_node", "yk_dict_node_remove", "yk_dict_pod",
                "yk_dict_pod_required_node", "yk_dict_generation", "yk_dict_node_bits"]


class _Req(C.Structure):
    _fields_ = [("key", C.c_char_p), ("op", C.c_uint32), ("n_values", C.c_uint32), ("values", C.POINTER(C.c_char_p))]


class _Term(C.Structure):
    _fields_ = [("n_expressions", C.c_uint32), ("expressions", C.POINTER(_Req)), ("n_fields", C.c_uint32), ("fields", C.POINTER(_Req))]


class _Taint(C.Structure):
    _fields_ = [("key", C.c_char_p), ("value", C.c_char_p), ("effect", C.c_uint32)]


class _Tol(C.Structure):
    _fields_ = [("key", C.c_char_p), ("op", C.c_uint32), ("value", C.c_char_p), ("effect", C.c_uint32)]


class _PodSpec(C.Structure):
    _fields_ = [("n_selector", C.c_uint32), ("selector_keys", C.POINTER(C.c_char_p)), ("selector_values", C.POINTER(C.c_char_p)),
                ("has_required_affinity", C.c_int32), ("n_terms", C.c_uint32), ("terms", C.POINTER(_Term)),
                ("n_tolerations", C.c_uint32), ("tolerations", C.POINTER(_Tol)), ("node_name", C.c_char_p)]


class PodMasks(C.Structure):
    _fields_ = [("tolerated_bits", C.c_uint64), ("required_bits", C.c_uint64), ("forbidden_bits", C.c_uint64),
                ("required_node", C.c_uint32), ("flags", C.c_uint32)]


def _strs(xs):
    arr = (C.c_char_p * max(len(xs), 1))(*[x.encode() for x in xs])
    return arr


def _reqs(rs, keep):
    arr = (_Req * max(len(rs), 1))()
    for i, r in enumerate(rs):
        vals = _strs(r.get("values") or [])
        keep.append(vals)
        arr[i] = _Req(r["key"].encode(), OPS[r["op"]], len(r.get("values") or []), C.cast(vals, C.POINTER(C.c_char_p)))
    keep.append(arr)
    return arr


class Dictionary:
    def __init__(self):
        self._lib = load_library()
        self._lib.yk_dict_create.restype = C.c_void_p
        self._lib.yk_dict_destroy.argtypes = [C.c_void_p]
        self._lib.yk_dict_destroy.restype = None
        self._lib.yk_dict_generation.restype = C.c_uint64
        self._lib.yk_dict_generation.argtypes = [C.c_void_p]
        self._h = C.c_void_p(self._lib.yk_dict_create())

    def close(self):
        if self._h:
            self._lib.yk_dict_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def generation(self):
        return self._lib.yk_dict_generation(self._h)

    def node(self, idx, name, labels=None, taints=None, unschedulable=False):
        """-> (label_bits, taint_bits)"""
        labels = labels or {}
        taints = taints or []
        ks, vs = _strs(list(labels.keys())), _strs(list(labels.values()))
        ta = (_Taint * max(len(taints), 1))()
        for i, t in enumerate(taints):
            ta[i] = _Taint(t["key"].encode(), t.get("value", "").encode(), EFFECTS[t.get("effect", "NoSchedule")])
        lb, tb = C.c_uint64(0), C.c_uint64(0)
        rc = self._lib.yk_dict_node(self._h, C.c_uint32(idx), name.encode(), C.c_uint32(len(labels)),
                                    C.cast(ks, C.POINTER(C.c_char_p)), C.cast(vs, C.POINTER(C.c_char_p)),
                                    C.c_uint32(len(taints)), ta, C.c_int32(1 if unschedulable else 0), C.byref(lb), C.byref(tb))
        if rc != 0:
            raise YkError(rc, "yk_dict_node")
        return lb.value, tb.value

    def node_bits(self, idx):
        lb, tb = C.c_uint64(0), C.c_uint64(0)
        rc = self._lib.yk_dict_node_bits(self._h, C.c_uint32(idx), C.byref(lb), C.byref(tb))
        if rc != 0:
            raise YkError(rc, "yk_dict_node_bits")
        return lb.value, tb.value

    def pod(self, node_selector=None, affinity_terms=None, has_affinity=None, tolerations=None, node_name=None) -> PodMasks:
        """affinity_terms: list of {"expr": [...], "fields": [...]} or None; has_affinity defaults to
        (affinity_terms is not None) -- pass has_affinity=True with affinity_terms=None for a nil term list."""
        keep = []
        spec = _spec(keep, node_selector, affinity_terms, has_affinity, tolerations, node_name)
        out = PodMasks()
        rc = self._lib.yk_dict_pod(self._h, C.byref(spec), C.byref(out))
        if rc != 0:
            raise YkError(rc, "yk_dict_pod")
        return out

    def pod_required_node(self, required_node, node_selector=None, affinity_terms=None, has_affinity=None, tolerations=None,
                          node_name=None) -> PodMasks:
        """a pod whose node is fixed (a DaemonSet pod): masks as pod(...) gives, with required_node = the index of the node
        named required_node and the affinity terms resolved against that name"""
        keep = []
        spec = _spec(keep, node_selector, affinity_terms, has_affinity, tolerations, node_name)
        out = PodMasks()
        rc = self._lib.yk_dict_pod_required_node(self._h, C.byref(spec), required_node.encode(), C.byref(out))
        if rc != 0:
            raise YkError(rc, "yk_dict_pod_required_node")
        return out


def _spec(keep, node_selector, affinity_terms, has_affinity, tolerations, node_name):
    sel = node_selector or {}
    ks, vs = _strs(list(sel.keys())), _strs(list(sel.values()))
    keep += [ks, vs]
    terms = affinity_terms or []
    if has_affinity is None:
        has_affinity = affinity_terms is not None
    ta = (_Term * max(len(terms), 1))()
    for i, t in enumerate(terms):
        ex, fl = t.get("expr") or [], t.get("fields") or []
        ta[i] = _Term(len(ex), C.cast(_reqs(ex, keep), C.POINTER(_Req)), len(fl), C.cast(_reqs(fl, keep), C.POINTER(_Req)))
    tols = tolerations or []
    to = (_Tol * max(len(tols), 1))()
    for i, t in enumerate(tols):
        to[i] = _Tol(t.get("key", "").encode(), TOL_OPS[t.get("op", "")], t.get("value", "").encode(), EFFECTS[t.get("effect", "")])
    keep += [ta, to]
    return _PodSpec(len(sel), C.cast(ks, C.POINTER(C.c_char_p)), C.cast(vs, C.POINTER(C.c_char_p)),
                    1 if has_affinity else 0, len(terms), ta, len(tols), to, (node_name or "").encode())
