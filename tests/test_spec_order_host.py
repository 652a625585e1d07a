"""The speculative round-commit launch's order and screen (csrc/yk_spec.h), on the CPU: tests/host/spec_shim.cpp builds the
device's static order with the shared key and keep rules and runs the engine's own cycle set-up on the same tables.  On
fuzzed pending sets -- states left by an earlier cycle, causes, slow-path asks, absent applications, ties in create and
submit time, max_bindings cuts, masks, gangs, mixed priorities, several leaves, quotas -- the order must be
Orderer::extend_static's, and the screen must agree with the commit choice (yklt::Scan, round_eligible, plan_segments)."""
import ctypes as C

import numpy as np
import pytest

from device_shim import load

U32_NONE = 0xFFFFFFFF
ST_PENDING, ST_ALLOCATED, ST_NOFIT, ST_SKIPPED, ST_SLOWPATH, ST_INVALID, ST_ABSENT = 0, 1, 2, 3, 4, 5, 255
W_STATUS, W_COUNT, W_KEPT, W_BAD = 0, 1, 2, 3
GO = 0


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def fuzz_case(rng, variant):
    D = int(rng.integers(1, 5))
    nA = int(rng.integers(40, 400))
    nP = int(rng.integers(1, 12))
    nN = int(rng.integers(0, 6))
    # queues: root 0, leaf 1; "two_leaves" adds leaf 2; "fair" makes leaf 1 fair; "quota" puts a max on the root
    nQ = 3 if variant == "two_leaves" else 2
    q_parent = np.array([U32_NONE, 0, 0][:nQ], dtype=np.uint32)
    q_sort = np.zeros(nQ, dtype=np.uint8)
    if variant == "fair":
        q_sort[1] = 1
    q_max = np.full((D, nQ), -1, dtype=np.int64)
    if variant == "quota":
        q_max[:, 0] = 10 ** 9
    p_queue = np.ones(nP, dtype=np.uint32)
    if variant == "two_leaves":
        p_queue[rng.random(nP) < 0.5] = 2
    p_submit = rng.integers(0, 4, nP).astype(np.int64)              # ties in submit time
    p_present = (rng.random(nP) < 0.85).astype(np.uint8)              # absent applications
    a_app = rng.integers(0, nP, nA).astype(np.uint32)
    a_create = rng.integers(-3, 6, nA).astype(np.int64)               # ties (and negative) create times
    a_req = rng.integers(1, 9, (D, nA)).astype(np.int64)
    a_req[:, rng.random(nA) < 0.03] = 0                                # a request that is not strictly positive: a cause
    a_flags = (rng.random(nA) < 0.03).astype(np.uint32)                # slow path: a cause
    a_state = np.full(nA, ST_PENDING, dtype=np.uint8)
    left = rng.random(nA)                                              # states an earlier cycle left behind
    for st, share in ((ST_ALLOCATED, 0.1), (ST_NOFIT, 0.05), (ST_SKIPPED, 0.03), (ST_SLOWPATH, 0.02), (ST_INVALID, 0.02), (ST_ABSENT, 0.08)):
        a_state[(left >= 0) & (left < share)] = st
        left -= share
    a_prio = np.zeros(nA, dtype=np.int32) + int(rng.integers(-2, 3))
    if variant == "prio":
        a_prio[rng.random(nA) < 0.1] += 1
    a_tol = np.full(nA, 0xFFFF, dtype=np.uint64)
    a_need = np.zeros(nA, dtype=np.uint64)
    a_deny = np.zeros(nA, dtype=np.uint64)
    a_node = np.full(nA, U32_NONE, dtype=np.uint32)
    a_gang = np.full(nA, U32_NONE, dtype=np.uint32)
    if variant == "masks":
        a_need[rng.random(nA) < 0.05] = 1
        a_node[rng.random(nA) < 0.02] = 0
    if variant == "gang":
        a_gang[rng.random(nA) < 0.1] = 7
    if variant == "taint":
        a_tol[rng.random(nA) < 0.05] = 0
    n_taint = np.zeros(max(nN, 1), dtype=np.uint64)
    if nN:
        n_taint[0] = 0x10
    # signature ids in runs: asks of one application mostly share one
    base = rng.integers(0, 3, nP)
    a_sigid = (base[a_app] * 4 + (rng.random(nA) < 0.2) * rng.integers(0, 4, nA)).astype(np.uint32)
    if variant == "one_sig":
        a_sigid[:] = 5
    kept = int(np.sum((a_state != ST_ABSENT) & (a_state != ST_ALLOCATED) & (p_present[a_app] == 1)))
    max_bindings = int(rng.integers(1, max(kept, 1) + 1)) if rng.random() < 0.3 else nA   # max_bindings cuts
    rd_min = int(rng.integers(1, 40))
    un_min = int(rng.integers(3, 30))
    return dict(D=D, nA=nA, nP=nP, nQ=nQ, nN=nN, a_req=np.ascontiguousarray(a_req), a_tol=a_tol, a_need=a_need, a_deny=a_deny,
                a_node=a_node, a_prio=a_prio, a_create=a_create, a_app=a_app, a_flags=a_flags, a_gang=a_gang, a_sigid=a_sigid,
                a_state=a_state, p_queue=p_queue, p_submit=p_submit, p_present=p_present, q_parent=q_parent,
                q_max=np.ascontiguousarray(q_max), q_sort=q_sort, n_taint=n_taint, max_bindings=max_bindings, rd_min=rd_min,
                un_min=un_min)


def run(shim, c):
    nA = c["nA"]
    dev_order = np.zeros(nA, dtype=np.uint32)
    words = np.zeros(16, dtype=np.uint32)
    static = np.zeros(nA, dtype=np.uint32)
    batch = np.zeros(nA, dtype=np.uint32)
    n_static, n_batch = C.c_uint32(0), C.c_uint32(0)
    flags = np.zeros(8, dtype=np.int64)
    rc = shim.spec_run(C.c_int(c["D"]), C.c_uint32(nA), C.c_uint32(c["nP"]), C.c_uint32(c["nQ"]), C.c_uint32(c["nN"]),
                       _p(c["a_req"]), _p(c["a_tol"]), _p(c["a_need"]), _p(c["a_deny"]), _p(c["a_node"]), _p(c["a_prio"]),
                       _p(c["a_create"]), _p(c["a_app"]), _p(c["a_flags"]), _p(c["a_gang"]), _p(c["a_sigid"]), _p(c["a_state"]),
                       _p(c["p_queue"]), _p(c["p_submit"]), _p(c["p_present"]), _p(c["q_parent"]), _p(c["q_max"]), _p(c["q_sort"]),
                       _p(c["n_taint"]), C.c_uint32(c["max_bindings"]), C.c_int(c["rd_min"]), C.c_int(c["un_min"]),
                       _p(dev_order), _p(words), _p(static), C.byref(n_static), _p(batch), C.byref(n_batch), _p(flags))
    assert rc == 0
    n = int(words[W_COUNT])
    return dev_order[:n], words, static[:n_static.value], batch[:n_batch.value], flags


def pending_caused(c):
    """some ask the pending scan keeps carries a cause: the host's hints count it, the device's screen does not"""
    a = np.arange(c["nA"])
    pend = (c["a_state"] != ST_ABSENT) & (c["a_state"] != ST_ALLOCATED) & (c["p_present"][c["a_app"]] == 1)
    caused = (c["a_flags"] & 1).astype(bool) | ~np.all(c["a_req"] > 0, axis=0)
    return bool(np.any(pend[a] & caused))


VARIANTS = ("plain", "one_sig", "masks", "gang", "taint", "prio", "two_leaves", "fair", "quota")


@pytest.mark.parametrize("variant", VARIANTS)
def test_spec_order_matches_static_order_and_commit_choice(variant):
    shim = load("spec_shim")
    rng = np.random.default_rng(sum(map(ord, variant)))
    adopted = 0
    for _ in range(150):
        c = fuzz_case(rng, variant)
        dev, w, static, batch, f = run(shim, c)
        insensitive, device, plan_ready, one, adopt = (bool(x) for x in f[:5])
        n = int(w[W_COUNT])
        assert n == min(int(w[W_KEPT]), c["max_bindings"])
        # the keep and key rules are extend_static's: in a placement-insensitive cycle without kept gang members the device's
        # order is the static order, cut at max_bindings
        if insensitive and not w[W_BAD]:
            assert int(w[W_KEPT]) == len(static)
            assert np.array_equal(dev, static[:n])
        # the screen is never looser than the commit choice: GO in a cycle the host gates let through (one fifo leaf, no max)
        # is adopted, unless an ask with a cause changes the host's hints (its priority or masks count there)
        gate = variant not in ("two_leaves", "fair", "quota")
        if w[W_STATUS] == GO:
            if gate and not pending_caused(c):
                assert adopt, (variant, f.tolist(), w.tolist())
        # ... nor stricter: a cycle the host puts on one round stretch over its whole first batch gets GO
        if insensitive and device and plan_ready and one and not pending_caused(c):
            assert w[W_STATUS] == GO, (variant, f.tolist(), w.tolist())
        if adopt:
            adopted += 1
            assert insensitive and w[W_STATUS] == GO and np.array_equal(batch, dev)
            if variant == "one_sig":
                assert n < c["un_min"]           # one signature throughout: only a stretch shorter than a uniform run
    if variant in ("plain", "taint", "masks"):
        assert adopted > 0, variant          # the fuzz reaches the adopted case
    if variant in ("fair", "quota"):
        assert adopted == 0, variant         # an order that depends on placements is never adopted
