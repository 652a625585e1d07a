"""The device-resident ordered commit ("lattice commit", csrc/yk_lattice.h) on the CPU: the header is single-source, so
tests/host/device_shim.cpp compiles the very code of yk_lattice_kernel into plain loops and drives it with the real
ordering engine; here under forced `device`, where the lattice kernel takes every stretch.  Bindings, ask states and node
availability must equal the oracle's; after every batch the shim also checks that the patched node order is exactly
"every node once, ascending by (current key, NodeID rank)"."""
import ctypes as C
import functools

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
import device_shim
from device_shim import INELIGIBLE, dshim  # noqa: F401  (dshim: the shim fixture)

run = functools.partial(device_shim.run, rounds=0)
check = functools.partial(device_shim.check, rounds=0)


@pytest.mark.parametrize("batch", [7, 64, 1024])
def test_lattice_matches_oracle_on_fuzz(dshim, oracle, batch):
    checked = 0
    for seed in range(120):
        s = synth.fuzz(seed)
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > batch:
            continue
        if check(dshim, oracle, s, tag=(seed, batch), batch=batch)[0] is not None:
            checked += 1
    assert checked > 20


def test_config_shapes_small(dshim, oracle):
    for s, batch in ((synth.kwok(60, 6, 30), 64), (synth.kwok(60, 6, 30, variant="bare"), 64),
                     (synth.perf(300, 20, 40), 128), (synth.perf(300, 20, 40, masks=True), 128),
                     (synth.perf(1500, 20, 100), 4096), (synth.perf(1500, 20, 100, masks=True), 700),
                     (synth.hier(400, 3, 3, 2, 40), 96), (synth.hier(400, 2, 3, 2, 40, masks=True, leaf_sort=synth.SORT_FAIR), 96),
                     (synth.gangs(300, 60, 5), 100)):
        want, st = check(dshim, oracle, s, tag=s.name, batch=batch)
        assert want is not None and len(want["ask"]) > 0, s.name
        assert st["subruns"] > 0


def test_binpacking_is_left_to_the_host_commit(dshim):
    assert run(dshim, synth.perf(50, 2, 10, policy=synth.POLICY_BINPACKING))[0] == INELIGIBLE


def test_full_cluster_and_gang_rollbacks(dshim, oracle):
    """over-committed clusters: certain NOFITs by full scan, the capacity bound that rejects later asks without one, gangs
    that do not fit (decided on the device when no node takes the first member, handed over otherwise); with a max on the
    queue the order is placement-sensitive, so a failed gang ends its batch and the orderer rewinds to its first member"""
    for seed in range(6):
        for fill in (1.05, 2.0):
            for quota in (False, True):
                s = synth.gangs(120, 40, 5, seed=seed, fill=fill)
                if quota:
                    s.q_max[-1, 0] = 1 << 60   # never binds
                want, _ = check(dshim, oracle, s, tag=(seed, fill, quota), batch=1000)
                assert want is not None and (want["state"] == 2).sum() > 0
    # a gang whose members differ in what they request never reaches the lattice commit
    assert run(dshim, synth.poisoned_gangs(3))[0] == INELIGIBLE


def test_tiny_requests_stack_on_the_front_nodes(dshim, oracle):
    """requests much smaller than the key distance between nodes: one node takes many allocations in a row, the extras of
    the lattice carry the run and the elements have to be sorted"""
    s = synth.perf(40, 4, 300)
    s.ask_req[:, 0] = 10
    s.ask_req[:, 1] = 1_000_000
    want, st = check(dshim, oracle, s, batch=4096)
    assert want is not None
    assert st["sorts"] > 0
    # requests that do not move the key at all ({pods: 1}: no weighted resource): every element of a node ties with
    # the next one
    s = synth.kwok(30, 3, 200, variant="bare")
    assert check(dshim, oracle, s, batch=4096)[0] is not None


def test_max_bindings(dshim, oracle):
    for seed in (1, 4, 9, 12, 30):
        s = synth.fuzz(seed)
        full = oracle.run(s)
        k = max(1, len(full["ask"]) // 2)
        want = oracle.run(s, max_bindings=k)
        rc, ask, node, _, avail = run(dshim, s, batch=8 if not (s.ask_gang >= 0).any() else 64, max_bindings=k)
        if rc == INELIGIBLE:
            continue
        assert rc == 0
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
        assert np.array_equal(avail, want["avail"])


@pytest.mark.parametrize("D", [1, 2, 3, 5, 8])
def test_other_dimension_counts(dshim, oracle, D):
    for seed in range(12):
        s = synth.redim(synth.fuzz(seed), D, seed)
        check(dshim, oracle, s, tag=(seed, D), batch=64)
    s = synth.redim(synth.perf(200, 8, 40, masks=True), D, 1)
    assert check(dshim, oracle, s, batch=512)[0] is not None


def test_many_shapes_and_signatures(dshim, oracle):
    """windows that hit the shape and signature caps, boxes with six and more sides (their state count overflows an int
    unless it saturates), ids that collide in the per-sub-run tables (an entry whose id differs from its slot's leader
    leads itself)"""
    for seed in range(6):
        s = synth.perf(60, 6, 50, masks=True, seed=60 + seed)
        s.ask_req[:, 0] += (np.arange(s.n_asks) * 7919) % 13 * 10          # 13 x 4 request vectors, interleaved
        assert check(dshim, oracle, s, tag=("shapes", seed), batch=512)[0] is not None
        s = synth.perf(60, 6, 50, seed=70 + seed)
        s.ask_req[:, 1] += np.arange(s.n_asks) * 4096                       # every ask its own request vector
        assert check(dshim, oracle, s, tag=("unique", seed), batch=512)[0] is not None
        s = synth.perf(40, 4, 200, seed=80 + seed)
        s.ask_req[:, 0] = 10 + (np.arange(s.n_asks) % 7)                    # seven tiny shapes: deep boxes on every side
        s.ask_req[:, 1] = 1_000_000
        assert check(dshim, oracle, s, tag=("tiny7", seed), batch=4096)[0] is not None


# ---- uniform runs (csrc/yk_uniform.h): consecutive asks with one request vector and one predicate signature ----------------
@pytest.mark.parametrize("batch,uniform", [(64, (2, 0)), (1024, (3, 1)), (1024, (2, 2)), (7, (2, 0))])
def test_uniform_runs_match_oracle_on_fuzz(dshim, oracle, batch, uniform):
    checked = asks = 0
    for seed in range(150):
        s = synth.runny(synth.fuzz(seed), seed)
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > batch:
            continue
        want, st = check(dshim, oracle, s, tag=(seed, batch, uniform), batch=batch, uniform=uniform)
        if want is not None:
            checked += 1
            asks += st["uniform_asks"]
    assert checked > 20 and asks > 200


def test_uniform_reference_shape(dshim, oracle):
    """the reference's benchmark shape, small: identical nodes, identical pods -> every key ties across nodes at every depth"""
    for nodes, apps, tasks in ((50, 4, 125), (7, 3, 50), (100, 10, 110)):
        s = synth.reference_shape(nodes, apps, tasks)
        for uniform in ((16, 0), (16, 1), (16, 3), (16, 1 << 20)):   # a first depth past every node's capacity is cut back to it
            want, st = check(dshim, oracle, s, tag=(nodes, uniform), batch=1 << 20, uniform=uniform)
            assert want is not None
            assert st["uniform_asks"] == len(want["ask"]) == s.n_asks and st["subruns"] == 0
            if uniform[1] == 1:
                assert st["uniform_retries"] > 0


@pytest.mark.parametrize("nodes,apps,tasks", [(20, 4, 100), (50, 2, 100)])
def test_uniform_flat_request_takes_one_attempt(dshim, oracle, nodes, apps, tasks):
    """{pods: 1} requests no weighted resource, so no key moves and the run fills the front nodes to the brim: the first
    attempt generates a node's whole capacity (110 here, more than the mean-share depth) and never retries"""
    s = synth.kwok(nodes, apps, tasks, variant="bare")
    want, st = check(dshim, oracle, s, batch=1 << 20, uniform=(16, 0))
    assert want is not None and len(want["ask"]) == s.n_asks
    assert st["uniform_asks"] == s.n_asks and st["subruns"] == 0
    assert st["uniform_attempts"] == 1 and st["uniform_retries"] == 0


def test_uniform_run_overflows_the_cluster(dshim, oracle):
    """more identical pods than the nodes hold: the run places what fits and the rest fail (placement-insensitive order), or the
    batch stops at the first failure (quota'd queues: the order depends on what was placed)"""
    s = synth.reference_shape(6, 3, 300)
    s.node_total[:, 2] = s.node_avail[:, 2] = 110        # 660 pods fit, 900 asked
    want, st = check(dshim, oracle, s, batch=1 << 20, uniform=(8, 0))
    assert want is not None and len(want["ask"]) == 660 and st["uniform_asks"] > 0
    for seed in range(5):
        s = synth.hier(12, 2, 2, 2, 40, seed=seed)
        s.ask_req[:] = s.ask_req[0]
        for col in (s.ask_tol, s.ask_need, s.ask_deny):
            col[:] = col[0]
        want, st = check(dshim, oracle, s, tag=seed, batch=512, uniform=(4, 0))
        assert want is not None and st["uniform_asks"] > 0


def test_uniform_gangs(dshim, oracle):
    """homogeneous gangs inside a run: fine while everything fits; a run that cannot place all of its members goes to the
    windowed commit (which rolls gangs back)"""
    for seed in range(6):
        for fill in (0.5, 1.05, 2.0):
            s = synth.gangs(60, 30, 5, seed=seed, fill=fill)
            s.ask_req[:] = s.ask_req[0]
            want, st = check(dshim, oracle, s, tag=(seed, fill), batch=1000, uniform=(4, 0))
            assert want is not None
            assert st["uniform_attempts"] > 0


def test_plan_segments_and_capacity_rules(dshim):
    """the host-side pieces of the uniform-run path: batches are cut into uniform runs and the stretches between them, never
    inside a gang; a node's capacity for a request is yklt::fits applied repeatedly"""
    GANG, GSTART = 8, 4

    def plan(meta, shp, sig, min_run):
        B = len(shp)
        m, s, g = (np.ascontiguousarray(x, dtype=np.uint32) for x in (meta, shp, sig))
        off, ln, un = (np.zeros(B + 1, dtype=np.int32) for _ in range(3))
        n = dshim.host_plan_segments(m.ctypes.data_as(C.c_void_p), s.ctypes.data_as(C.c_void_p), g.ctypes.data_as(C.c_void_p), B, min_run,
                                     off.ctypes.data_as(C.c_void_p), ln.ctypes.data_as(C.c_void_p), un.ctypes.data_as(C.c_void_p), B + 1)
        segs = [(int(off[i]), int(ln[i]), bool(un[i])) for i in range(n)]
        assert sum(l for _, l, _ in segs) == B and all(segs[i][0] + segs[i][1] == segs[i + 1][0] for i in range(n - 1))   # a partition, in order
        return segs

    z = [0] * 10
    assert plan(z, [1] * 10, [7] * 10, 4) == [(0, 10, True)]
    assert plan(z, [1] * 10, [7] * 10, 11) == [(0, 10, False)]
    assert plan(z, [1, 1, 1, 2, 2, 2, 2, 2, 3, 3], [0] * 10, 4) == [(0, 3, False), (3, 5, True), (8, 2, False)]
    assert plan(z, [1] * 10, [0, 0, 0, 0, 0, 9, 9, 9, 9, 9], 5) == [(0, 5, True), (5, 5, True)]       # same request, two signatures
    assert plan([], [], [], 1) == []
    # a gang that straddles the start / the end of a run of equal (shape, signature) is kept whole on the windowed side
    meta = [0, GANG | GSTART, GANG, GANG, 0, 0, 0, 0, GANG | GSTART, GANG]
    shp = [5, 5, 1, 1, 1, 1, 1, 1, 1, 2]
    segs = plan(meta, shp, [0] * 10, 3)
    assert segs == [(0, 4, False), (4, 4, True), (8, 2, False)]
    for o, l, u in segs:   # no segment starts inside a gang
        assert not (meta[o] & GANG) or (meta[o] & GSTART)
    # capacity: request <= min(max(0, total), max(0, available)) on every dimension, as often as it goes
    cap = lambda av, to, rq, lim=10**9, usable=1: dshim.host_cap_of(len(rq), usable, (C.c_int64 * len(rq))(*av), (C.c_int64 * len(rq))(*to), (C.c_int64 * len(rq))(*rq), C.c_int64(lim))
    dshim.host_cap_of.restype = C.c_int64
    assert cap([1000, 64], [1000, 64], [100, 1]) == 10
    assert cap([1000, 64], [1000, 64], [100, 0]) == 10            # a zero request never limits
    assert cap([1000, -5], [1000, 64], [100, 1]) == 0             # over-committed dimension: clamped at 0
    assert cap([1000, 64], [50, 64], [100, 1]) == 0               # larger than the node's total: never fits
    assert cap([1000, 64], [1000, 64], [100, 1], lim=3) == 3
    assert cap([1000, 64], [1000, 64], [100, 1], usable=0) == 0
    assert cap([5, 5], [5, 5], [0, 0]) == 10**9                   # (never reaches the commit: the orderer marks it invalid)
    assert dshim.host_first_depth(50_000, 5_000) == 32 and dshim.host_first_depth(10, 5_000) == 4
