"""The engine's host side end to end, without a GPU: tests/host/engine_shim.cpp drives the REAL ordering engine
(csrc/yk_orderer.hpp) and the REAL ordered commit (csrc/yk_commit.hpp) through yk_cycle's own batch loop
(yk::host_commit in csrc/yk_lattice_host.hpp) -- batches, speculative next batch, rewind, epochs with lazy order merges --
with the device sweep replaced by a plain CPU loop.
Bindings, ask states and node availability must equal the oracle's, for every batch size / epoch length."""
import ctypes as C

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth

NONE = 0xFFFFFFFF


@pytest.fixture(scope="module")
def shim():
    from device_shim import load   # (device_shim imports this module)
    return load("engine_shim")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _u32(x):
    x = np.asarray(x).astype(np.int64).copy()
    x[x < 0] = NONE
    return x.astype(np.uint32)


def run_engine_host(shim, s, batch=256, epoch_limit=None, speculate=1, max_bindings=None, share_rows=1, rows=None,
                    fn="engine_host_run"):
    N, A, P, Q, D = s.n_nodes, s.n_asks, s.n_apps, s.n_queues, s.D
    if epoch_limit is None:
        epoch_limit = max(2 * batch, N * 5 // 8)
    if max_bindings is None:
        max_bindings = A
    keep = dict(
        w=np.ascontiguousarray(s.weights, dtype=np.float64),
        total=np.ascontiguousarray(s.node_total.T), avail=np.ascontiguousarray(s.node_avail.T),
        taint=np.ascontiguousarray(s.node_taint), label=np.ascontiguousarray(s.node_label),
        nflags=np.ascontiguousarray(s.node_flags, dtype=np.uint32), rank=s.node_rank(),
        req=np.ascontiguousarray(s.ask_req.T), tol=np.ascontiguousarray(s.ask_tol), need=np.ascontiguousarray(s.ask_need),
        deny=np.ascontiguousarray(s.ask_deny), anode=_u32(s.ask_node), prio=np.ascontiguousarray(s.ask_prio, dtype=np.int32),
        create=np.ascontiguousarray(s.ask_create), app=_u32(s.ask_app), aflags=np.ascontiguousarray(s.ask_flags, dtype=np.uint32),
        gang=_u32(s.ask_gang), queue=_u32(s.app_queue), submit=np.ascontiguousarray(s.app_submit), par=_u32(s.q_parent),
        guar=np.ascontiguousarray(s.q_guaranteed.T), mx=np.ascontiguousarray(s.q_max.T),
        alloc=np.ascontiguousarray(s.q_alloc.T).copy(), sort=np.ascontiguousarray(s.q_sort, dtype=np.uint8))
    k = keep
    # queue properties priority.offset / priority.policy=fence go through a setter (keeps the argument list short)
    k["qoff"] = np.ascontiguousarray(s.q_prio_offset, dtype=np.int32) if getattr(s, "q_prio_offset", None) is not None else None
    k["qfen"] = np.ascontiguousarray(s.q_prio_fence, dtype=np.uint8) if getattr(s, "q_prio_fence", None) is not None else None
    setter = getattr(shim, "host_set_queue_priority", None)
    if setter is not None:
        setter(_p(k["qoff"]) if k["qoff"] is not None else None, _p(k["qfen"]) if k["qfen"] is not None else None)
    setter = getattr(shim, "host_set_user_limits", None)
    if setter is not None:
        if getattr(s, "ul_queue", None) is not None and len(s.ul_queue):
            k["puser"] = _u32(s.app_user)
            k["ulq"], k["ulu"] = _u32(s.ul_queue), _u32(s.ul_user)
            k["ulm"] = np.ascontiguousarray(np.asarray(s.ul_max, dtype=np.int64).T)
            k["ula"] = np.ascontiguousarray(np.asarray(s.ul_alloc if s.ul_alloc is not None else np.zeros_like(s.ul_max), dtype=np.int64).T).copy()
            setter(_p(k["puser"]), C.c_uint32(len(s.ul_queue)), _p(k["ulq"]), _p(k["ulu"]), _p(k["ulm"]), _p(k["ula"]))
        else:
            setter(None, C.c_uint32(0), None, None, None, None)
    setter = getattr(shim, "host_set_app_alloc", None)
    if setter is not None:
        held = getattr(s, "app_alloc", None)
        k["palloc"] = np.ascontiguousarray(np.asarray(held, dtype=np.int64).reshape(P, D).T) if held is not None else None
        setter(_p(k["palloc"]) if held is not None else None)
    out_ask = np.zeros(max(A, 1), dtype=np.uint32)
    out_node = np.zeros(max(A, 1), dtype=np.uint32)
    n = C.c_uint32(0)
    state = np.zeros(max(A, 1), dtype=np.uint8)
    avail = np.zeros((D, max(N, 1)), dtype=np.int64)
    nrows = np.zeros(32, dtype=np.uint64)   # engine shim: [0] rows swept; device shim: its counters
    rc = getattr(shim, fn)(
        C.c_int(D), C.c_uint32(s.policy), _p(k["w"]),
        C.c_uint32(N), _p(k["total"]), _p(k["avail"]), _p(k["taint"]), _p(k["label"]), _p(k["nflags"]), _p(k["rank"]),
        C.c_uint32(A), C.c_uint32(P), C.c_uint32(Q), _p(k["req"]), _p(k["tol"]), _p(k["need"]), _p(k["deny"]), _p(k["anode"]),
        _p(k["prio"]), _p(k["create"]), _p(k["app"]), _p(k["aflags"]), _p(k["gang"]), _p(k["queue"]), _p(k["submit"]),
        _p(k["par"]), _p(k["guar"]), _p(k["mx"]), _p(k["alloc"]), _p(k["sort"]),
        C.c_uint32(batch), C.c_uint32(epoch_limit), C.c_int(speculate), C.c_int(share_rows), C.c_uint32(max_bindings),
        _p(out_ask), _p(out_node), C.byref(n), _p(state), _p(avail), _p(nrows))
    if rows is not None:
        rows.append(int(nrows[0]) if fn == "engine_host_run" else [int(x) for x in nrows])
        if fn == "engine_host_run":
            run_engine_host.last_counters = [int(x) for x in nrows]
    return rc, out_ask[:n.value].astype(np.int64), out_node[:n.value].astype(np.int64), state[:A], avail[:, :N].T.copy()


def check(shim, oracle, s, tag=None, **kw):
    want = oracle.run(s, max_bindings=kw.get("max_bindings") or -1)
    rc, ask, node, state, avail = run_engine_host(shim, s, **kw)
    assert rc == 0, (tag, rc)
    assert np.array_equal(ask, want["ask"]), tag
    assert np.array_equal(node, want["node"]), tag
    if kw.get("max_bindings") is None:
        assert np.array_equal(state, want["state"]), tag
    assert np.array_equal(avail, want["avail"]), tag
    return want


@pytest.mark.parametrize("batch", [7, 64, 1024])
def test_host_engine_matches_oracle_on_fuzz(shim, oracle, batch):
    checked = 0
    for seed in range(60):
        s = synth.fuzz(seed)
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > batch:
            rc = run_engine_host(shim, s, batch=batch)[0]
            assert rc == -1                      # documented error: a gang larger than the sweep batch
            continue
        for spec, share in ((1, 1), (0, 1), (1, 0)):
            check(shim, oracle, s, tag=(seed, batch, spec, share), batch=batch, speculate=spec, share_rows=share)
        checked += 1
    assert checked > 30


@pytest.mark.parametrize("epoch", [1, 3, 40, 10 ** 9])
def test_epoch_length_never_changes_the_result(shim, oracle, epoch):
    """epoch_limit 1 = a fresh sorted view for every batch; 1e9 = one view for the whole cycle: the touched-node
    index and the clean-bit scan must give the same placements either way."""
    for seed in range(0, 60, 3):
        s = synth.fuzz(seed)
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > 16:
            continue
        check(shim, oracle, s, tag=(seed, epoch), batch=16, epoch_limit=epoch)


@pytest.mark.parametrize("policy", [synth.POLICY_FAIR, synth.POLICY_BINPACKING])
def test_config_shapes_small(shim, oracle, policy):
    """the bench configurations, scaled down (the CPU stand-in sweep is O(asks x nodes))"""
    for s, batch in ((synth.kwok(60, 6, 30, policy=policy), 64),
                     (synth.perf(300, 20, 40, policy=policy), 128),
                     (synth.perf(300, 20, 40, masks=True, policy=policy), 128),
                     (synth.hier(400, 3, 3, 2, 40, policy=policy), 96),
                     (synth.hier(400, 2, 3, 2, 40, masks=True, leaf_sort=synth.SORT_FAIR, policy=policy), 96),
                     (synth.gangs(300, 60, 5, policy=policy), 100)):
        want = check(shim, oracle, s, tag=s.name, batch=batch)
        assert len(want["ask"]) > 0


def test_max_bindings_stops_the_cycle(shim, oracle):
    for seed in (1, 4, 9):
        s = synth.fuzz(seed)
        full = oracle.run(s)
        k = max(1, len(full["ask"]) // 2)
        want = oracle.run(s, max_bindings=k)
        rc, ask, node, _, avail = run_engine_host(shim, s, batch=8 if not (s.ask_gang >= 0).any() else 64, max_bindings=k)
        assert rc == 0
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
        assert np.array_equal(avail, want["avail"])


@pytest.mark.parametrize("policy", [synth.POLICY_FAIR, synth.POLICY_BINPACKING])
def test_gang_rollback_restores_every_index(shim, oracle, policy):
    """Gangs that are placed and then undone, in a placement-insensitive order (the batch goes on after the failure,
    inside one long epoch): the touched bitmap, the scan front, the pruning bound and the ordered index must all be
    back to where they were, or later asks miss the nodes the roll-back handed back.  (Each of those four restores
    was checked to be necessary by deleting it: this test then fails.)"""
    for seed in range(40):
        s = synth.poisoned_gangs(seed, policy=policy)
        for batch in (16, 1000):
            want = check(shim, oracle, s, tag=(seed, batch), batch=batch, epoch_limit=10 ** 9)
        assert (want["state"] == 2).sum() > 0


@pytest.mark.parametrize("fill", [1.05, 2.0])
def test_overcommitted_gangs(shim, oracle, fill):
    for seed in range(6):
        for policy in (synth.POLICY_FAIR, synth.POLICY_BINPACKING):
            s = synth.gangs(120, 40, 5, seed=seed, fill=fill, policy=policy)
            check(shim, oracle, s, tag=(seed, policy), batch=64, epoch_limit=10 ** 9)
            check(shim, oracle, s, tag=(seed, policy), batch=1000)


def test_shared_rows_sweep_one_row_per_signature(shim, oracle):
    """asks with identical predicate inputs share one swept row: same bindings, far fewer rows; asks that differ in
    any input (request, toleration, required / forbidden label, node name) never share"""
    s = synth.perf(300, 20, 40)
    shared, single = [], []
    want = check(shim, oracle, s, batch=128, rows=shared)
    check(shim, oracle, s, batch=128, share_rows=0, rows=single)
    assert single[0] >= len(want["ask"]) and shared[0] * 4 < single[0]
    # make every ask distinct in one input at a time: nothing may be shared any more
    for field in ("req", "tol", "need", "deny", "node"):
        t = synth.perf(64, 4, 20)
        i = np.arange(t.n_asks)
        if field == "req":
            t.ask_req[:, 3] = i                      # a dimension every node has plenty of
            t.node_total[:, 3] = t.node_avail[:, 3] = 1 << 40
        elif field == "tol":
            t.ask_tol[:] = (i.astype(np.uint64) << np.uint64(8))
        elif field == "need":
            t.node_label[:] |= np.uint64((1 << 40) - 1) << np.uint64(8)
            t.ask_need[:] = (i.astype(np.uint64) << np.uint64(8))
        elif field == "deny":
            t.ask_deny[:] = (i.astype(np.uint64) << np.uint64(48))
        else:
            t.ask_node[:] = i % t.n_nodes
            t.ask_req[:, 0] = 1                      # all can fit their node
        rows = []
        check(shim, oracle, t, batch=t.n_asks, rows=rows, tag=field)
        sig = np.column_stack([t.ask_req, t.ask_tol.astype(np.int64), t.ask_need.astype(np.int64), t.ask_deny.astype(np.int64), t.ask_node])
        distinct = len(np.unique(sig, axis=0))
        assert distinct >= min(t.n_asks, t.n_nodes), field        # the fixture really separates the asks
        assert rows[0] >= distinct, (field, rows, distinct)


def test_shared_rows_survive_hash_collisions(shim, oracle):
    """the signature hash only finds candidates: with every hash equal (share_rows=2 in the harness) rows are still
    shared exactly between asks whose full signatures are equal, and the bindings do not change"""
    for seed in (0, 3, 7, 11):
        s = synth.fuzz(seed)
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > 64:
            continue
        good, collide = [], []
        check(shim, oracle, s, batch=64, rows=good, tag=seed)
        check(shim, oracle, s, batch=64, share_rows=2, rows=collide, tag=seed)
        assert good == collide
    s = synth.perf(300, 20, 40)
    good, collide = [], []
    check(shim, oracle, s, batch=128, rows=good)
    check(shim, oracle, s, batch=128, share_rows=2, rows=collide)
    assert good == collide


def test_cut_cycle_leaves_no_tentative_gang_members(shim, oracle):
    """placement-insensitive order + gangs + max_bindings: members queued behind the cut must read PENDING again"""
    s = synth.gangs(200, 40, 5, fill=0.5)
    full = oracle.run(s)
    k = (len(full["ask"]) // 2) // 5 * 5 + 5
    want = oracle.run(s, max_bindings=k)
    rc, ask, node, state, avail = run_engine_host(shim, s, batch=20, max_bindings=k)
    assert rc == 0
    assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
    assert set(np.unique(state)) <= {0, 1}, np.unique(state)        # pending or allocated, nothing in between
    assert np.array_equal(state, want["state"])


def test_score_bits_match_the_oracle(shim, oracle):
    """csrc/yk_score.h (host build of the code the device runs; it forms usage/W without a divide when W is 1 or 2)
    against the oracle's plain restatement: identical IEEE-754 bits, including tiny and huge operands"""
    shim.score_host.restype = C.c_double
    rng = np.random.default_rng(5)
    cases = 0
    for wts in ([1.0, 1.0, 0.0, 0.0], [1.0, 0.0, 0.0, 0.0], [1.0, 1.0, 1.0, 0.0], [0.5, 1.5, 0.0, 0.0], [2.0, 0.0, 0.0, 0.0],
                [1.0, 1.0, 1.0, 1.0], [0.25, 0.25, 0.5, 1.0]):
        w = np.array(wts, dtype=np.float64)
        for _ in range(3000):
            mag = rng.integers(0, 62, size=4)
            total = (rng.integers(0, 1 << 62, size=4) >> (62 - mag)).astype(np.int64)
            total[rng.random(4) < 0.1] = 0
            avail = (total * rng.random(4)).astype(np.int64)
            if rng.random() < 0.2:
                avail = avail - rng.integers(0, 5, size=4)            # slightly negative / over-committed
            if rng.random() < 0.1:
                avail = total.copy()                                 # empty node: shares exactly 0
            if rng.random() < 0.05:
                avail = total - 1                                    # shares of 1 ulp-ish size
            for policy in (0, 1):
                got = shim.score_host(C.c_int(4), C.c_uint32(policy), _p(w), _p(total), _p(avail))
                want = oracle.node_score(policy, w, total, avail)
                assert np.float64(got).tobytes() == np.float64(want).tobytes() or (got != got and want != want), \
                    (wts, total, avail, policy, got, want)
                cases += 1
    assert cases > 40000


def test_reference_e2e_scenarios_through_the_host_engine(shim, oracle):
    """the two behaviour-level known answers the reference's e2e suites give for this path (priority order across
    sibling queues, binpacking node order; tests/test_oracle_golden.py states them) through the real orderer + commit"""
    done = []
    for expect in ("high", "normal", "low"):
        s = synth.priority_fence(quota_pods=1, done=done)
        for batch in (1, 64):
            rc, ask, node, state, avail = run_engine_host(shim, s, batch=batch)
            assert rc == 0 and [s.meta["apps"][a] for a in ask] == [expect]
        check(shim, oracle, s, batch=8)
        done.append(expect)
    s = synth.priority_fence(quota_pods=3)
    rc, ask, node, state, avail = run_engine_host(shim, s, batch=2)
    assert [s.meta["apps"][a] for a in ask] == ["high", "normal", "low"]
    s = synth.binpacking_e2e()
    rc, ask, node, state, avail = run_engine_host(shim, s, batch=4)
    assert [s.node_id[n] for n in node] == ["nodeA"] * 3 + ["nodeB"] * 3
    check(shim, oracle, s, batch=4)
    done = []
    for expect in ("high", "normal", "low"):                      # the same order from queue offsets (:179-251)
        s = synth.priority_offsets(quota_pods=1, done=done)
        for batch in (1, 64):
            rc, ask, node, state, avail = run_engine_host(shim, s, batch=batch)
            assert rc == 0 and [s.meta["apps"][a] for a in ask] == [expect]
        check(shim, oracle, s, batch=8)
        done.append(expect)
    from test_oracle_golden import _fence_snapshot
    for fenced, want in ((False, [2, 3, 0, 1]), (True, [0, 2, 1, 3])):
        s = _fence_snapshot(fenced)
        for batch in (1, 3, 64):
            for spec in (0, 1):
                rc, ask, node, state, avail = run_engine_host(shim, s, batch=batch, speculate=spec)
                assert rc == 0 and list(ask) == want, (fenced, batch, spec)


@pytest.mark.parametrize("prio", [False, True])
def test_speculated_empty_batch_is_undone_too(shim, oracle, prio):
    """a cluster far too small for its queues' quotas (tests/test_gpu_parity.py::test_config4_overcommitted_rewinds): near
    the end every in-flight batch fails at its first ask while the batch speculated behind it comes out EMPTY -- but has
    marked the remaining asks SKIPPED against a quota that the failing asks never consumed.  Those marks must be rolled
    back like any other speculated decision (they once were not: the asks ended SKIPPED where the oracle says NOFIT)."""
    s = synth.hier(6, 3, 3, 2, 60, priorities=prio, seed=22)
    for batch in (8, 64, 256):
        for spec in (0, 1):
            want = check(shim, oracle, s, tag=(batch, spec), batch=batch, speculate=spec)
    assert (want["state"] == 2).sum() > 100
    for nodes in (4, 6):          # the same shape over more seeds: about a third of them hit the condition
        for seed in range(12):
            s = synth.hier(nodes, 3, 3, 2, 60, priorities=prio, seed=seed)
            check(shim, oracle, s, tag=(nodes, seed), batch=64, speculate=1)


def test_gpu_suite_snapshots_through_the_host_engine(shim, oracle):
    """every single-cycle snapshot of tests/test_gpu_parity.py (minus the full-size ones), so that a change to the orderer
    or the commit that would fail on the GPU box already fails here"""
    cases = []
    for variant in ("bare", "sized"):
        for pol in (synth.POLICY_FAIR, synth.POLICY_BINPACKING):
            cases.append((synth.kwok(100, 10, 50, variant=variant, policy=pol), 128))
    for b in (64, 1000, 4096):
        cases.append((synth.perf(700, 20, 100), b))
    for pol in (synth.POLICY_FAIR, synth.POLICY_BINPACKING):
        cases.append((synth.perf(900, 20, 100, masks=True, policy=pol), 512))
        cases.append((synth.gangs(60, 40, 5, fill=1.4, policy=pol), 64))
    cases.append((synth.perf(8, 10, 200, masks=True), 256))
    for prio in (False, True):
        cases.append((synth.hier(300, 3, 4, 2, 40, masks=True, priorities=prio, seed=21), 128))
    cases.append((synth.hier(200, 2, 3, 3, 30, masks=True, priorities=True, seed=23, leaf_sort=synth.SORT_FAIR), 64))
    s = synth.hier(30, 2, 3, 2, 24, seed=9)
    s.ask_gang[:] = np.arange(s.n_asks) // 4
    cases.append((s, 32))
    s = synth.perf(5, 2, 10); s.node_flags[:] = 0; cases.append((s, 16))
    s = synth.perf(5, 2, 10); s.ask_req[::3] = 0; cases.append((s, 16))
    s = synth.perf(5, 2, 10); s.ask_flags[::2] = 1; cases.append((s, 16))
    s = synth.perf(9, 2, 10); s.ask_node[:] = 3; cases.append((s, 16))
    s = synth.perf(9, 2, 10); s.node_flags[4] = synth.NODE_SCHEDULABLE | synth.NODE_RESERVED; s.node_avail[2, 0] = -5000
    cases.append((s, 16))
    for s, b in cases:
        check(shim, oracle, s, tag=(s.name, b), batch=b)


def test_randomized_queue_trees_through_the_host_engine(shim, oracle):
    """random queue trees on clusters from far too small to roomy: priorities on/off, fair or fifo leaves, both node
    policies, masks, gangs -- every run with and without the speculative next batch.  (The overcommitted ones are what
    exercises rewind after rewind; this family found the 'empty speculated batch' bug once the GPU suite had shown it.)"""
    import random
    rng = random.Random(1)
    runs = 0
    for it in range(120):
        nn = rng.choice([3, 6, 10, 25, 80])
        par, lv, apps, tasks = rng.randrange(1, 4), rng.randrange(1, 4), rng.randrange(1, 4), rng.choice([5, 20, 60])
        s = synth.hier(nn, par, lv, apps, tasks, masks=rng.random() < 0.3, priorities=rng.random() < 0.7, seed=rng.randrange(1000),
                       leaf_sort=rng.choice([synth.SORT_FAIR, synth.SORT_FIFO]), policy=rng.choice([synth.POLICY_FAIR, synth.POLICY_BINPACKING]))
        if rng.random() < 0.3:
            g = rng.choice([2, 4, 5])
            if tasks % g == 0:
                s.ask_gang[:] = np.arange(s.n_asks) // g
        if rng.random() < 0.4:       # queue priority properties: offsets and fences
            s.q_prio_offset = np.array([rng.choice([0, 0, 5, -5, 100]) for _ in range(s.n_queues)], dtype=np.int32)
            s.q_prio_fence = np.array([rng.random() < 0.25 for _ in range(s.n_queues)], dtype=np.uint8)
        for b in (8, 64, 256):
            if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > b:
                continue
            for spec in (0, 1):
                check(shim, oracle, s, tag=(it, s.name, b, spec), batch=b, speculate=spec)
                runs += 1
    assert runs > 500


def test_max_bindings_and_a_gang_sunk_by_its_own_members(shim, oracle):
    """max_bindings ends the cycle at a gang that would need more bindings than are left -- unless the gang is sunk by its
    queue-side checks (an invalid / slow-path member, no headroom): that gang needs no room, gets its cause, and the
    cycle goes on.  (Found by scripts/host_campaign.py: the static order of a single-leaf cycle already behaved that way,
    the oracle and the tree walk stopped at the gang.)"""
    from oracle import py_oracle
    s = synth.fuzz(17513)                       # ask 70 is binding #53; then a 3-member gang with an invalid member; then ask 77
    for k in (53, 54, 55, 60):
        want = oracle.run(s, max_bindings=k)
        assert len(want["ask"]) == min(k, len(oracle.run(s)["ask"]))
        p = py_oracle.run(s, max_bindings=k)
        assert list(want["ask"]) == p["ask"] and list(want["node"]) == p["node"]
        for b in (8, 64, 300):
            for spec in (0, 1):
                rc, ask, node, state, avail = run_engine_host(shim, s, batch=b, max_bindings=k, speculate=spec)
                assert rc == 0 and np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"]), (k, b, spec)


@pytest.mark.parametrize("D", [1, 2, 3, 5, 8])
def test_other_dimension_counts(shim, oracle, D):
    """the commit's node record and the orderer's accounting are sized by D (1..8): same snapshots, other widths"""
    from oracle import py_oracle
    n = 0
    for seed in range(0, 60, 4):
        s = synth.redim(synth.fuzz(seed), D, seed)
        try:
            want = oracle.run(s)
        except RuntimeError:
            continue                              # a zero total on a weighted dimension: NaN score, rejected up front
        if seed % 12 == 0:
            p = py_oracle.run(s)
            assert list(want["ask"]) == p["ask"] and list(want["node"]) == p["node"]
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > 64:
            continue
        check(shim, oracle, s, tag=(seed, D), batch=64)
        n += 1
    assert n >= 8


def test_extreme_priorities_and_everything_tied(shim, oracle):
    """identical nodes, identical requests, priorities at the int32 limits (the application key once stored -priority in
    32 bits: -INT32_MIN wrapped and the application sorted last instead of first), extreme queue offsets"""
    import random
    rng = random.Random(4)
    runs = 0
    for it in range(60):
        nn = rng.choice([1, 2, 5, 33, 64, 65])
        s = synth.hier(nn, rng.randrange(1, 3), rng.randrange(1, 4), rng.randrange(1, 3), rng.choice([4, 16, 50]),
                       seed=rng.randrange(1000), leaf_sort=rng.choice([synth.SORT_FIFO, synth.SORT_FAIR]),
                       policy=rng.choice([synth.POLICY_FAIR, synth.POLICY_BINPACKING]), quota_frac=rng.choice([1.0, 3.0]))
        s.node_total[:] = s.node_total[0]
        s.node_avail[:] = s.node_total
        s.ask_req[:] = s.ask_req[0]
        s.ask_prio[:] = np.array([rng.choice([-(1 << 31), (1 << 31) - 1, 0, 1, -1]) for _ in range(s.n_asks)], dtype=np.int32)
        if rng.random() < 0.5:
            s.q_prio_offset = np.array([rng.choice([0, (1 << 31) - 1, -(1 << 31), 7]) for _ in range(s.n_queues)], dtype=np.int32)
            s.q_prio_fence = np.array([rng.random() < 0.3 for _ in range(s.n_queues)], dtype=np.uint8)
        for b in (7, 64):
            check(shim, oracle, s, tag=(it, b), batch=b, speculate=it % 2)
            runs += 1
    assert runs == 120
