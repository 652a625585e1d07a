"""The round commit (csrc/yk_rounds.h) on the GPU at the edges where its device-only code differs from the CPU build.

tests/test_rounds_host.py runs the header's `#else` branches.  On the device the same rounds run through a shuffle scan
and a cross-warp exclusive minimum (block_prefmin), a warp-bounded merge (merge_into), a register bitonic sort
(block_sort_fast), block_scan, warp_append and the red_* reductions.  A round that stops too early is still exact -- the
next round or a single step decides the same ask, only more slowly -- so bindings alone can hide a device fault.  The shim
(tests/host/rounds_shim.cpp) runs the same deterministic rounds under the engine's own driver, so here every case runs
twice: through the C ABI under the default `auto` commit, and through the shim with the same window, guard and uniform
minimum.  Bindings, node choices, final availability and ask states must equal the oracle's; passes, single steps, round
asks, hand-offs and uniform asks must equal the shim's exactly.

Part B replays long mask-free sessions (node resizes, foreign occupancy, cordons, reservations, taints, tied renames,
removals below n_hi) on the round commit and requires every cycle with work to have been decided by rounds.  The CPU tests
check the fixtures themselves: both oracles agree, every round case is round-eligible, and the shim matches the oracle on
every fixture, so that a GPU failure here points at device-only code."""
import functools

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from oracle import py_oracle
from test_rounds_host import ALL, check, infinite_shares, maskfree, rshim, shrunk  # noqa: F401  (rshim: the shim fixture)
from test_engine_host import run_engine_host
from test_gpu_dims import ST_PENDING, YK_ERR_RANGE, _device_eligible, extreme, nan_node, nan_repaired, widen
import test_sessions as ts

GI, MI = synth.GI, synth.MI
NO_UNIFORM = 1 << 30      # YK_UNIFORM_MIN that no run reaches: identical asks stay in round stretches (0 would turn the
                          # device commit off)
GUARD = 32                # the engine's own guard (ykrd::GUARD)
WCAP = 1024               # candidates per round at most (ykrd::WCAP)
# device counter -> shim counter (tests/host/rounds_shim.cpp stats order, test_rounds_host.STATS)
COUNTERS = {"round_passes": "passes", "round_single_steps": "singles", "round_asks": "round_asks",
            "lattice_handoffs": "handoffs", "uniform_asks": "uniform_asks"}
PY_ORACLE_PAIRS = 1_500_000   # node x ask pairs above which the Python oracle takes minutes (it is an exhaustive argmin)


class Run:
    """one snapshot and the knobs both sides use: candidates per round, the guard, the shortest uniform run, a max_bindings
    cut; `rounds` False for the routing cases that must NOT take rounds; `expect(counters)` what the case targets"""
    def __init__(self, snap, window=WCAP, guard=0, umin=NO_UNIFORM, mb=None, rounds=True, expect=None):
        self.snap, self.window, self.guard, self.umin, self.mb = snap, window, guard, umin, mb
        self.rounds, self.expect = rounds, expect

    def __repr__(self):
        return f"{self.snap.name} (window {self.window}, guard {self.guard}, uniform min {self.umin}, max_bindings {self.mb})"


def insensitive(s):
    """one fifo leaf, no max, one priority: a placement-insensitive order (NOFIT fails in place)"""
    s.q_max[:] = -1
    s.q_sort[:] = 0
    s.ask_prio[:] = 0
    s.app_queue[:] = s.app_queue[0]
    return s


def _whole(c):
    return c["round_asks"] > 0 and c["lattice_handoffs"] == 0


# ---- A. the fixtures ----
def fuzz_runs(D):
    """mask-free fuzz made placement-insensitive; configured weights on some seeds, +-Inf shares on some at D >= 2 (seeds
    with a NaN score are skipped by both sides: the oracle rejects them), and one config-2 shape taken entirely by rounds"""
    runs = []
    for seed in range(12):
        s = insensitive(maskfree(synth.redim(synth.fuzz(seed), D, seed)))
        s.policy = synth.POLICY_FAIR
        if seed % 3 == 1:
            s = synth.reweigh(s, np.linspace(0.25, 2.0, D))
        if seed % 4 == 2 and D >= 2 and s.n_nodes > 3:
            s = infinite_shares(s)
        s.name += f"-fuzz{seed}"
        runs.append(Run(s, guard=0 if seed % 2 else GUARD))
    s = maskfree(synth.redim(synth.perf(600, 12, 60), D, 3))
    runs.append(Run(s, expect=lambda c, n=s.n_asks: c["round_asks"] == n and c["lattice_handoffs"] == 0))
    return runs


def ladder(n_nodes=1200, n_asks=2400, seed=0):
    """node keys climb in steps of ~1/6 400 (10 mCPU of 32 CPU, vcore only): an allocation of 100..1 000 mCPU moves a node
    10..100 positions back, so a round stops where a node taken earlier -- often in an earlier warp -- now sorts before the
    next candidate, and the cross-warp minimum decides m.  A quarter of the asks request pods only (no weighted resource):
    the node keeps its key, and only an exclusive prefix minimum lets such a candidate be taken."""
    rng = np.random.default_rng(seed)
    s = synth.perf(n_nodes, n_asks // 100, 100, seed=seed + 20)
    s.node_total[:] = [32_000, 256 * GI, 1000, 0]
    s.node_avail[:] = s.node_total
    s.node_avail[:, 0] -= 10 * rng.permutation(n_nodes)
    s.node_id = [f"n{x:05d}" for x in rng.permutation(n_nodes)]          # NodeID ranks unrelated to the keys
    s.ask_req[:] = 0
    s.ask_req[:, 0] = rng.choice([100, 250, 400, 1000], n_asks)
    s.ask_req[:, 2] = 1
    s.ask_req[rng.random(n_asks) < 0.25, 0] = 0
    s.name = f"ladder-{n_nodes}x{n_asks}"
    return s


def long_order(n_front):
    """n_front empty small nodes sort first (key 0) and take the small asks, but reject the large ones by capacity without
    being spent; the first large node sits at position n_front.  The first ask is large: a single step whose hit is exactly
    there (1 055: lane 31 of the second chunk of 1 024; 2 048: lane 0 of the third; 2 061: mid-warp)."""
    s = synth.perf(n_front + 300, 16, 40, seed=5)
    s.node_total[:n_front] = [2000, 8 * GI, 110, 0]
    s.node_total[n_front:] = [32_000, 256 * GI, 110, 0]
    s.node_avail[:] = s.node_total
    s.node_avail[n_front:, :2] -= s.node_total[n_front:, :2] // 10
    s.node_id = [f"n{i:05d}" for i in range(s.n_nodes)]                   # rank = index: the front is exactly the small nodes
    s.ask_req[:] = [100, 128 * MI, 1, 0]
    s.ask_req[::31] = [4000, 16 * GI, 1, 0]
    s.name = f"long-order-{n_front}"
    return s


def spent_many():
    """one pod per node: every node leaves the order with its first allocation, ~2 700 of them in one stretch (the return
    merge runs in three chunks of 1 024); cordoned, reserved, over-committed and zero-capacity nodes scattered over the rank
    order leave at once; 3 000 asks for ~2 700 usable nodes: the cluster fills up and the rest fail in place"""
    s = synth.perf(3000, 40, 75, seed=9)
    s.node_total[:, 2] = s.node_avail[:, 2] = 1
    s.node_flags[::37] = 0
    s.node_flags[5::41] |= synth.NODE_RESERVED
    s.node_avail[7::43, 0] = -1000
    s.node_total[11::47, 2] = s.node_avail[11::47, 2] = 0
    s.name = "spent-many"
    return s


def ties():
    """2 000 identical empty nodes whose NodeID ranks are shuffled against their indices, 5 000 identical asks kept out of
    uniform runs: the re-keyed nodes tie on key and only the rank orders them"""
    s = synth.reference_shape(2000, 40, 125)
    s.node_id = [f"n{x:05d}" for x in np.random.default_rng(6).permutation(s.n_nodes)]
    s.name = "ties"
    return s


def runs_between(D):
    """small nodes that fill up (spent nodes leave the stretches) and two runs of 300 identical asks inside 10 000 others:
    uniform runs and round stretches alternate, each run reading the order the stretch before it left behind"""
    s = shrunk(widen(synth.perf(1500, 80, 125, seed=11), D, D), 12)
    for lo in (3000, 7000):
        s.ask_req[lo:lo + 300] = s.ask_req[lo]
    s.name += "-runs"
    return s


def guard_trip(D):
    """vcore only weighted, totals 2^60: 300 asks of 2^52 move keys and fill a side list; 60 empty nodes of exactly 2^52
    sort first and are spent (parked) by their first ask; then 500 asks of 1 unit leave every key where it is (2^-60 is
    below half an ulp of a share of 0.5), so every round decides one ask and the guard hands over after 16 passes, with the
    side list non-empty and nodes parked"""
    s = synth.perf(500, 8, 100, seed=12)
    s = synth.redim(s, 1, 0) if D == 1 else widen(s, D, 1)
    w = np.zeros(D)
    w[0] = 1.0
    s = synth.reweigh(s, w)
    big = np.arange(60, 500)
    s.node_total[:60, 0] = s.node_avail[:60, 0] = 1 << 52
    s.node_total[big, 0] = 1 << 60
    s.node_avail[big, 0] = (1 << 59) - (big - 60) * (1 << 45)
    s.node_total[:, 1:] = s.node_avail[:, 1:] = 1000
    s.ask_req[:] = 1
    s.ask_req[:300, 0] = 1 << 52
    s.name = f"guard-trip-D{D}"
    return s


def flat_handoff(D):
    """zero weights: every key is 0, every round decides one ask, the guard hands over after 16 passes"""
    return synth.reweigh(widen(synth.perf(2000, 40, 125), D, D), np.zeros(D))


def routing(case):
    s = synth.perf(800, 16, 50, seed=14)
    s.node_taint[::5] = 1 << 3
    s.ask_tol[:] = (1 << 3) | 1                    # every ask tolerates every taint of the cluster: rounds
    s.name = f"routing-{case}"
    if case == "untolerated":                       # one ask does not: no round pass
        s.ask_tol[17] = 1
    elif case == "queue-max":                       # a max on the queue: placement-sensitive, no round pass
        s.q_max[1, 0] = 1 << 60
    return s


def _mb_base(f=1):
    return shrunk(synth.perf(600, 12, 60, seed=3), f)


CASES = {
    **{f"dims-D{D}": functools.partial(fuzz_runs, D) for D in range(1, 9)},
    "windows": lambda: [Run(ladder(), window=w, expect=lambda c, w=w: c["round_asks"] == 2400 and c["round_passes"] > 2400 // max(w, 100))
                        for w in (1, 3, 31, 32, 33, 64, 1000, 1024)],
    "side-list-overflow": lambda: [Run(synth.perf(3000, 60, 125, seed=8),
                                       expect=lambda c: c["round_asks"] == 7500 and c["round_single_steps"] == 0)],
    "single-steps-long-order": lambda: [Run(long_order(n), expect=lambda c, n=n: c["round_single_steps"] > 0 and _whole(c))
                                        for n in (1055, 2048, 2061)],
    "spent-nodes": lambda: [Run(spent_many(), expect=lambda c: c["parked"] > 2 * WCAP and c["round_single_steps"] > 0 and _whole(c))],
    "key-ties": lambda: [Run(ties(), expect=lambda c: c["round_asks"] == 5000)],
    "uniform-around-stretches": lambda: [Run(runs_between(D), umin=200,
                                             expect=lambda c: c["uniform_asks"] >= 600 and c["round_asks"] > 0 and c["stretches"] >= 3
                                             and c["parked"] > 0) for D in (1, 8)],
    "guard-handoff": lambda: [Run(guard_trip(D), guard=GUARD,
                                  expect=lambda c: c["lattice_handoffs"] == 1 and c["round_passes"] == 16 and c["parked"] >= 60
                                  and 300 <= c["round_asks"] < 400) for D in (1, 8)]
                             + [Run(flat_handoff(D), guard=GUARD,
                                    expect=lambda c: c["lattice_handoffs"] == 1 and c["round_asks"] == 16) for D in (1, 8)],
    "max-bindings": lambda: [Run(_mb_base(), mb=1, expect=lambda c: c["round_asks"] == 1),
                             Run(_mb_base(), mb=100, expect=lambda c: c["round_asks"] == 100),
                             Run(_mb_base(), window=64, mb=500, expect=lambda c: c["round_asks"] == 500 and c["round_passes"] >= 8),
                             Run(_mb_base(40), mb=300, expect=lambda c: c["round_asks"] > 300 and c["round_single_steps"] > 0)],
    "extreme": lambda: [Run(extreme(D), expect=lambda c: c["round_asks"] == 240 and c["lattice_handoffs"] == 0) for D in (1, 4, 8)],
    "routing": lambda: [Run(routing("tolerated"), expect=lambda c: c["round_asks"] == 800 and c["lattice_handoffs"] == 0),
                        Run(routing("untolerated"), rounds=False), Run(routing("queue-max"), rounds=False)],
}


@functools.lru_cache(maxsize=None)
def case_runs(name):
    return CASES[name]()


def all_runs():
    for name in CASES:
        for r in case_runs(name):
            yield name, r


def _shim(rshim, oracle, r):
    """the shim on the run's snapshot and knobs -> (oracle result or None for a NaN snapshot, counters by device name)"""
    want, st = check(rshim, oracle, r.snap, tag=repr(r), uniform=(r.umin, 0), window=r.window, guard=r.guard,
                     batch=1 << 16, max_bindings=r.mb)
    c = {dev: st[sh] for dev, sh in COUNTERS.items()}
    c.update(parked=st["parked"], stretches=st["round_stretches"])
    return want, c


def _knobs(monkeypatch, r):
    monkeypatch.setenv("YK_ROUND_MIN", "1")
    monkeypatch.setenv("YK_ROUND_GUARD", str(r.guard))
    monkeypatch.setenv("YK_ROUND_WINDOW", str(r.window))
    monkeypatch.setenv("YK_UNIFORM_MIN", str(r.umin))


def _device(monkeypatch, r, want):
    from yunikorn_k8shim_b200 import Engine
    s = r.snap
    _knobs(monkeypatch, r)
    with Engine.for_snapshot(s, batch=4096) as e:
        ask, node, _ = e.cycle(s.n_asks if r.mb is None else r.mb)
        avail = e.nodes_available(np.arange(s.n_nodes))
        states = e.ask_states(np.arange(s.n_asks))
        st = e.stats()
    assert np.array_equal(ask, want["ask"]), ("ask order differs", r)
    assert np.array_equal(node, want["node"]), ("node choice differs", r)
    assert np.array_equal(avail, want["avail"]), ("final availability differs", r)
    if r.mb is None:
        assert np.array_equal(states, want["state"]), ("ask states differ", r)
    return st


# ---- A. on the GPU ----
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_round_commit_matches_oracle_and_shim(rshim, oracle, monkeypatch, name):
    ran = 0
    for r in case_runs(name):
        want, shim = _shim(rshim, oracle, r)
        if want is None:
            continue                              # a NaN score: test_nan_snapshot_on_the_round_route
        st = _device(monkeypatch, r, want)
        got = {k: st[k] for k in COUNTERS}
        assert got == {k: shim[k] for k in COUNTERS}, (r, "device", got, "shim", shim)
        if r.rounds:
            assert st["lattice_cycles"] == 1 and st["round_asks"] > 0, (r, st["lattice_cycles"])
        else:
            assert st["round_passes"] == 0 and st["lattice_cycles"] == 0, r
        if r.expect is not None:
            assert r.expect({**shim, **got}), (r, shim)
        ran += 1
    assert ran >= (8 if name.startswith("dims") else 1)


@pytest.mark.gpu
def test_nan_snapshot_on_the_round_route(rshim, oracle, monkeypatch):
    """node 5 scores NaN: the cycle on the round route is a clean YK_ERR_RANGE (nothing bound, every ask pending, the node
    tables unchanged); with node 5 repaired the next cycle on the same engine is the oracle's, by rounds, with the shim's
    counters"""
    from yunikorn_k8shim_b200 import Engine, YkError
    s = nan_node()
    t = nan_repaired(s)
    r = Run(t)
    want, shim = _shim(rshim, oracle, r)
    assert shim["round_asks"] == t.n_asks
    A, N = np.arange(s.n_asks), np.arange(s.n_nodes)
    _knobs(monkeypatch, r)
    with Engine.for_snapshot(s, batch=4096) as e:
        with pytest.raises(YkError) as ei:
            e.cycle(s.n_asks)
        assert ei.value.code == YK_ERR_RANGE
        st = e.stats()
        assert st["allocations"] == 0 and st["lattice_cycles"] == 1 and st["round_asks"] == 0
        assert (e.ask_states(A) == ST_PENDING).all()
        assert np.array_equal(e.nodes_available(N), s.node_avail)
        e.nodes_upsert([5], t.node_total[[5]], t.node_avail[[5]], t.node_taint[[5]], t.node_label[[5]], s.node_rank()[[5]],
                       t.node_flags[[5]])
        ask, node, _ = e.cycle(s.n_asks)
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
        assert np.array_equal(e.nodes_available(N), want["avail"])
        assert np.array_equal(e.ask_states(A), want["state"])
        st2 = e.stats()
    assert st2["lattice_cycles"] == 2
    assert {k: st2[k] - st[k] for k in COUNTERS} == {k: shim[k] for k in COUNTERS}


# ---- A. on the CPU ----
def _placement_insensitive(s):
    leaves = set(int(q) for q in s.app_queue[np.unique(s.ask_app)])
    if len(leaves) != 1 or len(set(s.ask_prio.tolist())) > 1:
        return False
    if getattr(s, "q_prio_offset", None) is not None and np.any(s.q_prio_offset):
        return False
    if getattr(s, "q_prio_fence", None) is not None and np.any(s.q_prio_fence):
        return False
    if getattr(s, "ul_queue", None) is not None and len(s.ul_queue):
        return False
    q = leaves.pop()
    if s.q_sort[q] != 0:
        return False
    while q >= 0:
        if (s.q_max[q] != -1).any():
            return False
        q = int(s.q_parent[q])
    return True


def _mask_free(s):
    taints = np.bitwise_or.reduce(s.node_taint) if s.n_nodes else np.uint64(0)
    return bool((s.ask_need == 0).all() and (s.ask_deny == 0).all() and (s.ask_node < 0).all() and (s.ask_gang < 0).all()
                and ((taints & ~s.ask_tol) == 0).all())


def test_fixtures_are_round_eligible():
    """every round case is mask-free, placement-insensitive and accepted by the device commit; the routing cases fail
    exactly one of the first two"""
    n = 0
    for name, r in all_runs():
        s = r.snap
        assert _device_eligible(s), (name, r)
        if r.rounds:
            assert _mask_free(s) and _placement_insensitive(s), (name, r)
        else:
            assert _mask_free(s) != _placement_insensitive(s), (name, r)
        n += 1
    assert n > 100


@pytest.mark.parametrize("name", list(CASES))
def test_shim_matches_oracle(rshim, oracle, name):
    """the shim (the kernel's own code, CPU build) decides every fixture as the oracle does and hits what the case targets;
    the GPU test compares the device's counters with these"""
    ran = 0
    for r in case_runs(name):
        want, c = _shim(rshim, oracle, r)
        if want is None:
            continue
        assert (c["round_asks"] > 0) == r.rounds, (r, c)
        if r.expect is not None:
            assert r.expect(c), (r, c)
        ran += 1
    assert ran >= (8 if name.startswith("dims") else 1)


def test_nan_snapshot_fixture(rshim, oracle):
    with pytest.raises(RuntimeError):
        oracle.run(nan_node())
    rc, *_ = run_engine_host(rshim, nan_node(), fn="rounds_host_run", batch=1 << 16)
    assert rc == YK_ERR_RANGE
    _, c = _shim(rshim, oracle, Run(nan_repaired(nan_node())))
    assert c["round_asks"] == 5000


def test_fixtures_oracles_agree(oracle):
    """both oracle restatements (C++ and Python) agree on every fixture above, where the Python one runs in seconds; the
    largest fixtures (side list, spent nodes, key ties, long orders, runs between stretches) are left to the C++ oracle"""
    n = 0
    for name, r in all_runs():
        s = r.snap
        if s.n_nodes * s.n_asks > PY_ORACLE_PAIRS:
            continue
        mb = -1 if r.mb is None else r.mb
        try:
            w = oracle.run(s, mb)
        except RuntimeError:
            with pytest.raises(Exception):
                py_oracle.run(s, mb)
            continue
        p = py_oracle.run(s, mb)
        assert list(w["ask"]) == p["ask"] and list(w["node"]) == p["node"], (name, r)
        if r.mb is None:
            assert list(w["state"]) == p["state"], (name, r)
        n += 1
    assert n > 90


# ---- B. mask-free sessions on the round commit ----
TOL_ALL = np.uint64(ALL)
LEAF = ts.LEAVES[0]


class MaskFreeGenerator(ts.Generator):
    """test_sessions.Generator with every application in one fifo leaf at priority 0, no queue max, no user limits, no
    gangs, asks that tolerate everything and carry no labels or node name; the node operations are all kept"""

    def new_asks(self):
        m, rng = self.m, self.rng
        apps = np.nonzero(m.p_present)[0]
        if not len(apps):
            return
        p = int(rng.choice(apps))
        if rng.random() < 0.25:                       # identical asks: round stretches, not uniform runs
            idx = self.ask_indices(int(rng.integers(8, 21)))
            if idx:
                m.asks_upsert(idx, ts._ask_shape(rng, m.D), p, TOL_ALL, text="asks_upsert(run)")
                m.note("asks_uniform_run")
        else:
            idx = self.ask_indices(int(rng.integers(1, 10)))
            if idx:
                m.asks_upsert(idx, np.stack([ts._ask_shape(rng, m.D) for _ in idx]), p, TOL_ALL)
                m.note("asks_new")

    def reupsert_asks(self):
        m, rng = self.m, self.rng
        cand = [a for a in np.nonzero(m.a_state == ts.PENDING)[0] if m.p_present[m.a_app[a]]]
        if cand:
            for a in sorted(rng.choice(cand, min(len(cand), int(rng.integers(1, 6))), replace=False).tolist()):
                m.asks_upsert([a], ts._ask_shape(rng, m.D), m.a_app[a], TOL_ALL, text="asks_upsert(re-upsert)")
            m.note("asks_reupsert")

    def new_app(self):
        m = self.m
        live = set(m.a_app[:m.a_hi][m.a_state[:m.a_hi] != ts.ABSENT].tolist())
        free = [p for p in range(m.maxP) if not m.p_present[p] and p not in live]
        if free:
            m.apps_upsert([free[0]], LEAF)
            m.note("apps_upsert")

    def queues(self, first=False):
        m, rng = self.m, self.rng
        guar = np.full((m.maxQ, m.D), -1, np.int64)
        for q in range(1, m.maxQ):
            if rng.random() < 0.5:
                guar[q, 0] = int(rng.integers(1, 20)) * 1000
        m.queues_set(guar, np.full((m.maxQ, m.D), -1, np.int64), np.zeros(m.maxQ, np.uint8))
        if not first:
            m.note("queues_set")

    def priorities(self):
        pass

    def limits(self):
        pass

    def start(self, n_nodes, n_apps=4):
        m, rng = self.m, self.rng
        self.queues(first=True)
        m.apps_upsert(list(range(n_apps)), LEAF)
        tied = int(rng.integers(3, 7))
        shape = ts._node_shape(rng, m.D)
        for n in range(n_nodes):
            ts._random_node(m, n, rng, shape if n < tied else None)
        m.nodes_upsert(list(range(n_nodes)), "nodes_upsert(initial)")
        for _ in range(3):
            self.new_asks()


SESSIONS = [(s, 4) for s in range(10)] + [(10, 1), (11, 8)]


@functools.lru_cache(maxsize=None)
def maskfree_session(seed, D=4):
    from oracle import oracle_ctypes
    oracle_ctypes.build()
    rng = np.random.default_rng([seed, D, 61])
    m = ts.Model(oracle_ctypes, f"maskfree-session(seed={seed}, D={D})", D, synth.POLICY_FAIR, max_nodes=128, max_asks=1024,
                 seed=seed + 1000 * D)
    g = MaskFreeGenerator(m, rng)
    g.start(int(rng.integers(12, 40)))
    for c in range(int(rng.integers(12, 31))):
        if c:
            g.step()
        m.check_conservation()
        m.cycle(*g.max_bindings())
        m.check_conservation()
    ts.finish(m)
    return m


def _has_work(c):
    """the cycle binds something or fails something in place: a valid ask (no slow path, some request, none negative), a
    binding allowed, a usable node"""
    s = c.snap
    valid = (s.ask_flags == 0) & (s.ask_req >= 0).all(axis=1) & (s.ask_req > 0).any(axis=1)
    usable = ((s.node_flags & ts.SCHED) != 0) & ((s.node_flags & ts.RESERVED) == 0)
    return bool(valid.any()) and c.max_bindings != 0 and bool(usable.any())


@pytest.mark.gpu
@pytest.mark.parametrize("batch", [64, 4096])
@pytest.mark.parametrize("seed,D", SESSIONS, ids=[f"seed{s}-D{d}" for s, d in SESSIONS])
def test_maskfree_session_on_the_round_commit(monkeypatch, seed, D, batch):
    """every cycle equals the model (oracle) bit for bit, and every cycle with work was decided by rounds -- otherwise the
    session silently tested the host commit"""
    monkeypatch.setenv("YK_ROUND_MIN", "1")
    monkeypatch.setenv("YK_ROUND_GUARD", "0")      # test_sessions._stats_ok allows hand-offs only with gangs
    monkeypatch.setenv("YK_UNIFORM_MIN", str(NO_UNIFORM))
    m = maskfree_session(seed, D)
    per = []
    ts.replay(m, "auto", batch, on_cycle=lambda e, c, d: per.append((c, d)))
    worked = 0
    for c, d in per:
        if _has_work(c):
            assert d["lattice_cycles"] == 1 and d["round_asks"] > 0, (m.name, batch, c.number, d["lattice_cycles"], d["round_asks"])
            worked += 1
    assert worked >= len(per) // 2, (m.name, worked, len(per))


# ---- B. on the CPU ----
@pytest.mark.parametrize("seed,D", SESSIONS, ids=[f"seed{s}-D{d}" for s, d in SESSIONS])
def test_maskfree_sessions_oracles_agree(seed, D):
    """every cycle's snapshot: both oracles agree, and it is mask-free and placement-insensitive"""
    m = maskfree_session(seed, D)
    ts._oracles_agree(m, every=1)
    for c in ts._cycles(m):
        assert _mask_free(c.snap) and _device_eligible(c.snap), (m.name, c.number)
        assert c.snap.n_asks == 0 or _placement_insensitive(c.snap), (m.name, c.number)


def test_maskfree_sessions_cover_node_changes():
    total = {}
    for args in SESSIONS:
        for k, v in maskfree_session(*args).count.items():
            total[k] = total.get(k, 0) + v
    need = {"node_resize": 5, "node_foreign_occupancy": 5, "node_cordon": 3, "node_reserved": 3, "node_taint": 3,
            "rename_tied": 3, "rename_with_allocations": 2, "remove_below_hi": 5, "cycle_after_removal_below_hi": 5,
            "release": 20, "asks_uniform_run": 10, "mb_one": 3, "mb_random": 3}
    short = {k: (total.get(k, 0), n) for k, n in need.items() if total.get(k, 0) < n}
    assert not short, short
