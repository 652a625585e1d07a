"""The device kernels away from the one point the rest of the GPU suite sits on (D = 4 resources, weights vcore = memory = 1).

Every kernel that decides a binding is a template on D = 1..8 (sweep, lattice, uniform runs), the node score has three
quotient branches (total weight 2, 1, anything else), and a zero total on a weighted resource turns a share into +-Inf.
Here each of those is run through the C ABI and compared bit for bit with the oracle -- ask order, node choice, final
availability, ask states -- and every test also checks from the engine's counters that the path it targets really ran,
so a cycle that quietly took another path fails instead of passing.  The CPU test at the end checks that the two oracles
agree on every snapshot built here."""
import copy

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from oracle import py_oracle

DIMS = [1, 2, 3, 5, 6, 7, 8]
FUZZ_SEEDS = range(12)
ST_PENDING = 0
YK_ERR_RANGE = -5
GI = synth.GI


# ---- snapshot builders (each one is also checked on the CPU by test_fixtures_oracles_agree) ----
def fuzz_dims(D, seed):
    return synth.redim(synth.fuzz(seed), D, seed)


def widen(s, D, seed=0):
    """synth.redim, with every added dimension a consistent copy of vcore, memory or pods (redim draws the copied column
    separately for totals, available and requests, which can leave no ask fitting anywhere)"""
    t = synth.redim(s, D, seed)
    for k in range(s.D, D):
        src = (k - s.D + seed) % 3
        t.node_total[:, k], t.node_avail[:, k], t.ask_req[:, k] = s.node_total[:, src], s.node_avail[:, src], s.ask_req[:, src]
    return t


def last_binds(s, seed):
    """the last dimension becomes a scarce resource of its own (an accelerator count, 1..4 per node): a third of the asks
    need one or two, and the node that is first in the order often has too few"""
    s = copy.deepcopy(s)
    rng = np.random.default_rng(seed)
    k = s.D - 1
    tot = rng.integers(1, 5, s.n_nodes)
    s.node_total[:, k] = tot
    s.node_avail[:, k] = tot - rng.integers(0, 2, s.n_nodes)
    s.ask_req[:, k] = rng.choice([0, 0, 0, 0, 1, 1, 2], s.n_asks)
    s.name += "-lastbinds"
    return s


def big(D):
    """over two sweep node tiles (512) and above the lattice's scan window (PMAX 512 / 256) at every D"""
    s = widen(synth.perf(1100, 20, 50, masks=True), D, D)
    return last_binds(s, D) if D >= 2 else s


def runny_big(D):
    return widen(synth.runny(synth.perf(1100, 20, 50), D), D, D)


def tiny_stack(D):
    s = synth.perf(40, 4, 300)
    s.ask_req[:, 0], s.ask_req[:, 1] = 10, 1_000_000
    return widen(s, D, D)


def uniform_shape(D):
    """5 000 identical asks: the shortest reference-shape cycle the default (auto) commit choice decides on the device
    (one uniform run costs about as much as 4 500 asks on the host commit)"""
    return widen(synth.reference_shape(600, 40, 125), D, D)


def gang_handoff(D):
    """300 empty small nodes at the front of the order (key 0), 100 big nodes behind them (10 % used): no gang member fits
    a small node, so the first gang cannot be placed from the front of the order and the device commit hands the rest of
    the cycle to the host commit"""
    s = synth.gangs(400, 30, 4, fill=0.5)
    s.node_total[:300, 0], s.node_total[:300, 1] = 1000, 4 * GI
    s.node_total[300:, 0], s.node_total[300:, 1] = 64_000, 512 * GI
    s.node_avail[:, :2] = s.node_total[:, :2]
    s.node_avail[300:, :2] -= s.node_total[300:, :2] // 10
    s.ask_req[:, 0], s.ask_req[:, 1] = 2000, 8 * GI
    return widen(s, D, D)


def weighted(case):
    base = synth.perf(600, 10, 60, masks=True, seed=3)
    if case == "tw1_second":          # total weight 1 on a dimension other than the first: the `usage` branch
        return synth.reweigh(base, [0, 1, 0, 0])
    if case == "tw1.5":               # a real divide by 1.5
        return synth.reweigh(base, [1, 0.5, 0, 0])
    if case == "tenths":              # 0.1 + 0.2 + 0.3 != 0.6: the order of the running sum shows in the last bit
        return synth.reweigh(widen(base, 3), [0.1, 0.2, 0.3])
    if case == "wide":
        return synth.reweigh(widen(base, 2), [1e-3, 1e3])
    if case == "pods":                # kwok {pods: 1} asks: with a weight on pods their keys move
        return synth.reweigh(synth.kwok(200, 10, 50, variant="bare"), [1, 1, 1, 0])
    if case == "d8":
        return synth.reweigh(widen(base, 8, 5), [1, 1, 0.5, 0.25, 0.5, 0, 0.75, 0.25])   # sums to 4.25
    raise KeyError(case)


WEIGHT_CASES = ["tw1_second", "tw1.5", "tenths", "wide", "pods", "d8"]


def _inf_nodes(s):
    """node 3: total 0 and available < 0 on vcore (+Inf share), node 7: available > 0 (-Inf), node 11: available 0 (0/0,
    the share is skipped); vcore stays weighted"""
    s = copy.deepcopy(s)
    for n, av in ((3, -100), (7, 500), (11, 0)):
        s.node_total[n, 0] = 0
        s.node_avail[n, 0] = av
    return s


def infinite(D):
    s = _inf_nodes(widen(synth.perf(40, 4, 30, seed=7), D, 1))
    s.ask_req[::2, 0] = 0                 # these can land on the zero-vcore nodes
    s.ask_node[0::10] = 3                 # the +Inf node sorts last: some asks name it (pod.Spec.NodeName)
    s.ask_node[2::10] = 11
    return s


def infinite_uniform(D):
    """more identical pods than the cluster holds: every node fills up, the +Inf one last"""
    s = _inf_nodes(widen(synth.reference_shape(12, 12, 125), D, 1))
    s.ask_req[:, 0] = 0
    return s


def nan_node():
    """node 5 has a +Inf and a -Inf share: its score is NaN, which neither the oracle nor the library accepts"""
    s = synth.reference_shape(300, 40, 125)
    s.node_total[5, 0], s.node_avail[5, 0] = 0, -10
    s.node_total[5, 1], s.node_avail[5, 1] = 0, GI
    return s


def nan_repaired(s):
    t = copy.deepcopy(s)
    t.node_total[5, 0] = t.node_avail[5, 0] = 32_000
    t.node_total[5, 1] = t.node_avail[5, 1] = 256 * GI
    return t


def extreme(D, uniform=False):
    """totals and available near 2^62 on the last dimension (weighted), requests of 1 and of about 2^61 on it: reaches the
    64-bit overflow guards of the lattice, the uniform runs' capacity divide and the j * request products.  At most three
    asks request 2^61, so what the queues hold stays below 2^63."""
    rng = np.random.default_rng(D)
    s = widen(synth.reference_shape(60, 4, 60) if uniform else synth.perf(60, 6, 40, seed=13), D, D)
    k = D - 1
    tot = (1 << 62) - rng.integers(0, 1 << 20, s.n_nodes)
    s.node_total[:, k] = tot
    s.node_avail[:, k] = tot - rng.choice([0, 1 << 60, 1 << 61], s.n_nodes) - rng.integers(0, 1 << 10, s.n_nodes)
    s.ask_req[:, k] = 1
    if uniform:
        s.ask_req[:3, k] = (1 << 61) - 12345   # three asks of one run ask for half a node, the rest for one unit
    else:
        s.ask_req[rng.choice(s.n_asks, 3, replace=False), k] = (1 << 61) - rng.integers(0, 1 << 20, 3)
    w = np.array(s.weights)
    w[k] = 1.0
    return synth.reweigh(s, w)


def _device_eligible(s):
    """what the device commit accepts (yklt::eligible): fair node sort, weighted totals >= 0, unique node names, every gang's
    members request one vector"""
    if s.policy != synth.POLICY_FAIR:
        return False
    if (s.node_total[:, s.weights != 0] < 0).any():
        return False
    first = {}
    for a in np.nonzero(s.ask_gang >= 0)[0]:
        key = (int(s.ask_app[a]), int(s.ask_gang[a]))
        if key in first and not np.array_equal(s.ask_req[a], s.ask_req[first[key]]):
            return False
        first.setdefault(key, a)
    return True


# ---- the GPU runs ----
def _engine():
    from yunikorn_k8shim_b200 import Engine
    return Engine


def _run(s, want, **kw):
    with _engine().for_snapshot(s, **kw) as e:
        ask, node, _ = e.cycle(s.n_asks)
        avail = e.nodes_available(np.arange(s.n_nodes))
        states = e.ask_states(np.arange(s.n_asks))
        st = e.stats()
    tag = (s.name, kw)
    assert np.array_equal(ask, want["ask"]), ("ask order differs", tag)
    assert np.array_equal(node, want["node"]), ("node choice differs", tag)
    assert np.array_equal(avail, want["avail"]), ("final availability differs", tag)
    assert np.array_equal(states, want["state"]), ("ask states differ", tag)
    return st


def _host(s, want, **kw):
    st = _run(s, want, commit="host", **kw)
    assert st["lattice_launches"] == 0 and st["lattice_cycles"] == 0
    assert st["sweep_launches"] > 0 or s.n_nodes == 0 or (s.node_flags == 0).all()
    return st


def _device(s, want, **kw):
    st = _run(s, want, commit="device", **kw)
    assert st["lattice_cycles"] == 1 and st["lattice_launches"] > 0, (s.name, st["lattice_cycles"])
    return st


def _both(s, want, **kw):
    return _host(s, want, **kw), _device(s, want, **kw)


# 1. every D, both commits
@pytest.mark.gpu
@pytest.mark.parametrize("D", DIMS)
def test_fuzz_every_dimension_count(oracle, D):
    ran = dev = 0
    for seed in FUZZ_SEEDS:
        s = fuzz_dims(D, seed)
        try:
            want = oracle.run(s)
        except RuntimeError:
            continue                      # a zero total on a weighted dimension: NaN score, rejected up front
        if (s.ask_gang >= 0).any() and np.bincount(s.ask_gang[s.ask_gang >= 0]).max() > 64:
            continue
        _host(s, want, batch=64)
        st = _run(s, want, commit="device", batch=64)
        eligible = _device_eligible(s)
        assert st["lattice_cycles"] == int(eligible), (s.name, eligible)   # forced device commit: every eligible cycle
        assert st["lattice_launches"] > 0 or not eligible or st["uniform_runs"] > 0
        ran += 1
        dev += int(eligible)
    assert ran >= 8 and dev >= 3, (ran, dev)


@pytest.mark.gpu
@pytest.mark.parametrize("D", DIMS)
def test_large_snapshot_every_dimension_count(oracle, D):
    s = big(D)
    want = oracle.run(s)
    assert len(want["ask"]) > 500
    host, dev = _both(s, want, batch=512)
    assert host["sweep_launches"] > 1
    assert dev["lattice_subruns"] > 1 and dev["lattice_asks"] == s.n_asks and dev["sweep_launches"] == 0


@pytest.mark.gpu
@pytest.mark.parametrize("D", DIMS)
def test_uniform_runs_every_dimension_count(oracle, monkeypatch, D):
    monkeypatch.setenv("YK_UNIFORM_MIN", "6")
    s = runny_big(D)
    want = oracle.run(s)
    st = _device(s, want, batch=4096)
    assert st["uniform_asks"] > 0 and st["lattice_subruns"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("D", DIMS)
def test_tiny_requests_stack_every_dimension_count(oracle, D):
    """requests far below the key distance between nodes: a node takes many allocations in a row, so the lattice's boxes
    run deep and the bound just outside them decides which elements are known"""
    s = tiny_stack(D)
    want = oracle.run(s)
    _host(s, want, batch=4096)
    st = _device(s, want, batch=4096)
    assert st["lattice_subruns"] > 0 and st["lattice_elements"] > s.n_asks and st["lattice_asks"] == s.n_asks


@pytest.mark.gpu
@pytest.mark.parametrize("D", DIMS)
def test_default_commit_one_uniform_run_every_dimension_count(oracle, monkeypatch, D):
    s = uniform_shape(D)
    want = oracle.run(s)
    st = _run(s, want, batch=4096)
    assert st["lattice_cycles"] == 1 and st["uniform_runs"] == 1 and st["uniform_asks"] == s.n_asks
    assert st["sweep_launches"] == 0 and st["lattice_subruns"] == 0
    if D in (1, 8):                        # a first depth of 1 makes the run retry deeper
        monkeypatch.setenv("YK_UNIFORM_DEPTH", "1")
        st = _run(s, want, batch=4096)
        assert st["uniform_runs"] == 1 and st["uniform_asks"] == s.n_asks and st["uniform_retries"] > 0


@pytest.mark.gpu
@pytest.mark.parametrize("D", [5, 8])
def test_gang_handoff_above_four_dimensions(oracle, D):
    s = gang_handoff(D)
    want = oracle.run(s)
    assert len(want["ask"]) == s.n_asks and set(want["node"].tolist()) <= set(range(300, 400))
    st = _device(s, want, batch=64)
    assert st["lattice_handoffs"] == 1 and st["sweep_launches"] > 0


# 2. single-pair kernels at every D
@pytest.mark.gpu
@pytest.mark.parametrize("D", range(1, 9))
def test_scores_and_predicates_every_dimension_count(oracle, D):
    s = widen(synth.perf(300, 4, 20, masks=True, seed=9), D, D)
    for k in range(D):
        s.node_avail[:, k] -= (np.arange(s.n_nodes) * (37 + 11 * k)) % np.maximum(s.node_total[:, k] // 3, 1)
    s.node_avail[::17, 0] = -5                                 # over-committed
    s.node_flags[4] = 0
    s.ask_node[5] = 9
    s.ask_req[6] = 0                                           # nothing requested: invalid
    N = np.arange(s.n_nodes)
    for w in (s.weights, np.linspace(0.3, 1.7, D)):           # the configured weights, and a vector whose sum needs a divide
        t = synth.reweigh(s, w)
        with _engine().for_snapshot(t) as e:
            got = e.node_scores(N)
        want = [oracle.node_score(t.policy, t.weights, t.node_total[n], t.node_avail[n]) for n in N]
        assert got.tolist() == want, (D, w)                    # float64, bit for bit
    fails = 0
    with _engine().for_snapshot(s) as e:
        for a in range(0, s.n_asks, 3):
            for n in range(0, s.n_nodes, 13):
                got, exp = e.evaluate(a, n), oracle.predicate(s, a, n)
                assert (got == 0) == (exp == 0) and (got == exp or {got, exp} <= {4, 8}), (D, a, n, got, exp)
                got_r, exp_r = e.evaluate_reserve(a, n), oracle.predicate_reserve(s, a, n)
                assert got_r == exp_r, (D, a, n, got_r, exp_r)
                fails += int(exp != 0)
        assert e.stats()["other_launches"] > 0
    assert 0 < fails


@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 8])
def test_preemption_search_at_one_and_eight_dimensions(oracle, D):
    s = widen(synth.perf(64, 4, 40, masks=True, seed=31), D, D)
    s.node_avail //= 50                                        # nearly full nodes: victims are needed
    rng = np.random.default_rng(D)
    asks = rng.integers(0, s.n_asks, 300)
    nodes = rng.integers(0, s.n_nodes, 300)
    scale = np.maximum(s.ask_req.max(axis=0), 1)
    victims, starts = [], []
    for q in range(300):
        nv = int(rng.integers(0, 70))                          # crosses the 32-victim warp step
        v = (rng.random((nv, D)) * scale * 1.2).astype(np.int64)
        victims.append(v)
        starts.append(int(rng.integers(0, nv + 2)) if q % 10 else nv + int(rng.integers(1, 4)))   # some start past the end
    want = [oracle.preemption_index(s, int(a), int(n), v, st) for a, n, v, st in zip(asks, nodes, victims, starts)]
    with _engine().for_snapshot(s) as e:
        got = e.preemption_search(asks, nodes, victims, starts)
    assert got.tolist() == want
    assert any(w >= 0 for w in want) and any(w < 0 for w in want)


# 3. weights
@pytest.mark.gpu
@pytest.mark.parametrize("case", WEIGHT_CASES)
def test_configured_weights(oracle, case):
    s = weighted(case)
    want = oracle.run(s)
    _both(s, want, batch=256)
    t = copy.deepcopy(s)
    t.node_avail = want["avail"]                               # after the cycle: every node in its own state
    with _engine().for_snapshot(t) as e:
        got = e.node_scores(np.arange(t.n_nodes))
    exp = [oracle.node_score(t.policy, t.weights, t.node_total[n], t.node_avail[n]) for n in range(t.n_nodes)]
    assert got.tolist() == exp
    if case == "pods":                                         # keys move with every pod: the asks spread over all nodes
        assert len(set(want["node"].tolist())) == s.n_nodes and len(set(exp)) > 1
    else:
        assert len(set(exp)) > 10


# 4. infinite shares on the device
@pytest.mark.gpu
@pytest.mark.parametrize("D", [4, 8])
def test_infinite_shares(oracle, monkeypatch, D):
    s = infinite(D)
    want = oracle.run(s)
    assert {3, 7, 11} <= set(want["node"].tolist())             # the zero-vcore nodes are used
    _both(s, want, batch=64)
    with _engine().for_snapshot(s) as e:
        sc = e.node_scores(np.array([3, 7, 11]))
    assert sc[0] == np.inf and sc[1] == -np.inf and np.isfinite(sc[2])
    monkeypatch.setenv("YK_UNIFORM_MIN", "64")
    u = infinite_uniform(D)
    want = oracle.run(u)
    assert {3, 7, 11} <= set(want["node"].tolist())
    st = _device(u, want, batch=4096)
    assert st["uniform_asks"] > 0


# 5. a NaN score is an error, and a clean one
@pytest.mark.gpu
@pytest.mark.parametrize("commit", ["host", "device", "auto"])
def test_nan_score_is_a_clean_error(oracle, commit):
    from yunikorn_k8shim_b200 import YkError
    s = nan_node()
    with pytest.raises(RuntimeError):
        oracle.run(s)
    t = nan_repaired(s)
    want = oracle.run(t)
    A, N = np.arange(s.n_asks), np.arange(s.n_nodes)
    with _engine().for_snapshot(s, batch=4096, commit=commit) as e:
        with pytest.raises(YkError) as ei:
            e.cycle(s.n_asks)
        assert ei.value.code == YK_ERR_RANGE
        st = e.stats()
        assert st["allocations"] == 0
        assert st["lattice_cycles"] == (0 if commit == "host" else 1)   # auto: 5 000 identical asks go to the device
        assert (e.ask_states(A) == ST_PENDING).all()
        assert np.array_equal(e.nodes_available(N), s.node_avail)
        e.nodes_upsert([5], t.node_total[[5]], t.node_avail[[5]], t.node_taint[[5]], t.node_label[[5]], s.node_rank()[[5]],
                       t.node_flags[[5]])
        ask, node, _ = e.cycle(s.n_asks)
        assert np.array_equal(ask, want["ask"]) and np.array_equal(node, want["node"])
        assert np.array_equal(e.nodes_available(N), want["avail"])
        assert np.array_equal(e.ask_states(A), want["state"])
        assert e.stats()["lattice_cycles"] == (0 if commit == "host" else 2)


# 6. extreme magnitudes
@pytest.mark.gpu
@pytest.mark.parametrize("D", [1, 4, 8])
def test_extreme_magnitudes(oracle, monkeypatch, D):
    s = extreme(D)
    want = oracle.run(s)
    _both(s, want, batch=64)
    monkeypatch.setenv("YK_UNIFORM_MIN", "2")
    u = extreme(D, uniform=True)
    want = oracle.run(u)
    st = _device(u, want, batch=4096)
    assert st["uniform_asks"] > 0
    if D in (1, 8):
        monkeypatch.setenv("YK_UNIFORM_DEPTH", "1")
        st = _device(u, want, batch=4096)
        assert st["uniform_asks"] > 0 and st["uniform_retries"] > 0


# 8. the fixtures, on the CPU
def _all_fixtures():
    for D in DIMS:
        for seed in FUZZ_SEEDS:
            yield fuzz_dims(D, seed)
    # the large builders once or twice each: the Python oracle takes seconds on them
    for s in (big(1), big(8), runny_big(5), uniform_shape(1)):
        yield s
    for D in DIMS:
        yield tiny_stack(D)
    for D in (5, 8):
        yield gang_handoff(D)
    for case in WEIGHT_CASES:
        yield weighted(case)
    for D in (4, 8):
        yield infinite(D)
        yield infinite_uniform(D)
    yield nan_repaired(nan_node())
    for D in (1, 4, 8):
        yield extreme(D)
        yield extreme(D, uniform=True)


def test_fixtures_oracles_agree(oracle):
    """every snapshot the GPU tests above compare against gets the same bindings from both oracle restatements (C++ and
    Python) -- also at 2^62 totals, with +-Inf shares and with configured weights"""
    n = 0
    for s in _all_fixtures():
        try:
            r = oracle.run(s)
        except RuntimeError:
            with pytest.raises(Exception):
                py_oracle.run(s)
            continue
        p = py_oracle.run(s)
        assert list(r["ask"]) == p["ask"], s.name
        assert list(r["node"]) == p["node"], s.name
        assert list(r["state"]) == p["state"], s.name
        n += 1
    assert n > 100
    with pytest.raises(RuntimeError):
        oracle.run(nan_node())
