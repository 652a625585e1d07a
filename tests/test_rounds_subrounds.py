"""Sub-rounds of the round commit (csrc/yk_rounds.h): a round runs on what is left of the staged window merged with the new
entries that sort before the fence (the first entry of order + side list behind the window), without a fresh staging.
Each case runs on the CPU through the shim against the oracle, and on the GPU through the C ABI against the oracle and the
shim's passes, single steps, round asks, hand-offs and uniform asks.

The cases aim at the window's edges: re-keyed nodes that land inside the window (pods-only asks keep their keys) and behind
it (a ladder of keys, narrow windows), a window that runs empty in mid-pass and is staged afresh, single steps right after
sub-rounds, a side list that fills up while the window lives on, the guard's hand-off and max_bindings cuts with a
non-empty window and side list.  A window that took every new entry, the fence test dropped, fails every CPU case here:
a node re-keyed behind an entry that was never staged would be taken before it."""
import functools

import numpy as np
import pytest

from yunikorn_k8shim_b200 import synth
from device_shim import check, dshim  # noqa: F401  (dshim: the shim fixture)
from test_rounds_parity import COUNTERS, WCAP, Run, _device, _mb_base, _shim, guard_trip, ladder, long_order


def keep_keys(n_nodes=900, n_asks=2700, seed=3):
    """the ladder with half of the asks pods only: the node they take keeps its key, so its new entry sorts before the
    fence and stays in the window, in the middle of it when the ladder's re-keyed nodes sort behind it"""
    s = ladder(n_nodes, n_asks, seed)
    s.ask_req[np.random.default_rng(seed).random(n_asks) < 0.5, 0] = 0
    s.name = f"keep-keys-{n_nodes}x{n_asks}"
    return s


CASES = {
    "windows": lambda: [Run(ladder(600, 1800, seed=4), window=w,
                            expect=lambda c: c["round_asks"] == 1800 and c["lattice_handoffs"] == 0)
                        for w in (1, 31, 32, 33, WCAP)],
    "inside-the-window": lambda: [Run(keep_keys(), window=w, expect=lambda c: c["round_asks"] == 2700) for w in (33, 200, WCAP)],
    "single-step-after-sub-round": lambda: [Run(long_order(n), window=w, expect=lambda c: c["round_single_steps"] > 0
                                                and c["lattice_handoffs"] == 0) for n, w in ((1055, 64), (2048, 33))],
    "side-list-fills": lambda: [Run(synth.perf(3000, 60, 125, seed=8), window=w,
                                    expect=lambda c: c["round_asks"] == 7500 and c["round_single_steps"] == 0) for w in (600, WCAP)],
    "guard-handoff": lambda: [Run(guard_trip(D), window=w, guard=32,
                                  expect=lambda c: c["lattice_handoffs"] == 1 and 0 < c["round_asks"] < 800)
                              for D, w in ((1, 100), (8, 600))],
    "max-bindings": lambda: [Run(_mb_base(), window=w, mb=mb, expect=lambda c, mb=mb: c["round_asks"] == mb)
                             for w, mb in ((33, 250), (WCAP, 333), (600, 1))],
}


@functools.lru_cache(maxsize=None)
def case_runs(name):
    return CASES[name]()


@pytest.mark.parametrize("name", list(CASES))
def test_sub_rounds_match_oracle(dshim, oracle, name):
    for r in case_runs(name):
        want, c = _shim(dshim, oracle, r)
        assert want is not None, r
        assert r.expect(c), (r, c)


def test_narrow_windows_need_the_fence(dshim, oracle):
    """windows of 1 to 33 on a ladder: most new entries sort behind the fence, so the side list and the fresh stagings
    carry them; every stretch is also checked for an exact node order by the shim"""
    for w in (1, 2, 31, 32, 33):
        s = ladder(300, 900, seed=w)
        _, st = check(dshim, oracle, s, tag=w, batch=1 << 16, window=w, guard=0)
        assert st["round_asks"] == 900 and st["passes"] >= 900 // w


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_sub_rounds_on_the_gpu(dshim, oracle, monkeypatch, name):
    for r in case_runs(name):
        want, shim = _shim(dshim, oracle, r)
        st = _device(monkeypatch, r, want)
        got = {k: st[k] for k in COUNTERS}
        assert got == {k: shim[k] for k in COUNTERS}, (r, "device", got, "shim", shim)
        assert st["lattice_cycles"] == 1 and r.expect({**shim, **got}), (r, got)
