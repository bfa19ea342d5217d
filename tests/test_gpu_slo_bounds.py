"""wva_slo_bounds: per (load pair, search), the targets at which the reference's candidate turns nil and at which its
target stops binding.

The expected result is composed from the C oracle: per pair an Analyzer built as create_allocation builds it, its
rate_range, EvalTTFT / EvalITL at lambda_min and lambda_max, BinarySearch's boundary checks restated with the
oracle's WithinTolerance, and the breakpoints found by bisecting the float32 bit patterns.  The CPU tests pin that
composition to the oracle's own binary_search and Analyzer.size; the GPU tests compare the CUDA path with it bit for
bit, and check the exact statements on wva_slo_grid without the oracle."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (F32, FREE, INF_BITS, NIL, PAST, SEARCHED, _adversarial_fleet, analyzer, check_slo_bounds,
                          from_bits, lam_range, mixed_fleet, overflow_fleet, ref_slo_bounds, u32_bits)
from tests.util import ALLOC_FIELDS, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, error_code
from workload_variant_autoscaler_b200 import Engine, WvaError, slo_envelope, synth_fleet
from workload_variant_autoscaler_b200 import _abi

def _key(x):
    return PAST if np.isnan(x) else u32_bits(x)


def stretch(kind, b1, b2, t):
    """The class of target t from one entry: NIL, SEARCHED or FREE."""
    first = not t >= b1
    last = t >= b2
    pos = 0 if first else (2 if last else 1)
    return pos if kind == 2 else 2 - pos


def edge_fleet(seed, keep=False):
    """mixed_fleet with a flat ITL (beta = 0) on one accelerator and an empty rate range on another model."""
    f = mixed_fleet(14, 3, seed, keep)
    f.perf_beta[:, 1] = 0.0
    f.perf_alpha[:, 2] = -1.0  # negative service times: lambda_min > lambda_max or below zero
    f.perf_gamma[:, 2] = -1.0
    return f


def probe_targets(y0, y1, b1, b2, rng):
    """The targets the composition is pinned at: b1, b2 and the float below each, +-64 ulps around y0 and y1,
    denormals, +Inf, MaxFloat32 and random targets in each stretch."""
    keys = {1, 2, 0x00400000, 0x7F7FFFFF, INF_BITS}
    for b in (b1, b2):
        if not np.isnan(b):
            keys |= {u32_bits(b), max(u32_bits(b) - 1, 1)}
    for y in (y0, y1):
        if y > 0 and np.isfinite(y):
            keys |= {k for k in range(u32_bits(y) - 64, u32_bits(y) + 65, 8) if 0 < k <= INF_BITS}
            keys |= {u32_bits(y) - 1, u32_bits(y), u32_bits(y) + 1}
    edges = sorted({1} | {_key(b) for b in (b1, b2)} | {INF_BITS + 1})
    for lo, hi in zip(edges, edges[1:]):
        if hi - 1 > lo:
            keys |= set(int(k) for k in rng.integers(lo, min(hi, INF_BITS + 1), 3))
    return [from_bits(k) for k in sorted(keys) if 0 < k <= INF_BITS]


# ---- CPU: the composition against the oracle's own search ------------------------------------------

@pytest.mark.parametrize("seed", [5, 6])
def test_composition_is_binary_search_and_size(oracle_mod, seed):
    """At every probe target: NIL <=> BinarySearch's ind < 0, and FREE => Size's rate for that search equals its
    rate with that target 0 (lambda_max, bit for bit)."""
    fleet = edge_fleet(seed)
    kind, y_lo, y_hi, b1, b2 = ref_slo_bounds(oracle_mod, fleet)
    rng = np.random.default_rng(seed)
    seen = {k: 0 for k in (1, 2, 3)}
    classes = set()
    for s in range(fleet.n_servers):
        for a in range(fleet.n_acc):
            if kind[s, a, 0] == 0:
                continue
            for w in range(2):
                k = int(kind[s, a, w])
                seen[k] += 1
                qa = analyzer(oracle_mod, fleet, s, a)
                lmin, lmax = lam_range(qa)
                ev = qa.eval_ttft if w == 0 else qa.eval_itl

                def fn(x):
                    err, y = ev(x)
                    if err:
                        raise ValueError("invalid model")
                    return y
                ts = [from_bits(1), from_bits(INF_BITS), F32(1.0), F32(100.0)] if k == 1 else \
                    probe_targets(y_lo[s, a, w], y_hi[s, a, w], b1[s, a, w], b2[s, a, w], rng)
                err0, r0, _, _ = qa.size(0.0, 0.0, 0.0)
                for t in ts:
                    args = (float(t), 0.0, 0.0) if w == 0 else (0.0, float(t), 0.0)
                    err, rates, _, _ = qa.size(*args)
                    if k == 1:
                        assert err, (s, a, w, t)
                        continue
                    c = stretch(k, b1[s, a, w], b2[s, a, w], t)
                    classes.add((k, c))
                    e, xs, ind = oracle_mod.binary_search(float(lmin), float(lmax), float(t), fn)
                    assert (c == NIL) == (ind < 0 or e != 0), (s, a, w, t, c, ind)
                    assert (c == NIL) == (err != 0), (s, a, w, t, c, err)
                    if c == FREE:
                        assert not err0
                        name = "rate_ttft" if w == 0 else "rate_itl"
                        assert u32_bits(rates[name]) == u32_bits(r0[name]), (s, a, w, t)
                        assert u32_bits(xs) == u32_bits(lmax), (s, a, w, t)
    assert seen[1] >= 1 and seen[2] >= 4 and seen[3] >= 2, seen
    assert {(2, NIL), (2, SEARCHED), (2, FREE)} <= classes, classes


def test_flat_itl_and_tolerance_edges(oracle_mod):
    """beta = 0: ITL is flat (y_lo == y_hi), its SEARCHED stretch is the tolerance band around it; targets within
    1e-6 of y_lo or y_hi land in the stretch the restated checks give, on the oracle's own search."""
    fleet = edge_fleet(7)
    kind, y_lo, y_hi, b1, b2 = ref_slo_bounds(oracle_mod, fleet)
    flat = [(s, a) for s in range(fleet.n_servers) for a in range(fleet.n_acc)
            if kind[s, a, 1] >= 2 and y_lo[s, a, 1] == y_hi[s, a, 1]]
    assert flat
    for s, a in flat:
        assert kind[s, a, 1] == 3
        y = y_lo[s, a, 1]
        assert b1[s, a, 1] <= y < b2[s, a, 1]
        qa = analyzer(oracle_mod, fleet, s, a)
        for t in (b1[s, a, 1], from_bits(u32_bits(b1[s, a, 1]) - 1), from_bits(u32_bits(b2[s, a, 1]) - 1), b2[s, a, 1]):
            err, rates, _, _ = qa.size(0.0, float(t), 0.0)
            c = stretch(3, b1[s, a, 1], b2[s, a, 1], t)
            assert (c == NIL) == (err != 0)


# ---- GPU: bit for bit against the composition ---------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet(engine, oracle_mod, monkeypatch, keep, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    kind = check_slo_bounds(engine, oracle_mod, edge_fleet(31, keep), f"keep = {keep}, rounds = {rounds}")[0]
    assert (kind == 0).any() and (kind == 1).any() and (kind == 2).any() and (kind == 3).any()


@pytest.mark.gpu
@pytest.mark.parametrize("n_acc", [32, 33])
def test_many_accelerators(engine, oracle_mod, n_acc):
    check_slo_bounds(engine, oracle_mod, synth_fleet(4, n_acc, seed=41 + n_acc, zero_load_frac=0.2), f"A = {n_acc}")


@pytest.mark.gpu
def test_stored_vector_fallback(engine, oracle_mod):
    """N = 1024 near saturation: the lambda_max solves leave the streaming windows and re-run on the stored
    vector."""
    fleet = overflow_fleet()
    fleet.srv_arrival_rpm[:] = 600.0
    kind = check_slo_bounds(engine, oracle_mod, fleet, "stored-vector fallback")[0]
    assert (kind >= 2).all()


@pytest.mark.gpu
def test_adversarial(engine, oracle_mod):
    """levels._adversarial_fleet's fleets: where the call refuses, wva_analyze with every target positive
    refuses too."""
    rng = np.random.default_rng(0x5B0)
    checked = 0
    for case in range(24):
        fleet = _adversarial_fleet(rng, 80000 + case)
        code = error_code(lambda: engine.slo_bounds(fleet))[0]
        if code:
            assert code == WVA_ERR_UNSUPPORTED, case
            f = fleet.take_servers(np.arange(fleet.n_servers))
            f.srv_slo_itl[:] = 1.0
            f.srv_slo_ttft[:] = 1.0
            assert error_code(lambda: engine.analyze(f))[0] == WVA_ERR_UNSUPPORTED, case
            continue
        check_slo_bounds(engine, oracle_mod, fleet, f"adversarial case {case}")
        checked += 1
    assert checked >= 12


# ---- GPU: the exact statements on wva_slo_grid, no oracle ---------------------------------------

@pytest.mark.gpu
def test_statements_on_the_slo_grid(engine):
    """On synth_fleet(1500, 8): rows whose target for server s at level (a, point) is b1, the float below b1, b2,
    the float below b2 or 0.  A candidate at a NIL target is nil, one at a FREE target equals the target-0
    candidate byte for byte, and slo_envelope's floor and ceiling hold for the winners."""
    fleet = synth_fleet(1500, 8, seed=101)
    S, A = fleet.n_servers, fleet.n_acc
    bounds = engine.slo_bounds(fleet)
    kind, _, _, b1, b2 = bounds
    assert (kind[..., 1] >= 2).sum() > 1000
    for w, col in ((1, "slo_itl"), (0, "slo_ttft")):
        pts = []
        for a in range(A):
            for b in (b1[:, a, w], b2[:, a, w]):
                ok = np.isfinite(b) & (b > 0)
                below = np.where(ok, np.array(b).view(np.uint32) - np.uint32(1), 0).view(np.float32)
                pts += [np.where(ok, b, 0).astype(F32), np.where(ok & (below > 0), below, 0).astype(F32)]
        floor, ceiling = slo_envelope(fleet, bounds, w)
        fc = lambda x: np.where(np.isfinite(x), x, 0).astype(F32)  # noqa: E731
        pts += [fc(floor), fc(np.where(floor > from_bits(1), (floor.view(np.uint32) - 1).view(F32), 0)), fc(ceiling),
                fc(ceiling * F32(2))]
        rows = np.stack([np.zeros(S, F32)] + pts)
        own = {"slo_itl": fleet.srv_slo_itl, "slo_ttft": fleet.srv_slo_ttft, "slo_tps": fleet.srv_slo_tps}
        lists = {k: np.broadcast_to(v, rows.shape).astype(F32) for k, v in own.items()}
        lists[col] = rows
        cand, win = engine.slo_grid(fleet, lists["slo_itl"], lists["slo_ttft"], lists["slo_tps"],
                                    want_candidates=True)
        L = rows.shape[0]
        for l in range(1, L):
            t = rows[l]
            for a in range(A):
                k = kind[:, a, w]
                idx0, idx = np.arange(S) * A + a, (l * S + np.arange(S)) * A + a
                cls = np.array([stretch(k[s], b1[s, a, w], b2[s, a, w], t[s]) if k[s] >= 2 else -1
                                for s in range(S)])
                sel = (t > 0) & (k >= 1)
                nil = sel & ((k == 1) | (cls == NIL))
                assert not cand.feasible[idx[nil]].any(), (w, l, a)
                free = sel & (cls == FREE)
                for f in ALLOC_FIELDS:
                    g = np.asarray(getattr(cand, f))
                    assert g[idx[free]].tobytes() == g[idx0[free]].tobytes(), (w, l, a, f)
            below = (t > 0) & ~(t >= floor)
            assert not win.feasible[l * S + np.arange(S)][below].any(), (w, l)
            above = (t > 0) & (t >= ceiling)
            for f in ALLOC_FIELDS:
                g = np.asarray(getattr(win, f))
                assert g[l * S + np.arange(S)][above].tobytes() == g[np.arange(S)][above].tobytes(), (w, l, f)


# ---- GPU: API ---------------------------------------------------------------------------------

@pytest.mark.gpu
def test_argument_errors_and_refusals(engine):
    fleet = mixed_fleet(6, 2, 79, False)
    L, h = engine._L, engine._h
    fc = fleet.as_c()
    oc = _abi.SloBoundsC()
    assert L.wva_slo_bounds(None, C.byref(fc), C.byref(oc)) == WVA_ERR_BAD_ARG
    assert L.wva_slo_bounds(h, None, C.byref(oc)) == WVA_ERR_BAD_ARG
    assert L.wva_slo_bounds(h, C.byref(fc), None) == WVA_ERR_BAD_ARG
    # every column NULL: nothing written, the call still runs
    assert L.wva_slo_bounds(h, C.byref(fc), C.byref(oc)) == 0
    big = synth_fleet(2, 2, seed=83, zero_load_frac=0.0)
    big.srv_max_batch[:] = 1 << 20
    big.max_queue_to_batch_ratio = 1 << 12
    n0 = engine.launch_count
    assert error_code(lambda: engine.slo_bounds(big))[0] == WVA_ERR_UNSUPPORTED
    assert engine.launch_count == n0  # refused before any launch
    assert error_code(lambda: engine.analyze(big))[0] == WVA_ERR_UNSUPPORTED


@pytest.mark.gpu
def test_non_terminating_solve_names_the_pair(engine):
    fleet = synth_fleet(3, 2, seed=5, zero_load_frac=0.0)
    fleet.perf_alpha[int(fleet.srv_model[1]), 1] = np.nan
    with pytest.raises(WvaError) as e:
        engine.slo_bounds(fleet)
    assert e.value.code == WVA_ERR_UNSUPPORTED
    assert "server 1, accelerator 1" in str(e.value)


@pytest.mark.gpu
def test_no_servers(engine):
    fleet = synth_fleet(3, 3, seed=3).take_servers(np.arange(0))
    kind, y_lo, _, _, _ = engine.slo_bounds(fleet)
    assert kind.shape == (0, 3, 2) and y_lo.shape == (0, 3, 2)


@pytest.mark.gpu
def test_launch_count(engine):
    """The tables, the tail, its re-run and bounds_kernel, whatever the fleet."""
    def launches(f):
        n0 = engine.launch_count
        engine.slo_bounds(f)
        return engine.launch_count - n0
    small, large = synth_fleet(5, 2, seed=71, zero_load_frac=0.0), synth_fleet(3000, 8, seed=72)
    assert launches(small) == launches(large) == 4


@pytest.mark.gpu
def test_one_handle_with_the_other_paths(engine, oracle_mod):
    fleet = mixed_fleet(30, 3, 73, True)
    want = ref_slo_bounds(oracle_mod, fleet)
    fresh = Engine(0)
    try:
        def same_bounds(e, what):
            for g, w in zip(e.slo_bounds(fleet), want):
                assert g.tobytes() == w.tobytes(), what

        def same_allocs(x, y, what):
            for k in ALLOC_FIELDS:
                assert np.asarray(getattr(x, k)).tobytes() == np.asarray(getattr(y, k)).tobytes(), f"{what}: {k}"
        rows = [np.stack([getattr(fleet, c) * F32(f) for f in (0.5, 1.5)]) for c in
                ("srv_slo_itl", "srv_slo_ttft", "srv_slo_tps")]
        cand_s, win_s = engine.solve(fleet)
        same_bounds(engine, "bounds after solve")
        cand_r, win_r = engine.resolve(want_candidates=True)
        same_allocs(cand_r, cand_s, "resolve after the bounds")
        for x, y in zip(engine.slo_grid(fleet, *rows, want_candidates=True),
                        fresh.slo_grid(fleet, *rows, want_candidates=True)):
            same_allocs(x, y, "slo grid after the bounds")
        same_bounds(engine, "bounds after the slo grid")
        for x, y in zip(engine.solve(fleet), fresh.solve(fleet)):
            same_allocs(x, y, "solve after the bounds")
        engine.summarize(fleet.n_types)
        same_bounds(engine, "bounds before summarize")
        with pytest.raises(WvaError) as e:
            engine.summarize(fleet.n_types)
        assert e.value.code == WVA_ERR_STATE
    finally:
        fresh.close()
