"""The solvers' exponent windows at their edges, bit for bit against the oracle (DESIGN.md 3.1-3.2).

Every streaming solve divides with ``div_recip`` and keeps no ``p[0..K]`` vector; that is exact only while ``p``, the
running sum and the rates stay inside the windows of ``wva_device.cuh`` (``kHiPHi``, ``kHiSumHi``, ``kHiRowSumHi``,
``kHiRate*``, the pass-2 bound ``2^(E(sum) - 960)``).  Outside them a solve must bail out to the stored vector.  The
fleets here are steered onto those edges with beta = delta = 0: then ``servRate[n-1] = n / c`` and, with
``x = lambda * c``, ``p[n] ~ x^n / n!`` peaks near ``n = x`` at about ``2^(1.4427 x)``.  Which edge a case reaches is
decided by ``chain_profile`` (pass 1 of the reference in float64, same operations and order) and asserted by the CPU
tests below, so the GPU tests cannot silently drift off their edges.

Bands per path (E = binary exponent; each edge has cases at E = edge - 1 and E = edge):

* grid (``grid_kernel``, round-1 windows): E(max p) at 600, E(sum) at 620 for the cells that do not share their row;
  rows that share (``b >= j + 2``) with E(sum) at 620, and shared rows with p in [2^600, 2^620); chains that cross
  2^600 growing by 2^4 or more per step.
* size (``size_warp_kernel``, ``sz2_solve``) and sweep: E(max p) at 880, E(sum) at 680 and 900, the pass-2 IEEE path
  (sum in [2^882, 2^900), p < 2^880, states below 2^(E(sum) - 960) before termination), float64 overflow (the
  reference's rescale branch).  The sweep also has chains that cross 2^880 growing by 2^4 or more per step; the
  size path also has chains with K >= 2^23 (no early termination) whose pass 2 runs the IEEE path down to the
  smallest subnormal.
* every path: servRate[0] and servRate[N-1] at 2^-60 and 2^60, exactly on the boundary and just across it;
  lambda exactly at 2^-60 and one ulp below (grid, size).

Not reachable through the fleet interface, and so left out: a sum bail on its own (E(sum) 620 for unshared grid cells,
900 elsewhere) — the sum exceeds the peak by at most ~2^11 here, since Analyze keeps lambda below 0.999
servRate[N-1], so the cases at those sums have already crossed the p edge; on the size path no streaming solve sees p >= 2^880 after
its first one, because every later lambda of a candidate is at most the throughput of its first solve at lambda*
(0.9 RateRange.Max here) and a candidate whose first solve bails is re-run wholesale on the stored vector; steep
crossings on the size path, because lambda < servRate[N-1] keeps x below N and a crossing of 2^880 by 2^4 per step
needs x above 2600, where lambda* itself overflows; lambda alone at 2^60, because Analyze rejects lambda above
0.999 servRate[N-1], so lambda >= 2^60 always comes with servRate[N-1] above the window (the grid cases still put
lambda exactly on 2^60); exact lambda edges in the sweep, whose rates are spaced by the sweep itself.
"""
from __future__ import annotations

import numpy as np
import pytest

from tests.grid_cases import (LONG_RATIO, OVERFLOW_SEARCHES, SWEEP_RATES, _Lanes, _analyzer, _cat, _cells_equal, _exp2,
                              _fleet_model, _lam_of_rate, _lam_star, _rate_bands, _straddle, _sweep_equal,
                              chain_profile, f32, grid_cases, grid_points, long_queue_fleet, overflow_search_fleet,
                              size_fleet, sweep_fleet, sweep_points, wide_bands)
from tests.util import assert_allocs_equal
from workload_variant_autoscaler_b200 import synth_fleet

# ---------------------------------------------------------------------------------------------------------------
# the reference's pass 1 (mm1modelstatedependent.go:93-105) in float64, vectorised over lambda
# ---------------------------------------------------------------------------------------------------------------
# ---------------------------------------------------------------------------------------------------------------
# float32 lambdas exactly as the oracle forms them
# ---------------------------------------------------------------------------------------------------------------
# ---------------------------------------------------------------------------------------------------------------
# fleets: one model and one accelerator per server, beta = delta = 0 unless given
# ---------------------------------------------------------------------------------------------------------------
# ---------------------------------------------------------------------------------------------------------------
# the points each path evaluates, with their profiles
# ---------------------------------------------------------------------------------------------------------------
def size_points(fleet, cand):
    """Profiles of the lambdas a size candidate is known to solve: lambda* (0.9 RateRange.Max) and the final
    Analyze at total / replicas with the oracle's replica count."""
    L = _Lanes()
    for s in range(fleet.n_servers):
        a, g, d, it, ot, ratio = _fleet_model(fleet, s)
        N = int(fleet.srv_max_batch[s])
        qa = _analyzer(N, a, g, d, it, ot, ratio)
        lams = [_lam_star(qa)]
        if cand["feasible"][s]:
            total = f32(f32(fleet.srv_slo_tps[s]) / f32(ot))
            lams.append(_lam_of_rate(f32(total / f32(cand["replicas"][s]))))
        L.add(qa, N, lams)
    return L.profile()


# ---------------------------------------------------------------------------------------------------------------
# bands
# ---------------------------------------------------------------------------------------------------------------
def grid_bands(P):
    ok = ~P["over"]
    shareable = ok & ~P["tail"] & (P["N"] >= P["j"] + 2)
    kernel = ok & ~shareable
    b = {}
    b["grid_kernel E(max p) 599 / 600"] = _straddle(P["emax"], kernel, 600)
    b["grid_kernel E(sum) 619 / 620"] = _straddle(P["esum"], kernel, 620)
    b["shared row E(sum) 619 / 620"] = _straddle(P["esum"], shareable, 620)
    in_band = shareable & (P["emax"] >= 600) & (P["esum"] < 620)
    b["shared row with p in [2^600, 2^620)"] = (int(in_band.sum()),) * 2
    b["steep crossing of 2^600"] = (int(P["steep600"].sum()),) * 2
    for k, v in _rate_bands(P).items():
        b[k] = (int(v),) * 2
    return b


def _assert_bands(bands, skip=()):
    low = {k: v for k, v in bands.items() if k not in skip and min(v) < 3}
    assert not low, f"bands with fewer than 3 cases on a side: {low}"


# ---------------------------------------------------------------------------------------------------------------
# CPU: the helper is the reference's pass 1, and the cases reach their bands
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,x,delta", [(16, 3.0, 0.0), (64, 40.0, 1e-3), (512, 300.0, 0.0), (1024, 600.0, 0.0),
                                       (1024, 611.5, 0.0), (2048, 650.0, 2e-5)])
def test_chain_profile_matches_oracle_probs(oracle_mod, N, x, delta):
    """The helper's p[n] / sum equals the oracle's normalised vector bit for bit on non-overflowing chains."""
    qa = _analyzer(N, 1.0, 0.0, delta)
    lam = f32(x)
    prof = chain_profile(qa.serv_rate(), qa.K, [lam], keep=True)
    assert not prof["over"][0]
    st = qa.solve(float(lam))
    assert st["is_valid"]
    want = qa.probs()
    got = prof["p"][:, 0] / prof["sum"][0]
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    assert prof["emax"][0] == _exp2(prof["p"][:, 0].max())


def test_chain_profile_termination_rule_hand_checked():
    """N = 4, rates 1..4, lambda = 1/2: p = 1, 1/2, 1/8, 1/48, 1/384, and from state 4 on every step divides by 8
    (the tail rate 4), so p[n] = 2^-(3 (n - 4)) / 384.  p[1] = 1/2 puts the threshold at 2^-78 * 1/2 = 2^-79, and
    lambda is below every remaining rate from state 1 on.  p[27] = 2^-77.6 is above it, p[28] = 2^-80.6 below: j = 28,
    past the head (N - 1 = 3)."""
    sr = np.array([1, 2, 3, 4], np.float32)
    prof = chain_profile(sr, 40, [0.5], keep=True)
    p = prof["p"][:, 0]
    assert p[4] == 1.0 / 384 and p[27] > 2.0 ** -79 > p[28]
    assert prof["j"][0] == 28 and prof["tail"][0]
    # the same chain in a table of 40 rates 1..40 ends in its head: lambda = 1/2 is below all of them
    prof = chain_profile(np.arange(1, 41, dtype=np.float32), 80, [0.5])
    assert 0 < prof["j"][0] < 39 and not prof["tail"][0]
    # lambda not below the remaining rates: no termination however small p gets
    prof = chain_profile(sr, 40, [np.float32(3.99999)])
    assert prof["j"][0] == -1 and prof["tail"][0]


def test_grid_cases_reach_their_bands(oracle_mod):
    pts = []
    for fleet, grid in grid_cases():
        cells, _ = oracle_mod.grid_solve(fleet, grid, want_cells=True)
        pts.append(grid_points(fleet, grid, cells["flags"]))
    _assert_bands(grid_bands(_cat(pts)))


def test_size_cases_reach_their_bands(oracle_mod):
    fleet = size_fleet()
    cand, _ = oracle_mod.solve(fleet)
    P = size_points(fleet, cand.reshape(-1))
    _assert_bands(wide_bands(P, steep=False))
    _assert_bands({k: (int(v),) * 2 for k, v in _rate_bands(P).items()})


def test_long_queue_cases_reach_the_pass2_ieee_path(oracle_mod):
    fleet = long_queue_fleet()
    cand, _ = oracle_mod.solve(fleet)
    P = size_points(fleet, cand.reshape(-1))
    assert (P["N"] * (1 + LONG_RATIO) >= 1 << 23).all()
    ieee = ~P["over"] & (P["esum"] >= 882) & (P["esum"] < 900) & (P["emax"] < 880) & (P["elive"] < P["esum"] - 960)
    assert ieee.sum() >= 3, P["esum"]


def test_overflow_search_cases_bail_inside_the_search(oracle_mod):
    """The ITL bisection of overflow_search_fleet iterates (EvalITL crosses the targets between lambda_min and
    lambda_max), its end point lambda_max and 0.9 lambda_max overflow float64 while lambda_max / 2 does not, and the
    candidates are feasible."""
    import oracle
    f = overflow_search_fleet(7.55, 0.0)
    ratio = f.max_queue_to_batch_ratio
    qa = oracle.Analyzer(1024, 1024 * ratio, float(f.perf_alpha[0, 0]), float(f.perf_beta[0, 0]),
                         float(f.perf_gamma[0, 0]), float(f.perf_delta[0, 0]), int(f.srv_in_tokens[0]),
                         int(f.srv_out_tokens[0]))
    lo, hi = qa.rate_range()
    lmin, lmax = _lam_of_rate(lo), _lam_of_rate(hi)
    (e0, y0), (e1, y1) = qa.eval_itl(float(lmin)), qa.eval_itl(float(lmax))
    assert e0 == 0 and e1 == 0
    assert y0 < min(t for t, _, _ in OVERFLOW_SEARCHES) and y1 > max(t for t, _, _ in OVERFLOW_SEARCHES)
    P = chain_profile(qa.serv_rate(), qa.K, [lmax, f32(f32(0.9) * lmax), f32(lmax / f32(2))])
    assert P["over"].tolist() == [True, True, False]
    for slo_itl, slo_ttft, max_rate in OVERFLOW_SEARCHES:
        cand, _ = oracle_mod.solve(overflow_search_fleet(slo_itl, slo_ttft))
        assert (cand["feasible"] == 1).all() and (cand["replicas"] == 2).all()
        assert np.allclose(cand["max_rate"], max_rate, rtol=1e-4)


def test_sweep_cases_reach_their_bands(oracle_mod):
    fleet = sweep_fleet()
    o = oracle_mod.sweep(fleet, SWEEP_RATES)
    P = sweep_points(fleet, SWEEP_RATES, o["valid"])
    _assert_bands(wide_bands(P))
    _assert_bands({k: (int(v),) * 2 for k, v in _rate_bands(P).items() if not k.startswith("lam")})


# ---------------------------------------------------------------------------------------------------------------
# GPU: every path at these edges, bit for bit
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", range(3))
def test_grid_cells_at_window_edges(engine, oracle_mod, case):
    fleet, grid = grid_cases()[case]
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    cells_g, win_g = engine.grid_solve(fleet, grid, want_cells=True)
    _cells_equal(cells_g, cells_o, f"grid case {case}")
    assert_allocs_equal(win_g, win_o, f"grid case {case} winners (cell table)")


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(3))
def test_grid_winners_at_window_edges(engine, oracle_mod, case):
    """Without a cell table (grid_order pruning): the winners."""
    fleet, grid = grid_cases()[case]
    _, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=False)
    _, win_g = engine.grid_solve(fleet, grid, want_cells=False)
    assert_allocs_equal(win_g, win_o, f"grid case {case} winners")


@pytest.mark.gpu
def test_size_warp_kernel_at_window_edges(engine, oracle_mod):
    fleet = size_fleet()
    assert fleet.n_servers <= 1024  # size_warp_kernel's range
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, "size candidates (warp per candidate)")
    assert_allocs_equal(win_g, win_o, "winners (warp per candidate)")


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "5"])
def test_size_rounds_at_window_edges(engine, oracle_mod, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet = size_fleet()
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, f"size candidates (rounds, D = {depth})")
    assert_allocs_equal(win_g, win_o, f"winners (rounds, D = {depth})")


@pytest.mark.gpu
@pytest.mark.parametrize("small_max", ["1024", "0"])
def test_size_long_queue_at_window_edges(engine, oracle_mod, monkeypatch, small_max):
    """Chains without early termination (K >= 2^23) whose pass 2 must take the exact IEEE path below 2^(E(sum) - 960)."""
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", small_max)
    fleet = long_queue_fleet()
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, f"long-queue size candidates (small max {small_max})")
    assert_allocs_equal(win_g, win_o, f"long-queue winners (small max {small_max})")


@pytest.mark.gpu
@pytest.mark.parametrize("small_max,depth", [("1024", "5"), ("0", "1"), ("0", "5")])
@pytest.mark.parametrize("case", range(len(OVERFLOW_SEARCHES)))
def test_size_search_bails_to_stored_vector(engine, oracle_mod, monkeypatch, small_max, depth, case):
    """A bisection whose streaming solves overflow float64 (the warp kernel and the rounds at depths 1 and 5): the
    candidate is re-run on the stored vector, whose search crosses overflowing midpoints."""
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", small_max)
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    slo_itl, slo_ttft, _ = OVERFLOW_SEARCHES[case]
    fleet = overflow_search_fleet(slo_itl, slo_ttft)
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, f"size candidates (overflowing search, small max {small_max}, D = {depth})")
    assert_allocs_equal(win_g, win_o, f"winners (overflowing search, small max {small_max}, D = {depth})")


@pytest.mark.gpu
def test_sweep_at_window_edges(engine, oracle_mod):
    """Points outside the streaming windows (including float64 overflow) are re-run on the stored vector."""
    fleet = sweep_fleet()
    o = oracle_mod.sweep(fleet, SWEEP_RATES)
    g = engine.sweep(fleet, SWEEP_RATES)
    _sweep_equal(g, o, "window-edge sweep")


@pytest.mark.gpu
def test_sweep_overflow_fleet_falls_back_to_stored_vector(engine, oracle_mod):
    """The N = 1024 fleet of the grid's overflow test, swept with 64 rates: the chains of the upper rates overflow
    float64, where the reference rescales its stored vector."""
    fleet = synth_fleet(2, 1, seed=29, max_batch_choices=(1024,))
    fleet.perf_alpha[:] = 7.47
    fleet.perf_beta[:] = 0.0001
    fleet.perf_gamma[:] = 1.0
    fleet.perf_delta[:] = 0.00001
    fleet.srv_in_tokens[:] = 64
    fleet.srv_out_tokens[:] = 64
    o = oracle_mod.sweep(fleet, 64)
    assert o["valid"].sum() == 128
    g = engine.sweep(fleet, 64)
    _sweep_equal(g, o, "overflow sweep")
