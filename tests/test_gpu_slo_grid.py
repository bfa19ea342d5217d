"""wva_slo_grid: the reference's Server.Calculate and SolveUnlimited winner at many caller-given SLO target rows.

The expected result is composed from the CPU oracle, literally: for each level l, a copy of the fleet with
srv_slo_itl / srv_slo_ttft / srv_slo_tps = row l and unlimited = 1 goes through the oracle's Server.Calculate
(candidate block l) and Solver.Solve (winner block l).  The CPU tests pin that composition against the oracle's own
solve and show on the oracle that each bisection of QueueAnalyzer.Size reads only its own target, which is what lets
the library run each distinct (server, search, target) once; the GPU tests compare the CUDA path with the
composition bit for bit."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (F32, SLO, TARGETS, TPS_TARGETS, _adversarial_fleet, _search, at_row, check_level_call,
                          mixed_fleet, overflow_fleet, pair_batch, ref_grid, slo_levels, tail)
from tests.util import (ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, assert_allocs_equal,
                        error_code, f32_bits, same_bytes)
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, greedy_solve, synth_fleet

# ITL / TTFT targets at the edges: 0, -0 and NaN disable a search, a negative one makes the pair nil, the others run
# TPS targets: no NaN (totalRate NaN) and no tiny positive one (totalRate 0, so a min_replicas-0 pair solves at 0/0):
# the library refuses some such levels, see test_nan_or_tiny_tps_level_fails_as_solve_does
# ---- CPU: the composition and the premise -------------------------------------------------------

@pytest.mark.parametrize("keep", [False, True])
def test_one_level_is_the_oracle_solve(oracle_mod, keep):
    fleet = mixed_fleet(12, 3, 5, keep)
    rows = [c[None, :] for c in (fleet.srv_slo_itl, fleet.srv_slo_ttft, fleet.srv_slo_tps)]
    cand, win = ref_grid(oracle_mod, fleet, dict(zip(SLO, rows)))
    cand_o, win_o = oracle_mod.solve(at_row(fleet, {}, 0))
    assert same_bytes(cand, cand_o.reshape(-1))
    assert same_bytes(win, win_o)
    assert win["feasible"].sum() >= 4


def _analyzer(oracle_mod, fleet, s, a):
    m = fleet.srv_model[s]
    N = pair_batch(fleet, s, a)
    return N, oracle_mod.Analyzer(N, N * fleet.max_queue_to_batch_ratio, float(fleet.perf_alpha[m, a]),
                                  float(fleet.perf_beta[m, a]), float(fleet.perf_gamma[m, a]),
                                  float(fleet.perf_delta[m, a]), int(fleet.srv_in_tokens[s]),
                                  int(fleet.srv_out_tokens[s]))


def test_each_search_reads_only_its_own_target(oracle_mod):
    """On every load pair of a mixed fleet and every (TTFT, ITL, TPS) over the edge values: Size's TTFT rate is
    that of Size(t, 0, 0) and its ITL rate that of Size(0, t, 0); Size fails exactly when a target is negative or
    one of the two searches fails; and min(lambda*s, the TPS rule) followed by the tail is CreateAllocation."""
    fleet = mixed_fleet(8, 2, 7, False)
    typical = (float(np.median(fleet.srv_slo_ttft[fleet.srv_slo_ttft > 0])),
               float(np.median(fleet.srv_slo_itl[fleet.srv_slo_itl > 0])))
    tps_typ = float(np.median(fleet.srv_slo_tps[fleet.srv_slo_tps > 0]))
    ttfts, itls = TARGETS + (typical[0],), TARGETS + (typical[1],)
    checked = feasible = 0
    for s in range(fleet.n_servers):
        m = int(fleet.srv_model[s])
        if m < 0 or not fleet.srv_has_target[s] or fleet.srv_out_tokens[s] == 0 or fleet.srv_arrival_rpm[s] <= 0:
            continue
        for a in range(fleet.n_acc):
            if not fleet.perf_present[m, a]:
                continue
            N, qa = _analyzer(oracle_mod, fleet, s, a)
            one_t = {f32_bits(t): qa.size(t, 0.0, 0.0) for t in ttfts}
            one_i = {f32_bits(t): qa.size(0.0, t, 0.0) for t in itls}
            srch_t = {f32_bits(t): _search(oracle_mod, qa, 0, t) for t in ttfts}
            srch_i = {f32_bits(t): _search(oracle_mod, qa, 1, t) for t in itls}
            for tt in ttfts:
                for ti in itls:
                    for tp in TPS_TARGETS + (tps_typ,):
                        err, rates, _, _ = qa.size(tt, ti, tp)
                        neg = tt < 0 or ti < 0 or tp < 0
                        ok_t, xs_t = srch_t[f32_bits(tt)]
                        ok_i, xs_i = srch_i[f32_bits(ti)]
                        assert (err != 0) == (neg or not ok_t or not ok_i), (s, a, tt, ti, tp, err)
                        if err == 0:
                            assert f32_bits(rates["rate_ttft"]) == f32_bits(one_t[f32_bits(tt)][1]["rate_ttft"])
                            assert f32_bits(rates["rate_itl"]) == f32_bits(one_i[f32_bits(ti)][1]["rate_itl"])
                        # the tail from the two searches reproduces CreateAllocation at this level
                        f_l = at_row(fleet, {}, 0)
                        f_l.srv_slo_ttft[s], f_l.srv_slo_itl[s], f_l.srv_slo_tps[s] = tt, ti, tp
                        want = oracle_mod.create_allocation(f_l, s, a)
                        got = None
                        if err == 0:
                            lmax = F32(qa.rate_range()[1]) / F32(1000)
                            l_tps = lmax * (F32(1) - F32(0.1)) if tp > 0 else lmax
                            lam = min(xs_t, xs_i, l_tps)
                            e2, met = qa.analyze(float(F32(lam) * F32(1000)))
                            if e2 == 0:
                                got = tail(oracle_mod, qa, f_l, s, a, N, met["throughput"], fleet.srv_arrival_rpm[s])
                        if got is None:
                            assert want["feasible"] == 0, (s, a, tt, ti, tp)
                            continue
                        for k in ALLOC_FIELDS:
                            if k in ("cost", "value", "itl", "ttft", "rho", "max_rate"):
                                assert f32_bits(got[k]) == f32_bits(want[k]), (s, a, tt, ti, tp, k)
                            else:
                                assert int(got[k]) == int(want[k]), (s, a, tt, ti, tp, k)
                        checked += 1
                        feasible += int(want["feasible"])
    assert checked >= 500 and feasible >= 100, (checked, feasible)


# ---- GPU: bit for bit against the composition -------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet_warp_path(engine, oracle_mod, keep):
    fleet = mixed_fleet(14, 3, 31, keep)
    cand_o, win_o = check_level_call(engine, oracle_mod, "slo_grid", fleet, dict(zip(SLO, slo_levels(fleet, 7, 3))), f"small, keep = {keep}")
    assert cand_o["feasible"].sum() > 40
    assert len(set(win_o["replicas"][win_o["feasible"] == 1].tolist())) >= 3


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = mixed_fleet(60, 3, 37, False)
    fleet.srv_keep_acc[::2] = 1
    rows = slo_levels(fleet, 4, 11)
    return fleet, rows, ref_grid(oracle_mod, fleet, dict(zip(SLO, rows)))


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [None, "1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    if depth is not None:
        monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rows, (cand_o, win_o) = rounds_case
    cand_g, win_g = engine.slo_grid(fleet, *rows, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"rounds, D = {depth}: candidates")
    assert_allocs_equal(win_g, win_o, f"rounds, D = {depth}: winners")


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_cartesian_itl_ttft_tps_grid(engine, oracle_mod, monkeypatch, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = mixed_fleet(12, 3, 41, False)
    S = fleet.n_servers
    f = np.array([0.5, 1.0, 2.0], np.float32)
    tps_on = np.where(fleet.srv_slo_tps > 0, fleet.srv_slo_tps, F32(100))
    itl, ttft, tps = [], [], []
    for fi in f:
        for ft in f:
            for use_tps in (False, True):
                itl.append(fleet.srv_slo_itl * fi)
                ttft.append(fleet.srv_slo_ttft * ft)
                tps.append(tps_on if use_tps else np.zeros(S, np.float32))
    rows = tuple(np.array(x, np.float32) for x in (itl, ttft, tps))
    cand_o, _ = check_level_call(engine, oracle_mod, "slo_grid", fleet, dict(zip(SLO, rows)), f"Cartesian, rounds = {rounds}")
    assert cand_o["feasible"].sum() > 100


@pytest.mark.gpu
def test_own_targets_are_wva_solve(engine):
    fleet = mixed_fleet(30, 4, 43, True)
    rows = [c[None, :] for c in (fleet.srv_slo_itl, fleet.srv_slo_ttft, fleet.srv_slo_tps)]
    cand1, win1 = engine.slo_grid(fleet, *rows, want_candidates=True)
    cand_s, win_s = engine.solve(at_row(fleet, {}, 0))
    for k in ALLOC_FIELDS:
        assert same_bytes(getattr(cand1, k), getattr(cand_s, k)), k
        assert same_bytes(getattr(win1, k), getattr(win_s, k)), k


@pytest.mark.gpu
def test_stored_vector_fallback_both_phases(engine, oracle_mod):
    """N = 1024 near saturation: the chains overflow float64 near lambda_max, so the searches (targets just under
    the value at lambda_max, and above it) and the tail's solves (targets off: lambda* = lambda_max) re-run on the
    stored vector."""
    fleet = overflow_fleet()
    S = fleet.n_servers
    near = {0: [], 1: []}
    for s in range(S):
        _, qa = _analyzer(oracle_mod, fleet, s, 0)
        lmax = F32(qa.rate_range()[1]) / F32(1000)
        for which, ev in ((0, qa.eval_ttft), (1, qa.eval_itl)):
            err, y = ev(float(lmax))
            assert err == 0
            near[which].append(F32(y))
    ttft_near, itl_near = (np.array(near[w], np.float32) for w in (0, 1))
    rows_itl, rows_ttft = [], []
    for fi, ft in ((0, 0), (0.9999, 0), (0, 0.9999), (0.9999, 0.9999), (1.5, 0), (0, 1.5), (0.99, 1.5)):
        rows_itl.append(itl_near * F32(fi))
        rows_ttft.append(ttft_near * F32(ft))
    L = len(rows_itl)
    rows = (np.array(rows_itl, np.float32), np.array(rows_ttft, np.float32), np.zeros((L, S), np.float32))
    cand_o, _ = check_level_call(engine, oracle_mod, "slo_grid", fleet, dict(zip(SLO, rows)), "stored-vector fallback")
    assert cand_o["feasible"].sum() >= L


@pytest.mark.gpu
def test_nan_and_huge_values_and_ties(engine, oracle_mod):
    fleet = mixed_fleet(12, 3, 47, False)
    fleet.srv_cur_cost[::2] = np.nan     # penalty NaN except for the current (accelerator, replicas)
    fleet.srv_cur_cost[1::4] = -F32_MAX  # the current accelerator's penalty rounds to MaxFloat32
    fleet.acc_cost[2] = fleet.acc_cost[1]
    fleet.perf_alpha[:, 2] = fleet.perf_alpha[:, 1]  # accelerators 1 and 2 identical: ties on value
    for k in ("perf_beta", "perf_gamma", "perf_delta", "perf_acc_count"):
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]
    check_level_call(engine, oracle_mod, "slo_grid", fleet, dict(zip(SLO, slo_levels(fleet, 4, 17))), "NaN / huge values and ties")


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_searches_run_once_per_distinct_target(engine, monkeypatch, rounds):
    """The launch count does not grow with the number of levels: L = 1 and 64 identical rows launch the same, and
    so do 2 and 16 rows over the same two distinct target rows."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = synth_fleet(40, 4, seed=53, zero_load_frac=0.0)
    own = [c.copy() for c in (fleet.srv_slo_itl, fleet.srv_slo_ttft, fleet.srv_slo_tps)]
    other = [own[0] * F32(0.75), own[1] * F32(1.5), own[2]]

    def launches(pattern):
        rows = [np.array([(own, other)[p][i] for p in pattern], np.float32) for i in range(3)]
        n0 = engine.launch_count
        engine.slo_grid(fleet, *rows)
        return engine.launch_count - n0
    assert launches([0]) == launches([0] * 64)
    assert launches([0, 1]) == launches([0, 1] * 8) == launches([1, 0, 0, 1] * 4)


@pytest.mark.gpu
def test_one_handle_with_the_other_paths(engine):
    fleet = mixed_fleet(30, 3, 59, True)
    rows = slo_levels(fleet, 4, 23)
    rpm = np.stack([fleet.srv_arrival_rpm * F32(k) for k in (0.5, 1.0, 2.0)]).astype(np.float32)
    fresh = Engine(0)
    try:
        def same(got, want, what):
            for k in ALLOC_FIELDS:
                assert np.array_equal(getattr(got, k).view(np.uint8), getattr(want, k).view(np.uint8)), f"{what}: {k}"

        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if x is not None:
                    same(x, y, what)

        slo_grid = lambda e: e.slo_grid(fleet, *rows, want_candidates=True)  # noqa: E731
        load_grid = lambda e: e.load_grid(fleet, rpm, want_candidates=True)  # noqa: E731
        size_grid = lambda e: e.size_grid(fleet, [4, 16, 64], want_candidates=True)  # noqa: E731
        # wva_solve -> wva_slo_grid -> wva_resolve: the resident fleet and the solve's cache are untouched
        cand_s, win_s = engine.solve(fleet)
        slo_grid(engine)
        cand_r, win_r = engine.resolve(want_candidates=True)
        same(cand_r, cand_s, "resolve after the SLO grid: candidates")
        same(win_r, win_s, "resolve after the SLO grid: winners")
        check(slo_grid, "SLO grid")
        check(load_grid, "load grid after the SLO grid")
        check(slo_grid, "SLO grid after the load grid")
        check(size_grid, "size grid after the SLO grid")
        check(slo_grid, "SLO grid after the size grid")
        check(lambda e: e.solve(fleet), "solve at the end")
        # no single solution to summarise after an SLO grid
        engine.solve(fleet)
        engine.summarize(fleet.n_types)
        slo_grid(engine)
        with pytest.raises(WvaError) as e:
            engine.summarize(fleet.n_types)
        assert e.value.code == WVA_ERR_STATE
    finally:
        fresh.close()


@pytest.mark.gpu
def test_each_block_is_the_greedy_input_of_its_level(engine, oracle_mod):
    fleet = mixed_fleet(30, 4, 61, True)
    fleet.type_capacity[:] = [6, 9, 4, 12]
    rows = slo_levels(fleet, 4, 13)
    cand_g, _ = engine.slo_grid(fleet, *rows, want_candidates=True)
    S, A = fleet.n_servers, fleet.n_acc
    for l in range(4):
        fl = at_row(fleet, dict(zip(SLO, rows)), l, unlimited=False)
        block = Allocs(S * A)
        for k in ALLOC_FIELDS:
            getattr(block, k)[:] = getattr(cand_g, k)[l * S * A:(l + 1) * S * A]
        cand_lim, win_lim = greedy_solve(fl, block)
        cand_o, win_o = oracle_mod.solve(fl)
        assert_allocs_equal(win_lim, win_o, f"level {l}, limited: winners")
        assert_allocs_equal(cand_lim, cand_o, f"level {l}, limited: candidates")


@pytest.mark.gpu
def test_argument_errors_and_refusals(engine):
    from workload_variant_autoscaler_b200 import _abi
    fleet = mixed_fleet(6, 2, 67, False)
    L, h = engine._L, engine._h
    win = Allocs(fleet.n_servers)
    fc, wc = fleet.as_c(), win.as_c()
    one = np.ones(fleet.n_servers, np.float32)
    p = _abi.ptr(one)
    assert L.wva_slo_grid(h, C.byref(fc), -1, p, p, p, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    for k in range(3):
        rows = [p, p, p]
        rows[k] = None
        assert L.wva_slo_grid(h, C.byref(fc), 1, *rows, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_slo_grid(h, C.byref(fc), 1, p, p, p, None, None) == WVA_ERR_BAD_ARG
    # S * A * L = 2^20 * 2^6 * 32 = 2^31: refused before the fleet is read
    big = fleet.as_c()
    big.n_servers, big.n_acc, big.n_types = 1 << 20, 1 << 6, 0
    assert L.wva_slo_grid(h, C.byref(big), 32, p, p, p, None, C.byref(wc)) == WVA_ERR_UNSUPPORTED
    with pytest.raises(ValueError):
        engine.slo_grid(fleet, one, one, one)
    with pytest.raises(ValueError):
        engine.slo_grid(fleet, one[None, :], one[None, :], np.ones((2, fleet.n_servers), np.float32))
    # an empty list is valid
    z = np.zeros((0, fleet.n_servers), np.float32)
    cand, win0 = engine.slo_grid(fleet, z, z, z, want_candidates=True)
    assert cand.n == 0 and win0.n == 0


@pytest.mark.gpu
@pytest.mark.parametrize("s, value, fails", [(6, np.nan, True), (6, 1e-45, True), (0, np.nan, False)])
def test_nan_or_tiny_tps_level_fails_as_solve_does(engine, s, value, fails):
    """A NaN TPS target makes totalRate NaN, and a tiny one rounds it to 0 (a min_replicas-0 pair then gets 0
    replicas and Analyze solves at 0/0).  On server 6 of this fleet wva_solve of that level fails; on server 0 it
    gives NaN latencies.  The grid fails exactly where wva_solve does and gives its records where it does not; the
    grid without that level succeeds."""
    fleet = mixed_fleet(10, 3, 71, False)
    assert fleet.srv_arrival_rpm[s] > 0 and fleet.srv_min_replicas[s] == 0
    itl, ttft, tps = slo_levels(fleet, 3, 19, special=False)
    tps[1, s] = value
    want, res = error_code(lambda: engine.solve(at_row(fleet, dict(zip(SLO, (itl, ttft, tps))), 1)))
    got, grid = error_code(lambda: engine.slo_grid(fleet, itl, ttft, tps, want_candidates=True))
    assert got == want == (WVA_ERR_UNSUPPORTED if fails else 0)
    if want == 0:
        S, A = fleet.n_servers, fleet.n_acc
        for k in ALLOC_FIELDS:
            assert same_bytes(getattr(grid[0], k)[S * A:2 * S * A], getattr(res[0], k)), k
            assert same_bytes(getattr(grid[1], k)[S:2 * S], getattr(res[1], k)), k
    keep = [0, 2]
    assert error_code(lambda: engine.slo_grid(fleet, itl[keep], ttft[keep], tps[keep]))[0] == 0


N_ADV = 36


@pytest.mark.gpu
def test_slo_grid_adversarial(engine, oracle_mod, monkeypatch):
    """Fleets from levels._adversarial_fleet with random target rows from the same edge sets (0, tiny,
    loose; some rows with a target negative or disabled), half of them on the rounds."""
    rng = np.random.default_rng(0x510)
    feasible = 0
    for case in range(N_ADV):
        fleet = _adversarial_fleet(rng, 40000 + case)
        if case % 2:
            monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        else:
            monkeypatch.delenv("WVA_SIZE_SMALL_MAX", raising=False)
        S, L = fleet.n_servers, int(rng.integers(1, 6))
        itl = rng.choice(np.array([0.0, 1e-3, 5.0, 80.0, 1e6, -1.0, np.nan], np.float32), (L, S),
                         p=[.2, .15, .2, .2, .15, .05, .05])
        ttft = rng.choice(np.array([0.0, 1e-2, 50.0, 2000.0, 1e7, -0.0, np.inf], np.float32), (L, S),
                          p=[.2, .15, .2, .2, .15, .05, .05])
        tps = rng.choice(np.array([0.0, 1.0, 500.0, 1e6, -1.0], np.float32), (L, S), p=[.5, .15, .15, .15, .05])
        itl[0], ttft[0], tps[0] = fleet.srv_slo_itl, fleet.srv_slo_ttft, fleet.srv_slo_tps
        if L > 2:
            itl[2], ttft[2], tps[2] = itl[1], ttft[1], tps[1]  # a repeated row
        _, win_o = check_level_call(engine, oracle_mod, "slo_grid", fleet, dict(zip(SLO, (itl, ttft, tps))), f"adversarial case {case}")
        feasible += int(win_o["feasible"].sum())
    assert feasible > 60
