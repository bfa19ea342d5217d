"""wva_load_grid: the reference's Server.Calculate and SolveUnlimited winner at many caller-given arrival rates.

The expected result is composed from the CPU oracle, literally: for each level l, a copy of the fleet with
srv_arrival_rpm = row l and unlimited = 1 goes through the oracle's Server.Calculate (candidate block l) and
Solver.Solve (winner block l).  The CPU tests pin that composition against the oracle's own solve and show on the
oracle that CreateAllocation splits into a load-independent Size and a per-level tail; the GPU tests compare the
CUDA path with the composition bit for bit."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (at_row, check_level_call, load_levels, mixed_fleet, overflow_fleet, pair_batch,
                          rates_at_rate_star, ref_grid, tail)
from tests.util import (ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, assert_allocs_equal,
                        error_code, f32_bits, same_bytes)
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, greedy_solve, synth_fleet

# ---- CPU: the composition and the split --------------------------------------------------------

@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("seed", [1, 2])
def test_one_level_is_the_oracle_solve(oracle_mod, seed, keep):
    fleet = mixed_fleet(12, 3, seed, keep)
    cand, win = ref_grid(oracle_mod, fleet, {"arrival_rpm": fleet.srv_arrival_rpm[None, :]})
    cand_o, win_o = oracle_mod.solve(at_row(fleet, {}, 0))
    assert same_bytes(cand, cand_o.reshape(-1))
    assert same_bytes(win, win_o)
    assert win["feasible"].sum() >= 4


@pytest.mark.parametrize("seed", [3, 4])
def test_size_once_then_the_tail_is_create_allocation(oracle_mod, seed):
    """QueueAnalyzer.Size does not read the load: one Size per pair, then the replica / cost / Analyze tail at each
    level, reproduces the oracle's CreateAllocation at that level bit for bit."""
    fleet = mixed_fleet(16, 3, seed, False)
    assert fleet.srv_slo_tps.max() > 0 and (fleet.srv_min_replicas == 0).any()
    levels = [0.0, -1.0, 1e-3, 600.0, 1e6, np.inf]
    checked = 0
    for s in range(fleet.n_servers):
        m = int(fleet.srv_model[s])
        if m < 0 or not fleet.srv_has_target[s] or fleet.srv_out_tokens[s] == 0:
            continue
        for a in range(fleet.n_acc):
            if not fleet.perf_present[m, a]:
                continue
            N = pair_batch(fleet, s, a)
            try:
                qa = oracle_mod.Analyzer(N, N * fleet.max_queue_to_batch_ratio, float(fleet.perf_alpha[m, a]),
                                         float(fleet.perf_beta[m, a]), float(fleet.perf_gamma[m, a]),
                                         float(fleet.perf_delta[m, a]), int(fleet.srv_in_tokens[s]),
                                         int(fleet.srv_out_tokens[s]))
                err, _, met, _ = qa.size(float(fleet.srv_slo_ttft[s]), float(fleet.srv_slo_itl[s]),
                                         float(fleet.srv_slo_tps[s]))
            except ValueError:
                qa, err = None, 1
            for rpm in levels:
                want = oracle_mod.create_allocation(at_row(fleet, {"arrival_rpm": [np.full(fleet.n_servers, rpm, np.float32)]}, 0), s, a)
                if rpm < 0:
                    assert want["feasible"] == 0
                    continue
                if rpm == 0:  # zeroLoadAllocation: min_replicas, no queue
                    assert want["feasible"] == 1 and want["rho"] == 0
                    continue
                got = tail(oracle_mod, qa, fleet, s, a, N, met["throughput"], rpm) if not err else None
                if got is None:
                    assert want["feasible"] == 0, (s, a, rpm)
                    continue
                for k in ALLOC_FIELDS:
                    if k in ("cost", "value", "itl", "ttft", "rho", "max_rate"):
                        assert f32_bits(got[k]) == f32_bits(want[k]), (s, a, rpm, k, got[k], want[k])
                    else:
                        assert int(got[k]) == int(want[k]), (s, a, rpm, k, got[k], want[k])
                checked += int(want["feasible"])
    assert checked >= 40


def test_max_rate_is_the_same_at_every_load_level(oracle_mod):
    fleet = mixed_fleet(20, 3, 5, False)
    rpm = load_levels(fleet, 6, 7)
    cand, _ = ref_grid(oracle_mod, fleet, {"arrival_rpm": rpm})
    cand = cand.reshape(6, fleet.n_servers, fleet.n_acc)
    load = ~(rpm < 0) & (rpm != 0)
    seen = 0
    for s in range(fleet.n_servers):
        for a in range(fleet.n_acc):
            rates = {f32_bits(cand[l, s, a]["max_rate"]) for l in range(6) if load[l, s] and cand[l, s, a]["feasible"]}
            assert len(rates) <= 1, (s, a)
            seen += len(rates)
    assert seen >= 20


# ---- GPU: bit for bit against the composition -------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet(engine, oracle_mod, monkeypatch, keep, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = mixed_fleet(14, 3, 31, keep)
    rpm = load_levels(fleet, 7, 3)
    cand_o, win_o = check_level_call(engine, oracle_mod, "load_grid", fleet, {"arrival_rpm": rpm}, f"small, keep = {keep}, rounds = {rounds}")
    assert cand_o["feasible"].sum() > 40
    assert len(set(win_o["replicas"][win_o["feasible"] == 1].tolist())) >= 3


@pytest.fixture(scope="module")
def large_case(oracle_mod):
    fleet = mixed_fleet(560, 4, 37, False)  # > 2,000 load pairs: the rounds
    fleet.srv_keep_acc[::2] = 1
    rpm = load_levels(fleet, 3, 11)
    return fleet, rpm, ref_grid(oracle_mod, fleet, {"arrival_rpm": rpm})


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [None, "1", "2", "3", "4", "5"])
def test_large_fleet_every_tree_depth(engine, large_case, monkeypatch, depth):
    if depth is not None:
        monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rpm, (cand_o, win_o) = large_case
    cand_g, win_g = engine.load_grid(fleet, rpm, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"large, D = {depth}: candidates")
    assert_allocs_equal(win_g, win_o, f"large, D = {depth}: winners")


@pytest.mark.gpu
def test_stored_vector_fallback_both_phases(engine, oracle_mod):
    fleet = overflow_fleet()
    cols = [rates_at_rate_star(oracle_mod, fleet, s, 0) for s in range(2)]
    L = min(len(c) for c in cols)
    rpm = np.stack([np.array(c[:L], np.float32) for c in cols], axis=1)
    cand_o, _ = check_level_call(engine, oracle_mod, "load_grid", fleet, {"arrival_rpm": rpm}, "stored-vector fallback")
    assert cand_o["feasible"].sum() >= L


@pytest.mark.gpu
def test_each_level_is_analyze_and_solve(engine, oracle_mod):
    fleet = mixed_fleet(30, 4, 41, True)
    fleet.type_capacity[:] = [6, 9, 4, 12]
    rpm = load_levels(fleet, 5, 13)
    cand_g, win_g = engine.load_grid(fleet, rpm, want_candidates=True)
    S, A = fleet.n_servers, fleet.n_acc
    for l in range(5):
        f = at_row(fleet, {"arrival_rpm": rpm}, l)
        cand_a = engine.analyze(f)
        _, win_s = engine.solve(f)
        for k in ALLOC_FIELDS:
            assert same_bytes(getattr(cand_g, k)[l * S * A:(l + 1) * S * A], getattr(cand_a, k)), (l, k)
            assert same_bytes(getattr(win_g, k)[l * S:(l + 1) * S], getattr(win_s, k)), (l, k)
        # limited mode by composition: the level's candidate block into the greedy pass
        fl = at_row(fleet, {"arrival_rpm": rpm}, l, unlimited=False)
        block = Allocs(S * A)
        for k in ALLOC_FIELDS:
            getattr(block, k)[:] = getattr(cand_g, k)[l * S * A:(l + 1) * S * A]
        cand_lim, win_lim = greedy_solve(fl, block)
        cand_o, win_o = oracle_mod.solve(fl)
        assert_allocs_equal(win_lim, win_o, f"level {l}, limited: winners")
        assert_allocs_equal(cand_lim, cand_o, f"level {l}, limited: candidates")
    # one level is wva_solve
    _, win1 = engine.load_grid(fleet, fleet.srv_arrival_rpm[None, :])
    _, win_s = engine.solve(fleet)
    for k in ALLOC_FIELDS:
        assert same_bytes(getattr(win1, k), getattr(win_s, k)), k


@pytest.mark.gpu
def test_nan_and_huge_values_and_ties(engine, oracle_mod):
    fleet = mixed_fleet(12, 3, 43, False)
    fleet.srv_cur_cost[::2] = np.nan     # penalty NaN except for the current (accelerator, replicas)
    fleet.srv_cur_cost[1::4] = -F32_MAX  # the current accelerator's penalty rounds to MaxFloat32
    fleet.acc_cost[2] = fleet.acc_cost[1]
    fleet.perf_alpha[:, 2] = fleet.perf_alpha[:, 1]  # accelerators 1 and 2 identical: ties on value
    for k in ("perf_beta", "perf_gamma", "perf_delta", "perf_acc_count"):
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]
    check_level_call(engine, oracle_mod, "load_grid", fleet, {"arrival_rpm": load_levels(fleet, 4, 17)}, "NaN / huge values and ties")


@pytest.mark.gpu
def test_nan_level_fails_as_analyze_does(engine):
    fleet = mixed_fleet(10, 3, 47, False)
    rpm = load_levels(fleet, 3, 19)
    rpm[1, 5] = np.nan
    want, cand_a = error_code(lambda: engine.analyze(at_row(fleet, {"arrival_rpm": rpm}, 1)))
    got, res = error_code(lambda: engine.load_grid(fleet, rpm, want_candidates=True))
    assert got == want
    if want == 0:
        S, A = fleet.n_servers, fleet.n_acc
        for k in ALLOC_FIELDS:
            assert same_bytes(getattr(res[0], k)[S * A:2 * S * A], getattr(cand_a, k)), k


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_sizing_runs_once_per_pair(engine, monkeypatch, rounds):
    """The launch count does not grow with the number of levels: the bisections run once per pair."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = synth_fleet(40, 4, seed=53, zero_load_frac=0.0)
    assert (fleet.srv_arrival_rpm > 0).all()
    rng = np.random.default_rng(5)
    counts = []
    for L in (1, 64):
        rpm = (fleet.srv_arrival_rpm[None, :] * rng.lognormal(0.0, 0.5, (L, fleet.n_servers))).astype(np.float32)
        n0 = engine.launch_count
        engine.load_grid(fleet, rpm)
        counts.append(engine.launch_count - n0)
    assert counts[0] == counts[1], counts


@pytest.mark.gpu
def test_cache_interplay_on_one_handle(engine):
    fleet = mixed_fleet(30, 3, 59, True)
    rpm = load_levels(fleet, 4, 23)
    fresh = Engine(0)
    try:
        def same(got, want, what):
            for k in ALLOC_FIELDS:
                assert np.array_equal(getattr(got, k).view(np.uint8), getattr(want, k).view(np.uint8)), f"{what}: {k}"

        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if x is not None:
                    same(x, y, what)

        solve = lambda e: e.solve(fleet)  # noqa: E731
        size_grid = lambda e: e.size_grid(fleet, [4, 16, 64], want_candidates=True)  # noqa: E731
        load_grid = lambda e: e.load_grid(fleet, rpm, want_candidates=True)  # noqa: E731
        check(solve, "solve")
        check(load_grid, "load grid")
        check(size_grid, "size grid after the load grid")
        check(solve, "solve after the load grid")
        check(load_grid, "load grid after the size grid")
        fleet.srv_out_tokens[:] = np.maximum(1, fleet.srv_out_tokens // 3)
        engine.update_load(out_tokens=fleet.srv_out_tokens)
        check(load_grid, "load grid after a token change")
        check(solve, "solve at the end")
    finally:
        fresh.close()


@pytest.mark.gpu
def test_argument_errors_empty_list_and_summary(engine):
    from workload_variant_autoscaler_b200 import _abi
    fleet = mixed_fleet(6, 2, 61, False)
    L, h = engine._L, engine._h
    win = Allocs(fleet.n_servers)
    fc, wc = fleet.as_c(), win.as_c()
    one = np.ones(fleet.n_servers, np.float32)
    assert L.wva_load_grid(h, C.byref(fc), -1, _abi.ptr(one), None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_load_grid(h, C.byref(fc), 1, None, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_load_grid(h, C.byref(fc), 1, _abi.ptr(one), None, None) == WVA_ERR_BAD_ARG
    # S * A * L = 2^20 * 2^6 * 32 = 2^31: refused before the fleet is read
    big = fleet.as_c()
    big.n_servers, big.n_acc, big.n_types = 1 << 20, 1 << 6, 0
    assert L.wva_load_grid(h, C.byref(big), 32, _abi.ptr(one), None, C.byref(wc)) == WVA_ERR_UNSUPPORTED
    with pytest.raises(ValueError):
        engine.load_grid(fleet, one)
    # an empty list is valid
    cand, win0 = engine.load_grid(fleet, np.zeros((0, fleet.n_servers), np.float32), want_candidates=True)
    assert cand.n == 0 and win0.n == 0
    # no single solution to summarise after a load grid
    engine.solve(fleet)
    engine.summarize(fleet.n_types)
    engine.load_grid(fleet, load_levels(fleet, 2, 29))
    with pytest.raises(WvaError) as e:
        engine.summarize(fleet.n_types)
    assert e.value.code == WVA_ERR_STATE
