"""wva_price_thresholds: the exact price of each accelerator at which each server's unlimited winner leaves it.

The expected result is composed from the CPU oracle: Server.Calculate once, then for each (server s, accelerator a)
a's record re-priced at p (cost = p * f32(NumInstances * replicas), value = TransitionPenalty, restated as in
test_gpu_workload_trace), the winner decided by the oracle's Solver.Solve on the one-server fleet, and the first
price at which a stops winning found by bisecting the float32 bit patterns.  The CPU tests pin that composition:
the re-priced table is Server.Calculate at the price, "a wins" holds exactly below the threshold on dense price
samples, and accelerator_demand is AllocateByType of the winners.  The GPU tests compare the CUDA path with the
composition bit for bit, and with wva_profile_grid at every threshold without the oracle."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (PRICE_MAX_BITS, PriceServer, _adversarial_fleet, at_price, edge_fleet, from_bits, mixed_fleet,
                          overflow_fleet, pred, priced, rates_at_rate_star, ref_price_fleet, u32_bits)
from tests.util import (ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, assert_allocs_equal,
                        assert_f32_bits_equal, error_code, same_bytes)
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, accelerator_demand, synth_fleet

F32 = np.float32


# ---- CPU: the composition ---------------------------------------------------------------------

def _prices(th, rng, n):
    """Each finite positive threshold and the float below it, 0, MaxFloat32 and n random bit patterns."""
    t = th[np.isfinite(th) & (th > 0)]
    ps = [F32(0.0), from_bits(PRICE_MAX_BITS)] + [x for v in np.unique(t) for x in (v, pred(v))]
    ps += [from_bits(int(b)) for b in rng.integers(0, PRICE_MAX_BITS + 1, n)]
    return ps


@pytest.mark.parametrize("seed,factor", [(3, 0.1), (4, 0.0)])
def test_repriced_table_is_calculate_at_the_price(oracle_mod, seed, factor):
    """CreateAllocation reads acc_cost[a] only in the cost of a's records: at each threshold, the float below it and
    random prices, re-pricing column a of the fleet's table gives Server.Calculate on f(p) bit for bit."""
    fleet = edge_fleet(seed, factor=factor, n=14)
    th, _, cand = ref_price_fleet(oracle_mod, fleet)[:3]
    cand = cand.reshape(fleet.n_servers, fleet.n_acc)
    rng = np.random.default_rng(seed)
    checked = 0
    for a in range(fleet.n_acc):
        for p in _prices(th[:, a], rng, 6):
            want = oracle_mod.calculate(at_price(fleet, a, p))
            got = cand.copy()
            for s in range(fleet.n_servers):
                got[s, a] = priced(fleet, s, a, cand[s, a], p)
            assert same_bytes(got, want), (a, p)
            checked += 1
    assert checked > 30


@pytest.mark.parametrize("keep,factor", [(False, 0.1), (True, 0.1), (False, 0.0), (False, 3.0)])
def test_a_wins_exactly_below_the_threshold(oracle_mod, keep, factor):
    """The monotonicity claim, checked on the predicate itself: at dense prices (every threshold and the float
    below it, random bit patterns, 0 and MaxFloat32) a wins iff p < threshold, with ties between accelerators,
    penalty factor 0, NaN and MaxFloat32 values, and current costs 0 and huge."""
    fleet = edge_fleet(11, keep, factor, n=14)
    th, _, cand = ref_price_fleet(oracle_mod, fleet)[:3]
    cand = cand.reshape(fleet.n_servers, fleet.n_acc)
    rng = np.random.default_rng(7)
    kinds = set()
    for s in range(fleet.n_servers):
        sp = PriceServer(oracle_mod, fleet, cand, s)
        for a in range(fleet.n_acc):
            t = th[s, a]
            kinds.add("0" if t == 0 else "inf" if np.isinf(t) else "finite")
            ps = _prices(th[s], rng, 24)
            for p in ps:
                assert sp.wins(a, p) == (p < t), (s, a, p, t)
    assert {"0", "finite"} <= kinds


def test_accelerator_demand_is_allocate_by_type(oracle_mod):
    """accelerator_demand equals AllocateByType's count of a's type (one accelerator per type) over the oracle's
    winners on f(p), at each stretch's start and one ulp below each breakpoint."""
    fleet = edge_fleet(5, n=14)
    th, _, cand_o = ref_price_fleet(oracle_mod, fleet)[:3]
    cand = Allocs(cand_o.size)
    for k in ALLOC_FIELDS:
        getattr(cand, k)[:] = cand_o[k]
    moved = 0
    for a in range(fleet.n_acc):
        bp, units = accelerator_demand(fleet, th, cand, a)
        assert units.size == bp.size + 1 and (np.diff(bp) > 0).all() and (np.diff(units) <= 0).all()
        starts = [F32(0.0)] + list(bp)
        for j, x in enumerate(starts):
            pts = [(x, units[j])] + ([(pred(x), units[j - 1])] if j else [])
            for p, want in pts:
                win = oracle_mod.solve(at_price(fleet, a, p))[1]
                t = oracle_mod.allocate_by_type(at_price(fleet, a, p), win)[a]
                assert int(t["count"]) == int(want), (a, j, p)
        moved += bp.size
    assert moved >= 3
    with pytest.raises(ValueError):
        accelerator_demand(fleet, th, cand, fleet.n_acc)


# ---- GPU: bit for bit against the composition ---------------------------------------------------

def _check(engine, oracle_mod, fleet, what):
    th_o, above_o, cand_o = ref_price_fleet(oracle_mod, fleet)[:3]
    th_g, above_g, cand_g = engine.price_thresholds(fleet, want_candidates=True)
    assert_f32_bits_equal(th_g.reshape(-1), th_o.reshape(-1), f"{what}: threshold")
    assert_allocs_equal(above_g, above_o, f"{what}: above")
    assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
    return th_o, above_o, cand_o


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet_warp_path(engine, oracle_mod, keep):
    th, _, _ = _check(engine, oracle_mod, edge_fleet(31, keep, n=14), f"warp path, keep = {keep}")
    assert ((th > 0) & np.isfinite(th)).sum() >= 3


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = mixed_fleet(60, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    return fleet, ref_price_fleet(oracle_mod, fleet)[:3]


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, (th_o, above_o, cand_o) = rounds_case
    th_g, above_g, cand_g = engine.price_thresholds(fleet, want_candidates=True)
    assert_f32_bits_equal(th_g.reshape(-1), th_o.reshape(-1), f"rounds, D = {depth}: threshold")
    assert_allocs_equal(above_g, above_o, f"rounds, D = {depth}: above")
    assert_allocs_equal(cand_g, cand_o, f"rounds, D = {depth}: candidates")


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_current_allocation_with_the_same_replica_count(engine, oracle_mod, keep):
    """Servers whose current allocation is a's candidate itself (same accelerator and replica count): the value
    is 0 at every price, so the threshold is 0 or +Inf."""
    fleet = edge_fleet(13, keep, n=14)
    cand = oracle_mod.calculate(fleet)
    same = []
    for s in range(fleet.n_servers):
        fe = np.nonzero(cand[s]["feasible"] & (cand[s]["acc"] >= 0))[0]
        if fe.size and s % 2 == 0:
            a = int(fe[-1])
            fleet.srv_cur_acc[s], fleet.srv_cur_replicas[s] = a, cand[s, a]["replicas"]
            fleet.srv_cur_cost[s] = cand[s, a]["cost"]
            same.append((s, a))
    th, _, _ = _check(engine, oracle_mod, fleet, f"same replica count, keep = {keep}")
    assert len(same) >= 3
    assert all(th[s, a] == 0 or np.isinf(th[s, a]) for s, a in same)


@pytest.mark.gpu
def test_zero_load_min_replicas_zero(engine, oracle_mod):
    """Zero-load servers with min_replicas 0 (the accelerator-"" record, cost 0 at every price) and 1."""
    fleet = edge_fleet(17, n=14)
    fleet.srv_arrival_rpm[::2] = 0.0
    fleet.srv_min_replicas[::4] = 0
    fleet.srv_min_replicas[2::4] = 1
    _, _, cand = _check(engine, oracle_mod, fleet, "zero load")
    assert ((cand["acc"] == -1) & (cand["feasible"] == 1)).sum() >= 2


@pytest.mark.gpu
@pytest.mark.parametrize("n_acc", [32, 33])
def test_many_accelerators(engine, oracle_mod, n_acc):
    """A = 32 and 33: lanes own one accelerator, or lane 0 owns two."""
    fleet = synth_fleet(5, n_acc, seed=41 + n_acc, zero_load_frac=0.2)
    fleet.accel_penalty_factor = 0.0
    fleet.acc_cost[n_acc - 1] = fleet.acc_cost[0]
    for k in ("perf_alpha", "perf_beta", "perf_gamma", "perf_delta", "perf_acc_count", "perf_max_batch",
              "perf_at_tokens", "perf_present"):
        getattr(fleet, k)[:, n_acc - 1] = getattr(fleet, k)[:, 0]  # ties across the strided lanes
    _check(engine, oracle_mod, fleet, f"A = {n_acc}")


@pytest.mark.gpu
def test_stored_vector_fallback(engine, oracle_mod):
    """N = 1024 near saturation: phase 1 re-runs the solves on the stored vector."""
    fleet = overflow_fleet()
    fleet.srv_arrival_rpm[:] = [rates_at_rate_star(oracle_mod, fleet, s, 0)[k] for s, k in ((0, 0), (1, 3))]
    _, _, cand = _check(engine, oracle_mod, fleet, "stored-vector fallback")
    assert cand["feasible"].sum() >= 1


@pytest.mark.gpu
def test_nan_and_huge_values_and_ties(engine, oracle_mod):
    """Values that are NaN (an overflowed cost under factor 0) or MaxFloat32, huge prices, and ties on value."""
    fleet = edge_fleet(19, factor=0.0, n=14)
    fleet.acc_cost[0] = F32(1e38)
    fleet.acc_cost[3] = F32_MAX
    th, _, cand = _check(engine, oracle_mod, fleet, "NaN / huge values and ties")
    assert np.isnan(cand["value"]).any() or (cand["value"] >= F32_MAX).any()


N_ADV = 30


@pytest.mark.gpu
def test_price_thresholds_adversarial(engine, oracle_mod, monkeypatch):
    """Fleets from levels._adversarial_fleet, half of them on the rounds.  Where wva_analyze refuses the
    fleet, the thresholds refuse too."""
    rng = np.random.default_rng(0xB1D)
    checked = refused = 0
    for case in range(N_ADV):
        fleet = _adversarial_fleet(rng, 70000 + case)
        if case % 2:
            monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        else:
            monkeypatch.delenv("WVA_SIZE_SMALL_MAX", raising=False)
        code = error_code(lambda: engine.analyze(fleet))[0]
        if code:
            assert error_code(lambda: engine.price_thresholds(fleet))[0] == code, case
            refused += 1
            continue
        _check(engine, oracle_mod, fleet, f"adversarial case {case}")
        checked += 1
    assert checked > N_ADV // 2


# ---- GPU: self-consistency with wva_profile_grid, no oracle -------------------------------------

@pytest.mark.gpu
def test_profile_grid_at_every_threshold(engine):
    """One wva_profile_grid over rows acc_cost[a] = each distinct finite threshold and the float below it: for
    every pair with 0 < threshold < +Inf, a wins just below and not at the threshold, and above is the winner there
    byte for byte.  Changing the fleet's own acc_cost[a] leaves column a unchanged."""
    fleet = synth_fleet(200, 8, seed=97)
    S, A = fleet.n_servers, fleet.n_acc
    th, above, cand = engine.price_thresholds(fleet, want_candidates=True)
    analyze = engine.analyze(fleet)
    for k in ALLOC_FIELDS:
        assert same_bytes(getattr(cand, k), getattr(analyze, k)), k
    rows, index = [], {}
    for a in range(A):
        for t in np.unique(th[:, a][(th[:, a] > 0) & np.isfinite(th[:, a])]):
            for p in (t, pred(t)):
                index[(a, u32_bits(p))] = len(rows)
                r = fleet.acc_cost.copy()
                r[a] = p
                rows.append(r)
    assert len(rows) >= 40
    _, win = engine.profile_grid(fleet, acc_cost=np.array(rows, F32))
    pairs = 0
    for s in range(S):
        for a in range(A):
            t = th[s, a]
            if not (t > 0 and np.isfinite(t)):
                continue
            at, below = index[(a, u32_bits(t))] * S + s, index[(a, u32_bits(pred(t)))] * S + s
            assert win.feasible[below] == 1 and win.acc[below] == a, (s, a)
            assert not (win.feasible[at] == 1 and win.acc[at] == a), (s, a)
            for k in ALLOC_FIELDS:
                assert same_bytes(getattr(win, k)[at], getattr(above, k)[s * A + a]), (s, a, k)
            pairs += 1
    assert pairs >= 40
    inf = np.isinf(th).reshape(-1)
    for k in ALLOC_FIELDS:
        assert not getattr(above, k)[inf].any(), k
    for a in range(A):
        f = fleet.take_servers(np.arange(S))
        f.acc_cost[a] *= F32(3.0) if a % 2 else F32(0.25)
        th2 = engine.price_thresholds(f)[0]
        assert same_bytes(th2[:, a], th[:, a]), a


# ---- GPU: API ---------------------------------------------------------------------------------

@pytest.mark.gpu
def test_argument_errors_and_refusals(engine):
    fleet = mixed_fleet(6, 2, 79, False)
    L, h = engine._L, engine._h
    fc = fleet.as_c()
    above = Allocs(fleet.n_servers * fleet.n_acc)
    assert L.wva_price_thresholds(None, C.byref(fc), None, None, None) == WVA_ERR_BAD_ARG
    assert L.wva_price_thresholds(h, None, None, None, None) == WVA_ERR_BAD_ARG
    assert L.wva_price_thresholds(h, C.byref(fc), None, C.byref(above.as_c()), None) == WVA_ERR_BAD_ARG
    # above and candidates NULL: the thresholds alone
    th = np.zeros(fleet.n_servers * fleet.n_acc, F32)
    assert L.wva_price_thresholds(h, C.byref(fc), th.ctypes.data_as(C.POINTER(C.c_float)), None, None) == 0
    assert same_bytes(th, engine.price_thresholds(fleet)[0].reshape(-1))
    for factor in (np.nan, -0.5, np.inf):
        f = fleet.take_servers(np.arange(fleet.n_servers))
        f.accel_penalty_factor = factor
        assert error_code(lambda: engine.price_thresholds(f))[0] == WVA_ERR_UNSUPPORTED, factor
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.accel_penalty_factor = 0.0
    assert error_code(lambda: engine.price_thresholds(f))[0] == 0
    for cost in (np.nan, np.inf, -np.inf):
        f = fleet.take_servers(np.arange(fleet.n_servers))
        f.srv_cur_cost[0] = cost
        assert error_code(lambda: engine.price_thresholds(f))[0] == WVA_ERR_UNSUPPORTED, cost
        f.srv_model[0] = -1  # no candidate on that server: nothing to refuse
        assert error_code(lambda: engine.price_thresholds(f))[0] == 0, cost
    # the queue-size rule refuses as wva_analyze does
    big = synth_fleet(2, 2, seed=83, zero_load_frac=0.0)
    big.srv_max_batch[:] = 1 << 20
    big.max_queue_to_batch_ratio = 1 << 12
    code = error_code(lambda: engine.analyze(big))[0]
    assert code == WVA_ERR_UNSUPPORTED
    assert error_code(lambda: engine.price_thresholds(big))[0] == code


@pytest.mark.gpu
def test_no_servers(engine):
    fleet = synth_fleet(3, 3, seed=3).take_servers(np.arange(0))
    th, above, cand = engine.price_thresholds(fleet, want_candidates=True)
    assert th.shape == (0, 3) and above.n == 0 and cand.n == 0
    assert engine._L.wva_price_thresholds(engine._h, C.byref(fleet.as_c()), None, None, None) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_launch_count(engine, monkeypatch, rounds):
    """One price_kernel launch on top of wva_analyze's."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = synth_fleet(40, 4, seed=71, zero_load_frac=0.0)

    def launches(call):
        n0 = engine.launch_count
        call()
        return engine.launch_count - n0
    assert launches(lambda: engine.price_thresholds(fleet)) == launches(lambda: engine.analyze(fleet)) + 1


@pytest.mark.gpu
def test_one_handle_with_the_other_paths(engine):
    fleet = mixed_fleet(30, 3, 73, True)
    fresh = Engine(0)
    try:
        def same(x, y, what):
            if isinstance(x, np.ndarray):
                assert same_bytes(x, y), what
                return
            for k in ALLOC_FIELDS:
                assert same_bytes(getattr(x, k), getattr(y, k)), f"{what}: {k}"

        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if x is not None:
                    same(x, y, what)

        prices = lambda e: e.price_thresholds(fleet, want_candidates=True)  # noqa: E731
        cand_s, win_s = engine.solve(fleet)
        prices(engine)
        cand_r, win_r = engine.resolve(want_candidates=True)
        same(cand_r, cand_s, "resolve after the thresholds: candidates")
        same(win_r, win_s, "resolve after the thresholds: winners")
        check(prices, "thresholds")
        check(lambda e: e.profile_grid(fleet, acc_cost=fleet.acc_cost[None] * F32(0.5), want_candidates=True),
              "profile grid after the thresholds")
        check(lambda e: e.load_grid(fleet, fleet.srv_arrival_rpm[None], want_candidates=True),
              "load grid after the thresholds")
        check(prices, "thresholds after the grids")
        check(lambda e: e.solve(fleet), "solve at the end")
        engine.solve(fleet)
        engine.summarize(fleet.n_types)
        prices(engine)
        with pytest.raises(WvaError) as e:
            engine.summarize(fleet.n_types)
        assert e.value.code == WVA_ERR_STATE
    finally:
        fresh.close()
