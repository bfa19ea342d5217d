"""wva_profile_grid: the reference's Server.Calculate and SolveUnlimited winner at many caller-given rows of
accelerator costs and model x accelerator performance profiles.

The expected result is composed from the CPU oracle, literally: for each level l, a copy of the fleet with acc_cost
and the perf_* columns = row l and unlimited = 1 goes through the oracle's Server.Calculate (candidate block l) and
Solver.Solve (winner block l).  The CPU tests pin that composition against the oracle's own solve and show on the
oracle that CreateAllocation splits into a record fixed by the row's (alpha, beta, gamma, delta, N) and a cost that
alone reads the row's price and AccCount; the GPU tests compare the CUDA path with the composition bit for bit."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (COLUMNS, F32, PERF, _adversarial_fleet, at_row, check_level_call, mixed_fleet, overflow_fleet,
                          profile_fleet, profile_rows, rates_at_rate_star, ref_grid)
from tests.util import (ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, assert_allocs_equal,
                        error_code, f32_bits, same_bytes)
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, greedy_solve, synth_fleet

# ---- CPU: the composition and the split --------------------------------------------------------

@pytest.mark.parametrize("keep", [False, True])
def test_one_level_is_the_oracle_solve(oracle_mod, keep):
    fleet = profile_fleet(12, 3, 5, keep)
    cand, win = ref_grid(oracle_mod, fleet, {"acc_cost": fleet.acc_cost[None]})
    cand_o, win_o = oracle_mod.solve(at_row(fleet, {}, 0))
    assert same_bytes(cand, cand_o.reshape(-1))
    assert same_bytes(win, win_o)
    assert win["feasible"].sum() >= 4


@pytest.mark.parametrize("seed", [3, 4])
def test_cost_and_acc_count_enter_only_the_cost(oracle_mod, seed):
    """A load pair's CreateAllocation at f_l equals the record at f_l with the fleet's own acc_cost and AccCount,
    with cost (and value) replaced by acc_cost_l[a] * f32(NumInstances_l * replicas): every other field is equal bit
    for bit.  This is what lets the grid size one key per distinct (alpha .. delta, N)."""
    fleet = profile_fleet(14, 3, seed, False)
    L = 5
    rows = profile_rows(fleet, L, seed + 10)
    rows["acc_cost"][1] = [np.nan, -2.0, F32_MAX][:fleet.n_acc]
    rng = np.random.default_rng(seed)
    rows["perf_acc_count"][2] = rng.choice([-1, 0, 3, 8], rows["perf_acc_count"][2].shape)
    checked = 0
    for l in range(L):
        fl = at_row(fleet, rows, l)
        fk = at_row(fleet, {k: v for k, v in rows.items() if k not in ("acc_cost", "perf_acc_count")}, l)
        for s in range(fleet.n_servers):
            m = int(fleet.srv_model[s])
            if m < 0 or not fleet.srv_has_target[s] or not (fleet.srv_arrival_rpm[s] > 0):
                continue
            for a in range(fleet.n_acc):
                if not fl.perf_present[m, a] or fleet.srv_out_tokens[s] == 0:
                    continue
                want = oracle_mod.create_allocation(fl, s, a)
                got = oracle_mod.create_allocation(fk, s, a)
                if got["feasible"]:
                    inst = int(fl.perf_acc_count[m, a])
                    inst = 1 if inst <= 0 else inst
                    with np.errstate(all="ignore"):
                        cost = F32(fl.acc_cost[a]) * np.array([inst * int(got["replicas"])], np.int64).astype(F32)[0]
                    got["cost"] = got["value"] = float(cost)
                    checked += 1
                for k in ALLOC_FIELDS:
                    if k in ("cost", "value", "itl", "ttft", "rho", "max_rate"):
                        assert f32_bits(got[k]) == f32_bits(want[k]), (l, s, a, k)
                    else:
                        assert int(got[k]) == int(want[k]), (l, s, a, k)
    assert checked >= 40


# ---- GPU: bit for bit against the composition -------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet_warp_path(engine, oracle_mod, keep):
    fleet = profile_fleet(14, 3, 31, keep)
    cand_o, win_o = check_level_call(engine, oracle_mod, "profile_grid", fleet, profile_rows(fleet, 7, 3), f"warp path, keep = {keep}")
    assert cand_o["feasible"].sum() > 40
    assert len(set(win_o["acc"][win_o["feasible"] == 1].tolist())) >= 2


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = profile_fleet(120, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    rows = profile_rows(fleet, 5, 11)
    return fleet, rows, ref_grid(oracle_mod, fleet, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rows, (cand_o, win_o) = rounds_case
    cand_g, win_g = engine.profile_grid(fleet, **rows, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"rounds, D = {depth}: candidates")
    assert_allocs_equal(win_g, win_o, f"rounds, D = {depth}: winners")


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_cost_only_rows(engine, oracle_mod, monkeypatch, rounds):
    """NaN, +-0, negative, +Inf and MaxFloat32 prices, equal prices on identical accelerators (ties to the lower
    id), and a price sweep of accelerator 0 that makes winners switch to and from it."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = profile_fleet(16, 3, 41, False)
    fleet.srv_cur_cost[::3] = np.nan
    for k in PERF:
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]  # accelerators 1 and 2 identical
    base = fleet.acc_cost
    special = [[np.nan, 1.0, 1.0], [0.0, -0.0, -0.0], [-5.0, 2.0, 2.0], [np.inf, 1.0, 1.0], [F32_MAX, F32_MAX, 1.0],
               [1.0, F32_MAX, F32_MAX]]
    sweep = [np.concatenate([[base[0] * F32(f)], base[1:]]) for f in (1.0, 0.3, 0.1, 0.03, 0.01, 3.0, 10.0)]
    acc = np.array(special + sweep, F32)
    cand_o, win_o = check_level_call(engine, oracle_mod, "profile_grid", fleet, {"acc_cost": acc}, f"cost rows, rounds = {rounds}")
    S = fleet.n_servers
    w = win_o.reshape(len(acc), S)
    fe = w["feasible"] == 1
    switched = ((w["acc"][len(special):] != w["acc"][len(special)]) & fe[len(special):]).sum()
    assert switched >= 2, "the price rows must make some winner switch accelerator"
    tie = w[1][fleet.srv_cur_acc != 2]  # prices zero: accelerators 1 and 2 tie, and 1 wins
    assert not ((tie["acc"] == 2) & (tie["feasible"] == 1)).any()


@pytest.mark.gpu
def test_perf_rows(engine, oracle_mod):
    """alpha / beta / gamma / delta perturbations, one that makes Size fail (a nil record at that level only), an
    accelerator turned on at some levels only (the new-accelerator case), AccCount <= 0, and perf batch sizes that
    change N where srv_max_batch is 0 and are ignored where it is set."""
    fleet = profile_fleet(18, 3, 43, True)
    fleet.perf_present[:, 2] = 0  # accelerator 2 is listed without profiles
    fleet.srv_slo_tps[::5] = F32(800.0)
    M, A = fleet.n_models, fleet.n_acc
    L = 8
    rows = {k: np.repeat(getattr(fleet, k)[None], L, axis=0).copy() for k in PERF}
    rows["perf_beta"][1] *= F32(1.1)
    rows["perf_alpha"][2] *= F32(0.9)
    rows["perf_gamma"][3] *= F32(1.1)
    rows["perf_delta"][3] *= F32(0.9)
    rows["perf_alpha"][4, :, 0] = F32(1e6)  # ITL targets unreachable on accelerator 0: Size fails there
    for l in (5, 6):  # accelerator 2 switched on with a measured profile
        rows["perf_present"][l, :, 2] = 1
        for k in PERF[1:]:
            rows[k][l, :, 2] = rows[k][l, :, 1]
        rows["perf_beta"][l, :, 2] *= F32(0.8)
    rows["perf_acc_count"][5, :, 0] = 0
    rows["perf_acc_count"][6, :, 1] = -2
    rows["perf_max_batch"][7] = np.maximum(rows["perf_max_batch"][7] // 4, 1)
    rows["perf_at_tokens"][7] *= 3
    cand_o, _ = check_level_call(engine, oracle_mod, "profile_grid", fleet, rows, "perf rows")
    c = cand_o.reshape(L, fleet.n_servers, A)
    assert (c[0, :, 0]["feasible"] > c[4, :, 0]["feasible"]).any()
    assert not c[0, :, 2]["feasible"].any() and c[5, :, 2]["feasible"].any()
    srv_n = fleet.srv_max_batch == 0
    assert (c[7][srv_n]["batch"] != c[0][srv_n]["batch"])[c[0][srv_n]["feasible"] == 1].any()
    fixed = (~srv_n) & (c[0, :, 0]["feasible"] == 1) & (c[0, :, 0]["rho"] > 0)
    assert (c[7, :, 0]["batch"][fixed] == fleet.srv_max_batch[fixed]).all()


@pytest.mark.gpu
def test_zero_load_servers(engine, oracle_mod):
    """Zero-load servers with min_replicas 0 and 1 and TPS targets: zeroLoadAllocation at each row's profile and
    price."""
    fleet = profile_fleet(16, 3, 47, False)
    fleet.srv_arrival_rpm[::2] = 0.0
    fleet.srv_min_replicas[::4] = 0
    fleet.srv_min_replicas[2::4] = 1
    fleet.srv_slo_tps[1::3] = F32(500.0)
    rows = profile_rows(fleet, 5, 7)
    cand_o, _ = check_level_call(engine, oracle_mod, "profile_grid", fleet, rows, "zero load")
    c = cand_o.reshape(5, fleet.n_servers, fleet.n_acc)
    z = c[:, ::2]
    assert (z["feasible"] == 1).sum() > 10 and (z["rho"] == 0).all()
    assert len(set(z["itl"][z["replicas"] > 0].tolist())) > 3


@pytest.mark.gpu
def test_repeated_rows_give_identical_blocks(engine, oracle_mod):
    fleet = profile_fleet(14, 3, 53, True)
    rows = profile_rows(fleet, 3, 9)
    rep = {k: v[[0, 1, 0, 2, 1, 1]] for k, v in rows.items()}
    check_level_call(engine, oracle_mod, "profile_grid", fleet, rep, "repeated rows")
    cand, win = engine.profile_grid(fleet, **rep, want_candidates=True)
    S, A = fleet.n_servers, fleet.n_acc
    for k in ALLOC_FIELDS:
        c = getattr(cand, k).reshape(6, S * A)
        w = getattr(win, k).reshape(6, S)
        for x, y in ((0, 2), (1, 4), (1, 5)):
            assert same_bytes(c[x], c[y]) and same_bytes(w[x], w[y]), (k, x, y)


@pytest.mark.gpu
def test_stored_vector_fallback(engine, oracle_mod):
    """N = 1024 near saturation: the chains overflow float64 and the solves re-run on the stored vector; rows change
    the price and move N to 512 and 2048 through the perf batch size."""
    fleet = overflow_fleet()
    fleet.srv_max_batch[:] = 0
    fleet.perf_max_batch[:] = 1024
    fleet.perf_at_tokens[:] = 64
    fleet.srv_arrival_rpm[:] = [rates_at_rate_star(oracle_mod, fleet, s, 0)[k] for s, k in ((0, 0), (1, 3))]
    L = 4
    rows = {"acc_cost": np.array([[1.0], [2.5], [1.0], [0.25]], F32),
            "perf_max_batch": np.array([1024, 1024, 512, 2048], np.int32).reshape(L, 1, 1).repeat(fleet.n_models, 1)}
    cand_o, _ = check_level_call(engine, oracle_mod, "profile_grid", fleet, rows, "stored-vector fallback")
    assert cand_o["feasible"].sum() >= L


@pytest.mark.gpu
def test_against_the_existing_calls(engine, oracle_mod):
    """L = 0; no rows and one level of the fleet's own columns are wva_solve, byte for byte; every level is wva_solve
    on f_l; each candidate block with its level's table is the oracle's greedy in limited mode."""
    fleet = profile_fleet(30, 4, 59, True)
    fleet.type_capacity[:] = [6, 9, 4, 12]
    S, A = fleet.n_servers, fleet.n_acc
    cand0, win0 = engine.profile_grid(fleet, acc_cost=np.zeros((0, A), F32), want_candidates=True)
    assert cand0.n == 0 and win0.n == 0
    cand_s, win_s = engine.solve(at_row(fleet, {}, 0))
    cand1, win1 = engine.profile_grid(fleet, perf_beta=fleet.perf_beta[None], want_candidates=True)
    for k in ALLOC_FIELDS:
        assert same_bytes(getattr(cand1, k), getattr(cand_s, k)) and same_bytes(getattr(win1, k), getattr(win_s, k)), k
    rows = profile_rows(fleet, 5, 13)
    cand_g, win_g = engine.profile_grid(fleet, **rows, want_candidates=True)
    for l in range(5):
        cand_l, win_l = engine.solve(at_row(fleet, rows, l))
        for k in ALLOC_FIELDS:
            assert same_bytes(getattr(cand_g, k)[l * S * A:(l + 1) * S * A], getattr(cand_l, k)), (l, k)
            assert same_bytes(getattr(win_g, k)[l * S:(l + 1) * S], getattr(win_l, k)), (l, k)
        fl = at_row(fleet, rows, l, unlimited=False)
        block = Allocs(S * A)
        for k in ALLOC_FIELDS:
            getattr(block, k)[:] = getattr(cand_g, k)[l * S * A:(l + 1) * S * A]
        cand_lim, win_lim = greedy_solve(fl, block)
        cand_o, win_o = oracle_mod.solve(fl)
        assert_allocs_equal(win_lim, win_o, f"level {l}, limited: winners")
        assert_allocs_equal(cand_lim, cand_o, f"level {l}, limited: candidates")


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_price_rows_size_every_pair_once(engine, monkeypatch, rounds):
    """The launch count depends on the keys, not on L: 1 and 48 price rows launch the same, and so do 2 and 48
    profile rows over the same two beta values."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = synth_fleet(40, 4, seed=71, zero_load_frac=0.0)
    rng = np.random.default_rng(5)

    def launches(**rows):
        n0 = engine.launch_count
        engine.profile_grid(fleet, **rows)
        return engine.launch_count - n0
    A = fleet.n_acc
    price = lambda L: (fleet.acc_cost[None] * rng.uniform(0.5, 2.0, (L, A))).astype(F32)  # noqa: E731
    assert launches(acc_cost=price(1)) == launches(acc_cost=price(48))
    betas = np.stack([fleet.perf_beta, fleet.perf_beta * F32(1.1)])
    assert launches(perf_beta=betas) == launches(perf_beta=betas[[0, 1] * 24], acc_cost=price(48))


@pytest.mark.gpu
def test_batch_size_refusal_at_its_level_only(engine):
    """N = MaxBatchSize * AtTokens / out_tokens: a row with MaxBatchSize 2^16 puts server 0's N above 2^20 on
    accelerator 0.  The grid fails as wva_analyze of that level does; the same row on a server whose batch size is
    fixed, or on an accelerator no loaded server reaches, does not fail."""
    fleet = synth_fleet(4, 2, seed=83, zero_load_frac=0.0)
    fleet.srv_max_batch[0] = 0
    fleet.perf_at_tokens[:] = 1 << 12
    fleet.perf_max_batch[:] = 512
    fleet.srv_out_tokens[:] = 1 << 7
    m0 = int(fleet.srv_model[0])
    mb = np.repeat(fleet.perf_max_batch[None], 3, axis=0).copy()
    mb[1, m0, 0] = 1 << 16  # N = 2^16 * 2^12 / 2^7 = 2^21
    code = error_code(lambda: engine.analyze(at_row(fleet, {"perf_max_batch": mb}, 1)))[0]
    assert code == WVA_ERR_UNSUPPORTED
    assert error_code(lambda: engine.profile_grid(fleet, perf_max_batch=mb))[0] == code
    assert error_code(lambda: engine.profile_grid(fleet, perf_max_batch=mb[[0, 2]]))[0] == 0
    # the same row where it cannot reach a loaded pair: server 0 on a fixed batch size, or accelerator 0 absent
    fixed = fleet.take_servers(np.arange(fleet.n_servers))
    fixed.srv_max_batch[0] = 8
    assert error_code(lambda: engine.profile_grid(fixed, perf_max_batch=mb))[0] == 0
    absent = np.repeat(fleet.perf_present[None], 3, axis=0).copy()
    absent[1, m0, 0] = 0
    assert error_code(lambda: engine.profile_grid(fleet, perf_max_batch=mb, perf_present=absent))[0] == 0


@pytest.mark.gpu
def test_one_handle_with_the_other_paths(engine):
    fleet = profile_fleet(30, 3, 73, True)
    rows = profile_rows(fleet, 4, 23)
    fresh = Engine(0)
    try:
        def same(got, want, what):
            for k in ALLOC_FIELDS:
                assert np.array_equal(getattr(got, k).view(np.uint8), getattr(want, k).view(np.uint8)), f"{what}: {k}"

        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if x is not None:
                    same(x, y, what)

        profile_grid = lambda e: e.profile_grid(fleet, **rows, want_candidates=True)  # noqa: E731
        workload_grid = lambda e: e.workload_grid(fleet, fleet.srv_arrival_rpm[None], want_candidates=True)  # noqa
        # wva_solve -> wva_profile_grid -> wva_resolve: the resident fleet and the solve's cache are untouched
        cand_s, win_s = engine.solve(fleet)
        profile_grid(engine)
        cand_r, win_r = engine.resolve(want_candidates=True)
        same(cand_r, cand_s, "resolve after the profile grid: candidates")
        same(win_r, win_s, "resolve after the profile grid: winners")
        check(profile_grid, "profile grid")
        check(workload_grid, "workload grid after the profile grid")
        check(profile_grid, "profile grid after the workload grid")
        check(lambda e: e.solve(fleet), "solve at the end")
        engine.solve(fleet)
        engine.summarize(fleet.n_types)
        profile_grid(engine)
        with pytest.raises(WvaError) as e:
            engine.summarize(fleet.n_types)
        assert e.value.code == WVA_ERR_STATE
    finally:
        fresh.close()


@pytest.mark.gpu
def test_argument_errors(engine, oracle_mod):
    from workload_variant_autoscaler_b200 import _abi
    fleet = mixed_fleet(6, 2, 79, False)
    L, h = engine._L, engine._h
    win = Allocs(fleet.n_servers)
    fc, wc = fleet.as_c(), win.as_c()
    cost = np.ascontiguousarray(fleet.acc_cost[None])
    rows = _abi.ProfileRowsC(_abi.ptr(cost), *[None] * 8)
    assert L.wva_profile_grid(h, C.byref(fc), -1, C.byref(rows), None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_profile_grid(h, None, 1, C.byref(rows), None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_profile_grid(h, C.byref(fc), 1, C.byref(rows), None, None) == WVA_ERR_BAD_ARG
    # rows NULL: the fleet's own columns, i.e. wva_solve's winners at every level
    win3 = Allocs(3 * fleet.n_servers)
    assert L.wva_profile_grid(h, C.byref(fc), 3, None, None, C.byref(win3.as_c())) == 0
    _, win_s = engine.solve(fleet)
    for k in ALLOC_FIELDS:
        assert same_bytes(getattr(win3, k), np.tile(getattr(win_s, k), 3)), k
    # S * A * L = 2^20 * 2^6 * 32 = 2^31, and L * M * A = 2^25 * 2^6 = 2^31: refused before the fleet is read
    big = fleet.as_c()
    big.n_servers, big.n_acc, big.n_types = 1 << 20, 1 << 6, 0
    assert L.wva_profile_grid(h, C.byref(big), 32, C.byref(rows), None, C.byref(wc)) == WVA_ERR_UNSUPPORTED
    big = fleet.as_c()
    big.n_servers, big.n_models, big.n_acc, big.n_types = 1, 1 << 25, 1 << 6, 0
    assert L.wva_profile_grid(h, C.byref(big), 1, C.byref(rows), None, C.byref(wc)) == WVA_ERR_UNSUPPORTED
    with pytest.raises(ValueError):
        engine.profile_grid(fleet)
    with pytest.raises(ValueError):
        engine.profile_grid(fleet, acc_cost=fleet.acc_cost)
    with pytest.raises(ValueError):
        engine.profile_grid(fleet, acc_cost=cost, perf_beta=np.repeat(fleet.perf_beta[None], 2, axis=0))
    with pytest.raises(ValueError):
        engine.profile_grid(fleet, perf_beta=fleet.perf_beta[None, :, :1])


N_ADV = 30


@pytest.mark.gpu
def test_profile_grid_adversarial(engine, oracle_mod, monkeypatch):
    """Fleets from levels._adversarial_fleet with random rows: prices from an edge set and profiles
    redrawn from the same decades, half of them on the rounds.  Where some level's wva_analyze refuses the level,
    the grid must refuse too."""
    rng = np.random.default_rng(0x9F0)
    feasible = refused = 0
    for case in range(N_ADV):
        fleet = _adversarial_fleet(rng, 60000 + case)
        if case % 2:
            monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        else:
            monkeypatch.delenv("WVA_SIZE_SMALL_MAX", raising=False)
        M, A, L = fleet.n_models, fleet.n_acc, int(rng.integers(1, 6))
        rows = {k: np.repeat(getattr(fleet, k)[None], L, axis=0).copy() for k in COLUMNS}
        rows["acc_cost"] = rng.choice(np.array([0.0, 1e-3, 3.0, 40.0, 1e30, -1.0, np.inf, np.nan], F32), (L, A))
        for k, lo, hi in (("perf_alpha", 1e-3, 1e3), ("perf_beta", 1e-5, 1e2), ("perf_gamma", 1e-3, 1e4),
                          ("perf_delta", 1e-7, 1.0)):
            redraw = rng.random((L, M, A)) < 0.3
            rows[k] = np.where(redraw, np.exp(rng.uniform(np.log(lo), np.log(hi), (L, M, A))), rows[k]).astype(F32)
        rows["perf_present"] = (rng.random((L, M, A)) < 0.85).astype(np.uint8)
        rows["perf_acc_count"] = rng.choice(np.array([-1, 0, 1, 2, 8], np.int32), (L, M, A))
        rows["perf_max_batch"] = rng.choice(np.array([1, 2, 8, 33, 120], np.int32), (L, M, A))
        rows["perf_at_tokens"] = rng.choice(np.array([1, 64, 512, 4096], np.int32), (L, M, A))
        for k in COLUMNS:
            rows[k][0] = getattr(fleet, k)
        if L > 2:
            for k in COLUMNS:
                rows[k][2] = rows[k][1]
        codes = [error_code(lambda: engine.analyze(at_row(fleet, rows, l)))[0] for l in range(L)]
        if any(codes):
            got, _ = error_code(lambda: engine.profile_grid(fleet, **rows))
            assert got == next(c for c in codes if c), (case, codes, got)
            refused += 1
            continue
        _, win_o = check_level_call(engine, oracle_mod, "profile_grid", fleet, rows, f"adversarial case {case}")
        feasible += int(win_o["feasible"].sum())
    assert feasible > 30 and refused < N_ADV // 2
