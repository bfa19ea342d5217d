"""wva_load_grid: the reference's Server.Calculate and SolveUnlimited winner at many caller-given arrival rates.

The expected result is composed from the CPU oracle, literally: for each level l, a copy of the fleet with
srv_arrival_rpm = row l and unlimited = 1 goes through the oracle's Server.Calculate (candidate block l) and
Solver.Solve (winner block l).  The CPU tests pin that composition against the oracle's own solve and show on the
oracle that CreateAllocation splits into a load-independent Size and a per-level tail; the GPU tests compare the
CUDA path with the composition bit for bit."""
import ctypes as C

import numpy as np
import pytest

from tests.util import assert_allocs_equal
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, greedy_solve, synth_fleet

F32_MAX = np.float32(np.finfo(np.float32).max)
WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED = -1, -5, -6
ALLOC_FIELDS = ("feasible", "acc", "replicas", "batch", "cost", "value", "itl", "ttft", "rho", "max_rate")


def at_level(fleet, row, unlimited=True):
    """A copy of the fleet with srv_arrival_rpm = row."""
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_arrival_rpm[:] = row
    f.unlimited = unlimited
    return f


def ref_load_grid(oracle_mod, fleet, rpm):
    """(candidates [L*S*A], winners [L*S]): Server.Calculate and Solver.Solve (unlimited) per level."""
    cands, wins = [np.zeros(0, oracle_mod.ALLOC_DTYPE)], [np.zeros(0, oracle_mod.ALLOC_DTYPE)]
    for row in rpm:
        f = at_level(fleet, row)
        cand = oracle_mod.calculate(f)
        cands.append(cand.reshape(-1))
        wins.append(oracle_mod.solve(f, cand)[1])
    return np.concatenate(cands), np.concatenate(wins)


def mixed_fleet(n_servers, n_acc, seed, keep):
    """Zero load, TPS targets, an unknown model, a server without a target, a missing profile, min_replicas = 0,
    an unknown current accelerator, keepAccelerator on or off."""
    f = synth_fleet(n_servers, n_acc, seed=seed, keep_accelerator=keep, zero_load_frac=0.2, tps_frac=0.3)
    f.srv_min_replicas[::3] = 0
    f.perf_present[1, n_acc - 1] = 0
    f.srv_has_target[2] = 0
    f.srv_model[3] = -1
    f.srv_cur_acc[4] = -2
    f.srv_keep_acc[4] = 1
    return f


def load_levels(fleet, L, seed):
    """[L, S]: each server's own load times a seeded log-normal factor per (level, server), so the levels are
    per-server and non-monotone, with 0, negative, +Inf, tiny and huge rates scattered over them."""
    rng = np.random.default_rng(seed)
    S = fleet.n_servers
    base = np.maximum(fleet.srv_arrival_rpm, 1.0)
    rpm = (base[None, :] * rng.lognormal(0.0, 0.8, (L, S))).astype(np.float32)
    for k, v in enumerate((0.0, -1.0, np.inf, 1e-3, 1e6)):
        rpm[k % L, k::5 + k] = v
    return rpm


def _same(a, b):
    return np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


def _f32_bits(x):
    v = np.float32(x)
    return 0x7FC00000 if np.isnan(v) else int(np.array([v]).view(np.uint32)[0])


# ---- CPU: the composition and the split --------------------------------------------------------

@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("seed", [1, 2])
def test_one_level_is_the_oracle_solve(oracle_mod, seed, keep):
    fleet = mixed_fleet(12, 3, seed, keep)
    cand, win = ref_load_grid(oracle_mod, fleet, fleet.srv_arrival_rpm[None, :])
    cand_o, win_o = oracle_mod.solve(at_level(fleet, fleet.srv_arrival_rpm))
    assert _same(cand, cand_o.reshape(-1))
    assert _same(win, win_o)
    assert win["feasible"].sum() >= 4


def pair_batch(fleet, s, a):
    """allocation.go:77-87."""
    if fleet.srv_max_batch[s] > 0:
        return int(fleet.srv_max_batch[s])
    m = fleet.srv_model[s]
    return max(int(fleet.perf_max_batch[m, a]) * int(fleet.perf_at_tokens[m, a]) // int(fleet.srv_out_tokens[s]), 1)


def go_f64_to_int(x):
    return int(x) if -2.0 ** 63 <= x < 2.0 ** 63 else -(1 << 63)


def tail(oracle_mod, qa, fleet, s, a, N, rate_star, rpm):
    """allocation.go:134-163 at arrival rate rpm, with the pair's analyzer after one Size: the record."""
    f32 = np.float32
    rec = np.zeros(1, oracle_mod.ALLOC_DTYPE)[0]
    rec["acc"] = -1
    m = fleet.srv_model[s]
    with np.errstate(all="ignore"):
        tps = f32(fleet.srv_slo_tps[s])
        total = f32(rpm) / f32(60) if tps == 0 else tps / f32(fleet.srv_out_tokens[s])
        nrep = go_f64_to_int(np.ceil(np.float64(total) / np.float64(rate_star)))
        nrep = max(nrep, int(fleet.srv_min_replicas[s]))
        inst = int(fleet.perf_acc_count[m, a])
        inst = 1 if inst <= 0 else inst
        cost = f32(fleet.acc_cost[a]) * np.array([inst * nrep], np.int64).astype(f32)[0]
        rate = total / np.array([nrep], np.int64).astype(f32)[0]
    err, met = qa.analyze(float(rate))
    if err:
        return rec
    rec["feasible"], rec["acc"], rec["replicas"], rec["batch"] = 1, a, nrep, N
    rec["cost"] = rec["value"] = cost
    rec["itl"] = met["avg_token_time"]
    rec["ttft"] = f32(met["avg_wait_time"]) + f32(met["avg_prefill_time"])
    rec["rho"] = met["rho"]
    rec["max_rate"] = f32(rate_star) / f32(1000)
    return rec


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
                want = oracle_mod.create_allocation(at_level(fleet, np.full(fleet.n_servers, rpm, np.float32)), s, a)
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
                        assert _f32_bits(got[k]) == _f32_bits(want[k]), (s, a, rpm, k, got[k], want[k])
                    else:
                        assert int(got[k]) == int(want[k]), (s, a, rpm, k, got[k], want[k])
                checked += int(want["feasible"])
    assert checked >= 40


def test_max_rate_is_the_same_at_every_load_level(oracle_mod):
    fleet = mixed_fleet(20, 3, 5, False)
    rpm = load_levels(fleet, 6, 7)
    cand, _ = ref_load_grid(oracle_mod, fleet, rpm)
    cand = cand.reshape(6, fleet.n_servers, fleet.n_acc)
    load = ~(rpm < 0) & (rpm != 0)
    seen = 0
    for s in range(fleet.n_servers):
        for a in range(fleet.n_acc):
            rates = {_f32_bits(cand[l, s, a]["max_rate"]) for l in range(6) if load[l, s] and cand[l, s, a]["feasible"]}
            assert len(rates) <= 1, (s, a)
            seen += len(rates)
    assert seen >= 20


# ---- GPU: bit for bit against the composition -------------------------------------------------

def _check(engine, oracle_mod, fleet, rpm, what):
    cand_o, win_o = ref_load_grid(oracle_mod, fleet, rpm)
    cand_g, win_g = engine.load_grid(fleet, rpm, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
    assert_allocs_equal(win_g, win_o, f"{what}: winners")
    return cand_o, win_o


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet(engine, oracle_mod, monkeypatch, keep, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = mixed_fleet(14, 3, 31, keep)
    rpm = load_levels(fleet, 7, 3)
    cand_o, win_o = _check(engine, oracle_mod, fleet, rpm, f"small, keep = {keep}, rounds = {rounds}")
    assert cand_o["feasible"].sum() > 40
    assert len(set(win_o["replicas"][win_o["feasible"] == 1].tolist())) >= 3


@pytest.fixture(scope="module")
def large_case(oracle_mod):
    fleet = mixed_fleet(560, 4, 37, False)  # > 2,000 load pairs: the rounds
    fleet.srv_keep_acc[::2] = 1
    rpm = load_levels(fleet, 3, 11)
    return fleet, rpm, ref_load_grid(oracle_mod, fleet, rpm)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [None, "1", "2", "3", "4", "5"])
def test_large_fleet_every_tree_depth(engine, large_case, monkeypatch, depth):
    if depth is not None:
        monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rpm, (cand_o, win_o) = large_case
    cand_g, win_g = engine.load_grid(fleet, rpm, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"large, D = {depth}: candidates")
    assert_allocs_equal(win_g, win_o, f"large, D = {depth}: winners")


def overflow_fleet():
    """The overflow fleet of test_overflow_rescale_falls_back_to_stored_vector: near saturation at N = 1024 the
    chain overflows float64, and the solves re-run on the stored vector with the reference's rescale loops."""
    fleet = synth_fleet(2, 1, seed=29, max_batch_choices=(1024,))
    fleet.perf_alpha[:] = 7.47
    fleet.perf_beta[:] = 0.0001
    fleet.perf_gamma[:] = 1.0
    fleet.perf_delta[:] = 0.00001
    fleet.srv_in_tokens[:] = 64
    fleet.srv_out_tokens[:] = 64
    fleet.srv_slo_tps[:] = 0
    fleet.srv_slo_itl[:] = 0
    fleet.srv_slo_ttft[:] = 0
    fleet.srv_min_replicas[:] = 1
    return fleet


def rates_at_rate_star(oracle_mod, fleet, s, a):
    """Arrival rates (req/min) at which totalRate / replicas lands at rateStar or one ulp under it, for 1..3
    replicas."""
    m = fleet.srv_model[s]
    N = pair_batch(fleet, s, a)
    qa = oracle_mod.Analyzer(N, N * fleet.max_queue_to_batch_ratio, float(fleet.perf_alpha[m, a]),
                             float(fleet.perf_beta[m, a]), float(fleet.perf_gamma[m, a]), float(fleet.perf_delta[m, a]),
                             int(fleet.srv_in_tokens[s]), int(fleet.srv_out_tokens[s]))
    err, _, met, _ = qa.size(0.0, 0.0, 0.0)
    assert err == 0
    star = np.float32(met["throughput"])
    under = np.nextafter(star, np.float32(0))
    out = []
    for k in (1, 2, 3):
        x = np.float32(star * np.float32(k * 60))
        hits = set()
        for _ in range(200):
            x = np.nextafter(x, np.float32(0))
        for _ in range(400):
            x = np.nextafter(x, np.float32(np.inf))
            total = x / np.float32(60)
            n = go_f64_to_int(np.ceil(np.float64(total) / np.float64(star)))
            r = total / np.float32(n)
            if n == k and r in (star, under):
                hits.add(r == star)
                out.append(float(x))
        assert hits, k
    return out


@pytest.mark.gpu
def test_stored_vector_fallback_both_phases(engine, oracle_mod):
    fleet = overflow_fleet()
    cols = [rates_at_rate_star(oracle_mod, fleet, s, 0) for s in range(2)]
    L = min(len(c) for c in cols)
    rpm = np.stack([np.array(c[:L], np.float32) for c in cols], axis=1)
    cand_o, _ = _check(engine, oracle_mod, fleet, rpm, "stored-vector fallback")
    assert cand_o["feasible"].sum() >= L


@pytest.mark.gpu
def test_each_level_is_analyze_and_solve(engine, oracle_mod):
    fleet = mixed_fleet(30, 4, 41, True)
    fleet.type_capacity[:] = [6, 9, 4, 12]
    rpm = load_levels(fleet, 5, 13)
    cand_g, win_g = engine.load_grid(fleet, rpm, want_candidates=True)
    S, A = fleet.n_servers, fleet.n_acc
    for l in range(5):
        f = at_level(fleet, rpm[l])
        cand_a = engine.analyze(f)
        _, win_s = engine.solve(f)
        for k in ALLOC_FIELDS:
            assert _same(getattr(cand_g, k)[l * S * A:(l + 1) * S * A], getattr(cand_a, k)), (l, k)
            assert _same(getattr(win_g, k)[l * S:(l + 1) * S], getattr(win_s, k)), (l, k)
        # limited mode by composition: the level's candidate block into the greedy pass
        fl = at_level(fleet, rpm[l], unlimited=False)
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
        assert _same(getattr(win1, k), getattr(win_s, k)), k


@pytest.mark.gpu
def test_nan_and_huge_values_and_ties(engine, oracle_mod):
    fleet = mixed_fleet(12, 3, 43, False)
    fleet.srv_cur_cost[::2] = np.nan     # penalty NaN except for the current (accelerator, replicas)
    fleet.srv_cur_cost[1::4] = -F32_MAX  # the current accelerator's penalty rounds to MaxFloat32
    fleet.acc_cost[2] = fleet.acc_cost[1]
    fleet.perf_alpha[:, 2] = fleet.perf_alpha[:, 1]  # accelerators 1 and 2 identical: ties on value
    for k in ("perf_beta", "perf_gamma", "perf_delta", "perf_acc_count"):
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]
    _check(engine, oracle_mod, fleet, load_levels(fleet, 4, 17), "NaN / huge values and ties")


def _code(fn):
    try:
        return 0, fn()
    except WvaError as e:
        return e.code, None


@pytest.mark.gpu
def test_nan_level_fails_as_analyze_does(engine):
    fleet = mixed_fleet(10, 3, 47, False)
    rpm = load_levels(fleet, 3, 19)
    rpm[1, 5] = np.nan
    want, cand_a = _code(lambda: engine.analyze(at_level(fleet, rpm[1])))
    got, res = _code(lambda: engine.load_grid(fleet, rpm, want_candidates=True))
    assert got == want
    if want == 0:
        S, A = fleet.n_servers, fleet.n_acc
        for k in ALLOC_FIELDS:
            assert _same(getattr(res[0], k)[S * A:2 * S * A], getattr(cand_a, k)), k


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
