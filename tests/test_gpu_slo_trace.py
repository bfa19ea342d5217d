"""wva_slo_trace: the reference's reconcile replayed over caller-given ticks of load and service-class targets, each
tick's winner becoming the next tick's current allocation.

The expected result is composed from the CPU oracle, literally: for each tick t, a copy of the fleet with the six
columns (arrival rate, in / out tokens, ITL / TTFT / TPS targets) at row t and current allocation c_t goes through the
oracle's Server.Calculate (candidate block t) and Solver.Solve with unlimited = 1 (winner block t), and c_{t+1} =
Fleet.apply_winners.  The CPU tests pin that composition against the oracle's own solve, show on the oracle that a
search at given (tokens, target) gives the same lambda* whatever the tick's rate, TPS and other target (the premise
of the library's search key), and cross-check the oracle against its restatement on this file's ticks.  The GPU tests
compare the CUDA path with the composition bit for bit."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_load_grid import _code, _f32_bits, _same, mixed_fleet, overflow_fleet, pair_batch, \
    rates_at_rate_star
from tests.test_gpu_parity import _adversarial_fleet
from tests.test_gpu_slo_grid import TARGETS, TPS_TARGETS, _search, at_slo, slo_levels
from tests.test_gpu_workload_grid import at_level, token_fleet, workload_levels
from tests.test_gpu_workload_trace import _moves, _records, low_penalty_fleet, pinned, ref_trace, wva_fleet
from tests.util import ALLOC_FIELDS, assert_allocs_equal
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, synth_fleet

F32 = np.float32
F32_MAX = F32(np.finfo(np.float32).max)
ACC_NONE = -1
WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED = -1, -5, -6
NAMES = ("arrival_rpm", "in_tokens", "out_tokens", "slo_itl", "slo_ttft", "slo_tps")


def at_tick(fleet, rows, t):
    """f_t without the current allocation: a copy of the fleet with the six columns at row t (unlimited)."""
    rpm, in_tok, out_tok, itl, ttft, tps = rows
    return at_slo(at_level(fleet, rpm[t], in_tok[t], out_tok[t]), itl[t], ttft[t], tps[t])


def ref_slo_trace(oracle_mod, fleet, rows):
    """(candidates [L*S*A], winners [L*S]): per tick, the workload trace's composition (Server.Calculate, Solver.Solve
    unlimited, apply_winners) on the fleet whose targets are row t."""
    rpm, in_tok, out_tok, itl, ttft, tps = rows
    cands, wins = [np.zeros(0, oracle_mod.ALLOC_DTYPE)], [np.zeros(0, oracle_mod.ALLOC_DTYPE)]
    cur = fleet
    for t in range(rpm.shape[0]):
        one = slice(t, t + 1)
        cand, win, cur = ref_trace(oracle_mod, at_slo(cur, itl[t], ttft[t], tps[t]), rpm[one], in_tok[one],
                                   out_tok[one])
        cands.append(cand)
        wins.append(win)
    return np.concatenate(cands), np.concatenate(wins)


def slo_trace_rows(fleet, L, seed, special=True):
    """The six row lists, each [L, S]: workload_levels' load and slo_levels' targets (with their edge values when
    `special`)."""
    return (*workload_levels(fleet, L, seed, special), *slo_levels(fleet, L, seed + 7, special))


def schedule(fleet, L, seed):
    """A time-of-day schedule on workload_levels' load (no edge values): ITL x 0.75 in the middle third of the ticks,
    TTFT x 1.5 in the first quarter, the fleet's own TPS."""
    rpm, in_tok, out_tok = workload_levels(fleet, L, seed, special=False)
    S = fleet.n_servers
    itl = np.repeat(fleet.srv_slo_itl[None, :], L, 0).astype(F32)
    ttft = np.repeat(fleet.srv_slo_ttft[None, :], L, 0).astype(F32)
    tps = np.repeat(fleet.srv_slo_tps[None, :], L, 0).astype(F32)
    itl[L // 3:2 * L // 3] *= F32(0.75)
    ttft[:max(L // 4, 1)] *= F32(1.5)
    assert itl.shape == (L, S)
    return rpm, in_tok, out_tok, itl, ttft, tps


def _call(engine, fleet, rows, **kw):
    return engine.slo_trace(fleet, **dict(zip(NAMES, rows)), **kw)


def _check(engine, oracle_mod, fleet, rows, what):
    cand_o, win_o = ref_slo_trace(oracle_mod, fleet, rows)
    cand_g, win_g = _call(engine, fleet, rows, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
    assert_allocs_equal(win_g, win_o, f"{what}: winners")
    return cand_o, win_o


def _same_allocs(got, want, what):
    for k in ALLOC_FIELDS:
        assert _same(getattr(got, k), getattr(want, k)), f"{what}: {k}"


# ---- CPU: the composition, the premise and the restatement -------------------------------------------

@pytest.mark.parametrize("keep", [False, True])
def test_one_tick_is_the_oracle_solve(oracle_mod, keep):
    fleet = token_fleet(12, 3, 5, keep)
    rows = slo_trace_rows(fleet, 3, 9, special=False)
    one = tuple(r[1:2] for r in rows)
    cand, win = ref_slo_trace(oracle_mod, fleet, one)
    cand_o, win_o = oracle_mod.solve(at_tick(fleet, one, 0))
    assert _same(cand, cand_o.reshape(-1))
    assert _same(win, win_o)
    assert win["feasible"].sum() >= 3


def test_search_reads_neither_rate_nor_tps_nor_the_other_target(oracle_mod):
    """The premise of the search key: at a tick's tokens (the Analyzer, which takes no rate) and a given target, the
    TTFT rate of Size is the same under every other tick's ITL and TPS targets, and so is the ITL rate under every
    other tick's TTFT and TPS targets; Size fails exactly when a target is negative or one of the two searches does."""
    fleet = token_fleet(10, 2, 21, False)
    L = 6
    rows = slo_trace_rows(fleet, L, 23)
    checked = 0
    for s in range(fleet.n_servers):
        for t in range(L):
            f = at_tick(fleet, rows, t)
            m = int(f.srv_model[s])
            if m < 0 or not f.srv_has_target[s] or f.srv_out_tokens[s] <= 0 or f.srv_in_tokens[s] < 0 or \
                    not f.srv_arrival_rpm[s] > 0 or pair_batch(f, s, 0) > 4096:
                continue
            for a in range(f.n_acc):
                if not f.perf_present[m, a]:
                    continue
                N = pair_batch(f, s, a)
                qa = oracle_mod.Analyzer(N, N * f.max_queue_to_batch_ratio, float(f.perf_alpha[m, a]),
                                         float(f.perf_beta[m, a]), float(f.perf_gamma[m, a]),
                                         float(f.perf_delta[m, a]), int(f.srv_in_tokens[s]),
                                         int(f.srv_out_tokens[s]))
                tt, ti = float(f.srv_slo_ttft[s]), float(f.srv_slo_itl[s])
                ok_t, _ = _search(oracle_mod, qa, 0, tt)
                ok_i, _ = _search(oracle_mod, qa, 1, ti)
                lone_t, lone_i = qa.size(tt, 0.0, 0.0), qa.size(0.0, ti, 0.0)
                for u in range(L):  # every other tick's other target and TPS
                    other_i, other_t, tp = float(rows[3][u, s]), float(rows[4][u, s]), float(rows[5][u, s])
                    for got, own, lone, key in (((tt, other_i, tp), ok_t, lone_t, "rate_ttft"),
                                                ((other_t, ti, tp), ok_i, lone_i, "rate_itl")):
                        err, rates, _, _ = qa.size(*got)
                        neg = min(got) < 0
                        if neg or err:
                            continue
                        assert own and lone[0] == 0, (s, t, a, u, key)
                        assert _f32_bits(rates[key]) == _f32_bits(lone[1][key]), (s, t, a, u, key)
                        checked += 1
    assert checked >= 100, checked


def test_oracle_agrees_with_the_restatement_on_schedule_ticks(oracle_mod):
    """oracle/restate_np.py against the oracle on a sample of this file's tick fleets f_t (cross_fleet)."""
    from tests.test_oracle_cross import Tally, cross_fleet
    t = Tally()
    f = token_fleet(10, 3, 41, False)
    rows = slo_trace_rows(f, 6, 43)
    for k in (0, 2, 5):
        cross_fleet(oracle_mod, at_tick(f, rows, k), t, f"edge rows, tick {k}")
    g = low_penalty_fleet(10, 3, 45, True)
    rows = schedule(g, 8, 47)
    for k in (0, 3, 7):
        cross_fleet(oracle_mod, at_tick(g, rows, k), t, f"schedule, tick {k}")
    t.report("SLO trace ticks", min_feasible=40, min_infeasible=10)


# ---- GPU: bit for bit against the composition ------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet_warp_path(engine, oracle_mod, keep):
    fleet = token_fleet(14, 3, 31, keep)
    cand_o, win_o = _check(engine, oracle_mod, fleet, slo_trace_rows(fleet, 7, 3), f"warp path, keep = {keep}")
    assert cand_o["feasible"].sum() > 30
    assert len(set(win_o["replicas"][win_o["feasible"] == 1].tolist())) >= 3


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = token_fleet(120, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    fleet.accel_penalty_factor = 0.02
    rows = slo_trace_rows(fleet, 4, 11)
    return fleet, rows, ref_slo_trace(oracle_mod, fleet, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rows, (cand_o, win_o) = rounds_case
    cand_g, win_g = _call(engine, fleet, rows, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"rounds, D = {depth}: candidates")
    assert_allocs_equal(win_g, win_o, f"rounds, D = {depth}: winners")


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("rounds", [False, True])
def test_schedule_moves_winners_and_back(engine, oracle_mod, monkeypatch, keep, rounds):
    """No penalty for a switch, the fleet's own load, ITL tightened in the middle ticks: winners leave their
    accelerator when the target tightens and come back when it relaxes."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = low_penalty_fleet(40, 4, 89, keep)
    if keep:
        fleet.srv_min_replicas[::2] = 0
    L, S = 9, fleet.n_servers
    rows = list(schedule(fleet, L, 29))
    for k in range(3):
        rows[k] = np.repeat(rows[k][:1], L, 0)  # one load: only the targets move
    rows[3][3:6] = rows[3][3:6] * F32(0.5)
    rows[0][7, ::3] = 0.0
    _, win_o = _check(engine, oracle_mod, fleet, tuple(rows), f"schedule, keep = {keep}")
    assert _moves(win_o, S) >= (2 if keep else 4)


@pytest.mark.gpu
def test_wva_configuration_every_server_pinned(engine, oracle_mod):
    fleet = wva_fleet(60, 4, 97)
    assert pinned(fleet).all()
    rows = schedule(fleet, 6, 31)
    _, win_o = _check(engine, oracle_mod, fleet, rows, "WVA configuration")
    win = win_o.reshape(6, -1)
    for t in range(6):
        f = win[t]["feasible"] != 0
        assert f.sum() >= 20
        assert (win[t]["acc"][f] == fleet.srv_cur_acc[f]).all()


@pytest.mark.gpu
def test_edge_targets_with_edge_loads(engine, oracle_mod):
    """Per tick the TARGETS edges (0, -0, NaN, negative, denormal, +Inf, MaxFloat32) in ITL and TTFT and the
    TPS_TARGETS in TPS, mixed with rate 0, a negative rate, out_tokens 0, a nil winner that keeps c_t, and a zero-load
    winner with min_replicas 0."""
    fleet = token_fleet(24, 3, 53, True)
    fleet.srv_min_replicas[::3] = 0
    L, S = 8, fleet.n_servers
    rows = [np.array(r) for r in slo_trace_rows(fleet, L, 57)]
    rpm, _, out_tok, itl, ttft, tps = rows
    for t, v in enumerate(TARGETS):
        itl[t, ::5] = v
        ttft[(t + 3) % L, 1::5] = v
    for t, v in enumerate(TPS_TARGETS):
        tps[t, 2::7] = v
    rpm[1, ::4] = 0.0
    rpm[2, 1::6] = -1.0
    out_tok[3, 2::6] = 0
    cand_o, win_o = _check(engine, oracle_mod, fleet, tuple(rows), "edge targets and loads")
    win = win_o.reshape(L, S)
    assert (win["feasible"] == 0).sum() >= 10
    assert ((win["feasible"] == 1) & (win["acc"] == ACC_NONE)).sum() >= 1


@pytest.mark.gpu
def test_stored_vector_fallback_both_phases(engine, oracle_mod):
    """N = 1024 near saturation: the searches and the tail re-run on the stored vector, under a TTFT / ITL schedule."""
    fleet = overflow_fleet()
    fleet.srv_max_batch[:] = 0
    fleet.perf_max_batch[:] = 1024
    fleet.perf_at_tokens[:] = 64
    S = fleet.n_servers
    cols = [rates_at_rate_star(oracle_mod, fleet, s, 0) for s in range(S)]
    L = min(len(c) for c in cols)
    rpm = np.stack([np.array(c[:L], np.float32) for c in cols], axis=1)
    out_tok = np.full((L, S), 64, np.int32)
    out_tok[1::4] = 128
    in_tok = np.full((L, S), 64, np.int32)
    itl = np.zeros((L, S), F32)
    ttft = np.zeros((L, S), F32)
    tps = np.zeros((L, S), F32)
    itl[::3] = 1e6
    ttft[1::3] = 1e9
    cand_o, _ = _check(engine, oracle_mod, fleet, (rpm, in_tok, out_tok, itl, ttft, tps), "stored-vector fallback")
    assert cand_o["feasible"].sum() >= L


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_nan_and_huge_values_and_ties(engine, oracle_mod, keep):
    fleet = token_fleet(12, 3, 47, keep)
    fleet.srv_cur_cost[::2] = np.nan
    fleet.srv_cur_cost[1::4] = -F32_MAX
    fleet.acc_cost[2] = fleet.acc_cost[1]
    fleet.perf_alpha[:, 2] = fleet.perf_alpha[:, 1]
    for k in ("perf_beta", "perf_gamma", "perf_delta", "perf_acc_count"):
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]
    _check(engine, oracle_mod, fleet, slo_trace_rows(fleet, 5, 17), f"NaN / huge values and ties, keep = {keep}")


@pytest.mark.gpu
@pytest.mark.parametrize("s, value, fails", [(6, np.nan, True), (6, 1e-45, True), (0, np.nan, False)])
def test_nan_or_tiny_tps_tick_fails_as_solve_does(engine, s, value, fails):
    """The SLO grid's NaN / tiny TPS case at tick 1 of a trace: the trace fails exactly when wva_solve of that tick
    fails, and otherwise gives its records; the trace without that tick succeeds."""
    fleet = mixed_fleet(10, 3, 71, False)
    assert fleet.srv_arrival_rpm[s] > 0 and fleet.srv_min_replicas[s] == 0
    L, S, A = 3, fleet.n_servers, fleet.n_acc
    itl, ttft, tps = slo_levels(fleet, L, 19, special=False)
    tps[1, s] = value
    rows = (None, None, None, itl, ttft, tps)
    cur = fleet
    _, res0 = _code(lambda: engine.solve(at_slo(cur, itl[0], ttft[0], tps[0])))
    cur = fleet.apply_winners(res0[1])
    want, res = _code(lambda: engine.solve(at_slo(cur, itl[1], ttft[1], tps[1])))
    got, tr = _code(lambda: _call(engine, fleet, rows, want_candidates=True))
    assert got == want == (WVA_ERR_UNSUPPORTED if fails else 0)
    if want == 0:
        for k in ALLOC_FIELDS:
            assert _same(getattr(tr[0], k)[S * A:2 * S * A], getattr(res[0], k)), k
            assert _same(getattr(tr[1], k)[S:2 * S], getattr(res[1], k)), k
    keep = [0, 2]
    assert _code(lambda: engine.slo_trace(fleet, slo_itl=itl[keep], slo_ttft=ttft[keep], slo_tps=tps[keep]))[0] == 0


# ---- GPU: against the library's other calls ---------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_no_targets_is_the_workload_trace(engine, monkeypatch, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = token_fleet(40, 4, 61, True)
    fleet.accel_penalty_factor = 0.01
    rows = workload_levels(fleet, 6, 63)
    got = engine.slo_trace(fleet, *rows, want_candidates=True)
    want = engine.workload_trace(fleet, *rows, want_candidates=True)
    _same_allocs(got[0], want[0], "candidates")
    _same_allocs(got[1], want[1], "winners")
    # a NULL load list is the fleet's own column
    got = engine.slo_trace(fleet, rows[0], want_candidates=True)
    want = engine.workload_trace(fleet, rows[0], want_candidates=True)
    _same_allocs(got[0], want[0], "own tokens: candidates")


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_one_tick_is_the_slo_grid(engine, monkeypatch, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = token_fleet(40, 4, 65, True)
    rows = slo_trace_rows(fleet, 3, 67)
    for t in range(3):
        one = [r[t:t + 1] for r in rows]
        got = _call(engine, fleet, one, want_candidates=True)
        want = engine.slo_grid(at_level(fleet, rows[0][t], rows[1][t], rows[2][t]), *one[3:], want_candidates=True)
        _same_allocs(got[0], want[0], f"tick {t}: candidates")
        _same_allocs(got[1], want[1], f"tick {t}: winners")


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3, 5])
def test_continuation(engine, k):
    fleet = low_penalty_fleet(30, 3, 103, True)
    fleet.srv_min_replicas[::2] = 0
    L, S = 7, fleet.n_servers
    rows = [np.array(r) for r in slo_trace_rows(fleet, L, 37)]
    rows[0][2, ::3] = 0.0
    cand, win = _call(engine, fleet, rows, want_candidates=True)
    cand_a, win_a = _call(engine, fleet, [r[:k] for r in rows], want_candidates=True)
    cur = fleet
    for t in range(k):
        cur = cur.apply_winners(_records(win_a)[t * S:(t + 1) * S])
    cand_b, win_b = _call(engine, cur, [r[k:] for r in rows], want_candidates=True)
    for n in ALLOC_FIELDS:
        assert _same(getattr(cand, n), np.concatenate([getattr(cand_a, n), getattr(cand_b, n)])), n
        assert _same(getattr(win, n), np.concatenate([getattr(win_a, n), getattr(win_b, n)])), n
    assert _moves(_records(win), S) >= 1


@pytest.mark.gpu
def test_each_tick_is_solve_on_the_advanced_fleet(engine):
    fleet = synth_fleet(1500, 8, seed=69)
    L, S, A = 6, fleet.n_servers, fleet.n_acc
    rows = schedule(fleet, L, 71)
    cand_g, win_g = _call(engine, fleet, rows, want_candidates=True)
    cur = fleet
    for t in range(L):
        cand_s, win_s = engine.solve(at_tick(cur, rows, t))
        for k in ALLOC_FIELDS:
            assert _same(getattr(cand_g, k)[t * S * A:(t + 1) * S * A], getattr(cand_s, k)), (t, k)
            assert _same(getattr(win_g, k)[t * S:(t + 1) * S], getattr(win_s, k)), (t, k)
        cur = cur.apply_winners(win_s)
    assert win_g.feasible.sum() >= L * S // 4


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_launches_do_not_grow_with_identical_ticks(engine, monkeypatch, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = synth_fleet(40, 4, seed=71, zero_load_frac=0.0)

    def launches(L):
        rows = [np.repeat(r[:1], L, 0) for r in schedule(fleet, 2, 73)]
        n0 = engine.launch_count
        _call(engine, fleet, rows)
        return engine.launch_count - n0
    assert launches(1) == launches(64)


@pytest.mark.gpu
def test_argument_errors_and_refusals(engine):
    from workload_variant_autoscaler_b200 import _abi
    fleet = mixed_fleet(6, 2, 79, False)
    L, h = engine._L, engine._h
    win = Allocs(fleet.n_servers)
    fc, wc = fleet.as_c(), win.as_c()
    one = np.ones(fleet.n_servers, np.float32)
    tok = np.ones(fleet.n_servers, np.int32)
    p, t = _abi.ptr(one), _abi.ptr(tok)
    assert L.wva_slo_trace(h, C.byref(fc), -1, p, t, t, p, p, p, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_slo_trace(h, C.byref(fc), 1, p, t, t, p, p, p, None, None) == WVA_ERR_BAD_ARG
    assert L.wva_slo_trace(h, None, 1, p, t, t, p, p, p, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    # every list NULL is valid: the fleet's own columns
    assert L.wva_slo_trace(h, C.byref(fc), 1, None, None, None, None, None, None, None, C.byref(wc)) == 0
    # S * A * L = 2^20 * 2^6 * 32 = 2^31: refused before the fleet is read
    big = fleet.as_c()
    big.n_servers, big.n_acc, big.n_types = 1 << 20, 1 << 6, 0
    assert L.wva_slo_trace(h, C.byref(big), 32, p, t, t, p, p, p, None, C.byref(wc)) == WVA_ERR_UNSUPPORTED
    with pytest.raises(ValueError):
        engine.slo_trace(fleet)
    with pytest.raises(ValueError):
        engine.slo_trace(fleet, one)
    with pytest.raises(ValueError):
        engine.slo_trace(fleet, one[None, :], slo_itl=np.ones((2, fleet.n_servers), np.float32))
    with pytest.raises(ValueError):
        engine.slo_trace(fleet, slo_itl=one[None, :], out=Allocs(2 * fleet.n_servers))
    z = np.zeros((0, fleet.n_servers), np.float32)
    cand, win0 = engine.slo_trace(fleet, slo_ttft=z, want_candidates=True)
    assert cand.n == 0 and win0.n == 0
    # a load pair outside the queue-size rule at some tick is refused, as the workload trace refuses it
    g = synth_fleet(4, 2, seed=83, zero_load_frac=0.0)
    g.srv_max_batch[0] = 0
    g.perf_max_batch[:] = 512
    g.perf_at_tokens[:] = 1 << 12
    out_tok = np.full((2, 4), 1 << 16, np.int32)
    out_tok[1, 0] = 1
    assert _code(lambda: engine.slo_trace(g, out_tokens=out_tok))[0] == WVA_ERR_UNSUPPORTED
    engine.solve(fleet)


@pytest.mark.gpu
def test_one_handle_with_the_other_paths(engine):
    fleet = token_fleet(30, 3, 73, True)
    rows = slo_trace_rows(fleet, 4, 23)
    fresh = Engine(0)
    try:
        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if x is not None:
                    for k in ALLOC_FIELDS:
                        assert np.array_equal(getattr(x, k).view(np.uint8), getattr(y, k).view(np.uint8)), \
                            f"{what}: {k}"

        trace = lambda e: _call(e, fleet, rows, want_candidates=True)  # noqa: E731
        cand_s, win_s = engine.solve(fleet)
        trace(engine)
        cand_r, win_r = engine.resolve(want_candidates=True)
        _same_allocs(cand_r, cand_s, "resolve after the trace: candidates")
        _same_allocs(win_r, win_s, "resolve after the trace: winners")
        check(trace, "trace")
        check(lambda e: e.slo_grid(fleet, *rows[3:], want_candidates=True), "SLO grid after the trace")
        check(trace, "trace after the SLO grid")
        check(lambda e: e.workload_trace(fleet, *rows[:3], want_candidates=True), "workload trace")
        check(trace, "trace after the workload trace")
        check(lambda e: e.solve(fleet), "solve at the end")
        engine.solve(fleet)
        engine.summarize(fleet.n_types)
        trace(engine)
        with pytest.raises(WvaError) as e:
            engine.summarize(fleet.n_types)
        assert e.value.code == WVA_ERR_STATE
    finally:
        fresh.close()


N_ADV = 30


@pytest.mark.gpu
def test_slo_trace_adversarial(engine, oracle_mod, monkeypatch):
    """Fleets from test_gpu_parity's _adversarial_fleet, keep on half the servers, with random load and target rows
    from the edge sets, half of them on the rounds.  Where the per-tick wva_solve loop refuses a tick the trace
    refuses too; it may refuse beyond that only through a keep server that is not pinned."""
    rng = np.random.default_rng(0x5107)
    feasible = refused = extra = 0
    for case in range(N_ADV):
        fleet = _adversarial_fleet(rng, 70000 + case)
        S, A, L = fleet.n_servers, fleet.n_acc, int(rng.integers(1, 6))
        fleet.srv_keep_acc[:] = rng.random(S) < 0.5
        fleet.srv_cur_acc[:] = rng.integers(-2, A, S)
        fleet.accel_penalty_factor = float(rng.choice([0.0, 0.1]))
        if case % 2:
            monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        else:
            monkeypatch.delenv("WVA_SIZE_SMALL_MAX", raising=False)
        rpm = rng.choice(np.array([0.0, 1e-3, 3.0, 600.0, 1e6, -1.0, np.inf], np.float32), (L, S),
                         p=[.15, .1, .25, .25, .1, .05, .1])
        in_tok = rng.choice(np.array([0, 1, 7, 512, 100000], np.int32), (L, S), p=[.15, .15, .2, .3, .2])
        out_tok = rng.choice(np.array([0, 1, 2, 9, 300, 50000], np.int32), (L, S), p=[.1, .1, .15, .15, .3, .2])
        itl = rng.choice(np.array([0.0, 1e-3, 5.0, 80.0, 1e6, -1.0, np.nan], np.float32), (L, S),
                         p=[.2, .15, .2, .2, .15, .05, .05])
        ttft = rng.choice(np.array([0.0, 1e-2, 50.0, 2000.0, 1e7, -0.0, np.inf], np.float32), (L, S),
                          p=[.2, .15, .2, .2, .15, .05, .05])
        tps = rng.choice(np.array([0.0, 10.0, 1e4, -1.0, np.inf], np.float32), (L, S), p=[.5, .2, .15, .05, .1])
        rows = (rpm, in_tok, out_tok, itl, ttft, tps)
        code, cur = 0, fleet
        for t in range(L):
            code, res = _code(lambda: engine.solve(at_tick(cur, rows, t)))
            if code:
                break
            cur = cur.apply_winners(res[1])
        got, _ = _code(lambda: _call(engine, fleet, rows))
        if code:
            assert got == code, (case, code, got)
            refused += 1
            continue
        if got:
            assert got == WVA_ERR_UNSUPPORTED and ((fleet.srv_keep_acc != 0) & ~pinned(fleet)).any(), (case, got)
            extra += 1
            continue
        _, win_o = _check(engine, oracle_mod, fleet, rows, f"adversarial case {case}")
        feasible += int(win_o["feasible"].sum())
    assert feasible > 30 and refused + extra < N_ADV // 2
