"""wva_profile_trace: the reference's reconcile replayed over caller-given ticks of load (arrival rate, in_tokens,
out_tokens), accelerator costs and model x accelerator performance profiles, each tick's winner becoming the next
tick's current allocation.

The expected result is composed from the CPU oracle, literally: for each tick t, a copy of the fleet with workload
row t, profile row t and current allocation c_t goes through the oracle's Server.Calculate (candidate block t) and
Solver.Solve with unlimited = 1 (winner block t), and c_{t+1} = Fleet.apply_winners (Server.ApplyDesiredAlloc).  The
CPU tests pin that composition against the oracle's own solve and show on the oracle that a price change between
ticks carries the winner's allocation, cost included, as the winner recorded it.  The GPU tests compare the CUDA
path with the composition bit for bit."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (COLUMNS, LOAD, PERF, ROW_COLUMN, _adversarial_fleet, _moves, _records, at_row, check_level_call, overflow_fleet,
                          pinned, profile_fleet, profile_rows, rates_at_rate_star, ref_trace, transition_penalty,
                          workload_levels)
from tests.util import (ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, assert_allocs_equal,
                        error_code, f32_bits, same_bytes)
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, synth_fleet

F32 = np.float32
def load_rows(fleet, L, seed, special=True):
    rpm, in_tok, out_tok = workload_levels(fleet, L, seed, special=special)
    return {"arrival_rpm": rpm, "in_tokens": in_tok, "out_tokens": out_tok}
LOAD_COLUMN = {k: ROW_COLUMN[k] for k in LOAD}


def hourly_prices(fleet, L, seed):
    """acc_cost [L, A]: a daily curve per accelerator with its own phase and depth, plus noise."""
    rng = np.random.default_rng(seed)
    A = fleet.n_acc
    t = np.arange(L)[:, None]
    phase, depth = rng.uniform(0, 2 * np.pi, A), rng.uniform(0.2, 0.8, A)
    curve = 1.0 + depth * np.sin(2 * np.pi * t / 24.0 + phase) + rng.normal(0, 0.03, (L, A))
    return (fleet.acc_cost[None] * np.maximum(curve, 0.05)).astype(F32)


def _bytes_equal(got, want, what):
    for k in ALLOC_FIELDS:
        assert np.array_equal(getattr(got, k).view(np.uint8), getattr(want, k).view(np.uint8)), f"{what}: {k}"


# ---- CPU: the composition and the carried allocation --------------------------------------------

@pytest.mark.parametrize("keep", [False, True])
def test_one_tick_is_the_oracle_solve(oracle_mod, keep):
    fleet = profile_fleet(12, 3, 5, keep)
    rows = {"arrival_rpm": fleet.srv_arrival_rpm[None] * F32(1.5), "acc_cost": fleet.acc_cost[None] * F32(0.7)}
    rows["perf_beta"] = fleet.perf_beta[None] * F32(0.9)
    cand, win, _ = ref_trace(oracle_mod, fleet, rows)
    cand_o, win_o = oracle_mod.solve(at_row(fleet, rows, 0))
    assert same_bytes(cand, cand_o.reshape(-1))
    assert same_bytes(win, win_o)
    assert win["feasible"].sum() >= 4


@pytest.mark.parametrize("seed", [3, 4])
def test_price_change_carries_the_winners_allocation(oracle_mod, seed):
    """Along an oracle trace whose prices change at every tick, c_{t+1} is winner t's (acc, replicas, cost) as the
    winner recorded it, the cost at tick t's prices, and tick t+1's values are TransitionPenalty against that cost,
    not against the cost re-priced at tick t+1."""
    fleet = profile_fleet(16, 3, seed, False)
    fleet.accel_penalty_factor = 0.1
    L = 5
    price = fleet.acc_cost[None] * np.array([[1.0], [2.0], [0.5], [3.0], [0.8]], F32)
    rows = {"acc_cost": price.astype(F32)}
    S, A = fleet.n_servers, fleet.n_acc
    cur, carried, repriced = fleet, 0, 0
    for t in range(L):
        f = at_row(cur, rows, t)
        cand = oracle_mod.calculate(f)
        win = oracle_mod.solve(f, cand)[1]
        if t > 0:
            for s in range(S):
                for a in range(A):
                    c = cand[s, a]
                    if not c["feasible"]:
                        continue
                    want = transition_penalty(f.accel_penalty_factor, cur.srv_cur_acc[s], cur.srv_cur_replicas[s],
                                              cur.srv_cur_cost[s], c["acc"], c["replicas"], c["cost"])
                    assert f32_bits(c["value"]) == f32_bits(want), (t, s, a)
                    if a == cur.srv_cur_acc[s] and c["replicas"] == cur.srv_cur_replicas[s]:
                        repriced += f32_bits(c["cost"]) != f32_bits(cur.srv_cur_cost[s])
        nxt = cur.apply_winners(win)
        for s in range(S):
            if win[s]["feasible"]:
                assert (nxt.srv_cur_acc[s], nxt.srv_cur_replicas[s]) == (win[s]["acc"], win[s]["replicas"])
                assert f32_bits(nxt.srv_cur_cost[s]) == f32_bits(win[s]["cost"])
                carried += 1
            else:
                assert (nxt.srv_cur_acc[s], nxt.srv_cur_replicas[s]) == (cur.srv_cur_acc[s], cur.srv_cur_replicas[s])
                assert f32_bits(nxt.srv_cur_cost[s]) == f32_bits(cur.srv_cur_cost[s])
        cur = nxt
    assert carried >= 20 and repriced >= 5


# ---- GPU: bit for bit against the composition -------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet_warp_path(engine, oracle_mod, keep):
    fleet = profile_fleet(14, 3, 31, keep)
    rows = {**load_rows(fleet, 7, 3), **profile_rows(fleet, 7, 3)}
    cand_o, win_o = check_level_call(engine, oracle_mod, "profile_trace", fleet, rows, f"warp path, keep = {keep}")
    assert cand_o["feasible"].sum() > 40
    assert len(set(win_o["acc"][win_o["feasible"] == 1].tolist())) >= 2


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = profile_fleet(120, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    fleet.accel_penalty_factor = 0.02
    rows = {**load_rows(fleet, 5, 11), **profile_rows(fleet, 5, 11)}
    return fleet, rows, ref_trace(oracle_mod, fleet, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rows, (cand_o, win_o, _) = rounds_case
    cand_g, win_g = engine.profile_trace(fleet, **rows, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"rounds, D = {depth}: candidates")
    assert_allocs_equal(win_g, win_o, f"rounds, D = {depth}: winners")


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("penalty", [0.0, None])
@pytest.mark.parametrize("rounds", [False, True])
def test_hourly_price_rows(engine, oracle_mod, monkeypatch, keep, penalty, rounds):
    """Price rows alone: NaN, +-0, negative, +Inf and MaxFloat32 prices, ties between identical accelerators 1 and
    2, then an hourly curve in which accelerator 0 becomes very cheap and then very dear.  Without keep some winner
    switches accelerator mid-trace, at penalty factor 0 and at the fleet's default; and the chain is not the profile
    grid's, whose every row is solved against c_0."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = profile_fleet(16, 3, 41, keep)
    if penalty is not None:
        fleet.accel_penalty_factor = penalty
    fleet.srv_cur_cost[::5] = np.nan
    for k in PERF:
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]
    base = fleet.acc_cost
    special = [[np.nan, 1.0, 1.0], [0.0, -0.0, -0.0], [-5.0, 2.0, 2.0], [np.inf, 1.0, 1.0], [F32_MAX, F32_MAX, 1.0],
               [1.0, F32_MAX, F32_MAX]]
    hourly = hourly_prices(fleet, 12, 5)
    hourly[3:7, 0] = base[0] * F32(0.01)
    hourly[7:, 0] = base[0] * F32(20.0)
    acc = np.concatenate([hourly[:2], np.array(special, F32), hourly[2:]]).astype(F32)
    rows = {"acc_cost": acc}
    _, win_o = check_level_call(engine, oracle_mod, "profile_trace", fleet, rows, f"price rows, keep = {keep}, penalty = {penalty}")
    S = fleet.n_servers
    _, win_trace = engine.profile_trace(fleet, **rows)
    _, win_grid = engine.profile_grid(fleet, **rows)
    assert any(not same_bytes(getattr(win_trace, k), getattr(win_grid, k)) for k in ALLOC_FIELDS)
    if not keep:
        assert _moves(win_o[(len(special) + 2) * S:], S) >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_price_and_workload_rows(engine, oracle_mod, keep):
    """Price rows with workload rows, rate-0 ticks included: with keep, a min_replicas 0 server is released by its
    zero-load tick and moves; every zero-load record carries its tick's price."""
    fleet = profile_fleet(40, 4, 89, keep)
    fleet.accel_penalty_factor = 0.0
    fleet.srv_min_replicas[:] = 1
    fleet.srv_min_replicas[::2] = 0
    L = 10
    rows = load_rows(fleet, L, 29, special=False)
    rows["arrival_rpm"][3::4, ::3] = 0.0
    rows["acc_cost"] = hourly_prices(fleet, L, 7)
    cand_o, win_o = check_level_call(engine, oracle_mod, "profile_trace", fleet, rows, f"prices and load, keep = {keep}")
    S, A = fleet.n_servers, fleet.n_acc
    c = cand_o.reshape(L, S, A)
    zero = 0
    for t in range(L):
        for s in range(S):
            if rows["arrival_rpm"][t, s] != 0:
                continue
            for a in range(A):
                r = c[t, s, a]
                if r["feasible"] and r["replicas"] > 0:
                    m = fleet.srv_model[s]
                    inst = max(int(fleet.perf_acc_count[m, a]), 1) * int(r["replicas"])
                    assert f32_bits(r["cost"]) == f32_bits(F32(rows["acc_cost"][t, a]) * F32(inst)), (t, s, a)
                    zero += 1
    assert zero >= 10
    assert _moves(win_o, S) >= 3


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_accelerator_switched_on_and_off(engine, oracle_mod, keep):
    """Accelerator 2 is listed without profiles, switched on (and cheap) at tick 2 and off again at tick 5, while
    servers 0..5 sit on it.  With keep (min_replicas 1) they are pinned: nil winners while it is off, and they stay.
    Without keep they move off it at tick 0, onto it while it is cheap and on, and off it again."""
    fleet = profile_fleet(24, 3, 43, keep)
    fleet.accel_penalty_factor = 0.0
    M, A = fleet.n_models, fleet.n_acc
    fleet.perf_present[:, 2] = 0
    sit = np.arange(6)
    fleet.srv_cur_acc[sit] = 2
    fleet.srv_cur_replicas[sit] = 1
    fleet.srv_cur_cost[sit] = fleet.acc_cost[2]
    fleet.srv_min_replicas[sit] = 1
    fleet.srv_arrival_rpm[sit] = np.maximum(fleet.srv_arrival_rpm[sit], F32(30.0))
    fleet.srv_has_target[sit] = 1
    fleet.srv_model[sit] = np.abs(fleet.srv_model[sit])
    L, on, off = 8, 2, 5
    rows = {k: np.repeat(getattr(fleet, k)[None], L, axis=0).copy() for k in PERF}
    rows["acc_cost"] = np.repeat(fleet.acc_cost[None], L, axis=0).copy()
    rows["perf_present"][on:off, :, 2] = 1
    for k in PERF[1:]:
        rows[k][on:off, :, 2] = rows[k][on:off, :, 1]
    rows["acc_cost"][:, 2] = fleet.acc_cost.min() * F32(0.05)
    cand_o, win_o = check_level_call(engine, oracle_mod, "profile_trace", fleet, rows, f"accelerator on and off, keep = {keep}")
    w = win_o.reshape(L, -1)
    if keep:
        assert pinned(fleet)[sit].all()
        for t in range(L):
            if on <= t < off:
                f = w[t, sit]["feasible"] == 1
                assert f.sum() >= 3 and (w[t, sit]["acc"][f] == 2).all(), t
            else:
                assert not w[t, sit]["feasible"].any(), t
    else:
        assert not (w[:on]["acc"][w[:on]["feasible"] == 1] == 2).any()
        assert ((w[on:off]["acc"] == 2) & (w[on:off]["feasible"] == 1)).sum() >= 6
        assert not (w[off:]["acc"][w[off:]["feasible"] == 1] == 2).any()
        assert ((w[0, sit]["feasible"] == 1) & (w[0, sit]["acc"] != 2)).sum() >= 3


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_profile_changes_from_a_tick(engine, oracle_mod, keep):
    """alpha / beta / gamma / delta changes that hold from some tick on, one alpha that makes Size fail at one tick
    only, AccCount 0 and negative, and a perf batch size that moves N where srv_max_batch is 0 and does not where it
    is set; together with workload rows."""
    fleet = profile_fleet(18, 3, 47, keep)
    fleet.srv_slo_tps[::5] = F32(800.0)
    L = 8
    rows = {k: np.repeat(getattr(fleet, k)[None], L, axis=0).copy() for k in PERF}
    rows["perf_beta"][2:, :, 1] *= F32(0.9)
    rows["perf_alpha"][3:] *= F32(0.95)
    rows["perf_gamma"][5:, :, 0] *= F32(1.1)
    rows["perf_delta"][5:, :, 2] *= F32(0.9)
    rows["perf_alpha"][4, :, 0] = F32(1e6)  # ITL targets unreachable on accelerator 0 at tick 4 only
    rows["perf_acc_count"][6:, :, 0] = 0
    rows["perf_acc_count"][6:, :, 1] = -2
    rows["perf_max_batch"][7] = np.maximum(rows["perf_max_batch"][7] // 4, 1)
    rows["perf_at_tokens"][7] *= 3
    rows.update(load_rows(fleet, L, 13, special=False))
    cand_o, _ = check_level_call(engine, oracle_mod, "profile_trace", fleet, rows, f"profile changes, keep = {keep}")
    c = cand_o.reshape(L, fleet.n_servers, fleet.n_acc)
    assert (c[3, :, 0]["feasible"] > c[4, :, 0]["feasible"]).any()
    srv_n = fleet.srv_max_batch == 0
    both = (c[6][srv_n]["feasible"] == 1) & (c[7][srv_n]["feasible"] == 1) & (c[7][srv_n]["rho"] > 0)
    assert (c[7][srv_n]["batch"] != c[6][srv_n]["batch"])[both].any()
    fixed = (~srv_n)[:, None] & (c[7]["feasible"] == 1) & (c[7]["rho"] > 0)
    assert (c[7]["batch"][fixed] == np.broadcast_to(fleet.srv_max_batch[:, None], c[7].shape)[fixed]).all()


@pytest.mark.gpu
def test_stored_vector_fallback_both_phases(engine, oracle_mod):
    """N = 1024 near saturation: the chains overflow float64, so phase 1's solves and the tail's re-run on the
    stored vector, tick after tick; the ticks change the price and move N through out_tokens and the perf batch
    size."""
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
    rows = {"arrival_rpm": rpm, "in_tokens": np.full((L, S), 64, np.int32), "out_tokens": out_tok,
            "acc_cost": (np.arange(1, L + 1, dtype=F32)[:, None] * F32(0.75)).astype(F32),
            "perf_max_batch": np.where(np.arange(L) % 3 == 2, 512, 1024).astype(np.int32)[:, None, None]
            .repeat(fleet.n_models, 1)}
    cand_o, _ = check_level_call(engine, oracle_mod, "profile_trace", fleet, rows, "stored-vector fallback")
    assert cand_o["feasible"].sum() >= L


# ---- GPU: equivalences ------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_without_profile_rows_is_the_workload_trace(engine, monkeypatch, rounds):
    """Every profile column NULL: wva_workload_trace's bytes and launch count (the same keys, sized the same way)."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = profile_fleet(30, 4, 61, True)
    fleet.accel_penalty_factor = 0.01
    rows = load_rows(fleet, 6, 19)
    n0 = engine.launch_count
    got = engine.profile_trace(fleet, **rows, want_candidates=True)
    n1 = engine.launch_count
    want = engine.workload_trace(fleet, **rows, want_candidates=True)
    n2 = engine.launch_count
    for g, w in zip(got, want):
        _bytes_equal(g, w, "profile trace without profile rows")
    assert n1 - n0 == n2 - n1


@pytest.mark.gpu
def test_model_without_profiles(engine, oracle_mod):
    """Model 0 has no profile at any accelerator, and model 1's MaxBatchSize * AtTokens is 2^22.  Server 0, on model
    0 without keep, is loaded with out_tokens 1: it has no candidate at any tick, and nothing may size it on model 1's
    rows (N = 2^22 would be refused).  Without a perf column the call is wva_workload_trace, bytes and launches; with
    one it is the per-tick composition."""
    fleet = synth_fleet(4, 2, seed=83, n_models=2, zero_load_frac=0.0)
    fleet.srv_model[:] = [0, 1, 1, 1]
    fleet.perf_present[0] = 0
    fleet.perf_present[1] = 1
    fleet.perf_max_batch[1] = 1024
    fleet.perf_at_tokens[1] = 4096
    fleet.srv_max_batch[:] = [0, 8, 16, 8]
    fleet.srv_out_tokens[0] = 1
    fleet.srv_keep_acc[:] = 0
    fleet.srv_has_target[:] = 1
    fleet.srv_arrival_rpm[:] = np.maximum(fleet.srv_arrival_rpm, F32(30.0))
    L = 3
    load = {k: np.repeat(getattr(fleet, c)[None], L, axis=0).copy() for k, c in LOAD_COLUMN.items()}
    load["arrival_rpm"][1] *= F32(2.0)
    n0 = engine.launch_count
    got = engine.profile_trace(fleet, **load, want_candidates=True)
    n1 = engine.launch_count
    want = engine.workload_trace(fleet, *load.values(), want_candidates=True)
    n2 = engine.launch_count
    for g, w in zip(got, want):
        _bytes_equal(g, w, "no perf column")
    assert n1 - n0 == n2 - n1
    cand_o, win_o = check_level_call(engine, oracle_mod, "profile_trace", fleet, {**load, "acc_cost": hourly_prices(fleet, L, 5)}, "prices")
    assert not cand_o.reshape(L, 4, 2)[:, 0]["feasible"].any() and win_o["feasible"].sum() >= 2 * L
    beta = np.repeat(fleet.perf_beta[None], L, axis=0).copy()
    beta[1:] *= F32(1.1)
    check_level_call(engine, oracle_mod, "profile_trace", fleet, {**load, "perf_beta": beta}, "perf rows")


@pytest.mark.gpu
def test_one_tick_is_the_profile_grid(engine):
    """L = 1 and the workload lists NULL: wva_profile_grid's bytes for that row."""
    fleet = profile_fleet(30, 4, 59, True)
    rows = profile_rows(fleet, 5, 13)
    for l in range(5):
        one = {k: v[l:l + 1] for k, v in rows.items()}
        for g, w in zip(engine.profile_trace(fleet, **one, want_candidates=True),
                        engine.profile_grid(fleet, **one, want_candidates=True)):
            _bytes_equal(g, w, f"row {l}")


@pytest.mark.gpu
def test_each_tick_is_solve_on_the_advanced_fleet(engine):
    fleet = profile_fleet(30, 4, 67, True)
    fleet.accel_penalty_factor = 0.01
    L = 6
    rows = {**load_rows(fleet, L, 19), **profile_rows(fleet, L, 21)}
    cand_g, win_g = engine.profile_trace(fleet, **rows, want_candidates=True)
    S, A = fleet.n_servers, fleet.n_acc
    cur = fleet
    for t in range(L):
        cand_s, win_s = engine.solve(at_row(cur, rows, t))
        for k in ALLOC_FIELDS:
            assert same_bytes(getattr(cand_g, k)[t * S * A:(t + 1) * S * A], getattr(cand_s, k)), (t, k)
            assert same_bytes(getattr(win_g, k)[t * S:(t + 1) * S], getattr(win_s, k)), (t, k)
        cur = cur.apply_winners(win_s)


CONTINUATION_L = {1: 7, 3: 7, 5: 7, 32: 70, 33: 70, 65: 100}  # the trace length per split tick k


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3, 5, 32, 33, 65])
def test_continuation(engine, k):
    """The trace over [0, L) is the trace over [0, k) followed by the trace over [k, L) from c_k."""
    fleet = profile_fleet(30, 3, 103, True)
    fleet.accel_penalty_factor = 0.0
    fleet.srv_min_replicas[:] = 1
    fleet.srv_min_replicas[::2] = 0
    L = CONTINUATION_L[k]
    rows = {**load_rows(fleet, L, 37), **profile_rows(fleet, L, 39)}
    rows["arrival_rpm"][2, ::3] = 0.0
    S = fleet.n_servers
    cand, win = engine.profile_trace(fleet, **rows, want_candidates=True)
    cand_a, win_a = engine.profile_trace(fleet, **{n: r[:k] for n, r in rows.items()}, want_candidates=True)
    cur = fleet
    for t in range(k):
        cur = cur.apply_winners(_records(win_a)[t * S:(t + 1) * S])
    cand_b, win_b = engine.profile_trace(cur, **{n: r[k:] for n, r in rows.items()}, want_candidates=True)
    for n in ALLOC_FIELDS:
        assert same_bytes(getattr(cand, n), np.concatenate([getattr(cand_a, n), getattr(cand_b, n)])), n
        assert same_bytes(getattr(win, n), np.concatenate([getattr(win_a, n), getattr(win_b, n)])), n
    assert _moves(_records(win), S) >= 1


# ---- GPU: refusals, arguments and the handle ---------------------------------------------------------

@pytest.mark.gpu
def test_batch_size_refusal_and_the_pinned_pair(engine):
    """N = MaxBatchSize * AtTokens / out_tokens: a row with MaxBatchSize 2^16 puts server 0's N on accelerator 0
    at 2^21 at tick 1.  The trace refuses as that tick's wva_analyze does.  With server 0 pinned to accelerator 1
    the pair is excluded at every tick, so the per-tick loop never sizes it, and neither does the trace."""
    fleet = synth_fleet(4, 2, seed=83, zero_load_frac=0.0)
    fleet.srv_max_batch[0] = 0
    fleet.perf_at_tokens[:] = 1 << 12
    fleet.perf_max_batch[:] = 512
    fleet.srv_out_tokens[:] = 1 << 7
    m0 = int(fleet.srv_model[0])
    L = 3
    mb = np.repeat(fleet.perf_max_batch[None], L, axis=0).copy()
    mb[1, m0, 0] = 1 << 16
    rows = {"perf_max_batch": mb, "acc_cost": hourly_prices(fleet, L, 3)}
    code = error_code(lambda: engine.analyze(at_row(fleet, rows, 1)))[0]
    assert code == WVA_ERR_UNSUPPORTED
    assert error_code(lambda: engine.profile_trace(fleet, **rows))[0] == code
    assert error_code(lambda: engine.profile_trace(fleet, **{k: v[[0, 2]] for k, v in rows.items()}))[0] == 0
    pin = fleet.take_servers(np.arange(fleet.n_servers))
    pin.srv_keep_acc[0] = 1
    pin.srv_cur_acc[0] = 1
    pin.srv_cur_replicas[0] = 1
    pin.srv_min_replicas[0] = 1
    assert pinned(pin)[0]
    cand_g, win_g = engine.profile_trace(pin, **rows, want_candidates=True)
    S, A = pin.n_servers, pin.n_acc
    cur = pin
    for t in range(L):
        cand_s, win_s = engine.solve(at_row(cur, rows, t))
        for k in ALLOC_FIELDS:
            assert same_bytes(getattr(cand_g, k)[t * S * A:(t + 1) * S * A], getattr(cand_s, k)), (t, k)
            assert same_bytes(getattr(win_g, k)[t * S:(t + 1) * S], getattr(win_s, k)), (t, k)
        cur = cur.apply_winners(win_s)
    assert (win_g.acc[0::S][win_g.feasible[0::S] == 1] == 1).all()


@pytest.mark.gpu
def test_argument_errors(engine):
    from workload_variant_autoscaler_b200 import _abi
    fleet = profile_fleet(6, 2, 79, False)
    L, h = engine._L, engine._h
    win = Allocs(fleet.n_servers)
    fc, wc = fleet.as_c(), win.as_c()
    cost = np.ascontiguousarray(fleet.acc_cost[None])
    rows = _abi.ProfileRowsC(_abi.ptr(cost), *[None] * 8)
    assert L.wva_profile_trace(h, C.byref(fc), -1, None, None, None, C.byref(rows), None, C.byref(wc)) == \
        WVA_ERR_BAD_ARG
    assert L.wva_profile_trace(h, None, 1, None, None, None, C.byref(rows), None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_profile_trace(h, C.byref(fc), 1, None, None, None, C.byref(rows), None, None) == WVA_ERR_BAD_ARG
    # every list NULL: the fleet's own columns at every tick, i.e. wva_workload_trace on the fleet's own load
    win3 = Allocs(3 * fleet.n_servers)
    assert L.wva_profile_trace(h, C.byref(fc), 3, None, None, None, None, None, C.byref(win3.as_c())) == 0
    own = [np.repeat(getattr(fleet, c)[None], 3, axis=0) for c in LOAD_COLUMN.values()]
    _bytes_equal(win3, engine.workload_trace(fleet, *own)[1], "every list NULL")
    # S * A * L = 2^20 * 2^6 * 32 = 2^31, and L * M * A = 2^25 * 2^6 = 2^31: refused before the fleet is read
    big = fleet.as_c()
    big.n_servers, big.n_acc, big.n_types = 1 << 20, 1 << 6, 0
    assert L.wva_profile_trace(h, C.byref(big), 32, None, None, None, C.byref(rows), None, C.byref(wc)) == \
        WVA_ERR_UNSUPPORTED
    big = fleet.as_c()
    big.n_servers, big.n_models, big.n_acc, big.n_types = 1, 1 << 25, 1 << 6, 0
    assert L.wva_profile_trace(h, C.byref(big), 1, None, None, None, C.byref(rows), None, C.byref(wc)) == \
        WVA_ERR_UNSUPPORTED
    with pytest.raises(ValueError):
        engine.profile_trace(fleet)
    with pytest.raises(ValueError):
        engine.profile_trace(fleet, acc_cost=fleet.acc_cost)
    with pytest.raises(ValueError):
        engine.profile_trace(fleet, fleet.srv_arrival_rpm[None], acc_cost=np.repeat(cost, 2, axis=0))
    with pytest.raises(ValueError):
        engine.profile_trace(fleet, out_tokens=fleet.srv_out_tokens[None, :1])
    with pytest.raises(ValueError):
        engine.profile_trace(fleet, acc_cost=cost, out=Allocs(2 * fleet.n_servers))
    # an empty list is valid, and the handle then solves as usual
    cand, win0 = engine.profile_trace(fleet, acc_cost=np.zeros((0, fleet.n_acc), F32), want_candidates=True)
    assert cand.n == 0 and win0.n == 0
    engine.solve(fleet)


@pytest.mark.gpu
def test_one_handle_with_the_other_paths(engine):
    fleet = profile_fleet(30, 3, 73, True)
    rows = {**load_rows(fleet, 4, 23), **profile_rows(fleet, 4, 25)}
    fresh = Engine(0)
    try:
        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if x is not None:
                    _bytes_equal(x, y, what)

        trace = lambda e: e.profile_trace(fleet, **rows, want_candidates=True)  # noqa: E731
        grid = lambda e: e.profile_grid(fleet, **{k: v for k, v in rows.items() if k in COLUMNS})  # noqa: E731
        # wva_solve -> wva_profile_trace -> wva_resolve: the resident fleet and the solve's cache are untouched
        cand_s, win_s = engine.solve(fleet)
        trace(engine)
        cand_r, win_r = engine.resolve(want_candidates=True)
        _bytes_equal(cand_r, cand_s, "resolve after the trace: candidates")
        _bytes_equal(win_r, win_s, "resolve after the trace: winners")
        check(trace, "trace")
        check(grid, "profile grid after the trace")
        check(trace, "trace after the profile grid")
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
def test_profile_trace_adversarial(engine, oracle_mod, monkeypatch):
    """Fleets from levels._adversarial_fleet, keep on half the servers, with random load rows from the
    workload grid's edge sets and random profile rows from the profile grid's, half of them on the rounds.  Where
    the per-tick wva_solve loop refuses a tick, the trace must refuse too; it may refuse beyond that only through a
    keep server that is not pinned."""
    rng = np.random.default_rng(0x9A7E)
    feasible = refused = extra = 0
    for case in range(N_ADV):
        fleet = _adversarial_fleet(rng, 70000 + case)
        S, M, A, L = fleet.n_servers, fleet.n_models, fleet.n_acc, int(rng.integers(1, 6))
        fleet.srv_keep_acc[:] = rng.random(S) < 0.5
        fleet.srv_cur_acc[:] = rng.integers(-2, A, S)
        fleet.accel_penalty_factor = float(rng.choice([0.0, 0.1]))
        if case % 2:
            monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        else:
            monkeypatch.delenv("WVA_SIZE_SMALL_MAX", raising=False)
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
        rows["arrival_rpm"] = rng.choice(np.array([0.0, 1e-3, 3.0, 600.0, 1e6, -1.0, np.inf], F32), (L, S),
                                         p=[.15, .1, .25, .25, .1, .05, .1])
        rows["in_tokens"] = rng.choice(np.array([0, 1, 7, 512, 100000, -1], np.int32), (L, S),
                                       p=[.15, .15, .2, .25, .2, .05])
        rows["out_tokens"] = rng.choice(np.array([0, 1, 2, 9, 300, 50000, -1], np.int32), (L, S),
                                        p=[.1, .1, .15, .15, .25, .2, .05])
        for k in rows:
            rows[k][0] = getattr(fleet, LOAD_COLUMN.get(k, k))
        # the per-tick wva_solve loop
        code, cur = 0, fleet
        for t in range(L):
            code, res = error_code(lambda: engine.solve(at_row(cur, rows, t)))
            if code:
                break
            cur = cur.apply_winners(res[1])
        got, _ = error_code(lambda: engine.profile_trace(fleet, **rows))
        if code:
            assert got == code, (case, code, got)
            refused += 1
            continue
        if got:
            assert got == WVA_ERR_UNSUPPORTED and ((fleet.srv_keep_acc != 0) & ~pinned(fleet)).any(), (case, got)
            extra += 1
            continue
        _, win_o = check_level_call(engine, oracle_mod, "profile_trace", fleet, rows, f"adversarial case {case}")
        feasible += int(win_o["feasible"].sum())
    assert feasible > 30 and refused + extra < N_ADV // 2
