"""The traces over long horizons: nil runs that push the price trace's look-back for c_l past one or more 32-tick
ballots, a day of ticks (288 at a 5-minute period, 1,440 at a 1-minute one) and the int32 bound of every level call.

The expected results are the compositions of tests/levels.py (ref_trace, ref_grid, ref_price_rows), computed once
per module in fixtures.  The CPU tests show that the cases bite: the gap rows make exactly the intended nil runs,
two wrong look-backs in price_kernel (stop after one ballot; take the earliest feasible tick of a ballot) would change
the thresholds on them, and the day rows keep the chain moving past tick 32.  The GPU tests compare every trace with
the oracle bit for bit on those rows, and at 256 x 8 x 1,440 with itself: continuation, each block against the
single-fleet call on the advanced fleet, and a grid's repeating days."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (PERF, PriceServer, _moves, _records, at_row, check_level_call,
                          check_price_rows, day_profile_rows, day_rows, day_slo_rows, edge_fleet, gap_mask, gap_rows,
                          last_feasible, mixed_fleet, moving_fleet, pinned, ref_grid, ref_price_rows,
                          ref_trace, token_fleet, wva_fleet)
from tests.util import ACC_UNKNOWN, ALLOC_FIELDS, WVA_ERR_UNSUPPORTED, error_code, same_bytes
from workload_variant_autoscaler_b200 import Allocs, Engine, _abi, synth_fleet

F32 = np.float32
SLO_NAMES = ("slo_itl", "slo_ttft", "slo_tps")


# ---- the gap rows: (server, nil-run length, first nil tick); the tick after the run looks back length + 1 ticks ----

GAPS = [(0, 31, 8),   # look-back 32: the last tick of the first ballot
        (1, 32, 8),   # 33: the latest tick of the second ballot
        (5, 63, 9),   # 64: the earliest tick of the second ballot
        (9, 64, 9),   # 65: the latest tick of the third ballot
        (4, 95, 3),   # 96: the earliest tick of the third ballot
        (8, 32, 1),   # l = 33, whose only feasible winner before is tick 0
        (6, 64, 1)]   # l = 65, likewise
L_GAP = 100
GAP_SEED = 44


def gap_arrays(S=10):
    gaps, start = np.zeros(S, np.int64), np.zeros(S, np.int64)
    for s, g, t in GAPS:
        gaps[s], start[s] = g, t
    return gaps, start


def gap_fleet(factor, keep):
    """moving_fleet (penalty factor 0) or edge_fleet at factor 0.1, min_replicas 1, keepAccelerator on every server
    or none.  Servers 2 (no target), 3 (unknown model) and, under keep, 4 (pinned to an unknown accelerator) have
    no feasible winner at any tick; the gap servers have one before and after their run."""
    f = moving_fleet(43) if factor == 0.0 else edge_fleet(43, keep, factor)
    f.srv_min_replicas[:] = 1
    f.srv_keep_acc[:] = keep
    return f


def gap_servers(fleet):
    """The GAPS entries whose server has a feasible winner at all (not pinned to an unknown accelerator)."""
    dead = pinned(fleet) & (fleet.srv_cur_acc == ACC_UNKNOWN)
    return [(s, g, t) for s, g, t in GAPS if not dead[s]]


def assert_nil_runs(fleet, win, gaps, start, what):
    """On the oracle's winners: infeasible on every tick of each run, feasible at the tick after and before it."""
    w = win.reshape(-1, fleet.n_servers)
    for s, g, t in gap_servers(fleet):
        if not gaps[s]:
            continue
        assert not w["feasible"][t:t + g, s].any(), (what, s)
        assert w["feasible"][t - 1, s] and w["feasible"][t + g, s], (what, s)


CASES = [(0.0, False), (0.0, True), (0.1, False), (0.1, True)]


@pytest.fixture(scope="module")
def gap_cases(oracle_mod):
    """{(factor, keep): (fleet, rows, ref_price_rows over L_GAP ticks)}."""
    gaps, start = gap_arrays()
    out = {}
    for factor, keep in CASES:
        f = gap_fleet(factor, keep)
        rows = gap_rows(f, L_GAP, gaps, start, GAP_SEED)
        out[(factor, keep)] = f, rows, ref_price_rows(oracle_mod, f, rows, True)
    return out


# price_kernel's look-back, and two wrong ones: each maps (t = the last feasible tick before l or -1, l, the server's
# feasible flags per tick) to the tick whose winner is read as c_l (-1: the fleet's own current allocation)
def one_ballot(t, l, feasible):
    return t if t >= 0 and l - t <= 32 else -1


def earliest_in_ballot(t, l, feasible):
    if t < 0:
        return -1
    t0 = l - 1 - 32 * ((l - 1 - t) // 32)  # the latest tick of the ballot that holds t
    return next(u for u in range(max(t0 - 31, 0), t + 1) if feasible[u])


MUTANTS = {"one ballot": one_ballot, "earliest in the ballot": earliest_in_ballot}


def mutant_diffs(oracle_mod, fleet, ref, mutant, l, s):
    """How many of server s's thresholds at tick l change when price_kernel reads c_l from the mutant's tick instead
    of the last feasible winner's (the candidates, and so the other columns' values, stay the trace's); None when
    the mutant reads the same tick."""
    th, _, cand, win, fleets = ref
    S, A = fleet.n_servers, fleet.n_acc
    w = win.reshape(-1, S)
    t = int(last_feasible(win, S)[l, s])
    m = mutant(t, l, w["feasible"][:, s] != 0)
    if m == t:
        return None
    f = fleets[l].take_servers(np.arange(S))
    src = (fleet.srv_cur_acc[s], fleet.srv_cur_replicas[s], fleet.srv_cur_cost[s]) if m < 0 else \
        (w[m, s]["acc"], w[m, s]["replicas"], w[m, s]["cost"])
    f.srv_cur_acc[s], f.srv_cur_replicas[s], f.srv_cur_cost[s] = src
    sp = PriceServer(oracle_mod, f, cand.reshape(-1, S, A)[l], s)
    return sum(int(sp.threshold(a) != th[l, s, a]) for a in range(A))


# ---- CPU: the cases bite -------------------------------------------------------------------------------------

def test_gap_rows_make_the_intended_nil_runs(gap_cases):
    gaps, start = gap_arrays()
    for (factor, keep), (fleet, rows, ref) in gap_cases.items():
        what = f"factor {factor}, keep = {keep}"
        rpm = rows["arrival_rpm"]
        nil = gap_mask(fleet.n_servers, L_GAP, gaps, start)
        assert (rpm[nil] == -1).all() and (rpm[~nil] > 0).all() and np.isfinite(rpm).all(), what
        assert_nil_runs(fleet, ref[3], gaps, start, what)
        assert len(gap_servers(fleet)) == (6 if keep else 7), what
        if not keep:
            # several feasible winners that differ within the first ballot of the runs' look-backs
            w = ref[3].reshape(L_GAP, fleet.n_servers)
            varied = [s for s, _, t in GAPS if len({(int(r["acc"]), int(r["replicas"])) for r in w[:t, s]}) >= 2]
            assert len(varied) >= 3, (what, varied)


def test_price_look_back_mutants_change_the_thresholds(oracle_mod, gap_cases):
    """At the tick after each run: the one-ballot mutant reads the same tick at look-back 32 and the fleet's own c_0
    beyond it; the earliest-tick mutant reads the same tick where the last feasible one opens its ballot (32, 64,
    96) and an earlier one at 33 and 65.  Where they read another tick, the thresholds change: on every such server
    without keep, and on some with keep (a pinned server's one candidate wins at every finite value)."""
    for (factor, keep), (fleet, rows, ref) in gap_cases.items():
        changed = {name: {} for name in MUTANTS}
        for s, g, t in gap_servers(fleet):
            l = t + g
            for name, mutant in MUTANTS.items():
                changed[name][g + 1 if t > 1 else f"l = {l} from tick 0"] = mutant_diffs(oracle_mod, fleet, ref,
                                                                                       mutant, l, s)
        what = f"factor {factor}, keep = {keep}: {changed}"
        one, early = changed["one ballot"], changed["earliest in the ballot"]
        assert one[32] is None and all(early[d] is None for d in (32, 64, 96) if d in early), what
        reads_c0 = [d for d in one if d != 32]
        assert all(one[d] is not None for d in reads_c0), what
        if keep:
            assert sum(one[d] for d in reads_c0) >= 1, what
        else:
            assert all(one[d] >= 1 for d in reads_c0) and sum(one[d] for d in reads_c0) >= 15, what
            assert early[33] >= 1 and early[65] >= 1, what


# ---- CPU: the day rows -----------------------------------------------------------------------------------------

DAY_L, DAY_PERIOD = 288, 96


def day_fleet(n=10, seed=133):
    """token_fleet at penalty factor 0.1 with min_replicas 1: winners move with the daily load, and the penalty
    makes c_t matter, so the trace is not the grid."""
    f = token_fleet(n, 3, seed, False)
    f.srv_min_replicas[:] = 1
    f.accel_penalty_factor = 0.1
    return f


def day_load(fleet):
    return day_rows(fleet, DAY_L, DAY_PERIOD, 135)


@pytest.fixture(scope="module")
def day_cases(oracle_mod):
    """{name: (fleet, rows, reference)} of the four traces over a day of 288 ticks, and of the workload grid."""
    fleet = day_fleet()
    load = day_load(fleet)
    prof = {**load, **day_profile_rows(fleet, DAY_L, DAY_PERIOD, 137)}
    slo = {**load, **day_slo_rows(fleet, DAY_L, DAY_PERIOD)}
    price_fleet = day_fleet(8, 141)
    price_load = day_rows(price_fleet, DAY_L, DAY_PERIOD, 143)
    return {"workload_trace": (fleet, load, ref_trace(oracle_mod, fleet, load)),
            "workload_grid": (fleet, load, ref_grid(oracle_mod, fleet, load)),
            "profile_trace": (fleet, prof, ref_trace(oracle_mod, fleet, prof)),
            "slo_trace": (fleet, slo, ref_trace(oracle_mod, fleet, slo)),
            "price_threshold_trace": (price_fleet, price_load, ref_price_rows(oracle_mod, price_fleet, price_load,
                                                                              True))}


def test_day_rows_repeat_and_carry_the_edge_values():
    fleet = day_fleet()
    rows = {**day_load(fleet), **day_profile_rows(fleet, DAY_L, DAY_PERIOD, 137),
            **day_slo_rows(fleet, DAY_L, DAY_PERIOD)}
    for k, v in rows.items():
        assert v.shape[0] == DAY_L, k
        if k != "perf_beta":  # beta changes once, at L // 2
            assert same_bytes(v[:-DAY_PERIOD], v[DAY_PERIOD:]), k
    rpm, in_tok, out_tok = rows["arrival_rpm"], rows["in_tokens"], rows["out_tokens"]
    for v in (0.0, -1.0, np.inf, F32(1e-3), F32(1e6)):
        assert (rpm == v).any(), v
    assert {-1, 0, 100000} <= set(in_tok.ravel().tolist()) and {-1, 0, 1, 20000} <= set(out_tok.ravel().tolist())
    assert (rows["perf_present"][:, :, fleet.n_acc - 1] == 0).any() and (rows["perf_beta"][-1] != fleet.perf_beta).any()
    assert (rows["slo_itl"] != fleet.srv_slo_itl[None]).any() and (rows["slo_ttft"] != fleet.srv_slo_ttft[None]).any()


def test_day_rows_keep_the_chain_moving(day_cases):
    """Past tick 32 the winners still change accelerator, and the trace is not the grid: c_t matters there."""
    for name in ("workload_trace", "profile_trace", "slo_trace", "price_threshold_trace"):
        fleet, _, ref = day_cases[name]
        S = fleet.n_servers
        win = ref[3] if name == "price_threshold_trace" else ref[1]
        assert _moves(win[33 * S:], S) >= 5, name
    fleet, _, (_, win_t, _) = day_cases["workload_trace"]
    win_g = day_cases["workload_grid"][2][1]
    S = fleet.n_servers
    keys = lambda w: np.stack([w["feasible"], w["acc"], w["replicas"]])[:, 33 * S:]  # noqa: E731
    assert (keys(win_t) != keys(win_g)).any(axis=0).sum() >= 10


# ---- GPU: bit for bit against the oracle ---------------------------------------------------------------------

def _prefix(ref, L, S, A):
    th, above, cand, win, fleets = ref
    return th[:L], above[:L * S * A], cand[:L * S * A], win[:L * S], fleets[:L]


@pytest.mark.gpu
@pytest.mark.parametrize("L", [33, 34, 65, 66, L_GAP])
@pytest.mark.parametrize("factor,keep", CASES)
def test_price_trace_on_gap_rows(engine, oracle_mod, gap_cases, factor, keep, L):
    """L = 34 and 66 end at the ticks that look back to tick 0 across one and two ballots."""
    fleet, rows, ref = gap_cases[(factor, keep)]
    check_price_rows(engine, oracle_mod, fleet, {k: v[:L] for k, v in rows.items()}, True,
                     f"gap rows, factor {factor}, keep = {keep}, L = {L}", _prefix(ref, L, fleet.n_servers, fleet.n_acc))


@pytest.fixture(scope="module")
def gap_level_cases(oracle_mod):
    """The workload, SLO and profile traces on the gap rows of moving_fleet: every other run by rate -1, the others
    by an ITL target of -1 (SLO) or perf_present 0 on every accelerator of the server's model (profile)."""
    fleet = gap_fleet(0.0, False)
    gaps, start = gap_arrays()
    by_rate = np.zeros_like(gaps)
    for s, g, _ in GAPS[::2]:
        by_rate[s] = g
    load = gap_rows(fleet, L_GAP, gaps, start, GAP_SEED)
    mixed = gap_rows(fleet, L_GAP, by_rate, start, GAP_SEED)
    other = gap_mask(fleet.n_servers, L_GAP, gaps - by_rate, start)
    slo = {**mixed, **{k: np.repeat(getattr(fleet, "srv_" + k)[None], L_GAP, 0).astype(F32) for k in SLO_NAMES}}
    slo["slo_itl"][other] = -1.0
    present = np.repeat(fleet.perf_present[None], L_GAP, 0)
    for t, s in zip(*np.nonzero(other)):
        present[t, fleet.srv_model[s], :] = 0
    prof = {**mixed, "perf_present": present}
    return {name: (fleet, rows, ref_trace(oracle_mod, fleet, rows))
            for name, rows in (("workload_trace", load), ("slo_trace", slo), ("profile_trace", prof))}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["workload_trace", "slo_trace", "profile_trace"])
def test_traces_on_gap_rows(engine, oracle_mod, gap_level_cases, name):
    fleet, rows, ref = gap_level_cases[name]
    assert_nil_runs(fleet, ref[1], *gap_arrays(), name)
    check_level_call(engine, oracle_mod, name, fleet, rows, f"{name} on gap rows", ref)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["workload_trace", "profile_trace", "slo_trace", "price_threshold_trace"])
def test_traces_over_a_day(engine, oracle_mod, day_cases, name):
    """288 ticks (a day at a 5-minute period) of rows that repeat every 96 ticks, edge values included."""
    fleet, rows, ref = day_cases[name]
    if name == "price_threshold_trace":
        check_price_rows(engine, oracle_mod, fleet, rows, True, "price trace over a day", ref)
    else:
        check_level_call(engine, oracle_mod, name, fleet, rows, f"{name} over a day", ref)


@pytest.mark.gpu
def test_workload_trace_over_1440_ticks(engine, oracle_mod):
    """A day at a 1-minute period: each key of the tick lists holds 15 ticks."""
    fleet = day_fleet(8, 141)
    rows = day_rows(fleet, 1440, 96, 143)
    _, win = check_level_call(engine, oracle_mod, "workload_trace", fleet, rows, "1,440 ticks")
    assert _moves(win[1000 * fleet.n_servers:], fleet.n_servers) >= 10


@pytest.mark.gpu
def test_wva_configuration_over_a_day(engine, oracle_mod):
    """keepAccelerator and min_replicas 1 on every server, each pinned to a real accelerator."""
    fleet = wva_fleet(10, 3, 145)
    assert pinned(fleet).all()
    check_level_call(engine, oracle_mod, "workload_trace", fleet, day_rows(fleet, DAY_L, DAY_PERIOD, 147),
                     "WVA's configuration over a day")


@pytest.mark.gpu
def test_carried_infinite_cost_survives_a_nil_run(engine):
    """A cost of +Inf carried into c_1 (as in test_gpu_price_levels.test_trace_refuses_a_carried_infinite_cost)
    stays c_t through a 40-tick nil run: the trace is refused at the tick after the run, not before it."""
    fleet = synth_fleet(3, 1, seed=87, zero_load_frac=0.0)
    fleet.acc_cost[0] = np.finfo(F32).max
    fleet.perf_acc_count[:, 0] = 2
    cand = engine.analyze(fleet)
    assert cand.feasible.all()
    fleet.srv_keep_acc[:] = 0
    fleet.srv_cur_acc[:] = 0
    fleet.srv_cur_replicas[:] = cand.replicas
    fleet.srv_cur_cost[:] = 0.0
    rpm = np.repeat(fleet.srv_arrival_rpm[None], 43, axis=0).astype(F32)
    rpm[1:41] = -1.0
    _, win = engine.workload_trace(fleet, rpm)
    assert np.isinf(win.cost[:3]).all() and not win.feasible[3:41 * 3].any()
    call = lambda L: error_code(lambda: engine.price_threshold_trace(fleet, rpm[:L]))[0]  # noqa: E731
    assert call(41) == 0
    assert call(42) == WVA_ERR_UNSUPPORTED
    assert b"tick 41)" in engine._L.wva_last_error(engine._h)
    assert call(43) == WVA_ERR_UNSUPPORTED
    assert b"tick 41)" in engine._L.wva_last_error(engine._h)


# ---- GPU: 256 servers x 8 accelerators x 1,440 ticks, without the oracle ------------------------------------------

BIG_L, BIG_PERIOD = 1440, 96


@pytest.fixture(scope="module")
def scale_case():
    """(fleet, {trace: rows}, ticks right after nil runs of >= 33 ticks): day rows with a nil run (rate -1) of 33 to
    120 ticks on every eighth server, and the profile and SLO traces' own day rows on top."""
    fleet = synth_fleet(256, 8, seed=151)
    S = fleet.n_servers
    rng = np.random.default_rng(153)
    gaps = np.zeros(S, np.int64)
    gaps[::8] = rng.integers(33, 121, gaps[::8].size)
    start = rng.integers(1, BIG_L - 121, S)
    load = day_rows(fleet, BIG_L, BIG_PERIOD, 155)
    load["arrival_rpm"][gap_mask(S, BIG_L, gaps, start)] = -1.0
    rows = {"workload_trace": load, "price_threshold_trace": load,
            "profile_trace": {**load, **day_profile_rows(fleet, BIG_L, BIG_PERIOD, 157)},
            "slo_trace": {**load, **day_slo_rows(fleet, BIG_L, BIG_PERIOD)}}
    after = sorted({int(t) for t in (start + gaps)[gaps > 0]})
    return fleet, rows, after


def _trace(engine, name, fleet, rows, want_candidates=False):
    """{column: output} of one trace call (threshold and above for the price trace, candidates when wanted)."""
    out = getattr(engine, name)(fleet, **rows, want_candidates=want_candidates)
    return {"threshold": out[0], "above": out[1], "candidates": out[2], "winners": out[3]} \
        if name == "price_threshold_trace" else {"candidates": out[0], "winners": out[1]}


def _block(x, t, n):
    """Block t of n records (or floats) per tick, as bytes per column."""
    if isinstance(x, np.ndarray):
        return x.reshape(-1)[t * n:(t + 1) * n].tobytes()
    return tuple(getattr(x, k)[t * n:(t + 1) * n].tobytes() for k in ALLOC_FIELDS)


def _advance(fleet, win, ticks):
    S = fleet.n_servers
    rec = _records(win)
    for t in range(ticks):
        fleet = fleet.apply_winners(rec[t * S:(t + 1) * S])
    return fleet


TRACES = ["workload_trace", "profile_trace", "slo_trace", "price_threshold_trace"]


@pytest.mark.gpu
@pytest.mark.parametrize("name", TRACES)
def test_continuation_at_scale(engine, scale_case, name):
    """The trace over [0, L) is the trace over [0, k) then the trace over [k, L) from the fleet advanced through
    ticks < k, byte for byte, at k = 32, 33 and 720."""
    fleet, rows_of, _ = scale_case
    rows = rows_of[name]
    S, A = fleet.n_servers, fleet.n_acc
    full = _trace(engine, name, fleet, rows)
    for k in (32, 33, 720):
        head = _trace(engine, name, fleet, {n: r[:k] for n, r in rows.items()})
        tail = _trace(engine, name, _advance(fleet, head["winners"], k), {n: r[k:] for n, r in rows.items()})
        for col, x in full.items():
            if x is None:
                continue
            cut = k * (S if col == "winners" else S * A)
            for f in (None,) if isinstance(x, np.ndarray) else ALLOC_FIELDS:
                get = (lambda y: y.reshape(-1)) if f is None else (lambda y: getattr(y, f))  # noqa: E731
                assert same_bytes(get(x)[:cut], get(head[col])), (name, k, col, f)
                assert same_bytes(get(x)[cut:], get(tail[col])), (name, k, col, f)


@pytest.mark.gpu
@pytest.mark.parametrize("name", TRACES)
def test_blocks_are_the_single_call_on_the_advanced_fleet(engine, scale_case, name):
    """At ticks 0, 31, 32, 33 and 1,439 and right after every nil run: each block of the price trace is
    price_thresholds, each block of the other traces is solve, on the fleet advanced through the ticks before."""
    fleet, rows_of, after = scale_case
    rows = rows_of[name]
    S, A = fleet.n_servers, fleet.n_acc
    price = name == "price_threshold_trace"
    got = _trace(engine, name, fleet, rows, want_candidates=not price)
    ticks = sorted({0, 31, 32, 33, BIG_L - 1, *after})
    assert len(after) >= 20
    rec = _records(got["winners"])
    cur = fleet
    for t in range(BIG_L):
        if t in ticks:
            f = at_row(cur, rows, t)
            if price:
                th1, above1 = engine.price_thresholds(f)[:2]
                assert _block(got["threshold"], t, S * A) == th1.tobytes(), (name, t)
                assert _block(got["above"], t, S * A) == _block(above1, 0, S * A), (name, t)
            else:
                cand1, win1 = engine.solve(f)
                assert _block(got["candidates"], t, S * A) == _block(cand1, 0, S * A), (name, t)
                assert _block(got["winners"], t, S) == _block(win1, 0, S), (name, t)
        cur = cur.apply_winners(rec[t * S:(t + 1) * S])


@pytest.mark.gpu
def test_grid_days_repeat(engine, scale_case):
    """workload_grid on rows that repeat every 96 ticks (without the nil runs): blocks l and l + 96 are the same
    bytes."""
    fleet, _, _ = scale_case
    S, A = fleet.n_servers, fleet.n_acc
    rows = day_rows(fleet, BIG_L, BIG_PERIOD, 155)
    cand, win = engine.workload_grid(fleet, **rows, want_candidates=True)
    for x, n in ((cand, S * A), (win, S)):
        for k in ALLOC_FIELDS:
            c = getattr(x, k).reshape(BIG_L, n)
            assert same_bytes(c[:-BIG_PERIOD], c[BIG_PERIOD:]), k
    assert len({_block(win, t, S) for t in range(BIG_PERIOD)}) >= BIG_PERIOD // 2


# ---- GPU: the int32 bound of every level call -------------------------------------------------------------------

LEVEL_CALLS = ["load_grid", "slo_grid", "workload_grid", "profile_grid", "price_threshold_grid", "workload_trace",
               "slo_trace", "profile_trace", "price_threshold_trace"]


def _c_call(engine, name, fleet, n):
    """wva_<name> through the C ABI with n rows but row lists of one row: a refusal reads none of them."""
    S, A = fleet.n_servers, fleet.n_acc
    p = _abi.ptr
    rpm = np.ascontiguousarray(fleet.srv_arrival_rpm, F32)
    tin, tout = (np.ascontiguousarray(x, np.int32) for x in (fleet.srv_in_tokens, fleet.srv_out_tokens))
    slo = [np.ascontiguousarray(getattr(fleet, "srv_" + k), F32) for k in SLO_NAMES]
    prof = _abi.ProfileRowsC(p(np.ascontiguousarray(fleet.acc_cost, F32)), *[None] * len(PERF))
    th = np.zeros(S * A, F32)
    win = Allocs(S)
    fc, wc = fleet.as_c(), win.as_c()
    args = {"load_grid": (p(rpm),), "slo_grid": tuple(p(x) for x in slo), "workload_grid": (p(rpm), p(tin), p(tout)),
            "profile_grid": (C.byref(prof),), "workload_trace": (p(rpm), p(tin), p(tout)),
            "slo_trace": (p(rpm), p(tin), p(tout), *(p(x) for x in slo)),
            "profile_trace": (p(rpm), p(tin), p(tout), C.byref(prof)),
            "price_threshold_grid": (p(rpm), p(tin), p(tout), p(th), None),
            "price_threshold_trace": (p(rpm), p(tin), p(tout), p(th), None)}[name]
    return getattr(engine._L, "wva_" + name)(engine._h, C.byref(fc), n, *args, None, C.byref(wc))


def _normal_call(e, name, fleet):
    rows = {"arrival_rpm": np.repeat(fleet.srv_arrival_rpm[None], 3, 0) * F32(1.5)}
    if name == "slo_grid":
        rows = {k: np.repeat(getattr(fleet, "srv_" + k)[None], 3, 0) * F32(0.9) for k in SLO_NAMES}
    if name == "profile_grid":
        rows = {"acc_cost": np.repeat(fleet.acc_cost[None], 3, 0) * F32(0.8)}
    return getattr(e, name)(fleet, **rows, want_candidates=True)


def _same_results(x, y, what):
    for a, b in zip(x, y):
        if isinstance(a, np.ndarray):
            assert same_bytes(a, b), what
        elif a is not None:
            for k in ALLOC_FIELDS:
                assert same_bytes(getattr(a, k), getattr(b, k)), (what, k)


@pytest.fixture(scope="module")
def fresh_engine(engine):
    e = Engine(0)
    yield e
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", LEVEL_CALLS)
def test_level_calls_refuse_the_int32_bound(engine, fresh_engine, name):
    """n = floor(2^31 / (S * A)) + 1 rows: S * A * n >= 2^31 candidates, refused before any row is read (the row
    lists hold one row).  The handle then returns what a fresh one does."""
    fleet = mixed_fleet(6, 2, 79, False)
    S, A = fleet.n_servers, fleet.n_acc
    n = (1 << 31) // (S * A) + 1
    assert S * A * n >= 1 << 31 and S * A * (n - 1) < 1 << 31
    assert _c_call(engine, name, fleet, n) == WVA_ERR_UNSUPPORTED
    assert b"2^31" in engine._L.wva_last_error(engine._h)
    _same_results(_normal_call(engine, name, fleet), _normal_call(fresh_engine, name, fleet), name)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["profile_grid", "profile_trace"])
def test_profile_calls_refuse_the_row_entry_bound(engine, fresh_engine, name):
    """64 models on 2 servers: L * M * A >= 2^31 row entries while S * A * L < 2^31 candidates."""
    fleet = synth_fleet(2, 2, seed=161, n_models=64)
    S, A, M = fleet.n_servers, fleet.n_acc, fleet.n_models
    n = (1 << 31) // (M * A) + 1
    assert n * M * A >= 1 << 31 and S * A * n < 1 << 31
    assert _c_call(engine, name, fleet, n) == WVA_ERR_UNSUPPORTED
    assert b"row entries" in engine._L.wva_last_error(engine._h)
    _same_results(_normal_call(engine, name, fleet), _normal_call(fresh_engine, name, fleet), name)
