"""wva_slo_margins and wva_slo_margin_trace: the load margins (grid and trace) at rows that carry their own ITL, TTFT
and TPS targets, as well as their own load and tokens.

The expected margins come from slo_margin_levels.ref_slo_margins: per row, levels.ref_margins with one level on the
fleet with the row's rate, tokens and targets, on a trace also with the c_t that apply_winners of each tick's `at`
carries.  The GPU tests compare the CUDA path with it bit for bit, and without the oracle with wva_load_margins on the
row's fleet, with the SLO grid and trace, and with the workload margins."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (F32, SLO, _moves, at_row, below, day_rows, day_slo_rows, mixed_fleet, overflow_fleet,
                          pinned, rates_at_rate_star, ref_grid, ref_slo_bounds, ref_trace, token_fleet)
from tests.profile_margin_levels import scale_to_rows
from tests.slo_margin_levels import (CALLS, KINDS, check_slo_margins, own_targets, ref_slo_margins, run,
                                     slo_margin_case, split)
from tests.util import (ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, error_code,
                        same_bytes)
from tests.workload_margin_levels import (CALLS as WORKLOAD_CALLS, assert_same, block, part, ref_workload_margins,
                                          unpinned_case)
from workload_variant_autoscaler_b200 import (MARGIN_HI_OPEN, MARGIN_LO_OPEN, MARGIN_TRUNCATED, Allocs, Engine,
                                              WvaError, synth_fleet, _lib)

TRACES = [False, True]


def same_records(x, y, fields=ALLOC_FIELDS):
    return all(same_bytes(x[k], y[k]) for k in fields)


def unpinned_slo_case():
    """workload_margin_levels.unpinned_case with the ITL target x 0.5 .. x 2 per tick and TTFT x 1.5 from tick 3 on."""
    fleet, rows, lo, hi = unpinned_case()
    L = rows["arrival_rpm"].shape[0]
    rng = np.random.default_rng(31)
    own = own_targets(fleet, L)
    rows["slo_itl"] = (own["slo_itl"] * rng.choice(np.array([0.5, 0.75, 1.0, 2.0], F32), (L, 1))).astype(F32)
    rows["slo_ttft"] = own["slo_ttft"]
    rows["slo_ttft"][3:] *= F32(1.5)
    return fleet, rows, lo, hi


# ---- CPU: the composition ---------------------------------------------------------------------

@pytest.mark.parametrize("trace", TRACES)
@pytest.mark.parametrize("kind", ["schedule", "mixed"])
def test_composition_at_blocks_are_the_slo_winners(oracle_mod, kind, trace):
    fleet = token_fleet(12, 3, 5, trace)
    rows, lo, hi = slo_margin_case(oracle_mod, fleet, 5, kind, 7)
    ref = ref_slo_margins(oracle_mod, fleet, rows, lo, hi, trace)
    win = (ref_trace if trace else ref_grid)(oracle_mod, fleet, rows)[1]
    assert same_records(ref[3], win)


@pytest.mark.parametrize("trace", TRACES)
def test_composition_without_target_lists_is_the_workload_margins(oracle_mod, trace):
    fleet = token_fleet(12, 3, 5, False)
    rows, lo, hi = slo_margin_case(oracle_mod, fleet, 4, "mixed", 9)
    load, _ = split(rows)
    ref = ref_slo_margins(oracle_mod, fleet, {**load, "slo_itl": None, "slo_ttft": None, "slo_tps": None}, lo, hi,
                          trace)
    want = ref_workload_margins(oracle_mod, fleet, load, lo, hi, trace)
    for k in range(3):
        assert same_bytes(ref[k], want[k]), k
    for k in range(3, 6):
        assert same_records(ref[k], want[k]), k


def test_composition_reads_the_itl_rows(oracle_mod):
    """On ITL rows at least two rows' stretch or record differs from the margins at the fleet's own targets."""
    fleet = token_fleet(12, 3, 5, False)
    rows, lo, hi = slo_margin_case(oracle_mod, fleet, 5, "itl", 7)
    ref = ref_slo_margins(oracle_mod, fleet, rows, lo, hi, False)
    fixed = ref_workload_margins(oracle_mod, fleet, split(rows)[0], lo, hi, False)
    S = fleet.n_servers
    differs = [not same_bytes(ref[0][l], fixed[0][l]) or not same_bytes(ref[1][l], fixed[1][l])
               or not same_records(ref[3].reshape(-1, S)[l], fixed[3].reshape(-1, S)[l]) for l in range(5)]
    assert sum(differs) >= 2, differs


def test_composition_negative_target_rows_have_nil_load_records(oracle_mod):
    """A negative target makes every load pair of the row nil (TargetPerf.check), whatever the rate."""
    fleet = token_fleet(12, 3, 5, False)
    fleet.srv_min_replicas[:] = np.maximum(fleet.srv_min_replicas, 1)
    rows, lo, hi = slo_margin_case(oracle_mod, fleet, 3, "mixed", 11, tokens=False)
    rows["slo_itl"][1] = -1.0
    ref = ref_slo_margins(oracle_mod, fleet, rows, lo, hi, False)
    at = ref[3].reshape(3, -1)
    load = rows["arrival_rpm"][1] > 0
    assert load.sum() >= 6
    assert (at[1]["feasible"][load] == 0).all()
    assert (at[0]["feasible"][load] == 1).sum() >= 3


def test_unpinned_case_is_reached_with_targets_moving(oracle_mod):
    fleet, rows, lo, hi = unpinned_slo_case()
    assert not pinned(fleet).any()
    tr = ref_slo_margins(oracle_mod, fleet, rows, lo, hi, True)
    at = tr[3].reshape(-1, fleet.n_servers)
    assert (at[0]["acc"] == -1).all() and ((at[1]["acc"] != fleet.srv_cur_acc) & (at[1]["feasible"] == 1)).any()


def test_the_calls_are_exported():
    assert {"wva_slo_margins", "wva_slo_margin_trace"} <= set(_lib.EXPORTS)


# ---- GPU: bit for bit against the composition ---------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("fleet_kind", ["token", "mixed"])
@pytest.mark.parametrize("kind", KINDS)
def test_small_fleets(engine, oracle_mod, kind, fleet_kind, keep, trace):
    fleet = (token_fleet if fleet_kind == "token" else mixed_fleet)(14, 3, 31, keep)
    rows, lo, hi = slo_margin_case(oracle_mod, fleet, 5, kind, 7)
    check_slo_margins(engine, oracle_mod, fleet, rows, lo, hi, trace,
                      f"{kind} on {fleet_kind}, keep = {keep}, trace = {trace}")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_tps_rows_and_current_costs(engine, oracle_mod, trace):
    """TPS rows, and a NaN and a MaxFloat32 current cost, under ITL and TPS rows."""
    fleet = token_fleet(12, 3, 17, False)
    fleet.srv_cur_cost[5] = np.nan
    fleet.srv_cur_cost[6] = F32_MAX
    fleet.accel_penalty_factor = 0.0
    for kind in ("tps", "itl"):
        rows, lo, hi = slo_margin_case(oracle_mod, fleet, 4, kind, 19)
        check_slo_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"TPS / costs, {kind}, {trace}")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
@pytest.mark.parametrize("which", [0, 1])
def test_targets_at_the_nil_bound_and_below_it(engine, oracle_mod, which, trace):
    """Per server, row 0 puts the TTFT (which = 0) or ITL (1) target at wva_slo_bounds' b1 of its first
    accelerator, where the candidate turns nil, and row 1 at the float below it; rows 2 and 3 repeat them at 1.5 times
    the load."""
    fleet = token_fleet(12, 3, 37, False)
    fleet.srv_slo_tps[:] = 0
    kind, _, _, b1, _ = ref_slo_bounds(oracle_mod, fleet)
    col = ("slo_ttft", "slo_itl")[which]
    own = own_targets(fleet, 4)
    t = own[col]
    S = fleet.n_servers
    ok = np.zeros(S, bool)
    for s in range(S):
        for a in range(fleet.n_acc):
            b = F32(b1[s, a, which])
            if kind[s, a, which] in (2, 3) and np.isfinite(b) and b > 0:
                t[0, s] = t[2, s] = b
                t[1, s] = t[3, s] = below(b)
                ok[s] = True
                break
    assert ok.sum() >= 4
    rows = {col: t}
    rows["in_tokens"] = rows["out_tokens"] = None
    x = np.maximum(fleet.srv_arrival_rpm, 1.0).astype(np.float32)
    rate = (np.stack([x] * 4) * np.array([[1], [1], [1.5], [1.5]])).astype(np.float32)
    rows["arrival_rpm"] = scale_to_rows(oracle_mod, fleet, rows, rate)
    lo, hi = (rows["arrival_rpm"] * F32(0.5)).astype(np.float32), (rows["arrival_rpm"] * F32(2)).astype(np.float32)
    check_slo_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"b1 of search {which}, {trace}")


@pytest.mark.gpu
def test_unpinned_server_lifts_its_mask(engine, oracle_mod):
    fleet, rows, lo, hi = unpinned_slo_case()
    ref = check_slo_margins(engine, oracle_mod, fleet, rows, lo, hi, True, "unpinned")
    assert _moves(ref[3], fleet.n_servers) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_rate_zero_rows_between_target_rows(engine, oracle_mod, trace):
    fleet = token_fleet(12, 3, 13, True)
    fleet.srv_min_replicas[:] = np.maximum(fleet.srv_min_replicas, 1)
    rows, lo, hi = slo_margin_case(oracle_mod, fleet, 6, "mixed", 13)
    for t in (1, 3):
        rows["arrival_rpm"][t] = 0
        lo[t] = 0
        hi[t] = np.where(np.arange(fleet.n_servers) % 2, rows["arrival_rpm"][t + 1] * F32(2), 0).astype(np.float32)
    lo[4, ::3] = 0  # a window bottom of 0 crossed on the way down
    _, _, flags, *_ = check_slo_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"zero rows, {trace}")
    assert (flags[1] & MARGIN_LO_OPEN).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n_acc", [32, 33])
def test_many_accelerators(engine, oracle_mod, n_acc):
    fleet = token_fleet(6, n_acc, 43, False)
    fleet.accel_penalty_factor = 0.0
    rows, lo, hi = slo_margin_case(oracle_mod, fleet, 4, "mixed", 13)
    for trace in TRACES:
        check_slo_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"A = {n_acc}, trace = {trace}")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_stored_vector_fallback_at_each_record(engine, oracle_mod, trace):
    """N = 1024 near saturation: rows 0 .. 2 put totalRate / replicas at rateStar as r, below lo and at hi at the
    fleet's own targets, given as lists; row 3 tightens the ITL target."""
    fleet = overflow_fleet()
    fleet.perf_max_batch[:] = 1024
    fleet.perf_at_tokens[:] = 64
    fleet.srv_max_batch[:] = 0
    fleet.srv_out_tokens[:] = 64
    rates = np.array(rates_at_rate_star(oracle_mod, fleet, 0, 0), np.float32)
    fleet = fleet.take_servers(np.zeros(len(rates), np.int64))
    up = np.array([np.nextafter(r, F32(np.inf)) for r in rates], np.float32)
    rate = np.stack([rates, up, below(rates), rates])
    lo = np.stack([rates, rates, np.zeros_like(rates), rates * F32(0.5)]).astype(np.float32)
    hi = np.stack([rates, up, rates, rates * F32(2)]).astype(np.float32)
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": None, **own_targets(fleet, 4)}
    rows["slo_itl"][3] *= F32(0.75)
    check_slo_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, "stored-vector fallback")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_replica_overflow_truncates_at_an_itl_row(engine, oracle_mod, trace):
    """Rates far above a pair's INT32_MAX-replica point truncate the stretch, at ITL rows."""
    fleet = synth_fleet(3, 2, seed=5, tps_frac=0.0, zero_load_frac=0.0)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    rate = np.stack([x, x])
    rate[1, 0] = F32(3e38)
    with np.errstate(over="ignore"):
        lo, hi = (rate * F32(0.5)).astype(np.float32), np.minimum(rate * F32(2), F32_MAX).astype(np.float32)
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": None,
            "slo_itl": (own_targets(fleet, 2)["slo_itl"] * np.array([[0.75], [1.5]])).astype(F32)}
    _, _, flags, *_ = check_slo_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, "overflow")
    assert flags[1, 0] & MARGIN_TRUNCATED


# ---- GPU: refusals ------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
@pytest.mark.parametrize("value", [np.nan, np.inf, float(F32_MAX)])
def test_nan_tps_refuses_only_under_a_window(engine, oracle_mod, value, trace):
    """A NaN, +Inf or MaxFloat32 TPS target at row 1 on a min_replicas-0 server: the call refuses exactly where
    wva_load_margins on the row's fleet does (NaN refused) when the row's window top is above 0, and the key is never
    sized where the window is [0, 0]."""
    fleet = mixed_fleet(10, 3, 71, False)
    s = 6
    assert fleet.srv_arrival_rpm[s] > 0 and fleet.srv_min_replicas[s] == 0
    fleet.srv_min_replicas[:s] = np.maximum(fleet.srv_min_replicas[:s], 1)
    fleet.srv_min_replicas[s + 1:] = np.maximum(fleet.srv_min_replicas[s + 1:], 1)
    x = np.maximum(fleet.srv_arrival_rpm, 10.0).astype(np.float32)
    rate = np.stack([x, x])
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    tps = own_targets(fleet, 2)["slo_tps"]
    tps[1, s] = value
    single, _ = error_code(lambda: engine.load_margins(at_row(fleet, {"slo_tps": tps}, 1), rate[1:], lo[1:], hi[1:]))
    got, _ = error_code(lambda: getattr(engine, CALLS[trace])(fleet, rate, None, None, lo, hi, slo_tps=tps))
    assert got == single
    assert single == WVA_ERR_UNSUPPORTED or not np.isnan(value)
    rate[1, s] = lo[1, s] = hi[1, s] = 0
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": None, "slo_tps": tps}
    check_slo_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, "NaN TPS under [0, 0]")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_argument_errors_and_summary(engine, oracle_mod, trace):
    from workload_variant_autoscaler_b200 import _abi
    fleet = token_fleet(6, 2, 61, False)
    fn = getattr(engine._L, "wva_" + CALLS[trace])
    h, S = engine._h, fleet.n_servers
    fc = fleet.as_c()
    rows, lo, hi = slo_margin_case(oracle_mod, fleet, 4, "mixed", 3, tokens=False)
    rate = rows["arrival_rpm"][:2].copy()
    lo, hi = lo[:2].copy(), hi[:2].copy()
    slo = {k: np.ascontiguousarray(rows[k][:2]) for k in SLO}
    lo_o, hi_o, flags = np.zeros(2 * S, np.float32), np.zeros(2 * S, np.float32), np.zeros(2 * S, np.uint8)
    recs = [Allocs(2 * S) for _ in range(3)]

    def call(rate_=rate, lo_=lo, hi_=hi, n=2, flags_=flags, out=True, targets=True):
        oc = _abi.MarginsC(_abi.ptr(lo_o), _abi.ptr(hi_o), _abi.ptr(flags_) if flags_ is not None else None,
                           *(r.as_c() for r in recs))
        p = lambda a: _abi.ptr(np.ascontiguousarray(a, np.float32).reshape(-1)) if a is not None else None  # noqa
        tg = [p(slo[k]) if targets else None for k in SLO]
        return fn(h, C.byref(fc), n, p(rate_), None, None, *tg, p(lo_), p(hi_), C.byref(oc) if out else None)

    assert call() == 0
    assert call(targets=False) == 0
    assert call(n=0) == 0
    assert call(rate_=None, n=0) == 0
    assert call(rate_=None) == WVA_ERR_BAD_ARG
    assert call(out=False) == WVA_ERR_BAD_ARG
    assert call(n=-1) == WVA_ERR_BAD_ARG
    assert call(lo_=None) == WVA_ERR_BAD_ARG
    assert call(flags_=None) == WVA_ERR_BAD_ARG
    for bad in (np.nan, np.inf, -1.0):
        for which in range(3):
            args = [rate.copy(), lo.copy(), hi.copy()]
            args[which][1, 2] = bad
            assert call(*args) == WVA_ERR_BAD_ARG, (bad, which)
    assert call(lo_=(rate + 1).astype(np.float32)) == WVA_ERR_BAD_ARG  # lo > r
    assert call(n=(1 << 31) // (3 * S) + 1) == WVA_ERR_UNSUPPORTED  # refused before the rows are read
    with pytest.raises(ValueError):
        getattr(engine, CALLS[trace])(fleet, None)
    with pytest.raises(ValueError):
        getattr(engine, CALLS[trace])(fleet, rate, slo_itl=slo["slo_itl"][:1])
    engine.solve(fleet)
    engine.summarize(fleet.n_types)
    getattr(engine, CALLS[trace])(fleet, rate, None, None, lo, hi, **slo)
    with pytest.raises(WvaError) as e:
        engine.summarize(fleet.n_types)
    assert e.value.code == WVA_ERR_STATE
    # the default window is [0, 2 * rate] (on servers with min_replicas > 0: a bottom of 0 is refused otherwise)
    fleet = synth_fleet(14, 3, seed=33)
    rate = np.stack([fleet.srv_arrival_rpm, fleet.srv_arrival_rpm * 1.5]).astype(np.float32)
    itl = (np.stack([fleet.srv_slo_itl] * 2) * np.array([[0.75], [1.25]])).astype(F32)
    got = getattr(engine, CALLS[trace])(fleet, rate, slo_itl=itl)
    want = getattr(engine, CALLS[trace])(fleet, rate, None, None, np.zeros_like(rate),
                                         (rate * F32(2)).astype(np.float32), slo_itl=itl)
    assert_same(got, want, "default window")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_no_rows_and_no_servers(engine, trace):
    call = getattr(engine, CALLS[trace])
    fleet = synth_fleet(6, 2, seed=61)
    got = call(fleet, np.zeros((0, 6), np.float32), slo_itl=np.zeros((0, 6), np.float32))
    assert got[0].shape == (0, 6) and got[3].n == 0
    empty = fleet.take_servers(np.zeros(0, np.int64))
    got = call(empty, np.zeros((3, 0), np.float32), slo_tps=np.zeros((3, 0), np.float32))
    assert got[0].shape == (3, 0) and got[3].n == 0


# ---- GPU: against the other calls, without the oracle -------------------------------------------

def big_rows(kind):
    fleet = synth_fleet(1500, 8, seed=42)
    if kind == "24":
        x = np.maximum(fleet.srv_arrival_rpm, 1.0).astype(np.float32)
        rng = np.random.default_rng(5)
        rate = (x[None, :] * rng.lognormal(0, 0.6, (24, x.size))).astype(np.float32)
        out = (fleet.srv_out_tokens[None, :] * rng.choice([0.75, 1.0, 1.5], (24, x.size))).astype(np.int32)
        rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": np.maximum(out, 1), **day_slo_rows(fleet, 24, 24)}
    else:
        rows = {**day_rows(fleet, 288, 288, 3, special=False), **day_slo_rows(fleet, 288, 288)}
    rate = rows["arrival_rpm"]
    return fleet, rows, (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)


@pytest.fixture(scope="module", params=["24", "288"])
def big_case(request):
    return big_rows(request.param)


def slo_trace_of(engine, fleet, rows):
    return engine.slo_trace(fleet, **{k: v for k, v in rows.items()})


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_at_blocks_are_the_slo_winners(engine, big_case, trace):
    fleet, rows, lo, hi = big_case
    got = run(engine, trace, fleet, rows, lo, hi)
    if trace:
        _, win = slo_trace_of(engine, fleet, rows)
        for f in ALLOC_FIELDS:
            assert same_bytes(getattr(got[3], f), getattr(win, f)), f
    else:
        S = fleet.n_servers
        for t in range(0, rows["arrival_rpm"].shape[0], 5):
            _, win = slo_trace_of(engine, fleet, {k: None if v is None else v[t:t + 1] for k, v in rows.items()})
            for f in ALLOC_FIELDS:
                assert same_bytes(getattr(part(got[3], t, S), f), getattr(win, f)), (t, f)


@pytest.mark.gpu
def test_at_blocks_at_the_fleets_own_load_are_the_slo_grid(engine, big_case):
    fleet, rows, lo, hi = big_case
    L, S = lo.shape
    slo = split(rows)[1]
    rate = np.ascontiguousarray(np.broadcast_to(fleet.srv_arrival_rpm, (L, S)), np.float32)
    got = engine.slo_margins(fleet, rate, None, None, (rate * F32(0.5)).astype(np.float32),
                             (rate * F32(2)).astype(np.float32), **slo)
    _, win = engine.slo_grid(fleet, slo["slo_itl"], slo["slo_ttft"], slo["slo_tps"])
    for f in ALLOC_FIELDS:
        assert same_bytes(getattr(got[3], f), getattr(win, f)), f


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_blocks_are_the_load_margins_on_the_rows_fleet(engine, big_case, trace):
    fleet, rows, lo, hi = big_case
    L, S = lo.shape
    got = run(engine, trace, fleet, rows, lo, hi)
    cur = fleet
    step = 1 if L <= 24 else 7
    for t in range(L):
        f = at_row(cur, {k: v for k, v in rows.items() if k != "arrival_rpm"}, t)
        if t % step == 0 or trace:
            one = engine.load_margins(f, rows["arrival_rpm"][t:t + 1], lo[t:t + 1], hi[t:t + 1])
            if t % step == 0:
                assert_same(block(got, t, S), one, f"row {t}")
            if trace:
                cur = cur.apply_winners(one[3])


@pytest.mark.gpu
def test_below_and_above_are_a_one_tick_slo_trace_at_their_rates(engine, big_case):
    fleet, rows, lo, hi = big_case
    L, S = lo.shape
    lo_e, hi_e, flags, _, bel, abv = run(engine, False, fleet, rows, lo, hi)
    for name, rec, rates, skip in (("below", bel, below(lo_e), MARGIN_LO_OPEN | MARGIN_TRUNCATED),
                                   ("above", abv, hi_e, MARGIN_HI_OPEN | MARGIN_TRUNCATED)):
        use = (flags & skip) == 0
        assert use.any(), name
        r = np.where(use, rates, rows["arrival_rpm"]).astype(np.float32)
        for t in range(0, L, max(L // 12, 1)):
            one = {k: None if v is None else v[t:t + 1] for k, v in rows.items()}
            one["arrival_rpm"] = r[t:t + 1]
            _, win = slo_trace_of(engine, fleet, one)
            for f in ALLOC_FIELDS:
                g, w = getattr(part(rec, t, S), f)[use[t]], getattr(win, f)[use[t]]
                assert same_bytes(g, w), f"{name}.{f}, row {t}"


@pytest.mark.gpu
def test_trace_continuation(engine, big_case):
    fleet, rows, lo, hi = big_case
    L, S = lo.shape
    whole = run(engine, True, fleet, rows, lo, hi)
    cut = lambda a, sl: None if a is None else a[sl]  # noqa: E731
    for k in sorted({1, 32, 33, L - 1} & set(range(1, L))):
        head = run(engine, True, fleet, {n: cut(v, slice(None, k)) for n, v in rows.items()}, lo[:k], hi[:k])
        cur = fleet
        for t in range(k):
            cur = cur.apply_winners(part(head[3], t, S))
        tail = run(engine, True, cur, {n: cut(v, slice(k, None)) for n, v in rows.items()}, lo[k:], hi[k:])
        for t in range(L):
            piece = block(head, t, S) if t < k else block(tail, t - k, S)
            assert_same(block(whole, t, S), piece, f"k = {k}, tick {t}")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_null_target_lists_are_the_workload_margin_calls(engine, big_case, trace):
    fleet, rows, lo, hi = big_case
    load = split(rows)[0]
    n0 = engine.launch_count
    got = getattr(engine, CALLS[trace])(fleet, load["arrival_rpm"], load["in_tokens"], load["out_tokens"], lo, hi)
    n1 = engine.launch_count
    want = getattr(engine, WORKLOAD_CALLS[trace])(fleet, load["arrival_rpm"], load["in_tokens"], load["out_tokens"],
                                                  lo, hi)
    assert n1 - n0 == engine.launch_count - n1
    assert_same(got, want, "NULL target lists")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_launch_count_does_not_depend_on_rows(engine, trace):
    """One key set (the same row repeated) launches the same kernels at L = 1 and L = 64."""
    fleet = synth_fleet(40, 4, seed=71, zero_load_frac=0.0)
    rows = day_slo_rows(fleet, 2, 2)

    def launches(L):
        x = np.repeat(np.maximum(fleet.srv_arrival_rpm, 1.0)[None].astype(np.float32), L, 0)
        slo = {k: np.repeat(v[:1], L, 0) for k, v in rows.items()}
        n0 = engine.launch_count
        getattr(engine, CALLS[trace])(fleet, x, **slo)
        return engine.launch_count - n0
    assert launches(1) == launches(64)


@pytest.mark.gpu
def test_calls_interleaved_on_one_handle(engine, oracle_mod):
    fleet = token_fleet(30, 3, 59, False)
    fleet.accel_penalty_factor = 0.0
    rows, lo, hi = slo_margin_case(oracle_mod, fleet, 4, "mixed", 23)
    fresh = Engine(0)
    try:
        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if isinstance(x, Allocs):
                    for k in ALLOC_FIELDS:
                        assert same_bytes(getattr(x, k), getattr(y, k)), f"{what}: {k}"
                elif x is not None:
                    assert same_bytes(x, y), what

        load = split(rows)[0]
        grid = lambda e: run(e, False, fleet, rows, lo, hi)  # noqa: E731
        trace = lambda e: run(e, True, fleet, rows, lo, hi)  # noqa: E731
        workload = lambda e: e.workload_margins(fleet, load["arrival_rpm"], None, load["out_tokens"], lo, hi)  # noqa
        strace = lambda e: e.slo_trace(fleet, **rows, want_candidates=True)  # noqa: E731

        def resolve(e):
            e.upload(fleet)
            e.update_load(arrival_rpm=rows["arrival_rpm"][1])
            return e.resolve(want_candidates=True)

        check(grid, "grid")
        check(trace, "trace after the grid")
        check(strace, "SLO trace after the trace")
        check(grid, "grid after the SLO trace")
        check(workload, "workload margins after the grid")
        check(trace, "trace after the workload margins")
        check(resolve, "resolve after the trace")
        check(grid, "grid after a resolve")
    finally:
        fresh.close()
