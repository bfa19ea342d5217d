"""wva_profile_margins and wva_profile_margin_trace: the load margins (grid and trace) at rows that carry their own
accelerator costs and performance profiles, as well as their own load and tokens.

The expected margins come from profile_margin_levels.ref_profile_margins: per row, levels.ref_margins with one level
on the fleet with the row's rate, tokens, acc_cost and perf_* columns, on a trace also with the c_t that apply_winners
of each tick's `at` carries.  The GPU tests compare the CUDA path with it bit for bit, and without the oracle with
wva_load_margins on the row's fleet, with the profile grid and trace, and with the workload margins."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (COLUMNS, F32, _moves, at_row, below, day_profile_rows, day_rows, mixed_fleet,
                          overflow_fleet, pinned, profile_fleet, rates_at_rate_star, ref_grid, ref_trace)
from tests.profile_margin_levels import (CALLS, check_profile_margins, own_profile, profile_margin_case,
                                         ref_profile_margins, run, split)
from tests.util import ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, same_bytes
from tests.workload_margin_levels import (CALLS as WORKLOAD_CALLS, assert_same, block, part, ref_workload_margins,
                                          unpinned_case)
from workload_variant_autoscaler_b200 import (MARGIN_HI_OPEN, MARGIN_LO_OPEN, MARGIN_TRUNCATED, Allocs, Engine,
                                              WvaError, synth_fleet, _lib)

TRACES = [False, True]
KINDS = ["prices", "edge_prices", "acc_count", "present", "beta", "batch", "mixed"]


def same_records(x, y, fields=ALLOC_FIELDS):
    return all(same_bytes(x[k], y[k]) for k in fields)


def unpinned_profile_case():
    """workload_margin_levels.unpinned_case with a price row per tick (every price x 0.5 .. x 1.25) and beta x 1.1 from
    tick 3 on."""
    fleet, rows, lo, hi = unpinned_case()
    L = rows["arrival_rpm"].shape[0]
    rng = np.random.default_rng(29)
    own = own_profile(fleet, L)
    rows["acc_cost"] = (own["acc_cost"] * rng.choice([0.5, 0.8, 1.0, 1.25], own["acc_cost"].shape)).astype(F32)
    rows["perf_beta"] = own["perf_beta"]
    rows["perf_beta"][3:] *= F32(1.1)
    return fleet, rows, lo, hi


# ---- CPU: the composition ---------------------------------------------------------------------

@pytest.mark.parametrize("trace", TRACES)
@pytest.mark.parametrize("kind", ["prices", "mixed"])
def test_composition_at_blocks_are_the_profile_winners(oracle_mod, kind, trace):
    fleet = profile_fleet(12, 3, 5, trace)
    rows, lo, hi = profile_margin_case(oracle_mod, fleet, 5, kind, 7)
    ref = ref_profile_margins(oracle_mod, fleet, rows, lo, hi, trace)
    win = (ref_trace if trace else ref_grid)(oracle_mod, fleet, rows)[1]
    assert same_records(ref[3], win)


@pytest.mark.parametrize("trace", TRACES)
def test_composition_without_profile_columns_is_the_workload_margins(oracle_mod, trace):
    fleet = profile_fleet(12, 3, 5, False)
    rows, lo, hi = profile_margin_case(oracle_mod, fleet, 4, "prices", 9)
    load, _ = split(rows)
    ref = ref_profile_margins(oracle_mod, fleet, load, lo, hi, trace)
    want = ref_workload_margins(oracle_mod, fleet, load, lo, hi, trace)
    for k in range(3):
        assert same_bytes(ref[k], want[k]), k
    for k in range(3, 6):
        assert same_records(ref[k], want[k]), k


@pytest.mark.parametrize("kind", ["prices", "beta"])
def test_composition_reads_the_profile_rows(oracle_mod, kind):
    """On profile rows some row's stretch or record differs from the margins at the fleet's own prices and profiles."""
    fleet = profile_fleet(12, 3, 5, False)
    rows, lo, hi = profile_margin_case(oracle_mod, fleet, 5, kind, 7)
    ref = ref_profile_margins(oracle_mod, fleet, rows, lo, hi, False)
    fixed = ref_workload_margins(oracle_mod, fleet, split(rows)[0], lo, hi, False)
    S = fleet.n_servers
    differs = [not same_bytes(ref[0][l], fixed[0][l]) or not same_bytes(ref[1][l], fixed[1][l])
               or not same_records(ref[3].reshape(-1, S)[l], fixed[3].reshape(-1, S)[l]) for l in range(5)]
    assert sum(differs) >= 2, differs


def test_unpinned_case_is_reached_on_profile_rows(oracle_mod):
    fleet, rows, lo, hi = unpinned_profile_case()
    assert not pinned(fleet).any()
    tr = ref_profile_margins(oracle_mod, fleet, rows, lo, hi, True)
    at = tr[3].reshape(-1, fleet.n_servers)
    assert (at[0]["acc"] == -1).all() and ((at[1]["acc"] != fleet.srv_cur_acc) & (at[1]["feasible"] == 1)).any()


def test_the_calls_are_exported():
    assert {"wva_profile_margins", "wva_profile_margin_trace"} <= set(_lib.EXPORTS)


# ---- GPU: bit for bit against the composition ---------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("fleet_kind", ["profile", "mixed"])
@pytest.mark.parametrize("kind", KINDS)
def test_small_fleets(engine, oracle_mod, kind, fleet_kind, keep, trace):
    fleet = (profile_fleet if fleet_kind == "profile" else mixed_fleet)(14, 3, 31, keep)
    rows, lo, hi = profile_margin_case(oracle_mod, fleet, 5, kind, 7)
    check_profile_margins(engine, oracle_mod, fleet, rows, lo, hi, trace,
                          f"{kind} on {fleet_kind}, keep = {keep}, trace = {trace}")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_tps_targets_and_current_costs(engine, oracle_mod, trace):
    """TPS-target servers, and a NaN and a MaxFloat32 current cost, under price and beta rows."""
    fleet = profile_fleet(12, 3, 17, False)
    fleet.srv_slo_tps[:3] = (2e4, 1e5, 5e5)
    fleet.srv_cur_cost[5] = np.nan
    fleet.srv_cur_cost[6] = F32_MAX
    fleet.accel_penalty_factor = 0.0
    for kind in ("prices", "beta"):
        rows, lo, hi = profile_margin_case(oracle_mod, fleet, 4, kind, 19)
        check_profile_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"TPS / costs, {kind}, {trace}")


@pytest.mark.gpu
def test_unpinned_server_lifts_its_mask(engine, oracle_mod):
    fleet, rows, lo, hi = unpinned_profile_case()
    ref = check_profile_margins(engine, oracle_mod, fleet, rows, lo, hi, True, "unpinned")
    assert _moves(ref[3], fleet.n_servers) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_rate_zero_rows_between_profile_rows(engine, oracle_mod, trace):
    fleet = profile_fleet(12, 3, 13, True)
    fleet.srv_min_replicas[:] = np.maximum(fleet.srv_min_replicas, 1)
    rows, lo, hi = profile_margin_case(oracle_mod, fleet, 6, "mixed", 13)
    for t in (1, 3):
        rows["arrival_rpm"][t] = 0
        lo[t] = 0
        hi[t] = np.where(np.arange(fleet.n_servers) % 2, rows["arrival_rpm"][t + 1] * F32(2), 0).astype(np.float32)
    _, _, flags, *_ = check_profile_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"zero rows, {trace}")
    assert (flags[1] & MARGIN_LO_OPEN).all()


@pytest.mark.gpu
@pytest.mark.parametrize("n_acc", [32, 33])
def test_many_accelerators(engine, oracle_mod, n_acc):
    fleet = profile_fleet(6, n_acc, 43, False)
    fleet.accel_penalty_factor = 0.0
    rows, lo, hi = profile_margin_case(oracle_mod, fleet, 4, "mixed", 13)
    for trace in TRACES:
        check_profile_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"A = {n_acc}, trace = {trace}")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_stored_vector_fallback_at_a_perf_row(engine, oracle_mod, trace):
    """The overflow fleet at its own perf data has N = 2048 (perf_max_batch 1024 x perf_at_tokens 64 / out_tokens 32);
    rows 0 .. 2 halve perf_at_tokens, so N = 1024 there, and their rates put totalRate / replicas at rateStar as r,
    below lo and at hi."""
    base = overflow_fleet()
    base.perf_max_batch[:] = 1024
    base.perf_at_tokens[:] = 32
    base.srv_max_batch[:] = 0
    rates = np.array(rates_at_rate_star(oracle_mod, base, 0, 0), np.float32)
    fleet = base.take_servers(np.zeros(len(rates), np.int64))
    fleet.srv_out_tokens[:] = 32
    fleet.perf_at_tokens[:] = 64
    up = np.array([np.nextafter(r, F32(np.inf)) for r in rates], np.float32)
    rate = np.stack([rates, up, below(rates)])
    lo = np.stack([rates, rates, np.zeros_like(rates)])
    hi = np.stack([rates, up, rates])
    at_tok = own_profile(fleet, 3)["perf_at_tokens"]
    at_tok[:] = 32
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": None, "perf_at_tokens": at_tok}
    check_profile_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, "stored-vector fallback")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_replica_overflow_truncates_at_a_price_row(engine, oracle_mod, trace):
    """Rates far above a pair's INT32_MAX-replica point truncate the stretch, at price rows."""
    fleet = synth_fleet(3, 2, seed=5, tps_frac=0.0, zero_load_frac=0.0)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    rate = np.stack([x, x])
    rate[1, 0] = F32(3e38)
    with np.errstate(over="ignore"):
        lo, hi = (rate * F32(0.5)).astype(np.float32), np.minimum(rate * F32(2), F32_MAX).astype(np.float32)
    own = own_profile(fleet, 2)
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": None,
            "acc_cost": (own["acc_cost"] * np.array([[0.5], [1.25]])).astype(F32)}
    _, _, flags, *_ = check_profile_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, "overflow")
    assert flags[1, 0] & MARGIN_TRUNCATED


# ---- GPU: refusals ------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_perf_row_pushing_n_past_the_queue_rule_refuses_only_under_a_window(engine, oracle_mod, trace):
    """N = perf_max_batch * perf_at_tokens / out_tokens: row 1 puts server 0's N at 2^21 (N = 32 at row 0), outside
    the queue-size rule.  Refused, as wva_load_margins on the row's fleet refuses, where the row's window top is above
    0; never sized where the window is [0, 0]."""
    fleet = synth_fleet(4, 2, seed=83, zero_load_frac=0.0)
    fleet.srv_max_batch[0] = 0
    fleet.perf_max_batch[:] = 512
    fleet.perf_at_tokens[:] = 1 << 12
    fleet.srv_out_tokens[0] = 1 << 16
    fleet.srv_min_replicas[:] = np.maximum(fleet.srv_min_replicas, 1)
    x = np.maximum(fleet.srv_arrival_rpm, 10.0).astype(np.float32)
    rate = np.stack([x, x])
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    at_tok = own_profile(fleet, 2)["perf_at_tokens"]
    at_tok[1] = 1 << 28
    f1 = at_row(fleet, {"perf_at_tokens": at_tok}, 1)
    with pytest.raises(WvaError) as single:
        engine.load_margins(f1, rate[1:], lo[1:], hi[1:])
    with pytest.raises(WvaError) as e:
        getattr(engine, CALLS[trace])(fleet, rate, None, None, lo, hi, perf_at_tokens=at_tok)
    assert e.value.code == single.value.code == WVA_ERR_UNSUPPORTED
    rate[1, 0] = lo[1, 0] = hi[1, 0] = 0
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": None, "perf_at_tokens": at_tok}
    check_profile_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, "N past the rule under [0, 0]")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_argument_errors_and_summary(engine, oracle_mod, trace):
    from workload_variant_autoscaler_b200 import _abi
    from workload_variant_autoscaler_b200.engine import _profile_rows_c
    fleet = profile_fleet(6, 2, 61, False)
    fn = getattr(engine._L, "wva_" + CALLS[trace])
    h, S = engine._h, fleet.n_servers
    fc = fleet.as_c()
    rows, lo, hi = profile_margin_case(oracle_mod, fleet, 4, "mixed", 3, tokens=False)
    rate = rows["arrival_rpm"][:2].copy()
    lo, hi = lo[:2].copy(), hi[:2].copy()
    prof = {k: np.ascontiguousarray(v[:2]) for k, v in split(rows)[1].items()}
    prc = _profile_rows_c(prof)
    lo_o, hi_o, flags = np.zeros(2 * S, np.float32), np.zeros(2 * S, np.float32), np.zeros(2 * S, np.uint8)
    recs = [Allocs(2 * S) for _ in range(3)]

    def call(rate_=rate, lo_=lo, hi_=hi, n=2, flags_=flags, out=True, rows_=True):
        oc = _abi.MarginsC(_abi.ptr(lo_o), _abi.ptr(hi_o), _abi.ptr(flags_) if flags_ is not None else None,
                           *(r.as_c() for r in recs))
        p = lambda a: _abi.ptr(np.ascontiguousarray(a, np.float32).reshape(-1)) if a is not None else None  # noqa
        return fn(h, C.byref(fc), n, p(rate_), None, None, C.byref(prc) if rows_ else None, p(lo_), p(hi_),
                  C.byref(oc) if out else None)

    assert call() == 0
    assert call(rows_=False) == 0
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
    big = synth_fleet(2, 64, seed=3, n_models=64)
    bc = big.as_c()
    n_rows = (1 << 31) // (64 * 64) + 1  # L*M*A >= 2^31 with 3*S*L < 2^31, refused before any row is read
    assert fn(h, C.byref(bc), n_rows, None, None, None, None, None, None, C.byref(_abi.MarginsC())) == \
        WVA_ERR_UNSUPPORTED
    with pytest.raises(ValueError):
        getattr(engine, CALLS[trace])(fleet, None)
    with pytest.raises(ValueError):
        getattr(engine, CALLS[trace])(fleet, rate, acc_cost=prof["acc_cost"][:1])
    engine.solve(fleet)
    engine.summarize(fleet.n_types)
    getattr(engine, CALLS[trace])(fleet, rate, None, None, lo, hi, **prof)
    with pytest.raises(WvaError) as e:
        engine.summarize(fleet.n_types)
    assert e.value.code == WVA_ERR_STATE
    # the default window is [0, 2 * rate] (on servers with min_replicas > 0: a bottom of 0 is refused otherwise)
    fleet = synth_fleet(14, 3, seed=33)
    rate = np.stack([fleet.srv_arrival_rpm, fleet.srv_arrival_rpm * 1.5]).astype(np.float32)
    cost = (np.stack([fleet.acc_cost] * 2) * np.array([[0.5], [1.25]])).astype(F32)
    got = getattr(engine, CALLS[trace])(fleet, rate, acc_cost=cost)
    want = getattr(engine, CALLS[trace])(fleet, rate, None, None, np.zeros_like(rate),
                                         (rate * F32(2)).astype(np.float32), acc_cost=cost)
    assert_same(got, want, "default window")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_no_rows_and_no_servers(engine, trace):
    call = getattr(engine, CALLS[trace])
    fleet = synth_fleet(6, 2, seed=61)
    got = call(fleet, np.zeros((0, 6), np.float32), acc_cost=np.zeros((0, 2), np.float32))
    assert got[0].shape == (0, 6) and got[3].n == 0
    empty = fleet.take_servers(np.zeros(0, np.int64))
    got = call(empty, np.zeros((3, 0), np.float32), acc_cost=np.stack([empty.acc_cost] * 3))
    assert got[0].shape == (3, 0) and got[3].n == 0


# ---- GPU: against the other calls, without the oracle -------------------------------------------

def big_rows(kind):
    fleet = synth_fleet(1500, 8, seed=42)
    if kind == "24":
        x = np.maximum(fleet.srv_arrival_rpm, 1.0).astype(np.float32)
        rng = np.random.default_rng(5)
        rate = (x[None, :] * rng.lognormal(0, 0.6, (24, x.size))).astype(np.float32)
        out = (fleet.srv_out_tokens[None, :] * rng.choice([0.75, 1.0, 1.5], (24, x.size))).astype(np.int32)
        rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": np.maximum(out, 1),
                **day_profile_rows(fleet, 24, 24, 5)}
    else:
        rows = {**day_rows(fleet, 288, 288, 3, special=False), **day_profile_rows(fleet, 288, 288, 3)}
    rate = rows["arrival_rpm"]
    return fleet, rows, (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)


@pytest.fixture(scope="module", params=["24", "288"])
def big_case(request):
    return big_rows(request.param)


def prices_only(rows):
    return {k: v for k, v in rows.items() if k not in COLUMNS or k == "acc_cost"}


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_at_blocks_are_the_profile_winners(engine, big_case, trace):
    fleet, rows, lo, hi = big_case
    got = run(engine, trace, fleet, rows, lo, hi)
    if trace:
        _, win = engine.profile_trace(fleet, **rows)
        for f in ALLOC_FIELDS:
            assert same_bytes(getattr(got[3], f), getattr(win, f)), f
    else:
        S = fleet.n_servers
        for t in range(0, rows["arrival_rpm"].shape[0], 5):
            _, win = engine.profile_trace(fleet, **{k: None if v is None else v[t:t + 1] for k, v in rows.items()})
            for f in ALLOC_FIELDS:
                assert same_bytes(getattr(part(got[3], t, S), f), getattr(win, f)), (t, f)


@pytest.mark.gpu
def test_at_blocks_at_the_fleets_own_load_are_the_profile_grid(engine, big_case):
    fleet, rows, lo, hi = big_case
    L, S = lo.shape
    prof = split(rows)[1]
    rate = np.ascontiguousarray(np.broadcast_to(fleet.srv_arrival_rpm, (L, S)), np.float32)
    got = engine.profile_margins(fleet, rate, None, None, (rate * F32(0.5)).astype(np.float32),
                                 (rate * F32(2)).astype(np.float32), **prof)
    _, win = engine.profile_grid(fleet, **prof)
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
def test_below_and_above_are_a_one_tick_profile_trace_at_their_rates(engine, big_case):
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
            _, win = engine.profile_trace(fleet, **one)
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
def test_null_profile_columns_are_the_workload_margin_calls(engine, big_case, trace):
    fleet, rows, lo, hi = big_case
    load = split(rows)[0]
    n0 = engine.launch_count
    got = getattr(engine, CALLS[trace])(fleet, load["arrival_rpm"], load["in_tokens"], load["out_tokens"], lo, hi)
    n1 = engine.launch_count
    want = getattr(engine, WORKLOAD_CALLS[trace])(fleet, load["arrival_rpm"], load["in_tokens"], load["out_tokens"],
                                                  lo, hi)
    assert n1 - n0 == engine.launch_count - n1
    assert_same(got, want, "NULL profile columns")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_prices_alone_launch_what_the_workload_margins_launch(engine, big_case, trace):
    fleet, rows, lo, hi = big_case
    load = split(rows)[0]
    n0 = engine.launch_count
    run(engine, trace, fleet, prices_only(rows), lo, hi)
    n1 = engine.launch_count
    getattr(engine, WORKLOAD_CALLS[trace])(fleet, load["arrival_rpm"], load["in_tokens"], load["out_tokens"], lo, hi)
    assert n1 - n0 == engine.launch_count - n1


@pytest.mark.gpu
def test_calls_interleaved_on_one_handle(engine, oracle_mod):
    fleet = profile_fleet(30, 3, 59, False)
    fleet.accel_penalty_factor = 0.0
    rows, lo, hi = profile_margin_case(oracle_mod, fleet, 4, "mixed", 23)
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
        ptrace = lambda e: e.profile_trace(fleet, **rows, want_candidates=True)  # noqa: E731

        def resolve(e):
            e.upload(fleet)
            e.update_load(arrival_rpm=rows["arrival_rpm"][1])
            return e.resolve(want_candidates=True)

        check(grid, "grid")
        check(trace, "trace after the grid")
        check(ptrace, "profile trace after the trace")
        check(grid, "grid after the profile trace")
        check(workload, "workload margins after the grid")
        check(trace, "trace after the workload margins")
        check(resolve, "resolve after the trace")
        check(grid, "grid after a resolve")
    finally:
        fresh.close()
