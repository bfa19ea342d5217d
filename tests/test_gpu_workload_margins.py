"""wva_workload_margins and wva_workload_margin_trace: the load margins (grid and trace) at rows that carry their own
token lengths.

The expected margins come from workload_margin_levels.ref_workload_margins: per row, levels.ref_margins with one level
on the fleet with the row's rate and tokens, on a trace also with the c_t that apply_winners of each tick's `at`
carries.  The GPU tests compare the CUDA path with it bit for bit, and without the oracle with wva_load_margins on
the row's fleet, with the workload grid and trace, and with the load-margin calls at the fleet's own tokens."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (F32, TINY, _moves, below, day_rows, edge_fleet, from_bits, load_pair, mixed_fleet,
                          overflow_fleet, pair_state, pinned, rates_at_rate_star, ref_grid, ref_margins, ref_trace,
                          token_fleet, u32_bits)
from tests.margin_trace_levels import margin_windows, ref_margin_trace
from tests.util import ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, same_bytes
from tests.workload_margin_levels import (CALLS, assert_same, block, check_workload_margins, own_tokens, part,
                                          ref_workload_margins, unpinned_case, workload_margin_rows)
from workload_variant_autoscaler_b200 import (MARGIN_HI_OPEN, MARGIN_LO_OPEN, MARGIN_TRUNCATED, Allocs, Engine,
                                              WvaError, synth_fleet, _lib)

TRACES = [False, True]


def case(oracle_mod, fleet, L, seed, special=True):
    rows = workload_margin_rows(oracle_mod, fleet, L, seed, special)
    lo, hi = margin_windows(fleet, rows["arrival_rpm"], seed)
    return rows, lo, hi


def same_records(x, y, fields=ALLOC_FIELDS):
    return all(same_bytes(x[k], y[k]) for k in fields)


def tps_case():
    """Servers with a TPS target (totalRate = TPS / out_tokens of the row) at out_tokens 0.5x, 1x and 2x their own."""
    fleet = synth_fleet(6, 3, seed=71, zero_load_frac=0.0, tps_frac=0.0)
    fleet.srv_slo_tps[:3] = (2e4, 1e5, 5e5)
    x = np.maximum(fleet.srv_arrival_rpm, 50.0).astype(np.float32)
    rate = np.stack([x, x, x])
    out = np.stack([np.maximum(fleet.srv_out_tokens // 2, 1), fleet.srv_out_tokens, fleet.srv_out_tokens * 2])
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": out.astype(np.int32)}
    return fleet, rows, (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)


# ---- CPU: the composition ---------------------------------------------------------------------

@pytest.mark.parametrize("trace", TRACES)
def test_composition_at_blocks_are_the_workload_winners(oracle_mod, trace):
    fleet = token_fleet(12, 3, 5, trace)
    rows, lo, hi = case(oracle_mod, fleet, 5, 7)
    ref = ref_workload_margins(oracle_mod, fleet, rows, lo, hi, trace)
    win = (ref_trace if trace else ref_grid)(oracle_mod, fleet, rows)[1]
    assert same_records(ref[3], win)


@pytest.mark.parametrize("trace", TRACES)
def test_composition_at_own_tokens_is_the_load_margins(oracle_mod, trace):
    fleet = mixed_fleet(12, 3, 5, False)
    rows, lo, hi = case(oracle_mod, fleet, 4, 9)
    rows = own_tokens(fleet, rows["arrival_rpm"])
    ref = ref_workload_margins(oracle_mod, fleet, rows, lo, hi, trace)
    want = (ref_margin_trace if trace else ref_margins)(oracle_mod, fleet, rows["arrival_rpm"], lo, hi)
    for k in range(3):
        assert same_bytes(ref[k], want[k]), k
    for k in range(3, 6):
        assert same_records(ref[k], want[k]), k


def test_composition_reads_the_tokens(oracle_mod):
    """On token rows some level's stretch or record differs from the margins at the fleet's own tokens."""
    fleet = token_fleet(12, 3, 5, False)
    rows, lo, hi = case(oracle_mod, fleet, 5, 7)
    ref = ref_workload_margins(oracle_mod, fleet, rows, lo, hi, False)
    fixed = ref_margins(oracle_mod, fleet, rows["arrival_rpm"], lo, hi)
    S = fleet.n_servers
    differs = [not same_bytes(ref[0][l], fixed[0][l]) or not same_bytes(ref[1][l], fixed[1][l])
               or not same_records(ref[3].reshape(-1, S)[l], fixed[3].reshape(-1, S)[l]) for l in range(5)]
    assert sum(differs) >= 2, differs


def test_tps_records_follow_the_rows_out_tokens(oracle_mod):
    fleet, rows, lo, hi = tps_case()
    ref = ref_workload_margins(oracle_mod, fleet, rows, lo, hi, False)
    at = ref[3].reshape(3, -1)
    for s in range(3):
        assert len({int(at[l]["replicas"][s]) for l in range(3)}) == 3, s
    assert (ref[2][:, :3] & MARGIN_HI_OPEN).all()  # totalRate does not read the load


def test_unpinned_case_is_reached_on_token_rows(oracle_mod):
    fleet, rows, lo, hi = unpinned_case()
    assert not pinned(fleet).any()
    tr = ref_workload_margins(oracle_mod, fleet, rows, lo, hi, True)
    at = tr[3].reshape(-1, fleet.n_servers)
    assert (at[0]["acc"] == -1).all() and ((at[1]["acc"] != fleet.srv_cur_acc) & (at[1]["feasible"] == 1)).any()


def test_the_calls_are_exported():
    assert {"wva_workload_margins", "wva_workload_margin_trace"} <= set(_lib.EXPORTS)


# ---- GPU: bit for bit against the composition ---------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("kind", ["mixed", "token"])
def test_small_fleets(engine, oracle_mod, kind, keep, trace):
    """workload_levels' rows: rate-only, token-only and joint changes, and in -1, out -1, out 0, in 0, in 100,000
    and out 20,000 scattered over them."""
    fleet = (mixed_fleet if kind == "mixed" else token_fleet)(14, 3, 31, keep)
    rows, lo, hi = case(oracle_mod, fleet, 5, 7)
    _, _, flags, *_ = check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace,
                                             f"{kind}, keep = {keep}, trace = {trace}")
    assert (flags == 0).any() and (flags & MARGIN_HI_OPEN).any()


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_tps_targets(engine, oracle_mod, trace):
    fleet, rows, lo, hi = tps_case()
    check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"TPS, trace = {trace}")


@pytest.mark.gpu
def test_unpinned_server_lifts_its_mask(engine, oracle_mod):
    fleet, rows, lo, hi = unpinned_case()
    ref = check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, True, "unpinned")
    assert _moves(ref[3], fleet.n_servers) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_rate_zero_rows_between_load_rows(engine, oracle_mod, trace):
    """Rate-0 rows (window [0, 2 x a later load] on min_replicas > 0 servers, [0, 0] elsewhere) between token rows."""
    fleet = token_fleet(12, 3, 13, True)
    fleet.srv_min_replicas[::4] = 0
    rows, lo, hi = case(oracle_mod, fleet, 7, 13)
    zero_min = (fleet.srv_min_replicas == 0)[None, :]
    lo[(lo == 0) & zero_min] = rows["arrival_rpm"][(lo == 0) & zero_min]
    for t in (1, 3, 4):
        rows["arrival_rpm"][t] = 0
        lo[t] = 0
        hi[t] = np.where(fleet.srv_min_replicas > 0, rows["arrival_rpm"][min(t + 2, 6)] * F32(2), 0).astype(np.float32)
    _, _, flags, *_ = check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"zero rows, {trace}")
    assert (flags[1] & MARGIN_LO_OPEN).all()


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = token_fleet(40, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    fleet.accel_penalty_factor = 0.0
    rows, lo, hi = case(oracle_mod, fleet, 4, 11)
    return fleet, rows, lo, hi, {t: ref_workload_margins(oracle_mod, fleet, rows, lo, hi, t) for t in TRACES}


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
@pytest.mark.parametrize("depth", [None, "1", "2", "3", "4", "5"])
def test_warp_path_and_every_tree_depth(engine, oracle_mod, rounds_case, monkeypatch, depth, trace):
    if depth is not None:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rows, lo, hi, want = rounds_case
    check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"D = {depth}", ref=want[trace])


@pytest.mark.gpu
@pytest.mark.parametrize("n_acc", [32, 33])
def test_many_accelerators(engine, oracle_mod, n_acc):
    fleet = token_fleet(6, n_acc, 43, False)
    fleet.accel_penalty_factor = 0.0
    rows, lo, hi = case(oracle_mod, fleet, 3, 13)
    for trace in TRACES:
        check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"A = {n_acc}, trace = {trace}")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_nan_and_huge_values_and_ties(engine, oracle_mod, trace):
    fleet = edge_fleet(43, keep=False, factor=0.0)
    fleet.srv_cur_cost[::4] = np.nan
    fleet.srv_cur_cost[1::4] = -F32_MAX
    rows, lo, hi = case(oracle_mod, fleet, 4, 17)
    check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, f"NaN / huge values and ties, {trace}")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_stored_vector_fallback_at_each_record(engine, oracle_mod, trace):
    """The overflow fleet with its batch size from the perf data: out_tokens 64 gives N = 1024 at the row (the fleet's
    own out_tokens are 32, N = 2048), and the rates put totalRate / replicas at rateStar as r, below lo and at hi."""
    base = overflow_fleet()
    base.perf_max_batch[:] = 1024
    base.perf_at_tokens[:] = 64
    base.srv_max_batch[:] = 0
    rates = np.array(rates_at_rate_star(oracle_mod, base, 0, 0), np.float32)
    fleet = base.take_servers(np.zeros(len(rates), np.int64))
    fleet.srv_out_tokens[:] = 32
    up = np.array([np.nextafter(r, F32(np.inf)) for r in rates], np.float32)
    rate = np.stack([rates, up, below(rates)])
    lo = np.stack([rates, rates, np.zeros_like(rates)])
    hi = np.stack([rates, up, rates])
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": np.full(rate.shape, 64, np.int32)}
    check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, "stored-vector fallback")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_replica_overflow_truncates(engine, oracle_mod, trace):
    """A replica overflow above and at a row's rate, at the row's out_tokens."""
    fleet = synth_fleet(3, 2, seed=5, tps_frac=0.0, zero_load_frac=0.0)
    s = 0
    out_row = np.int32(fleet.srv_out_tokens[s] * 2)
    f = fleet.take_servers(np.arange(3))
    f.srv_out_tokens[s] = out_row
    rs, rmax, _, _ = load_pair(oracle_mod, f, s, 0)
    lo_b, hi_b = u32_bits(F32(1)), u32_bits(F32_MAX)
    while hi_b - lo_b > 1:
        m = (lo_b + hi_b) // 2
        if pair_state(f, s, rs, rmax, from_bits(m))[2]:
            hi_b = m
        else:
            lo_b = m
    x = fleet.srv_arrival_rpm.astype(np.float32)
    rate = np.stack([x, x, x])
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    rate[0, s], lo[0, s], hi[0, s] = from_bits(hi_b - 3), from_bits(hi_b - 6), from_bits(hi_b + 6)
    rate[1, s], lo[1, s], hi[1, s] = from_bits(hi_b), from_bits(hi_b - 6), from_bits(hi_b + 6)
    out = np.stack([fleet.srv_out_tokens] * 3).astype(np.int32)
    out[:2, s] = out_row
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": out}
    _, _, flags, *_ = check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, "overflow")
    assert flags[1, s] == MARGIN_TRUNCATED


# ---- GPU: refusals ------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_out_tokens_one_refuses_only_under_a_window(engine, oracle_mod, trace):
    """N = MaxBatchSize * AtTokens / out_tokens: out_tokens 1 puts server 0's N at 2^21, outside the queue-size rule
    (N = 32 at its other rows).  Refused, as wva_load_margins on the row's fleet refuses, where the row's window top is
    above 0; never sized where the window is [0, 0]."""
    fleet = synth_fleet(4, 2, seed=83, zero_load_frac=0.0)
    fleet.srv_max_batch[0] = 0
    fleet.perf_max_batch[:] = 512
    fleet.perf_at_tokens[:] = 1 << 12
    fleet.srv_min_replicas[:] = np.maximum(fleet.srv_min_replicas, 1)
    x = np.maximum(fleet.srv_arrival_rpm, 10.0).astype(np.float32)
    rate = np.stack([x, x])
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    out = np.stack([fleet.srv_out_tokens] * 2).astype(np.int32)
    out[:, 0] = 1 << 16
    out[1, 0] = 1
    f1 = fleet.take_servers(np.arange(4))
    f1.srv_out_tokens[:] = out[1]
    with pytest.raises(WvaError) as single:
        engine.load_margins(f1, rate[1:], lo[1:], hi[1:])
    with pytest.raises(WvaError) as e:
        getattr(engine, CALLS[trace])(fleet, rate, None, out, lo, hi)
    assert e.value.code == single.value.code == WVA_ERR_UNSUPPORTED
    rate[1, 0] = lo[1, 0] = hi[1, 0] = 0
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": out}
    check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, "out 1 under [0, 0]")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_tiny_rates_are_refused_as_the_margins_refuse(engine, oracle_mod, trace):
    fleet = synth_fleet(4, 2, seed=3, tps_frac=0.0, zero_load_frac=0.0)
    fleet.srv_min_replicas[:] = np.maximum(fleet.srv_min_replicas, 1)
    rate = np.array([[1e-41, TINY, 0, 2.0], [2.0, 3.0, 4.0, 5.0]], np.float32)
    lo = np.array([[0, TINY, 0, 0], [1.0, 1.0, 1.0, 1.0]], np.float32)
    hi = np.array([[1e-40, 1e-42, 1e-40, 5.0], [4.0, 6.0, 8.0, 10.0]], np.float32)
    out = (np.stack([fleet.srv_out_tokens] * 2) * np.array([[1.5], [1]])).astype(np.int32)
    rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": out}
    check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, "tiny rates")
    fleet.srv_min_replicas[0] = 0
    with pytest.raises(WvaError) as e:
        getattr(engine, CALLS[trace])(fleet, rate, None, out, lo, hi)
    assert e.value.code == WVA_ERR_UNSUPPORTED


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_argument_errors_and_summary(engine, oracle_mod, trace):
    from workload_variant_autoscaler_b200 import _abi
    fleet = mixed_fleet(6, 2, 61, False)
    fn = getattr(engine._L, "wva_" + CALLS[trace])
    h, S = engine._h, fleet.n_servers
    fc = fleet.as_c()
    rows, lo, hi = case(oracle_mod, fleet, 2, 3, special=False)
    rate = rows["arrival_rpm"]
    lo_o, hi_o, flags = np.zeros(2 * S, np.float32), np.zeros(2 * S, np.float32), np.zeros(2 * S, np.uint8)
    recs = [Allocs(2 * S) for _ in range(3)]

    def call(rate_=rate, lo_=lo, hi_=hi, n=2, flags_=flags, out=True):
        oc = _abi.MarginsC(_abi.ptr(lo_o), _abi.ptr(hi_o), _abi.ptr(flags_) if flags_ is not None else None,
                           *(r.as_c() for r in recs))
        p = lambda a: _abi.ptr(np.ascontiguousarray(a, np.float32).reshape(-1)) if a is not None else None  # noqa
        t = lambda a: _abi.ptr(np.ascontiguousarray(a, np.int32).reshape(-1))  # noqa: E731
        return fn(h, C.byref(fc), n, p(rate_), t(rows["in_tokens"]), t(rows["out_tokens"]), p(lo_), p(hi_),
                  C.byref(oc) if out else None)

    assert call() == 0
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
    assert call(hi_=(rate * F32(0.5)).astype(np.float32)) == WVA_ERR_BAD_ARG  # r > hi
    assert call(n=(1 << 31) // (3 * S) + 1) == WVA_ERR_UNSUPPORTED  # refused before the rows are read
    with pytest.raises(ValueError):
        getattr(engine, CALLS[trace])(fleet, None)
    with pytest.raises(ValueError):
        getattr(engine, CALLS[trace])(fleet, rate, rows["in_tokens"][:, :-1])
    engine.solve(fleet)
    engine.summarize(fleet.n_types)
    getattr(engine, CALLS[trace])(fleet, rate, rows["in_tokens"], rows["out_tokens"], lo, hi)
    with pytest.raises(WvaError) as e:
        engine.summarize(fleet.n_types)
    assert e.value.code == WVA_ERR_STATE
    # the default window is [0, 2 * rate] (on servers with min_replicas > 0: a bottom of 0 is refused otherwise)
    fleet = synth_fleet(14, 3, seed=33)
    rate = np.stack([fleet.srv_arrival_rpm, fleet.srv_arrival_rpm * 1.5]).astype(np.float32)
    out = (np.stack([fleet.srv_out_tokens] * 2) * np.array([[1], [1.5]])).astype(np.int32)
    got = getattr(engine, CALLS[trace])(fleet, rate, None, out)
    want = getattr(engine, CALLS[trace])(fleet, rate, None, out, np.zeros_like(rate), (rate * F32(2)).astype(np.float32))
    assert_same(got, want, "default window")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_no_rows_and_no_servers(engine, trace):
    call = getattr(engine, CALLS[trace])
    fleet = synth_fleet(6, 2, seed=61)
    got = call(fleet, np.zeros((0, 6), np.float32), np.zeros((0, 6), np.int32), np.zeros((0, 6), np.int32))
    assert got[0].shape == (0, 6) and got[3].n == 0
    empty = fleet.take_servers(np.zeros(0, np.int64))
    got = call(empty, np.zeros((3, 0), np.float32), np.zeros((3, 0), np.int32))
    assert got[0].shape == (3, 0) and got[3].n == 0


# ---- GPU: against the other calls, without the oracle -------------------------------------------

def big_rows(kind):
    fleet = synth_fleet(1500, 8, seed=42)
    if kind == "24":
        x = np.maximum(fleet.srv_arrival_rpm, 1.0).astype(np.float32)
        rng = np.random.default_rng(5)
        rate = (x[None, :] * rng.lognormal(0, 0.6, (24, x.size))).astype(np.float32)
        out = (fleet.srv_out_tokens[None, :] * rng.choice([0.75, 1.0, 1.5], (24, x.size))).astype(np.int32)
        rows = {"arrival_rpm": rate, "in_tokens": None, "out_tokens": np.maximum(out, 1)}
    else:
        rows = day_rows(fleet, 288, 288, 3, special=False)
    rate = rows["arrival_rpm"]
    return fleet, rows, (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)


@pytest.fixture(scope="module", params=["24", "288"])
def big_case(request):
    return big_rows(request.param)


def run(engine, trace, fleet, rows, lo, hi):
    return getattr(engine, CALLS[trace])(fleet, rows["arrival_rpm"], rows["in_tokens"], rows["out_tokens"], lo, hi)


def at_tokens(fleet, rows, l):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    for k, col in (("in_tokens", "srv_in_tokens"), ("out_tokens", "srv_out_tokens")):
        if rows[k] is not None:
            getattr(f, col)[:] = rows[k][l]
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_at_blocks_are_the_workload_winners(engine, big_case, trace):
    fleet, rows, lo, hi = big_case
    got = run(engine, trace, fleet, rows, lo, hi)
    _, win = (engine.workload_trace if trace else engine.workload_grid)(fleet, **rows)
    for f in ALLOC_FIELDS:
        assert same_bytes(getattr(got[3], f), getattr(win, f)), f


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
def test_blocks_are_the_load_margins_on_the_rows_fleet(engine, big_case, trace):
    fleet, rows, lo, hi = big_case
    L, S = lo.shape
    got = run(engine, trace, fleet, rows, lo, hi)
    cur = fleet
    for t in range(L):
        one = engine.load_margins(at_tokens(cur, rows, t), rows["arrival_rpm"][t:t + 1], lo[t:t + 1], hi[t:t + 1])
        assert_same(block(got, t, S), one, f"row {t}")
        if trace:
            cur = cur.apply_winners(one[3])


@pytest.mark.gpu
def test_below_and_above_are_the_workload_grid_at_their_rates(engine, big_case):
    fleet, rows, lo, hi = big_case
    lo_e, hi_e, flags, _, bel, abv = run(engine, False, fleet, rows, lo, hi)
    for name, rec, rates, skip in (("below", bel, below(lo_e), MARGIN_LO_OPEN | MARGIN_TRUNCATED),
                                   ("above", abv, hi_e, MARGIN_HI_OPEN | MARGIN_TRUNCATED)):
        use = (flags & skip) == 0
        assert use.any(), name
        r = np.where(use, rates, rows["arrival_rpm"]).astype(np.float32)
        _, win = engine.workload_grid(fleet, r, rows["in_tokens"], rows["out_tokens"])
        for f in ALLOC_FIELDS:
            g, w = getattr(rec, f)[use.reshape(-1)], getattr(win, f)[use.reshape(-1)]
            assert same_bytes(g, w), f"{name}.{f}"


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
def test_null_tokens_are_the_load_margin_calls(engine, big_case, trace):
    fleet, rows, lo, hi = big_case
    rate = rows["arrival_rpm"]
    n0 = engine.launch_count
    got = getattr(engine, CALLS[trace])(fleet, rate, None, None, lo, hi)
    n1 = engine.launch_count
    want = (engine.load_margin_trace if trace else engine.load_margins)(fleet, rate, lo, hi)
    assert n1 - n0 == engine.launch_count - n1
    assert_same(got, want, "NULL tokens")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", TRACES)
@pytest.mark.parametrize("rounds", [False, True])
def test_launch_count_does_not_depend_on_rows(engine, monkeypatch, rounds, trace):
    """The same token key set at L = 1, 24 and 1,440 (each server's rows take its own and 1.5x its out_tokens)."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = synth_fleet(40, 4, seed=53, zero_load_frac=0.0)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    counts = []
    for L, wide in ((2, 1.01), (24, 2.0), (1440, 100.0)):
        rate = (np.stack([x] * L) * np.linspace(0.5, 2.0, L, dtype=np.float32)[:, None]).astype(np.float32)
        out = (np.stack([fleet.srv_out_tokens] * L) * np.where(np.arange(L) % 2, 1.5, 1.0)[:, None]).astype(np.int32)
        n0 = engine.launch_count
        getattr(engine, CALLS[trace])(fleet, rate, None, out, (rate / F32(wide)).astype(np.float32),
                                      (rate * F32(wide)).astype(np.float32))
        counts.append(engine.launch_count - n0)
    assert counts[0] == counts[1] == counts[2], counts


@pytest.mark.gpu
def test_calls_interleaved_on_one_handle(engine, oracle_mod):
    fleet = token_fleet(30, 3, 59, False)
    fleet.accel_penalty_factor = 0.0
    rows, lo, hi = case(oracle_mod, fleet, 4, 23)
    fresh = Engine(0)
    try:
        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if isinstance(x, Allocs):
                    for k in ALLOC_FIELDS:
                        assert same_bytes(getattr(x, k), getattr(y, k)), f"{what}: {k}"
                elif x is not None:
                    assert same_bytes(x, y), what

        grid = lambda e: run(e, False, fleet, rows, lo, hi)  # noqa: E731
        trace = lambda e: run(e, True, fleet, rows, lo, hi)  # noqa: E731
        margins = lambda e: e.load_margins(fleet, rows["arrival_rpm"], lo, hi)  # noqa: E731
        workload = lambda e: e.workload_grid(fleet, **rows, want_candidates=True)  # noqa: E731

        def resolve(e):
            e.upload(fleet)
            e.update_load(arrival_rpm=rows["arrival_rpm"][1])
            return e.resolve(want_candidates=True)

        check(grid, "grid")
        check(trace, "trace after the grid")
        check(workload, "workload grid after the trace")
        check(grid, "grid after the workload grid")
        check(margins, "load margins after the grid")
        check(trace, "trace after the load margins")
        check(resolve, "resolve after the trace")
        check(grid, "grid after a resolve")
    finally:
        fresh.close()
