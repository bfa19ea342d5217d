"""wva_load_margin_trace: wva_load_margins at every tick of a replayed reconcile, each tick against the current
allocation c_t that the workload trace carries into it.

The expected margins come from margin_trace_levels.ref_margin_trace: per tick, levels.ref_margins with one level on
the chained fleet, advanced by apply_winners of each tick's `at` records.  The GPU tests compare the CUDA path with it
bit for bit, and without the oracle with wva_workload_trace, with wva_load_margins on the advanced fleet and with
itself split in two.

A nil winner keeps c_t.  At the margins' non-negative rates a load pair is nil only in the gate-2 fleets of DESIGN.md
§3.19 (past 2^24 replicas, where the margins truncate), so the nil winners here come from pairs that are nil at every
rate: no target, an unknown model, a missing profile, and keepAccelerator against an unknown accelerator."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (F32, TINY, _moves, below, day_rows, edge_fleet, from_bits, load_pair, mixed_fleet,
                          moving_fleet, overflow_fleet, pair_state, pinned, rates_at_rate_star, ref_margins, ref_trace,
                          u32_bits, wva_fleet)
from tests.margin_trace_levels import check_margin_trace, margin_levels, margin_windows, ref_margin_trace
from tests.util import (ACC_NONE, ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED,
                        same_bytes)
from workload_variant_autoscaler_b200 import (MARGIN_HI_OPEN, MARGIN_LO_OPEN, MARGIN_TRUNCATED, Allocs, Engine,
                                              WvaError, synth_fleet, _lib)

INF = F32(np.inf)
RECORDS = ("at", "below", "above")


def trace_case(oracle_mod, fleet, L, seed):
    rate = margin_levels(oracle_mod, fleet, L, seed)
    lo, hi = margin_windows(fleet, rate, seed)
    return rate, lo, hi


def unpinned_case():
    """keepAccelerator on, min_replicas 0 and c_0 on each server's dearest accelerator: tick 0 at rate 0 is won by
    the zero-load record with accelerator "", which lifts the mask, so that the load ticks after it are won by
    cheaper accelerators (pairs a phase 1 that honoured keepAccelerator against c_0 would not have sized).  Rate-0
    ticks come back at ticks 3 and 5."""
    fleet = synth_fleet(8, 3, seed=23, keep_accelerator=True, zero_load_frac=0.0, tps_frac=0.0)
    fleet.srv_min_replicas[:] = 0
    fleet.accel_penalty_factor = 0.0
    a = int(np.argmax(fleet.acc_cost))
    fleet.srv_cur_acc[:] = a
    fleet.srv_cur_replicas[:] = 1
    fleet.srv_cur_cost[:] = (fleet.acc_cost[a] * fleet.perf_acc_count[fleet.srv_model, a]).astype(np.float32)
    x = np.maximum(fleet.srv_arrival_rpm, 100.0).astype(np.float32)
    scale = np.array([0, 1, 2.5, 0, 0.7, 0, 4], np.float32)
    rate = (scale[:, None] * x[None, :]).astype(np.float32)
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    return fleet, rate, lo, hi


def zero_gap_case(oracle_mod, seed, keep):
    """Load ticks with rate-0 ticks between them, where a zero-load winner becomes c_{t+1}.  A rate-0 tick's window is
    [0, 2 x the next load] on min_replicas > 0 servers (the walk up crosses from 0 into the load) and [0, 0] on the
    others, whose pairs have 0 replicas just above rate 0 (refused there, as the intervals refuse)."""
    fleet = moving_fleet(seed)
    fleet.srv_keep_acc[:] = keep
    fleet.srv_min_replicas[::4] = 0
    rate = margin_levels(oracle_mod, fleet, 7, seed)
    zero = np.array([1, 3, 4], np.int64)
    lo, hi = margin_windows(fleet, rate, seed)
    lo[(lo == 0) & (fleet.srv_min_replicas == 0)[None, :]] = rate[(lo == 0) & (fleet.srv_min_replicas == 0)[None, :]]
    for t in zero:
        rate[t] = 0
        lo[t] = 0
        hi[t] = np.where(fleet.srv_min_replicas > 0, rate[min(t + 2, 6)] * F32(2), 0).astype(np.float32)
    return fleet, rate, lo, hi


def same_records(x, y, fields=ALLOC_FIELDS):
    return all(same_bytes(x[k], y[k]) for k in fields)


# ---- CPU: the composition ---------------------------------------------------------------------

@pytest.mark.parametrize("name", ["moving", "mixed_keep_off", "mixed_keep_on"])
def test_composition_at_blocks_are_the_workload_trace_winners(oracle_mod, name):
    fleet = {"moving": lambda: moving_fleet(4), "mixed_keep_off": lambda: mixed_fleet(12, 3, 5, False),
             "mixed_keep_on": lambda: mixed_fleet(12, 3, 5, True)}[name]()
    rate, lo, hi = trace_case(oracle_mod, fleet, 6, 7)
    ref = ref_margin_trace(oracle_mod, fleet, rate, lo, hi)
    _, win, _ = ref_trace(oracle_mod, fleet, {"arrival_rpm": rate})
    assert same_records(ref[3], win)


@pytest.mark.parametrize("name", ["moving", "mixed_keep_off"])
def test_composition_is_not_the_grid(oracle_mod, name):
    """Against c_0 at every row (ref_margins of the grid) some tick's lo, hi or `at` differs, and c_t changes
    accelerator along the trace."""
    fleet = moving_fleet(4) if name == "moving" else mixed_fleet(12, 3, 5, False)
    rate, lo, hi = trace_case(oracle_mod, fleet, 6, 7)
    tr = ref_margin_trace(oracle_mod, fleet, rate, lo, hi)
    grid = ref_margins(oracle_mod, fleet, rate, lo, hi)
    S = fleet.n_servers
    assert _moves(tr[3], S) > 0
    differs = [not same_bytes(tr[0][t], grid[0][t]) or not same_bytes(tr[1][t], grid[1][t])
               or not same_records(tr[3].reshape(-1, S)[t], grid[3].reshape(-1, S)[t]) for t in range(6)]
    assert any(differs[1:]) and not differs[0]


def test_wva_configuration_is_the_grid_up_to_value(oracle_mod):
    """Every server pinned, one candidate: c_t never leaves c_0's accelerator, so the stretches are the grid's and the
    records differ at most in value (TransitionPenalty against c_t instead of c_0)."""
    fleet = wva_fleet(12, 3, 9)
    assert pinned(fleet).all()
    rate, lo, hi = trace_case(oracle_mod, fleet, 5, 9)
    tr = ref_margin_trace(oracle_mod, fleet, rate, lo, hi)
    grid = ref_margins(oracle_mod, fleet, rate, lo, hi)
    assert same_bytes(tr[0], grid[0]) and same_bytes(tr[1], grid[1]) and np.array_equal(tr[2], grid[2])
    rest = [k for k in ALLOC_FIELDS if k != "value"]
    for k in range(3, 6):
        assert same_records(tr[k], grid[k], rest)
    assert not same_records(tr[3], grid[3])  # the chain does move the penalty


def test_unpinned_case_is_reached(oracle_mod):
    fleet, rate, lo, hi = unpinned_case()
    assert not pinned(fleet).any()
    tr = ref_margin_trace(oracle_mod, fleet, rate, lo, hi)
    at = tr[3].reshape(-1, fleet.n_servers)
    assert (at[0]["feasible"] == 1).all() and (at[0]["acc"] == ACC_NONE).all()
    assert ((at[1]["acc"] != fleet.srv_cur_acc) & (at[1]["feasible"] == 1)).any()


def test_the_call_is_exported():
    assert "wva_load_margin_trace" in _lib.EXPORTS


# ---- GPU: bit for bit against the composition ---------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("kind", ["mixed", "edge"])
def test_small_fleets(engine, oracle_mod, kind, keep):
    fleet = mixed_fleet(14, 3, 31, keep) if kind == "mixed" else edge_fleet(31, keep=keep)
    rate, lo, hi = trace_case(oracle_mod, fleet, 5, 7)
    _, _, flags, *_ = check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, f"{kind}, keep = {keep}")
    assert (flags == 0).any() and (flags & MARGIN_HI_OPEN).any()


@pytest.mark.gpu
def test_moving_fleet(engine, oracle_mod):
    fleet = moving_fleet(4)
    rate, lo, hi = trace_case(oracle_mod, fleet, 8, 7)
    ref = check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, "moving")
    assert _moves(ref[3], fleet.n_servers) > 0


@pytest.mark.gpu
def test_unpinned_server_lifts_its_mask(engine, oracle_mod):
    fleet, rate, lo, hi = unpinned_case()
    check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, "unpinned")


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_rate_zero_ticks_between_load_ticks(engine, oracle_mod, keep):
    fleet, rate, lo, hi = zero_gap_case(oracle_mod, 13, keep)
    _, _, flags, at, *_ = check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, f"zero gaps, keep = {keep}")
    assert (flags[1] & MARGIN_LO_OPEN).all()
    assert (at["acc"].reshape(7, -1)[1][fleet.srv_min_replicas == 0] == ACC_NONE).all()


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = mixed_fleet(40, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    fleet.accel_penalty_factor = 0.0
    rate, lo, hi = trace_case(oracle_mod, fleet, 4, 11)
    return fleet, rate, lo, hi, ref_margin_trace(oracle_mod, fleet, rate, lo, hi)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [None, "1", "2", "3", "4", "5"])
def test_warp_path_and_every_tree_depth(engine, oracle_mod, rounds_case, monkeypatch, depth):
    if depth is not None:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rate, lo, hi, want = rounds_case
    check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, f"D = {depth}", ref=want)


@pytest.mark.gpu
@pytest.mark.parametrize("n_acc", [32, 33])
def test_many_accelerators(engine, oracle_mod, n_acc):
    fleet = mixed_fleet(6, n_acc, 43, False)
    fleet.accel_penalty_factor = 0.0
    rate, lo, hi = trace_case(oracle_mod, fleet, 3, 13)
    check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, f"A = {n_acc}")


@pytest.mark.gpu
def test_nan_and_huge_values_and_ties(engine, oracle_mod):
    """NaN, 1e38, 0 and -MaxFloat32 current costs, and accelerators 1 and 2 tied on value (edge_fleet), with NaN
    penalties on a keepAccelerator-off fleet whose chain moves."""
    fleet = edge_fleet(43, keep=False, factor=0.0)
    fleet.srv_cur_cost[::4] = np.nan
    fleet.srv_cur_cost[1::4] = -F32_MAX
    rate, lo, hi = trace_case(oracle_mod, fleet, 5, 17)
    check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, "NaN / huge values and ties")


@pytest.mark.gpu
def test_windows_that_are_one_point(engine, oracle_mod):
    fleet = mixed_fleet(12, 3, 41, False)
    rate, _, _ = trace_case(oracle_mod, fleet, 3, 13)
    _, _, flags, *_ = check_margin_trace(engine, oracle_mod, fleet, rate, rate.copy(), rate.copy(), "lo = r = hi")
    assert ((flags & (MARGIN_LO_OPEN | MARGIN_HI_OPEN)) == (MARGIN_LO_OPEN | MARGIN_HI_OPEN)).all()


@pytest.mark.gpu
def test_tps_targets_out_tokens_zero_and_nil_winners(engine, oracle_mod):
    """A TPS target and out_tokens 0: the key does not read the load above rate 0.  No target, an unknown model, a
    missing profile and keepAccelerator against an unknown accelerator: nil winners, which keep c_t."""
    fleet = synth_fleet(9, 3, seed=19, zero_load_frac=0.0, tps_frac=0.0)
    fleet.srv_slo_tps[0] = 500
    fleet.srv_out_tokens[1] = 0
    fleet.srv_has_target[2] = 0
    fleet.srv_model[3] = -1
    fleet.perf_present[fleet.srv_model[4], :] = 0
    fleet.srv_cur_acc[5], fleet.srv_keep_acc[5] = -2, 1
    rate, lo, hi = trace_case(oracle_mod, fleet, 3, 19)
    lo[:, :2] = 0
    _, _, flags, at, *_ = check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, "TPS, out 0, nil")
    assert (flags[:, 0:2] & MARGIN_HI_OPEN).all()
    assert (at["feasible"].reshape(3, -1)[:, 2:6] == 0).all()


@pytest.mark.gpu
def test_replica_overflow_truncates(engine, oracle_mod):
    """A replica overflow above, at and below a tick's rate."""
    fleet = synth_fleet(3, 2, seed=5, tps_frac=0.0, zero_load_frac=0.0)
    s = 0
    rs, rmax, _, _ = load_pair(oracle_mod, fleet, s, 0)
    lo_b, hi_b = u32_bits(F32(1)), u32_bits(F32_MAX)
    while hi_b - lo_b > 1:
        m = (lo_b + hi_b) // 2
        if pair_state(fleet, s, rs, rmax, from_bits(m))[2]:
            hi_b = m
        else:
            lo_b = m
    over = from_bits(hi_b)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    rate = np.stack([x, x, x, x])
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    rate[0, s], lo[0, s], hi[0, s] = from_bits(hi_b - 3), from_bits(hi_b - 6), from_bits(hi_b + 6)  # above r
    rate[1, s], lo[1, s], hi[1, s] = over, from_bits(hi_b - 6), from_bits(hi_b + 6)                 # at r
    rate[2, s], lo[2, s], hi[2, s] = from_bits(hi_b + 2), from_bits(hi_b - 6), from_bits(hi_b + 6)  # below r
    _, _, flags, *_ = check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, "overflow")
    assert flags[1, s] == flags[2, s] == MARGIN_TRUNCATED


@pytest.mark.gpu
def test_stored_vector_fallback_at_each_record(engine, oracle_mod):
    """Rates at which totalRate / replicas lands at rateStar, where the chain leaves the streaming windows: as r, as
    the float below lo and as hi."""
    base = overflow_fleet()
    rates = np.array(rates_at_rate_star(oracle_mod, base, 0, 0), np.float32)
    fleet = base.take_servers(np.zeros(len(rates), np.int64))
    up = np.array([np.nextafter(r, INF) for r in rates], np.float32)
    rate = np.stack([rates, up, below(rates)])
    lo = np.stack([rates, rates, np.zeros_like(rates)])
    hi = np.stack([rates, up, rates])
    check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, "stored-vector fallback")


@pytest.mark.gpu
def test_tiny_rates_are_refused_as_the_margins_refuse(engine, oracle_mod):
    fleet = synth_fleet(4, 2, seed=3, tps_frac=0.0, zero_load_frac=0.0)
    fleet.srv_min_replicas[:] = np.maximum(fleet.srv_min_replicas, 1)
    rate = np.array([[1e-41, TINY, 0, 2.0], [2.0, 3.0, 4.0, 5.0]], np.float32)
    lo = np.array([[0, TINY, 0, 0], [1.0, 1.0, 1.0, 1.0]], np.float32)
    hi = np.array([[1e-40, 1e-42, 1e-40, 5.0], [4.0, 6.0, 8.0, 10.0]], np.float32)
    check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, "tiny rates")
    fleet.srv_min_replicas[0] = 0
    with pytest.raises(WvaError) as mg:
        engine.load_margins(fleet, rate[:1], lo[:1], hi[:1])
    with pytest.raises(WvaError) as tr:
        engine.load_margin_trace(fleet, rate, lo, hi)
    assert mg.value.code == tr.value.code == WVA_ERR_UNSUPPORTED
    rate[0, 0] = lo[0, 0] = F32(1e-40)  # the same window above the underflow is fine
    engine.load_margin_trace(fleet, rate, lo, hi)


# ---- GPU: against the other calls, without the oracle -------------------------------------------

def big_rows(kind):
    if kind == "24":
        fleet = synth_fleet(1500, 8, seed=42)
        x = fleet.srv_arrival_rpm.astype(np.float32)
        rng = np.random.default_rng(5)
        rate = (np.maximum(x, 1.0)[None, :] * rng.lognormal(0, 0.6, (24, x.size))).astype(np.float32)
    else:
        fleet = synth_fleet(1500, 8, seed=42)
        rate = day_rows(fleet, 288, 288, 3, special=False)["arrival_rpm"]
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    return fleet, rate, lo, hi


@pytest.fixture(scope="module", params=["24", "288"])
def big_case(request):
    return big_rows(request.param)


def part(allocs, t, S):
    """Block t (records t*S .. t*S + S - 1) of an Allocs."""
    x = Allocs(S)
    for f in ALLOC_FIELDS:
        getattr(x, f)[:] = getattr(allocs, f)[t * S:(t + 1) * S]
    return x


def block(result, t, S):
    lo, hi, flags, *recs = result
    return (lo[t], hi[t], flags[t]) + tuple(part(r, t, S) for r in recs)


def assert_same(x, y, what):
    for k, (a, b) in enumerate(zip(x, y)):
        if isinstance(a, Allocs):
            for f in ALLOC_FIELDS:
                assert same_bytes(getattr(a, f), getattr(b, f)), f"{what}: {RECORDS[k - 3]}.{f}"
        else:
            assert same_bytes(a, b), f"{what}: column {k}"


@pytest.mark.gpu
def test_at_blocks_are_the_workload_trace_winners(engine, big_case):
    fleet, rate, lo, hi = big_case
    got = engine.load_margin_trace(fleet, rate, lo, hi)
    _, win = engine.workload_trace(fleet, rate)
    for f in ALLOC_FIELDS:
        assert same_bytes(getattr(got[3], f), getattr(win, f)), f


@pytest.mark.gpu
def test_blocks_are_the_single_call_on_the_advanced_fleet(engine, big_case):
    fleet, rate, lo, hi = big_case
    L, S = rate.shape
    got = engine.load_margin_trace(fleet, rate, lo, hi)
    cur = fleet
    for t in range(L):
        one = engine.load_margins(cur, rate[t:t + 1], lo[t:t + 1], hi[t:t + 1])
        assert_same(block(got, t, S), one, f"tick {t}")
        cur = cur.apply_winners(one[3])


@pytest.mark.gpu
def test_continuation(engine, big_case):
    fleet, rate, lo, hi = big_case
    L, S = rate.shape
    whole = engine.load_margin_trace(fleet, rate, lo, hi)
    for k in sorted({1, 32, 33, L - 1} & set(range(1, L))):  # the split points that lie inside the trace
        head = engine.load_margin_trace(fleet, rate[:k], lo[:k], hi[:k])
        cur = fleet
        for t in range(k):
            cur = cur.apply_winners(part(head[3], t, S))
        tail = engine.load_margin_trace(cur, rate[k:], lo[k:], hi[k:])
        for t in range(L):
            piece = block(head, t, S) if t < k else block(tail, t - k, S)
            assert_same(block(whole, t, S), piece, f"k = {k}, tick {t}")


# ---- GPU: call mechanics ------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_launch_count_does_not_depend_on_ticks(engine, monkeypatch, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = synth_fleet(40, 4, seed=53, zero_load_frac=0.0)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    counts = []
    for L, wide in ((1, 1.01), (24, 2.0), (1440, 100.0)):
        rate = (np.stack([x] * L) * np.linspace(0.5, 2.0, L, dtype=np.float32)[:, None]).astype(np.float32)
        n0 = engine.launch_count
        engine.load_margin_trace(fleet, rate, (rate / F32(wide)).astype(np.float32),
                                 (rate * F32(wide)).astype(np.float32))
        counts.append(engine.launch_count - n0)
    n0 = engine.launch_count
    engine.load_margins(fleet, rate[:1], rate[:1], rate[:1])
    assert counts[0] == counts[1] == counts[2] == engine.launch_count - n0 + 1, counts


@pytest.mark.gpu
def test_no_ticks_and_no_servers(engine):
    fleet = synth_fleet(6, 2, seed=61)
    got = engine.load_margin_trace(fleet, np.zeros((0, 6), np.float32))
    assert got[0].shape == (0, 6) and got[3].n == 0
    empty = fleet.take_servers(np.zeros(0, np.int64))
    got = engine.load_margin_trace(empty, np.zeros((3, 0), np.float32))
    assert got[0].shape == (3, 0) and got[3].n == 0


@pytest.mark.gpu
def test_argument_errors_and_summary(engine, oracle_mod):
    from workload_variant_autoscaler_b200 import _abi
    fleet = mixed_fleet(6, 2, 61, False)
    L, h = engine._L, engine._h
    S = fleet.n_servers
    fc = fleet.as_c()
    rate = margin_levels(oracle_mod, fleet, 2, 3)
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    lo_o, hi_o, flags = (np.zeros(2 * S, np.float32), np.zeros(2 * S, np.float32), np.zeros(2 * S, np.uint8))
    recs = [Allocs(2 * S) for _ in range(3)]

    def call(rate_=rate, lo_=lo, hi_=hi, n=2, flags_=flags, out=True):
        oc = _abi.MarginsC(_abi.ptr(lo_o), _abi.ptr(hi_o), _abi.ptr(flags_) if flags_ is not None else None,
                           *(r.as_c() for r in recs))
        p = lambda a: _abi.ptr(np.ascontiguousarray(a, np.float32).reshape(-1)) if a is not None else None  # noqa
        return L.wva_load_margin_trace(h, C.byref(fc), n, p(rate_), p(lo_), p(hi_), C.byref(oc) if out else None)

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
        engine.load_margin_trace(fleet, None)
    with pytest.raises(ValueError):
        engine.load_margin_trace(fleet, rate, lo[:, :-1], hi)
    engine.solve(fleet)
    engine.summarize(fleet.n_types)
    engine.load_margin_trace(fleet, rate, lo, hi)
    with pytest.raises(WvaError) as e:
        engine.summarize(fleet.n_types)
    assert e.value.code == WVA_ERR_STATE
    # the default window is [0, 2 * rate] (on servers with min_replicas > 0: a bottom of 0 is refused otherwise)
    fleet = synth_fleet(14, 3, seed=33)
    rate = np.stack([fleet.srv_arrival_rpm, fleet.srv_arrival_rpm * 1.5]).astype(np.float32)
    got = engine.load_margin_trace(fleet, rate)
    want = engine.load_margin_trace(fleet, rate, np.zeros_like(rate), (rate * F32(2)).astype(np.float32))
    assert_same(got, want, "default window")


@pytest.mark.gpu
def test_calls_interleaved_on_one_handle(engine, oracle_mod):
    fleet = mixed_fleet(30, 3, 59, False)
    fleet.accel_penalty_factor = 0.0
    rate, lo, hi = trace_case(oracle_mod, fleet, 4, 23)
    fresh = Engine(0)
    try:
        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if isinstance(x, Allocs):
                    for k in ALLOC_FIELDS:
                        assert same_bytes(getattr(x, k), getattr(y, k)), f"{what}: {k}"
                elif x is not None:
                    assert same_bytes(x, y), what

        trace = lambda e: e.load_margin_trace(fleet, rate, lo, hi)  # noqa: E731
        margins = lambda e: e.load_margins(fleet, rate, lo, hi)  # noqa: E731
        workload = lambda e: e.workload_trace(fleet, rate, want_candidates=True)  # noqa: E731

        def resolve(e):
            e.upload(fleet)
            e.update_load(arrival_rpm=rate[1])
            return e.resolve(want_candidates=True)

        check(trace, "trace")
        check(margins, "margins after the trace")
        check(trace, "trace after the margins")
        check(workload, "workload trace after the trace")
        check(trace, "trace after the workload trace")
        check(resolve, "resolve after the trace")
        check(trace, "trace after a resolve")
    finally:
        fresh.close()
