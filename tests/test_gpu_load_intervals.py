"""wva_load_intervals: the float32 arrival rates at which each server's load-grid winner changes its decision.

The expected intervals come from ref_intervals, a Python composition over the CPU oracle: one Analyzer.size per
pair gives rateStar and RateRange.Max; each load pair's state (replica count, Analyze's rate check) is stepped
through the range by float32 bit bisection with the arithmetic of the load-grid test's `tail`; the union of the
step points is then evaluated with the oracle's Server.Calculate + Solver.Solve (ref_grid), and an interval
starts wherever the winner's decision key changes.  The CPU tests pin that composition against the oracle at the
starts, one ulp below them, at the steps that start nothing and at random interior points; the GPU tests compare
the CUDA path with it, and with wva_load_grid, bit for bit."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (F32, KEY_FIELDS, TINY, at_row, check_intervals, from_bits, load_pair, mixed_fleet,
                          overflow_fleet, pair_state, rates_at_rate_star, rec_key, ref_intervals, u32_bits, winners_at)
from tests.util import (ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, assert_allocs_equal,
                        same_bytes)
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, synth_fleet

# ---- the oracle composition ---------------------------------------------------------------------

def ranges(fleet, seed):
    """[0.5x, 2x] of each server's load, with lo = hi on one loaded server and lo = 0 on another."""
    rng = np.random.default_rng(seed)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    lo = (x * F32(0.5)).astype(np.float32)
    hi = (x * F32(2.0)).astype(np.float32)
    loaded = np.nonzero(x > 0)[0]
    i, j = rng.choice(loaded, 2, replace=False)
    lo[i] = hi[i] = x[i]
    lo[j] = 0
    return lo, hi


# ---- CPU: the composition against the oracle ----------------------------------------------------

@pytest.mark.parametrize("keep", [False, True])
def test_ref_intervals_are_the_oracle_winners(oracle_mod, keep):
    fleet = mixed_fleet(12, 3, 71, keep)
    lo, hi = ranges(fleet, 5)
    M = 1024
    count, trunc, start, rec, steps = ref_intervals(oracle_mod, fleet, lo, hi, M)
    assert (count >= 1).all() and not trunc.any()
    assert count.max() >= 4
    rng = np.random.default_rng(3)
    probes, want = [[] for _ in range(fleet.n_servers)], [[] for _ in range(fleet.n_servers)]
    for s in range(fleet.n_servers):
        n = int(count[s])
        st = [F32(v) for v in start[s, :n]]
        assert st[0] == lo[s] and all(x < y for x, y in zip(st, st[1:])) and st[-1] <= hi[s]
        ends = st[1:] + [np.nextafter(F32(hi[s]), F32(np.inf))]
        for j in range(n):
            k = rec_key(rec[s * M + j])
            if j > 0:  # one ulp below a start: the previous interval
                probes[s].append(np.nextafter(st[j], F32(-np.inf)))
                want[s].append(rec_key(rec[s * M + j - 1]))
            inside = [p for p in steps[s] if st[j] < p < ends[j]]  # steps that start nothing
            if st[j] > 0:
                inside += [F32(v) for v in rng.uniform(st[j], ends[j], 3).astype(np.float32) if st[j] <= v < ends[j]]
            probes[s] += inside
            want[s] += [k] * len(inside)
    got = winners_at(oracle_mod, fleet, probes)
    n_probes = 0
    for s in range(fleet.n_servers):
        for x, w, k in zip(probes[s], got[s], want[s]):
            assert rec_key(w) == k, (s, x)
            n_probes += 1
    assert n_probes >= 40


def test_truncation_at_M_and_lo_equal_hi(oracle_mod):
    fleet = mixed_fleet(12, 3, 71, False)
    lo, hi = ranges(fleet, 5)
    full = ref_intervals(oracle_mod, fleet, lo, hi, 64)
    M = 2
    count, trunc, start, rec, _ = ref_intervals(oracle_mod, fleet, lo, hi, M)
    for s in range(fleet.n_servers):
        assert count[s] == min(M, full[0][s])
        assert trunc[s] == (full[0][s] > M)
        assert same_bytes(start[s], full[2][s, :M])
        if lo[s] == hi[s]:
            assert count[s] == 1
    assert trunc.any()


def test_tail_at_a_tiny_rate_is_zero_replicas(oracle_mod):
    """Below 60 * 2^-150 req/min totalRate is 0: with min_replicas 0 the pair has 0 replicas and Analyze's check
    sees 0/0, which passes; the oracle reports a feasible record of 0 replicas and cost 0 there."""
    fleet = synth_fleet(3, 2, seed=3, tps_frac=0.0, zero_load_frac=0.0)
    fleet.srv_min_replicas[:] = 0
    for rpm in (TINY, F32(4.2e-44)):
        assert F32(rpm) / F32(60) == 0
        cand = oracle_mod.calculate(at_row(fleet, {"arrival_rpm": [np.full(3, rpm, np.float32)]}, 0)).reshape(-1)
        assert (cand["feasible"] == 1).all() and (cand["replicas"] == 0).all() and (cand["cost"] == 0).all()


# ---- GPU: bit for bit -------------------------------------------------------------------------------

def cross_check_load_grid(engine, fleet, lo, hi, M, seed, max_levels=None):
    """One wva_load_grid over every start, every start's predecessor and random interior points reproduces the
    records at the starts and the interval's key everywhere else.  Returns the number of intervals."""
    count, trunc, start, rec = engine.load_intervals(fleet, lo, hi, M)
    S = fleet.n_servers
    rng = np.random.default_rng(seed)
    pts, want = [[] for _ in range(S)], [[] for _ in range(S)]
    keys = [[tuple(u32_bits(getattr(rec, k)[s * M + j]) if k in ("cost", "value", "max_rate")
                   else int(getattr(rec, k)[s * M + j]) for k in KEY_FIELDS) for j in range(count[s])] for s in range(S)]
    for s in range(S):
        n = int(count[s])
        st = [F32(v) for v in start[s, :n]]
        ends = st[1:] + [np.nextafter(F32(hi[s]), F32(np.inf))]
        for j in range(n):
            pts[s].append(("start", j, st[j]))
            if j > 0:
                pts[s].append(("key", j - 1, np.nextafter(st[j], F32(-np.inf))))
            if st[j] > 0 and not (trunc[s] and j == n - 1):  # a truncated list's last interval ends unreported
                for v in rng.uniform(st[j], ends[j], 2).astype(np.float32):
                    if st[j] <= v < ends[j]:
                        pts[s].append(("key", j, F32(v)))
    L = max(len(p) for p in pts)
    if max_levels is not None:
        assert L <= max_levels, L
    rows = np.zeros((L, S), np.float32)
    for s in range(S):
        vals = [v for _, _, v in pts[s]] or [F32(lo[s])]
        rows[:, s] = vals[-1]
        rows[:len(vals), s] = vals
    _, win = engine.load_grid(fleet, rows)
    for s in range(S):
        for l, (kind, j, v) in enumerate(pts[s]):
            i = l * S + s
            if kind == "start":
                for k in ALLOC_FIELDS:
                    assert same_bytes(getattr(win, k)[i:i + 1], getattr(rec, k)[s * M + j:s * M + j + 1]), (s, j, k)
            else:
                got = tuple(u32_bits(getattr(win, k)[i]) if k in ("cost", "value", "max_rate") else int(getattr(win, k)[i])
                            for k in KEY_FIELDS)
                assert got == keys[s][j], (s, j, v)
    return int(count.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet(engine, oracle_mod, monkeypatch, keep, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = mixed_fleet(14, 3, 31, keep)
    lo, hi = ranges(fleet, 7)
    count, _ = check_intervals(engine, oracle_mod, fleet, lo, hi, 64, f"small, keep = {keep}, rounds = {rounds}")
    assert count.max() >= 4
    cross_check_load_grid(engine, fleet, lo, hi, 64, 1)


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = mixed_fleet(48, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    lo, hi = ranges(fleet, 11)
    return fleet, lo, hi, ref_intervals(oracle_mod, fleet, lo, hi, 32)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, lo, hi, (count_o, trunc_o, start_o, rec_o, _) = rounds_case
    count, trunc, start, rec = engine.load_intervals(fleet, lo, hi, 32)
    assert np.array_equal(count, count_o) and np.array_equal(trunc, trunc_o)
    assert same_bytes(start, start_o)
    assert_allocs_equal(rec, rec_o, f"D = {depth}: records")


@pytest.mark.gpu
def test_configs3_shape_against_the_load_grid(engine):
    fleet = synth_fleet(1500, 8, seed=42)
    x = fleet.srv_arrival_rpm
    n = cross_check_load_grid(engine, fleet, (x * F32(0.5)).astype(np.float32), (x * F32(2)).astype(np.float32), 64, 2)
    assert n > 3 * fleet.n_servers


@pytest.mark.gpu
@pytest.mark.parametrize("n_acc", [32, 33])
def test_many_accelerators(engine, oracle_mod, n_acc):
    fleet = mixed_fleet(6, n_acc, 43, False)
    lo, hi = ranges(fleet, 13)
    check_intervals(engine, oracle_mod, fleet, lo, hi, 64, f"A = {n_acc}")


@pytest.mark.gpu
def test_M_one_and_tight_M(engine, oracle_mod):
    fleet = mixed_fleet(12, 3, 71, False)
    lo, hi = ranges(fleet, 5)
    count, trunc = check_intervals(engine, oracle_mod, fleet, lo, hi, 1, "M = 1")
    assert (count[hi > 0] == 1).all() and trunc.any()
    count, trunc = check_intervals(engine, oracle_mod, fleet, lo, hi, 3, "M = 3")
    assert trunc.any()


@pytest.mark.gpu
def test_replica_overflow_stops_the_list(engine, oracle_mod):
    fleet = synth_fleet(3, 2, seed=5, tps_frac=0.0, zero_load_frac=0.0)
    s, a = 0, 0
    rs, rmax, _, _ = load_pair(oracle_mod, fleet, s, a)
    # the first rate at which ceil(totalRate / rateStar) exceeds INT32_MAX, found on the oracle's rateStar
    lo_b, hi_b = u32_bits(F32(1)), u32_bits(F32_MAX)
    while hi_b - lo_b > 1:
        m = (lo_b + hi_b) // 2
        if pair_state(fleet, s, rs, rmax, from_bits(m))[2]:
            hi_b = m
        else:
            lo_b = m
    over = from_bits(hi_b)
    lo = fleet.srv_arrival_rpm.astype(np.float32).copy()
    hi = lo.copy()
    lo[s] = from_bits(hi_b - 6)
    hi[s] = from_bits(hi_b + 6)
    count, trunc = check_intervals(engine, oracle_mod, fleet, lo, hi, 64, "overflow")
    _, _, start, _ = engine.load_intervals(fleet, lo, hi, 64)
    assert trunc[s] == 1 and 1 <= count[s] <= 6 and start[s, count[s] - 1] < over
    lo[s] = over  # overflow at rpm_lo itself: nothing is written
    count, trunc, _, _ = engine.load_intervals(fleet, lo, hi, 64)
    assert count[s] == 0 and trunc[s] == 1


@pytest.mark.gpu
def test_nan_and_huge_values_and_ties(engine, oracle_mod):
    fleet = mixed_fleet(12, 3, 43, False)
    fleet.srv_cur_cost[::2] = np.nan
    fleet.srv_cur_cost[1::4] = -F32_MAX
    fleet.acc_cost[2] = fleet.acc_cost[1]
    fleet.perf_alpha[:, 2] = fleet.perf_alpha[:, 1]
    for k in ("perf_beta", "perf_gamma", "perf_delta", "perf_acc_count"):
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]
    lo, hi = ranges(fleet, 17)
    check_intervals(engine, oracle_mod, fleet, lo, hi, 64, "NaN / huge values and ties")


@pytest.mark.gpu
def test_stored_vector_fallback_at_the_starts(engine, oracle_mod):
    base = overflow_fleet()
    rates = rates_at_rate_star(oracle_mod, base, 0, 0)
    fleet = base.take_servers(np.zeros(len(rates), np.int64))
    lo = np.array(rates, np.float32)
    hi = np.array([np.nextafter(F32(r), F32(np.inf)) for r in rates], np.float32)
    count, _ = check_intervals(engine, oracle_mod, fleet, lo, hi, 4, "stored-vector fallback")
    assert count.sum() >= len(rates)
    cross_check_load_grid(engine, fleet, lo, hi, 4, 3)


@pytest.mark.gpu
def test_tiny_rates_where_total_rate_underflows(engine, oracle_mod):
    """Below 60 * 2^-150 req/min totalRate is 0.  With min_replicas >= 1 the final rate is 0 and Analyze rejects it
    (a nil stretch).  With min_replicas 0 Analyze solves at 0/0: the oracle reports NaN latencies there, but the
    load grid fails at such a rate (the rescale loop does not terminate), and so do the intervals."""
    fleet = synth_fleet(4, 2, seed=3, tps_frac=0.0, zero_load_frac=0.0)
    fleet.srv_min_replicas[:] = np.maximum(fleet.srv_min_replicas, 1)
    lo = np.array([0, TINY, 0, 0], np.float32)
    hi = np.array([1e-40, 1e-42, 1e-40, 5.0], np.float32)
    check_intervals(engine, oracle_mod, fleet, lo, hi, 16, "tiny rates")
    count, _, start, rec = engine.load_intervals(fleet, lo, hi, 16)
    # server 0: rate 0, then nil while totalRate is 0, then feasible
    assert count[0] >= 3 and start[0, 1] == TINY and rec.feasible[1] == 0 and rec.feasible[2] == 1
    cross_check_load_grid(engine, fleet, lo, hi, 16, 4)
    fleet.srv_min_replicas[0] = 0
    with pytest.raises(WvaError) as grid:
        engine.load_grid(fleet, np.full((1, 4), TINY, np.float32))
    with pytest.raises(WvaError) as iv:
        engine.load_intervals(fleet, lo, hi, 16)
    assert iv.value.code == grid.value.code == WVA_ERR_UNSUPPORTED
    lo[0] = F32(1e-40)  # above the underflow the same server is fine
    engine.load_intervals(fleet, lo, hi, 16)


@pytest.mark.gpu
def test_argument_errors_and_summary(engine):
    from workload_variant_autoscaler_b200 import _abi
    fleet = mixed_fleet(6, 2, 61, False)
    L, h = engine._L, engine._h
    S = fleet.n_servers
    fc = fleet.as_c()
    count, trunc, start, rec = np.zeros(S, np.int32), np.zeros(S, np.uint8), np.zeros(S * 4, np.float32), Allocs(S * 4)
    lo = (fleet.srv_arrival_rpm * F32(0.5)).astype(np.float32)
    hi = (fleet.srv_arrival_rpm * F32(2)).astype(np.float32)

    def call(lo_=lo, hi_=hi, M=4, count_=count, out=True, f=fc):
        oc = _abi.IntervalsC(M, _abi.ptr(count_) if count_ is not None else None, _abi.ptr(trunc), _abi.ptr(start),
                             rec.as_c())
        return L.wva_load_intervals(h, C.byref(f), _abi.ptr(lo_) if lo_ is not None else None,
                                    _abi.ptr(hi_) if hi_ is not None else None, C.byref(oc) if out else None)

    assert call() == 0
    assert call(out=False) == WVA_ERR_BAD_ARG
    assert call(M=0) == WVA_ERR_BAD_ARG
    assert call(lo_=None) == WVA_ERR_BAD_ARG
    assert call(count_=None) == WVA_ERR_BAD_ARG
    for bad in (np.nan, np.inf, -1.0):
        b = lo.copy()
        b[1] = bad
        assert call(lo_=b, hi_=np.full(S, np.inf if bad != np.inf else 1, np.float32)) == WVA_ERR_BAD_ARG
        assert call(hi_=np.where(np.arange(S) == 2, F32(bad), hi).astype(np.float32)) == WVA_ERR_BAD_ARG
    assert call(lo_=(hi + 1).astype(np.float32)) == WVA_ERR_BAD_ARG  # lo > hi
    assert call(M=(1 << 31) // S + 1) == WVA_ERR_UNSUPPORTED     # S * M >= 2^31
    with pytest.raises(ValueError):
        engine.load_intervals(fleet, lo[:-1], hi, 4)
    engine.solve(fleet)
    engine.summarize(fleet.n_types)
    engine.load_intervals(fleet, lo, hi, 4)
    with pytest.raises(WvaError) as e:
        engine.summarize(fleet.n_types)
    assert e.value.code == WVA_ERR_STATE


@pytest.mark.gpu
def test_cache_interplay_on_one_handle(engine):
    fleet = mixed_fleet(30, 3, 59, True)
    lo, hi = ranges(fleet, 23)
    rpm = np.stack([lo, hi, (lo + hi) / 2]).astype(np.float32)
    fresh = Engine(0)
    try:
        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if isinstance(x, Allocs):
                    for k in ALLOC_FIELDS:
                        assert same_bytes(getattr(x, k), getattr(y, k)), f"{what}: {k}"
                elif x is not None:
                    assert same_bytes(x, y), what

        solve = lambda e: e.solve(fleet)  # noqa: E731
        size_grid = lambda e: e.size_grid(fleet, [4, 16, 64], want_candidates=True)  # noqa: E731
        load_grid = lambda e: e.load_grid(fleet, rpm, want_candidates=True)  # noqa: E731
        intervals = lambda e: e.load_intervals(fleet, lo, hi, 16)  # noqa: E731
        check(solve, "solve")
        check(intervals, "intervals after a solve")
        check(solve, "solve after the intervals")
        check(load_grid, "load grid after the intervals")
        check(intervals, "intervals after the load grid")
        check(size_grid, "size grid after the intervals")
        check(intervals, "intervals after the size grid")
    finally:
        fresh.close()


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_launch_count_does_not_depend_on_M(engine, monkeypatch, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = synth_fleet(40, 4, seed=53, zero_load_frac=0.0)
    x = fleet.srv_arrival_rpm
    lo, hi = (x * F32(0.5)).astype(np.float32), (x * F32(2)).astype(np.float32)
    counts = []
    for M in (1, 64):
        n0 = engine.launch_count
        engine.load_intervals(fleet, lo, hi, M)
        counts.append(engine.launch_count - n0)
    assert counts[0] == counts[1], counts
