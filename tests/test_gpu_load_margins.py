"""wva_load_margins: the stretch of float32 arrival rates around each level's rate on which the load-grid winner keeps
its decision.

The expected margins come from levels.ref_margins, a composition over the CPU oracle: levels.ref_intervals over each level's
window (with M large enough never to truncate at M) lists the intervals; the margin is the one that holds the level's
rate r, the next start is hi, and the records are the oracle's winners (levels.winners_at) at r, one float32 below lo
and at hi.  A replica overflow (levels.server_steps) ends the stretch as it ends the interval list.  The GPU tests
compare the CUDA path with it bit for bit, and with wva_load_intervals, wva_load_grid and wva_solve."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from tests.levels import (F32, KEY_FIELDS, TINY, below, check_margins, from_bits, load_levels, load_pair, mixed_fleet,
                          overflow_fleet, pair_state, rates_at_rate_star, rec_key, ref_margins, u32_bits, winners_at)
from tests.util import (ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED, assert_allocs_equal,
                        same_bytes)
from workload_variant_autoscaler_b200 import (MARGIN_HI_OPEN, MARGIN_LO_OPEN, MARGIN_TRUNCATED, Allocs, Engine,
                                              WvaError, synth_fleet, within_margins)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = F32(np.inf)


def windows(fleet, rate, seed):
    """[0.5x, 2x] of each rate, with the window bottom at 0 for some and lo = r = hi for others.  A bottom of 0 is
    kept off min_replicas-0 servers, whose pairs have 0 replicas just above it (refused, as the intervals refuse)."""
    rng = np.random.default_rng(seed)
    r = np.asarray(rate, np.float32)
    lo, hi = (r * F32(0.5)).astype(np.float32), (r * F32(2)).astype(np.float32)
    pick = rng.random(r.shape)
    lo[(pick < 0.15) & (fleet.srv_min_replicas > 0)[None, :]] = 0
    lo[pick > 0.92] = hi[pick > 0.92] = r[pick > 0.92]
    return lo, hi


def clean_levels(oracle_mod, fleet, L, seed):
    """load_levels' rows without the negative and infinite rates, which the margins refuse, scaled per server so that
    its own load sits at 1.5 times its first replica step (60 * rateStar of its fastest load pair) and capped at 20
    steps: the windows around the rates hold a few steps each, and the composition's step walk stays short."""
    rows = load_levels(fleet, L, seed).astype(np.float64)
    rows[~np.isfinite(rows) | (rows < 0)] = 7.5
    for s in range(fleet.n_servers):
        steps = [60.0 * float(p[0]) for p in (load_pair(oracle_mod, fleet, s, a) for a in range(fleet.n_acc)) if p]
        if steps:
            step = min(steps)
            rows[:, s] = np.minimum(rows[:, s] * (1.5 * step / max(float(fleet.srv_arrival_rpm[s]), 1.0)), 20 * step)
    return rows.astype(np.float32)


# ---- CPU ----------------------------------------------------------------------------------------

def test_margins_struct_matches_the_header():
    from workload_variant_autoscaler_b200 import _abi
    prog = ('#include <stdio.h>\n#include "wva_b200.h"\nint main(){printf("%zu %d %d %d\\n", sizeof(wva_margins), '
            'WVA_MARGIN_LO_OPEN, WVA_MARGIN_HI_OPEN, WVA_MARGIN_TRUNCATED);return 0;}')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(prog)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"),
                        os.path.join(d, "t.c")], check=True)
        out = subprocess.run([os.path.join(d, "t")], check=True, capture_output=True, text=True).stdout.split()
    assert [int(x) for x in out] == [C.sizeof(_abi.MarginsC), MARGIN_LO_OPEN, MARGIN_HI_OPEN, MARGIN_TRUNCATED]
    assert C.sizeof(_abi.MarginsC) == 3 * 8 + 3 * C.sizeof(_abi.AllocsC)


def test_within_margins_open_ends():
    lo = np.array([[1, 1, 1, 2, 0]], np.float32)
    hi = np.array([[3, INF, 3, 2, INF]], np.float32)
    flags = np.array([[0, MARGIN_HI_OPEN, MARGIN_LO_OPEN, MARGIN_TRUNCATED, MARGIN_LO_OPEN | MARGIN_HI_OPEN]], np.uint8)
    top = np.array([[4, 4, 4, 4, 4]], np.float32)
    for x, want in ((1, [1, 1, 1, 0, 1]), (np.nextafter(F32(3), F32(0)), [1, 1, 1, 0, 1]), (3, [0, 1, 0, 0, 1]),
                    (4, [0, 1, 0, 0, 1]), (np.nextafter(F32(4), F32(5)), [0, 0, 0, 0, 0]),
                    (np.nextafter(F32(1), F32(0)), [0, 0, 0, 0, 1]), (2, [1, 1, 1, 0, 1]), (np.nan, [0] * 5)):
        got = within_margins(lo, hi, flags, np.full((1, 5), x, np.float32), top)
        assert got.tolist() == [[bool(v) for v in want]], (x, got)
    with pytest.raises(ValueError):
        within_margins(lo, hi, flags, np.zeros((1, 4), np.float32), top)


def test_ref_margins_hold_their_key_inside(oracle_mod):
    """The composition against the oracle: the key at r holds at lo, one ulp below hi and at random interior rates,
    and differs one ulp below lo and at hi where those are changes."""
    fleet = mixed_fleet(10, 3, 71, False)
    rate = clean_levels(oracle_mod, fleet, 2, 5)
    lo, hi = windows(fleet, rate, 3)
    lo_e, hi_e, flags, at, below_r, above_r = ref_margins(oracle_mod, fleet, rate, lo, hi)
    L, S = rate.shape
    rng = np.random.default_rng(9)
    probes, want = [[] for _ in range(S)], [[] for _ in range(S)]
    for l in range(L):
        for s in range(S):
            i, f = l * S + s, flags[l, s]
            if f & MARGIN_TRUNCATED and lo_e[l, s] == hi_e[l, s]:
                continue
            k = rec_key(at[i])
            top = hi_e[l, s] if not f & MARGIN_HI_OPEN else np.nextafter(hi[l, s], INF)
            inside = [lo_e[l, s], below(top)] + [F32(v) for v in rng.uniform(lo_e[l, s], top, 3).astype(np.float32)
                                                 if lo_e[l, s] <= v < top and v > 0]
            probes[s] += inside
            want[s] += [k] * len(inside)
            if not f & MARGIN_LO_OPEN:
                probes[s].append(below(lo_e[l, s]))
                want[s].append(("differs", k))
            if not f & (MARGIN_HI_OPEN | MARGIN_TRUNCATED):
                probes[s].append(hi_e[l, s])
                want[s].append(("differs", k))
    got = winners_at(oracle_mod, fleet, probes)
    n_open = n_closed = 0
    for s in range(S):
        for x, w, k in zip(probes[s], got[s], want[s]):
            if k[0] == "differs":
                assert rec_key(w) != k[1], (s, x)
                n_closed += 1
            else:
                assert rec_key(w) == k, (s, x)
                n_open += 1
    assert n_open >= 40 and n_closed >= 4


# ---- GPU: bit for bit against the composition ---------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet(engine, oracle_mod, monkeypatch, keep, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = mixed_fleet(14, 3, 31, keep)
    rate = clean_levels(oracle_mod, fleet, 3, 7)
    lo, hi = windows(fleet, rate, 7)
    _, _, flags, _, _, _ = check_margins(engine, oracle_mod, fleet, rate, lo, hi, f"keep = {keep}, rounds = {rounds}")
    assert (flags == 0).any() and (flags & MARGIN_LO_OPEN).any() and (flags & MARGIN_HI_OPEN).any()


@pytest.mark.gpu
def test_one_level_at_the_fleet_load(engine, oracle_mod):
    fleet = mixed_fleet(14, 3, 33, True)
    rate = fleet.srv_arrival_rpm[None, :].astype(np.float32)
    lo, hi = windows(fleet, rate, 2)
    check_margins(engine, oracle_mod, fleet, rate, lo, hi, "arrival_rpm = None", own_rate=True)
    # the default window is [0, 2 * rate]
    fleet = synth_fleet(14, 3, seed=33)
    rate = fleet.srv_arrival_rpm[None, :].astype(np.float32)
    got = engine.load_margins(fleet)
    want = engine.load_margins(fleet, rate, np.zeros_like(rate), (rate * F32(2)).astype(np.float32))
    for g, w in zip(got[:3], want[:3]):
        assert same_bytes(g, w)


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = mixed_fleet(48, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    rate = clean_levels(oracle_mod, fleet, 2, 11)
    lo, hi = windows(fleet, rate, 11)
    return fleet, rate, lo, hi, ref_margins(oracle_mod, fleet, rate, lo, hi)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rate, lo, hi, want = rounds_case
    got = engine.load_margins(fleet, rate, lo, hi)
    assert same_bytes(got[0], want[0]) and same_bytes(got[1], want[1]) and np.array_equal(got[2], want[2])
    for name, g, w in zip(("at", "below", "above"), got[3:], want[3:]):
        assert_allocs_equal(g, w, f"D = {depth}: {name}")


@pytest.mark.gpu
def test_rates_at_and_next_to_a_replica_step(engine, oracle_mod):
    """r exactly at a step (lo = r) and one ulp below it (hi = the next float), found from the load intervals; a
    window bottom of 0 that the downward walk reaches, and rate 0 itself."""
    fleet = synth_fleet(6, 2, seed=17, keep_accelerator=True, zero_load_frac=0.0, tps_frac=0.0)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    count, _, start, _ = engine.load_intervals(fleet, np.zeros_like(x), (x * F32(3)).astype(np.float32), 64)
    assert (count >= 3).all()
    step = np.array([start[s, 2] for s in range(fleet.n_servers)], np.float32)
    rate = np.stack([step, below(step), np.zeros_like(x), np.full_like(x, TINY), (x * F32(0.01)).astype(np.float32)])
    lo = np.zeros_like(rate)
    hi = np.stack([(x * F32(3)).astype(np.float32)] * 4 + [x])
    lo_e, hi_e, flags, *_ = check_margins(engine, oracle_mod, fleet, rate, lo, hi, "at a step")
    assert same_bytes(lo_e[0], step) and same_bytes(hi_e[1], step)
    assert (flags[2] & MARGIN_LO_OPEN).all() and (lo_e[2] == 0).all()


@pytest.mark.gpu
def test_windows_that_are_one_point(engine, oracle_mod):
    fleet = mixed_fleet(12, 3, 41, False)
    rate = clean_levels(oracle_mod, fleet, 2, 13)
    lo, hi = rate.copy(), rate.copy()
    _, hi_e, flags, *_ = check_margins(engine, oracle_mod, fleet, rate, lo, hi, "lo = r = hi")
    assert ((flags & (MARGIN_LO_OPEN | MARGIN_HI_OPEN)) == (MARGIN_LO_OPEN | MARGIN_HI_OPEN)).all()


@pytest.mark.gpu
def test_tps_targets_out_tokens_zero_and_nil_winners(engine, oracle_mod):
    """A TPS target and out_tokens 0: the key does not read the load above rate 0.  No target, an unknown model and
    a missing profile: nil winners."""
    fleet = synth_fleet(8, 3, seed=19, zero_load_frac=0.0, tps_frac=0.0)
    fleet.srv_slo_tps[0] = 500
    fleet.srv_out_tokens[1] = 0
    fleet.srv_has_target[2] = 0
    fleet.srv_model[3] = -1
    fleet.perf_present[fleet.srv_model[4], :] = 0
    rate = clean_levels(oracle_mod, fleet, 2, 19)
    lo, hi = windows(fleet, rate, 19)
    lo[:, :2] = 0
    _, _, flags, at, *_ = check_margins(engine, oracle_mod, fleet, rate, lo, hi, "TPS, out 0, nil")
    assert (flags[:, 0:2] & MARGIN_HI_OPEN).all()
    assert (at["feasible"].reshape(2, -1)[:, 2:5] == 0).all()


@pytest.mark.gpu
def test_nan_and_huge_values_and_ties(engine, oracle_mod):
    fleet = mixed_fleet(12, 3, 43, False)
    fleet.srv_cur_cost[::2] = np.nan
    fleet.srv_cur_cost[1::4] = -F32_MAX
    fleet.acc_cost[2] = fleet.acc_cost[1]
    fleet.perf_alpha[:, 2] = fleet.perf_alpha[:, 1]
    for k in ("perf_beta", "perf_gamma", "perf_delta", "perf_acc_count"):
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]
    rate = clean_levels(oracle_mod, fleet, 2, 17)
    lo, hi = windows(fleet, rate, 17)
    check_margins(engine, oracle_mod, fleet, rate, lo, hi, "NaN / huge values and ties")


@pytest.mark.gpu
@pytest.mark.parametrize("n_acc", [32, 33])
def test_many_accelerators(engine, oracle_mod, n_acc):
    fleet = mixed_fleet(6, n_acc, 43, False)
    rate = clean_levels(oracle_mod, fleet, 2, 13)
    lo, hi = windows(fleet, rate, 13)
    check_margins(engine, oracle_mod, fleet, rate, lo, hi, f"A = {n_acc}")


@pytest.mark.gpu
def test_replica_overflow_truncates(engine, oracle_mod):
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
    rate = np.stack([x, x, x])
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    rate[0, s], lo[0, s], hi[0, s] = from_bits(hi_b - 3), from_bits(hi_b - 6), from_bits(hi_b + 6)  # above r
    rate[1, s], lo[1, s], hi[1, s] = over, from_bits(hi_b - 6), from_bits(hi_b + 6)                 # at r
    rate[2, s], lo[2, s], hi[2, s] = from_bits(hi_b + 2), from_bits(hi_b - 6), from_bits(hi_b + 6)  # below r
    lo_e, hi_e, flags, *_ = check_margins(engine, oracle_mod, fleet, rate, lo, hi, "overflow")
    assert hi_e[0, s] <= over and not flags[0, s] & MARGIN_LO_OPEN
    assert flags[1, s] == flags[2, s] == MARGIN_TRUNCATED and lo_e[1, s] == hi_e[1, s] == over


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
    check_margins(engine, oracle_mod, fleet, rate, lo, hi, "stored-vector fallback")


@pytest.mark.gpu
def test_tiny_rates_are_refused_as_the_intervals_refuse(engine, oracle_mod):
    fleet = synth_fleet(4, 2, seed=3, tps_frac=0.0, zero_load_frac=0.0)
    fleet.srv_min_replicas[:] = np.maximum(fleet.srv_min_replicas, 1)
    rate = np.array([[1e-41, TINY, 0, 2.0]], np.float32)
    lo = np.array([[0, TINY, 0, 0]], np.float32)
    hi = np.array([[1e-40, 1e-42, 1e-40, 5.0]], np.float32)
    check_margins(engine, oracle_mod, fleet, rate, lo, hi, "tiny rates")
    fleet.srv_min_replicas[0] = 0
    with pytest.raises(WvaError) as iv:
        engine.load_intervals(fleet, lo[0], hi[0], 16)
    with pytest.raises(WvaError) as mg:
        engine.load_margins(fleet, rate, lo, hi)
    assert iv.value.code == mg.value.code == WVA_ERR_UNSUPPORTED
    lo[0, 0] = F32(1e-40)  # the same window above the underflow is fine
    rate[0, 0] = F32(1e-40)
    engine.load_intervals(fleet, lo[0], hi[0], 16)
    engine.load_margins(fleet, rate, lo, hi)


@pytest.mark.gpu
def test_argument_errors_and_summary(engine, oracle_mod):
    from workload_variant_autoscaler_b200 import _abi
    fleet = mixed_fleet(6, 2, 61, False)
    L, h = engine._L, engine._h
    S = fleet.n_servers
    fc = fleet.as_c()
    rate = clean_levels(oracle_mod, fleet, 2, 3)
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    lo_o, hi_o, flags = (np.zeros(2 * S, np.float32), np.zeros(2 * S, np.float32), np.zeros(2 * S, np.uint8))
    recs = [Allocs(2 * S) for _ in range(3)]

    def call(rate_=rate, lo_=lo, hi_=hi, n=2, flags_=flags, out=True):
        oc = _abi.MarginsC(_abi.ptr(lo_o), _abi.ptr(hi_o), _abi.ptr(flags_) if flags_ is not None else None,
                           *(r.as_c() for r in recs))
        p = lambda a: _abi.ptr(np.ascontiguousarray(a, np.float32).reshape(-1)) if a is not None else None  # noqa
        return L.wva_load_margins(h, C.byref(fc), n, p(rate_), p(lo_), p(hi_), C.byref(oc) if out else None)

    assert call() == 0
    assert call(n=0) == 0
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
        engine.load_margins(fleet, rate, lo[:, :-1], hi)
    engine.solve(fleet)
    engine.summarize(fleet.n_types)
    engine.load_margins(fleet, rate, lo, hi)
    with pytest.raises(WvaError) as e:
        engine.summarize(fleet.n_types)
    assert e.value.code == WVA_ERR_STATE


# ---- GPU: against the other calls, without the oracle -------------------------------------------

def key_of(allocs, i):
    return tuple(u32_bits(getattr(allocs, k)[i]) if k in ("cost", "value", "max_rate") else int(getattr(allocs, k)[i])
                 for k in KEY_FIELDS)


@pytest.fixture(scope="module")
def big_case():
    fleet = synth_fleet(1500, 8, seed=42)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    rng = np.random.default_rng(5)
    rate = np.stack([x, (x * rng.lognormal(0, 0.3, x.size)).astype(np.float32)])
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    return fleet, rate, lo, hi


@pytest.mark.gpu
def test_configs3_shape_against_the_load_intervals(engine, big_case):
    fleet, rate, lo, hi = big_case
    S, M = fleet.n_servers, 256
    lo_m, hi_m, flags, at, below_r, above_r = engine.load_margins(fleet, rate, lo, hi)
    n_checked = 0
    for l in range(rate.shape[0]):
        count, trunc, start, rec = engine.load_intervals(fleet, lo[l], hi[l], M)
        for s in range(S):
            i = l * S + s
            if trunc[s] and count[s] == M:
                continue
            if flags[l, s] & MARGIN_TRUNCATED:
                assert trunc[s], s
                continue
            n = int(count[s])
            j = max(k for k in range(n) if start[s, k] <= rate[l, s])
            assert same_bytes(lo_m[l, s], lo[l, s] if j == 0 else start[s, j]), (l, s)
            assert bool(flags[l, s] & MARGIN_LO_OPEN) == (j == 0), (l, s)
            assert key_of(at, i) == key_of(rec, s * M + j), (l, s)
            if j + 1 < n:
                assert same_bytes(hi_m[l, s], start[s, j + 1]), (l, s)
                nx = s * M + j + 1
                for k in ALLOC_FIELDS:
                    assert same_bytes(getattr(above_r, k)[i:i + 1], getattr(rec, k)[nx:nx + 1]), (l, s)
            else:
                assert flags[l, s] & MARGIN_HI_OPEN and not trunc[s], (l, s)
            n_checked += 1
    assert n_checked > 0.9 * rate.size and (flags == 0).any()


@pytest.mark.gpu
def test_configs3_shape_against_the_load_grid(engine, big_case):
    """wva_load_grid at r, below lo, lo, hi - 1 ulp, hi and random interior rates reproduces the records and keys."""
    fleet, rate, lo, hi = big_case
    L, S = rate.shape
    lo_m, hi_m, flags, at, below_r, above_r = engine.load_margins(fleet, rate, lo, hi)
    rng = np.random.default_rng(7)
    for l in range(L):
        r = rate[l]
        closed_lo = (flags[l] & (MARGIN_LO_OPEN | MARGIN_TRUNCATED)) == 0
        closed_hi = (flags[l] & (MARGIN_HI_OPEN | MARGIN_TRUNCATED)) == 0
        ok = (flags[l] & MARGIN_TRUNCATED) == 0
        top = np.where(closed_hi, hi_m[l], np.nextafter(hi[l], INF)).astype(np.float32)
        pts = {"r": r, "below": np.where(closed_lo, below(lo_m[l]), r), "lo": np.where(ok, lo_m[l], r),
               "hi-": np.where(ok, below(top), r), "hi": np.where(closed_hi, hi_m[l], r)}
        for k in range(3):
            u = rng.uniform(lo_m[l], top).astype(np.float32)
            pts[f"in{k}"] = np.where(ok & (u >= lo_m[l]) & (u < top), u, r).astype(np.float32)
        rows = np.stack(list(pts.values())).astype(np.float32)
        _, win = engine.load_grid(fleet, rows)
        for j, name in enumerate(pts):
            for s in range(S):
                g = j * S + s
                if name in ("r", "below", "hi"):
                    ref = {"r": at, "below": below_r if closed_lo[s] else at,
                           "hi": above_r if closed_hi[s] else at}[name]
                    i = l * S + s
                    for k in ALLOC_FIELDS:
                        assert same_bytes(getattr(win, k)[g:g + 1], getattr(ref, k)[i:i + 1]), (name, s, k)
                else:
                    assert key_of(win, g) == key_of(at, l * S + s), (name, l, s)


@pytest.mark.gpu
def test_within_margins_means_the_same_solve(engine, big_case):
    fleet, rate, lo, hi = big_case
    lo_m, hi_m, flags, at, _, _ = engine.load_margins(fleet, rate[:1], lo[:1], hi[:1])
    rng = np.random.default_rng(11)
    new = (rate[:1] * rng.uniform(0.4, 2.2, rate[:1].shape)).astype(np.float32)
    inside = within_margins(lo_m, hi_m, flags, new, hi[:1])
    assert inside.any() and not inside.all()
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_arrival_rpm[:] = new[0]
    f.unlimited = True
    _, win = engine.solve(f, want_candidates=False)
    S = fleet.n_servers
    same = np.array([key_of(win, s) == key_of(at, s) for s in range(S)])
    assert same[inside[0]].all()


# ---- GPU: handle behaviour ----------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_launch_count_does_not_depend_on_levels_or_windows(engine, monkeypatch, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = synth_fleet(40, 4, seed=53, zero_load_frac=0.0)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    counts = []
    for L, wide in ((1, 1.01), (1, 100.0), (12, 2.0)):
        rate = np.stack([x] * L)
        n0 = engine.launch_count
        engine.load_margins(fleet, rate, (rate / F32(wide)).astype(np.float32), (rate * F32(wide)).astype(np.float32))
        counts.append(engine.launch_count - n0)
    assert counts[0] == counts[1] == counts[2], counts


@pytest.mark.gpu
def test_cache_interplay_on_one_handle(engine, oracle_mod):
    fleet = mixed_fleet(30, 3, 59, True)
    rate = clean_levels(oracle_mod, fleet, 3, 23)
    lo, hi = windows(fleet, rate, 23)
    fresh = Engine(0)
    try:
        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if isinstance(x, Allocs):
                    for k in ALLOC_FIELDS:
                        assert same_bytes(getattr(x, k), getattr(y, k)), f"{what}: {k}"
                elif x is not None:
                    assert same_bytes(x, y), what

        margins = lambda e: e.load_margins(fleet, rate, lo, hi)  # noqa: E731
        intervals = lambda e: e.load_intervals(fleet, lo[0], hi[0], 16)  # noqa: E731
        load_grid = lambda e: e.load_grid(fleet, rate, want_candidates=True)  # noqa: E731

        def resolve(e):
            e.upload(fleet)
            e.update_load(arrival_rpm=rate[1])
            return e.resolve(want_candidates=True)

        check(margins, "margins")
        check(intervals, "intervals after the margins")
        check(margins, "margins after the intervals")
        check(load_grid, "load grid after the margins")
        check(margins, "margins after the load grid")
        check(resolve, "resolve after the margins")
        check(margins, "margins after a resolve")
    finally:
        fresh.close()
