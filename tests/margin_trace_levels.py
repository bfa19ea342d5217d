"""The load margin trace's reference side: the oracle composition that tests/test_gpu_load_margin_trace.py compares
wva_load_margin_trace with, and the rates and windows it judges the call on.  It builds on the load margins'
composition in tests/levels.py (ref_margins) and advances the current allocation tick by tick as ref_trace does."""
import numpy as np

from tests.levels import F32, at_row, load_levels, load_pair, ref_margins
from tests.util import assert_allocs_equal, same_bytes


def ref_margin_trace(oracle_mod, fleet, rate, lo, hi):
    """(lo (L, S), hi (L, S), flags (L, S), at, below, above, the tick fleets): wva_load_margin_trace's contract.
    Per tick t, ref_margins with one level on f_t = at_row of the chained fleet, whose current allocation is c_t;
    c_{t+1} is apply_winners of tick t's `at` records, as ref_price_rows(trace=True) advances."""
    L, S = rate.shape
    out, fleets, cur = [], [], fleet
    for t in range(L):
        f = at_row(cur, {"arrival_rpm": rate}, t)
        r = ref_margins(oracle_mod, f, rate[t:t + 1], lo[t:t + 1], hi[t:t + 1])
        out.append(r)
        fleets.append(f)
        cur = cur.apply_winners(r[3])
    if not out:
        z, empty = np.zeros((0, S), np.float32), np.zeros(0, oracle_mod.ALLOC_DTYPE)
        return z, z.copy(), np.zeros((0, S), np.uint8), empty, empty, empty, fleets
    return tuple(np.concatenate([r[k] for r in out]) for k in range(6)) + (fleets,)


def check_margin_trace(engine, oracle_mod, fleet, rate, lo, hi, what, ref=None):
    """Engine.load_margin_trace against ref_margin_trace (or `ref`, its result), bit for bit."""
    want = ref_margin_trace(oracle_mod, fleet, rate, lo, hi) if ref is None else ref
    got = engine.load_margin_trace(fleet, rate, lo, hi)
    for name, g, w in zip(("lo", "hi"), got[:2], want[:2]):
        assert same_bytes(g, w), f"{what}: {name}: got {g[g.view(np.uint32) != w.view(np.uint32)]}"
    assert np.array_equal(got[2], want[2]), f"{what}: flags {got[2]} vs {want[2]}"
    for name, g, w in zip(("at", "below", "above"), got[3:6], want[3:6]):
        assert_allocs_equal(g, w, f"{what}: {name}")
    return want


def margin_levels(oracle_mod, fleet, L, seed):
    """[L, S] rates the margins accept: load_levels' rows with the negative and infinite rates at 7.5, scaled per
    server so that its own load sits at 1.5 times its first replica step (60 * rateStar of its fastest load pair) and
    capped at 20 steps, so that each window holds a few steps and the composition's step walk stays short (the rows
    of the load margins' tests)."""
    rows = load_levels(fleet, L, seed).astype(np.float64)
    rows[~np.isfinite(rows) | (rows < 0)] = 7.5
    for s in range(fleet.n_servers):
        steps = [60.0 * float(p[0]) for p in (load_pair(oracle_mod, fleet, s, a) for a in range(fleet.n_acc)) if p]
        if steps:
            step = min(steps)
            rows[:, s] = np.minimum(rows[:, s] * (1.5 * step / max(float(fleet.srv_arrival_rpm[s]), 1.0)), 20 * step)
    return rows.astype(np.float32)


def margin_windows(fleet, rate, seed):
    """[0.5x, 2x] of each rate, with the window bottom at 0 for some and lo = r = hi for others.  A bottom of 0 is
    kept off min_replicas-0 servers, whose pairs have 0 replicas just above it (refused, as the intervals refuse)."""
    rng = np.random.default_rng(seed)
    r = np.asarray(rate, np.float32)
    lo, hi = (r * F32(0.5)).astype(np.float32), (r * F32(2)).astype(np.float32)
    pick = rng.random(r.shape)
    lo[(pick < 0.15) & (fleet.srv_min_replicas > 0)[None, :]] = 0
    lo[pick > 0.92] = hi[pick > 0.92] = r[pick > 0.92]
    return lo, hi
