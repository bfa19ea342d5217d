"""The workload margins' reference side: the oracle composition that tests/test_gpu_workload_margins.py compares
wva_workload_margins and wva_workload_margin_trace with, and the rows and windows it judges them on.  It builds on the
load margins' composition in tests/levels.py (ref_margins): per row, ref_margins with one level on the fleet with the
row's rate and tokens; on a trace that fleet also carries c_t, advanced by apply_winners of each tick's `at`."""
import numpy as np

from tests.levels import F32, at_row, load_pair, ref_margins, workload_levels
from tests.util import ALLOC_FIELDS, assert_allocs_equal, same_bytes
from workload_variant_autoscaler_b200 import Allocs, synth_fleet

CALLS = {False: "workload_margins", True: "workload_margin_trace"}


def ref_workload_margins(oracle_mod, fleet, rows, lo, hi, trace):
    """(lo (L, S), hi (L, S), flags (L, S), at, below, above, the row fleets): the call's contract.  rows holds
    arrival_rpm, in_tokens and out_tokens ([L, S]; a token list of None is the fleet's own column).  Row l is
    ref_margins with one level on f_l = at_row of the fleet (on a trace: of the chained fleet, whose current
    allocation is c_t)."""
    rate = rows["arrival_rpm"]
    L, S = rate.shape
    out, fleets, cur = [], [], fleet
    for t in range(L):
        f = at_row(cur, rows, t)
        r = ref_margins(oracle_mod, f, rate[t:t + 1], lo[t:t + 1], hi[t:t + 1])
        out.append(r)
        fleets.append(f)
        if trace:
            cur = cur.apply_winners(r[3])
    if not out:
        z, empty = np.zeros((0, S), np.float32), np.zeros(0, oracle_mod.ALLOC_DTYPE)
        return z, z.copy(), np.zeros((0, S), np.uint8), empty, empty, empty, fleets
    return tuple(np.concatenate([r[k] for r in out]) for k in range(6)) + (fleets,)


def check_workload_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, what, ref=None):
    """Engine.workload_margins / workload_margin_trace against ref_workload_margins (or `ref`, its result), bit for
    bit."""
    want = ref_workload_margins(oracle_mod, fleet, rows, lo, hi, trace) if ref is None else ref
    got = getattr(engine, CALLS[trace])(fleet, rows["arrival_rpm"], rows.get("in_tokens"), rows.get("out_tokens"),
                                        lo, hi)
    for name, g, w in zip(("lo", "hi"), got[:2], want[:2]):
        assert same_bytes(g, w), f"{what}: {name}: got {g[g.view(np.uint32) != w.view(np.uint32)]}"
    assert np.array_equal(got[2], want[2]), f"{what}: flags {got[2]} vs {want[2]}"
    for name, g, w in zip(("at", "below", "above"), got[3:6], want[3:6]):
        assert_allocs_equal(g, w, f"{what}: {name}")
    return want


def first_step(oracle_mod, fleet, s):
    """60 * rateStar of server s's fastest load pair at its own tokens (None: no load pair)."""
    steps = [60.0 * float(p[0]) for p in (load_pair(oracle_mod, fleet, s, a) for a in range(fleet.n_acc)) if p]
    return min(steps) if steps else None


def workload_margin_rows(oracle_mod, fleet, L, seed, special=True):
    """{"arrival_rpm", "in_tokens", "out_tokens"} [L, S] the workload margins accept: workload_levels' rows with the
    negative and infinite rates at 7.5 and out_tokens 1 (a 2^21 queue, refused) at the fleet's own, each rate scaled
    per (row, server) so that the server's own load sits at 1.5 times the first replica step of the row's tokens and
    capped at 20 steps (margin_levels scales to the fleet's own tokens, which a 1.5x out_tokens row moves)."""
    rpm, in_tok, out_tok = workload_levels(fleet, L, seed, special)
    out_tok = np.where(out_tok == 1, fleet.srv_out_tokens[None, :], out_tok).astype(np.int32)
    rows = rpm.astype(np.float64)
    rows[~np.isfinite(rows) | (rows < 0)] = 7.5
    for l in range(L):
        f = at_row(fleet, {"in_tokens": in_tok, "out_tokens": out_tok}, l)
        for s in range(fleet.n_servers):
            step = first_step(oracle_mod, f, s)
            if step:
                rows[l, s] = min(rows[l, s] * (1.5 * step / max(float(fleet.srv_arrival_rpm[s]), 1.0)), 20 * step)
    return {"arrival_rpm": rows.astype(np.float32), "in_tokens": in_tok, "out_tokens": out_tok}


def own_tokens(fleet, rate):
    """The load rows with the fleet's own tokens at every row."""
    shape = rate.shape
    return {"arrival_rpm": rate,
            "in_tokens": np.ascontiguousarray(np.broadcast_to(fleet.srv_in_tokens, shape), np.int32),
            "out_tokens": np.ascontiguousarray(np.broadcast_to(fleet.srv_out_tokens, shape), np.int32)}


def unpinned_case():
    """keepAccelerator on, min_replicas 0 and c_0 on each server's dearest accelerator: row 0 at rate 0 is won by the
    zero-load record with accelerator "", which lifts the mask, so that the load rows after it are won by cheaper
    accelerators (pairs a phase 1 that honoured keepAccelerator against c_0 would not have sized).  The tokens move
    from row to row."""
    fleet = synth_fleet(8, 3, seed=23, keep_accelerator=True, zero_load_frac=0.0, tps_frac=0.0)
    fleet.srv_min_replicas[:] = 0
    fleet.accel_penalty_factor = 0.0
    a = int(np.argmax(fleet.acc_cost))
    fleet.srv_cur_acc[:] = a
    fleet.srv_cur_replicas[:] = 1
    fleet.srv_cur_cost[:] = (fleet.acc_cost[a] * fleet.perf_acc_count[fleet.srv_model, a]).astype(np.float32)
    x = np.maximum(fleet.srv_arrival_rpm, 100.0).astype(np.float32)
    scale = np.array([0, 1, 2.5, 0, 0.7, 0, 4], np.float32)
    rows = own_tokens(fleet, (scale[:, None] * x[None, :]).astype(np.float32))
    rows["in_tokens"] = (rows["in_tokens"] * np.array([1, 2, 0.5, 1, 2, 1, 0.5])[:, None]).astype(np.int32)
    rows["out_tokens"] = (rows["out_tokens"] * np.array([1, 1.5, 0.75, 1, 1.5, 1, 0.75])[:, None]).astype(np.int32)
    rate = rows["arrival_rpm"]
    return fleet, rows, (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)


def part(allocs, t, S):
    """Block t (records t*S .. t*S + S - 1) of an Allocs."""
    x = Allocs(S)
    for f in ALLOC_FIELDS:
        getattr(x, f)[:] = getattr(allocs, f)[t * S:(t + 1) * S]
    return x


def block(result, t, S):
    """Block t of a margins result: (lo, hi, flags, at, below, above)."""
    lo, hi, flags, *recs = result
    return (lo[t], hi[t], flags[t]) + tuple(part(r, t, S) for r in recs)


def assert_same(x, y, what):
    """Two margins results (or blocks), byte for byte."""
    for k, (a, b) in enumerate(zip(x, y)):
        if isinstance(a, Allocs):
            for f in ALLOC_FIELDS:
                assert same_bytes(getattr(a, f), getattr(b, f)), f"{what}: record {k - 3}.{f}"
        else:
            assert same_bytes(a, b), f"{what}: column {k}"
