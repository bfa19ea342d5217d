"""The profile margins' reference side: the rows and windows tests/test_gpu_profile_margins.py judges
wva_profile_margins and wva_profile_margin_trace on, and the composition it compares them with.  The composition is
the workload margins' (workload_margin_levels.ref_workload_margins): its at_row writes every row list, acc_cost and
the perf_* columns included, and on a trace it advances c_t with apply_winners of each tick's `at`, whose cost is at
that tick's prices."""
import numpy as np

from tests.levels import COLUMNS, F32, at_row, load_levels, profile_rows
from tests.margin_trace_levels import margin_windows
from tests.util import F32_MAX, assert_allocs_equal, same_bytes
from tests.workload_margin_levels import first_step, ref_workload_margins

CALLS = {False: "profile_margins", True: "profile_margin_trace"}
LOAD = ("arrival_rpm", "in_tokens", "out_tokens")


def ref_profile_margins(oracle_mod, fleet, rows, lo, hi, trace):
    """(lo (L, S), hi (L, S), flags (L, S), at, below, above, the row fleets): the call's contract, row l being
    ref_margins with one level on the fleet with every list of rows at row l (on a trace also with c_t)."""
    return ref_workload_margins(oracle_mod, fleet, rows, lo, hi, trace)


def split(rows):
    """(the load lists, the profile columns) of rows, by keyword."""
    return ({k: rows.get(k) for k in LOAD}, {k: v for k, v in rows.items() if k in COLUMNS})


def run(engine, trace, fleet, rows, lo, hi):
    load, prof = split(rows)
    return getattr(engine, CALLS[trace])(fleet, load["arrival_rpm"], load["in_tokens"], load["out_tokens"], lo, hi,
                                         **prof)


def check_profile_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, what, ref=None):
    """Engine.profile_margins / profile_margin_trace against ref_profile_margins (or `ref`, its result), bit for
    bit."""
    want = ref_profile_margins(oracle_mod, fleet, rows, lo, hi, trace) if ref is None else ref
    got = run(engine, trace, fleet, rows, lo, hi)
    for name, g, w in zip(("lo", "hi"), got[:2], want[:2]):
        assert same_bytes(g, w), f"{what}: {name}: got {g[g.view(np.uint32) != w.view(np.uint32)]}"
    assert np.array_equal(got[2], want[2]), f"{what}: flags {got[2]} vs {want[2]}"
    for name, g, w in zip(("at", "below", "above"), got[3:6], want[3:6]):
        assert_allocs_equal(g, w, f"{what}: {name}")
    return want


def scale_to_rows(oracle_mod, fleet, rows, rate):
    """rate [L, S] with the negative and infinite rates at 7.5, each scaled per (row, server) so that the server's own
    load sits at 1.5 times the first replica step of the row's own fleet (its tokens, prices and profiles: a beta or a
    perf_max_batch change moves that step) and capped at 20 steps."""
    out = rate.astype(np.float64)
    out[~np.isfinite(out) | (out < 0)] = 7.5
    for l in range(out.shape[0]):
        f = at_row(fleet, {k: v for k, v in rows.items() if k != "arrival_rpm"}, l)
        for s in range(fleet.n_servers):
            step = first_step(oracle_mod, f, s)
            if step:
                out[l, s] = min(out[l, s] * (1.5 * step / max(float(fleet.srv_arrival_rpm[s]), 1.0)), 20 * step)
    return out.astype(np.float32)


def own_profile(fleet, L):
    """Every profile column of the fleet, repeated over L rows."""
    return {k: np.repeat(getattr(fleet, k)[None], L, axis=0).copy() for k in COLUMNS}


def edit_rows(fleet, L, kind, seed):
    """Profile rows of one kind over L >= 4 rows (the columns a kind does not name are left out):
    - "prices": every price x 0.5 .. x 1.25;
    - "edge_prices": price 0, NaN, +Inf and MaxFloat32 on accelerator 0 at rows 0 .. 3;
    - "acc_count": AccCount -3, 0 and 4 at rows 1 .. 3;
    - "present": the last accelerator's perf_present toggled at row 1;
    - "beta": beta x 2 and gamma x 0.5 at rows 1 and 3 (rateStar moves);
    - "batch": perf_max_batch / 4 at row 1 and perf_at_tokens x 2 at row 2 (N moves);
    - "mixed": profile_rows."""
    rng = np.random.default_rng(seed)
    own = own_profile(fleet, L)
    if kind == "mixed":
        return profile_rows(fleet, L, seed)
    if kind == "prices":
        return {"acc_cost": (own["acc_cost"] * rng.choice([0.5, 0.8, 1.0, 1.25], own["acc_cost"].shape)).astype(F32)}
    if kind == "edge_prices":
        c = own["acc_cost"]
        c[:4, 0] = (0.0, np.nan, np.inf, F32_MAX)
        return {"acc_cost": c}
    if kind == "acc_count":
        c = own["perf_acc_count"]
        c[1], c[2], c[3] = -3, 0, 4
        return {"perf_acc_count": c}
    if kind == "present":
        p = own["perf_present"]
        p[1, :, -1] ^= 1
        return {"perf_present": p}
    if kind == "beta":
        own["perf_beta"][[1, 3]] *= F32(2)
        own["perf_gamma"][[1, 3]] *= F32(0.5)
        return {"perf_beta": own["perf_beta"], "perf_gamma": own["perf_gamma"]}
    if kind == "batch":
        own["perf_max_batch"][1] = np.maximum(own["perf_max_batch"][1] // 4, 1)
        own["perf_at_tokens"][2] *= 2
        return {"perf_max_batch": own["perf_max_batch"], "perf_at_tokens": own["perf_at_tokens"]}
    raise ValueError(kind)


def profile_margin_case(oracle_mod, fleet, L, kind, seed, tokens=True):
    """(rows, lo, hi): edit_rows of `kind` plus load rows (load_levels, and with `tokens` out_tokens x 1 or 1.5), the
    rates scaled to each row's own fleet, windows from margin_windows."""
    rows = edit_rows(fleet, L, kind, seed)
    rng = np.random.default_rng(seed + 1)
    rows["in_tokens"] = None
    rows["out_tokens"] = None
    if tokens:
        rows["out_tokens"] = (fleet.srv_out_tokens[None, :] * rng.choice([1.0, 1.0, 1.5], (L, fleet.n_servers))
                              ).astype(np.int32)
    rows["arrival_rpm"] = scale_to_rows(oracle_mod, fleet, rows, load_levels(fleet, L, seed))
    lo, hi = margin_windows(fleet, rows["arrival_rpm"], seed)
    return rows, lo, hi
