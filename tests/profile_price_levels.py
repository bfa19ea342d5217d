"""The profile price thresholds' reference side: the rows tests/test_gpu_profile_price_levels.py judges
wva_profile_price_threshold_grid and wva_profile_price_threshold_trace on, and the checks it compares them with.
The composition is tests.levels.ref_price_rows: its at_row writes every row list, acc_cost and the perf_* columns
included, and on a trace it advances c_t with apply_winners of each tick's winners, whose cost is at that tick's
prices."""
import numpy as np

from tests.levels import F32, load_levels, ref_price_rows, workload_levels
from tests.profile_margin_levels import edit_rows, split
from tests.util import assert_allocs_equal, assert_f32_bits_equal

CALLS = {False: "profile_price_threshold_grid", True: "profile_price_threshold_trace"}
KINDS = ("prices", "edge_prices", "acc_count", "present", "beta", "batch", "mixed")


def price_case(fleet, L, kind, seed, tokens=False):
    """edit_rows of `kind` plus load rows: load_levels' rates, or with `tokens` workload_levels' rates and tokens."""
    rows = edit_rows(fleet, L, kind, seed)
    if tokens:
        rows.update(zip(("arrival_rpm", "in_tokens", "out_tokens"), workload_levels(fleet, L, seed + 1)))
    else:
        rows["arrival_rpm"] = load_levels(fleet, L, seed + 1)
    return rows


def run(engine, trace, fleet, rows, want_candidates=False):
    """Engine.profile_price_threshold_grid / _trace on rows (load lists and profile columns by keyword)."""
    load, prof = split(rows)
    return getattr(engine, CALLS[trace])(fleet, load["arrival_rpm"], load["in_tokens"], load["out_tokens"],
                                         want_candidates=want_candidates, **prof)


def not_nil(fleet, s, a):
    """The pairs wva_analyze does not class nil: those CreateAllocation sizes and the zero-load candidates."""
    if fleet.srv_keep_acc[s] and fleet.srv_cur_acc[s] != -1 and fleet.srv_cur_acc[s] != a:
        return False
    m = int(fleet.srv_model[s])
    if fleet.srv_arrival_rpm[s] < 0 or fleet.srv_in_tokens[s] < 0 or fleet.srv_out_tokens[s] < 0:
        return False
    return 0 <= m < fleet.n_models and bool(fleet.perf_present[m, a]) and bool(fleet.srv_has_target[s])


def cost_refused(fleets):
    """(row, server) of the first row fleet with a NaN or infinite current cost on a server with a pair not classed
    nil, None without one: where wva_price_thresholds refuses a row's fleet."""
    for l, f in enumerate(fleets):
        for s in range(f.n_servers):
            if not np.isfinite(f.srv_cur_cost[s]) and any(not_nil(f, s, a) for a in range(f.n_acc)):
                return l, s
    return None


def check_profile_price_rows(engine, oracle_mod, fleet, rows, trace, what, ref=None):
    """The call against ref_price_rows (or `ref`, its result), bit for bit: (threshold, candidates, winners, the
    row fleets) of the reference."""
    th_o, above_o, cand_o, win_o, fleets = ref if ref is not None else ref_price_rows(oracle_mod, fleet, rows, trace)
    th_g, above_g, cand_g, win_g = run(engine, trace, fleet, rows, want_candidates=True)
    assert th_g.dtype == F32
    assert_f32_bits_equal(th_g.reshape(-1), th_o.reshape(-1), f"{what}: threshold")
    assert_allocs_equal(above_g, above_o, f"{what}: above")
    assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
    assert_allocs_equal(win_g, win_o, f"{what}: winners")
    return th_o, cand_o, win_o, fleets
