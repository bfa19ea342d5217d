"""The SLO margins' reference side: the rows and windows tests/test_gpu_slo_margins.py judges wva_slo_margins and
wva_slo_margin_trace on, and the composition it compares them with.  The composition is the workload margins'
(workload_margin_levels.ref_workload_margins): its at_row writes every row list, the slo_* targets included, and on a
trace it advances c_t with apply_winners of each tick's `at`."""
import numpy as np

from tests.levels import F32, LOAD, SLO, TARGETS, TPS_TARGETS, day_slo_rows, load_levels, slo_levels
from tests.margin_trace_levels import margin_windows
from tests.profile_margin_levels import scale_to_rows
from tests.util import F32_MAX, assert_allocs_equal, same_bytes
from tests.workload_margin_levels import ref_workload_margins

CALLS = {False: "slo_margins", True: "slo_margin_trace"}
KINDS = ("schedule", "itl", "ttft", "tps", "edges", "mixed")


def ref_slo_margins(oracle_mod, fleet, rows, lo, hi, trace):
    """(lo (L, S), hi (L, S), flags (L, S), at, below, above, the row fleets): the call's contract, row l being
    ref_margins with one level on the fleet with every list of rows at row l (on a trace also with c_t)."""
    return ref_workload_margins(oracle_mod, fleet, rows, lo, hi, trace)


def split(rows):
    """(the load lists, the target lists) of rows, by keyword."""
    return {k: rows.get(k) for k in LOAD}, {k: rows.get(k) for k in SLO}


def run(engine, trace, fleet, rows, lo, hi):
    load, slo = split(rows)
    return getattr(engine, CALLS[trace])(fleet, load["arrival_rpm"], load["in_tokens"], load["out_tokens"], lo, hi,
                                         **slo)


def check_slo_margins(engine, oracle_mod, fleet, rows, lo, hi, trace, what, ref=None):
    """Engine.slo_margins / slo_margin_trace against ref_slo_margins (or `ref`, its result), bit for bit."""
    want = ref_slo_margins(oracle_mod, fleet, rows, lo, hi, trace) if ref is None else ref
    got = run(engine, trace, fleet, rows, lo, hi)
    for name, g, w in zip(("lo", "hi"), got[:2], want[:2]):
        assert same_bytes(g, w), f"{what}: {name}: got {g[g.view(np.uint32) != w.view(np.uint32)]}"
    assert np.array_equal(got[2], want[2]), f"{what}: flags {got[2]} vs {want[2]}"
    for name, g, w in zip(("at", "below", "above"), got[3:6], want[3:6]):
        assert_allocs_equal(g, w, f"{what}: {name}")
    return want


def own_targets(fleet, L):
    """The fleet's own targets, repeated over L rows."""
    return {k: np.repeat(getattr(fleet, "srv_" + k)[None], L, axis=0).astype(F32) for k in SLO}


def target_rows(fleet, L, kind, seed):
    """Target rows of one kind over L >= 4 rows (the targets a kind does not move are left out):
    - "schedule": ITL x 0.75 in the middle third of the rows, TTFT x 1.5 in the first quarter (day_slo_rows);
    - "itl": ITL alone x 0.5 .. x 2 per (row, server);
    - "ttft": TTFT alone x 0.5 .. x 2 per (row, server);
    - "tps": a TPS target on every third server (2e4 x 0.5 .. x 2) and 0 elsewhere, with TPS_TARGETS' 0, -0 and -1
      scattered over it (+Inf and MaxFloat32 overflow the replica count; test_gpu_slo_margins'
      test_nan_tps_refuses_only_under_a_window judges them against wva_load_margins on the row's fleet);
    - "edges": ITL and TTFT with the TARGETS edges scattered over them, the fleet's own TPS;
    - "mixed": slo_levels without edge values, all three moving."""
    rng = np.random.default_rng(seed)
    S = fleet.n_servers
    own = own_targets(fleet, L)
    factor = lambda: rng.choice(np.array([0.5, 0.75, 1.0, 1.5, 2.0], F32), (L, S))  # noqa: E731
    if kind == "schedule":
        rows = day_slo_rows(fleet, L, L)
        return {"slo_itl": rows["slo_itl"], "slo_ttft": rows["slo_ttft"]}
    if kind == "itl":
        return {"slo_itl": (own["slo_itl"] * factor()).astype(F32)}
    if kind == "ttft":
        return {"slo_ttft": (own["slo_ttft"] * factor()).astype(F32)}
    if kind == "tps":
        tps = np.zeros((L, S), F32)
        tps[:, ::3] = (F32(2e4) * factor()[:, ::3]).astype(F32)
        for k, v in enumerate(v for v in TPS_TARGETS if np.isfinite(v) and v < F32_MAX):
            tps[k % L, 1 + k::7] = v
        return {"slo_tps": tps}
    if kind == "edges":
        itl, ttft = own["slo_itl"], own["slo_ttft"]
        for k, v in enumerate(TARGETS):
            itl[k % L, k % S::3 + k] = v
            ttft[(k + 1) % L, (k + 1) % S::4 + k] = v
        return {"slo_itl": itl, "slo_ttft": ttft}
    if kind == "mixed":
        return dict(zip(SLO, slo_levels(fleet, L, seed, special=False)))
    raise ValueError(kind)


def slo_margin_case(oracle_mod, fleet, L, kind, seed, tokens=True):
    """(rows, lo, hi): target_rows of `kind` plus load rows (load_levels, and with `tokens` out_tokens x 1 or 1.5), the
    rates scaled to each row's own fleet (its tokens and targets: an ITL change moves rateStar), windows from
    margin_windows."""
    rows = target_rows(fleet, L, kind, seed)
    rng = np.random.default_rng(seed + 1)
    rows["in_tokens"] = None
    rows["out_tokens"] = None
    if tokens:
        rows["out_tokens"] = (fleet.srv_out_tokens[None, :] * rng.choice([1.0, 1.0, 1.5], (L, fleet.n_servers))
                              ).astype(np.int32)
    rows["arrival_rpm"] = scale_to_rows(oracle_mod, fleet, rows, load_levels(fleet, L, seed))
    lo, hi = margin_windows(fleet, rows["arrival_rpm"], seed)
    return rows, lo, hi
