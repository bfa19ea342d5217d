"""wva_slo_margins and wva_slo_margin_trace in five cases: synth_fleet(10000, 8, seed=42) (the configs[3] shape) x the
24 rows of workload_margins_bench.py (rates and out_tokens x {0.75, 1, 1.5} per (row, server)) under
slo_trace_bench.py's target schedule (each server's own ITL x 0.75 in rows 8-19, its own TTFT x 1.5 in rows 0-5, its
own TPS), grid and trace, each with keepAccelerator off and in WVA's configuration; and synth_fleet(256, 8) x 1,440
ticks (a day of minutes: workload_margins_bench.py's diurnal rate and token draw, the ITL target x 0.75 in the middle
third of the day and the TTFT target x 1.5 in its first quarter), trace.  Windows are [0.5x, 2x] of each row.

Prints one JSON line with the GPU's name, power limit and max SM clock, and per case: the median device / kernel /
host time over the repeated calls, the launches per call, the keys sized against L * S, the searches phase 1 runs
against those wva_slo_trace runs on the same rows, each kernel's own device time (torch.profiler, in a separate call:
margin_kernel, margin_chain and phase 1's sizing kernels), the workload-margin call on the same load rows at the
fleet's own targets (what the target rows cost), and the alternative a caller has without the call: one
wva_load_margins per row on the fleet with the row's tokens and targets (for the trace, after wva_slo_trace, on the
fleet advanced by Fleet.apply_winners), timed (device time summed over the calls, host wall time of the whole loop),
with a per-row byte comparison of every column.  Needs a GPU; run from the repository root.  --dry-run builds the
cases' rows and windows and prints their shapes without touching a GPU."""
import argparse
import json
import sys
import time

import numpy as np

sys.path.insert(0, ".")
sys.path.insert(0, "tools")
from profile_margins_bench import kernels_ms  # noqa: E402
from slo_trace_bench import slo_schedule  # noqa: E402
from workload_margins_bench import (FIELDS, gpu_label, rows_24, rows_day, same, timed,  # noqa: E402
                                    windows, wva_configuration)
from workload_variant_autoscaler_b200 import synth_fleet  # noqa: E402

F32 = np.float32
SLO = ("slo_itl", "slo_ttft", "slo_tps")


def day_schedule(fleet, L):
    """The day of minutes' targets: ITL x 0.75 in the middle third of the day, TTFT x 1.5 in its first quarter."""
    minute = np.arange(L) % 1440
    itl, ttft, tps = (np.repeat(getattr(fleet, "srv_" + k)[None, :], L, 0).astype(F32) for k in SLO)
    itl[(minute >= 480) & (minute < 960)] *= F32(0.75)
    ttft[minute < 360] *= F32(1.5)
    return itl, ttft, tps


def cases(S, A, L, day_S, day_L):
    off = synth_fleet(S, A, seed=42)
    wva = wva_configuration(synth_fleet(S, A, seed=42), 42)
    load = rows_24(off, L, 7)
    slo = dict(zip(SLO, slo_schedule(off, L)))
    small = synth_fleet(day_S, A, seed=42)
    out = {}
    for trace in (False, True):
        kind = "trace" if trace else "grid"
        out[f"{S}x{A}x{L}_{kind}_keep_off"] = (off, load, slo, trace)
        out[f"{S}x{A}x{L}_{kind}_wva_configuration"] = (wva, load, slo, trace)
    out[f"{day_S}x{A}x{day_L}_trace_day_of_minutes"] = (small, rows_day(small, day_L, 3),
                                                        dict(zip(SLO, day_schedule(small, day_L))), True)
    return out


def pairs_of(fleet, trace):
    """[S] the load pairs phase 1 sizes per key of a server: its present accelerators, only the current one where
    keepAccelerator masks the rest (on a trace on the pinned servers only)."""
    cur, keep = fleet.srv_cur_acc, fleet.srv_keep_acc != 0
    keep = keep & (cur != -1) & (((cur == -2) | (fleet.srv_min_replicas != 0)) if trace else True)
    prof = fleet.perf_present[np.maximum(fleet.srv_model, 0)] != 0
    own = np.arange(fleet.n_acc)[None, :] == cur[:, None]
    ok = (fleet.srv_model >= 0) & (fleet.srv_has_target != 0)
    return (prof & ok[:, None] & np.where(keep[:, None], own, True)).sum(1)


def n_keys_and_searches(fleet, hi, in_tok, out_tok, slo, trace):
    """(keys, searches the key rule runs, searches wva_slo_trace runs): keys are the distinct (server, in, out, target
    bits) over the rows whose window top is above 0 and whose tokens class a pair as a load; each key's pairs run
    Size's TTFT and ITL searches where the target is positive (none with a negative target).  wva_slo_trace runs each
    distinct (server, in, out, search, target bits) once per pair."""
    L, S = hi.shape
    use = (hi > 0) & (in_tok >= 0) & (out_tok >= 1)
    n_pairs = pairs_of(fleet, trace)
    bits = [slo[k].astype(F32).view(np.uint32) for k in SLO]
    keys, run, trace_run = 0, 0, 0
    for s in range(S):
        rows = np.nonzero(use[:, s])[0]
        k = {(int(in_tok[t, s]), int(out_tok[t, s]), *(int(b[t, s]) for b in bits)) for t in rows}
        keys += len(k)
        if not n_pairs[s]:
            continue
        srch = set()
        for ki, ko, bi, bt, bp in k:
            x = np.array([bi, bt, bp], np.uint32).view(F32)
            if (x < 0).any():
                continue
            for w, y, yb in ((0, x[1], bt), (1, x[0], bi)):
                if y > 0:
                    run += int(n_pairs[s])
                    srch.add((ki, ko, w, yb))
        trace_run += len(srch) * int(n_pairs[s])
    return keys, run, trace_run


def at_row(fleet, in_tok, out_tok, slo, l):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_in_tokens[:] = in_tok[l]
    f.srv_out_tokens[:] = out_tok[l]
    for k, v in slo.items():
        getattr(f, "srv_" + k)[:] = v[l]
    return f


def alternative(e, fleet, load, slo, lo, hi, trace, got):
    """One load_margins per row on the fleet with the row's columns (on a trace after slo_trace, along the
    apply_winners chain): (timing, rows differing, whether the `at` blocks are the SLO trace's winners)."""
    rate, in_tok, out_tok = load
    L, S = rate.shape
    t0 = time.perf_counter()
    dev = 0.0
    if trace:
        _, win = e.slo_trace(fleet, rate, in_tok, out_tok, **slo)
        dev = e.last_device_ms
    cur, differ = fleet, 0
    for t in range(L):
        one = e.load_margins(at_row(cur, in_tok, out_tok, slo, t), rate[t:t + 1], lo[t:t + 1], hi[t:t + 1])
        dev += e.last_device_ms
        if trace:
            cur = cur.apply_winners(one[3])
        sl = slice(t * S, (t + 1) * S)
        ok = same(one[0][0], got[0][t]) and same(one[1][0], got[1][t]) and same(one[2][0], got[2][t])
        ok = ok and all(same(getattr(x, f), getattr(y, f)[sl]) for x, y in zip(one[3:], got[3:]) for f in FIELDS)
        differ += not ok
    wall = (time.perf_counter() - t0) * 1e3
    res = {"device_ms_total": dev, "host_wall_ms": wall, "rows_differing": differ}
    if trace:
        res["at_blocks_equal_slo_trace_winners"] = all(same(getattr(got[3], f), getattr(win, f)) for f in FIELDS)
    return res


def run_case(e, fleet, load, slo, trace, reps):
    rate, in_tok, out_tok = load
    lo, hi = windows(rate)
    call = e.slo_margin_trace if trace else e.slo_margins
    go = lambda: call(fleet, rate, in_tok, out_tok, lo, hi, **slo)  # noqa: E731
    got, t = timed(go, reps, e)
    res = dict(t)
    res["keys"], res["searches"], res["slo_trace_searches"] = n_keys_and_searches(fleet, hi, in_tok, out_tok, slo,
                                                                                  trace)
    res["rows_x_servers"] = int(rate.size)
    res["kernels_ms"] = kernels_ms(go)
    own = e.workload_margin_trace if trace else e.workload_margins
    _, tw = timed(lambda: own(fleet, rate, in_tok, out_tok, lo, hi), reps, e)
    tw["kernels_ms"] = kernels_ms(lambda: own(fleet, rate, in_tok, out_tok, lo, hi))
    res["own_targets_workload_margin_call"] = tw
    res["alternative"] = alternative(e, fleet, load, slo, lo, hi, trace, got)
    return res


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--servers", type=int, default=10000)
    p.add_argument("--acc", type=int, default=8)
    p.add_argument("--rows", type=int, default=24)
    p.add_argument("--day-servers", type=int, default=256)
    p.add_argument("--day-ticks", type=int, default=1440)
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--dry-run", action="store_true", help="build the cases and print their shapes; no GPU")
    a = p.parse_args(argv)
    if min(a.servers, a.acc, a.rows, a.day_servers, a.day_ticks, a.reps) < 1:
        p.error("every size must be at least 1")
    cs = cases(a.servers, a.acc, a.rows, a.day_servers, a.day_ticks)
    if a.dry_run:
        shapes = {}
        for name, (fleet, (rate, in_tok, out_tok), slo, trace) in cs.items():
            lo, hi = windows(rate)
            assert rate.shape == lo.shape == hi.shape == in_tok.shape == out_tok.shape
            assert all(v.shape == rate.shape for v in slo.values())
            assert (lo <= rate).all() and (rate <= hi).all() and np.isfinite(hi).all()
            keys, run, trace_run = n_keys_and_searches(fleet, hi, in_tok, out_tok, slo, trace)
            shapes[name] = {"servers": fleet.n_servers, "acc": fleet.n_acc, "rows": rate.shape[0], "trace": trace,
                            "keys": keys, "searches": run, "slo_trace_searches": trace_run}
        print(json.dumps({"dry_run": True, "cases": shapes}))
        return
    from workload_variant_autoscaler_b200 import Engine
    e = Engine(0)
    out = {name: run_case(e, fleet, load, slo, trace, a.reps) for name, (fleet, load, slo, trace) in cs.items()}
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power,
                      "workload": "SLO margins, windows [0.5x, 2x]", "calls": a.reps, **out}))


if __name__ == "__main__":
    main()
