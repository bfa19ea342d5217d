"""wva_profile_price_threshold_grid and wva_profile_price_threshold_trace in five cases: synth_fleet(10000, 8,
seed=42) (the configs[3] shape) x the 24 rows of workload_margins_bench.py (rates and out_tokens x {0.75, 1, 1.5} per
(row, server)) with hourly prices on every accelerator (profile_margins_bench.py's rows), grid and trace, each with
keepAccelerator off and in WVA's configuration; and synth_fleet(256, 8) x 1,440 ticks (a day of minutes, prices
changing every hour, beta x 1.1 from the middle of the day and the last accelerator absent for the first third),
trace.

Prints one JSON line with the GPU's name, power limit and max SM clock, and per case: the median device / kernel /
host time over the repeated calls and the launches per call; wva_profile_trace alone on the same rows (what the
thresholds add); price_kernel's own device time (torch.profiler, in a separate call); and the alternative a caller has
without the call: one wva_price_thresholds per row on the fleet with the row's columns (for the trace with c_t from
wva_profile_trace's winners along Fleet.apply_winners), timed (device time summed over the calls, host wall time of
the whole loop), with a per-row byte comparison of threshold, above and the candidates.  Needs a GPU; run from the
repository root.  --dry-run builds the cases and prints their shapes without touching a GPU."""
import argparse
import json
import sys
import time

import numpy as np

sys.path.insert(0, ".")
sys.path.insert(0, "tools")
from profile_margins_bench import at_row, kernels_ms, profile  # noqa: E402
from workload_margins_bench import FIELDS, gpu_label, rows_24, rows_day, same, timed, wva_configuration  # noqa: E402
from workload_variant_autoscaler_b200 import synth_fleet  # noqa: E402


def cases(S, A, L, day_S, day_L):
    off = synth_fleet(S, A, seed=42)
    wva = wva_configuration(synth_fleet(S, A, seed=42), 42)
    load = rows_24(off, L, 7)
    prof = profile(off, L, 1, 11, False)
    small = synth_fleet(day_S, A, seed=42)
    out = {}
    for trace in (False, True):
        kind = "trace" if trace else "grid"
        out[f"{S}x{A}x{L}_{kind}_hourly_prices_keep_off"] = (off, load, prof, trace)
        out[f"{S}x{A}x{L}_{kind}_hourly_prices_wva_configuration"] = (wva, load, prof, trace)
    out[f"{day_S}x{A}x{day_L}_trace_day_of_minutes"] = (small, rows_day(small, day_L, 3),
                                                        profile(small, day_L, 60, 11, True), True)
    return out


def block(allocs, lo, hi):
    return {f: getattr(allocs, f)[lo:hi] for f in FIELDS}


def alternative(e, fleet, load, prof, trace, got):
    """One price_thresholds per row on the fleet with the row's columns (on a trace with c_t from profile_trace's
    winners along apply_winners): (timing, rows differing)."""
    rate, in_tok, out_tok = load
    L, S = rate.shape
    A = fleet.n_acc
    th, above, cand, _ = got
    t0 = time.perf_counter()
    dev = 0.0
    if trace:
        _, win = e.profile_trace(fleet, rate, in_tok, out_tok, **prof)
        dev = e.last_device_ms
    cur, differ = fleet, 0
    for t in range(L):
        f = at_row(cur, in_tok, out_tok, prof, t)
        f.srv_arrival_rpm[:] = rate[t]
        th1, above1, cand1 = e.price_thresholds(f, want_candidates=True)
        dev += e.last_device_ms
        if trace:
            one = type(win)(S)
            for k in FIELDS:
                getattr(one, k)[:] = getattr(win, k)[t * S:(t + 1) * S]
            cur = cur.apply_winners(one)
        sl = slice(t * S * A, (t + 1) * S * A)
        ok = same(th1, th[t]) and all(same(getattr(above1, k), getattr(above, k)[sl]) and
                                      same(getattr(cand1, k), getattr(cand, k)[sl]) for k in FIELDS)
        differ += not ok
    return {"device_ms_total": dev, "host_wall_ms": (time.perf_counter() - t0) * 1e3, "rows_differing": differ}


def run_case(e, fleet, load, prof, trace, reps):
    rate, in_tok, out_tok = load
    call = e.profile_price_threshold_trace if trace else e.profile_price_threshold_grid
    go = lambda: call(fleet, rate, in_tok, out_tok, want_candidates=True, **prof)  # noqa: E731
    got, t = timed(go, reps, e)
    res = dict(t)
    res["rows_x_servers"] = int(rate.size)
    k = kernels_ms(go)
    res["price_kernel_ms"] = sum(v for n, v in k.items() if "price_kernel" in n)
    res["kernels_ms"] = k
    # wva_profile_trace alone (the grid mode has no public call of its own; the trace is the same pipeline)
    _, tp = timed(lambda: e.profile_trace(fleet, rate, in_tok, out_tok, want_candidates=True, **prof), reps, e)
    res["profile_trace_alone"] = tp
    res["alternative"] = alternative(e, fleet, load, prof, trace, got)
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
        shapes = {name: {"servers": f.n_servers, "acc": f.n_acc, "rows": load[0].shape[0], "trace": trace,
                         "profile_columns": sorted(prof)} for name, (f, load, prof, trace) in cs.items()}
        print(json.dumps({"dry_run": True, "cases": shapes}))
        return
    from workload_variant_autoscaler_b200 import Engine
    e = Engine(0)
    out = {name: run_case(e, fleet, load, prof, trace, a.reps) for name, (fleet, load, prof, trace) in cs.items()}
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "workload": "profile price thresholds",
                      "calls": a.reps, **out}))


if __name__ == "__main__":
    main()
