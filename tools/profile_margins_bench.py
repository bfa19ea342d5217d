"""wva_profile_margins and wva_profile_margin_trace in nine cases: synth_fleet(10000, 8, seed=42) (the configs[3]
shape) x the 24 rows of workload_margins_bench.py (rates and out_tokens x {0.75, 1, 1.5} per (row, server)) with hourly
prices (profile_trace_bench.py's curve), grid and trace, each with keepAccelerator off and in WVA's configuration; the
same four with a beta change (x 1.1 from row 12 on) and a new accelerator (the last one absent until row 8) in the
rows; and synth_fleet(256, 8) x 1,440 ticks (a day of minutes, prices changing every hour, the beta change and the new
accelerator), trace.  Windows are [0.5x, 2x] of each row.

Prints one JSON line with the GPU's name, power limit and max SM clock, and per case: the median device / kernel /
host time over the repeated calls, the launches per call, the keys sized against L * S, each kernel's own device time
(torch.profiler, in a separate call: margin_kernel, margin_chain and phase 1's sizing kernels), the workload-margin
call on the same load rows at the fleet's own prices and profiles (what the profile rows cost), and the alternative a
caller has without the call: one wva_load_margins per row on the fleet with the row's tokens, prices and profiles
(for the trace, after wva_profile_trace, on the fleet advanced by Fleet.apply_winners), timed (device time summed over
the calls, host wall time of the whole loop), with a per-row byte comparison of every column.  Needs a GPU; run from
the repository root.  --dry-run builds the cases' rows and windows and prints their shapes without touching a GPU."""
import argparse
import json
import sys
import time

import numpy as np

sys.path.insert(0, ".")
sys.path.insert(0, "tools")
from workload_margins_bench import (FIELDS, gpu_label, rows_24, rows_day, same, timed,  # noqa: E402
                                    windows, wva_configuration)
from workload_variant_autoscaler_b200 import synth_fleet  # noqa: E402

F32 = np.float32
PROFILE = ("acc_cost", "perf_present", "perf_alpha", "perf_beta", "perf_gamma", "perf_delta", "perf_acc_count",
           "perf_max_batch", "perf_at_tokens")


def hourly_prices(fleet, L, ticks_per_hour, seed):
    """acc_cost [L, A]: a daily price curve per accelerator (own phase and depth), constant within each hour."""
    rng = np.random.default_rng(seed)
    A = fleet.n_acc
    hour = (np.arange(L) // ticks_per_hour)[:, None]
    phase, depth = rng.uniform(0, 2 * np.pi, A), rng.uniform(0.2, 0.6, A)
    curve = 1.0 + depth * np.sin(2 * np.pi * hour / 24 + phase) + rng.normal(0, 0.02, (L // ticks_per_hour + 1, A))[
        hour[:, 0]]
    return (fleet.acc_cost[None] * np.maximum(curve, 0.05)).astype(F32)


def profile(fleet, L, ticks_per_hour, seed, perf):
    """The profile rows: hourly prices, and with `perf` beta x 1.1 from row L // 2 on and the last accelerator
    absent (perf_present 0) before row L // 3."""
    rows = {"acc_cost": hourly_prices(fleet, L, ticks_per_hour, seed)}
    if perf:
        beta = np.repeat(fleet.perf_beta[None], L, axis=0).astype(F32)
        beta[L // 2:] *= F32(1.1)
        present = np.repeat(fleet.perf_present[None], L, axis=0)
        present[:L // 3, :, -1] = 0
        rows.update(perf_beta=beta, perf_present=present)
    return rows


def cases(S, A, L, day_S, day_L):
    off = synth_fleet(S, A, seed=42)
    wva = wva_configuration(synth_fleet(S, A, seed=42), 42)
    load = rows_24(off, L, 7)
    small = synth_fleet(day_S, A, seed=42)
    out = {}
    for perf in (False, True):
        what = "beta_and_new_acc" if perf else "prices"
        prof = profile(off, L, 1, 11, perf)
        for trace in (False, True):
            kind = "trace" if trace else "grid"
            out[f"{S}x{A}x{L}_{kind}_{what}_keep_off"] = (off, load, prof, trace)
            out[f"{S}x{A}x{L}_{kind}_{what}_wva_configuration"] = (wva, load, prof, trace)
    out[f"{day_S}x{A}x{day_L}_trace_day_of_minutes"] = (small, rows_day(small, day_L, 3),
                                                        profile(small, day_L, 60, 11, True), True)
    return out


def n_keys(fleet, hi, in_tok, out_tok, prof, trace):
    """Distinct (server, accelerator, in, out, alpha .. delta bits, N) over the rows whose window top is above 0 at
    which the pair is a load pair, keepAccelerator masking a pair at every row (on a trace on the pinned servers
    only); without a perf column the workload margins' (server, in, out) keys."""
    L, S = hi.shape
    use = (hi > 0) & (in_tok >= 0) & (out_tok >= 1)
    srv = np.broadcast_to(np.arange(S), (L, S))
    if not any(k in prof for k in PROFILE[1:]):
        keys = np.stack([srv[use], in_tok[use], out_tok[use]], axis=1)
        return int(np.unique(keys, axis=0).shape[0]) if keys.size else 0
    col = {k: prof.get(k, np.repeat(getattr(fleet, k)[None], L, axis=0)) for k in PROFILE[1:]}
    cur, keep = fleet.srv_cur_acc, fleet.srv_keep_acc != 0
    if trace:
        keep = keep & (cur != -1) & ((cur == -2) | (fleet.srv_min_replicas != 0))
    else:
        keep = keep & (cur != -1)
    m = fleet.srv_model
    found = []
    for a in range(fleet.n_acc):
        ok = use & ~(keep & (cur != a))[None, :] & col["perf_present"][:, m, a].astype(bool)
        ok &= fleet.srv_has_target[None, :].astype(bool)
        N = np.where(fleet.srv_max_batch[None, :] > 0, fleet.srv_max_batch[None, :],
                     np.maximum(col["perf_max_batch"][:, m, a].astype(np.int64) *
                                col["perf_at_tokens"][:, m, a] // np.maximum(out_tok, 1), 1))
        bits = [col[k][:, m, a].astype(F32).view(np.uint32).astype(np.int64)
                for k in ("perf_alpha", "perf_beta", "perf_gamma", "perf_delta")]
        found.append(np.stack([srv[ok], np.full(int(ok.sum()), a), in_tok[ok], out_tok[ok], *(b[ok] for b in bits),
                               N[ok]], axis=1))
    keys = np.concatenate(found)
    return int(np.unique(keys, axis=0).shape[0]) if keys.size else 0


def kernels_ms(call):
    """Device time (ms) per kernel name in one call."""
    from torch.profiler import ProfilerActivity, profile as tprofile
    with tprofile(activities=[ProfilerActivity.CUDA]) as p:
        call()
    out = {}
    for ev in p.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            out[ev.key[:80]] = t / 1e3
    return out


def at_row(fleet, in_tok, out_tok, prof, l):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_in_tokens[:] = in_tok[l]
    f.srv_out_tokens[:] = out_tok[l]
    for k, v in prof.items():
        getattr(f, k)[:] = v[l]
    return f


def alternative(e, fleet, load, prof, lo, hi, trace, got):
    """One load_margins per row on the fleet with the row's columns (on a trace after profile_trace, along the
    apply_winners chain): (timing, rows differing, whether the `at` blocks are the profile trace's winners)."""
    rate, in_tok, out_tok = load
    L, S = rate.shape
    t0 = time.perf_counter()
    dev = 0.0
    if trace:
        _, win = e.profile_trace(fleet, rate, in_tok, out_tok, **prof)
        dev = e.last_device_ms
    cur, differ = fleet, 0
    for t in range(L):
        one = e.load_margins(at_row(cur, in_tok, out_tok, prof, t), rate[t:t + 1], lo[t:t + 1], hi[t:t + 1])
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
        res["at_blocks_equal_profile_trace_winners"] = all(same(getattr(got[3], f), getattr(win, f)) for f in FIELDS)
    return res


def run_case(e, fleet, load, prof, trace, reps):
    rate, in_tok, out_tok = load
    lo, hi = windows(rate)
    call = e.profile_margin_trace if trace else e.profile_margins
    go = lambda: call(fleet, rate, in_tok, out_tok, lo, hi, **prof)  # noqa: E731
    got, t = timed(go, reps, e)
    res = dict(t)
    res["keys"] = n_keys(fleet, hi, in_tok, out_tok, prof, trace)
    res["rows_x_servers"] = int(rate.size)
    res["kernels_ms"] = kernels_ms(go)
    own = e.workload_margin_trace if trace else e.workload_margins
    _, tw = timed(lambda: own(fleet, rate, in_tok, out_tok, lo, hi), reps, e)
    tw["kernels_ms"] = kernels_ms(lambda: own(fleet, rate, in_tok, out_tok, lo, hi))
    res["own_prices_workload_margin_call"] = tw
    res["alternative"] = alternative(e, fleet, load, prof, lo, hi, trace, got)
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
        for name, (fleet, (rate, in_tok, out_tok), prof, trace) in cs.items():
            lo, hi = windows(rate)
            assert rate.shape == lo.shape == hi.shape == in_tok.shape == out_tok.shape
            assert (lo <= rate).all() and (rate <= hi).all() and np.isfinite(hi).all()
            shapes[name] = {"servers": fleet.n_servers, "acc": fleet.n_acc, "rows": rate.shape[0], "trace": trace,
                            "profile_columns": sorted(prof), "keys": n_keys(fleet, hi, in_tok, out_tok, prof, trace)}
        print(json.dumps({"dry_run": True, "cases": shapes}))
        return
    from workload_variant_autoscaler_b200 import Engine
    e = Engine(0)
    out = {name: run_case(e, fleet, load, prof, trace, a.reps) for name, (fleet, load, prof, trace) in cs.items()}
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power,
                      "workload": "profile margins, windows [0.5x, 2x]", "calls": a.reps, **out}))


if __name__ == "__main__":
    main()
