"""wva_workload_margins and wva_workload_margin_trace in five cases: synth_fleet(10000, 8, seed=42) (the configs[3]
shape) x the 24 rows of workload_grid_bench.py (rates as in load_grid_bench.py, out_tokens x {0.75, 1, 1.5} per
(row, server)), grid and trace, each with keepAccelerator off and in WVA's configuration (keepAccelerator on every
server, every current accelerator a real one with its cost, min_replicas 1); and synth_fleet(256, 8) x 1,440 ticks
(a day of minutes: a diurnal rate and the same token draw), trace.  Windows are [0.5x, 2x] of each row.

Prints one JSON line with the GPU's name, power limit and max SM clock, and per case: the median device / kernel /
host time over the repeated calls, the launches per call, the token keys sized against L * S, the own device time
of margin_kernel and margin_chain (torch.profiler, in a separate call), the load-margin call on the same rates at the
fleet's own tokens (what the token rows cost), and the alternative a caller has without the call: one
wva_load_margins per row on the fleet with the row's tokens (for the trace, after wva_workload_trace, on the fleet
advanced by Fleet.apply_winners), timed (device time summed over the calls, host wall time of the whole loop), with a
per-row byte comparison of every column.  Needs a GPU; run from the repository root.  --dry-run builds the cases'
rows and windows and prints their shapes without touching a GPU."""
import argparse
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
from workload_variant_autoscaler_b200 import synth_fleet  # noqa: E402

FIELDS = ("feasible", "acc", "replicas", "batch", "cost", "value", "itl", "ttft", "rho", "max_rate")
F32 = np.float32


def gpu_label():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # the label is informative only
        q = "unknown"
    return name, q


def wva_configuration(fleet, seed):
    """keepAccelerator and min_replicas 1 on every server, each current accelerator a real one with its cost."""
    rng = np.random.default_rng(seed)
    fleet.srv_keep_acc[:] = 1
    fleet.srv_min_replicas[:] = 1
    none = fleet.srv_cur_acc < 0
    fleet.srv_cur_acc[none] = rng.integers(0, fleet.n_acc, int(none.sum()))
    fleet.srv_cur_replicas[none] = 1
    a = fleet.srv_cur_acc
    fleet.srv_cur_cost[:] = (fleet.acc_cost[a] * fleet.perf_acc_count[fleet.srv_model, a] *
                             fleet.srv_cur_replicas).astype(np.float32)
    return fleet


def tokens(fleet, L, rng):
    """workload_grid_bench.py's tokens: in_tokens the server's own, out_tokens x {0.75, 1, 1.5} per (row, server)."""
    S = fleet.n_servers
    out = np.maximum(fleet.srv_out_tokens[None, :] * rng.choice([0.75, 1.0, 1.5], (L, S)), 1).astype(np.int32)
    return np.ascontiguousarray(np.broadcast_to(fleet.srv_in_tokens, (L, S)), np.int32), out


def rows_24(fleet, L, seed):
    """workload_grid_bench.py's rows."""
    rng = np.random.default_rng(seed)
    rpm = (fleet.srv_arrival_rpm[None, :] * rng.lognormal(0.0, 0.5, (L, fleet.n_servers))).astype(np.float32)
    return (rpm,) + tokens(fleet, L, rng)


def rows_day(fleet, L, seed):
    """A diurnal rate (load_margin_trace_bench.py's day of minutes) with the same token draw."""
    rng = np.random.default_rng(seed)
    t = np.arange(L)[:, None]
    phase = rng.uniform(0, 2 * np.pi, fleet.n_servers)
    daily = np.exp(1.5 * np.sin(2 * np.pi * t / 1440 + phase[None, :]))
    rpm = (np.maximum(fleet.srv_arrival_rpm, 1.0)[None, :] * daily *
           rng.lognormal(0.0, 0.1, (L, fleet.n_servers))).astype(np.float32)
    return (rpm,) + tokens(fleet, L, rng)


def cases(S, A, L, day_S, day_L):
    off = synth_fleet(S, A, seed=42)
    wva = wva_configuration(synth_fleet(S, A, seed=42), 42)
    rows = rows_24(off, L, 7)
    small = synth_fleet(day_S, A, seed=42)
    out = {}
    for trace in (False, True):
        kind = "trace" if trace else "grid"
        out[f"{S}x{A}x{L}_{kind}_keep_off"] = (off, rows, trace)
        out[f"{S}x{A}x{L}_{kind}_wva_configuration"] = (wva, rows, trace)
    out[f"{day_S}x{A}x{day_L}_trace_day_of_minutes"] = (small, rows_day(small, day_L, 3), True)
    return out


def windows(rate):
    return (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)


def n_keys(hi, in_tok, out_tok):
    """Distinct (server, in, out) over the rows whose window top is above 0 and whose tokens are a load."""
    L, S = hi.shape
    use = (hi > 0) & (in_tok >= 0) & (out_tok >= 1)
    srv = np.broadcast_to(np.arange(S), (L, S))
    keys = np.stack([srv[use], in_tok[use], out_tok[use]], axis=1)
    return int(np.unique(keys, axis=0).shape[0]) if keys.size else 0


def call_of(e, trace):
    return e.workload_margin_trace if trace else e.workload_margins


def kernel_ms(call):
    """Device time (ms) per margin kernel name in one call."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
    out = {}
    for ev in prof.key_averages():
        if "margin" in ev.key:
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            out[ev.key] = t / 1e3
    return out


def timed(call, reps, e, warm=3):
    for _ in range(warm):
        call()
    dev, ker, wall = [], [], []
    l0 = e.launch_count
    for _ in range(reps):
        t0 = time.perf_counter()
        out = call()
        wall.append(time.perf_counter() - t0)
        dev.append(e.last_device_ms)
        ker.append(e.last_kernel_ms)
    return out, {"device_ms_p50": float(np.median(dev)), "kernel_ms_p50": float(np.median(ker)),
                 "host_wall_ms_p50": float(np.median(wall)) * 1e3, "launches_per_call": (e.launch_count - l0) / reps}


def same(a, b):
    return np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


def with_tokens(fleet, in_tok, out_tok, l):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_in_tokens[:] = in_tok[l]
    f.srv_out_tokens[:] = out_tok[l]
    return f


def alternative(e, fleet, rows, lo, hi, trace, got):
    """One load_margins per row on the fleet with the row's tokens (on a trace after workload_trace, along the
    apply_winners chain): (timing, rows differing, whether the `at` blocks are the workload call's winners)."""
    rate, in_tok, out_tok = rows
    L, S = rate.shape
    if not trace:  # the grid's alternative needs no workload call: it runs only for the check of `at`
        _, win = e.workload_grid(fleet, rate, in_tok, out_tok)
    t0 = time.perf_counter()
    dev = 0.0
    if trace:
        _, win = e.workload_trace(fleet, rate, in_tok, out_tok)
        dev = e.last_device_ms
    cur, differ = fleet, 0
    for t in range(L):
        one = e.load_margins(with_tokens(cur, in_tok, out_tok, t), rate[t:t + 1], lo[t:t + 1], hi[t:t + 1])
        dev += e.last_device_ms
        if trace:
            cur = cur.apply_winners(one[3])
        sl = slice(t * S, (t + 1) * S)
        ok = same(one[0][0], got[0][t]) and same(one[1][0], got[1][t]) and same(one[2][0], got[2][t])
        ok = ok and all(same(getattr(x, f), getattr(y, f)[sl]) for x, y in zip(one[3:], got[3:]) for f in FIELDS)
        differ += not ok
    wall = (time.perf_counter() - t0) * 1e3
    at_equal = all(same(getattr(got[3], f), getattr(win, f)) for f in FIELDS)
    return {"device_ms_total": dev, "host_wall_ms": wall, "rows_differing": differ,
            "at_blocks_equal_workload_winners": at_equal}


def run_case(e, fleet, rows, trace, reps):
    rate, in_tok, out_tok = rows
    lo, hi = windows(rate)
    call = call_of(e, trace)
    got, t = timed(lambda: call(fleet, rate, in_tok, out_tok, lo, hi), reps, e)
    res = dict(t)
    res["keys"] = n_keys(hi, in_tok, out_tok)
    res["rows_x_servers"] = int(rate.size)
    res["kernels_ms"] = kernel_ms(lambda: call(fleet, rate, in_tok, out_tok, lo, hi))
    fixed = e.load_margin_trace if trace else e.load_margins
    _, tf = timed(lambda: fixed(fleet, rate, lo, hi), reps, e)
    tf["kernels_ms"] = kernel_ms(lambda: fixed(fleet, rate, lo, hi))
    res["own_tokens_load_margin_call"] = tf
    res["alternative"] = alternative(e, fleet, rows, lo, hi, trace, got)
    return res


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--servers", type=int, default=10000)
    p.add_argument("--acc", type=int, default=8)
    p.add_argument("--rows", type=int, default=24)
    p.add_argument("--day-servers", type=int, default=256)
    p.add_argument("--day-ticks", type=int, default=1440)
    p.add_argument("--reps", type=int, default=10)
    p.add_argument("--dry-run", action="store_true", help="build the cases and print their shapes; no GPU")
    a = p.parse_args(argv)
    if min(a.servers, a.acc, a.rows, a.day_servers, a.day_ticks, a.reps) < 1:
        p.error("every size must be at least 1")
    cs = cases(a.servers, a.acc, a.rows, a.day_servers, a.day_ticks)
    if a.dry_run:
        shapes = {}
        for name, (fleet, (rate, in_tok, out_tok), trace) in cs.items():
            lo, hi = windows(rate)
            assert rate.shape == lo.shape == hi.shape == in_tok.shape == out_tok.shape
            assert (lo <= rate).all() and (rate <= hi).all() and np.isfinite(hi).all()
            shapes[name] = {"servers": fleet.n_servers, "acc": fleet.n_acc, "rows": rate.shape[0], "trace": trace,
                            "keys": n_keys(hi, in_tok, out_tok)}
        print(json.dumps({"dry_run": True, "cases": shapes}))
        return
    from workload_variant_autoscaler_b200 import Engine
    e = Engine(0)
    out = {name: run_case(e, fleet, rows, trace, a.reps) for name, (fleet, rows, trace) in cs.items()}
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power,
                      "workload": "workload margins, windows [0.5x, 2x]", "calls": a.reps, **out}))


if __name__ == "__main__":
    main()
