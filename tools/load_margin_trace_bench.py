"""wva_load_margin_trace in three cases: synth_fleet(10000, 8, seed=42) (the configs[3] shape) × the 24 rows of
load_grid_bench.py, keepAccelerator off and in WVA's configuration (keepAccelerator on every server, every current
accelerator a real one with its cost, min_replicas 1); and synth_fleet(256, 8) × 1,440 ticks (a day of minutes, a
diurnal rate per server).  Windows are [0.5x, 2x] of each row.

Prints one JSON line with the GPU's name, power limit and max SM clock, and per case: the median device / kernel /
host time over the repeated calls, the launches per call, a histogram of the flags, the own device time of
margin_chain and margin_kernel (torch.profiler, in a separate call), and the alternative a caller has without the
call: wva_workload_trace, then one wva_load_margins call per tick on the fleet advanced by Fleet.apply_winners, timed
(device time summed over the calls, host wall time of the whole loop), with a per-tick byte comparison of every
column.  Needs a GPU; run from the repository root.  --dry-run builds the cases' rows and windows at the given
sizes and prints their shapes without touching a GPU."""
import argparse
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
from workload_variant_autoscaler_b200 import (MARGIN_HI_OPEN, MARGIN_LO_OPEN, MARGIN_TRUNCATED,  # noqa: E402
                                              synth_fleet)

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
    A = fleet.n_acc
    fleet.srv_keep_acc[:] = 1
    fleet.srv_min_replicas[:] = 1
    none = fleet.srv_cur_acc < 0
    fleet.srv_cur_acc[none] = rng.integers(0, A, int(none.sum()))
    fleet.srv_cur_replicas[none] = 1
    a = fleet.srv_cur_acc
    fleet.srv_cur_cost[:] = (fleet.acc_cost[a] * fleet.perf_acc_count[fleet.srv_model, a] *
                             fleet.srv_cur_replicas).astype(np.float32)
    return fleet


def levels(fleet, L, seed):
    """load_grid_bench.py's rows."""
    rng = np.random.default_rng(seed)
    return (fleet.srv_arrival_rpm[None, :] * rng.lognormal(0.0, 0.5, (L, fleet.n_servers))).astype(np.float32)


def day(fleet, L, seed):
    """A diurnal rate: the server's own load (at least 1 req/min) times e^(1.5 sin) with a per-server phase, times
    noise, one row per minute."""
    rng = np.random.default_rng(seed)
    t = np.arange(L)[:, None]
    phase = rng.uniform(0, 2 * np.pi, fleet.n_servers)
    daily = np.exp(1.5 * np.sin(2 * np.pi * t / 1440 + phase[None, :]))
    return (np.maximum(fleet.srv_arrival_rpm, 1.0)[None, :] * daily *
            rng.lognormal(0.0, 0.1, (L, fleet.n_servers))).astype(np.float32)


def cases(S, A, L, day_S, day_L):
    fleet = synth_fleet(S, A, seed=42)
    rows = levels(fleet, L, 7)
    small = synth_fleet(day_S, A, seed=42)
    return {f"{S}x{A}x{L}_keep_off": (fleet, rows),
            f"{S}x{A}x{L}_wva_configuration": (wva_configuration(synth_fleet(S, A, seed=42), 42), rows),
            f"{day_S}x{A}x{day_L}_day_of_minutes": (small, day(small, day_L, 3))}


def windows(rate):
    return (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)


def kernel_ms(e, fleet, rate, lo, hi):
    """Device time (ms) per margin kernel name in one call."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.load_margin_trace(fleet, rate, lo, hi)
    out = {}
    for ev in prof.key_averages():
        if "margin" in ev.key:
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            out[ev.key.split("(")[0]] = t / 1e3
    return out


def timed(call, reps, e):
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


def alternative(e, fleet, rate, lo, hi, got):
    """workload_trace, then one load_margins per tick on the apply_winners chain: (timing, ticks differing)."""
    L, S = rate.shape
    t0 = time.perf_counter()
    _, win = e.workload_trace(fleet, rate)
    dev = e.last_device_ms
    cur, differ = fleet, 0
    for t in range(L):
        one = e.load_margins(cur, rate[t:t + 1], lo[t:t + 1], hi[t:t + 1])
        dev += e.last_device_ms
        cur = cur.apply_winners(one[3])
        sl = slice(t * S, (t + 1) * S)
        ok = same(one[0][0], got[0][t]) and same(one[1][0], got[1][t]) and same(one[2][0], got[2][t])
        ok = ok and all(same(getattr(x, f), getattr(y, f)[sl]) for x, y in zip(one[3:], got[3:]) for f in FIELDS)
        differ += not ok
    wall = (time.perf_counter() - t0) * 1e3
    at_vs_trace = all(same(getattr(got[3], f), getattr(win, f)) for f in FIELDS)
    return {"device_ms_total": dev, "host_wall_ms": wall, "ticks_differing": differ,
            "at_blocks_equal_workload_trace": at_vs_trace}


def run_case(e, fleet, rate, reps, warm=3):
    lo, hi = windows(rate)
    for _ in range(warm):
        e.load_margin_trace(fleet, rate, lo, hi)
    got, t = timed(lambda: e.load_margin_trace(fleet, rate, lo, hi), reps, e)
    flags = got[2]
    res = dict(t)
    res["flags"] = {"closed": int((flags == 0).sum()), "lo_open": int(((flags & MARGIN_LO_OPEN) != 0).sum()),
                    "hi_open": int(((flags & MARGIN_HI_OPEN) != 0).sum()),
                    "truncated": int(((flags & MARGIN_TRUNCATED) != 0).sum())}
    res["kernels_ms"] = kernel_ms(e, fleet, rate, lo, hi)
    res["alternative"] = alternative(e, fleet, rate, lo, hi, got)
    return res


def main(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("--servers", type=int, default=10000)
    p.add_argument("--acc", type=int, default=8)
    p.add_argument("--ticks", type=int, default=24)
    p.add_argument("--day-servers", type=int, default=256)
    p.add_argument("--day-ticks", type=int, default=1440)
    p.add_argument("--reps", type=int, default=10)
    p.add_argument("--dry-run", action="store_true", help="build the cases and print their shapes; no GPU")
    a = p.parse_args(argv)
    if min(a.servers, a.acc, a.ticks, a.day_servers, a.day_ticks, a.reps) < 1:
        p.error("every size must be at least 1")
    cs = cases(a.servers, a.acc, a.ticks, a.day_servers, a.day_ticks)
    if a.dry_run:
        shapes = {}
        for name, (fleet, rate) in cs.items():
            lo, hi = windows(rate)
            assert rate.shape == lo.shape == hi.shape == (rate.shape[0], fleet.n_servers)
            assert (lo <= rate).all() and (rate <= hi).all() and np.isfinite(hi).all()
            shapes[name] = {"servers": fleet.n_servers, "acc": fleet.n_acc, "ticks": rate.shape[0]}
        print(json.dumps({"dry_run": True, "cases": shapes}))
        return
    from workload_variant_autoscaler_b200 import Engine
    e = Engine(0)
    out = {name: run_case(e, fleet, rate, a.reps) for name, (fleet, rate) in cs.items()}
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power,
                      "workload": "load_margin_trace, windows [0.5x, 2x]", "calls": a.reps, **out}))


if __name__ == "__main__":
    main()
