"""wva_load_margins on synth_fleet(10000, 8, seed=42) (the configs[3] shape) in three cases: one level at the fleet's
own load with windows [0.5x, 2x], keepAccelerator off and in WVA's configuration (keepAccelerator on every server,
every current accelerator a real one with its cost, min_replicas 1); and 24 levels, the rows of load_grid_bench.py,
with windows [0.5x, 2x] of each row.

Prints one JSON line with, per case: the median device / kernel / host time over 20 calls, the launches per call,
a histogram of the flags and margin_kernel's own device time (torch.profiler, one call).  Per case it also runs
wva_load_intervals on the same windows with M = 64 (level by level), timed, and checks that its interval holding each
level's rate equals the margin wherever the list is not truncated; and one wva_load_grid at the rows {r, below lo,
hi}, compared byte for byte with at / below / above.  Needs a GPU; run from the repository root."""
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
from workload_variant_autoscaler_b200 import (MARGIN_HI_OPEN, MARGIN_LO_OPEN, MARGIN_TRUNCATED, Engine,  # noqa: E402
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


def margin_kernel_ms(e, fleet, rate, lo, hi):
    """Device time (ms) per margin kernel name in one call."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.load_margins(fleet, rate, lo, hi)
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


def run_case(e, fleet, rate, reps, M=64, warm=3):
    L, S = rate.shape
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    for _ in range(warm):
        e.load_margins(fleet, rate, lo, hi)
    (lo_m, hi_m, flags, at, below, above), t = timed(lambda: e.load_margins(fleet, rate, lo, hi), reps, e)
    res = dict(t)
    res["flags"] = {"closed": int((flags == 0).sum()), "lo_open": int(((flags & MARGIN_LO_OPEN) != 0).sum()),
                    "hi_open": int(((flags & MARGIN_HI_OPEN) != 0).sum()),
                    "truncated": int(((flags & MARGIN_TRUNCATED) != 0).sum())}
    res["margin_kernels_ms"] = margin_kernel_ms(e, fleet, rate, lo, hi)
    # the load intervals on the same windows, one call per level
    iv_dev, iv_ker, iv_launch = 0.0, 0.0, 0
    checked = differ = truncated = 0
    for l in range(L):
        for _ in range(warm if l == 0 else 0):
            e.load_intervals(fleet, lo[l], hi[l], M)
        n0 = e.launch_count
        count, trunc, start, rec = e.load_intervals(fleet, lo[l], hi[l], M)
        iv_dev += e.last_device_ms
        iv_ker += e.last_kernel_ms
        iv_launch += e.launch_count - n0
        truncated += int(trunc.sum())
        for s in range(S):
            if trunc[s] or flags[l, s] & MARGIN_TRUNCATED:
                continue
            n = int(count[s])
            j = int(np.searchsorted(start[s, :n], rate[l, s], side="right")) - 1
            lo_want = start[s, j]
            hi_want = start[s, j + 1] if j + 1 < n else F32(np.inf)
            checked += 1
            differ += not (lo_m[l, s] == lo_want and hi_m[l, s] == hi_want and
                           all(getattr(at, k)[l * S + s] == getattr(rec, k)[s * M + j] or k in ("itl", "ttft", "rho")
                               for k in FIELDS))
    res["load_intervals_M64"] = {"device_ms_total": iv_dev, "kernel_ms_total": iv_ker, "launches": iv_launch,
                                 "servers_truncated": truncated, "margins_checked": checked,
                                 "margins_differing": differ}
    # the records through the load grid at {r, below lo, hi}
    closed_lo = (flags & (MARGIN_LO_OPEN | MARGIN_TRUNCATED)) == 0
    closed_hi = (flags & (MARGIN_HI_OPEN | MARGIN_TRUNCATED)) == 0
    rows = np.concatenate([rate, np.where(closed_lo, np.nextafter(lo_m, F32(0)), rate),
                           np.where(closed_hi, hi_m, rate)]).astype(np.float32)
    _, win = e.load_grid(fleet, rows)
    mismatches = 0
    for k, (recs, closed) in enumerate(((at, np.ones_like(closed_lo)), (below, closed_lo), (above, closed_hi))):
        for f in FIELDS:
            g = getattr(win, f)[k * L * S:(k + 1) * L * S].reshape(L, S)
            w = getattr(recs, f).reshape(L, S)
            same = g.view(np.uint8 if g.itemsize == 1 else np.uint32) == w.view(np.uint8 if w.itemsize == 1 else
                                                                                  np.uint32)
            mismatches += int((~same & closed).sum())
    res["load_grid_record_mismatches"] = mismatches
    return res


def main(S=10000, A=8, reps=20):
    e = Engine(0)
    out = {}
    fleet = synth_fleet(S, A, seed=42)
    own = fleet.srv_arrival_rpm[None, :].astype(np.float32)
    out["L1_keep_off"] = run_case(e, fleet, own, reps)
    wfleet = wva_configuration(synth_fleet(S, A, seed=42), 42)
    out["L1_wva_configuration"] = run_case(e, wfleet, own, reps)
    out["L24_load_grid_rows"] = run_case(e, fleet, levels(fleet, 24, 7), reps)
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power,
                      "workload": f"load_margins synth_fleet({S}, {A}, seed=42), windows [0.5x, 2x]", "calls": reps,
                      **out}))


if __name__ == "__main__":
    main()
