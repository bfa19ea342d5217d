"""wva_load_intervals on synth_fleet(10000, 8, seed=42) (the configs[3] shape), ranges [0.5x, 2x] of each server's
load, M = 64.

Prints one JSON line: the median device / kernel / host time over 20 calls, the launches per call, the intervals
found and the servers truncated, the per-kernel device time of the interval kernels (torch.profiler, one call),
and one wva_load_grid over every interval start, timed, with a byte comparison of its winners against the
interval records.  Needs a GPU; run from the repository root."""
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
from workload_variant_autoscaler_b200 import Engine, synth_fleet  # noqa: E402

FIELDS = ("feasible", "acc", "replicas", "batch", "cost", "value", "itl", "ttft", "rho", "max_rate")


def gpu_label():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # the label is informative only
        q = "unknown"
    return name, q


def kernel_times(e, fleet, lo, hi, M):
    """Device time per kernel name (ms) of one call, for the interval kernels."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.load_intervals(fleet, lo, hi, M)
    out = {}
    for ev in prof.key_averages():
        if "interval" in ev.key:
            t = getattr(ev, "device_time_total", None)
            if t is None:
                t = ev.cuda_time_total
            out[ev.key.split("(")[0]] = t / 1e3
    return out


def main(S=10000, A=8, M=64, reps=20, warm=3):
    e = Engine(0)
    fleet = synth_fleet(S, A, seed=42)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    lo, hi = (x * np.float32(0.5)).astype(np.float32), (x * np.float32(2)).astype(np.float32)
    for _ in range(warm):
        e.load_intervals(fleet, lo, hi, M)
    dev, ker, wall = [], [], []
    l0 = e.launch_count
    for _ in range(reps):
        t0 = time.perf_counter()
        count, trunc, start, rec = e.load_intervals(fleet, lo, hi, M)
        wall.append(time.perf_counter() - t0)
        dev.append(e.last_device_ms)
        ker.append(e.last_kernel_ms)
    launches = (e.launch_count - l0) / reps
    per_kernel = kernel_times(e, fleet, lo, hi, M)
    # the same records through the load grid: one level per interval start (shorter lists repeat their last start)
    L = int(count.max())
    rows = np.zeros((L, S), np.float32)
    for s in range(S):
        n = int(count[s])
        rows[:, s] = start[s, n - 1] if n else lo[s]
        rows[:n, s] = start[s, :n]
    e.load_grid(fleet, rows)
    lg_dev, lg_wall = [], []
    for _ in range(5):
        t0 = time.perf_counter()
        _, win = e.load_grid(fleet, rows)
        lg_wall.append(time.perf_counter() - t0)
        lg_dev.append(e.last_device_ms)
    mismatches = 0
    for s in range(S):
        for j in range(int(count[s])):
            i, r = j * S + s, s * M + j
            if any(getattr(win, k)[i:i + 1].tobytes() != getattr(rec, k)[r:r + 1].tobytes() for k in FIELDS):
                mismatches += 1
    name, power = gpu_label()
    print(json.dumps({
        "gpu": name, "power_limit_and_max_sm_clock": power,
        "workload": f"load_intervals synth_fleet({S}, {A}, seed=42), [0.5x, 2x], M = {M}", "calls": reps,
        "device_ms_p50": float(np.median(dev)), "kernel_ms_p50": float(np.median(ker)),
        "host_wall_ms_p50": float(np.median(wall)) * 1e3, "launches_per_call": launches,
        "intervals": int(count.sum()), "max_per_server_found": L, "servers_truncated": int(trunc.sum()),
        "interval_kernels_ms": per_kernel,
        "load_grid_over_starts_levels": L, "load_grid_device_ms_p50": float(np.median(lg_dev)),
        "load_grid_wall_ms_p50": float(np.median(lg_wall)) * 1e3, "record_mismatches": mismatches,
    }))


if __name__ == "__main__":
    main()
