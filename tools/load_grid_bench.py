"""wva_load_grid on two shapes: synth_fleet(10000, 8, seed=42) x 24 load levels, and synth_fleet(100, 4) x 256.

Each level is the fleet's own load times a seeded log-normal factor per (level, server), the shape of a load
forecast.  Prints one JSON line: per shape, the median device / kernel / host time over repeated calls and the
launches per call, then the same answer obtained the existing way (one wva_update_load + wva_resolve per level on a
resident fleet), timed, with a per-level byte comparison of candidates and winners against the load grid.  Needs a
GPU; run from the repository root."""
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


def levels(fleet, L, seed):
    rng = np.random.default_rng(seed)
    return (fleet.srv_arrival_rpm[None, :] * rng.lognormal(0.0, 0.5, (L, fleet.n_servers))).astype(np.float32)


def same_block(got, lo, hi, want):
    return all(getattr(got, k)[lo:hi].tobytes() == getattr(want, k).tobytes() for k in FIELDS)


def run_shape(e, S, A, L, reps, base_reps, warm=3):
    fleet = synth_fleet(S, A, seed=42)
    rpm = levels(fleet, L, 7)
    for _ in range(warm):
        e.load_grid(fleet, rpm)
    dev, ker, wall = [], [], []
    l0 = e.launch_count
    for _ in range(reps):
        t0 = time.perf_counter()
        e.load_grid(fleet, rpm)
        wall.append(time.perf_counter() - t0)
        dev.append(e.last_device_ms)
        ker.append(e.last_kernel_ms)
    launches = (e.launch_count - l0) / reps
    # the existing way: update_load + resolve per level on the resident fleet
    e.upload(fleet)
    for l in range(min(L, warm)):
        e.update_load(arrival_rpm=rpm[l])
        e.resolve()
    base_wall, base_dev = [], []
    for _ in range(base_reps):
        t0 = time.perf_counter()
        d = 0.0
        for l in range(L):
            e.update_load(arrival_rpm=rpm[l])
            e.resolve()
            d += e.last_device_ms
        base_wall.append(time.perf_counter() - t0)
        base_dev.append(d)
    # per-level byte comparison
    cand, win = e.load_grid(fleet, rpm, want_candidates=True)
    e.upload(fleet)
    mismatched = []
    for l in range(L):
        e.update_load(arrival_rpm=rpm[l])
        c, w = e.resolve(want_candidates=True)
        if not (same_block(cand, l * S * A, (l + 1) * S * A, c) and same_block(win, l * S, (l + 1) * S, w)):
            mismatched.append(l)
    med_wall, med_base = float(np.median(wall)) * 1e3, float(np.median(base_wall)) * 1e3
    return {
        "workload": f"load_grid synth_fleet({S}, {A}, seed=42) x {L} levels", "pairs": S * A, "levels": L,
        "calls": reps, "device_ms_p50": float(np.median(dev)), "kernel_ms_p50": float(np.median(ker)),
        "host_wall_ms_p50": med_wall, "launches_per_call": launches,
        "resolve_levels_wall_ms_p50": med_base, "resolve_levels_device_ms_p50": float(np.median(base_dev)),
        "resolve_levels_reps": base_reps, "speedup_wall": med_base / med_wall,
        "feasible_candidates": int(cand.feasible.sum()), "level_mismatches": len(mismatched),
    }


def main():
    e = Engine(0)
    shapes = [run_shape(e, 10000, 8, 24, reps=20, base_reps=5), run_shape(e, 100, 4, 256, reps=20, base_reps=3)]
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "shapes": shapes}))


if __name__ == "__main__":
    main()
