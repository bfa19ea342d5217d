"""wva_workload_grid on two shapes: synth_fleet(10000, 8, seed=42) x 24 levels, and synth_fleet(100, 4) x 256.

Each level is the fleet's own load with the arrival rate times a seeded log-normal factor per (level, server), as in
load_grid_bench.py, and out_tokens drawn from {0.75, 1, 1.5} x the server's own per (level, server): a forecast in
which answers get shorter or longer, with at most 3 token keys per server.  Prints one JSON line: per shape, the
median device / kernel / host time over repeated calls and the launches per call, the number of token keys against
L * S, the same answer obtained the existing way (one wva_update_load + wva_resolve per level on a resident fleet),
timed, with a per-level byte comparison against the workload grid, and wva_load_grid at the same rates with the
tokens fixed (what the token dimension costs).  Needs a GPU; run from the repository root."""
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
    S = fleet.n_servers
    rpm = (fleet.srv_arrival_rpm[None, :] * rng.lognormal(0.0, 0.5, (L, S))).astype(np.float32)
    in_tok = np.broadcast_to(fleet.srv_in_tokens, (L, S)).astype(np.int32)
    out_f = rng.choice([0.75, 1.0, 1.5], (L, S))
    out_tok = np.maximum(fleet.srv_out_tokens[None, :] * out_f, 1).astype(np.int32)
    return rpm, in_tok, out_tok


def n_keys(rpm, in_tok, out_tok):
    """Distinct (server, in, out) over the levels where the server is a load."""
    L, S = rpm.shape
    load = ~(rpm < 0) & (rpm != 0) & (in_tok >= 0) & (out_tok >= 1)
    srv = np.broadcast_to(np.arange(S), (L, S))
    keys = np.stack([srv[load], in_tok[load], out_tok[load]], axis=1)
    return int(np.unique(keys, axis=0).shape[0]) if keys.size else 0


def same_block(got, lo, hi, want):
    return all(getattr(got, k)[lo:hi].tobytes() == getattr(want, k).tobytes() for k in FIELDS)


def timed(e, fn, reps, warm):
    for _ in range(warm):
        fn()
    dev, ker, wall = [], [], []
    l0 = e.launch_count
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        wall.append(time.perf_counter() - t0)
        dev.append(e.last_device_ms)
        ker.append(e.last_kernel_ms)
    return (float(np.median(dev)), float(np.median(ker)), float(np.median(wall)) * 1e3,
            (e.launch_count - l0) / reps)


def run_shape(e, S, A, L, reps, base_reps, warm=3):
    fleet = synth_fleet(S, A, seed=42)
    rpm, in_tok, out_tok = levels(fleet, L, 7)
    dev, ker, wall, launches = timed(e, lambda: e.workload_grid(fleet, rpm, in_tok, out_tok), reps, warm)
    lg_dev, lg_ker, lg_wall, lg_launches = timed(e, lambda: e.load_grid(fleet, rpm), reps, warm)
    # the existing way: update_load + resolve per level on the resident fleet
    e.upload(fleet)
    for l in range(min(L, warm)):
        e.update_load(rpm[l], in_tok[l], out_tok[l])
        e.resolve()
    base_wall, base_dev = [], []
    for _ in range(base_reps):
        t0 = time.perf_counter()
        d = 0.0
        for l in range(L):
            e.update_load(rpm[l], in_tok[l], out_tok[l])
            e.resolve()
            d += e.last_device_ms
        base_wall.append(time.perf_counter() - t0)
        base_dev.append(d)
    # per-level byte comparison
    cand, win = e.workload_grid(fleet, rpm, in_tok, out_tok, want_candidates=True)
    e.upload(fleet)
    mismatched = []
    for l in range(L):
        e.update_load(rpm[l], in_tok[l], out_tok[l])
        c, w = e.resolve(want_candidates=True)
        if not (same_block(cand, l * S * A, (l + 1) * S * A, c) and same_block(win, l * S, (l + 1) * S, w)):
            mismatched.append(l)
    med_base = float(np.median(base_wall)) * 1e3
    return {
        "workload": f"workload_grid synth_fleet({S}, {A}, seed=42) x {L} levels, out_tokens x {{0.75, 1, 1.5}}",
        "pairs": S * A, "levels": L, "calls": reps, "keys": n_keys(rpm, in_tok, out_tok), "level_servers": L * S,
        "device_ms_p50": dev, "kernel_ms_p50": ker, "host_wall_ms_p50": wall, "launches_per_call": launches,
        "resolve_levels_wall_ms_p50": med_base, "resolve_levels_device_ms_p50": float(np.median(base_dev)),
        "resolve_levels_reps": base_reps, "speedup_wall": med_base / wall,
        "load_grid_same_rates": {"device_ms_p50": lg_dev, "kernel_ms_p50": lg_ker, "host_wall_ms_p50": lg_wall,
                                 "launches_per_call": lg_launches},
        "feasible_candidates": int(cand.feasible.sum()), "level_mismatches": len(mismatched),
    }


def main():
    e = Engine(0)
    shapes = [run_shape(e, 10000, 8, 24, reps=20, base_reps=5), run_shape(e, 100, 4, 256, reps=20, base_reps=3)]
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "shapes": shapes}))


if __name__ == "__main__":
    main()
