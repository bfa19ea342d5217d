"""wva_size_grid at config-2 shape: 100 servers x 4 accelerators x batch sizes 1..256 (102,400 size candidates).

Prints one JSON line: median device / kernel time over repeated calls, launches per call, size candidates per
second, the same answer obtained the other way (one wva_solve per batch size with srv_max_batch overwritten), and
the C oracle's size candidates per second on one core over a sample of the candidates (which the GPU result must
match bit for bit).  Needs a GPU; run from the repository root."""
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
import oracle  # noqa: E402
from workload_variant_autoscaler_b200 import Engine, synth_fleet  # noqa: E402

INT_FIELDS = ("feasible", "acc", "replicas", "batch")
FLOAT_FIELDS = ("cost", "value", "itl", "ttft", "rho", "max_rate")


def with_batch(fleet, b):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_max_batch[:] = b
    return f


def gpu_label():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # the label is informative only
        q = "unknown"
    return name, q


def main(reps=20, warm=3):
    fleet = synth_fleet(100, 4, seed=42)
    batches = np.arange(1, 257, dtype=np.int32)
    S, A, B = fleet.n_servers, fleet.n_acc, batches.size
    e = Engine(0)
    for _ in range(warm):
        cand, _ = e.size_grid(fleet, batches, want_candidates=True)
    dev, ker, wall = [], [], []
    l0 = e.launch_count
    for _ in range(reps):
        t0 = time.perf_counter()
        e.size_grid(fleet, batches)
        wall.append(time.perf_counter() - t0)
        dev.append(e.last_device_ms)
        ker.append(e.last_kernel_ms)
    launches = (e.launch_count - l0) / reps
    # the same candidates the other way: one solve per batch size
    fleets = [with_batch(fleet, int(b)) for b in batches]
    for f in fleets[:2]:
        e.solve(f, want_candidates=False)
    t0 = time.perf_counter()
    for f in fleets:
        e.solve(f, want_candidates=False)
    per_batch_ms = (time.perf_counter() - t0) * 1e3
    # the C oracle on one core over a sample: every 10th server, every 32nd batch size
    oracle.build()
    s_idx, b_idx = np.arange(0, S, 10), np.arange(0, B, 32)
    sample = fleet.take_servers(s_idx)
    t0 = time.perf_counter()
    ref = [oracle.calculate(with_batch(sample, int(batches[bi]))) for bi in b_idx]
    oracle_s = time.perf_counter() - t0
    n_sample = s_idx.size * A * b_idx.size
    mismatches = 0
    for k, bi in enumerate(b_idx):
        for i, s in enumerate(s_idx):
            for a in range(A):
                j = (s * A + a) * B + bi
                same = all(int(getattr(cand, n)[j]) == int(ref[k][i, a][n]) for n in INT_FIELDS) and all(
                    np.float32(getattr(cand, n)[j]).tobytes() == np.float32(ref[k][i, a][n]).tobytes()
                    for n in FLOAT_FIELDS)
                mismatches += int(not same)
    name, power = gpu_label()
    n = S * A * B
    med_dev, med_ker = float(np.median(dev)), float(np.median(ker))
    print(json.dumps({
        "workload": "size_grid synth_fleet(100, 4, seed=42) x batch 1..256", "gpu": name,
        "power_limit_and_max_sm_clock": power, "size_candidates": n, "calls": reps,
        "device_ms_p50": med_dev, "kernel_ms_p50": med_ker, "host_wall_ms_p50": float(np.median(wall)) * 1e3,
        "launches_per_call": launches, "candidates_per_s_device": n / (med_dev * 1e-3),
        "per_batch_solve_ms": per_batch_ms,
        "oracle_candidates_per_s_1core": n_sample / oracle_s, "oracle_sample": n_sample,
        "sample_mismatches": mismatches,
    }))


if __name__ == "__main__":
    main()
