"""wva_slo_bounds on synth_fleet(10000, 8, seed=42) (the configs[3] shape) and synth_fleet(100, 4, seed=42).

Prints one JSON line.  Per shape: the median device / kernel / host time over 20 calls and the launches per call;
the device time of each of the call's kernels (torch.profiler, one call); wva_analyze on the same fleet; and the
sampled alternative, one wva_slo_grid of 64 rows along one ITL axis (each server's own ITL target times 0.25 ..
4, geometric), which cannot give the breakpoints.  Needs a GPU; run from the repository root."""
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
from workload_variant_autoscaler_b200 import Engine, synth_fleet  # noqa: E402

KERNELS = ("build_pair_tables", "bounds_tail", "bounds_fallback", "bounds_kernel")


def gpu_label():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # the label is informative only
        q = "unknown"
    return name, q


def kernel_split(e, fleet):
    """Device ms per kernel of one call, by name."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.slo_bounds(fleet)
    out = {}
    for ev in prof.key_averages():
        for k in KERNELS:
            if k in ev.key:
                t = getattr(ev, "device_time_total", None)
                out[k] = out.get(k, 0.0) + (t if t is not None else ev.cuda_time_total) / 1e3
    return out


def timed(e, call, reps, warm):
    for _ in range(warm):
        call()
    dev, ker, wall = [], [], []
    l0 = e.launch_count
    for _ in range(reps):
        t0 = time.perf_counter()
        call()
        wall.append(time.perf_counter() - t0)
        dev.append(e.last_device_ms)
        ker.append(e.last_kernel_ms)
    return {"device_ms": float(np.median(dev)), "kernel_ms": float(np.median(ker)),
            "host_ms": float(np.median(wall)) * 1e3, "launches": (e.launch_count - l0) // reps}


def shape(e, S, A, reps=20, warm=3, rows=64):
    fleet = synth_fleet(S, A, seed=42)
    out = {"shape": f"{S}x{A}"}
    out["bounds"] = timed(e, lambda: e.slo_bounds(fleet), reps, warm)
    out["kernels_ms"] = kernel_split(e, fleet)
    kind = e.slo_bounds(fleet)[0]
    out["entries_by_kind"] = [int((kind == k).sum()) for k in range(4)]
    out["analyze"] = timed(e, lambda: e.analyze(fleet), reps, warm)
    itl = (fleet.srv_slo_itl[None, :] * np.geomspace(0.25, 4.0, rows)[:, None]).astype(np.float32)
    ttft = np.broadcast_to(fleet.srv_slo_ttft, itl.shape).astype(np.float32)
    tps = np.broadcast_to(fleet.srv_slo_tps, itl.shape).astype(np.float32)
    out["slo_grid_64"] = timed(e, lambda: e.slo_grid(fleet, itl, ttft, tps), 5, 1)
    return out


def main():
    name, q = gpu_label()
    e = Engine(0)
    res = {"bench": "slo_bounds", "gpu": name, "power_limit_and_max_sm_clock": q,
           "shapes": [shape(e, 10000, 8), shape(e, 100, 4)]}
    e.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
