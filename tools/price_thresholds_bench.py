"""wva_price_thresholds on synth_fleet(10000, 8, seed=42) (the configs[3] shape) and synth_fleet(100, 4, seed=42).

Prints one JSON line.  Per shape: the median device / kernel / host time over 20 calls and the launches per call;
price_kernel's device time (torch.profiler, one call); wva_analyze on the same fleet, which is the sizing the
thresholds add to; and the existing alternative, one wva_profile_grid over 64 evenly spaced prices of accelerator 0
(0.25x to 4x its own price).  For the scan it counts the winner changes between adjacent rows, how many of them
the thresholds place exactly (a threshold of accelerator 0 inside the rows' bracket, and `above` equal to the
winner after it, byte for byte), and how many thresholds of accelerator 0 the scan misses (outside its range).  A
change is a new (feasible, accelerator, replicas): while accelerator 0 wins, its cost moves at every row.
Needs a GPU; run from the repository root."""
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


def price_kernel_ms(e, fleet):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.price_thresholds(fleet)
    for ev in prof.key_averages():
        if "price_kernel" in ev.key:
            t = getattr(ev, "device_time_total", None)
            return (t if t is not None else ev.cuda_time_total) / 1e3
    return None


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


def shape(e, S, A, reps=20, warm=3, a=0, rows=64):
    fleet = synth_fleet(S, A, seed=42)
    out = {"shape": f"{S}x{A}"}
    out["thresholds"] = timed(e, lambda: e.price_thresholds(fleet), reps, warm)
    out["price_kernel_ms"] = price_kernel_ms(e, fleet)
    out["analyze"] = timed(e, lambda: e.analyze(fleet), reps, warm)
    th, above, _ = e.price_thresholds(fleet)
    col = th[:, a]
    out["finite_thresholds"] = int((np.isfinite(th) & (th > 0)).sum())
    prices = (fleet.acc_cost[a] * np.linspace(0.25, 4.0, rows)).astype(np.float32)
    acc = np.repeat(fleet.acc_cost[None], rows, axis=0)
    acc[:, a] = prices
    out["profile_grid_64"] = timed(e, lambda: e.profile_grid(fleet, acc_cost=acc), 5, 1)
    _, win = e.profile_grid(fleet, acc_cost=acc)
    w = {k: getattr(win, k).reshape(rows, S) for k in FIELDS}
    changes = exact = 0
    for j in range(rows - 1):
        # a decision change: the winner moves to another accelerator or replica count (its cost moves with a's
        # price at every row while a wins)
        moved = np.zeros(S, bool)
        for k in ("feasible", "acc", "replicas"):
            moved |= w[k][j] != w[k][j + 1]
        for s in np.nonzero(moved)[0]:
            changes += 1
            inside = prices[j] < col[s] <= prices[j + 1]
            same = all(getattr(above, k)[s * A + a].tobytes() == w[k][j + 1, s].tobytes() for k in FIELDS)
            exact += bool(inside and same)
    finite = col[np.isfinite(col) & (col > 0)]
    out["scan"] = {"changes": changes, "placed_exactly": exact,
                   "thresholds_missed": int(((finite <= prices[0]) | (finite > prices[-1])).sum()),
                   "thresholds_of_acc": int(finite.size)}
    return out


def main():
    name, q = gpu_label()
    e = Engine(0)
    res = {"bench": "price_thresholds", "gpu": name, "power_limit_and_max_sm_clock": q,
           "shapes": [shape(e, 10000, 8), shape(e, 100, 4)]}
    e.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
