"""wva_price_threshold_grid / wva_price_threshold_trace on synth_fleet(10000, 8, seed=42) x 24 levels (the rows of
load_grid_bench.py), keepAccelerator off and in WVA's configuration, and on synth_fleet(100, 4, seed=42) x 256.

Prints one JSON line.  Per shape, configuration and call: the median device / kernel / host time over repeated calls
and the launches per call; price_kernel's device time (torch.profiler, a separate call); the same call's
wva_workload_grid / wva_workload_trace alone, which is what the thresholds add to; and the existing way, L single
wva_price_thresholds calls on the row fleets (f_t built with Fleet.apply_winners for the trace), timed, with a
per-row byte comparison of threshold, above and candidates.  The card's name, power limit and maximum SM clock are
read in the same run.  Needs a GPU; run from the repository root."""
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
    """load_grid_bench.py's rows: each server's own load times a seeded log-normal factor per (level, server)."""
    rng = np.random.default_rng(seed)
    return (fleet.srv_arrival_rpm[None, :] * rng.lognormal(0.0, 0.5, (L, fleet.n_servers))).astype(np.float32)


def wva_configuration(fleet, seed):
    """keepAccelerator and min_replicas 1 on every server, each current accelerator a real one with its cost
    (internal/utils/utils.go:290)."""
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


def price_kernel_ms(call):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
    for ev in prof.key_averages():
        if "price_kernel" in ev.key:
            t = getattr(ev, "device_time_total", None)
            return (t if t is not None else ev.cuda_time_total) / 1e3
    return None


def row_fleet(fleet, rpm, l):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_arrival_rpm[:] = rpm[l]
    return f


class _Block(dict):
    """One tick's winner columns, read by attribute as Fleet.apply_winners reads an Allocs."""
    __getattr__ = dict.__getitem__


def run(e, S, A, L, wva, trace, reps, warm=2):
    fleet = synth_fleet(S, A, seed=42)
    if wva:
        wva_configuration(fleet, 42)
    rpm = levels(fleet, L, 7)
    price = e.price_threshold_trace if trace else e.price_threshold_grid
    workload = e.workload_trace if trace else e.workload_grid
    out = {"shape": f"{S}x{A}x{L}", "config": "wva" if wva else "keep_off", "call": "trace" if trace else "grid"}
    out["thresholds"] = timed(e, lambda: price(fleet, rpm), reps, warm)
    out["price_kernel_ms"] = price_kernel_ms(lambda: price(fleet, rpm))
    out["workload_alone"] = timed(e, lambda: workload(fleet, rpm), reps, warm)
    th, above, cand, win = price(fleet, rpm, want_candidates=True)
    # the existing way: L single calls on the row fleets, f_t taking c_t from this call's winners for the trace
    res, cur, dev, t0 = [], fleet, 0.0, time.perf_counter()
    for l in range(L):
        res.append(e.price_thresholds(row_fleet(cur, rpm, l), want_candidates=True))
        dev += e.last_device_ms
        if trace:
            cur = cur.apply_winners(_Block({k: getattr(win, k)[l * S:(l + 1) * S] for k in FIELDS}))
    wall = (time.perf_counter() - t0) * 1e3
    same = 0
    n = S * A
    for l, (th1, above1, cand1) in enumerate(res):
        ok = th[l].tobytes() == th1.tobytes()
        for k in FIELDS:
            ok &= getattr(above, k)[l * n:(l + 1) * n].tobytes() == getattr(above1, k).tobytes()
            ok &= getattr(cand, k)[l * n:(l + 1) * n].tobytes() == getattr(cand1, k).tobytes()
        same += bool(ok)
    out["single_calls"] = {"host_ms": wall, "device_ms": dev, "rows_byte_identical": same, "rows": L}
    out["finite_thresholds"] = int((np.isfinite(th) & (th > 0)).sum())
    return out


def main():
    name, q = gpu_label()
    e = Engine(0)
    res = {"bench": "price_levels", "gpu": name, "power_limit_and_max_sm_clock": q, "runs": []}
    for wva in (False, True):
        for trace in (False, True):
            res["runs"].append(run(e, 10000, 8, 24, wva, trace, reps=10))
    for trace in (False, True):
        res["runs"].append(run(e, 100, 4, 256, False, trace, reps=10))
    e.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
