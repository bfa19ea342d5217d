"""wva_slo_grid on two shapes: synth_fleet(10000, 8, seed=42) x a 4 x 4 ITL x TTFT grid, and synth_fleet(100, 4) x
8 x 8.

Row (i, j) of a grid holds each server's own ITL target times factor i and its own TTFT target times factor j (TPS
unchanged): the question "what does a tighter or looser ITL / TTFT cost across the fleet".  Prints one JSON line: per
shape, the median device / kernel / host time over repeated calls, the launches per call, the searches run against
the 2 L (load pairs) a per-level solve runs, and the tail kernel's own device time (torch.profiler, a separate call);
then the same answer obtained the existing way (one wva_solve per level on a copy of the fleet with the level's
srv_slo_* columns), timed, with a per-level byte comparison of candidates and winners.  Needs a GPU; run from the
repository root."""
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


def cartesian(fleet, factors):
    """(itl, ttft, tps), each [len(factors)^2, S]: row i * n + j = (ITL x factors[i], TTFT x factors[j], own TPS)."""
    f = np.asarray(factors, np.float32)
    n = f.size
    itl = np.repeat(fleet.srv_slo_itl[None, :] * f[:, None], n, axis=0)
    ttft = np.tile(fleet.srv_slo_ttft[None, :] * f[:, None], (n, 1))
    tps = np.repeat(fleet.srv_slo_tps[None, :], n * n, axis=0)
    return tuple(np.ascontiguousarray(x, np.float32) for x in (itl, ttft, tps))


def load_pairs(fleet):
    """Load pairs per server (the gates of CreateAllocation with keepAccelerator, at the fleet's own load)."""
    S, A = fleet.n_servers, fleet.n_acc
    n = np.zeros(S, np.int64)
    for s in range(S):
        m = int(fleet.srv_model[s])
        if (fleet.srv_arrival_rpm[s] <= 0 or fleet.srv_in_tokens[s] < 0 or fleet.srv_out_tokens[s] <= 0
                or not fleet.srv_has_target[s] or m < 0 or m >= fleet.n_models):
            continue
        for a in range(A):
            if fleet.srv_keep_acc[s] and fleet.srv_cur_acc[s] != -1 and fleet.srv_cur_acc[s] != a:
                continue
            n[s] += int(fleet.perf_present[m, a] != 0)
    return n


def searches(fleet, rows):
    """Searches the grid runs: per server, its distinct positive TTFT and ITL targets over the levels whose three
    targets are not negative, times its load pairs."""
    itl, ttft, tps = rows
    n = load_pairs(fleet)
    total = 0
    for s in range(fleet.n_servers):
        ok = ~((itl[:, s] < 0) | (ttft[:, s] < 0) | (tps[:, s] < 0))
        keys = {(w, float(t)) for w, col in ((0, ttft), (1, itl)) for t in col[ok, s] if t > 0}
        total += len(keys) * int(n[s])
    return total, 2 * itl.shape[0] * int(n.sum())


def tail_ms(e, fleet, rows):
    """Device time (ms) of slo_kernel in one call."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.slo_grid(fleet, *rows)
    t = 0.0
    for ev in prof.key_averages():
        if "slo_kernel" in ev.key:
            d = getattr(ev, "device_time_total", None)
            t += (d if d is not None else ev.cuda_time_total) / 1e3
    return t


def at_level(fleet, rows, l):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_slo_itl[:], f.srv_slo_ttft[:], f.srv_slo_tps[:] = rows[0][l], rows[1][l], rows[2][l]
    f.unlimited = True
    return f


def same_block(got, lo, hi, want):
    return all(getattr(got, k)[lo:hi].tobytes() == getattr(want, k).tobytes() for k in FIELDS)


def run_shape(e, S, A, factors, reps, base_reps, warm=3):
    fleet = synth_fleet(S, A, seed=42)
    rows = cartesian(fleet, factors)
    L = rows[0].shape[0]
    for _ in range(warm):
        e.slo_grid(fleet, *rows)
    dev, ker, wall = [], [], []
    l0 = e.launch_count
    for _ in range(reps):
        t0 = time.perf_counter()
        e.slo_grid(fleet, *rows)
        wall.append(time.perf_counter() - t0)
        dev.append(e.last_device_ms)
        ker.append(e.last_kernel_ms)
    launches = (e.launch_count - l0) / reps
    tail = tail_ms(e, fleet, rows)
    # the existing way: one wva_solve per level on a copy of the fleet with the level's targets
    fl = [at_level(fleet, rows, l) for l in range(L)]
    for l in range(min(L, warm)):
        e.solve(fl[l], want_candidates=False)
    base_wall, base_dev = [], []
    for _ in range(base_reps):
        t0 = time.perf_counter()
        d = 0.0
        for l in range(L):
            e.solve(fl[l], want_candidates=False)
            d += e.last_device_ms
        base_wall.append(time.perf_counter() - t0)
        base_dev.append(d)
    # per-level byte comparison
    cand, win = e.slo_grid(fleet, *rows, want_candidates=True)
    mismatched = []
    for l in range(L):
        c, w = e.solve(fl[l])
        if not (same_block(cand, l * S * A, (l + 1) * S * A, c) and same_block(win, l * S, (l + 1) * S, w)):
            mismatched.append(l)
    run, per_level = searches(fleet, rows)
    med_wall, med_base = float(np.median(wall)) * 1e3, float(np.median(base_wall)) * 1e3
    n = len(factors)
    return {
        "workload": f"slo_grid synth_fleet({S}, {A}, seed=42) x {n} x {n} ITL x TTFT", "pairs": S * A, "levels": L,
        "calls": reps, "device_ms_p50": float(np.median(dev)), "kernel_ms_p50": float(np.median(ker)),
        "host_wall_ms_p50": med_wall, "launches_per_call": launches, "tail_kernel_ms": tail,
        "searches_run": run, "searches_per_level_solves": per_level,
        "solve_levels_wall_ms_p50": med_base, "solve_levels_device_ms_p50": float(np.median(base_dev)),
        "solve_levels_reps": base_reps, "speedup_wall": med_base / med_wall,
        "feasible_candidates": int(cand.feasible.sum()), "level_mismatches": len(mismatched),
    }


def main():
    e = Engine(0)
    shapes = [run_shape(e, 10000, 8, (0.5, 0.75, 1.5, 2.0), reps=20, base_reps=5),
              run_shape(e, 100, 4, tuple(np.geomspace(0.5, 2.0, 8).astype(np.float32)), reps=20, base_reps=3)]
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "shapes": shapes}))


if __name__ == "__main__":
    main()
