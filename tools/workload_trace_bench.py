"""wva_workload_trace on three shapes: synth_fleet(10000, 8, seed=42) x 24 ticks as synthesised (keepAccelerator off),
the same in WVA's configuration (keepAccelerator on every server, every current accelerator a real one with its
cost, min_replicas 1), and synth_fleet(100, 4) x 256 ticks.

The ticks are workload_grid_bench.py's levels: the fleet's own load with the arrival rate times a seeded log-normal
factor per (tick, server), and out_tokens drawn from {0.75, 1, 1.5} x the server's own.  Prints one JSON line: per
shape, the median device / kernel / host time over repeated calls, the launches per call, the (server, accelerator)
pairs the trace sizes against the workload grid's, and the same answer obtained the existing way (per tick,
Fleet.apply_winners of the previous tick's winners and one wva_solve), timed, with a per-tick byte comparison against
the trace.  Needs a GPU; run from the repository root."""
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


def ticks(fleet, L, seed):
    rng = np.random.default_rng(seed)
    S = fleet.n_servers
    rpm = (fleet.srv_arrival_rpm[None, :] * rng.lognormal(0.0, 0.5, (L, S))).astype(np.float32)
    in_tok = np.broadcast_to(fleet.srv_in_tokens, (L, S)).astype(np.int32)
    out_f = rng.choice([0.75, 1.0, 1.5], (L, S))
    out_tok = np.maximum(fleet.srv_out_tokens[None, :] * out_f, 1).astype(np.int32)
    return rpm, in_tok, out_tok


def wva_configuration(fleet, seed):
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


def pairs_sized(fleet):
    """Pairs with a profile that the trace sizes (the pinned rule of wva_workload_trace) and that the grid sizes."""
    cur = fleet.srv_cur_acc
    pin = (fleet.srv_keep_acc != 0) & (cur != -1) & ((cur == -2) | (fleet.srv_min_replicas != 0))
    ok = (fleet.srv_model >= 0) & (fleet.srv_has_target != 0)
    prof = fleet.perf_present[np.maximum(fleet.srv_model, 0)] != 0  # [S, A]
    A = fleet.n_acc
    own = np.arange(A)[None, :] == cur[:, None]
    keep_mask = (fleet.srv_keep_acc != 0)[:, None] & (cur != -1)[:, None] & ~own
    trace = prof & ok[:, None] & np.where(pin[:, None], own, True)
    grid = prof & ok[:, None] & ~keep_mask
    return int(trace.sum()), int(grid.sum())


def tick_of(allocs, t, S):
    return np.rec.fromarrays([getattr(allocs, k)[t * S:(t + 1) * S] for k in FIELDS], names=",".join(FIELDS))


def at_tick(fleet, rpm, in_tok, out_tok):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_arrival_rpm[:], f.srv_in_tokens[:], f.srv_out_tokens[:] = rpm, in_tok, out_tok
    return f


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


def solve_loop(e, fleet, rows, L, want=False):
    """The existing way: per tick, wva_solve on the fleet advanced by the previous winners."""
    cur, out, dev = fleet, [], 0.0
    for t in range(L):
        cand, win = e.solve(at_tick(cur, rows[0][t], rows[1][t], rows[2][t]), want_candidates=want)
        dev += e.last_device_ms
        if want:
            out.append((cand, win))
        cur = cur.apply_winners(win)
    return out, dev


def run_shape(e, label, fleet, L, reps, base_reps, warm=3):
    S, A = fleet.n_servers, fleet.n_acc
    rows = ticks(fleet, L, 7)
    dev, ker, wall, launches = timed(e, lambda: e.workload_trace(fleet, *rows), reps, warm)
    gdev, gker, gwall, glaunches = timed(e, lambda: e.workload_grid(fleet, *rows), reps, warm)
    solve_loop(e, fleet, rows, min(L, warm))
    base_wall, base_dev = [], []
    for _ in range(base_reps):
        t0 = time.perf_counter()
        _, d = solve_loop(e, fleet, rows, L)
        base_wall.append(time.perf_counter() - t0)
        base_dev.append(d)
    # per-tick byte comparison
    cand, win = e.workload_trace(fleet, *rows, want_candidates=True)
    per_tick, _ = solve_loop(e, fleet, rows, L, want=True)
    mismatched = [t for t, (c, w) in enumerate(per_tick)
                  if not all(getattr(cand, k)[t * S * A:(t + 1) * S * A].tobytes() == getattr(c, k).tobytes() and
                             getattr(win, k)[t * S:(t + 1) * S].tobytes() == getattr(w, k).tobytes() for k in FIELDS)]
    moves = sum(int(((tick_of(win, t, S).feasible != 0) & (tick_of(win, t - 1, S).feasible != 0) &
                     (tick_of(win, t, S).acc != tick_of(win, t - 1, S).acc)).sum()) for t in range(1, L))
    trace_pairs, grid_pairs = pairs_sized(fleet)
    med_base = float(np.median(base_wall)) * 1e3
    return {
        "workload": f"workload_trace {label} x {L} ticks, out_tokens x {{0.75, 1, 1.5}}",
        "pairs": S * A, "ticks": L, "calls": reps, "pairs_sized": trace_pairs, "grid_pairs_sized": grid_pairs,
        "device_ms_p50": dev, "kernel_ms_p50": ker, "host_wall_ms_p50": wall, "launches_per_call": launches,
        "solve_loop_wall_ms_p50": med_base, "solve_loop_device_ms_p50": float(np.median(base_dev)),
        "solve_loop_reps": base_reps, "speedup_wall": med_base / wall,
        "workload_grid_same_rows": {"device_ms_p50": gdev, "kernel_ms_p50": gker, "host_wall_ms_p50": gwall,
                                    "launches_per_call": glaunches},
        "feasible_winners": int(win.feasible.sum()), "accelerator_moves": moves, "tick_mismatches": len(mismatched),
    }


def main():
    e = Engine(0)
    shapes = [
        run_shape(e, "synth_fleet(10000, 8, seed=42), keep off", synth_fleet(10000, 8, seed=42), 24, 20, 3),
        run_shape(e, "synth_fleet(10000, 8, seed=42), WVA configuration",
                  wva_configuration(synth_fleet(10000, 8, seed=42), 5), 24, 20, 3),
        run_shape(e, "synth_fleet(100, 4, seed=42)", synth_fleet(100, 4, seed=42), 256, 20, 3),
    ]
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "shapes": shapes}))


if __name__ == "__main__":
    main()
