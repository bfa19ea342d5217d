"""wva_profile_trace on four shapes:
1. synth_fleet(10000, 8, seed=42) x 24 ticks: workload_trace_bench.py's rows plus an hourly price curve per
   accelerator;
2. shape 1 in WVA's configuration (keepAccelerator on every server, every current accelerator a real one with its
   cost, min_replicas 1);
3. shape 1 plus accelerator 7 switched on at tick 12 (perf_present 0 before) and beta x 0.9 on accelerator 3 from
   tick 8;
4. synth_fleet(100, 4, seed=42) x 256 ticks with price rows.

Prints one JSON line: per shape, the median device / kernel / host time over repeated calls, the launches per call,
the keys the call sizes, wva_workload_trace on the same workload rows (the price of the profile dimension), and the
same answer obtained the existing way (per tick, Fleet.apply_winners of the previous tick's winners and one wva_solve
on f_t), timed, with a per-tick byte comparison against the trace.  Needs a GPU; run from the repository root."""
import json
import sys
import time

import numpy as np

sys.path.insert(0, ".")
sys.path.insert(0, "tools")
from workload_trace_bench import FIELDS, gpu_label, ticks, timed, wva_configuration  # noqa: E402
from workload_variant_autoscaler_b200 import Engine, synth_fleet  # noqa: E402

LOAD_COLUMN = {"arrival_rpm": "srv_arrival_rpm", "in_tokens": "srv_in_tokens", "out_tokens": "srv_out_tokens"}


def hourly_prices(fleet, L, seed):
    """acc_cost [L, A]: a daily curve per accelerator with its own phase and depth, plus noise."""
    rng = np.random.default_rng(seed)
    A = fleet.n_acc
    t = np.arange(L)[:, None]
    phase, depth = rng.uniform(0, 2 * np.pi, A), rng.uniform(0.2, 0.8, A)
    curve = 1.0 + depth * np.sin(2 * np.pi * t / 24.0 + phase) + rng.normal(0, 0.03, (L, A))
    return (fleet.acc_cost[None] * np.maximum(curve, 0.05)).astype(np.float32)


def at_tick(fleet, rows, t):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    for k, v in rows.items():
        getattr(f, LOAD_COLUMN.get(k, k))[:] = v[t]
    f.unlimited = True
    return f


def keys_sized(fleet, rows, L):
    """Distinct (s, a, in, out, bits of alpha .. delta, N) over the (tick, pair) loads, pinned servers on their
    current pair only (wva_profile_trace's keys)."""
    S, A = fleet.n_servers, fleet.n_acc
    col = lambda k: rows[k] if k in rows else np.broadcast_to(getattr(fleet, LOAD_COLUMN.get(k, k))[None],  # noqa
                                                              (L,) + getattr(fleet, LOAD_COLUMN.get(k, k)).shape)
    rpm, tin, tout = col("arrival_rpm"), col("in_tokens"), col("out_tokens")
    m = fleet.srv_model
    ok = (m >= 0) & (fleet.srv_has_target != 0)
    mm = np.maximum(m, 0)
    cur = fleet.srv_cur_acc
    pin = (fleet.srv_keep_acc != 0) & (cur != -1) & ((cur == -2) | (fleet.srv_min_replicas != 0))
    allowed = np.where(pin[:, None], np.arange(A)[None] == cur[:, None], True)
    load = ~(rpm < 0) & (rpm != 0) & (tin >= 0) & (tout >= 1) & ok[None]
    per = {k: col(k)[:, mm, :] for k in ("perf_present", "perf_alpha", "perf_beta", "perf_gamma", "perf_delta",
                                         "perf_max_batch", "perf_at_tokens")}  # [L, S, A]
    live = load[:, :, None] & (per["perf_present"] != 0) & allowed[None]
    t_, s_, a_ = np.nonzero(live)
    out = tout[t_, s_].astype(np.int64)
    n = (per["perf_max_batch"][t_, s_, a_].astype(np.int64) * per["perf_at_tokens"][t_, s_, a_]) // out
    n = np.where(fleet.srv_max_batch[s_] > 0, fleet.srv_max_batch[s_], np.maximum(n, 1))
    bits = [per[k][t_, s_, a_].astype(np.float32).view(np.uint32).astype(np.int64)
            for k in ("perf_alpha", "perf_beta", "perf_gamma", "perf_delta")]
    key = np.stack([s_, a_, tin[t_, s_], out, *bits, n], axis=1)
    return int(len(np.unique(key, axis=0))) if len(key) else 0


def solve_loop(e, fleet, rows, L, want=False):
    cur, out = fleet, []
    for t in range(L):
        cand, win = e.solve(at_tick(cur, rows, t), want_candidates=want)
        if want:
            out.append((cand, win))
        cur = cur.apply_winners(win)
    return out


def run_shape(e, label, fleet, L, rows, reps, base_reps, warm=3):
    S, A = fleet.n_servers, fleet.n_acc
    dev, ker, wall, launches = timed(e, lambda: e.profile_trace(fleet, **rows), reps, warm)
    load = [rows[k] for k in LOAD_COLUMN]
    wdev, wker, wwall, wlaunches = timed(e, lambda: e.workload_trace(fleet, *load), reps, warm)
    solve_loop(e, fleet, rows, min(L, warm))
    base_wall = []
    for _ in range(base_reps):
        t0 = time.perf_counter()
        solve_loop(e, fleet, rows, L)
        base_wall.append(time.perf_counter() - t0)
    cand, win = e.profile_trace(fleet, **rows, want_candidates=True)
    per_tick = solve_loop(e, fleet, rows, L, want=True)
    mismatched = [t for t, (c, w) in enumerate(per_tick)
                  if not all(getattr(cand, k)[t * S * A:(t + 1) * S * A].tobytes() == getattr(c, k).tobytes() and
                             getattr(win, k)[t * S:(t + 1) * S].tobytes() == getattr(w, k).tobytes() for k in FIELDS)]
    acc = win.acc.reshape(L, S)
    fe = win.feasible.reshape(L, S) != 0
    moves = int((fe[1:] & fe[:-1] & (acc[1:] != acc[:-1])).sum())
    med_base = float(np.median(base_wall)) * 1e3
    return {
        "workload": f"profile_trace {label} x {L} ticks", "pairs": S * A, "ticks": L, "calls": reps,
        "keys_sized": keys_sized(fleet, rows, L), "device_ms_p50": dev, "kernel_ms_p50": ker, "host_wall_ms_p50": wall,
        "launches_per_call": launches, "solve_loop_wall_ms_p50": med_base, "solve_loop_reps": base_reps,
        "speedup_wall": med_base / wall,
        "workload_trace_same_load": {"device_ms_p50": wdev, "kernel_ms_p50": wker, "host_wall_ms_p50": wwall,
                                     "launches_per_call": wlaunches},
        "feasible_winners": int(win.feasible.sum()), "accelerator_moves": moves, "tick_mismatches": len(mismatched),
    }


def shape_rows(fleet, L, seed):
    rpm, in_tok, out_tok = ticks(fleet, L, 7)
    return {"arrival_rpm": rpm, "in_tokens": in_tok, "out_tokens": out_tok, "acc_cost": hourly_prices(fleet, L, seed)}


def main():
    e = Engine(0)
    big = synth_fleet(10000, 8, seed=42)
    wva = wva_configuration(synth_fleet(10000, 8, seed=42), 5)
    small = synth_fleet(100, 4, seed=42)
    rows3 = shape_rows(big, 24, 11)
    for k in ("perf_present", "perf_beta"):
        rows3[k] = np.repeat(getattr(big, k)[None], 24, axis=0).copy()
    rows3["perf_present"][:12, :, 7] = 0
    rows3["perf_beta"][8:, :, 3] *= np.float32(0.9)
    shapes = [
        run_shape(e, "synth_fleet(10000, 8, seed=42), hourly prices", big, 24, shape_rows(big, 24, 11), 20, 3),
        run_shape(e, "synth_fleet(10000, 8, seed=42), hourly prices, WVA configuration", wva, 24,
                  shape_rows(wva, 24, 11), 20, 3),
        run_shape(e, "synth_fleet(10000, 8, seed=42), hourly prices, accelerator 7 on at tick 12, beta x 0.9 on "
                  "accelerator 3 from tick 8", big, 24, rows3, 20, 3),
        run_shape(e, "synth_fleet(100, 4, seed=42), hourly prices", small, 256, shape_rows(small, 256, 13), 20, 3),
    ]
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "shapes": shapes}))


if __name__ == "__main__":
    main()
