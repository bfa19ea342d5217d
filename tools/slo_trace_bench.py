"""wva_slo_trace on three shapes: synth_fleet(10000, 8, seed=42) x 24 ticks as synthesised (keepAccelerator off),
the same in WVA's configuration (keepAccelerator on every server, every current accelerator a real one with its cost,
min_replicas 1), and synth_fleet(100, 4, seed=42) x 256 ticks.

The load is workload_trace_bench.py's (arrival rate times a seeded log-normal factor per (tick, server), out_tokens
from {0.75, 1, 1.5} x the server's own), and the targets follow a time-of-day schedule: each server's own ITL x 0.75
in ticks 8-19 of every 24 and its own TTFT x 1.5 in ticks 0-5, its own TPS throughout.  Prints one JSON line: per
shape, the median device / kernel / host time over repeated calls, the launches per call, the searches the call runs
against the 2 x L x (pairs sized) a per-tick solve runs, wva_workload_trace on the same load (the price of the SLO
axis), and the same answer obtained the existing way (per tick, Fleet.apply_winners of the previous tick's winners and
one wva_solve on the fleet with all six columns overwritten), timed, with a per-tick byte comparison against the
trace.  Needs a GPU; run from the repository root."""
import json
import sys
import time

import numpy as np

sys.path.insert(0, ".")
sys.path.insert(0, "tools")
from workload_trace_bench import FIELDS, gpu_label, pairs_sized, ticks, timed, wva_configuration  # noqa: E402
from workload_variant_autoscaler_b200 import Engine, synth_fleet  # noqa: E402

NAMES = ("arrival_rpm", "in_tokens", "out_tokens", "slo_itl", "slo_ttft", "slo_tps")


def slo_schedule(fleet, L):
    """(itl, ttft, tps), each [L, S]: ITL x 0.75 in hours 8-19, TTFT x 1.5 in hours 0-5, TPS the fleet's own."""
    hour = np.arange(L) % 24
    itl = np.repeat(fleet.srv_slo_itl[None, :], L, 0).astype(np.float32)
    ttft = np.repeat(fleet.srv_slo_ttft[None, :], L, 0).astype(np.float32)
    tps = np.repeat(fleet.srv_slo_tps[None, :], L, 0).astype(np.float32)
    itl[(hour >= 8) & (hour < 20)] *= np.float32(0.75)
    ttft[hour < 6] *= np.float32(1.5)
    return itl, ttft, tps


def searches(fleet, rows):
    """The searches the call runs (distinct (server, in, out, search, target bits) x the server's pairs sized) and
    the 2 x L x (pairs sized) that a wva_solve per tick runs."""
    rpm, in_tok, out_tok, itl, ttft, tps = rows
    L, S = rpm.shape
    cur = fleet.srv_cur_acc
    pin = (fleet.srv_keep_acc != 0) & (cur != -1) & ((cur == -2) | (fleet.srv_min_replicas != 0))
    prof = fleet.perf_present[np.maximum(fleet.srv_model, 0)] != 0
    own = np.arange(fleet.n_acc)[None, :] == cur[:, None]
    ok = (fleet.srv_model >= 0) & (fleet.srv_has_target != 0)
    n_pairs = (prof & ok[:, None] & np.where(pin[:, None], own, True)).sum(1)
    load = ~(rpm < 0) & (rpm != 0) & (in_tok >= 0) & (out_tok >= 1)
    run = 0
    for s in range(S):
        if not n_pairs[s]:
            continue
        keys = set()
        for t in np.nonzero(load[:, s])[0]:
            if itl[t, s] < 0 or ttft[t, s] < 0 or tps[t, s] < 0:
                continue
            for w, x in ((0, ttft[t, s]), (1, itl[t, s])):
                if x > 0:
                    keys.add((int(in_tok[t, s]), int(out_tok[t, s]), w, int(np.float32(x).view(np.uint32))))
        run += len(keys) * int(n_pairs[s])
    return run, 2 * L * int(pairs_sized(fleet)[0])


def at_tick(fleet, rows, t):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    (f.srv_arrival_rpm[:], f.srv_in_tokens[:], f.srv_out_tokens[:], f.srv_slo_itl[:], f.srv_slo_ttft[:],
     f.srv_slo_tps[:]) = (r[t] for r in rows)
    return f


def solve_loop(e, fleet, rows, L, want=False):
    """The existing way: per tick, wva_solve on f_t, the fleet advanced by the previous winners."""
    cur, out, dev = fleet, [], 0.0
    for t in range(L):
        cand, win = e.solve(at_tick(cur, rows, t), want_candidates=want)
        dev += e.last_device_ms
        if want:
            out.append((cand, win))
        cur = cur.apply_winners(win)
    return out, dev


def run_shape(e, label, fleet, L, reps, base_reps, warm=3):
    S, A = fleet.n_servers, fleet.n_acc
    rows = (*ticks(fleet, L, 7), *slo_schedule(fleet, L))
    kw = dict(zip(NAMES, rows))
    dev, ker, wall, launches = timed(e, lambda: e.slo_trace(fleet, **kw), reps, warm)
    wdev, wker, wwall, wlaunches = timed(e, lambda: e.workload_trace(fleet, *rows[:3]), reps, warm)
    solve_loop(e, fleet, rows, min(L, warm))
    base_wall, base_dev = [], []
    for _ in range(base_reps):
        t0 = time.perf_counter()
        _, d = solve_loop(e, fleet, rows, L)
        base_wall.append(time.perf_counter() - t0)
        base_dev.append(d)
    cand, win = e.slo_trace(fleet, want_candidates=True, **kw)
    per_tick, _ = solve_loop(e, fleet, rows, L, want=True)
    mismatched = [t for t, (c, w) in enumerate(per_tick)
                  if not all(getattr(cand, k)[t * S * A:(t + 1) * S * A].tobytes() == getattr(c, k).tobytes() and
                             getattr(win, k)[t * S:(t + 1) * S].tobytes() == getattr(w, k).tobytes() for k in FIELDS)]
    run, per_tick_searches = searches(fleet, rows)
    med_base = float(np.median(base_wall)) * 1e3
    return {
        "workload": f"slo_trace {label} x {L} ticks, ITL x 0.75 in hours 8-19, TTFT x 1.5 in hours 0-5",
        "pairs": S * A, "ticks": L, "calls": reps, "searches_run": run, "searches_per_tick_solve": per_tick_searches,
        "device_ms_p50": dev, "kernel_ms_p50": ker, "host_wall_ms_p50": wall, "launches_per_call": launches,
        "solve_loop_wall_ms_p50": med_base, "solve_loop_device_ms_p50": float(np.median(base_dev)),
        "solve_loop_reps": base_reps, "speedup_wall": med_base / wall,
        "workload_trace_same_load": {"device_ms_p50": wdev, "kernel_ms_p50": wker, "host_wall_ms_p50": wwall,
                                     "launches_per_call": wlaunches},
        "feasible_winners": int(win.feasible.sum()), "tick_mismatches": len(mismatched),
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
