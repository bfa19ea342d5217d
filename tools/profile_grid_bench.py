"""wva_profile_grid on four shapes: synth_fleet(10000, 8, seed=42) x 24 price rows (perf columns the fleet's own), the
same fleet x 24 rows in which level l scales beta of accelerator l mod 8 by 0.9 (l // 8 even) or 1.1, that shape in
WVA's configuration (keepAccelerator on every server, min_replicas 1), and synth_fleet(100, 4, seed=42) x 256 rows
that perturb alpha and beta of every (model, accelerator) entry (no two rows alike: the no-deduplication case).

Prints one JSON line: per shape, the median device / kernel / host wall time over repeated calls, the launches per
call, the keys sized (distinct (server, accelerator, alpha, beta, gamma, delta, N) used as a load pair), the bytes of
row lists passed in, and the same answer obtained the existing way (one wva_solve per level on the fleet with that
level's columns), timed, with a per-level byte comparison.  device - kernel time is what runs outside the sizing
kernels: the host's key build, the uploads, the record and winner kernels and the copy back.  Needs a GPU; run from
the repository root."""
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, ".")
from workload_variant_autoscaler_b200 import Engine, synth_fleet  # noqa: E402

FIELDS = ("feasible", "acc", "replicas", "batch", "cost", "value", "itl", "ttft", "rho", "max_rate")
PERF = ("perf_present", "perf_alpha", "perf_beta", "perf_gamma", "perf_delta", "perf_acc_count", "perf_max_batch",
        "perf_at_tokens")


def gpu_label():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:  # the label is informative only
        q = "unknown"
    return name, q


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


def price_rows(fleet, L, seed):
    rng = np.random.default_rng(seed)
    return {"acc_cost": (fleet.acc_cost[None] * rng.uniform(0.7, 1.3, (L, fleet.n_acc))).astype(np.float32)}


def beta_rows(fleet, L):
    beta = np.repeat(fleet.perf_beta[None], L, axis=0).copy()
    for l in range(L):
        beta[l, :, l % fleet.n_acc] *= np.float32(0.9 if (l // fleet.n_acc) % 2 == 0 else 1.1)
    return {"perf_beta": beta}


def alpha_beta_rows(fleet, L, seed):
    rng = np.random.default_rng(seed)
    shape = (L,) + fleet.perf_alpha.shape
    return {"perf_alpha": (fleet.perf_alpha[None] * rng.lognormal(0.0, 0.05, shape)).astype(np.float32),
            "perf_beta": (fleet.perf_beta[None] * rng.lognormal(0.0, 0.05, shape)).astype(np.float32)}


def at_level(fleet, rows, l):
    f = fleet.take_servers(np.arange(fleet.n_servers))
    for k, v in rows.items():
        getattr(f, k)[:] = v[l]
    f.unlimited = True
    return f


def keys_sized(fleet, rows, L):
    """Distinct (server, accelerator, bits of alpha .. delta, N) over the levels at which the pair is a load."""
    S, A = fleet.n_servers, fleet.n_acc
    m = fleet.srv_model
    cur = fleet.srv_cur_acc
    rate = fleet.srv_arrival_rpm
    ok = (m >= 0) & (m < fleet.n_models) & (fleet.srv_has_target != 0) & ~(rate < 0) & (rate != 0) & \
        (fleet.srv_in_tokens >= 0) & (fleet.srv_out_tokens > 0)
    keep = (fleet.srv_keep_acc != 0)[:, None] & (cur != -1)[:, None] & (np.arange(A)[None, :] != cur[:, None])
    base = ok[:, None] & ~keep
    mm = np.maximum(m, 0)
    out = []
    for l in range(L):
        col = {k: (rows[k][l] if k in rows else getattr(fleet, k))[mm] for k in PERF}  # [S, A]
        load = base & (col["perf_present"] != 0)
        N = np.where(fleet.srv_max_batch[:, None] > 0, fleet.srv_max_batch[:, None],
                     np.maximum(col["perf_max_batch"].astype(np.int64) * col["perf_at_tokens"] //
                                np.maximum(fleet.srv_out_tokens[:, None], 1), 1))
        s_idx, a_idx = np.nonzero(load)
        out.append(np.stack([s_idx, a_idx] + [col[k].view(np.uint32)[load].astype(np.int64)
                                              for k in ("perf_alpha", "perf_beta", "perf_gamma", "perf_delta")] +
                            [N[load]], axis=1))
    return int(len(np.unique(np.concatenate(out), axis=0)))


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


def run_shape(e, label, fleet, rows, reps, base_reps, warm=3):
    S, A = fleet.n_servers, fleet.n_acc
    L = len(next(iter(rows.values())))
    dev, ker, wall, launches = timed(e, lambda: e.profile_grid(fleet, **rows), reps, warm)
    levels = [at_level(fleet, rows, l) for l in range(L)]
    for f in levels[:warm]:
        e.solve(f, want_candidates=False)
    base_wall = []
    for _ in range(base_reps):
        t0 = time.perf_counter()
        for f in levels:
            e.solve(f, want_candidates=False)
        base_wall.append(time.perf_counter() - t0)
    cand, win = e.profile_grid(fleet, **rows, want_candidates=True)
    mismatched = []
    for l, f in enumerate(levels):
        c, w = e.solve(f)
        if not all(getattr(cand, k)[l * S * A:(l + 1) * S * A].tobytes() == getattr(c, k).tobytes() and
                   getattr(win, k)[l * S:(l + 1) * S].tobytes() == getattr(w, k).tobytes() for k in FIELDS):
            mismatched.append(l)
    perf_given = any(k != "acc_cost" for k in rows)
    row_bytes = sum(int(v.nbytes) for v in rows.values())
    rank_bytes = 4 * L * fleet.n_models * A if perf_given else 0
    med_base = float(np.median(base_wall)) * 1e3
    moves = int(sum(((win.acc[l * S:(l + 1) * S] != win.acc[:S]) & (win.feasible[l * S:(l + 1) * S] != 0)).sum()
                    for l in range(1, L)))
    return {
        "workload": f"profile_grid {label} x {L} rows", "pairs": S * A, "levels": L, "calls": reps,
        "keys_sized": keys_sized(fleet, rows, L), "row_bytes": row_bytes, "rank_table_bytes": rank_bytes,
        "device_ms_p50": dev, "kernel_ms_p50": ker, "host_wall_ms_p50": wall, "launches_per_call": launches,
        "solve_loop_wall_ms_p50": med_base, "solve_loop_reps": base_reps, "speedup_wall": med_base / wall,
        "feasible_winners": int(win.feasible.sum()), "winners_off_level_0_accelerator": moves,
        "level_mismatches": len(mismatched),
    }


def main():
    e = Engine(0)
    big = synth_fleet(10000, 8, seed=42)
    wva = wva_configuration(synth_fleet(10000, 8, seed=42), 5)
    small = synth_fleet(100, 4, seed=42)
    shapes = [
        run_shape(e, "synth_fleet(10000, 8, seed=42), prices only", big, price_rows(big, 24, 7), 20, 3),
        run_shape(e, "synth_fleet(10000, 8, seed=42), beta of accelerator l mod 8 x 0.9 / 1.1", big,
                  beta_rows(big, 24), 20, 3),
        run_shape(e, "synth_fleet(10000, 8, seed=42), WVA configuration, beta rows", wva, beta_rows(wva, 24), 20, 3),
        run_shape(e, "synth_fleet(100, 4, seed=42), alpha and beta of every pair perturbed", small,
                  alpha_beta_rows(small, 256, 11), 20, 3),
    ]
    name, power = gpu_label()
    print(json.dumps({"gpu": name, "power_limit_and_max_sm_clock": power, "shapes": shapes}))


if __name__ == "__main__":
    main()
