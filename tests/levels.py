"""The level calls' reference side: the oracle compositions the GPU tests compare the library with, and the fleets
and rows more than one test module judges them on.

Every grid is the same composition: per row l, a copy of the fleet with row l of each given list written into its
column and unlimited = 1 goes through the oracle's Server.Calculate (candidate block l) and Solver.Solve (winner block
l).  A trace does the same per tick on the fleet whose current allocation is the previous tick's winner
(Fleet.apply_winners, the reference's Server.ApplyDesiredAlloc).  The row lists are keyed by the Engine level calls'
argument names, so one dict serves the call and its reference."""
import collections

import numpy as np
import pytest

from tests.util import (ACC_NONE, ACC_UNKNOWN, ALLOC_FIELDS, F32_MAX, assert_allocs_equal, assert_f32_bits_equal,
                        same_bytes)
from workload_variant_autoscaler_b200 import synth_fleet
from workload_variant_autoscaler_b200._abi import SAT_NONE

F32 = np.float32
LOAD = ("arrival_rpm", "in_tokens", "out_tokens")
SLO = ("slo_itl", "slo_ttft", "slo_tps")
PERF = ("perf_present", "perf_alpha", "perf_beta", "perf_gamma", "perf_delta", "perf_acc_count", "perf_max_batch",
        "perf_at_tokens")
COLUMNS = ("acc_cost",) + PERF


# the fleet column of each row-list argument; the profile lists are named after their columns
ROW_COLUMN = {"arrival_rpm": "srv_arrival_rpm", "in_tokens": "srv_in_tokens", "out_tokens": "srv_out_tokens",
              "slo_itl": "srv_slo_itl", "slo_ttft": "srv_slo_ttft", "slo_tps": "srv_slo_tps"}


# ITL / TTFT targets at the edges: 0, -0 and NaN disable a search, a negative one makes the pair nil, the others run
TARGETS = (0.0, -0.0, np.nan, -1.0, 1e-30, 1e-40, np.inf, float(F32_MAX))


# TPS targets: no NaN (totalRate NaN) and no tiny positive one (totalRate 0, so a min_replicas-0 pair solves at 0/0):
# the library refuses some such levels, see test_gpu_slo_grid.test_nan_or_tiny_tps_level_fails_as_solve_does
TPS_TARGETS = (0.0, -0.0, -1.0, np.inf, float(F32_MAX))


def n_rows(rows):
    return next(len(v) for v in rows.values() if v is not None)


def at_row(fleet, rows, l, unlimited=True):
    """A copy of the fleet with row l of every list in rows (a list that is None or missing leaves the fleet's own
    column)."""
    f = fleet.take_servers(np.arange(fleet.n_servers))
    for k, v in rows.items():
        if v is not None:
            getattr(f, ROW_COLUMN.get(k, k))[:] = v[l]
    f.unlimited = unlimited
    return f


def ref_grid(oracle_mod, fleet, rows):
    """(candidates [L*S*A], winners [L*S]): Server.Calculate and Solver.Solve (unlimited) per row."""
    cands, wins = [np.zeros(0, oracle_mod.ALLOC_DTYPE)], [np.zeros(0, oracle_mod.ALLOC_DTYPE)]
    for l in range(n_rows(rows)):
        f = at_row(fleet, rows, l)
        cand = oracle_mod.calculate(f)
        cands.append(cand.reshape(-1))
        wins.append(oracle_mod.solve(f, cand)[1])
    return np.concatenate(cands), np.concatenate(wins)


def ref_trace(oracle_mod, fleet, rows):
    """(candidates [L*S*A], winners [L*S], the fleet with c_L): per tick, Server.Calculate and Solver.Solve
    (unlimited) on the fleet with row t and current allocation c_t, then c_{t+1} = apply_winners."""
    cands, wins = [np.zeros(0, oracle_mod.ALLOC_DTYPE)], [np.zeros(0, oracle_mod.ALLOC_DTYPE)]
    cur = fleet
    for t in range(n_rows(rows)):
        f = at_row(cur, rows, t)
        cand = oracle_mod.calculate(f)
        win = oracle_mod.solve(f, cand)[1]
        cands.append(cand.reshape(-1))
        wins.append(win)
        cur = cur.apply_winners(win)
    return np.concatenate(cands), np.concatenate(wins), cur


def check_level_call(engine, oracle_mod, name, fleet, rows, what, ref=None):
    """Engine.<name> against its composition (ref_trace for a trace, ref_grid for a grid; or `ref`, its result),
    bit for bit: the oracle's (candidates, winners)."""
    if ref is None:
        ref = (ref_trace if name.endswith("_trace") else ref_grid)(oracle_mod, fleet, rows)
    cand_o, win_o = ref[:2]
    cand_g, win_g = getattr(engine, name)(fleet, **rows, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
    assert_allocs_equal(win_g, win_o, f"{what}: winners")
    return cand_o, win_o


def mixed_fleet(n_servers, n_acc, seed, keep):
    """Zero load, TPS targets, an unknown model, a server without a target, a missing profile, min_replicas = 0,
    an unknown current accelerator, keepAccelerator on or off."""
    f = synth_fleet(n_servers, n_acc, seed=seed, keep_accelerator=keep, zero_load_frac=0.2, tps_frac=0.3)
    f.srv_min_replicas[::3] = 0
    f.perf_present[1, n_acc - 1] = 0
    f.srv_has_target[2] = 0
    f.srv_model[3] = -1
    f.srv_cur_acc[4] = -2
    f.srv_keep_acc[4] = 1
    return f


def load_levels(fleet, L, seed):
    """[L, S]: each server's own load times a seeded log-normal factor per (level, server), so the levels are
    per-server and non-monotone, with 0, negative, +Inf, tiny and huge rates scattered over them."""
    rng = np.random.default_rng(seed)
    S = fleet.n_servers
    base = np.maximum(fleet.srv_arrival_rpm, 1.0)
    rpm = (base[None, :] * rng.lognormal(0.0, 0.8, (L, S))).astype(np.float32)
    for k, v in enumerate((0.0, -1.0, np.inf, 1e-3, 1e6)):
        rpm[k % L, k::5 + k] = v
    return rpm


def pair_batch(fleet, s, a):
    """allocation.go:77-87."""
    if fleet.srv_max_batch[s] > 0:
        return int(fleet.srv_max_batch[s])
    m = fleet.srv_model[s]
    return max(int(fleet.perf_max_batch[m, a]) * int(fleet.perf_at_tokens[m, a]) // int(fleet.srv_out_tokens[s]), 1)


def go_f64_to_int(x):
    return int(x) if -2.0 ** 63 <= x < 2.0 ** 63 else -(1 << 63)


def tail(oracle_mod, qa, fleet, s, a, N, rate_star, rpm):
    """allocation.go:134-163 at arrival rate rpm, with the pair's analyzer after one Size: the record."""
    f32 = np.float32
    rec = np.zeros(1, oracle_mod.ALLOC_DTYPE)[0]
    rec["acc"] = -1
    m = fleet.srv_model[s]
    with np.errstate(all="ignore"):
        tps = f32(fleet.srv_slo_tps[s])
        total = f32(rpm) / f32(60) if tps == 0 else tps / f32(fleet.srv_out_tokens[s])
        nrep = go_f64_to_int(np.ceil(np.float64(total) / np.float64(rate_star)))
        nrep = max(nrep, int(fleet.srv_min_replicas[s]))
        inst = int(fleet.perf_acc_count[m, a])
        inst = 1 if inst <= 0 else inst
        cost = f32(fleet.acc_cost[a]) * np.array([inst * nrep], np.int64).astype(f32)[0]
        rate = total / np.array([nrep], np.int64).astype(f32)[0]
    err, met = qa.analyze(float(rate))
    if err:
        return rec
    rec["feasible"], rec["acc"], rec["replicas"], rec["batch"] = 1, a, nrep, N
    rec["cost"] = rec["value"] = cost
    rec["itl"] = met["avg_token_time"]
    rec["ttft"] = f32(met["avg_wait_time"]) + f32(met["avg_prefill_time"])
    rec["rho"] = met["rho"]
    rec["max_rate"] = f32(rate_star) / f32(1000)
    return rec


def overflow_fleet():
    """The overflow fleet of test_overflow_rescale_falls_back_to_stored_vector: near saturation at N = 1024 the
    chain overflows float64, and the solves re-run on the stored vector with the reference's rescale loops."""
    fleet = synth_fleet(2, 1, seed=29, max_batch_choices=(1024,))
    fleet.perf_alpha[:] = 7.47
    fleet.perf_beta[:] = 0.0001
    fleet.perf_gamma[:] = 1.0
    fleet.perf_delta[:] = 0.00001
    fleet.srv_in_tokens[:] = 64
    fleet.srv_out_tokens[:] = 64
    fleet.srv_slo_tps[:] = 0
    fleet.srv_slo_itl[:] = 0
    fleet.srv_slo_ttft[:] = 0
    fleet.srv_min_replicas[:] = 1
    return fleet


def rates_at_rate_star(oracle_mod, fleet, s, a):
    """Arrival rates (req/min) at which totalRate / replicas lands at rateStar or one ulp under it, for 1..3
    replicas."""
    m = fleet.srv_model[s]
    N = pair_batch(fleet, s, a)
    qa = oracle_mod.Analyzer(N, N * fleet.max_queue_to_batch_ratio, float(fleet.perf_alpha[m, a]),
                             float(fleet.perf_beta[m, a]), float(fleet.perf_gamma[m, a]), float(fleet.perf_delta[m, a]),
                             int(fleet.srv_in_tokens[s]), int(fleet.srv_out_tokens[s]))
    err, _, met, _ = qa.size(0.0, 0.0, 0.0)
    assert err == 0
    star = np.float32(met["throughput"])
    under = np.nextafter(star, np.float32(0))
    out = []
    for k in (1, 2, 3):
        x = np.float32(star * np.float32(k * 60))
        hits = set()
        for _ in range(200):
            x = np.nextafter(x, np.float32(0))
        for _ in range(400):
            x = np.nextafter(x, np.float32(np.inf))
            total = x / np.float32(60)
            n = go_f64_to_int(np.ceil(np.float64(total) / np.float64(star)))
            r = total / np.float32(n)
            if n == k and r in (star, under):
                hits.add(r == star)
                out.append(float(x))
        assert hits, k
    return out


def with_batch(fleet, b):
    """A copy of the fleet with every server's MaxBatchSize override set to b."""
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_max_batch[:] = b
    return f


def ref_candidates(oracle_mod, fleet, batches):
    """[S, A, B]: Server.Calculate at each batch size."""
    cand = np.zeros((fleet.n_servers, fleet.n_acc, len(batches)), oracle_mod.ALLOC_DTYPE)
    for bi, b in enumerate(batches):
        cand[:, :, bi] = oracle_mod.calculate(with_batch(fleet, int(b)))
    return cand


def ref_winners(oracle_mod, cand, batches):
    """Per server: the feasible candidate with the smallest value, strict '<' from MaxFloat32 (a NaN value or one
    not below MaxFloat32 never wins); ties to the smaller batch size, then the lower accelerator id."""
    S, A, B = cand.shape
    win = np.zeros(S, oracle_mod.ALLOC_DTYPE)
    win["acc"] = -1
    for s in range(S):
        best = None  # (value, batch, a, bi)
        for a in range(A):
            for bi in range(B):
                c = cand[s, a, bi]
                if not c["feasible"]:
                    continue
                v = np.float32(c["value"])
                if not v < F32_MAX:
                    continue
                key = (int(batches[bi]), a, bi)
                if best is None or v < best[0] or (v == best[0] and key < best[1:]):
                    best = (v,) + key
        if best is not None:
            win[s] = cand[s, best[2], best[3]]
    return win


def ref_size_grid(oracle_mod, fleet, batches):
    cand = ref_candidates(oracle_mod, fleet, batches)
    return cand.reshape(-1), ref_winners(oracle_mod, cand, batches)


def slo_levels(fleet, L, seed, special=True):
    """(itl, ttft, tps), each [L, S]: every server's own targets times a seeded factor per (level, server), so the
    rows are per-server and non-monotone, with the edge values of TARGETS and TPS_TARGETS scattered over them."""
    rng = np.random.default_rng(seed)
    S = fleet.n_servers
    factors = np.array([0.5, 0.75, 1.0, 1.5, 2.0], np.float32)
    rows = []
    for col in (fleet.srv_slo_itl, fleet.srv_slo_ttft, fleet.srv_slo_tps):
        rows.append((col[None, :] * rng.choice(factors, (L, S))).astype(np.float32))
    itl, ttft, tps = rows
    if special:
        for k, v in enumerate(TARGETS):
            itl[k % L, k % S::3 + k] = v
            ttft[(k + 1) % L, (k + 1) % S::4 + k] = v
        for k, v in enumerate(TPS_TARGETS):
            tps[(k + 2) % L, (2 * k) % S::5 + k] = v
    return itl, ttft, tps


def _search(oracle_mod, qa, which, target):
    """One BinarySearch of Size (queueanalyzer.go:204-228) on its own: (ok, lambdaStar); ok False when it errs or
    the target is below the bounded region."""
    lo, hi = qa.rate_range()
    lmin, lmax = F32(lo) / F32(1000), F32(hi) / F32(1000)
    if not target > 0:
        return True, lmax
    ev = qa.eval_ttft if which == 0 else qa.eval_itl

    def fn(x):
        err, y = ev(x)
        if err:
            raise ValueError(err)
        return y
    err, xs, ind = oracle_mod.binary_search(float(lmin), float(lmax), float(target), fn)
    return (err == 0 and ind >= 0), F32(xs)


def token_fleet(n_servers, n_acc, seed, keep):
    """mixed_fleet with every other server's batch size from the perf data (N = MaxBatchSize * AtTokens /
    out_tokens, so N follows the level's out_tokens), and perf batch sizes kept small so that out_tokens 1 stays a
    cheap model."""
    f = mixed_fleet(n_servers, n_acc, seed, keep)
    f.srv_max_batch[::2] = 0
    f.perf_max_batch[:] = np.minimum(f.perf_max_batch, 32)
    return f


def workload_levels(fleet, L, seed, special=True):
    """(rpm, in, out), each [L, S]: per (level, server) a rate-only, token-only or joint change of the server's own
    load (non-monotone over the levels), out_tokens from {0.75, 1, 1.5} x own, and with `special` the edge tokens
    scattered over them: in -1, out -1, out 0, in 0, in large, out 1 and out large enough for N = 1."""
    rng = np.random.default_rng(seed)
    S = fleet.n_servers
    rpm = load_levels(fleet, L, seed + 1)
    own_in = np.broadcast_to(fleet.srv_in_tokens, (L, S))
    own_out = np.broadcast_to(fleet.srv_out_tokens, (L, S))
    in_f = rng.choice([0.5, 1.0, 2.0], (L, S))
    out_f = rng.choice([0.75, 1.0, 1.5], (L, S))
    mode = rng.integers(0, 3, (L, S))  # 0: rate only, 1: tokens only, 2: both
    in_tok = np.where(mode == 0, own_in, np.maximum(own_in * in_f, 0)).astype(np.int32)
    out_tok = np.where(mode == 0, own_out, np.maximum(own_out * out_f, 1)).astype(np.int32)
    rpm = np.where(mode == 1, fleet.srv_arrival_rpm[None, :], rpm).astype(np.float32)
    if special:
        for k, (col, v) in enumerate((("in", -1), ("out", -1), ("out", 0), ("in", 0), ("in", 100000), ("out", 1),
                                      ("out", 20000))):
            (in_tok if col == "in" else out_tok)[(k + 1) % L, k % 3::4 + k] = v
    return rpm, in_tok, out_tok


def profile_fleet(n_servers, n_acc, seed, keep):
    """mixed_fleet with every other server's batch size from the perf data, perf batch sizes kept small, and a few
    servers sharing a model so that rows of one model reach several servers."""
    f = mixed_fleet(n_servers, n_acc, seed, keep)
    f.srv_max_batch[::2] = 0
    f.perf_max_batch[:] = np.minimum(f.perf_max_batch, 64)
    f.srv_model[5::4] = f.srv_model[0]
    return f


def profile_rows(fleet, L, seed):
    """Mixed rows: per level a price change of every accelerator, a +-10 % change of one profile coefficient on
    some (model, accelerator) entries, AccCount changes (0 and negative included), perf batch sizes, and a level
    that turns the last accelerator off or on."""
    rng = np.random.default_rng(seed)
    M, A = fleet.n_models, fleet.n_acc
    rows = {k: np.repeat(getattr(fleet, k)[None], L, axis=0).copy() for k in COLUMNS}
    rows["acc_cost"] *= rng.choice([0.5, 0.8, 1.0, 1.0, 1.25], (L, A)).astype(F32)
    for l in range(1, L):
        k = PERF[1 + (l - 1) % 4]
        mask = rng.random((M, A)) < 0.4
        rows[k][l] = np.where(mask, rows[k][l] * rng.choice([F32(0.9), F32(1.1)], (M, A)), rows[k][l])
    rows["perf_acc_count"][L // 2] = rng.choice([-3, 0, 1, 2, 4], (M, A))
    rows["perf_max_batch"][-1] = np.maximum(rows["perf_max_batch"][-1] // 2, 1)
    rows["perf_at_tokens"][min(2, L - 1)] *= 2
    rows["perf_present"][min(1, L - 1), :, A - 1] ^= 1
    return rows


def pinned(fleet):
    """The servers whose accelerator no tick can change (include/wva_b200.h, wva_workload_trace)."""
    cur = fleet.srv_cur_acc
    return (fleet.srv_keep_acc != 0) & (cur != ACC_NONE) & ((cur == ACC_UNKNOWN) | (fleet.srv_min_replicas != 0))


def transition_penalty(factor, cur_acc, cur_rep, cur_cost, acc, rep, cost):
    """allocation.go:291-300 in float32; an unknown accelerator name equals no candidate's."""
    cur_cost, cost = F32(cur_cost), F32(cost)
    with np.errstate(all="ignore"):
        if cur_acc == acc and cur_acc != ACC_UNKNOWN:
            return F32(0.0) if cur_rep == rep else F32(cost - cur_cost)
        return F32(F32(F32(factor) * F32(cur_cost + cost)) + F32(cost - cur_cost))


def low_penalty_fleet(n_servers, n_acc, seed, keep):
    """token_fleet with AccelPenaltyFactor 0 and every min_replicas 1: the cheapest feasible accelerator wins, so the
    winners move between accelerators as the load moves."""
    f = token_fleet(n_servers, n_acc, seed, keep)
    f.accel_penalty_factor = 0.0
    f.srv_min_replicas[:] = 1
    return f


def wva_fleet(n_servers, n_acc, seed):
    """WVA's production configuration: keepAccelerator and min_replicas 1 on every server, each current accelerator
    a real one with its cost (internal/utils/utils.go:290)."""
    f = synth_fleet(n_servers, n_acc, seed=seed, keep_accelerator=True)
    rng = np.random.default_rng(seed)
    f.srv_min_replicas[:] = 1
    none = f.srv_cur_acc < 0
    f.srv_cur_acc[none] = rng.integers(0, n_acc, int(none.sum()))
    f.srv_cur_replicas[none] = 1
    a = f.srv_cur_acc
    f.srv_cur_cost[:] = (f.acc_cost[a] * f.perf_acc_count[f.srv_model, a] * f.srv_cur_replicas).astype(np.float32)
    return f


def _records(allocs):
    """An Allocs as a structured array (the oracle's layout)."""
    return np.rec.fromarrays([getattr(allocs, k) for k in ALLOC_FIELDS], names=",".join(ALLOC_FIELDS))


def _moves(win, S):
    """(tick, server) pairs at which a feasible winner sits on another real accelerator than the last feasible one."""
    win = win.reshape(-1, S)
    n = 0
    for s in range(S):
        accs = [int(a) for a, f in zip(win[:, s]["acc"], win[:, s]["feasible"]) if f and a >= 0]
        n += sum(x != y for x, y in zip(accs, accs[1:]))
    return n


TINY = F32(np.nextafter(F32(0), F32(1)))
KEY_FIELDS = ("feasible", "acc", "replicas", "batch", "cost", "value", "max_rate")
INT32_MAX = 2147483647


def u32_bits(x):
    return int(np.array([x], np.float32).view(np.uint32)[0])


def from_bits(bits):
    return F32(np.array([bits], np.uint32).view(np.float32)[0])


def rec_key(r):
    return tuple(u32_bits(r[k]) if k in ("cost", "value", "max_rate") else int(r[k]) for k in KEY_FIELDS)


def load_pair(oracle_mod, fleet, s, a):
    """(rateStar, RateRange.Max) of a pair whose key reads the load above rate 0, else None: the gates of
    CreateAllocation, the candidate rule, a TPS target (totalRate does not read the load) and a failed Size."""
    m = int(fleet.srv_model[s])
    if fleet.srv_keep_acc[s] and fleet.srv_cur_acc[s] != -1 and fleet.srv_cur_acc[s] != a:
        return None
    if m < 0 or m >= fleet.n_models or not fleet.perf_present[m, a] or not fleet.srv_has_target[s]:
        return None
    if fleet.srv_in_tokens[s] < 0 or fleet.srv_out_tokens[s] <= 0 or fleet.srv_slo_tps[s] != 0:
        return None
    N = pair_batch(fleet, s, a)
    try:
        qa = oracle_mod.Analyzer(N, N * fleet.max_queue_to_batch_ratio, float(fleet.perf_alpha[m, a]),
                                 float(fleet.perf_beta[m, a]), float(fleet.perf_gamma[m, a]),
                                 float(fleet.perf_delta[m, a]), int(fleet.srv_in_tokens[s]),
                                 int(fleet.srv_out_tokens[s]))
    except ValueError:
        return None
    err, _, met, _ = qa.size(float(fleet.srv_slo_ttft[s]), float(fleet.srv_slo_itl[s]), float(fleet.srv_slo_tps[s]))
    if err:
        return None
    return F32(met["throughput"]), F32(qa.rate_range()[1]), qa, N


def pair_state(fleet, s, rate_star, rmax, rpm):
    """(replicas, gate, over) at rpm > 0 with `tail`'s arithmetic: gate 0 = the final rate is not positive, 1 =
    Analyze accepts it, 2 = above RateRange.Max; over = more than INT32_MAX replicas."""
    with np.errstate(all="ignore"):
        total = F32(rpm) / F32(60)
        q = np.ceil(np.float64(total) / np.float64(rate_star))
        over = not (q <= INT32_MAX)
        nrep = max(go_f64_to_int(q), int(fleet.srv_min_replicas[s]))
        rate = total / np.array([nrep], np.int64).astype(F32)[0]
    ok = not (rate <= 0 or rate > rmax)
    return nrep, (1 if ok else (0 if rate <= 0 else 2)), over


def next_step(fleet, s, rate_star, rmax, x, hi):
    """The smallest float32 in (x, hi] whose state differs from x's (None: none)."""
    at = pair_state(fleet, s, rate_star, rmax, x)
    lo_b, hi_b = u32_bits(x), u32_bits(hi)
    if hi_b <= lo_b or pair_state(fleet, s, rate_star, rmax, from_bits(hi_b)) == at:
        return None
    while hi_b - lo_b > 1:
        mid = (lo_b + hi_b) // 2
        if pair_state(fleet, s, rate_star, rmax, from_bits(mid)) != at:
            hi_b = mid
        else:
            lo_b = mid
    return from_bits(hi_b)


def server_steps(oracle_mod, fleet, s, lo, hi):
    """(the points to evaluate in [lo, hi], the first rate at which a pair overflows or None)."""
    pts = {F32(lo)}
    lo_pos = F32(lo) if lo > 0 else TINY
    if lo == 0 and hi > 0:
        pts.add(TINY)
    over_at = None
    for a in range(fleet.n_acc):
        p = load_pair(oracle_mod, fleet, s, a) if hi > 0 else None
        if p is None:
            continue
        rs, rmax = p[0], p[1]
        x = lo_pos
        if pair_state(fleet, s, rs, rmax, x)[2]:
            over_at = x if over_at is None else min(over_at, x)
            continue
        while True:
            y = next_step(fleet, s, rs, rmax, x, F32(hi))
            if y is None:
                break
            if pair_state(fleet, s, rs, rmax, y)[2]:
                over_at = y if over_at is None else min(over_at, y)
                break
            pts.add(y)
            x = y
    pts = sorted(p for p in pts if over_at is None or p < over_at)
    return pts, over_at


def winners_at(oracle_mod, fleet, points):
    """The oracle's unlimited winner of server s at each rate of points[s] (a list per server)."""
    S = fleet.n_servers
    L = max(1, max(len(p) for p in points))
    rows = np.zeros((L, S), np.float32)
    for s, p in enumerate(points):
        if p:
            rows[:, s] = p[-1]
            rows[:len(p), s] = p
    _, win = ref_grid(oracle_mod, fleet, {"arrival_rpm": rows})
    win = win.reshape(L, S)
    return [[win[l, s] for l in range(len(p))] for s, p in enumerate(points)]


def ref_intervals(oracle_mod, fleet, lo, hi, M):
    """(count [S], truncated [S], start (S, M), records [S*M], the step points of each server)."""
    S = fleet.n_servers
    count = np.zeros(S, np.int32)
    trunc = np.zeros(S, np.uint8)
    start = np.zeros((S, M), np.float32)
    rec = np.zeros(S * M, oracle_mod.ALLOC_DTYPE)
    steps = [server_steps(oracle_mod, fleet, s, lo[s], hi[s]) for s in range(S)]
    wins = winners_at(oracle_mod, fleet, [p for p, _ in steps])
    for s in range(S):
        pts, over_at = steps[s]
        trunc[s] = over_at is not None
        prev = None
        for x, w in zip(pts, wins[s]):
            k = rec_key(w)
            if k == prev:
                continue
            if count[s] == M:
                trunc[s] = 1
                break
            start[s, count[s]] = x
            rec[s * M + count[s]] = w
            count[s] += 1
            prev = k
    return count, trunc, start, rec, [p for p, _ in steps]


def check_intervals(engine, oracle_mod, fleet, lo, hi, M, what):
    count_o, trunc_o, start_o, rec_o, _ = ref_intervals(oracle_mod, fleet, lo, hi, M)
    count, trunc, start, rec = engine.load_intervals(fleet, lo, hi, M)
    assert np.array_equal(count, count_o), f"{what}: count {count} vs {count_o}"
    assert np.array_equal(trunc, trunc_o), f"{what}: truncated {trunc} vs {trunc_o}"
    assert same_bytes(start, start_o), f"{what}: start_rpm"
    assert_allocs_equal(rec, rec_o, f"{what}: records")
    return count_o, trunc_o


INF_BITS, PAST = 0x7F800000, 0x7F800001
NIL, SEARCHED, FREE = 0, 1, 2


def is_load_pair(fleet, s, a):
    """CreateAllocation's gates and the candidate rule (allocation.go:42-75, server.go:70-82): a pair it sizes."""
    if fleet.srv_keep_acc[s] and fleet.srv_cur_acc[s] != -1 and fleet.srv_cur_acc[s] != a:
        return False
    rpm, m = fleet.srv_arrival_rpm[s], int(fleet.srv_model[s])
    if rpm < 0 or fleet.srv_in_tokens[s] < 0 or fleet.srv_out_tokens[s] < 0 or not 0 <= m < fleet.n_models:
        return False
    if not fleet.perf_present[m, a] or not fleet.srv_has_target[s]:
        return False
    return rpm != 0 and fleet.srv_out_tokens[s] != 0


def analyzer(oracle_mod, fleet, s, a):
    m, N = int(fleet.srv_model[s]), pair_batch(fleet, s, a)
    return oracle_mod.Analyzer(N, N * fleet.max_queue_to_batch_ratio, float(fleet.perf_alpha[m, a]),
                               float(fleet.perf_beta[m, a]), float(fleet.perf_gamma[m, a]),
                               float(fleet.perf_delta[m, a]), int(fleet.srv_in_tokens[s]),
                               int(fleet.srv_out_tokens[s]))


def lam_range(qa):
    rmin, rmax = qa.rate_range()
    return F32(rmin) / F32(1000), F32(rmax) / F32(1000)  # queueanalyzer.go:197-198


class Classifier:
    """BinarySearch's boundary checks (utils.go:36-51) restated with the oracle's WithinTolerance."""

    def __init__(self, oracle_mod):
        self.wt = oracle_mod.lib().wvao_within_tolerance

    def cls(self, y0, y1, t):
        if self.wt(y0, t, 1e-6):
            return SEARCHED
        if self.wt(y1, t, 1e-6):
            return FREE
        inc = y0 < y1
        if (inc and t < y0) or (not inc and t > y0):
            return NIL
        if (inc and t > y1) or (not inc and t < y1):
            return FREE
        return SEARCHED

    def rank(self, y0, y1, t):
        c = self.cls(y0, y1, t)
        return c if y0 < y1 else 2 - c

    def first(self, y0, y1, k):
        """Smallest positive float32 target of rank >= k, NaN past +Inf."""
        if self.rank(y0, y1, from_bits(INF_BITS)) < k:
            return F32(np.nan)
        if self.rank(y0, y1, from_bits(1)) >= k:
            return from_bits(1)
        lo, hi = 1, INF_BITS
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if self.rank(y0, y1, from_bits(mid)) >= k:
                hi = mid
            else:
                lo = mid
        return from_bits(hi)


def ref_slo_bounds(oracle_mod, fleet):
    """(kind, y_lo, y_hi, b1, b2), each (S, A, 2), from the oracle."""
    S, A = fleet.n_servers, fleet.n_acc
    kind = np.zeros((S, A, 2), np.uint8)
    y_lo, y_hi, b1, b2 = (np.zeros((S, A, 2), np.float32) for _ in range(4))
    cl = Classifier(oracle_mod)
    for s in range(S):
        for a in range(A):
            if not is_load_pair(fleet, s, a):
                continue
            N = pair_batch(fleet, s, a)
            if N + N * fleet.max_queue_to_batch_ratio < 2:
                continue
            qa = analyzer(oracle_mod, fleet, s, a)
            lmin, lmax = lam_range(qa)
            ends = [(qa.eval_ttft(float(x)), qa.eval_itl(float(x))) for x in (lmin, lmax)]
            if lmin > lmax or ends[0][0][0]:
                kind[s, a] = 1  # BinarySearch's range error, or an invalid model at the first evaluation
                continue
            for w in range(2):
                y0, y1 = F32(ends[0][w][1]), F32(ends[1][w][1])
                kind[s, a, w] = 2 if y0 < y1 else 3
                y_lo[s, a, w], y_hi[s, a, w] = y0, y1
                b1[s, a, w], b2[s, a, w] = cl.first(y0, y1, 1), cl.first(y0, y1, 2)
    return kind, y_lo, y_hi, b1, b2


def check_slo_bounds(engine, oracle_mod, fleet, what):
    want = ref_slo_bounds(oracle_mod, fleet)
    got = engine.slo_bounds(fleet)
    assert np.array_equal(got[0], want[0]), f"{what}: kind"
    for name, g, w in zip(("y_lo", "y_hi", "b1", "b2"), got[1:], want[1:]):
        assert_f32_bits_equal(g.reshape(-1), w.reshape(-1), f"{what}: {name}")
    return want


def limited_fleet(seed, cap, policy=SAT_NONE, delayed=False, n=24, n_acc=3):
    f = synth_fleet(n, n_acc, seed=seed, max_batch_choices=(2, 4, 8, 16), zero_load_frac=0.1)
    f.unlimited = False
    f.saturation_policy = policy
    f.delayed_best_effort = delayed
    f.type_capacity[:] = cap
    f.srv_priority[:] = np.random.default_rng(seed).choice([1, 5, 10], f.n_servers)
    return f


F = np.float32
ALLOC_FLOATS = ("cost", "itl", "ttft", "rho", "max_rate")
BIG_N = 4096


def same_f32(a, b):
    a, b = F(a), F(b)
    return (np.isnan(a) and np.isnan(b)) or a.view(np.uint32) == b.view(np.uint32)


class Tally:
    """Points a family covered: feasible / infeasible records (or cells, or sweep points), refusals by reason,
    probability vectors compared, and pairs left out for their batch size."""

    def __init__(self):
        self.n = collections.Counter()

    def report(self, what, min_feasible=1, min_infeasible=1, **at_least):
        print(f"{what}: {dict(self.n)}")
        assert self.n["feasible"] >= min_feasible, (what, dict(self.n))
        assert self.n["infeasible"] >= min_infeasible, (what, dict(self.n))
        for k, v in at_least.items():
            assert self.n[k] >= v, (what, k, dict(self.n))


def _restated(call, oracle_mod, oracle_call, tally):
    """call() on the restatement; on Unsupported, the oracle's side of the refusal (see the module docstring) and
    None."""
    from oracle import restate_np as R
    try:
        return call()
    except R.Unsupported as e:
        tally.n[f"refused ({e.reason})"] += 1
        if e.reason == "states":
            with pytest.raises(oracle_mod.Unsupported):
                oracle_call()
        return None


def cross_alloc(oracle_mod, f, s, a, tally, what=""):
    from oracle import restate_np as R
    r = _restated(lambda: R.create_allocation(f, s, a), oracle_mod, lambda: oracle_mod.create_allocation(f, s, a),
                  tally)
    if r is None:
        return
    o = oracle_mod.create_allocation(f, s, a)
    assert o["feasible"] == r["feasible"], (what, s, a, o, r)
    tally.n["feasible" if o["feasible"] else "infeasible"] += 1
    if not o["feasible"]:
        return
    assert (o["acc"], o["replicas"], o["batch"]) == (r["acc"], r["replicas"], r["batch"]), (what, s, a, o, r)
    for k in ALLOC_FLOATS:
        assert same_f32(o[k], r[k]), (what, s, a, k, o[k], r[k])


def pair_n(f, s, a):
    """The batch size N of a load pair (allocation.go:77-87), in Python's unbounded int."""
    if f.srv_max_batch[s] > 0:
        return int(f.srv_max_batch[s])
    m = int(f.srv_model[s])
    return max(int(f.perf_max_batch[m, a]) * int(f.perf_at_tokens[m, a]) // int(f.srv_out_tokens[s]), 1)


def _too_long(f, s, a):
    """A load pair whose N is above BIG_N but within the restated domain: left out of the samples for time."""
    m = int(f.srv_model[s])
    if m < 0 or not f.perf_present[m, a] or not (f.srv_arrival_rpm[s] > 0) or f.srv_out_tokens[s] <= 0:
        return False
    return BIG_N < pair_n(f, s, a) <= (1 << 20)


def cross_fleet(oracle_mod, f, tally, what="", pairs=None):
    """cross_alloc on every (server, accelerator) of f, or on the given pairs."""
    for s, a in (pairs if pairs is not None else ((s, a) for s in range(f.n_servers) for a in range(f.n_acc))):
        if _too_long(f, s, a):
            tally.n["left out (N > 4096)"] += 1
            continue
        cross_alloc(oracle_mod, f, s, a, tally, what)


TINY_TOTAL = F32(60) * F32(2.0 ** -149)  # below this positive rate totalRate rounds to 0


def _levels_to_rows(cols):
    """[L, S] rows from one list of rates per server, each padded with its own last rate."""
    L = max(1, max(len(c) for c in cols))
    rows = np.zeros((L, len(cols)), np.float32)
    for s, c in enumerate(cols):
        if c:
            rows[:, s] = c[-1]
            rows[:len(c), s] = c
    return rows


N_SIZE = 60


def size_grid_cases():
    """(fleet, batch list, rounds) per case: unsorted, repeated lists with 1 and 2, and every 15th case a long
    batch size (1024 or 2049) with ratio 1 so that the oracle stays fast."""
    rng = np.random.default_rng(0x51CE)
    out = []
    for case in range(N_SIZE):
        fleet = _adversarial_fleet(rng, 20000 + case)
        batches = [1, 2] + rng.integers(1, 65, int(rng.integers(0, 5))).tolist()
        batches += [batches[int(rng.integers(0, len(batches)))]]  # a repeat
        if case % 15 == 7:
            batches.append(1024 if case % 30 == 7 else 2049)
            fleet.max_queue_to_batch_ratio = 1
        rng.shuffle(batches)
        out.append((fleet, np.array(batches, np.int32), bool(case % 2)))
    return out


N_LOAD = 60


def _rate_star_rates(oracle_mod, fleet, s):
    """rates_at_rate_star for every pair of server s that has a rateStar (the others have no such rates)."""
    out = []
    for a in range(fleet.n_acc):
        if load_pair(oracle_mod, fleet, s, a) is None:
            continue
        try:
            out += rates_at_rate_star(oracle_mod, fleet, s, a)
        except AssertionError:  # no float32 rate lands exactly at 60 k rateStar (rateStar tiny or huge)
            pass
    return out


def adversarial_load_levels(oracle_mod, fleet):
    """Per server: 0, -1, 1e-3, 0.5x, x, 2x, 1e3 x of its load, MaxFloat32, +Inf, and the rates at and one ulp
    under 60 nrep rateStar (nrep = 1..3) of each of its pairs.  No NaN (test_nan_level_fails_as_analyze_does), and
    no positive rate below 60 * 2^-149 (the header's min_replicas-0 case)."""
    cols = []
    for s in range(fleet.n_servers):
        x = F32(fleet.srv_arrival_rpm[s])
        lv = [F32(0), F32(-1), F32(1e-3), x * F32(0.5), x, x * F32(2), x * F32(1e3), F32_MAX, F32(np.inf)]
        lv += [F32(r) for r in _rate_star_rates(oracle_mod, fleet, s)]
        cols.append([v for v in lv if not (0 < v < TINY_TOTAL)])
    return _levels_to_rows(cols)


def load_grid_cases(oracle_mod):
    rng = np.random.default_rng(0x10AD)
    return [(f, adversarial_load_levels(oracle_mod, f)) for f in (_adversarial_fleet(rng, 30000 + c) for c in range(N_LOAD))]


def go_queue(perf_max_batch, at_tokens, out_tokens, srv_max_batch, ratio):
    """(N, K) of a load pair as Go computes them, in 64-bit int (allocation.go:77-93)."""
    i64 = np.int64
    if srv_max_batch > 0:
        N = i64(srv_max_batch)
    else:
        N = max(i64(perf_max_batch) * i64(at_tokens) // i64(out_tokens), i64(1))
    return N, N + N * i64(ratio)


QUEUE_CASES = [
    ("at_tokens_wrap", 65536, 65537, 1, 0, 10, True),       # N = 4,295,032,832: int32 sees 65536
    ("ratio_wrap", 8, 512, 1, 4, 1 << 30, True),            # K = 2^32 + 4: int32 sees 4
    ("n_2p20", 1024, 1024, 1, 0, 10, False),                # N = 2^20: the largest batch size
    ("n_above_2p20", 1025, 1024, 1, 0, 10, True),           # N = 2^20 + 1024
    ("k_just_below_2p31", 8, 512, 1, 1 << 20, 2046, False),  # K = 2^31 - 2^20
    ("k_2p31", 8, 512, 1, 1 << 20, 2047, True),             # K = 2^31 exactly
]


def queue_fleet(name, n_servers=3):
    """A small fleet whose server 0 carries the named case of QUEUE_CASES on every accelerator (the others
    ordinary; ratio applies to all)."""
    _, pmb, at, out, smb, ratio, _ = next(c for c in QUEUE_CASES if c[0] == name)
    f = synth_fleet(n_servers, 2, seed=7, server_batch=False, zero_load_frac=0.0, tps_frac=0.0,
                    max_batch_choices=(4, 8, 16))
    m = int(f.srv_model[0])
    f.perf_max_batch[m, :] = pmb
    f.perf_at_tokens[m, :] = at
    f.srv_out_tokens[0] = out
    f.srv_max_batch[0] = smb
    f.max_queue_to_batch_ratio = ratio
    return f


def _adversarial_fleet(rng, case):
    """Small fleet whose parameters sit at the edges the reference never exercises on purpose: coefficients spread
    over many decades (and exactly 0), token counts 0 / 1 / huge, SLOs 0 / tiny / loose, loads from 1e-3 to 1e6
    requests per minute, TPS targets, batch sizes 1 and 2."""
    S, A = int(rng.integers(1, 7)), int(rng.integers(1, 4))
    f = synth_fleet(S, A, seed=9000 + case, zero_load_frac=0.1, tps_frac=0.3, server_batch=bool(case % 2),
                    max_batch_choices=(1, 2, 3, 8, 33, 120) if case % 25 else (2, 150, 400))
    M = f.n_models

    def logu(lo, hi, shape):
        return np.exp(rng.uniform(np.log(lo), np.log(hi), shape)).astype(np.float32)
    f.perf_alpha[:] = logu(1e-3, 1e3, (M, A))
    f.perf_beta[:] = logu(1e-5, 1e2, (M, A))
    f.perf_gamma[:] = logu(1e-3, 1e4, (M, A))
    f.perf_delta[:] = logu(1e-7, 1.0, (M, A))
    zero = rng.random((M, A))
    f.perf_beta[zero < 0.1] = 0.0
    f.perf_gamma[(zero > 0.1) & (zero < 0.2)] = 0.0
    f.perf_delta[(zero > 0.2) & (zero < 0.3)] = 0.0
    f.srv_in_tokens[:] = rng.choice([0, 1, 7, 512, 100000], S)
    f.srv_out_tokens[:] = rng.choice([1, 2, 9, 300, 50000], S)
    f.srv_arrival_rpm[:] = logu(1e-3, 1e6, S)
    f.srv_arrival_rpm[rng.random(S) < 0.15] = 0.0
    f.srv_slo_itl[:] = rng.choice([0.0, 1e-3, 5.0, 80.0, 1e6], S).astype(np.float32)
    f.srv_slo_ttft[:] = rng.choice([0.0, 1e-2, 50.0, 2000.0, 1e7], S).astype(np.float32)
    f.srv_slo_tps[:] = rng.choice([0.0, 0.0, 1.0, 500.0, 1e6], S).astype(np.float32)
    f.srv_min_replicas[:] = rng.integers(0, 3, S)
    f.max_queue_to_batch_ratio = int(rng.choice([1, 3, 10]))
    return f


# ---- price thresholds: wva_price_thresholds' composition at one fleet, and at each level's or tick's fleet ----

PRICE_MAX_BITS = 0x7F7FFFFF


def pred(x):
    """The largest float32 below x (x > 0)."""
    return from_bits(u32_bits(x) - 1)


def at_price(fleet, a, p):
    """A copy of the fleet with acc_cost[a] = p, unlimited."""
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.acc_cost[a] = p
    f.unlimited = True
    return f


def priced(fleet, s, a, rec, p):
    """a's record of server s at price p: cost = p * f32(NumInstances * replicas), value = TransitionPenalty against
    the fleet's current allocation (allocation.go:144-145, :274-275, :291-300); a nil record is unchanged."""
    r = rec.copy()
    if not r["feasible"]:
        return r
    inst = int(fleet.perf_acc_count[int(fleet.srv_model[s]), a])
    inst = 1 if inst <= 0 else inst
    with np.errstate(all="ignore"):
        r["cost"] = F32(p) * F32(inst * int(r["replicas"]))
    r["value"] = transition_penalty(F32(fleet.accel_penalty_factor), int(fleet.srv_cur_acc[s]),
                                    int(fleet.srv_cur_replicas[s]), fleet.srv_cur_cost[s], int(r["acc"]),
                                    int(r["replicas"]), r["cost"])
    return r


class PriceServer:
    """One server's winner as a's price moves: Server.Calculate's row with a's record re-priced, decided by the
    oracle's Solver.Solve on the one-server fleet.  SolveUnlimited reads only feasible and value, so the solve sees
    each record with its column id in the batch field, which names the winning column."""

    def __init__(self, oracle_mod, fleet, cand, s):
        self.o, self.fleet, self.row, self.s = oracle_mod, fleet, cand[s], s
        self.f1 = fleet.take_servers(np.array([s]))
        self.f1.unlimited = True

    def winner(self, a, p):
        """(winning column or -1, winner record) with a's record at price p."""
        row = self.row.copy()
        row[a] = priced(self.fleet, self.s, a, row[a], p)
        tagged = row.copy()
        tagged["batch"] = np.arange(row.size)
        w = self.o.solve(self.f1, tagged[None])[1][0]
        if not w["feasible"]:
            return -1, w
        return int(w["batch"]), row[int(w["batch"])]

    def wins(self, a, p):
        return self.winner(a, p)[0] == a

    def threshold(self, a):
        """The first float32 price in [+0, MaxFloat32] at which a stops winning, by bisecting the bit patterns."""
        if self.wins(a, from_bits(PRICE_MAX_BITS)):
            return F32(np.inf)
        if not self.wins(a, F32(0.0)):
            return F32(0.0)
        lo, hi = 0, PRICE_MAX_BITS
        while hi - lo > 1:
            mid = (lo + hi) // 2
            if self.wins(a, from_bits(mid)):
                lo = mid
            else:
                hi = mid
        return from_bits(hi)


def ref_price_fleet(oracle_mod, fleet):
    """(threshold [S, A], above [S*A], candidates [S*A], winners [S]) of one fleet: wva_price_thresholds' contract
    composed from the oracle."""
    cand = oracle_mod.calculate(fleet)
    S, A = fleet.n_servers, fleet.n_acc
    th = np.zeros((S, A), F32)
    above = np.zeros(S * A, oracle_mod.ALLOC_DTYPE)
    for s in range(S):
        sp = PriceServer(oracle_mod, fleet, cand, s)
        for a in range(A):
            th[s, a] = sp.threshold(a)
            if np.isfinite(th[s, a]):
                above[s * A + a] = sp.winner(a, th[s, a])[1]
    return th, above, cand.reshape(-1), oracle_mod.solve(fleet, cand)[1]


def ref_price_rows(oracle_mod, fleet, rows, trace):
    """(threshold [L, S, A], above [L*S*A], candidates [L*S*A], winners [L*S], the row fleets): ref_price_fleet on
    at_row(fleet, rows, l) per level, or with `trace` on ref_trace's fleet of tick t, whose current allocation is
    c_t (apply_winners of the ticks before)."""
    out, fleets, cur = [], [], fleet
    for l in range(n_rows(rows)):
        f = at_row(cur, rows, l)
        r = ref_price_fleet(oracle_mod, f)
        out.append(r)
        fleets.append(f)
        if trace:
            cur = cur.apply_winners(r[3])
    S, A = fleet.n_servers, fleet.n_acc
    if not out:
        empty = np.zeros(0, oracle_mod.ALLOC_DTYPE)
        return np.zeros((0, S, A), F32), empty, empty, empty, fleets
    return (np.stack([r[0] for r in out]),) + tuple(np.concatenate([r[k] for r in out]) for k in (1, 2, 3)) + (fleets,)


def edge_fleet(seed, keep=False, factor=0.1, n=10, n_acc=4):
    """mixed_fleet with one type per accelerator, accelerators 1 and 2 identical (ties on value), and current costs
    0, 1e38 and -MaxFloat32."""
    f = mixed_fleet(n, n_acc, seed, keep)
    f.accel_penalty_factor = factor
    for k in ("perf_alpha", "perf_beta", "perf_gamma", "perf_delta", "perf_acc_count", "perf_max_batch",
              "perf_at_tokens", "perf_present"):
        getattr(f, k)[:, 2] = getattr(f, k)[:, 1]
    f.acc_cost[2] = f.acc_cost[1]
    f.acc_type[:] = np.arange(n_acc)
    f.type_capacity = np.full(n_acc, 1000, np.int32)
    f.acc_multiplicity[:] = np.arange(n_acc) % 3 + 1
    f.srv_cur_cost[5::5] = 0.0
    f.srv_cur_cost[6::5] = F32(1e38)
    f.srv_cur_cost[7::5] = -F32_MAX
    return f


def moving_fleet(seed):
    """Penalty factor 0 and min_replicas 1: the cheapest accelerator wins, so c_t changes accelerator on the trace."""
    f = edge_fleet(seed, factor=0.0)
    f.srv_min_replicas[:] = 1
    return f


PRICE_CALLS = {False: "price_threshold_grid", True: "price_threshold_trace"}


def check_price_rows(engine, oracle_mod, fleet, rows, trace, what, ref=None):
    """Engine.price_threshold_grid / price_threshold_trace against ref_price_rows (or `ref`, its result), bit for
    bit: (threshold, candidates, winners) of the reference."""
    th_o, above_o, cand_o, win_o, _ = ref if ref is not None else ref_price_rows(oracle_mod, fleet, rows, trace)
    th_g, above_g, cand_g, win_g = getattr(engine, PRICE_CALLS[trace])(fleet, **rows, want_candidates=True)
    assert_f32_bits_equal(th_g.reshape(-1), th_o.reshape(-1), f"{what}: threshold")
    assert_allocs_equal(above_g, above_o, f"{what}: above")
    assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
    assert_allocs_equal(win_g, win_o, f"{what}: winners")
    return th_o, cand_o, win_o


# ---- long horizons: nil runs and periodic days ---------------------------------------------------------------

def gap_mask(n_servers, L, gaps, start):
    """[L, S] bool: server s is in its nil run on ticks [start[s], start[s] + gaps[s]) (gaps[s] 0: none)."""
    gaps = np.broadcast_to(np.asarray(gaps), (n_servers,))
    start = np.broadcast_to(np.asarray(start), (n_servers,))
    t = np.arange(L)[:, None]
    return (t >= start[None, :]) & (t < (start + gaps)[None, :])


def gap_rows(fleet, L, gaps, start, seed):
    """{"arrival_rpm": [L, S]}: each server's own load (at least 200 req/min) times a seeded log-uniform factor in
    [0.1, 50] per (tick, server), which spans many replica counts, so that a 32-tick window holds several feasible winners that differ;
    positive and finite everywhere except that server s is nil (rate -1) on ticks [start[s], start[s] + gaps[s])."""
    rng = np.random.default_rng(seed)
    S = fleet.n_servers
    base = np.maximum(fleet.srv_arrival_rpm, 200.0)
    rpm = (base[None, :] * np.exp(rng.uniform(np.log(0.1), np.log(50.0), (L, S)))).astype(F32)
    rpm[gap_mask(S, L, gaps, start)] = -1.0
    return {"arrival_rpm": rpm}


def _tile(x, L):
    """Rows t = x[t % period] for t < L."""
    return np.ascontiguousarray(x[np.arange(L) % x.shape[0]])


def day_rows(fleet, L, period, seed, special=True):
    """{"arrival_rpm", "in_tokens", "out_tokens"}, each [L, S], repeating every `period` ticks: a diurnal rate (the
    server's own load, at least 100 req/min, times a smooth daily factor from e^-2 to e^2 with a per-server phase,
    times per-server noise) and tokens from
    a small per-period set of the server's own.  With `special`, a few ticks of the day carry the edge values of
    load_levels and workload_levels (rates 0, -1, +Inf, tiny and huge; in -1 / 0 / large, out -1 / 0 / 1 / large),
    so they too repeat daily."""
    rng = np.random.default_rng(seed)
    S = fleet.n_servers
    base = np.maximum(fleet.srv_arrival_rpm, 100.0)
    t = np.arange(period)[:, None]
    phase = rng.uniform(0, 2 * np.pi, S)
    daily = np.exp(2.0 * np.sin(2 * np.pi * t / period + phase[None, :]))
    rpm = (base[None, :] * daily * rng.lognormal(0.0, 0.15, (period, S))).astype(F32)
    in_tok = (fleet.srv_in_tokens[None, :] * rng.choice([0.5, 1.0, 1.0, 2.0], (period, S))).astype(np.int32)
    out_tok = np.maximum(fleet.srv_out_tokens[None, :] * rng.choice([0.75, 1.0, 1.0, 1.5], (period, S)),
                         1).astype(np.int32)
    if special:
        for k, v in enumerate((0.0, -1.0, np.inf, 1e-3, 1e6)):
            rpm[(7 * k + 3) % period, k::5 + k] = v
        for k, (col, v) in enumerate((("in", -1), ("out", -1), ("out", 0), ("in", 0), ("in", 100000), ("out", 1),
                                      ("out", 20000))):
            (in_tok if col == "in" else out_tok)[(11 * k + 5) % period, k % 3::4 + k] = v
    return {"arrival_rpm": _tile(rpm, L), "in_tokens": _tile(in_tok, L), "out_tokens": _tile(out_tok, L)}


def day_profile_rows(fleet, L, period, seed):
    """Profile rows over a day that repeats every `period` ticks: acc_cost an hourly price curve per accelerator
    (own phase and depth), beta x 1.1 on every entry from tick L // 2 on, and the last accelerator withdrawn
    (perf_present 0) on ticks [period // 4, period // 2) of every day."""
    rng = np.random.default_rng(seed)
    A = fleet.n_acc
    t = np.arange(period)[:, None]
    phase, depth = rng.uniform(0, 2 * np.pi, A), rng.uniform(0.2, 0.8, A)
    curve = 1.0 + depth * np.sin(2 * np.pi * t / period + phase) + rng.normal(0, 0.03, (period, A))
    acc = (fleet.acc_cost[None] * np.maximum(curve, 0.05)).astype(F32)
    present = np.repeat(fleet.perf_present[None], period, axis=0)
    present[period // 4:period // 2, :, A - 1] = 0
    beta = np.repeat(fleet.perf_beta[None], L, axis=0).astype(F32)
    beta[L // 2:] *= F32(1.1)
    return {"acc_cost": _tile(acc, L), "perf_present": _tile(present, L), "perf_beta": beta}


def day_slo_rows(fleet, L, period):
    """SLO rows over a day that repeats every `period` ticks: the ITL target x 0.75 in the middle third of the day,
    the TTFT target x 1.5 in its first quarter, the fleet's own TPS target."""
    own = {k: np.repeat(getattr(fleet, ROW_COLUMN[k])[None], period, axis=0).astype(F32) for k in SLO}
    own["slo_itl"][period // 3:2 * period // 3] *= F32(0.75)
    own["slo_ttft"][:max(period // 4, 1)] *= F32(1.5)
    return {k: _tile(v, L) for k, v in own.items()}


def last_feasible(win, S):
    """[L, S]: the tick of each server's last feasible winner before tick t, -1 for none (c_t is then the fleet's
    own current allocation)."""
    feas = win.reshape(-1, S)["feasible"] != 0
    out = np.full(feas.shape, -1, np.int64)
    for t in range(1, feas.shape[0]):
        out[t] = np.where(feas[t - 1], t - 1, out[t - 1])
    return out


ACC_CM = {  # CreateAcceleratorUnitCostConfigMap, JSON-decoded as readAccFunc does (optimizer_test.go:72-86)
    "A100": {"device": "NVIDIA-A100-PCIE-80GB", "cost": "40.00"},
    "MI300X": {"device": "AMD-MI300X-192GB", "cost": "65.00"},
    "G2": {"device": "Intel-Gaudi-2-96GB", "cost": "23.00"},
}
SC_CM = {  # CreateServiceClassConfigMap
    "premium.yaml": "name: Premium\npriority: 1\ndata:\n  - model: default/default\n    slo-tpot: 24\n    slo-ttft: 500\n"
                    "  - model: meta/llama0-70b\n    slo-tpot: 80\n    slo-ttft: 500",
    "freemium.yaml": "name: Freemium\npriority: 10\ndata:\n  - model: ibm/granite-13b\n    slo-tpot: 200\n    slo-ttft: 2000\n"
                     "  - model: meta/llama0-7b\n    slo-tpot: 150\n    slo-ttft: 1500",
}


def _va(i, *, arrival="0.00", replicas=1):
    return {
        "metadata": {"name": f"test-variantautoscaling-{i}", "namespace": "default",
                     "labels": {"inference.optimization/acceleratorName": "A100"}},
        "spec": {"modelID": "meta/llama0-70b", "modelProfile": {"accelerators": [{
            "acc": "A100", "accCount": 1, "maxBatchSize": 4,
            "perfParms": {"decodeParms": {"alpha": "20.28", "beta": "0.72"}, "prefillParms": {"gamma": "0", "delta": "0"}}}]}},
        "status": {"currentAlloc": {"accelerator": "A100", "numReplicas": replicas, "maxBatch": 4, "variantCost": "40.00",
                                    "itlAverage": "0.00", "ttftAverage": "0.00",
                                    "load": {"arrivalRate": arrival, "avgInputTokens": "0.00", "avgOutputTokens": "0.00"}}},
    }
