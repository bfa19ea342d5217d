"""The size grid, load grid, load intervals, sweep and streaming paths on adversarial fleets, and the queue-size rule.

The fleets come from levels._adversarial_fleet (coefficients over many decades or exactly 0, token counts
0 / 1 / 100000, SLOs 0 / tiny / 1e7, loads from 1e-3 to 1e6 req/min), each path with a seed stream of its own.  The
expected values are the oracle compositions the other test modules pin: ref_size_grid, ref_grid,
ref_intervals and the oracle's sweep and solve.  The load intervals are also checked without the monotonicity
argument of DESIGN.md §3.10 that ref_intervals restates: a load grid over samples spread over every decade of each
range must give every sample the key of the interval that contains it.

The queue-size rule: the reference computes a load pair's batch size N and its queue model's
K = N + N * max_queue_to_batch_ratio in Go's 64-bit int.  The library and the oracle count states in int32, so a
model with N above 2^20 (library) or K of 2^31 or more (both) is refused instead of being built at a wrapped size."""
import numpy as np
import pytest

from tests.grid_cases import device_winners
from tests.levels import (F32, KEY_FIELDS, QUEUE_CASES, _adversarial_fleet, _levels_to_rows, _rate_star_rates,
                          from_bits, go_queue, load_grid_cases, load_pair, pair_batch, queue_fleet, ref_grid,
                          ref_intervals, ref_size_grid, size_grid_cases, u32_bits)
from tests.util import ALLOC_FIELDS, assert_allocs_equal, assert_f32_bits_equal
from workload_variant_autoscaler_b200 import Grid, WvaError, _abi, synth_fleet

SWEEP_COLS = ("rate", "ttft", "itl", "throughput", "rho")


def same_bytes(a, b):
    return np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


# ---- size grid ---------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_size_grid_adversarial(engine, oracle_mod, monkeypatch):
    feasible = 0
    for case, (fleet, batches, rounds) in enumerate(size_grid_cases()):
        if rounds:
            monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        else:
            monkeypatch.delenv("WVA_SIZE_SMALL_MAX", raising=False)
        cand_o, win_o = ref_size_grid(oracle_mod, fleet, batches)
        cand_g, win_g = engine.size_grid(fleet, batches, want_candidates=True)
        what = f"size grid, case {case}, batches {batches.tolist()}, rounds = {rounds}"
        assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
        assert_allocs_equal(win_g, win_o, f"{what}: winners")
        feasible += int(win_o["feasible"].sum())
    assert feasible > 30


# ---- load grid ---------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def load_cases(oracle_mod):
    return load_grid_cases(oracle_mod)


def test_load_levels_reach_the_replica_steps(oracle_mod, load_cases):
    """The levels include rates at which the replica count of some pair steps: at 60 k rateStar for k = 1..3 the
    count is k, one ulp under it too, so the tail's ceil and the rate check are exercised at their edges."""
    n_servers_with = 0
    for fleet, rpm in load_cases:
        for s in range(fleet.n_servers):
            if len(_rate_star_rates(oracle_mod, fleet, s)) >= 2:
                n_servers_with += 1
    assert n_servers_with >= 40


@pytest.mark.gpu
def test_load_grid_adversarial(engine, oracle_mod, monkeypatch, load_cases):
    feasible = 0
    for case, (fleet, rpm) in enumerate(load_cases):
        if case % 2:
            monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        else:
            monkeypatch.delenv("WVA_SIZE_SMALL_MAX", raising=False)
        cand_o, win_o = ref_grid(oracle_mod, fleet, {"arrival_rpm": rpm})
        cand_g, win_g = engine.load_grid(fleet, rpm, want_candidates=True)
        assert_allocs_equal(cand_g, cand_o, f"load grid, case {case}: candidates")
        assert_allocs_equal(win_g, win_o, f"load grid, case {case}: winners")
        feasible += int(win_o["feasible"].sum())
    assert feasible > 300


# ---- load intervals ----------------------------------------------------------------------------------

N_INTERVALS = 30
M_LONG = 64


def interval_ranges(oracle_mod, fleet, rng):
    """[lo, hi] per server, sized from its load pairs' rateStar so that no pair takes more than about 150 steps
    (ref_intervals walks every step in Python).  lo = 0 only on servers with min_replicas >= 1: below
    60 * 2^-149 req/min a min_replicas-0 load pair is unsupported."""
    S = fleet.n_servers
    lo, hi = np.zeros(S, np.float32), np.zeros(S, np.float32)
    for s in range(S):
        stars = [p[0] for p in (load_pair(oracle_mod, fleet, s, a) for a in range(fleet.n_acc)) if p is not None]
        x = F32(fleet.srv_arrival_rpm[s])
        if not stars:  # nothing steps: any range
            lo[s], hi[s] = x * F32(0.5), x * F32(2)
            continue
        step = F32(60) * min(stars)  # the replica count of the slowest-stepping pair changes every `step`
        n = F32(rng.integers(1, 120))
        base = x if x > 0 else step * F32(rng.uniform(0.5, 20))
        lo[s] = base * F32(rng.uniform(0.3, 1.0))
        if fleet.srv_min_replicas[s] >= 1 and rng.random() < 0.35:
            lo[s] = 0
        hi[s] = lo[s] + step * n
        if not np.isfinite(hi[s]):
            hi[s] = lo[s]
    return lo, hi


@pytest.fixture(scope="module")
def interval_cases(oracle_mod):
    """(fleet, lo, hi, the reference at M_LONG) per case."""
    rng = np.random.default_rng(0x1E7A)
    out = []
    for case in range(N_INTERVALS):
        fleet = _adversarial_fleet(rng, 40000 + case)
        # ref_intervals re-sizes every pair at every step point: batch sizes from the AtTokens rule above 2048
        # (up to 2^17 here) are replaced by the adversarial list's server batch sizes to keep it fast
        for s in range(fleet.n_servers):
            if fleet.srv_max_batch[s] == 0 and fleet.srv_out_tokens[s] > 0 and max(
                    pair_batch(fleet, s, a) for a in range(fleet.n_acc)) > 2048:
                fleet.srv_max_batch[s] = rng.choice([1, 2, 3, 8, 33, 120])
        lo, hi = interval_ranges(oracle_mod, fleet, rng)
        out.append((fleet, lo, hi, ref_intervals(oracle_mod, fleet, lo, hi, M_LONG)))
    return out


def _truncate(ref, M):
    """ref_intervals at M from its result at a larger M (test_truncation_at_M_and_lo_equal_hi pins this)."""
    count, trunc, start, rec, _ = ref
    S, ML = start.shape
    c = np.minimum(count, M).astype(np.int32)
    t = (trunc | (count > M)).astype(np.uint8)
    st = np.zeros((S, M), np.float32)
    r = np.zeros(S * M, rec.dtype)
    for s in range(S):
        st[s, :c[s]] = start[s, :c[s]]
        r[s * M:s * M + c[s]] = rec[s * ML:s * ML + c[s]]
    return c, t, st, r


def test_interval_cases_reach_their_regimes(interval_cases):
    """The ranges give truncated lists (at M = 3 and at M_LONG), lists longer than 3 and lo = 0 ranges."""
    long_lists = trunc3 = lo_zero = 0
    for fleet, lo, hi, ref in interval_cases:
        count = ref[0]
        long_lists += int((count > 3).sum())
        trunc3 += int(_truncate(ref, 3)[1].sum())
        lo_zero += int(((lo == 0) & (hi > 0)).sum())
    assert long_lists >= 10 and trunc3 >= 10 and lo_zero >= 5, (long_lists, trunc3, lo_zero)


@pytest.mark.gpu
def test_load_intervals_adversarial(engine, interval_cases):
    for case, (fleet, lo, hi, ref) in enumerate(interval_cases):
        for M in (M_LONG, 3):
            count_o, trunc_o, start_o, rec_o = _truncate(ref, M)
            count, trunc, start, rec = engine.load_intervals(fleet, lo, hi, M)
            what = f"intervals, case {case}, M = {M}"
            assert np.array_equal(count, count_o), f"{what}: count {count} vs {count_o}"
            assert np.array_equal(trunc, trunc_o), f"{what}: truncated {trunc} vs {trunc_o}"
            assert same_bytes(start, start_o), f"{what}: start_rpm"
            assert_allocs_equal(rec, rec_o, f"{what}: records")


def _key(win, i):
    return tuple(u32_bits(getattr(win, k)[i]) if k in ("cost", "value", "max_rate") else int(getattr(win, k)[i])
                 for k in KEY_FIELDS)


@pytest.mark.gpu
def test_load_intervals_against_sampled_load_grid(engine, oracle_mod, interval_cases):
    """Without §3.10: 256 rates uniform over the float32 bit patterns of [lo, hi], every start and one ulp either
    side of it, through one wva_load_grid.  Each sample's key is its interval's key, the record at a start is the
    interval's record, and about 64 of the load-grid winners per case are the oracle's."""
    rng = np.random.default_rng(0x5A3B)
    checked = 0
    for case, (fleet, lo, hi, _) in enumerate(interval_cases):
        S, M = fleet.n_servers, M_LONG
        count, trunc, start, rec = engine.load_intervals(fleet, lo, hi, M)
        cols, owner = [], []
        for s in range(S):
            n = int(count[s])
            st = [F32(v) for v in start[s, :n]]
            b_lo, b_hi = u32_bits(lo[s]), u32_bits(hi[s])
            pts = [from_bits(int(b)) for b in rng.integers(b_lo, b_hi + 1, 256)]
            for x in st:
                pts += [x, np.nextafter(x, F32(-np.inf)), np.nextafter(x, F32(np.inf))]
            pts = [p for p in pts if lo[s] <= p <= hi[s]]
            # the interval of each sample (-1: past a truncated list's last start, where nothing is reported)
            own = []
            for p in pts:
                j = int(np.searchsorted(np.array(st, np.float32), p, side="right")) - 1
                own.append(-1 if j < 0 or (trunc[s] and j == n - 1 and p > st[-1]) else j)
            cols.append(pts)
            owner.append(own)
        rows = _levels_to_rows(cols)
        _, win = engine.load_grid(fleet, rows)
        for s in range(S):
            for l, (p, j) in enumerate(zip(cols[s], owner[s])):
                if j < 0:
                    continue
                i = l * S + s
                assert _key(win, i) == _key(rec, s * M + j), (case, s, float(p), j)
                if p == start[s, j]:
                    for k in ALLOC_FIELDS:
                        assert same_bytes(getattr(win, k)[i:i + 1], getattr(rec, k)[s * M + j:s * M + j + 1]), (case, s, j, k)
                checked += 1
        # a random subset of the load-grid winners against the oracle
        pick = np.sort(rng.choice(rows.shape[0], min(64, rows.shape[0]), replace=False))
        _, win_o = ref_grid(oracle_mod, fleet, {"arrival_rpm": rows[pick]})
        idx = (pick[:, None] * S + np.arange(S)[None, :]).reshape(-1)
        for k in ALLOC_FIELDS:
            got = getattr(win, k)[idx]
            if k in ("feasible", "acc", "replicas", "batch"):
                assert np.array_equal(got.astype(np.int64), win_o[k].astype(np.int64)), (case, k)
            else:
                assert_f32_bits_equal(got, win_o[k], f"case {case}: sampled winners {k}")
    assert checked > 256 * 20


# ---- sweep -------------------------------------------------------------------------------------------

N_SWEEP = 40


@pytest.mark.gpu
def test_sweep_adversarial(engine, oracle_mod):
    rng = np.random.default_rng(0x5EE9)
    valid = 0
    for case in range(N_SWEEP):
        fleet = _adversarial_fleet(rng, 50000 + case)
        n_rates = (1, 2, 33, 64)[case % 4]
        o = oracle_mod.sweep(fleet, n_rates)
        g = engine.sweep(fleet, n_rates)
        assert np.array_equal(g["valid"], o["valid"]), f"sweep, case {case}, n_rates {n_rates}: valid"
        for k in SWEEP_COLS:
            assert_f32_bits_equal(g[k], o[k], f"sweep, case {case}, n_rates {n_rates}: {k}")
        valid += int(o["valid"].sum())
    assert valid > 1000


# ---- streaming ---------------------------------------------------------------------------------------

N_TICKS = 40


def streaming_fleet():
    """About 24 servers: the servers of an adversarial fleet repeated, each with load columns, SLOs and
    min_replicas of its own from the same adversarial sets, and small type capacities for limited mode.  The base
    case has server batch sizes (odd case numbers): out_tokens 1 under the AtTokens rule would give batch sizes up
    to 2^17, whose sizing costs seconds per tick."""
    rng = np.random.default_rng(0x57E4)
    case = 60001
    while True:
        base = _adversarial_fleet(rng, case)
        if base.n_servers >= 3 and base.n_acc >= 2:
            break
        case += 2
    assert (base.srv_max_batch > 0).all()
    fleet = base.take_servers(np.arange(24) % base.n_servers)
    S = fleet.n_servers
    fleet.srv_in_tokens[:] = rng.choice([0, 1, 7, 512, 100000], S)
    fleet.srv_out_tokens[:] = rng.choice([1, 2, 9, 300, 50000], S)
    fleet.srv_arrival_rpm[:] = np.exp(rng.uniform(np.log(1e-3), np.log(1e6), S)).astype(np.float32)
    fleet.srv_slo_itl[:] = rng.choice([0.0, 1e-3, 5.0, 80.0, 1e6], S).astype(np.float32)
    fleet.srv_slo_ttft[:] = rng.choice([0.0, 1e-2, 50.0, 2000.0, 1e7], S).astype(np.float32)
    fleet.srv_slo_tps[:] = rng.choice([0.0, 0.0, 1.0, 500.0, 1e6], S).astype(np.float32)
    fleet.srv_min_replicas[:] = rng.integers(0, 3, S)
    fleet.type_capacity[:] = rng.integers(0, 40, fleet.n_types)
    return fleet


def streaming_schedule(fleet):
    """N_TICKS updates (arrival, in_tokens, out_tokens), None = column not passed.  Ticks 3 / 6, 9 / 12 and
    15 / 18 take a group of servers' rate to 0 and back, to a negative rate and back, and their out_tokens to 0 and
    back; tick 21 sets a group's in_tokens to 0; every fifth tick passes nothing and tick 25 passes every column
    unchanged.  The other ticks move a random subset of the columns."""
    rng = np.random.default_rng(0x71C5)
    S = fleet.n_servers
    rate = fleet.srv_arrival_rpm.copy()
    inp = fleet.srv_in_tokens.copy()
    out = fleet.srv_out_tokens.copy()
    groups = rng.permutation(S)[:16].reshape(4, 4)
    saved = {}
    ticks = []
    for t in range(N_TICKS):
        cols = [None, None, None]
        if t in (3, 9):
            g = groups[0 if t == 3 else 1]
            saved[t] = rate[g].copy()
            rate[g] = 0.0 if t == 3 else -1.0
            cols[0] = rate.copy()
        elif t in (6, 12):
            g = groups[0 if t == 6 else 1]
            rate[g] = saved[t - 3]
            cols[0] = rate.copy()
        elif t == 15:
            saved[t] = out[groups[2]].copy()
            out[groups[2]] = 0
            cols[2] = out.copy()
        elif t == 18:
            out[groups[2]] = saved[15]
            cols[2] = out.copy()
        elif t == 21:
            inp[groups[3]] = 0
            cols[1] = inp.copy()
        elif t == 25:
            cols = [rate.copy(), inp.copy(), out.copy()]
        elif t % 5 != 0:
            for c in range(3):
                if rng.random() < 0.5:
                    continue
                k = rng.choice(S, int(rng.integers(1, 6)), replace=False)
                if c == 0:
                    rate[k] = (rate[k] * np.exp(rng.normal(0, 1.0, k.size))).astype(np.float32)
                    rate[k[rate[k] < 0]] = -rate[k[rate[k] < 0]]  # a negative stays negative only through ticks 9-12
                    cols[0] = rate.copy()
                elif c == 1:
                    inp[k] = rng.choice([1, 7, 512, 100000], k.size)
                    cols[1] = inp.copy()
                else:
                    out[k] = rng.choice([1, 2, 9, 300, 50000], k.size)
                    cols[2] = out.copy()
        ticks.append(cols)
    return ticks


def _apply(fleet, cols):
    for name, c in zip(("srv_arrival_rpm", "srv_in_tokens", "srv_out_tokens"), cols):
        if c is not None:
            getattr(fleet, name)[:] = c


def test_streaming_schedule_crosses_every_class_boundary():
    fleet = streaming_fleet()
    ticks = streaming_schedule(fleet)
    f = fleet.take_servers(np.arange(fleet.n_servers))
    seen = set()
    for cols in ticks:
        before = (f.srv_arrival_rpm.copy(), f.srv_in_tokens.copy(), f.srv_out_tokens.copy())
        _apply(f, cols)
        r0, r1 = before[0], f.srv_arrival_rpm
        seen.update({("rate>0->0", bool(((r0 > 0) & (r1 == 0)).any())), ("rate0->>0", bool(((r0 == 0) & (r1 > 0)).any())),
                     ("rate->neg", bool(((r0 >= 0) & (r1 < 0)).any())), ("neg->rate", bool(((r0 < 0) & (r1 >= 0)).any())),
                     ("out->0", bool(((before[2] > 0) & (f.srv_out_tokens == 0)).any())),
                     ("out0->", bool(((before[2] == 0) & (f.srv_out_tokens > 0)).any())),
                     ("in->0", bool(((before[1] > 0) & (f.srv_in_tokens == 0)).any()))})
    for name in ("rate>0->0", "rate0->>0", "rate->neg", "neg->rate", "out->0", "out0->", "in->0"):
        assert (name, True) in seen, name
    assert sum(all(c is None for c in cols) for cols in ticks) >= 5
    assert any(all(c is not None for c in cols) for cols in ticks)
    assert sum(sum(c is not None for c in cols) == 1 for cols in ticks) >= 10


def _device_block_columns(blk, S):
    raw = blk.cpu().numpy().view(np.uint8)
    out = {"feasible": raw[:S]}
    for k, name in enumerate(ALLOC_FIELDS[1:], start=1):
        dt = np.int32 if name in ("acc", "replicas", "batch") else np.float32
        out[name] = raw[4 * S * k:4 * S * (k + 1)].view(dt)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("unlimited", [True, False])
def test_streaming_adversarial(engine, oracle_mod, unlimited):
    fleet = streaming_fleet()
    fleet.unlimited = unlimited
    ticks = streaming_schedule(fleet)
    S = fleet.n_servers
    engine.upload(fleet)
    blk, cols_dev = device_winners(S) if unlimited else (None, None)
    feasible = 0
    for t, cols in enumerate(ticks):
        _apply(fleet, cols)
        engine.update_load(*cols)
        cand_g, win_g = engine.resolve(want_candidates=True)
        cand_o, win_o = oracle_mod.solve(fleet)
        what = f"tick {t}, unlimited = {unlimited}"
        assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
        assert_allocs_equal(win_g, win_o, f"{what}: winners")
        feasible += int(win_o["feasible"].sum())
        if unlimited:
            engine.resolve_device(cols_dev)
            engine.synchronize()
            dev = _device_block_columns(blk, S)
            for k in ALLOC_FIELDS:
                assert same_bytes(dev[k], getattr(win_g, k)), f"{what}: resolve_device {k}"
    assert feasible > 100


# ---- the queue-size rule -----------------------------------------------------------------------------

def _wrap32(x):
    return int(np.array([x], np.int64).astype(np.int32)[0])


# (name, perf_max_batch, at_tokens, out_tokens, srv_max_batch, ratio, refused by the library)
def test_queue_cases_sit_where_they_are_meant_to():
    for name, pmb, at, out, smb, ratio, refused in QUEUE_CASES:
        N, K = go_queue(pmb, at, out, smb, ratio)
        assert refused == bool(N > (1 << 20) or K >= (1 << 31)), name
        if name == "at_tokens_wrap":
            assert N >= (1 << 32) and _wrap32(N) == 65536 and 0 < _wrap32(N) <= (1 << 20)
        if name == "ratio_wrap":
            assert K >= (1 << 31) and _wrap32(K) == 4 and _wrap32(N * ratio) == 0
        if name == "n_2p20":
            assert N == (1 << 20) and K < (1 << 31)
        if name == "k_just_below_2p31":
            assert K == (1 << 31) - (1 << 20)
        if name == "k_2p31":
            assert K == (1 << 31) and _wrap32(K) < 0


@pytest.mark.parametrize("name", ["at_tokens_wrap", "ratio_wrap"])
def test_oracle_refuses_queue_models_outside_int32(oracle_mod, name):
    """The oracle computes N and K in 64 bits: it builds no model of 2^31 states or more and reports it, where it
    used to solve a wrapped model (batch 65536; the record of ratio 0)."""
    f = queue_fleet(name)
    with pytest.raises(oracle_mod.Unsupported):
        oracle_mod.calculate(f)
    with pytest.raises(oracle_mod.Unsupported):
        oracle_mod.solve(f)
    with pytest.raises(oracle_mod.Unsupported):
        oracle_mod.create_allocation(f, 0, 0)
    with pytest.raises(oracle_mod.Unsupported):
        oracle_mod.sweep(f, 4)
    if name == "ratio_wrap":  # the grid's batch list is its N
        with pytest.raises(oracle_mod.Unsupported):
            oracle_mod.grid_solve(f, Grid([4], [1, 2]))
    # the same pair without load builds no model: zeroLoadAllocation reads perf_max_batch directly (with the
    # ratio of 2^30 every load pair is refused, so there no server carries load)
    f.srv_arrival_rpm[0 if name == "at_tokens_wrap" else slice(None)] = 0
    cand = oracle_mod.calculate(f)
    assert cand[0]["feasible"].all()
    if name == "at_tokens_wrap":
        assert (cand[0]["batch"] == 65536).all()


def _refused(engine, call):
    n0 = engine.launch_count
    with pytest.raises(WvaError) as e:
        call()
    assert e.value.code == _abi.WVA_ERR_UNSUPPORTED, str(e.value)
    assert "2^" in str(e.value), str(e.value)
    assert engine.launch_count == n0, "a refused call launches nothing"


def _check_ordinary(engine, oracle_mod):
    f = synth_fleet(6, 3, seed=11, max_batch_choices=(4, 16, 64))
    cand_o, win_o = oracle_mod.solve(f)
    cand_g, win_g = engine.solve(f)
    assert_allocs_equal(cand_g, cand_o, "ordinary fleet after a refusal: candidates")
    assert_allocs_equal(win_g, win_o, "ordinary fleet after a refusal: winners")


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["at_tokens_wrap", "ratio_wrap"])
def test_library_refuses_queue_models_outside_int32(engine, oracle_mod, name):
    f = queue_fleet(name)
    S = f.n_servers
    x = f.srv_arrival_rpm
    rpm = np.stack([x, x * F32(2)]).astype(np.float32)
    lo, hi = (x * F32(0.5)).astype(np.float32), (x * F32(2)).astype(np.float32)
    _refused(engine, lambda: engine.analyze(f))
    _refused(engine, lambda: engine.solve(f))
    _refused(engine, lambda: engine.load_grid(f, rpm))
    _refused(engine, lambda: engine.load_intervals(f, lo, hi, 8))
    _refused(engine, lambda: engine.sweep(f, 4))
    # the resident path: for the AtTokens case a fleet whose server 0 has out_tokens 0 (a zero-load pair, solved),
    # then out_tokens 1 through wva_update_load; the ratio is not a load column, so that fleet is uploaded as is
    if name == "ratio_wrap":
        engine.upload(f)
    else:
        ok = queue_fleet(name)
        ok.srv_out_tokens[0] = 0
        engine.upload(ok)
        engine.resolve()
        engine.update_load(out_tokens=f.srv_out_tokens)
    _refused(engine, lambda: engine.resolve())
    blk, cols = device_winners(S)
    _refused(engine, lambda: engine.resolve_device(cols))
    if name == "ratio_wrap":
        # the grid's and the size grid's batch lists are their N
        _refused(engine, lambda: engine.grid_solve(f, Grid([2, 4], [1, 2])))
        engine.upload(f)
        _refused(engine, lambda: engine.grid_solve_device(Grid([2, 4], [1, 2]), cols))
        _refused(engine, lambda: engine.size_grid(f, [4, 2]))
    else:
        # the grid and the size grid do not read the AtTokens rule: the same fleet is solved there
        grid = Grid([2, 4], [1, 2, 3])
        _, win_o = oracle_mod.grid_solve(f, grid, want_cells=False)
        _, win_g = engine.grid_solve(f, grid)
        assert_allocs_equal(win_g, win_o, "grid winners, AtTokens fleet")
        cand_o, win_o = ref_size_grid(oracle_mod, f, [4, 2])
        cand_g, win_g = engine.size_grid(f, [4, 2], want_candidates=True)
        assert_allocs_equal(cand_g, cand_o, "size-grid candidates, AtTokens fleet")
        assert_allocs_equal(win_g, win_o, "size-grid winners, AtTokens fleet")
    _check_ordinary(engine, oracle_mod)


@pytest.mark.gpu
def test_zero_load_pair_outside_int32_is_not_refused(engine, oracle_mod):
    """Server 0 carries the AtTokens wrap but no load: zeroLoadAllocation reads perf_max_batch, and no queue model
    is built, so every path that builds models only for load pairs solves the fleet."""
    f = queue_fleet("at_tokens_wrap", n_servers=4)
    f.srv_arrival_rpm[0] = 0
    cand_o, win_o = oracle_mod.solve(f)
    cand_g, win_g = engine.solve(f)
    assert_allocs_equal(cand_g, cand_o, "candidates")
    assert_allocs_equal(win_g, win_o, "winners")
    assert int(np.asarray(cand_g.batch)[0]) == 65536
    rpm = np.stack([f.srv_arrival_rpm, f.srv_arrival_rpm * F32(3)]).astype(np.float32)
    cand_o, win_o = ref_grid(oracle_mod, f, {"arrival_rpm": rpm})
    cand_g, win_g = engine.load_grid(f, rpm, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, "load-grid candidates")
    assert_allocs_equal(win_g, win_o, "load-grid winners")
    lo = (f.srv_arrival_rpm * F32(0.9)).astype(np.float32)
    hi = (f.srv_arrival_rpm * F32(1.1)).astype(np.float32)
    count_o, trunc_o, start_o, rec_o, _ = ref_intervals(oracle_mod, f, lo, hi, 16)
    count, trunc, start, rec = engine.load_intervals(f, lo, hi, 16)
    assert np.array_equal(count, count_o) and np.array_equal(trunc, trunc_o) and same_bytes(start, start_o)
    assert_allocs_equal(rec, rec_o, "interval records")
    engine.upload(f)
    _, win_r = engine.resolve()
    assert_allocs_equal(win_r, win_o[:f.n_servers], "resolve")
