"""wva_profile_price_threshold_grid / wva_profile_price_threshold_trace: wva_price_thresholds at every row of load,
accelerator prices and performance profiles, in one call.

The expected result is tests.levels.ref_price_rows on profile rows: per level the fleet at_row(fleet, rows, l) with
every load list, acc_cost and perf_* column at row l, per tick the fleet of the profile trace's chain (current
allocation c_t, whose cost is at tick t-1's prices).  The CPU tests pin that composition to a full Server.Calculate +
Solver.Solve at the price on profile rows, and demand_by_level with per-row AccCount to AllocateByType.  The GPU tests
compare the CUDA path with it bit for bit, and on a larger fleet with the single call, the price threshold and
profile calls and wva_profile_grid without the oracle."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (PRICE_MAX_BITS, at_price, at_row, edge_fleet, from_bits, mixed_fleet, moving_fleet,
                          overflow_fleet, pred, rates_at_rate_star, ref_price_rows, u32_bits)
from tests.profile_margin_levels import own_profile
from tests.profile_price_levels import (CALLS, KINDS, check_profile_price_rows, cost_refused, price_case, run)
from tests.util import (ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_UNSUPPORTED, error_code, same_bytes)
from workload_variant_autoscaler_b200 import Allocs, Engine, demand_by_level, synth_fleet
from workload_variant_autoscaler_b200 import _abi

F32 = np.float32
PRICE_CALLS = {False: "price_threshold_grid", True: "price_threshold_trace"}


def _to_allocs(rec):
    out = Allocs(rec.size)
    for k in ALLOC_FIELDS:
        getattr(out, k)[:] = rec[k]
    return out


def _rec(allocs, lo, hi):
    """Records [lo, hi) of an Allocs, as an Allocs."""
    out = Allocs(hi - lo)
    for k in ALLOC_FIELDS:
        getattr(out, k)[:] = getattr(allocs, k)[lo:hi]
    return out


def _same(x, y, what):
    if isinstance(x, np.ndarray):
        assert same_bytes(x, y), what
        return
    for k in ALLOC_FIELDS:
        assert same_bytes(getattr(x, k), getattr(y, k)), f"{what}: {k}"


# ---- CPU: the composition on profile rows ---------------------------------------------------------

def _prices(col, rng, n):
    """Each finite positive threshold of a column and the float below it, 0, MaxFloat32 and n random bit
    patterns."""
    t = np.unique(col[np.isfinite(col) & (col > 0)])
    return ([F32(0.0), from_bits(PRICE_MAX_BITS)] + [x for v in t for x in (v, pred(v))] +
            [from_bits(int(b)) for b in rng.integers(0, PRICE_MAX_BITS + 1, n)])


def _a_wins(oracle_mod, f, a, p):
    """Per server, whether a's column wins on f with acc_cost[a] = p: a full Server.Calculate and Solver.Solve, the
    records tagged with their column id in the batch field (SolveUnlimited reads only feasible and value)."""
    fp = at_price(f, a, p)
    cand = oracle_mod.calculate(fp)
    cand["batch"] = np.arange(f.n_acc)[None, :]
    w = oracle_mod.solve(fp, cand)[1]
    return (w["feasible"] == 1) & (w["batch"] == a)


@pytest.mark.parametrize("kind,keep,trace,tokens", [
    ("prices", False, False, False), ("prices", True, True, True), ("edge_prices", False, False, False),
    ("acc_count", False, True, False), ("acc_count", True, False, True), ("present", False, True, False),
    ("present", True, False, False), ("beta", False, False, True), ("batch", True, True, False),
    ("mixed", False, True, True), ("mixed", True, False, False),
])
def test_a_wins_exactly_below_each_rows_threshold(oracle_mod, kind, keep, trace, tokens):
    """At every row's fleet (prices, AccCount and profiles of the row; on a trace c_t), "a wins" from a full
    Calculate + Solve at price p equals p < threshold, at every threshold, the float below it, 0, MaxFloat32 and
    random bit patterns."""
    fleet = moving_fleet(21 + keep) if trace else edge_fleet(21 + keep, keep)
    rows = price_case(fleet, 4, kind, 5, tokens)
    th, _, _, _, fleets = ref_price_rows(oracle_mod, fleet, rows, trace)
    assert cost_refused(fleets) is None
    rng = np.random.default_rng(9)
    kinds = set()
    for l, f in enumerate(fleets):
        for a in range(fleet.n_acc):
            for p in _prices(th[l, :, a], rng, 2):
                assert (_a_wins(oracle_mod, f, a, p) == (p < th[l, :, a])).all(), (l, a, p)
            kinds |= {"0" if t == 0 else "inf" if np.isinf(t) else "finite" for t in th[l, :, a]}
    assert {"0", "finite"} <= kinds


@pytest.mark.parametrize("trace", [False, True])
def test_column_a_does_not_read_the_rows_price_of_a(oracle_mod, trace):
    """Changing row l's acc_cost[a] leaves column a of threshold and above in block l unchanged (and, on a trace,
    every earlier block)."""
    fleet = moving_fleet(31)
    rows = price_case(fleet, 4, "mixed", 7)
    th, above, _, _, _ = ref_price_rows(oracle_mod, fleet, rows, trace)
    S, A = fleet.n_servers, fleet.n_acc
    for l, a in ((1, 0), (2, 3), (3, 1)):
        moved = {k: (v.copy() if v is not None else None) for k, v in rows.items()}
        moved["acc_cost"][l, a] *= F32(3.0)
        th2, above2, _, _, _ = ref_price_rows(oracle_mod, fleet, moved, trace)
        assert same_bytes(th2[l, :, a], th[l, :, a]), (l, a)
        idx = (l * S + np.arange(S)) * A + a
        for k in ALLOC_FIELDS:
            assert same_bytes(above2[k][idx], above[k][idx]), (l, a, k)
        if trace:
            assert same_bytes(th2[:l], th[:l]), (l, a)


@pytest.mark.parametrize("trace", [False, True])
def test_demand_by_level_with_row_acc_count_is_allocate_by_type(oracle_mod, trace):
    """units[l, j] with perf_acc_count rows equals AllocateByType's count of a's type over the oracle's winners on
    row l's fleet (its AccCount) at price p, at each union stretch's start and one ulp below each breakpoint."""
    fleet = moving_fleet(27)
    rows = price_case(fleet, 4, "acc_count", 12)
    rows["perf_acc_count"][2] = 3
    th, _, cand, _, fleets = ref_price_rows(oracle_mod, fleet, rows, trace)
    cand = _to_allocs(cand)
    spread = 0
    for a in range(fleet.n_acc):
        bp, units = demand_by_level(fleet, th, cand, a, perf_acc_count=rows["perf_acc_count"])
        assert units.shape == (len(fleets), bp.size + 1) and (np.diff(bp) > 0).all()
        starts = [F32(0.0)] + list(bp)
        for l, f in enumerate(fleets):
            for j, x in enumerate(starts):
                for p, want in [(x, units[l, j])] + ([(pred(x), units[l, j - 1])] if j else []):
                    fp = at_price(f, a, p)
                    got = oracle_mod.allocate_by_type(fp, oracle_mod.solve(fp)[1])[a]["count"]
                    assert int(got) == int(want), (a, l, j, p)
        spread += bp.size
    assert spread >= 3
    # without the rows the count reads the fleet's own AccCount: row 2 then differs somewhere
    assert any((demand_by_level(fleet, th, cand, a)[1] != demand_by_level(
        fleet, th, cand, a, perf_acc_count=rows["perf_acc_count"])[1]).any() for a in range(fleet.n_acc))
    with pytest.raises(ValueError):
        demand_by_level(fleet, th, cand, 0, perf_acc_count=rows["perf_acc_count"][:1])


# ---- GPU: bit for bit against the composition ---------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_profile_rows(engine, oracle_mod, kind, keep, trace):
    """Every kind of profile row with load rows (0, negative, +Inf, tiny and huge rates), and with token rows."""
    fleet = edge_fleet(41 + keep, keep)
    for tokens in (False, True):
        rows = price_case(fleet, 5, kind, 17, tokens)
        ref = ref_price_rows(oracle_mod, fleet, rows, trace)
        where = cost_refused(ref[4])
        if where is not None:  # a carried NaN or infinite cost: the call refuses, naming the server and tick
            assert trace
            assert error_code(lambda: run(engine, trace, fleet, rows))[0] == WVA_ERR_UNSUPPORTED
            assert f"server {where[1]}, tick {where[0]}".encode() in engine._L.wva_last_error(engine._h)
            continue
        check_profile_price_rows(engine, oracle_mod, fleet, rows, trace,
                                 f"{kind}, tokens = {tokens}, keep = {keep}, trace = {trace}", ref)


@pytest.mark.gpu
def test_trace_with_a_moving_current_allocation(engine, oracle_mod):
    fleet = moving_fleet(43)
    for kind in ("prices", "acc_count", "mixed"):
        check_profile_price_rows(engine, oracle_mod, fleet, price_case(fleet, 6, kind, 3), True, f"moving c_t, {kind}")


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = mixed_fleet(40, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    rows = price_case(fleet, 3, "mixed", 29, tokens=True)
    return fleet, rows, {t: ref_price_rows(oracle_mod, fleet, rows, t) for t in (False, True)}


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, oracle_mod, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rows, ref = rounds_case
    for trace in (False, True):
        check_profile_price_rows(engine, oracle_mod, fleet, rows, trace, f"rounds, D = {depth}, trace = {trace}",
                                 ref[trace])


@pytest.mark.gpu
@pytest.mark.parametrize("n_acc", [32, 33])
def test_many_accelerators(engine, oracle_mod, n_acc):
    """A = 32 and 33: lanes own one accelerator, or lane 0 owns two; ties across the strided lanes."""
    fleet = synth_fleet(4, n_acc, seed=41 + n_acc, zero_load_frac=0.2)
    fleet.accel_penalty_factor = 0.0
    fleet.acc_cost[n_acc - 1] = fleet.acc_cost[0]
    for k in ("perf_alpha", "perf_beta", "perf_gamma", "perf_delta", "perf_acc_count", "perf_max_batch",
              "perf_at_tokens", "perf_present"):
        getattr(fleet, k)[:, n_acc - 1] = getattr(fleet, k)[:, 0]
    for kind in ("prices", "acc_count"):
        rows = price_case(fleet, 4, kind, 7)
        rows["arrival_rpm"] = np.abs(rows["arrival_rpm"]).clip(1, 1e4).astype(F32)
        for trace in (False, True):
            check_profile_price_rows(engine, oracle_mod, fleet, rows, trace, f"A = {n_acc}, {kind}, trace = {trace}")


@pytest.mark.gpu
def test_stored_vector_fallback(engine, oracle_mod):
    """N = 1024 near saturation: the tail re-runs the solves on the stored vector."""
    fleet = overflow_fleet()
    rates = [rates_at_rate_star(oracle_mod, fleet, s, 0) for s in range(fleet.n_servers)]
    rows = own_profile(fleet, 3)
    rows = {"acc_cost": (rows["acc_cost"] * np.array([[1.0], [0.5], [2.0]])).astype(F32),
            "perf_acc_count": rows["perf_acc_count"] + np.arange(3)[:, None, None].astype(np.int32),
            "arrival_rpm": np.array([[r[k % len(r)] for r in rates] for k in range(3)], F32)}
    for trace in (False, True):
        _, cand, _, _ = check_profile_price_rows(engine, oracle_mod, fleet, rows, trace,
                                                 f"stored-vector fallback, trace = {trace}")
        assert cand["feasible"].sum() >= 1


@pytest.mark.gpu
def test_current_costs_at_the_edges(engine, oracle_mod):
    """Current costs 0, 1e38 and -MaxFloat32 (edge_fleet) under AccCount and price rows, grid and trace."""
    fleet = edge_fleet(19, factor=0.0)
    assert {0.0, F32(1e38), -F32_MAX} <= set(fleet.srv_cur_cost.tolist())
    for trace in (False, True):
        check_profile_price_rows(engine, oracle_mod, fleet, price_case(fleet, 4, "acc_count", 2), trace,
                                 f"edge costs, trace = {trace}")


@pytest.mark.gpu
@pytest.mark.parametrize("k", [32, 33])
def test_continuation(engine, oracle_mod, k):
    """Ticks 0..L-1 equal ticks 0..k-1 of one call then ticks k..L-1 on the fleet with c_k."""
    fleet = moving_fleet(53)
    L = 40
    rows = price_case(fleet, L, "mixed", 8)
    full = run(engine, True, fleet, rows, want_candidates=True)
    S, A = fleet.n_servers, fleet.n_acc
    head = {key: (v[:k] if v is not None else None) for key, v in rows.items()}
    tail = {key: (v[k:] if v is not None else None) for key, v in rows.items()}
    first = run(engine, True, fleet, head, want_candidates=True)
    cur = fleet
    for t in range(k):
        cur = cur.apply_winners(_rec(first[3], t * S, (t + 1) * S))
    second = run(engine, True, cur, tail, want_candidates=True)
    assert same_bytes(full[0][:k], first[0]) and same_bytes(full[0][k:], second[0])
    for i, n in ((1, S * A), (2, S * A), (3, S)):
        _same(_rec(full[i], 0, k * n), first[i], f"head {i}")
        _same(_rec(full[i], k * n, L * n), second[i], f"tail {i}")


@pytest.mark.gpu
def test_look_back_past_32_ticks(engine, oracle_mod):
    """perf_present off on every accelerator for 31 to 95 ticks: no feasible winner in that run, so price_kernel's
    look-back for c_t reaches over one, two or three ballots of 32 ticks."""
    fleet = synth_fleet(6, 3, seed=59, zero_load_frac=0.0)
    fleet.accel_penalty_factor = 0.0
    fleet.srv_min_replicas[:] = 1
    L = 110
    rows = own_profile(fleet, L)
    prof = {"perf_present": rows["perf_present"],
            "acc_cost": (rows["acc_cost"] * (1.0 + 0.5 * np.sin(np.arange(L) / 3.0))[:, None]).astype(F32)}
    for m, (start, gap) in enumerate(((4, 31), (5, 64), (6, 95))):
        prof["perf_present"][start:start + gap, m % fleet.n_models] = 0
    rows = {"arrival_rpm": np.repeat(fleet.srv_arrival_rpm[None], L, axis=0).astype(F32), **prof}
    ref = ref_price_rows(oracle_mod, fleet, rows, True)
    check_profile_price_rows(engine, oracle_mod, fleet, rows, True, "look-back", ref)
    win = ref[3].reshape(L, -1)
    assert (~win["feasible"].astype(bool)).sum(axis=0).max() >= 95


# ---- GPU: against the price threshold and profile calls, no oracle -------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
def test_null_profile_columns_are_the_price_threshold_calls(engine, trace):
    fleet = mixed_fleet(30, 3, 73, True)
    rows = price_case(fleet, 4, "prices", 19, tokens=True)
    del rows["acc_cost"]
    n0 = engine.launch_count
    want = getattr(engine, PRICE_CALLS[trace])(fleet, rows["arrival_rpm"], rows["in_tokens"], rows["out_tokens"],
                                               want_candidates=True)
    n1 = engine.launch_count
    got = run(engine, trace, fleet, rows, want_candidates=True)
    assert engine.launch_count - n1 == n1 - n0
    for x, y, what in zip(got, want, ("threshold", "above", "candidates", "winners")):
        _same(x, y, what)
    # rows == NULL in the C call is the same
    S, A, L = fleet.n_servers, fleet.n_acc, 4
    th = np.zeros(L * S * A, F32)
    win = Allocs(L * S)
    fn = getattr(engine._L, "wva_" + CALLS[trace])
    assert fn(engine._h, C.byref(fleet.as_c()), L, _abi.ptr(rows["arrival_rpm"].reshape(-1)),
              _abi.ptr(rows["in_tokens"].reshape(-1)), _abi.ptr(rows["out_tokens"].reshape(-1)), None,
              _abi.ptr(th), None, None, C.byref(win.as_c())) == 0
    assert same_bytes(th, want[0].reshape(-1))
    _same(win, want[3], "winners, rows NULL")


@pytest.fixture(scope="module")
def big_case():
    fleet = synth_fleet(1500, 8, seed=61)
    rng = np.random.default_rng(62)
    L = 24
    own = own_profile(fleet, L)
    hours = 1.0 + 0.4 * np.sin(2 * np.pi * (np.arange(L)[:, None] / L + rng.uniform(0, 1, fleet.n_acc)[None]))
    beta = own["perf_beta"].copy()
    beta[8:, :, 2] *= F32(0.9)
    present = own["perf_present"].copy()
    present[:12, :, 7] = 0
    acc_count = own["perf_acc_count"].copy()
    acc_count[16:, :, 1] = 2
    rows = {"arrival_rpm": (fleet.srv_arrival_rpm[None] * rng.lognormal(0, 0.6, (L, fleet.n_servers))).astype(F32),
            "out_tokens": np.maximum(fleet.srv_out_tokens[None] * rng.choice([0.5, 1, 2], (L, fleet.n_servers)),
                                     1).astype(np.int32),
            "acc_cost": (own["acc_cost"] * hours).astype(F32), "perf_beta": beta, "perf_present": present,
            "perf_acc_count": acc_count}
    return fleet, rows


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
def test_every_block_is_the_single_call(engine, big_case, trace):
    """Each block equals wva_price_thresholds on f_l (f_t, with c_t from the trace's own winners) byte for byte, and
    the candidates and winners equal wva_profile_trace's (grid: wva_solve's on f_l)."""
    fleet, rows = big_case
    S, A = fleet.n_servers, fleet.n_acc
    th, above, cand, win = run(engine, trace, fleet, rows, want_candidates=True)
    if trace:
        c_ref, w_ref = engine.profile_trace(fleet, **rows, want_candidates=True)
        _same(cand, c_ref, "candidates")
        _same(win, w_ref, "winners")
    cur = fleet
    for l in range(th.shape[0]):
        f = at_row(cur, rows, l)
        th1, above1, cand1 = engine.price_thresholds(f, want_candidates=True)
        assert same_bytes(th[l], th1), l
        _same(_rec(above, l * S * A, (l + 1) * S * A), above1, f"above {l}")
        _same(_rec(cand, l * S * A, (l + 1) * S * A), cand1, f"candidates {l}")
        if not trace and l in (0, 12, 23):
            _, w1 = engine.solve(f)
            _same(_rec(win, l * S, (l + 1) * S), w1, f"winners {l}")
        if trace:
            cur = cur.apply_winners(_rec(win, l * S, (l + 1) * S))
    assert ((th > 0) & np.isfinite(th)).sum() >= 100


@pytest.mark.gpu
def test_grid_at_the_fleets_own_load_is_the_profile_grid(engine, big_case):
    fleet, rows = big_case
    prof = {k: v for k, v in rows.items() if k not in ("arrival_rpm", "out_tokens")}
    L = rows["acc_cost"].shape[0]
    own = np.repeat(fleet.srv_arrival_rpm[None], L, axis=0).astype(F32)
    _, _, cand, win = engine.profile_price_threshold_grid(fleet, own, want_candidates=True, **prof)
    c_ref, w_ref = engine.profile_grid(fleet, want_candidates=True, **prof)
    _same(cand, c_ref, "candidates")
    _same(win, w_ref, "winners")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
def test_profile_grid_at_each_threshold(engine, big_case, trace):
    """wva_profile_grid on f_l at each finite threshold of level l and the float below it: a wins below and not at
    the threshold, and above is the winner there."""
    fleet, rows = big_case
    S, A = fleet.n_servers, fleet.n_acc
    th, above, _, win = run(engine, trace, fleet, rows)
    cur, pairs = fleet, 0
    for l in range(th.shape[0]):
        f = at_row(cur, rows, l)
        if trace:
            cur = cur.apply_winners(_rec(win, l * S, (l + 1) * S))
        if l not in (0, 13, 23):
            continue
        prices, index = [], {}
        for a in range(A):
            for t in np.unique(th[l, :, a][(th[l, :, a] > 0) & np.isfinite(th[l, :, a])])[:40]:
                for p in (t, pred(t)):
                    index[(a, u32_bits(p))] = len(prices)
                    r = f.acc_cost.copy()
                    r[a] = p
                    prices.append(r)
        _, pw = engine.profile_grid(f, acc_cost=np.array(prices, F32))
        for s in range(S):
            for a in range(A):
                t = th[l, s, a]
                if (a, u32_bits(t)) not in index or (a, u32_bits(pred(t))) not in index:
                    continue
                at, below = index[(a, u32_bits(t))] * S + s, index[(a, u32_bits(pred(t)))] * S + s
                assert pw.feasible[below] == 1 and pw.acc[below] == a, (l, s, a)
                assert not (pw.feasible[at] == 1 and pw.acc[at] == a), (l, s, a)
                for k in ALLOC_FIELDS:
                    assert same_bytes(getattr(pw, k)[at], getattr(above, k)[(l * S + s) * A + a]), (l, s, a, k)
                pairs += 1
    assert pairs >= 100


@pytest.mark.gpu
def test_a_price_at_tick_t_moves_nothing_before_it(engine, big_case):
    """Changing acc_cost[a] at tick t leaves trace blocks 0..t-1 and column a of block t unchanged."""
    fleet, rows = big_case
    th, above, _, _ = run(engine, True, fleet, rows)
    S, A = fleet.n_servers, fleet.n_acc
    for t, a in ((5, 0), (17, 6)):
        moved = dict(rows)
        moved["acc_cost"] = rows["acc_cost"].copy()
        moved["acc_cost"][t, a] *= F32(0.4)
        th2, above2, _, _ = run(engine, True, fleet, moved)
        assert same_bytes(th2[:t], th[:t]) and same_bytes(th2[t, :, a], th[t, :, a]), (t, a)
        idx = (t * S + np.arange(S)) * A + a
        for k in ALLOC_FIELDS:
            assert same_bytes(getattr(above2, k)[:t * S * A], getattr(above, k)[:t * S * A]), (t, k)
            assert same_bytes(getattr(above2, k)[idx], getattr(above, k)[idx]), (t, k)
        assert not same_bytes(th2[t], th[t]) or not same_bytes(th2[t + 1:], th[t + 1:])


# ---- GPU: refusals and bookkeeping ----------------------------------------------------------------

def _code(engine, trace, fleet, rows):
    return error_code(lambda: run(engine, trace, fleet, rows))[0]


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
def test_refusals(engine, trace):
    fleet = mixed_fleet(8, 2, 79, False)
    fleet.srv_model[3] = 0
    fleet.srv_model[0] = 0
    fleet.srv_has_target[0] = 1
    L = 3
    own = own_profile(fleet, L)
    rows = {"arrival_rpm": np.repeat(fleet.srv_arrival_rpm[None], L, axis=0), "acc_cost": own["acc_cost"]}
    assert _code(engine, trace, fleet, rows) == 0
    for factor in (np.nan, -0.5, np.inf):
        f = fleet.take_servers(np.arange(fleet.n_servers))
        f.accel_penalty_factor = factor
        assert _code(engine, trace, f, rows) == WVA_ERR_UNSUPPORTED, factor
    m = int(fleet.srv_model[0])
    for cost in (np.nan, np.inf, -np.inf):
        f = fleet.take_servers(np.arange(fleet.n_servers))
        f.srv_cur_cost[0] = cost
        f.srv_cur_acc[0] = -1
        f.srv_arrival_rpm[0] = 5.0
        r = dict(rows, perf_present=own["perf_present"].copy())
        r["arrival_rpm"] = rows["arrival_rpm"].copy()
        r["arrival_rpm"][:, 0] = 5.0
        r["perf_present"][:, m, :] = 0  # never present: nothing to refuse
        assert _code(engine, trace, f, r) == 0, cost
        r["perf_present"][1, m, 0] = 1  # present at row 1 only
        assert _code(engine, trace, f, r) == WVA_ERR_UNSUPPORTED, cost
        assert b"server 0" in engine._L.wva_last_error(engine._h)
        assert error_code(lambda: engine.price_thresholds(at_row(f, r, 1)))[0] == WVA_ERR_UNSUPPORTED


@pytest.mark.gpu
@pytest.mark.parametrize("price", [np.inf, np.nan])
def test_trace_refuses_a_carried_non_finite_cost(engine, price):
    """A winner with c_t's accelerator and replica count has value 0 whatever its cost; at an edge price of +Inf or
    NaN that cost becomes c_1's.  The trace refuses at tick 1; the grid, whose current cost stays the fleet's, does
    not."""
    fleet = synth_fleet(3, 1, seed=87, zero_load_frac=0.0)
    cand = engine.analyze(fleet)
    assert cand.feasible.all()
    fleet.srv_keep_acc[:] = 0
    fleet.srv_cur_acc[:] = 0
    fleet.srv_cur_replicas[:] = cand.replicas
    fleet.srv_cur_cost[:] = 0.0
    rows = {"arrival_rpm": np.repeat(fleet.srv_arrival_rpm[None], 2, axis=0).astype(F32),
            "acc_cost": np.array([[price], [fleet.acc_cost[0]]], F32)}
    assert _code(engine, False, fleet, rows) == 0
    _, win = engine.profile_trace(fleet, **rows)
    assert not np.isfinite(win.cost[:3]).any()
    assert _code(engine, True, fleet, rows) == WVA_ERR_UNSUPPORTED
    assert b"tick 1" in engine._L.wva_last_error(engine._h)


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
def test_argument_errors_and_empty_calls(engine, trace):
    fleet = mixed_fleet(6, 2, 79, False)
    S, A, L = fleet.n_servers, fleet.n_acc, 2
    fn = getattr(engine._L, "wva_" + CALLS[trace])
    h, fc = engine._h, fleet.as_c()
    rpm = np.repeat(fleet.srv_arrival_rpm[None], L, axis=0).astype(F32)
    cost = np.repeat(fleet.acc_cost[None], L, axis=0).astype(F32)
    rc_ = _abi.ProfileRowsC(_abi.ptr(cost.reshape(-1)), *([None] * 8))
    th = np.zeros(L * S * A, F32)
    win = Allocs(L * S)
    args = lambda n, r, t, w: (C.byref(fc), n, r, None, None, C.byref(rc_), t, None, None, w)  # noqa: E731
    assert fn(None, *args(L, _abi.ptr(rpm), _abi.ptr(th), C.byref(win.as_c()))) == WVA_ERR_BAD_ARG
    assert fn(h, *args(L, _abi.ptr(rpm), _abi.ptr(th), None)) == WVA_ERR_BAD_ARG
    assert fn(h, *args(-1, _abi.ptr(rpm), _abi.ptr(th), C.byref(win.as_c()))) == WVA_ERR_BAD_ARG
    assert fn(h, *args(L, None, _abi.ptr(th), C.byref(win.as_c()))) == WVA_ERR_BAD_ARG
    assert fn(h, *args(L, _abi.ptr(rpm), None, C.byref(win.as_c()))) == WVA_ERR_BAD_ARG
    assert fn(h, None, L, _abi.ptr(rpm), None, None, C.byref(rc_), _abi.ptr(th), None, None,
              C.byref(win.as_c())) == WVA_ERR_BAD_ARG
    assert fn(h, *args(L, _abi.ptr(rpm), _abi.ptr(th), C.byref(win.as_c()))) == 0
    ref = run(engine, trace, fleet, {"arrival_rpm": rpm, "acc_cost": cost})
    assert same_bytes(th, ref[0].reshape(-1))
    _same(win, ref[3], "winners")
    th0, above0, cand0, win0 = run(engine, trace, fleet, {"arrival_rpm": rpm[:0], "acc_cost": cost[:0]}, True)
    assert th0.shape == (0, S, A) and above0.n == cand0.n == win0.n == 0
    empty = fleet.take_servers(np.arange(0))
    th0, above0, _, win0 = run(engine, trace, empty, {"arrival_rpm": np.zeros((3, 0), F32),
                                                      "acc_cost": np.repeat(cost[:1], 3, axis=0)})
    assert th0.shape == (3, 0, A) and above0.n == win0.n == 0
    with pytest.raises(ValueError):
        getattr(engine, CALLS[trace])(fleet, None, acc_cost=cost)


@pytest.mark.gpu
def test_one_handle_with_the_other_paths(engine):
    fleet = mixed_fleet(30, 3, 73, True)
    rows = price_case(fleet, 4, "mixed", 19, tokens=True)
    fresh = Engine(0)
    try:
        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if x is not None:
                    _same(x, y, what)

        grid = lambda e: run(e, False, fleet, rows, True)  # noqa: E731
        trace = lambda e: run(e, True, fleet, rows, True)  # noqa: E731
        check(trace, "trace")
        check(lambda e: e.price_thresholds(fleet, want_candidates=True), "single call after the trace")
        check(grid, "grid after the single call")
        check(lambda e: e.profile_trace(fleet, **rows, want_candidates=True), "profile trace after the grid")
        check(lambda e: e.price_threshold_trace(fleet, rows["arrival_rpm"], rows["in_tokens"], rows["out_tokens"],
                                                want_candidates=True), "price threshold trace")
        check(trace, "trace after the price threshold trace")
    finally:
        fresh.close()
