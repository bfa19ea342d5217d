"""wva_price_threshold_grid / wva_price_threshold_trace: wva_price_thresholds at every level of a grid or tick of a
trace, in one call.

The expected result is ref_price_rows below: per level the fleet at_row(fleet, rows, l), per tick the fleet of
ref_trace's chain (current allocation c_t), each through the single-fleet composition of wva_price_thresholds
(Server.Calculate, a's record re-priced, the one-server Solver.Solve and a bisection over the float32 bit patterns).
The CPU tests pin that composition to a full Server.Calculate + Solver.Solve at the price, and demand_by_level to
AllocateByType.  The GPU tests compare the CUDA path with it bit for bit, and on a larger fleet with the single call,
the workload calls and wva_profile_grid without the oracle."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import (at_row, from_bits, load_levels, mixed_fleet, n_rows, overflow_fleet, rates_at_rate_star,
                          transition_penalty, u32_bits, workload_levels)
from tests.util import (ALLOC_FIELDS, F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED,
                        assert_allocs_equal, assert_f32_bits_equal, error_code, same_bytes)
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, demand_by_level, synth_fleet

F32 = np.float32
CALLS = {False: "price_threshold_grid", True: "price_threshold_trace"}


# ---- the reference: wva_price_thresholds' composition at each level's or tick's fleet ---------------------------

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


def load_rows(fleet, L, seed):
    return {"arrival_rpm": load_levels(fleet, L, seed)}


def token_rows(fleet, L, seed):
    return dict(zip(("arrival_rpm", "in_tokens", "out_tokens"), workload_levels(fleet, L, seed)))


def moving_fleet(seed):
    """Penalty factor 0 and min_replicas 1: the cheapest accelerator wins, so c_t changes accelerator on the trace."""
    f = edge_fleet(seed, factor=0.0)
    f.srv_min_replicas[:] = 1
    return f


def _to_allocs(rec):
    out = Allocs(rec.size)
    for k in ALLOC_FIELDS:
        getattr(out, k)[:] = rec[k]
    return out


def _check(engine, oracle_mod, fleet, rows, trace, what, ref=None):
    th_o, above_o, cand_o, win_o, _ = ref if ref is not None else ref_price_rows(oracle_mod, fleet, rows, trace)
    th_g, above_g, cand_g, win_g = getattr(engine, CALLS[trace])(fleet, **rows, want_candidates=True)
    assert_f32_bits_equal(th_g.reshape(-1), th_o.reshape(-1), f"{what}: threshold")
    assert_allocs_equal(above_g, above_o, f"{what}: above")
    assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
    assert_allocs_equal(win_g, win_o, f"{what}: winners")
    return th_o, cand_o, win_o


# ---- CPU: the composition ---------------------------------------------------------------------

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


@pytest.mark.parametrize("rows_of,keep,trace", [
    (load_rows, False, False), (load_rows, True, False), (token_rows, False, False), (token_rows, True, True),
    (load_rows, False, True),
])
def test_a_wins_exactly_below_each_rows_threshold(oracle_mod, rows_of, keep, trace):
    """At every level's (tick's) fleet, "a wins" from a full Calculate + Solve at price p equals p < threshold, at
    every threshold, the float below it, 0, MaxFloat32 and random bit patterns."""
    fleet = edge_fleet(21 + keep, keep)
    rows = rows_of(fleet, 3, 5)
    th, _, _, _, fleets = ref_price_rows(oracle_mod, fleet, rows, trace)
    rng = np.random.default_rng(9)
    kinds = set()
    for l, f in enumerate(fleets):
        for a in range(fleet.n_acc):
            for p in _prices(th[l, :, a], rng, 3):
                assert (_a_wins(oracle_mod, f, a, p) == (p < th[l, :, a])).all(), (l, a, p)
            kinds |= {"0" if t == 0 else "inf" if np.isinf(t) else "finite" for t in th[l, :, a]}
    assert {"0", "finite"} <= kinds


def test_trace_composition_with_a_moving_current_allocation(oracle_mod):
    """A trace whose c_t changes accelerator: the thresholds of tick t are read against c_t, not the fleet's own
    current allocation, and "a wins" still holds exactly below them."""
    fleet = moving_fleet(23)
    rows = load_rows(fleet, 4, 8)
    th, _, _, win, fleets = ref_price_rows(oracle_mod, fleet, rows, True)
    S = fleet.n_servers
    w = win.reshape(-1, S)
    moved = sum(1 for t in range(1, w.shape[0]) for s in range(S)
                if fleets[t].srv_cur_acc[s] != fleet.srv_cur_acc[s])
    assert moved >= 2
    assert (th != ref_price_rows(oracle_mod, fleet, rows, False)[0]).any()
    rng = np.random.default_rng(4)
    for t in range(1, len(fleets)):
        for a in range(fleet.n_acc):
            for p in _prices(th[t, :, a], rng, 2):
                assert (_a_wins(oracle_mod, fleets[t], a, p) == (p < th[t, :, a])).all(), (t, a, p)


@pytest.mark.parametrize("trace", [False, True])
def test_demand_by_level_is_allocate_by_type(oracle_mod, trace):
    """units[l, j] equals AllocateByType's count of a's type over the oracle's winners on level l's fleet at price
    p, at each union stretch's start and one ulp below each breakpoint."""
    fleet = moving_fleet(27)
    rows = load_rows(fleet, 3, 12)
    th, _, cand, _, fleets = ref_price_rows(oracle_mod, fleet, rows, trace)
    cand = _to_allocs(cand)
    spread = 0
    for a in range(fleet.n_acc):
        bp, units = demand_by_level(fleet, th, cand, a)
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
    with pytest.raises(ValueError):
        demand_by_level(fleet, th[0], cand, 0)


# ---- GPU: bit for bit against the composition ---------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("rows_of", [load_rows, token_rows])
def test_mixed_fleet_rows(engine, oracle_mod, rows_of, keep, trace):
    """mixed_fleet with load_levels rows (0, negative, +Inf, tiny and huge rates) or workload_levels rows."""
    fleet = edge_fleet(41 + keep, keep)
    th, _, _ = _check(engine, oracle_mod, fleet, rows_of(fleet, 5, 17), trace,
                      f"{rows_of.__name__}, keep = {keep}, trace = {trace}")
    assert ((th > 0) & np.isfinite(th)).sum() >= 3


@pytest.mark.gpu
def test_trace_with_a_moving_current_allocation(engine, oracle_mod):
    _check(engine, oracle_mod, moving_fleet(43), load_rows(moving_fleet(43), 6, 3), True, "moving c_t")


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = mixed_fleet(40, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    rows = token_rows(fleet, 3, 29)
    return fleet, rows, {t: ref_price_rows(oracle_mod, fleet, rows, t) for t in (False, True)}


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, oracle_mod, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rows, ref = rounds_case
    for trace in (False, True):
        _check(engine, oracle_mod, fleet, rows, trace, f"rounds, D = {depth}, trace = {trace}", ref[trace])


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
    rows = load_rows(fleet, 2, 7)
    for trace in (False, True):
        _check(engine, oracle_mod, fleet, rows, trace, f"A = {n_acc}, trace = {trace}")


@pytest.mark.gpu
def test_stored_vector_fallback(engine, oracle_mod):
    """N = 1024 near saturation: the tail re-runs the solves on the stored vector."""
    fleet = overflow_fleet()
    rates = [rates_at_rate_star(oracle_mod, fleet, s, 0) for s in range(fleet.n_servers)]
    rows = {"arrival_rpm": np.array([[r[k % len(r)] for r in rates] for k in range(3)], F32)}
    for trace in (False, True):
        _, cand, _ = _check(engine, oracle_mod, fleet, rows, trace, f"stored-vector fallback, trace = {trace}")
        assert cand["feasible"].sum() >= 1


@pytest.mark.gpu
def test_nan_and_huge_values_and_ties(engine, oracle_mod):
    """Values that are NaN (an overflowed cost under factor 0) or MaxFloat32, huge prices and ties on value."""
    fleet = edge_fleet(19, factor=0.0)
    fleet.acc_cost[0] = F32(1e38)
    fleet.acc_cost[3] = F32_MAX
    fleet.srv_cur_cost[fleet.srv_cur_cost > F32(1e37)] = 0.0  # keep the trace's carried costs finite
    for trace in (False, True):
        _check(engine, oracle_mod, fleet, load_rows(fleet, 3, 2), trace, f"NaN / huge values, trace = {trace}")


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_current_allocation_equal_to_a_candidate(engine, oracle_mod, keep):
    """A current allocation that is a's candidate itself at a level: its value is 0 at every price, so the
    threshold is 0 or +Inf."""
    fleet = edge_fleet(13, keep)
    rows = load_rows(fleet, 3, 6)
    cand = oracle_mod.calculate(at_row(fleet, rows, 0))
    same = []
    for s in range(0, fleet.n_servers, 2):
        fe = np.nonzero(cand[s]["feasible"] & (cand[s]["acc"] >= 0))[0]
        if fe.size:
            a = int(fe[-1])
            fleet.srv_cur_acc[s], fleet.srv_cur_replicas[s] = a, cand[s, a]["replicas"]
            fleet.srv_cur_cost[s] = cand[s, a]["cost"]
            same.append((s, a))
    assert len(same) >= 2
    th, _, _ = _check(engine, oracle_mod, fleet, rows, False, f"same replica count, keep = {keep}")
    assert all(th[0, s, a] == 0 or np.isinf(th[0, s, a]) for s, a in same)
    _check(engine, oracle_mod, fleet, rows, True, f"same replica count, trace, keep = {keep}")


@pytest.mark.gpu
def test_zero_load_min_replicas_zero(engine, oracle_mod):
    fleet = edge_fleet(17)
    fleet.srv_min_replicas[::4] = 0
    fleet.srv_min_replicas[2::4] = 1
    rows = load_rows(fleet, 3, 11)
    rows["arrival_rpm"][:, ::2] = 0.0
    for trace in (False, True):
        _, cand, _ = _check(engine, oracle_mod, fleet, rows, trace, f"zero load, trace = {trace}")
        assert ((cand["acc"] == -1) & (cand["feasible"] == 1)).sum() >= 2


# ---- GPU: against the single call and the workload calls, no oracle --------------------------------

@pytest.fixture(scope="module")
def big_case():
    fleet = synth_fleet(1500, 8, seed=61)
    rng = np.random.default_rng(62)
    rows = {"arrival_rpm": (fleet.srv_arrival_rpm[None] * rng.lognormal(0, 0.6, (24, fleet.n_servers))).astype(F32),
            "out_tokens": np.maximum(fleet.srv_out_tokens[None] * rng.choice([0.5, 1, 2], (24, fleet.n_servers)),
                                     1).astype(np.int32)}
    return fleet, rows


def _rec(allocs, lo, hi):
    """Records [lo, hi) of an Allocs, as an Allocs."""
    out = Allocs(hi - lo)
    for k in ALLOC_FIELDS:
        getattr(out, k)[:] = getattr(allocs, k)[lo:hi]
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
def test_every_block_is_the_single_call(engine, big_case, trace):
    """Each block equals wva_price_thresholds on f_l (f_t, with c_t from the trace's own winners) byte for byte, and
    the winners equal wva_workload_grid's (wva_workload_trace's)."""
    fleet, rows = big_case
    S, A = fleet.n_servers, fleet.n_acc
    th, above, cand, win = getattr(engine, CALLS[trace])(fleet, **rows, want_candidates=True)
    _, w_ref = (engine.workload_trace if trace else engine.workload_grid)(fleet, **rows)
    for k in ALLOC_FIELDS:
        assert same_bytes(getattr(win, k), getattr(w_ref, k)), k
    cur = fleet
    for l in range(th.shape[0]):
        f = at_row(cur, rows, l)
        th1, above1, cand1 = engine.price_thresholds(f, want_candidates=True)
        assert same_bytes(th[l], th1), l
        for k in ALLOC_FIELDS:
            assert same_bytes(getattr(above, k)[l * S * A:(l + 1) * S * A], getattr(above1, k)), (l, k)
            assert same_bytes(getattr(cand, k)[l * S * A:(l + 1) * S * A], getattr(cand1, k)), (l, k)
        if trace:
            cur = cur.apply_winners(_rec(win, l * S, (l + 1) * S))
    assert ((th > 0) & np.isfinite(th)).sum() >= 100


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
def test_profile_grid_at_each_threshold(engine, big_case, trace):
    """wva_profile_grid on f_l at each finite threshold of level l and the float below it: a wins below and not at
    the threshold, and above is the winner there."""
    fleet, rows = big_case
    S, A = fleet.n_servers, fleet.n_acc
    th, above, _, win = getattr(engine, CALLS[trace])(fleet, **rows)
    cur, pairs = fleet, 0
    for l in range(th.shape[0]):
        f = at_row(cur, rows, l)
        if trace:
            cur = cur.apply_winners(_rec(win, l * S, (l + 1) * S))
        if l not in (0, 7, 23):
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


# ---- GPU: refusals and bookkeeping ----------------------------------------------------------------

def _call(engine, trace, fleet, rows):
    return error_code(lambda: getattr(engine, CALLS[trace])(fleet, **rows))


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
def test_refusals(engine, trace):
    fleet = mixed_fleet(8, 2, 79, False)
    fleet.srv_model[3] = 0
    rows = {"arrival_rpm": np.repeat(fleet.srv_arrival_rpm[None], 3, axis=0)}
    assert _call(engine, trace, fleet, rows)[0] == 0
    for factor in (np.nan, -0.5, np.inf):
        f = fleet.take_servers(np.arange(fleet.n_servers))
        f.accel_penalty_factor = factor
        assert _call(engine, trace, f, rows)[0] == WVA_ERR_UNSUPPORTED, factor
    for cost in (np.nan, np.inf, -np.inf):
        f = fleet.take_servers(np.arange(fleet.n_servers))
        f.srv_cur_cost[0] = cost
        f.srv_arrival_rpm[0] = 5.0
        r = {"arrival_rpm": rows["arrival_rpm"].copy()}
        r["arrival_rpm"][:, 0] = -1.0  # nil at every level: nothing to refuse
        assert _call(engine, trace, f, r)[0] == 0, cost
        r["arrival_rpm"][2, 0] = 5.0  # a candidate at level 2 only
        assert _call(engine, trace, f, r)[0] == WVA_ERR_UNSUPPORTED, cost
        assert b"server 0" in engine._L.wva_last_error(engine._h)
        assert error_code(lambda: engine.price_thresholds(at_row(f, r, 2)))[0] == WVA_ERR_UNSUPPORTED
    # the queue-size rule refuses as the workload call does
    big = synth_fleet(2, 2, seed=83, zero_load_frac=0.0)
    big.srv_max_batch[:] = 1 << 20
    big.max_queue_to_batch_ratio = 1 << 12
    brows = {"arrival_rpm": big.srv_arrival_rpm[None]}
    code = error_code(lambda: (engine.workload_trace if trace else engine.workload_grid)(big, **brows))[0]
    assert code == WVA_ERR_UNSUPPORTED
    assert _call(engine, trace, big, brows)[0] == code


@pytest.mark.gpu
def test_trace_refuses_a_carried_infinite_cost(engine):
    """A winner with c_t's accelerator and replica count has value 0 whatever its cost; at acc_cost MaxFloat32 that
    cost is +Inf and becomes c_1's.  The trace refuses at tick 1, as the single call on f_1 does; the grid, whose
    current cost stays the fleet's, does not."""
    fleet = synth_fleet(3, 1, seed=87, zero_load_frac=0.0)
    fleet.acc_cost[0] = F32_MAX
    fleet.perf_acc_count[:, 0] = 2
    cand = engine.analyze(fleet)
    assert cand.feasible.all()
    fleet.srv_keep_acc[:] = 0
    fleet.srv_cur_acc[:] = 0
    fleet.srv_cur_replicas[:] = cand.replicas
    fleet.srv_cur_cost[:] = 0.0
    rows = {"arrival_rpm": np.repeat(fleet.srv_arrival_rpm[None], 2, axis=0)}
    assert _call(engine, False, fleet, rows)[0] == 0
    assert _call(engine, True, fleet, {"arrival_rpm": rows["arrival_rpm"][:1]})[0] == 0
    _, win = engine.workload_trace(fleet, **rows)
    assert np.isinf(win.cost[:3]).all()
    assert _call(engine, True, fleet, rows)[0] == WVA_ERR_UNSUPPORTED
    assert b"tick 1" in engine._L.wva_last_error(engine._h)
    f1 = at_row(fleet.apply_winners(_rec(win, 0, 3)), rows, 1)
    assert error_code(lambda: engine.price_thresholds(f1))[0] == WVA_ERR_UNSUPPORTED


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
def test_argument_errors_and_empty_calls(engine, trace):
    fleet = mixed_fleet(6, 2, 79, False)
    S, A, L = fleet.n_servers, fleet.n_acc, 2
    fn = getattr(engine._L, "wva_" + CALLS[trace])
    h, fc = engine._h, fleet.as_c()
    rpm = np.repeat(fleet.srv_arrival_rpm[None], L, axis=0).astype(F32)
    th = np.zeros(L * S * A, F32)
    win = Allocs(L * S)
    p = lambda x: x.ctypes.data_as(C.POINTER(C.c_float))  # noqa: E731
    args = lambda n, r, t, w: (C.byref(fc), n, r, None, None, t, None, None, w)  # noqa: E731
    assert fn(None, *args(L, p(rpm), p(th), C.byref(win.as_c()))) == WVA_ERR_BAD_ARG
    assert fn(h, *args(L, p(rpm), p(th), None)) == WVA_ERR_BAD_ARG
    assert fn(h, *args(-1, p(rpm), p(th), C.byref(win.as_c()))) == WVA_ERR_BAD_ARG
    assert fn(h, *args(L, None, p(th), C.byref(win.as_c()))) == WVA_ERR_BAD_ARG
    assert fn(h, *args(L, p(rpm), None, C.byref(win.as_c()))) == WVA_ERR_BAD_ARG
    assert fn(h, None, L, p(rpm), None, None, p(th), None, None, C.byref(win.as_c())) == WVA_ERR_BAD_ARG
    # NULL token lists, above and candidates: the thresholds alone, the fleet's own tokens
    assert fn(h, *args(L, p(rpm), p(th), C.byref(win.as_c()))) == 0
    ref = getattr(engine, CALLS[trace])(fleet, rpm, fleet.srv_in_tokens[None].repeat(L, 0),
                                        fleet.srv_out_tokens[None].repeat(L, 0))
    assert same_bytes(th, ref[0].reshape(-1))
    for k in ALLOC_FIELDS:
        assert same_bytes(getattr(win, k), getattr(ref[3], k)), k
    th0, above0, cand0, win0 = getattr(engine, CALLS[trace])(fleet, rpm[:0], want_candidates=True)
    assert th0.shape == (0, S, A) and above0.n == cand0.n == win0.n == 0
    empty = fleet.take_servers(np.arange(0))
    th0, above0, _, win0 = getattr(engine, CALLS[trace])(empty, np.zeros((3, 0), F32))
    assert th0.shape == (3, 0, A) and above0.n == win0.n == 0
    with pytest.raises(ValueError):
        getattr(engine, CALLS[trace])(fleet, None)


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
def test_launch_count_does_not_depend_on_the_rows(engine, trace):
    """One price_kernel launch on top of the workload call's, at any L."""
    fleet = synth_fleet(40, 4, seed=71, zero_load_frac=0.0)
    workload = engine.workload_trace if trace else engine.workload_grid

    def launches(call):
        n0 = engine.launch_count
        call()
        return engine.launch_count - n0
    extra = set()
    for L in (1, 4, 16):
        rows = load_rows(fleet, L, 3)
        rows["arrival_rpm"] = np.abs(rows["arrival_rpm"]).clip(1, 1e4)
        extra.add(launches(lambda: getattr(engine, CALLS[trace])(fleet, **rows)) -
                  launches(lambda: workload(fleet, **rows)))
    assert extra == {1}


@pytest.mark.gpu
def test_one_handle_with_the_other_paths(engine):
    fleet = mixed_fleet(30, 3, 73, True)
    rows = token_rows(fleet, 4, 19)
    fresh = Engine(0)
    try:
        def same(x, y, what):
            if isinstance(x, np.ndarray):
                assert same_bytes(x, y), what
                return
            for k in ALLOC_FIELDS:
                assert same_bytes(getattr(x, k), getattr(y, k)), f"{what}: {k}"

        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if x is not None:
                    same(x, y, what)

        grid = lambda e: e.price_threshold_grid(fleet, **rows, want_candidates=True)  # noqa: E731
        trace = lambda e: e.price_threshold_trace(fleet, **rows, want_candidates=True)  # noqa: E731
        cand_s, win_s = engine.solve(fleet)
        grid(engine)
        cand_r, win_r = engine.resolve(want_candidates=True)
        same(cand_r, cand_s, "resolve after the grid: candidates")
        same(win_r, win_s, "resolve after the grid: winners")
        check(trace, "trace")
        check(lambda e: e.price_thresholds(fleet, want_candidates=True), "single call after the trace")
        check(grid, "grid after the single call")
        check(lambda e: e.workload_trace(fleet, **rows, want_candidates=True), "workload trace after the grid")
        check(trace, "trace after the workload trace")
        engine.solve(fleet)
        engine.summarize(fleet.n_types)
        trace(engine)
        with pytest.raises(WvaError) as e:
            engine.summarize(fleet.n_types)
        assert e.value.code == WVA_ERR_STATE
    finally:
        fresh.close()
