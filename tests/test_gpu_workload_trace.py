"""wva_workload_trace: the reference's reconcile replayed over caller-given ticks of (arrival rate, in_tokens,
out_tokens), each tick's winner becoming the next tick's current allocation.

The expected result is composed from the CPU oracle, literally: for each tick t, a copy of the fleet with row t and
current allocation c_t goes through the oracle's Server.Calculate (candidate block t) and Solver.Solve with
unlimited = 1 (winner block t), and c_{t+1} = Fleet.apply_winners (Server.ApplyDesiredAlloc).  The CPU tests pin that
composition against the oracle's own solve and against the reference's ApplyDesiredAlloc, and show on the oracle why
one batched sizing serves every tick: CreateAllocation does not read the current allocation, which enters only
through the value and the keepAccelerator mask.  The GPU tests compare the CUDA path with the composition bit for
bit."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_load_grid import _code, _f32_bits, _same, mixed_fleet, overflow_fleet, rates_at_rate_star
from tests.test_gpu_parity import _adversarial_fleet
from tests.test_gpu_workload_grid import at_level, token_fleet, workload_levels
from tests.util import ALLOC_FIELDS, assert_allocs_equal
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, synth_fleet

F32 = np.float32
F32_MAX = F32(np.finfo(np.float32).max)
ACC_NONE, ACC_UNKNOWN = -1, -2
WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED = -1, -5, -6


def ref_trace(oracle_mod, fleet, rpm, in_tok, out_tok):
    """(candidates [L*S*A], winners [L*S], the fleet with c_L): per tick, Server.Calculate and Solver.Solve
    (unlimited) on the fleet with row t and current allocation c_t, then c_{t+1} = apply_winners."""
    cands, wins = [np.zeros(0, oracle_mod.ALLOC_DTYPE)], [np.zeros(0, oracle_mod.ALLOC_DTYPE)]
    cur = fleet
    for t in range(rpm.shape[0]):
        f = at_level(cur, rpm[t], in_tok[t], out_tok[t])
        cand = oracle_mod.calculate(f)
        win = oracle_mod.solve(f, cand)[1]
        cands.append(cand.reshape(-1))
        wins.append(win)
        cur = cur.apply_winners(win)
    return np.concatenate(cands), np.concatenate(wins), cur


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


# ---- CPU: the composition, the state transition and the split ---------------------------------

@pytest.mark.parametrize("keep", [False, True])
def test_one_tick_is_the_oracle_solve(oracle_mod, keep):
    fleet = token_fleet(12, 3, 5, keep)
    rows = [c[None, :] for c in (fleet.srv_arrival_rpm, fleet.srv_in_tokens, fleet.srv_out_tokens)]
    cand, win, _ = ref_trace(oracle_mod, fleet, *rows)
    cand_o, win_o = oracle_mod.solve(at_level(fleet, *[r[0] for r in rows]))
    assert _same(cand, cand_o.reshape(-1))
    assert _same(win, win_o)
    assert win["feasible"].sum() >= 4


def test_apply_winners_hand_built():
    """TestServer_ApplyDesiredAlloc (server_test.go:731-776): the desired allocation (a new accelerator, 3 replicas,
    cost 150) becomes current; a server without a winner keeps its allocation (the controller skips it); a zero-load
    winner with min_replicas 0 (accelerator "") gives NONE / 0 / 0."""
    fleet = synth_fleet(3, 3, seed=1)
    fleet.srv_cur_acc[:] = [0, 2, 1]
    fleet.srv_cur_replicas[:] = [1, 4, 2]
    fleet.srv_cur_cost[:] = [23.0, 260.0, 80.0]
    win = Allocs(3)
    win.feasible[:] = [1, 0, 1]
    win.acc[:] = [1, 0, ACC_NONE]
    win.replicas[:] = [3, 7, 0]
    win.cost[:] = [150.0, 99.0, 0.0]
    win.value[:] = [5.0, 6.0, 7.0]
    nxt = fleet.apply_winners(win)
    assert nxt.srv_cur_acc.tolist() == [1, 2, ACC_NONE]
    assert nxt.srv_cur_replicas.tolist() == [3, 4, 0]
    assert nxt.srv_cur_cost.tolist() == [150.0, 260.0, 0.0]
    # a copy: the fleet itself and every other column are unchanged
    assert fleet.srv_cur_acc.tolist() == [0, 2, 1] and fleet.srv_cur_cost.tolist() == [23.0, 260.0, 80.0]
    for n in ("srv_arrival_rpm", "srv_keep_acc", "srv_min_replicas", "acc_cost", "perf_alpha"):
        assert _same(getattr(nxt, n), getattr(fleet, n)), n
    # the oracle's structured winners work the same way
    rec = np.zeros(3, [("feasible", "<i4"), ("acc", "<i4"), ("replicas", "<i4"), ("cost", "<f4")])
    for k in rec.dtype.names:
        rec[k] = getattr(win, k)
    assert _same(fleet.apply_winners(rec).srv_cur_cost, nxt.srv_cur_cost)
    with pytest.raises(ValueError):
        fleet.apply_winners(Allocs(2))


@pytest.mark.parametrize("seed", [3, 4])
def test_create_allocation_does_not_read_the_current_allocation(oracle_mod, seed):
    """For random current allocations (keep off), CreateAllocation's records are the same in every field, and
    Server.Calculate's record is that record with value = TransitionPenalty(current, record)."""
    fleet = token_fleet(12, 3, seed, False)
    fleet.srv_keep_acc[:] = 0
    S, A = fleet.n_servers, fleet.n_acc
    rng = np.random.default_rng(seed)
    base = [[oracle_mod.create_allocation(fleet, s, a) for a in range(A)] for s in range(S)]
    checked = 0
    for trial in range(4):
        f = fleet.take_servers(np.arange(S))
        f.srv_cur_acc[:] = rng.integers(-2, A, S)
        f.srv_cur_replicas[:] = rng.integers(0, 6, S)
        f.srv_cur_cost[:] = rng.choice([0.0, 23.0, 150.0, 1e4], S).astype(np.float32)
        cand = oracle_mod.calculate(f)
        for s in range(S):
            for a in range(A):
                rec = oracle_mod.create_allocation(f, s, a)
                for k in ALLOC_FIELDS:
                    assert _f32_bits(rec[k]) == _f32_bits(base[s][a][k]), (trial, s, a, k)
                for k in ALLOC_FIELDS:
                    if k != "value":
                        assert _f32_bits(cand[s, a][k]) == _f32_bits(rec[k]), (trial, s, a, k)
                if rec["feasible"]:
                    want = transition_penalty(f.accel_penalty_factor, f.srv_cur_acc[s], f.srv_cur_replicas[s],
                                              f.srv_cur_cost[s], rec["acc"], rec["replicas"], rec["cost"])
                    assert _f32_bits(cand[s, a]["value"]) == _f32_bits(want), (trial, s, a)
                    checked += 1
    assert checked >= 60


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_pinned_servers_never_move(oracle_mod, seed):
    """Along oracle traces, a pinned server's current accelerator never changes, and a pinned server with an unknown
    accelerator has no feasible candidate at any tick; keep servers that are not pinned do move."""
    fleet = mixed_fleet(24, 3, seed, True)
    fleet.accel_penalty_factor = 0.0
    fleet.srv_cur_acc[5] = ACC_UNKNOWN
    fleet.srv_cur_acc[6] = ACC_NONE
    L = 8
    rpm, in_tok, out_tok = workload_levels(fleet, L, seed, special=False)
    rpm[2, ::4] = 0.0  # zero-load ticks release the min_replicas 0 servers
    pin = pinned(fleet)
    assert pin.sum() >= 8 and (~pin & (fleet.srv_keep_acc != 0)).sum() >= 4 and pin[4] and pin[5]
    cand, win, _ = ref_trace(oracle_mod, fleet, rpm, in_tok, out_tok)
    S, A = fleet.n_servers, fleet.n_acc
    cand, win = cand.reshape(L, S, A), win.reshape(L, S)
    cur = fleet.srv_cur_acc.copy()
    moved = 0
    for t in range(L):
        for s in range(S):
            if pin[s] and cur[s] == ACC_UNKNOWN:
                assert not cand[t, s]["feasible"].any(), (t, s)
            if pin[s]:
                assert not win[t, s]["feasible"] or win[t, s]["acc"] == fleet.srv_cur_acc[s], (t, s)
        nxt = np.where(win[t]["feasible"] != 0, win[t]["acc"], cur)
        assert (nxt[pin] == fleet.srv_cur_acc[pin]).all()
        moved += int((nxt[~pin] != cur[~pin]).sum())
        cur = nxt
    assert moved >= 3


# ---- GPU: bit for bit against the composition -------------------------------------------------

def _check(engine, oracle_mod, fleet, rows, what):
    cand_o, win_o, _ = ref_trace(oracle_mod, fleet, *rows)
    cand_g, win_g = engine.workload_trace(fleet, *rows, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
    assert_allocs_equal(win_g, win_o, f"{what}: winners")
    return cand_o, win_o


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


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet_warp_path(engine, oracle_mod, keep):
    fleet = token_fleet(14, 3, 31, keep)
    cand_o, win_o = _check(engine, oracle_mod, fleet, workload_levels(fleet, 7, 3), f"warp path, keep = {keep}")
    assert cand_o["feasible"].sum() > 40
    assert len(set(win_o["replicas"][win_o["feasible"] == 1].tolist())) >= 3


@pytest.fixture(scope="module")
def rounds_case(oracle_mod):
    fleet = token_fleet(120, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    fleet.accel_penalty_factor = 0.02
    rows = workload_levels(fleet, 4, 11)
    return fleet, rows, ref_trace(oracle_mod, fleet, *rows)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rows, (cand_o, win_o, _) = rounds_case
    cand_g, win_g = engine.workload_trace(fleet, *rows, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"rounds, D = {depth}: candidates")
    assert_allocs_equal(win_g, win_o, f"rounds, D = {depth}: winners")


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("rounds", [False, True])
def test_winners_move_between_accelerators(engine, oracle_mod, monkeypatch, keep, rounds):
    """No penalty for a switch: the winners follow the cheapest accelerator as the load moves, so the current
    accelerator changes along the chain, and with keep the released (min_replicas 0, zero-load) servers move."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = low_penalty_fleet(40, 4, 89, keep)
    if keep:
        fleet.srv_min_replicas[::2] = 0
    rpm, in_tok, out_tok = workload_levels(fleet, 10, 29, special=False)
    rpm[3::4, ::3] = 0.0
    _, win_o = _check(engine, oracle_mod, fleet, (rpm, in_tok, out_tok), f"moving, keep = {keep}")
    assert _moves(win_o, fleet.n_servers) >= (3 if keep else 10)


@pytest.mark.gpu
def test_wva_configuration_every_server_pinned(engine, oracle_mod):
    fleet = wva_fleet(60, 4, 97)
    assert pinned(fleet).all()
    rows = workload_levels(fleet, 6, 31, special=False)
    _, win_o = _check(engine, oracle_mod, fleet, rows, "WVA configuration")
    win = win_o.reshape(6, -1)
    for t in range(6):
        f = win[t]["feasible"] != 0
        assert f.sum() >= 30
        assert (win[t]["acc"][f] == fleet.srv_cur_acc[f]).all()


@pytest.mark.gpu
def test_chain_edges(engine, oracle_mod):
    """Server by server:
    0  no winner at tick 0 (negative rate): c_1 = c_0;
    1  no winner at tick 2 only: c_3 = winner 1;
    2  unknown current accelerator with keep: nil throughout;
    3  unknown current accelerator without keep: replaced at tick 0;
    4  keep, min_replicas 0, zero load at tick 1: winner 1 is NONE / 0 / 0, and tick 2 offers every accelerator;
    5  keep, min_replicas 1, zero load at tick 1: stays on its accelerator."""
    fleet = synth_fleet(6, 3, seed=101, zero_load_frac=0.0)
    fleet.accel_penalty_factor = 0.0
    fleet.srv_keep_acc[:] = [0, 0, 1, 0, 1, 1]
    fleet.srv_cur_acc[:] = [1, 2, ACC_UNKNOWN, ACC_UNKNOWN, 1, 2]
    fleet.srv_cur_replicas[:] = [2, 1, 3, 3, 1, 1]
    fleet.srv_cur_cost[:] = [80.0, 65.0, 10.0, 10.0, 40.0, 65.0]
    fleet.srv_min_replicas[:] = [1, 1, 1, 1, 0, 1]
    L, S, A = 4, fleet.n_servers, fleet.n_acc
    rpm = np.stack([fleet.srv_arrival_rpm] * L).astype(np.float32)
    in_tok = np.stack([fleet.srv_in_tokens] * L).astype(np.int32)
    out_tok = np.stack([fleet.srv_out_tokens] * L).astype(np.int32)
    rpm[0, 0] = -1.0
    rpm[2, 1] = -1.0
    rpm[1, 4] = rpm[1, 5] = 0.0
    cand_o, win_o = _check(engine, oracle_mod, fleet, (rpm, in_tok, out_tok), "chain edges")
    cand_o, win_o = cand_o.reshape(L, S, A), win_o.reshape(L, S)
    # 0: a nil winner at tick 0, so tick 1's values are against c_0
    assert not win_o[0, 0]["feasible"] and win_o[1, 0]["feasible"]
    c1 = cand_o[1, 0][cand_o[1, 0]["feasible"] != 0][0]
    assert _f32_bits(c1["value"]) == _f32_bits(transition_penalty(0.0, 1, 2, 80.0, c1["acc"], c1["replicas"],
                                                                  c1["cost"]))
    # 1: tick 3 is valued against winner 1
    assert win_o[1, 1]["feasible"] and not win_o[2, 1]["feasible"] and win_o[3, 1]["feasible"]
    w1 = win_o[1, 1]
    c3 = cand_o[3, 1][cand_o[3, 1]["feasible"] != 0][0]
    assert _f32_bits(c3["value"]) == _f32_bits(transition_penalty(0.0, w1["acc"], w1["replicas"], w1["cost"],
                                                                  c3["acc"], c3["replicas"], c3["cost"]))
    # 2 and 3
    assert not cand_o[:, 2]["feasible"].any() and not win_o[:, 2]["feasible"].any()
    assert win_o[0, 3]["feasible"] and win_o[0, 3]["acc"] >= 0
    # 4: released to every accelerator after the zero-load tick; 5 stays
    assert (win_o[1, 4]["feasible"], win_o[1, 4]["acc"], win_o[1, 4]["replicas"], win_o[1, 4]["cost"]) == \
        (1, ACC_NONE, 0, 0.0)
    assert cand_o[0, 4]["feasible"].sum() == 1 and cand_o[2, 4]["feasible"].sum() == A
    assert cand_o[2, 5]["feasible"].sum() == 1 and win_o[3, 5]["acc"] == 2


@pytest.mark.gpu
def test_stored_vector_fallback_both_phases(engine, oracle_mod):
    """N = 1024 from out_tokens 64 near saturation (the workload grid's case): the chains overflow float64, so phase
    1's solves and the tail's re-run on the stored vector, tick after tick."""
    fleet = overflow_fleet()
    fleet.srv_max_batch[:] = 0
    fleet.perf_max_batch[:] = 1024
    fleet.perf_at_tokens[:] = 64
    S = fleet.n_servers
    cols = [rates_at_rate_star(oracle_mod, fleet, s, 0) for s in range(S)]
    L = min(len(c) for c in cols)
    rpm = np.stack([np.array(c[:L], np.float32) for c in cols], axis=1)
    out_tok = np.full((L, S), 64, np.int32)
    out_tok[1::4] = 128
    out_tok[3::7, 0] = 32
    in_tok = np.full((L, S), 64, np.int32)
    cand_o, _ = _check(engine, oracle_mod, fleet, (rpm, in_tok, out_tok), "stored-vector fallback")
    assert cand_o["feasible"].sum() >= L


@pytest.mark.gpu
@pytest.mark.parametrize("keep", [False, True])
def test_nan_and_huge_values_and_ties(engine, oracle_mod, keep):
    fleet = token_fleet(12, 3, 47, keep)
    fleet.srv_cur_cost[::2] = np.nan     # penalty NaN except for the current (accelerator, replicas)
    fleet.srv_cur_cost[1::4] = -F32_MAX  # the current accelerator's penalty rounds to MaxFloat32
    fleet.acc_cost[2] = fleet.acc_cost[1]
    fleet.perf_alpha[:, 2] = fleet.perf_alpha[:, 1]  # accelerators 1 and 2 identical: ties on value
    for k in ("perf_beta", "perf_gamma", "perf_delta", "perf_acc_count"):
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]
    _check(engine, oracle_mod, fleet, workload_levels(fleet, 5, 17), f"NaN / huge values and ties, keep = {keep}")


@pytest.mark.gpu
def test_each_tick_is_solve_on_the_advanced_fleet(engine):
    """Tick t is wva_solve (unlimited) on the fleet advanced by apply_winners through ticks 0..t-1, byte for byte;
    an L = 1 trace is wva_workload_grid with L = 1."""
    fleet = token_fleet(30, 4, 67, True)
    fleet.accel_penalty_factor = 0.01
    L = 6
    rows = workload_levels(fleet, L, 19)
    cand_g, win_g = engine.workload_trace(fleet, *rows, want_candidates=True)
    S, A = fleet.n_servers, fleet.n_acc
    cur = fleet
    for t in range(L):
        cand_s, win_s = engine.solve(at_level(cur, rows[0][t], rows[1][t], rows[2][t]))
        for k in ALLOC_FIELDS:
            assert _same(getattr(cand_g, k)[t * S * A:(t + 1) * S * A], getattr(cand_s, k)), (t, k)
            assert _same(getattr(win_g, k)[t * S:(t + 1) * S], getattr(win_s, k)), (t, k)
        cur = cur.apply_winners(win_s)
    one = [r[:1] for r in rows]
    for got, want in zip(engine.workload_trace(fleet, *one, want_candidates=True),
                         engine.workload_grid(fleet, *one, want_candidates=True)):
        for k in ALLOC_FIELDS:
            assert _same(getattr(got, k), getattr(want, k)), k


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3, 5])
def test_continuation(engine, k):
    """The trace over [0, L) is the trace over [0, k) followed by the trace over [k, L) from c_k."""
    fleet = low_penalty_fleet(30, 3, 103, True)
    fleet.srv_min_replicas[::2] = 0
    L = 7
    rows = workload_levels(fleet, L, 37)
    rows[0][2, ::3] = 0.0
    S = fleet.n_servers
    cand, win = engine.workload_trace(fleet, *rows, want_candidates=True)
    cand_a, win_a = engine.workload_trace(fleet, *[r[:k] for r in rows], want_candidates=True)
    cur = fleet
    for t in range(k):
        cur = cur.apply_winners(_records(win_a)[t * S:(t + 1) * S])
    cand_b, win_b = engine.workload_trace(cur, *[r[k:] for r in rows], want_candidates=True)
    for n in ALLOC_FIELDS:
        assert _same(getattr(cand, n), np.concatenate([getattr(cand_a, n), getattr(cand_b, n)])), n
        assert _same(getattr(win, n), np.concatenate([getattr(win_a, n), getattr(win_b, n)])), n
    assert _moves(_records(win), S) >= 1


@pytest.mark.gpu
def test_pair_excluded_at_every_tick_does_not_fail(engine):
    """Server 0 is pinned to accelerator 0; at tick 1 its out_tokens 1 put accelerator 1's N at 2^21, outside the
    queue-size rule.  keepAccelerator excludes that pair at every tick, so the per-tick wva_solve loop never sizes
    it, and neither does the trace.  Without keep the same rows are refused."""
    fleet = synth_fleet(4, 2, seed=83, zero_load_frac=0.0)
    fleet.srv_max_batch[0] = 0
    fleet.perf_max_batch[:] = 512
    fleet.perf_at_tokens[:, 0] = 1
    fleet.perf_at_tokens[:, 1] = 1 << 12
    fleet.srv_keep_acc[0] = 1
    fleet.srv_cur_acc[0] = 0
    fleet.srv_min_replicas[0] = 1
    assert pinned(fleet)[0]
    L = 3
    rpm = np.stack([fleet.srv_arrival_rpm] * L).astype(np.float32)
    in_tok = np.stack([fleet.srv_in_tokens] * L).astype(np.int32)
    out_tok = np.stack([fleet.srv_out_tokens] * L).astype(np.int32)
    out_tok[:, 0] = 1 << 16
    out_tok[1, 0] = 1
    cand_g, win_g = engine.workload_trace(fleet, rpm, in_tok, out_tok, want_candidates=True)
    S, A = fleet.n_servers, fleet.n_acc
    cur = fleet
    for t in range(L):
        cand_s, win_s = engine.solve(at_level(cur, rpm[t], in_tok[t], out_tok[t]))
        for k in ALLOC_FIELDS:
            assert _same(getattr(cand_g, k)[t * S * A:(t + 1) * S * A], getattr(cand_s, k)), (t, k)
            assert _same(getattr(win_g, k)[t * S:(t + 1) * S], getattr(win_s, k)), (t, k)
        cur = cur.apply_winners(win_s)
    assert win_g.feasible[S] == 1 and win_g.acc[S] == 0
    free = fleet.take_servers(np.arange(S))
    free.srv_keep_acc[0] = 0
    assert _code(lambda: engine.workload_trace(free, rpm, in_tok, out_tok))[0] == WVA_ERR_UNSUPPORTED


@pytest.mark.gpu
def test_argument_errors(engine):
    from workload_variant_autoscaler_b200 import _abi
    fleet = mixed_fleet(6, 2, 79, False)
    L, h = engine._L, engine._h
    win = Allocs(fleet.n_servers)
    fc, wc = fleet.as_c(), win.as_c()
    one = np.ones(fleet.n_servers, np.float32)
    tok = np.ones(fleet.n_servers, np.int32)
    p, t = _abi.ptr(one), _abi.ptr(tok)
    assert L.wva_workload_trace(h, C.byref(fc), -1, p, t, t, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    for k in range(3):
        rows = [p, t, t]
        rows[k] = None
        assert L.wva_workload_trace(h, C.byref(fc), 1, *rows, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_workload_trace(h, C.byref(fc), 1, p, t, t, None, None) == WVA_ERR_BAD_ARG
    assert L.wva_workload_trace(h, None, 1, p, t, t, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    # S * A * L = 2^20 * 2^6 * 32 = 2^31: refused before the fleet is read
    big = fleet.as_c()
    big.n_servers, big.n_acc, big.n_types = 1 << 20, 1 << 6, 0
    assert L.wva_workload_trace(h, C.byref(big), 32, p, t, t, None, C.byref(wc)) == WVA_ERR_UNSUPPORTED
    with pytest.raises(ValueError):
        engine.workload_trace(fleet, one)
    with pytest.raises(ValueError):
        engine.workload_trace(fleet, one[None, :], in_tokens=np.ones((2, fleet.n_servers), np.int32))
    with pytest.raises(ValueError):
        engine.workload_trace(fleet, one[None, :], out=Allocs(2 * fleet.n_servers))
    # an empty list is valid, and the handle then solves as usual
    cand, win0 = engine.workload_trace(fleet, np.zeros((0, fleet.n_servers), np.float32), want_candidates=True)
    assert cand.n == 0 and win0.n == 0
    engine.solve(fleet)


@pytest.mark.gpu
def test_one_handle_with_the_other_paths(engine):
    fleet = token_fleet(30, 3, 73, True)
    rows = workload_levels(fleet, 4, 23)
    fresh = Engine(0)
    try:
        def same(got, want, what):
            for k in ALLOC_FIELDS:
                assert np.array_equal(getattr(got, k).view(np.uint8), getattr(want, k).view(np.uint8)), f"{what}: {k}"

        def check(call, what):
            for x, y in zip(call(engine), call(fresh)):
                if x is not None:
                    same(x, y, what)

        trace = lambda e: e.workload_trace(fleet, *rows, want_candidates=True)  # noqa: E731
        grid = lambda e: e.workload_grid(fleet, *rows, want_candidates=True)  # noqa: E731
        # wva_solve -> wva_workload_trace -> wva_resolve: the resident fleet and the solve's cache are untouched
        cand_s, win_s = engine.solve(fleet)
        trace(engine)
        cand_r, win_r = engine.resolve(want_candidates=True)
        same(cand_r, cand_s, "resolve after the trace: candidates")
        same(win_r, win_s, "resolve after the trace: winners")
        check(trace, "trace")
        check(grid, "workload grid after the trace")
        check(trace, "trace after the workload grid")
        check(lambda e: e.solve(fleet), "solve at the end")
        # no single solution to summarise after a trace
        engine.solve(fleet)
        engine.summarize(fleet.n_types)
        trace(engine)
        with pytest.raises(WvaError) as e:
            engine.summarize(fleet.n_types)
        assert e.value.code == WVA_ERR_STATE
    finally:
        fresh.close()


N_ADV = 30


@pytest.mark.gpu
def test_workload_trace_adversarial(engine, oracle_mod, monkeypatch):
    """Fleets from test_gpu_parity's _adversarial_fleet, keep on half the servers, with random (rate, in, out) rows
    from the workload grid's edge sets, half of them on the rounds.  Where the per-tick wva_solve loop refuses a
    tick, the trace must refuse too; the trace may refuse beyond that only through a keep server that is not
    pinned."""
    rng = np.random.default_rng(0x7ACE)
    feasible = refused = extra = 0
    for case in range(N_ADV):
        fleet = _adversarial_fleet(rng, 60000 + case)
        S, A, L = fleet.n_servers, fleet.n_acc, int(rng.integers(1, 6))
        fleet.srv_keep_acc[:] = rng.random(S) < 0.5
        fleet.srv_cur_acc[:] = rng.integers(-2, A, S)
        fleet.accel_penalty_factor = float(rng.choice([0.0, 0.1]))
        if case % 2:
            monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        else:
            monkeypatch.delenv("WVA_SIZE_SMALL_MAX", raising=False)
        rpm = rng.choice(np.array([0.0, 1e-3, 3.0, 600.0, 1e6, -1.0, np.inf], np.float32), (L, S),
                         p=[.15, .1, .25, .25, .1, .05, .1])
        in_tok = rng.choice(np.array([0, 1, 7, 512, 100000, -1], np.int32), (L, S), p=[.15, .15, .2, .25, .2, .05])
        out_tok = rng.choice(np.array([0, 1, 2, 9, 300, 50000, -1], np.int32), (L, S),
                             p=[.1, .1, .15, .15, .25, .2, .05])
        rpm[0], in_tok[0], out_tok[0] = fleet.srv_arrival_rpm, fleet.srv_in_tokens, fleet.srv_out_tokens
        # the per-tick wva_solve loop
        code, cur = 0, fleet
        for t in range(L):
            code, res = _code(lambda: engine.solve(at_level(cur, rpm[t], in_tok[t], out_tok[t])))
            if code:
                break
            cur = cur.apply_winners(res[1])
        got, _ = _code(lambda: engine.workload_trace(fleet, rpm, in_tok, out_tok))
        if code:
            assert got == code, (case, code, got)
            refused += 1
            continue
        if got:
            assert got == WVA_ERR_UNSUPPORTED and ((fleet.srv_keep_acc != 0) & ~pinned(fleet)).any(), (case, got)
            extra += 1
            continue
        _, win_o = _check(engine, oracle_mod, fleet, (rpm, in_tok, out_tok), f"adversarial case {case}")
        feasible += int(win_o["feasible"].sum())
    assert feasible > 30 and refused + extra < N_ADV // 2
