"""wva_workload_grid: the reference's Server.Calculate and SolveUnlimited winner at many caller-given rows of
(arrival rate, in_tokens, out_tokens).

The expected result is composed from the CPU oracle, literally: for each level l, a copy of the fleet with
srv_arrival_rpm / srv_in_tokens / srv_out_tokens = row l and unlimited = 1 goes through the oracle's
Server.Calculate (candidate block l) and Solver.Solve (winner block l).  The CPU tests pin that composition against
the oracle's own solve and show on the oracle that CreateAllocation splits into a Size per (in, out) token key and a
per-level tail that reads the level's rate and out_tokens; the GPU tests compare the CUDA path with the composition
bit for bit."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_load_grid import (_code, _f32_bits, _same, load_levels, mixed_fleet, overflow_fleet, pair_batch,
                                      rates_at_rate_star, tail)
from tests.test_gpu_parity import _adversarial_fleet
from tests.util import ALLOC_FIELDS, assert_allocs_equal
from workload_variant_autoscaler_b200 import Allocs, Engine, WvaError, greedy_solve, synth_fleet

F32 = np.float32
F32_MAX = F32(np.finfo(np.float32).max)
WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED = -1, -5, -6


def at_level(fleet, rpm, in_tok, out_tok, unlimited=True):
    """A copy of the fleet with the load of row (rpm, in_tok, out_tok)."""
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_arrival_rpm[:] = rpm
    f.srv_in_tokens[:] = in_tok
    f.srv_out_tokens[:] = out_tok
    f.unlimited = unlimited
    return f


def ref_workload_grid(oracle_mod, fleet, rpm, in_tok, out_tok):
    """(candidates [L*S*A], winners [L*S]): Server.Calculate and Solver.Solve (unlimited) per level."""
    cands, wins = [np.zeros(0, oracle_mod.ALLOC_DTYPE)], [np.zeros(0, oracle_mod.ALLOC_DTYPE)]
    for l in range(rpm.shape[0]):
        f = at_level(fleet, rpm[l], in_tok[l], out_tok[l])
        cand = oracle_mod.calculate(f)
        cands.append(cand.reshape(-1))
        wins.append(oracle_mod.solve(f, cand)[1])
    return np.concatenate(cands), np.concatenate(wins)


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


# ---- CPU: the composition and the split --------------------------------------------------------

@pytest.mark.parametrize("keep", [False, True])
def test_one_level_is_the_oracle_solve(oracle_mod, keep):
    fleet = token_fleet(12, 3, 5, keep)
    rows = [c[None, :] for c in (fleet.srv_arrival_rpm, fleet.srv_in_tokens, fleet.srv_out_tokens)]
    cand, win = ref_workload_grid(oracle_mod, fleet, *rows)
    cand_o, win_o = oracle_mod.solve(at_level(fleet, *[r[0] for r in rows]))
    assert _same(cand, cand_o.reshape(-1))
    assert _same(win, win_o)
    assert win["feasible"].sum() >= 4


def _size(oracle_mod, fleet, s, a):
    """One QueueAnalyzer.Size of pair (s, a) at the fleet's tokens: (analyzer, N, rateStar), or None when it fails."""
    m = fleet.srv_model[s]
    N = pair_batch(fleet, s, a)
    try:
        qa = oracle_mod.Analyzer(N, N * fleet.max_queue_to_batch_ratio, float(fleet.perf_alpha[m, a]),
                                 float(fleet.perf_beta[m, a]), float(fleet.perf_gamma[m, a]),
                                 float(fleet.perf_delta[m, a]), int(fleet.srv_in_tokens[s]),
                                 int(fleet.srv_out_tokens[s]))
        err, _, met, _ = qa.size(float(fleet.srv_slo_ttft[s]), float(fleet.srv_slo_itl[s]),
                                 float(fleet.srv_slo_tps[s]))
    except ValueError:
        return None
    return None if err else (qa, N, met["throughput"])


@pytest.mark.parametrize("seed", [3, 4])
def test_size_once_per_token_key_then_the_tail_is_create_allocation(oracle_mod, seed):
    """QueueAnalyzer.Size reads the tokens but not the rate: one Size per (pair, in, out) key, then the replica /
    cost / Analyze tail at each level's rate and out_tokens, reproduces the oracle's CreateAllocation at that level
    bit for bit."""
    fleet = token_fleet(12, 3, seed, False)
    assert fleet.srv_slo_tps.max() > 0 and (fleet.srv_min_replicas == 0).any() and (fleet.srv_max_batch == 0).any()
    rates = [0.0, -1.0, 1e-3, 600.0, 1e6, np.inf]
    checked = sized = 0
    S = fleet.n_servers
    for s in range(S):
        m = int(fleet.srv_model[s])
        if m < 0 or not fleet.srv_has_target[s]:
            continue
        own_in, own_out = int(fleet.srv_in_tokens[s]), int(fleet.srv_out_tokens[s])
        # out 20000 gives N = 1 where the perf data sets the batch size (MaxBatchSize * 512 < 20000)
        keys = {(0, own_out), (own_in, own_out), (100000, own_out), (own_in, 1), (own_in, 3 * own_out // 2),
                (own_in, 20000)}
        for a in range(fleet.n_acc):
            if not fleet.perf_present[m, a]:
                continue
            for in_tok, out_tok in sorted(keys):
                fk = at_level(fleet, fleet.srv_arrival_rpm, np.full(S, in_tok), np.full(S, out_tok))
                sz = _size(oracle_mod, fk, s, a)
                sized += 1
                for rpm in rates:
                    want = oracle_mod.create_allocation(at_level(fk, np.full(S, rpm, F32), in_tok, out_tok), s, a)
                    if rpm <= 0:
                        assert want["feasible"] == int(rpm == 0), (s, a, rpm)  # nil, or zeroLoadAllocation
                        continue
                    if sz is None:
                        assert want["feasible"] == 0, (s, a, rpm, in_tok, out_tok)
                        continue
                    qa, N, rate_star = sz
                    try:
                        got = tail(oracle_mod, qa, fk, s, a, N, rate_star, rpm)
                    except OverflowError:  # a replica count beyond int32, which the record cannot hold
                        continue
                    for k in ALLOC_FIELDS:
                        if k in ("cost", "value", "itl", "ttft", "rho", "max_rate"):
                            assert _f32_bits(got[k]) == _f32_bits(want[k]), (s, a, rpm, in_tok, out_tok, k)
                        else:
                            assert int(got[k]) == int(want[k]), (s, a, rpm, in_tok, out_tok, k)
                    checked += int(want["feasible"])
    assert sized >= 100 and checked >= 80


def test_same_tokens_give_the_same_rate_star_at_every_rate(oracle_mod):
    fleet = token_fleet(20, 3, 7, False)
    L = 8
    rpm, in_tok, out_tok = workload_levels(fleet, L, 9, special=False)
    cand, _ = ref_workload_grid(oracle_mod, fleet, rpm, in_tok, out_tok)
    cand = cand.reshape(L, fleet.n_servers, fleet.n_acc)
    load = ~(rpm < 0) & (rpm != 0)
    keys = multi = 0
    for s in range(fleet.n_servers):
        for a in range(fleet.n_acc):
            by_key = {}
            for l in range(L):
                if load[l, s] and cand[l, s, a]["feasible"]:
                    by_key.setdefault((in_tok[l, s], out_tok[l, s]), set()).add(_f32_bits(cand[l, s, a]["max_rate"]))
            assert all(len(v) == 1 for v in by_key.values()), (s, a, by_key)
            keys += len(by_key)
            multi += len(set().union(*by_key.values())) > 1 if by_key else 0
    assert keys >= 60 and multi >= 10  # the tokens do move rateStar


# ---- GPU: bit for bit against the composition -------------------------------------------------

def _check(engine, oracle_mod, fleet, rows, what):
    cand_o, win_o = ref_workload_grid(oracle_mod, fleet, *rows)
    cand_g, win_g = engine.workload_grid(fleet, *rows, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
    assert_allocs_equal(win_g, win_o, f"{what}: winners")
    return cand_o, win_o


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
    rows = workload_levels(fleet, 4, 11)
    return fleet, rows, ref_workload_grid(oracle_mod, fleet, *rows)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_rounds_every_tree_depth(engine, rounds_case, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, rows, (cand_o, win_o) = rounds_case
    cand_g, win_g = engine.workload_grid(fleet, *rows, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"rounds, D = {depth}: candidates")
    assert_allocs_equal(win_g, win_o, f"rounds, D = {depth}: winners")


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_cartesian_rate_by_out_tokens_grid(engine, oracle_mod, monkeypatch, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = token_fleet(16, 3, 41, False)
    rows = [[], [], []]
    for fr in (0.25, 1.0, 4.0):
        for fo in (0.5, 1.0, 1.5, 3.0):
            rows[0].append(fleet.srv_arrival_rpm * F32(fr))
            rows[1].append(fleet.srv_in_tokens)
            rows[2].append(np.maximum(fleet.srv_out_tokens * fo, 1).astype(np.int32))
    rows = [np.array(r) for r in rows]
    rows[0] = rows[0].astype(np.float32)
    _check(engine, oracle_mod, fleet, rows, f"rate x out_tokens, rounds = {rounds}")


@pytest.mark.gpu
def test_edge_tokens(engine, oracle_mod):
    """in -1 and out -1 give nil, out 0 gives zeroLoadAllocation at a positive rate, in 0 is a load, and TPS targets
    make totalRate differ per out_tokens key; keepAccelerator, min_replicas 0, unknown models and missing profiles
    come from mixed_fleet."""
    fleet = token_fleet(12, 3, 43, True)
    fleet.srv_slo_tps[::2] = F32(800.0)
    S = fleet.n_servers
    rpm = np.stack([np.maximum(fleet.srv_arrival_rpm, 10.0)] * 6).astype(np.float32)
    in_tok = np.stack([fleet.srv_in_tokens] * 6).astype(np.int32)
    out_tok = np.stack([fleet.srv_out_tokens] * 6).astype(np.int32)
    in_tok[0] = -1
    out_tok[1] = -1
    out_tok[2] = 0
    in_tok[3] = 0
    out_tok[4] = fleet.srv_out_tokens * 2
    out_tok[5] = np.maximum(fleet.srv_out_tokens // 3, 1)
    cand_o, win_o = _check(engine, oracle_mod, fleet, (rpm, in_tok, out_tok), "edge tokens")
    cand_o = cand_o.reshape(6, S, fleet.n_acc)
    assert not cand_o[0]["feasible"].any() and not cand_o[1]["feasible"].any()
    assert (cand_o[2]["rho"] == 0).all() and cand_o[2]["feasible"].sum() >= S
    assert cand_o[3]["feasible"].sum() >= S
    tps = fleet.srv_slo_tps > 0
    assert (cand_o[4]["replicas"][tps] != cand_o[5]["replicas"][tps]).any()


@pytest.mark.gpu
def test_stored_vector_fallback_both_phases(engine, oracle_mod):
    """N = 1024 from out_tokens 64 (MaxBatchSize 1024 x AtTokens 64 / 64) near saturation: the chains overflow
    float64, so phase 1's solves and the tail's re-run on the stored vector; other rows of the same servers use
    out_tokens 128 (N = 512) and 32 (N = 2048)."""
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
def test_nan_and_huge_values_and_ties(engine, oracle_mod):
    fleet = token_fleet(12, 3, 47, False)
    fleet.srv_cur_cost[::2] = np.nan     # penalty NaN except for the current (accelerator, replicas)
    fleet.srv_cur_cost[1::4] = -F32_MAX  # the current accelerator's penalty rounds to MaxFloat32
    fleet.acc_cost[2] = fleet.acc_cost[1]
    fleet.perf_alpha[:, 2] = fleet.perf_alpha[:, 1]  # accelerators 1 and 2 identical: ties on value
    for k in ("perf_beta", "perf_gamma", "perf_delta", "perf_acc_count"):
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]
    _check(engine, oracle_mod, fleet, workload_levels(fleet, 4, 17), "NaN / huge values and ties")


@pytest.mark.gpu
def test_each_block_is_the_greedy_input_of_its_level(engine, oracle_mod):
    fleet = token_fleet(30, 4, 53, True)
    fleet.type_capacity[:] = [6, 9, 4, 12]
    rows = workload_levels(fleet, 4, 13)
    cand_g, _ = engine.workload_grid(fleet, *rows, want_candidates=True)
    S, A = fleet.n_servers, fleet.n_acc
    for l in range(4):
        fl = at_level(fleet, rows[0][l], rows[1][l], rows[2][l], unlimited=False)
        block = Allocs(S * A)
        for k in ALLOC_FIELDS:
            getattr(block, k)[:] = getattr(cand_g, k)[l * S * A:(l + 1) * S * A]
        cand_lim, win_lim = greedy_solve(fl, block)
        cand_o, win_o = oracle_mod.solve(fl)
        assert_allocs_equal(win_lim, win_o, f"level {l}, limited: winners")
        assert_allocs_equal(cand_lim, cand_o, f"level {l}, limited: candidates")


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_own_tokens_are_the_load_grid(engine, monkeypatch, rounds):
    """Rows that repeat the fleet's tokens: the same bytes as wva_load_grid, with the same launches."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = mixed_fleet(40, 4, 59, False)
    rpm = load_levels(fleet, 6, 61)
    n0 = engine.launch_count
    cand_l, win_l = engine.load_grid(fleet, rpm, want_candidates=True)
    n1 = engine.launch_count
    cand_w, win_w = engine.workload_grid(fleet, rpm, want_candidates=True)
    n2 = engine.launch_count
    for k in ALLOC_FIELDS:
        assert _same(getattr(cand_w, k), getattr(cand_l, k)), k
        assert _same(getattr(win_w, k), getattr(win_l, k)), k
    assert n2 - n1 == n1 - n0


@pytest.mark.gpu
def test_each_level_is_update_load_and_resolve(engine):
    fleet = token_fleet(30, 4, 67, True)
    rows = workload_levels(fleet, 5, 19)
    cand_g, win_g = engine.workload_grid(fleet, *rows, want_candidates=True)
    S, A = fleet.n_servers, fleet.n_acc
    engine.upload(fleet)
    for l in range(5):
        engine.update_load(rows[0][l], rows[1][l], rows[2][l])
        cand_r, win_r = engine.resolve(want_candidates=True)
        for k in ALLOC_FIELDS:
            assert _same(getattr(cand_g, k)[l * S * A:(l + 1) * S * A], getattr(cand_r, k)), (l, k)
            assert _same(getattr(win_g, k)[l * S:(l + 1) * S], getattr(win_r, k)), (l, k)


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
def test_sizing_runs_once_per_token_key(engine, monkeypatch, rounds):
    """The launch count depends on the keys, not on L: 1 and 64 rows over one key per server launch the same, and
    so do 2 and 64 rows (rates varying) over the same two keys per server."""
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = synth_fleet(40, 4, seed=71, zero_load_frac=0.0)
    S = fleet.n_servers
    rng = np.random.default_rng(7)
    outs = (fleet.srv_out_tokens, np.maximum(fleet.srv_out_tokens * 3 // 2, 1).astype(np.int32))

    def launches(pattern):
        L = len(pattern)
        rpm = (fleet.srv_arrival_rpm[None, :] * rng.lognormal(0.0, 0.5, (L, S))).astype(np.float32)
        out = np.array([outs[p] for p in pattern], np.int32)
        n0 = engine.launch_count
        engine.workload_grid(fleet, rpm, None, out)
        return engine.launch_count - n0
    assert launches([0]) == launches([0] * 64)
    assert launches([0, 1]) == launches([0, 1] * 32) == launches([1, 0, 0, 1] * 16)


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

        workload_grid = lambda e: e.workload_grid(fleet, *rows, want_candidates=True)  # noqa: E731
        load_grid = lambda e: e.load_grid(fleet, rows[0], want_candidates=True)  # noqa: E731
        # wva_solve -> wva_workload_grid -> wva_resolve: the resident fleet and the solve's cache are untouched
        cand_s, win_s = engine.solve(fleet)
        workload_grid(engine)
        cand_r, win_r = engine.resolve(want_candidates=True)
        same(cand_r, cand_s, "resolve after the workload grid: candidates")
        same(win_r, win_s, "resolve after the workload grid: winners")
        check(workload_grid, "workload grid")
        check(load_grid, "load grid after the workload grid")
        check(workload_grid, "workload grid after the load grid")
        check(lambda e: e.solve(fleet), "solve at the end")
        # no single solution to summarise after a workload grid
        engine.solve(fleet)
        engine.summarize(fleet.n_types)
        workload_grid(engine)
        with pytest.raises(WvaError) as e:
            engine.summarize(fleet.n_types)
        assert e.value.code == WVA_ERR_STATE
    finally:
        fresh.close()


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
    assert L.wva_workload_grid(h, C.byref(fc), -1, p, t, t, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    for k in range(3):
        rows = [p, t, t]
        rows[k] = None
        assert L.wva_workload_grid(h, C.byref(fc), 1, *rows, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_workload_grid(h, C.byref(fc), 1, p, t, t, None, None) == WVA_ERR_BAD_ARG
    # S * A * L = 2^20 * 2^6 * 32 = 2^31: refused before the fleet is read
    big = fleet.as_c()
    big.n_servers, big.n_acc, big.n_types = 1 << 20, 1 << 6, 0
    assert L.wva_workload_grid(h, C.byref(big), 32, p, t, t, None, C.byref(wc)) == WVA_ERR_UNSUPPORTED
    with pytest.raises(ValueError):
        engine.workload_grid(fleet, one)
    with pytest.raises(ValueError):
        engine.workload_grid(fleet, one[None, :], out_tokens=np.ones((2, fleet.n_servers), np.int32))
    # an empty list is valid
    cand, win0 = engine.workload_grid(fleet, np.zeros((0, fleet.n_servers), np.float32), want_candidates=True)
    assert cand.n == 0 and win0.n == 0


@pytest.mark.gpu
def test_small_out_tokens_fail_only_under_load(engine):
    """N = MaxBatchSize * AtTokens / out_tokens: out_tokens 1 puts server 0's N at 2^21, above the queue-size rule.
    At a loaded level the grid fails as wva_analyze of that level does; at rate 0 or with out_tokens 0 the token
    pair is never sized and the grid gives wva_analyze's records."""
    fleet = synth_fleet(4, 2, seed=83, zero_load_frac=0.0)
    fleet.srv_max_batch[0] = 0
    fleet.perf_max_batch[:] = 512
    fleet.perf_at_tokens[:] = 1 << 12
    S = fleet.n_servers
    rpm = np.stack([fleet.srv_arrival_rpm] * 3).astype(np.float32)
    in_tok = np.stack([fleet.srv_in_tokens] * 3).astype(np.int32)
    out_tok = np.stack([fleet.srv_out_tokens] * 3).astype(np.int32)
    out_tok[:, 0] = 1 << 16  # N = 32 elsewhere
    out_tok[1, 0] = 1
    rpm[1, 0] = 0.0           # out_tokens 1 at rate 0: zeroLoadAllocation, no sizing
    out_tok[2, 1] = 1         # server 1 takes its batch size from the fleet: out_tokens 1 is fine there
    cand_g, _ = engine.workload_grid(fleet, rpm, in_tok, out_tok, want_candidates=True)
    for l in range(3):
        cand_a = engine.analyze(at_level(fleet, rpm[l], in_tok[l], out_tok[l]))
        for k in ALLOC_FIELDS:
            assert _same(getattr(cand_g, k)[l * S * 2:(l + 1) * S * 2], getattr(cand_a, k)), (l, k)
    rpm[1, 0] = 5.0
    want, _ = _code(lambda: engine.analyze(at_level(fleet, rpm[1], in_tok[1], out_tok[1])))
    assert want == WVA_ERR_UNSUPPORTED
    assert _code(lambda: engine.workload_grid(fleet, rpm, in_tok, out_tok))[0] == want
    out_tok[1, 0] = 0  # out_tokens 0: zeroLoadAllocation at a positive rate
    assert _code(lambda: engine.workload_grid(fleet, rpm, in_tok, out_tok))[0] == 0


N_ADV = 36


@pytest.mark.gpu
def test_workload_grid_adversarial(engine, oracle_mod, monkeypatch):
    """Fleets from test_gpu_parity's _adversarial_fleet with random (rate, in, out) rows from the same edge sets,
    half of them on the rounds.  Where some level's wva_analyze refuses the level, the grid must refuse too."""
    rng = np.random.default_rng(0x70C)
    feasible = refused = 0
    for case in range(N_ADV):
        fleet = _adversarial_fleet(rng, 50000 + case)
        if case % 2:
            monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
        else:
            monkeypatch.delenv("WVA_SIZE_SMALL_MAX", raising=False)
        S, L = fleet.n_servers, int(rng.integers(1, 6))
        rpm = rng.choice(np.array([0.0, 1e-3, 3.0, 600.0, 1e6, -1.0, np.inf], np.float32), (L, S),
                         p=[.15, .1, .25, .25, .1, .05, .1])
        in_tok = rng.choice(np.array([0, 1, 7, 512, 100000, -1], np.int32), (L, S), p=[.15, .15, .2, .25, .2, .05])
        out_tok = rng.choice(np.array([0, 1, 2, 9, 300, 50000, -1], np.int32), (L, S),
                             p=[.1, .1, .15, .15, .25, .2, .05])
        rpm[0], in_tok[0], out_tok[0] = fleet.srv_arrival_rpm, fleet.srv_in_tokens, fleet.srv_out_tokens
        if L > 2:
            in_tok[2], out_tok[2] = in_tok[1], out_tok[1]  # a repeated token row at other rates
        codes = [_code(lambda: engine.analyze(at_level(fleet, rpm[l], in_tok[l], out_tok[l])))[0] for l in range(L)]
        if any(codes):
            got, _ = _code(lambda: engine.workload_grid(fleet, rpm, in_tok, out_tok))
            assert got == next(c for c in codes if c), (case, codes, got)
            refused += 1
            continue
        _, win_o = _check(engine, oracle_mod, fleet, (rpm, in_tok, out_tok), f"adversarial case {case}")
        feasible += int(win_o["feasible"].sum())
    assert feasible > 40 and refused < N_ADV // 2
