"""wva_size_grid: the reference's CreateAllocation at every listed batch size, and the min-value
(accelerator, batch size) per server.

The expected result is composed from the CPU oracle, literally: candidate (s, a, bi) is the oracle's
Server.Calculate (CreateAllocation + TransitionPenalty) on a copy of the fleet with every srv_max_batch set to
batches[bi], and the winner is a loop over (a, bi) under the stated order.  The CPU tests pin that composition
against the oracle's own SolveUnlimited and on hand-built ties; the GPU tests compare the CUDA path with it bit
for bit."""
import ctypes as C

import numpy as np
import pytest

from tests.levels import mixed_fleet, ref_candidates, ref_size_grid, ref_winners, with_batch
from tests.util import F32_MAX, WVA_ERR_BAD_ARG, WVA_ERR_UNSUPPORTED, assert_allocs_equal, same_bytes
from workload_variant_autoscaler_b200 import Engine, synth_fleet

# ---- CPU: the composition itself --------------------------------------------------------------

@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_one_batch_size_is_the_oracle_solve(oracle_mod, seed, keep):
    fleet = mixed_fleet(12, 3, seed, keep)
    for b in (4, 32):
        cand, win = ref_size_grid(oracle_mod, fleet, [b])
        cand_o, win_o = oracle_mod.solve(with_batch(fleet, b))
        assert same_bytes(cand, cand_o.reshape(-1)), f"candidates, b = {b}"
        assert same_bytes(win, win_o), f"winners, b = {b}"
        assert win["feasible"].sum() >= 4


def _recs(oracle_mod, rows):
    """[S, A, B] candidates from {(s, a, bi): value}; every listed entry is feasible with acc = a."""
    S = 1 + max(k[0] for k in rows)
    A = 1 + max(k[1] for k in rows)
    B = 1 + max(k[2] for k in rows)
    cand = np.zeros((S, A, B), oracle_mod.ALLOC_DTYPE)
    cand["acc"] = -1
    for (s, a, bi), v in rows.items():
        cand[s, a, bi]["feasible"] = 1
        cand[s, a, bi]["acc"] = a
        cand[s, a, bi]["replicas"] = 1 + bi
        cand[s, a, bi]["value"] = v
    return cand


def test_winner_order_on_hand_built_ties(oracle_mod):
    batches = [16, 4, 8]
    nan, inf = np.float32(np.nan), np.float32(np.inf)
    cand = _recs(oracle_mod, {
        (0, 0, 0): 5.0, (0, 1, 0): 5.0,                     # equal value, same batch size: accelerator 0
        (1, 0, 0): 3.0, (1, 1, 1): 3.0, (1, 0, 2): 3.0,     # equal value: batch 4 (bi 1) before 8 and 16
        (2, 0, 1): nan, (2, 1, 2): 7.0,                     # a NaN value never wins
        (3, 0, 0): nan, (3, 1, 1): F32_MAX, (3, 1, 2): inf,  # nothing below MaxFloat32: nil
        (4, 0, 2): -1.0, (4, 1, 1): -2.0,                   # negative penalties are ordinary values
    })
    cand[4, 1, 0]["value"] = -9.0                            # infeasible: ignored
    win = ref_winners(oracle_mod, cand, batches)
    got = [(int(w["feasible"]), int(w["acc"]), int(w["replicas"])) for w in win]
    assert got == [(1, 0, 1), (1, 1, 2), (1, 1, 3), (0, -1, 0), (1, 1, 2)]
    assert win[2]["value"] == np.float32(7.0)


def test_repeated_batch_sizes_give_identical_records(oracle_mod):
    fleet = mixed_fleet(10, 3, 5, False)
    cand = ref_candidates(oracle_mod, fleet, [8, 4, 8])
    assert same_bytes(cand[:, :, 0], cand[:, :, 2])
    win = ref_winners(oracle_mod, cand, [8, 4, 8])
    win1 = ref_winners(oracle_mod, cand[:, :, :2].copy(), [8, 4])
    assert same_bytes(win, win1)


# ---- GPU: bit for bit against the composition -------------------------------------------------

def _check(engine, oracle_mod, fleet, batches, what):
    cand_o, win_o = ref_size_grid(oracle_mod, fleet, batches)
    cand_g, win_g = engine.size_grid(fleet, batches, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"{what}: candidates")
    assert_allocs_equal(win_g, win_o, f"{what}: winners")
    return cand_o, win_o


SMALL_BATCHES = [1, 3, 8, 16, 33]       # 10 x 3 x 5 = 150 candidates: warp-per-candidate kernel
LARGE_BATCHES = [1, 2, 3, 5, 8, 13, 21, 34, 55, 89, 144]  # 60 x 4 x 11 = 2,640: rounds


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True])
@pytest.mark.parametrize("keep", [False, True])
def test_small_fleet(engine, oracle_mod, monkeypatch, keep, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet = mixed_fleet(10, 3, 31, keep)
    cand_o, win_o = _check(engine, oracle_mod, fleet, SMALL_BATCHES, f"small, keep = {keep}, rounds = {rounds}")
    assert cand_o["feasible"].sum() > 20
    assert len(set(win_o["batch"][win_o["feasible"] == 1].tolist())) >= 2


@pytest.fixture(scope="module")
def large_case(oracle_mod):
    fleet = mixed_fleet(60, 4, 37, False)
    fleet.srv_keep_acc[::2] = 1
    return fleet, ref_size_grid(oracle_mod, fleet, LARGE_BATCHES)


@pytest.mark.gpu
@pytest.mark.parametrize("depth", [None, "1", "2", "3", "4", "5"])
def test_large_fleet_every_tree_depth(engine, large_case, monkeypatch, depth):
    if depth is not None:
        monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet, (cand_o, win_o) = large_case
    cand_g, win_g = engine.size_grid(fleet, LARGE_BATCHES, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, f"large, D = {depth}: candidates")
    assert_allocs_equal(win_g, win_o, f"large, D = {depth}: winners")


@pytest.mark.gpu
def test_nan_and_huge_values_never_win(engine, oracle_mod):
    fleet = mixed_fleet(12, 3, 43, False)
    fleet.srv_cur_cost[::2] = np.nan     # penalty NaN except for the current (accelerator, replicas)
    fleet.srv_cur_cost[1::4] = -F32_MAX  # the current accelerator's penalty rounds to MaxFloat32
    fleet.acc_cost[2] = fleet.acc_cost[1]
    fleet.perf_alpha[:, 2] = fleet.perf_alpha[:, 1]  # accelerators 1 and 2 identical: ties on value
    for k in ("perf_beta", "perf_gamma", "perf_delta", "perf_acc_count"):
        getattr(fleet, k)[:, 2] = getattr(fleet, k)[:, 1]
    _check(engine, oracle_mod, fleet, [2, 8, 8, 32], "NaN / huge values and ties")


@pytest.mark.gpu
@pytest.mark.parametrize("b", [1, 16, 100])
def test_one_batch_size_equals_solve(engine, b):
    fleet = mixed_fleet(24, 4, 47, True)
    cand_s, win_s = engine.solve(with_batch(fleet, b))
    cand_g, win_g = engine.size_grid(fleet, [b], want_candidates=True)
    for k, _ in cand_s.columns().items():
        assert np.array_equal(getattr(cand_g, k).view(np.uint8), getattr(cand_s, k).view(np.uint8)), k
        assert np.array_equal(getattr(win_g, k).view(np.uint8), getattr(win_s, k).view(np.uint8)), k


@pytest.mark.gpu
def test_stored_vector_fallback(engine, oracle_mod):
    # the overflow fleet of test_overflow_rescale_falls_back_to_stored_vector: near saturation at N = 1024 the
    # chain overflows float64, and the candidates re-run on the stored vector with the reference's rescale loops
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
    fleet.srv_arrival_rpm[:] = [60.0 * 2100, 60.0 * 1900]
    cand_o, _ = _check(engine, oracle_mod, fleet, [512, 1024], "stored-vector fallback")
    assert cand_o["feasible"].sum() >= 2


@pytest.mark.gpu
def test_cache_interplay_on_one_handle(engine):
    fleet = mixed_fleet(30, 3, 53, True)
    fresh = Engine(0)
    try:
        def same(got, want, what):
            for k in ("feasible", "acc", "replicas", "batch", "cost", "value", "itl", "ttft", "rho", "max_rate"):
                assert np.array_equal(getattr(got, k).view(np.uint8), getattr(want, k).view(np.uint8)), f"{what}: {k}"

        def check_solve(f, what):
            c, w = engine.solve(f)
            c0, w0 = fresh.solve(f)
            same(c, c0, what)
            same(w, w0, what)

        def check_grid(f, batches, what):
            c, w = engine.size_grid(f, batches, want_candidates=True)
            c0, w0 = fresh.size_grid(f, batches, want_candidates=True)
            same(c, c0, what)
            same(w, w0, what)

        check_solve(fleet, "solve")
        check_grid(fleet, [4, 16, 64], "size grid")
        check_solve(fleet, "solve after the size grid")
        check_grid(fleet, [2, 16, 128, 5], "size grid, another list")
        fleet.srv_out_tokens[:] = np.maximum(1, fleet.srv_out_tokens // 3)
        engine.update_load(out_tokens=fleet.srv_out_tokens)
        check_grid(fleet, [2, 16, 128, 5], "size grid after a token change")
        c, w = engine.size_grid(fleet, [2, 16, 128, 5])
        assert c is None
        check_solve(fleet, "solve at the end")
    finally:
        fresh.close()


@pytest.mark.gpu
def test_summarize_after_size_grid(engine, oracle_mod):
    fleet = mixed_fleet(40, 4, 59, False)
    fleet.acc_type[:] = [0, 1, 0, 2]
    fleet.type_capacity = np.array([7, 0, 100], np.int32)
    _, win_o = ref_size_grid(oracle_mod, fleet, [4, 32, 128])
    engine.size_grid(fleet, [4, 32, 128])
    got = engine.summarize(fleet.n_types)
    t = oracle_mod.allocate_by_type(fleet, win_o)
    d = oracle_mod.allocation_diffs(fleet, win_o)
    assert np.array_equal(got["by_type"]["present"], t["present"].astype(np.uint8))
    assert np.array_equal(got["by_type"]["count"], t["count"])
    assert np.array_equal(got["by_type"]["limit"], t["limit"])
    assert np.array_equal(got["by_type"]["cost"].view(np.uint32), np.ascontiguousarray(t["cost"]).view(np.uint32))
    for k in ("old_acc", "new_acc", "old_replicas", "new_replicas"):
        assert np.array_equal(got["diff"][k], d[k]), k
    assert np.array_equal(got["diff"]["cost"].view(np.uint32), np.ascontiguousarray(d["cost_diff"]).view(np.uint32))
    assert t["present"].sum() >= 2


@pytest.mark.gpu
def test_argument_errors_and_empty_list(engine):
    from workload_variant_autoscaler_b200 import Allocs, WvaError, _abi
    fleet = mixed_fleet(6, 2, 61, False)
    for bad in ([0], [4, 1 << 20 | 1], [-3]):
        with pytest.raises(WvaError) as e:
            engine.size_grid(fleet, bad)
        assert e.value.code == WVA_ERR_BAD_ARG, bad
    L, h = engine._L, engine._h
    win = Allocs(fleet.n_servers)
    fc, wc = fleet.as_c(), win.as_c()
    one = np.array([4], np.int32)
    assert L.wva_size_grid(h, C.byref(fc), -1, _abi.ptr(one), None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_size_grid(h, C.byref(fc), 1, None, None, C.byref(wc)) == WVA_ERR_BAD_ARG
    assert L.wva_size_grid(h, C.byref(fc), 1, _abi.ptr(one), None, None) == WVA_ERR_BAD_ARG
    # S * A * B = 2^20 * 2^6 * 32 = 2^31: refused before the fleet is read
    big = fleet.as_c()
    big.n_servers, big.n_acc, big.n_types = 1 << 20, 1 << 6, 0
    thirty_two = np.full(32, 4, np.int32)
    assert L.wva_size_grid(h, C.byref(big), 32, _abi.ptr(thirty_two), None, C.byref(wc)) == WVA_ERR_UNSUPPORTED
    # an empty list is valid: every winner is nil
    cand, win = engine.size_grid(fleet, [], want_candidates=True)
    assert cand.n == 0
    assert win.feasible.sum() == 0 and (win.acc == -1).all()
    assert engine.summarize(fleet.n_types)["diff"]["new_acc"].tolist() == [_abi.ACC_ABSENT] * fleet.n_servers
