"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle, bit for bit.

Integer decisions (feasible / accelerator / replicas / batch) must be identical and every
float32 output must have identical bits (north_star asks for <= 1e-9 relative; a single
float32 ulp is 6e-8, so the bar actually enforced is bit-exactness).
"""
import numpy as np
import pytest

from tests.util import assert_allocs_equal, assert_f32_bits_equal
from workload_variant_autoscaler_b200 import Grid, synth_fleet

pytestmark = pytest.mark.gpu


def _grid_check(engine, oracle_mod, fleet, grid):
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    cells_g, win_g = engine.grid_solve(fleet, grid, want_cells=True)
    assert np.array_equal(cells_g["flags"], cells_o["flags"]), "cell flags differ"
    for k in ("ttft", "itl", "rho", "throughput"):
        assert_f32_bits_equal(cells_g[k], cells_o[k], f"cells.{k}")
    assert_allocs_equal(win_g, win_o, "grid winners")
    return cells_o, win_o


def test_grid_small_bit_exact(engine, oracle_mod):
    fleet = synth_fleet(8, 3, seed=1)
    grid = Grid([1, 2, 3, 4, 7, 8, 16, 33], [1, 2, 3, 5, 8, 13, 21, 34, 55, 64])
    cells, win = _grid_check(engine, oracle_mod, fleet, grid)
    assert (cells["flags"] & 1).sum() > 100, "the case must exercise analysable cells"
    assert win["feasible"].sum() >= 4


def test_grid_keep_accelerator_and_zero_load(engine, oracle_mod):
    fleet = synth_fleet(12, 4, seed=7, keep_accelerator=True, zero_load_frac=0.3)
    fleet.srv_min_replicas[::3] = 0
    grid = Grid([1, 4, 16, 64], np.arange(1, 41))
    _grid_check(engine, oracle_mod, fleet, grid)


def test_grid_ragged_and_empty(engine, oracle_mod):
    fleet = synth_fleet(3, 2, seed=3)
    _grid_check(engine, oracle_mod, fleet, Grid([5], [3]))                      # one cell per pair
    _grid_check(engine, oracle_mod, fleet, Grid([2, 9], np.arange(1, 34)))      # R = 33: ragged chunks
    cells, win = engine.grid_solve(fleet, Grid([], []), want_cells=True)       # empty grid
    assert win.feasible.sum() == (fleet.srv_arrival_rpm == 0).sum()


def test_grid_missing_profiles_and_targets(engine, oracle_mod):
    fleet = synth_fleet(10, 4, seed=11)
    fleet.perf_present[0, 1] = 0
    fleet.perf_present[3, :] = 0
    fleet.srv_has_target[5] = 0
    fleet.srv_model[6] = -1
    fleet.srv_cur_acc[7] = -2  # current accelerator name not in the table
    fleet.srv_keep_acc[7] = 1
    fleet.srv_arrival_rpm[8] = -1.0
    _grid_check(engine, oracle_mod, fleet, Grid([2, 8, 32], [1, 2, 4, 8, 16, 32]))


def test_size_candidates_and_unlimited_winners(engine, oracle_mod):
    fleet = synth_fleet(48, 4, seed=5, max_batch_choices=(1, 2, 4, 8, 16, 32, 64))
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, "size candidates")
    assert_allocs_equal(win_g, win_o, "unlimited winners")
    assert cand_o["feasible"].sum() > 40
    assert (cand_o["replicas"] > 1).sum() > 5


def test_size_keep_accelerator_production_mode(engine, oracle_mod):
    # production: unlimited + KeepAccelerator (internal/utils/utils.go:170-173,290)
    fleet = synth_fleet(64, 4, seed=9, keep_accelerator=True, zero_load_frac=0.2,
                        max_batch_choices=(4, 8, 16, 32, 128, 256))
    fleet.srv_min_replicas[::4] = 0
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, "size candidates (keepAccelerator)")
    assert_allocs_equal(win_g, win_o, "winners (keepAccelerator)")


def test_size_at_tokens_batch_rule(engine, oracle_mod):
    # N = max(MaxBatchSize*AtTokens/outTokens, 1) when the server has no override (allocation.go:82-86)
    fleet = synth_fleet(24, 3, seed=13, server_batch=False, max_batch_choices=(4, 16, 64))
    fleet.perf_at_tokens[:] = 128
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, "size candidates (AtTokens rule)")
    assert_allocs_equal(win_g, win_o, "winners (AtTokens rule)")


def test_analyze_only_matches_calculate(engine, oracle_mod):
    fleet = synth_fleet(16, 3, seed=21, max_batch_choices=(2, 8, 32))
    cand_o = oracle_mod.calculate(fleet)
    cand_g = engine.analyze(fleet)
    assert_allocs_equal(cand_g, cand_o, "Server.Calculate")


def test_sweep_bit_exact(engine, oracle_mod):
    fleet = synth_fleet(10, 3, seed=17, max_batch_choices=(4, 16, 64, 128))
    n_rates = 40
    o = oracle_mod.sweep(fleet, n_rates)
    g = engine.sweep(fleet, n_rates)
    assert np.array_equal(g["valid"], o["valid"])
    assert o["valid"].sum() > 0.9 * o["valid"].size
    for k in ("rate", "ttft", "itl", "throughput", "rho"):
        assert_f32_bits_equal(g[k], o[k], f"sweep.{k}")


def test_streaming_update_matches_fresh_solve(engine, oracle_mod):
    fleet = synth_fleet(40, 4, seed=23, keep_accelerator=True, max_batch_choices=(4, 8, 16, 32))
    engine.upload(fleet)
    rng = np.random.default_rng(0)
    for _ in range(3):
        fleet.srv_arrival_rpm[:] = (fleet.srv_arrival_rpm * np.exp(rng.normal(0, 0.1, fleet.n_servers))).astype(np.float32)
        engine.update_load(arrival_rpm=fleet.srv_arrival_rpm)
        _, win_g = engine.resolve()
        _, win_o = oracle_mod.solve(fleet)
        assert_allocs_equal(win_g, win_o, "streaming winners")
    # token statistics change: service-rate tables must be rebuilt
    fleet.srv_out_tokens[:] = np.maximum(1, fleet.srv_out_tokens // 2)
    engine.update_load(out_tokens=fleet.srv_out_tokens)
    _, win_g = engine.resolve()
    _, win_o = oracle_mod.solve(fleet)
    assert_allocs_equal(win_g, win_o, "streaming winners after token change")


def test_overflow_rescale_falls_back_to_stored_vector(engine, oracle_mod):
    # N = 1024 near saturation: prod(lambda/servRate[n]) overflows float64, so the reference's
    # rescale branches (mm1modelstatedependent.go:84-89,96-104) run; the streaming solve must
    # bail out and the stored-vector fallback must reproduce the reference bits.
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
    grid = Grid([1024], [1, 2, 4])
    cells, win = _grid_check(engine, oracle_mod, fleet, grid)
    assert (cells["flags"] & 1).sum() >= 2
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, "size candidates (overflow)")


def test_full_size_properties_config2_slice(engine):
    """BASELINE config 2 at full batch/replica resolution on a slice of servers: properties
    that hold for any correct evaluation (no oracle at this size)."""
    from workload_variant_autoscaler_b200 import config2_grid
    fleet = synth_fleet(10, 4, seed=42)
    grid = config2_grid()
    cells, win = engine.grid_solve(fleet, grid, want_cells=True)
    S, A, B, R = fleet.n_servers, fleet.n_acc, 256, 64
    flags = cells["flags"].reshape(S, A, B, R)
    ok = (flags & 1) == 1
    feas = (flags & 2) == 2
    assert not (feas & ~ok).any()
    rho = cells["rho"].reshape(S, A, B, R)
    assert ((rho >= 0) & (rho <= 1))[ok].all()
    # more replicas => lower per-replica rate => analysable stays analysable
    assert (ok[..., 1:] | ~ok[..., :-1]).all()
    # utilisation is non-increasing in the replica count
    r0, r1 = rho[..., :-1], rho[..., 1:]
    both = ok[..., :-1] & ok[..., 1:]
    assert (r1[both] <= r0[both] + 1e-6).all()
    # winner is feasible wherever any cell is
    any_feas = feas.reshape(S, -1).any(axis=1) | (fleet.srv_arrival_rpm == 0)
    assert np.array_equal(win.feasible.astype(bool), any_feas)
    # idempotence
    _, win2 = engine.grid_solve(fleet, grid)
    for k, v in win.columns().items():
        assert np.array_equal(v.view(np.uint8), win2.columns()[k].view(np.uint8))


def test_exact_division_primitive_selfcheck(engine):
    """div_recip (4 dependent FP64 ops around a double-word reciprocal) must equal div.rn.f64 bit for bit
    on 2 x 10^9 pseudo-random operand pairs from the solver's exponent windows, including float32-valued
    divisors and divisors next to powers of two (DESIGN.md 3.1)."""
    import ctypes as C
    L = engine._L
    L.wva_dbg_div_selfcheck.restype = C.c_longlong
    L.wva_dbg_div_selfcheck.argtypes = [C.c_void_p, C.c_ulonglong, C.c_int, C.c_int]
    bad = L.wva_dbg_div_selfcheck(engine._h, 0x5EED, 148 * 16, 1800)   # 148*16*256*1800*2 = 2.2e9 divisions
    assert bad == 0


def test_config2_full_resolution_sample_bit_exact(engine, oracle_mod):
    """BASELINE configs[1] at full batch x replica resolution (256 x 64): five of the 100 models are
    checked cell-by-cell and winner-by-winner against the oracle (1.3 M cells)."""
    from workload_variant_autoscaler_b200 import config2_grid
    full = synth_fleet(100, 4, seed=42)
    grid = config2_grid()
    idx = np.array([0, 23, 47, 71, 99])
    sub = full.take_servers(idx)
    cells_o, win_o = oracle_mod.grid_solve(sub, grid, want_cells=True)
    # the sampled servers solved alone ...
    cells_g, win_g = engine.grid_solve(sub, grid, want_cells=True)
    assert np.array_equal(cells_g["flags"], cells_o["flags"])
    for k in ("ttft", "itl", "rho", "throughput"):
        assert_f32_bits_equal(cells_g[k], cells_o[k], f"cells.{k}")
    assert_allocs_equal(win_g, win_o, "winners of the sampled models")
    # ... and inside the full 100-model solve (scheduling differs, results must not)
    _, win_full = engine.grid_solve(full, grid)
    for name in ("feasible", "acc", "replicas", "batch"):
        assert np.array_equal(np.asarray(getattr(win_full, name))[idx].astype(np.int64), win_o[name].astype(np.int64)), name
    for name in ("cost", "value", "itl", "ttft", "rho", "max_rate"):
        assert_f32_bits_equal(getattr(win_full, name)[idx], win_o[name], f"full-solve winners {name}")


def test_queue_plans_do_not_change_results(engine, oracle_mod, monkeypatch):
    """grid_kernel's scheduling (how many long items share a sub-partition, which warps are parked; chosen per
    launch by grid_items_plan) must not leak into the results: the full config-2 solve of a fleet whose plan is
    L = 3 (seed 45) gives the same bits under every forced plan, and the sampled models match the oracle."""
    from workload_variant_autoscaler_b200 import config2_grid
    full = synth_fleet(100, 4, seed=45)
    grid = config2_grid()
    ref_cells, ref_win = engine.grid_solve(full, grid, want_cells=True)   # automatic plan
    for forced in ("0", "1", "2", "4"):
        monkeypatch.setenv("WVA_GRID_LONG", forced)
        cells, win = engine.grid_solve(full, grid, want_cells=True)
        for k in ("flags", "ttft", "itl", "rho", "throughput"):
            assert np.array_equal(cells[k].view(np.uint8), ref_cells[k].view(np.uint8)), f"plan {forced}: cells.{k}"
        for k, v in win.columns().items():
            assert np.array_equal(v.view(np.uint8), ref_win.columns()[k].view(np.uint8)), f"plan {forced}: winners.{k}"
    monkeypatch.delenv("WVA_GRID_LONG")
    idx = np.array([3, 58])
    sub = full.take_servers(idx)
    cells_o, win_o = oracle_mod.grid_solve(sub, grid, want_cells=True)
    n_per = full.n_acc * 256 * 64
    for j, srv in enumerate(idx):
        for k in ("ttft", "itl", "rho", "throughput"):
            assert_f32_bits_equal(ref_cells[k][srv * n_per:(srv + 1) * n_per], cells_o[k][j * n_per:(j + 1) * n_per], f"cells.{k}")
        assert np.array_equal(ref_cells["flags"][srv * n_per:(srv + 1) * n_per], cells_o["flags"][j * n_per:(j + 1) * n_per])
    for name in ("feasible", "acc", "replicas", "batch"):
        assert np.array_equal(np.asarray(getattr(ref_win, name))[idx].astype(np.int64), win_o[name].astype(np.int64)), name
    for name in ("cost", "value", "itl", "ttft", "rho", "max_rate"):
        assert_f32_bits_equal(getattr(ref_win, name)[idx], win_o[name], f"winners {name}")


def test_empty_and_degenerate_fleets(engine, oracle_mod):
    f0 = synth_fleet(4, 2, seed=1).take_servers(np.array([], dtype=np.int64))   # no servers
    cand, win = engine.solve(f0)
    assert cand.n == 0 and win.n == 0
    _, gw = engine.grid_solve(f0, Grid([1, 2], [1, 2]))
    assert gw.n == 0
    f1 = synth_fleet(3, 2, seed=2)
    f1.perf_present[:] = 0                                                        # nothing analysable
    cand, win = engine.solve(f1)
    assert cand.feasible.sum() == 0 and win.feasible.sum() == 0
    cells, gw = engine.grid_solve(f1, Grid([1, 4], [1, 2, 3]), want_cells=True)
    assert cells["flags"].sum() == 0 and gw.feasible.sum() == 0
    f2 = synth_fleet(5, 2, seed=3, max_batch_choices=(1,))                        # N = 1 everywhere (K = 11)
    _grid_check(engine, oracle_mod, f2, Grid([1], [1, 2, 50]))
    cand_o, win_o = oracle_mod.solve(f2)
    cand_g, win_g = engine.solve(f2)
    assert_allocs_equal(cand_g, cand_o, "N = 1 candidates")
    f3 = synth_fleet(5, 2, seed=4)
    f3.max_queue_to_batch_ratio = 0                                               # K = N: N = 1 is never valid
    _grid_check(engine, oracle_mod, f3, Grid([1, 2, 8], [1, 4]))
    f3.max_queue_to_batch_ratio = 3
    f3.accel_penalty_factor = 0.25
    _grid_check(engine, oracle_mod, f3, Grid([1, 2, 8], [1, 4]))
    cand_o, win_o = oracle_mod.solve(f3)
    cand_g, win_g = engine.solve(f3)
    assert_allocs_equal(win_g, win_o, "non-default tunables")


def test_abi_error_paths(engine):
    import ctypes as C
    from workload_variant_autoscaler_b200 import WvaError, _abi
    L = engine._L
    f = synth_fleet(3, 2, seed=5)
    win = _abi.Allocs(3).as_c()
    assert L.wva_solve(engine._h, None, None, C.byref(win)) == _abi.WVA_ERR_BAD_ARG          # NULL fleet
    fc = f.as_c()
    fc.srv_model = None
    assert L.wva_solve(engine._h, C.byref(fc), None, C.byref(win)) == _abi.WVA_ERR_BAD_ARG   # NULL column
    fc = f.as_c()
    fc.n_servers = -1
    assert L.wva_solve(engine._h, C.byref(fc), None, C.byref(win)) == _abi.WVA_ERR_BAD_ARG   # negative size
    with pytest.raises(WvaError):
        engine.grid_solve(f, Grid([0, 2], [1]))                                              # batch < 1
    with pytest.raises(WvaError):
        engine.grid_solve(f, Grid([2], [0]))                                                 # replicas < 1
    h2 = C.c_void_p()
    assert L.wva_create(C.byref(h2), 0) == 0
    assert L.wva_resolve(h2, None, C.byref(win)) == _abi.WVA_ERR_STATE                       # resolve before upload
    assert b"upload" in L.wva_last_error(h2)
    L.wva_destroy(h2)
    assert L.wva_create(C.byref(h2), 4096) == _abi.WVA_ERR_NO_DEVICE                        # no such device
    # infeasibility is data, not an error
    f.srv_has_target[:] = 0
    _, w = engine.solve(f)
    assert w.feasible.sum() == 0


def test_ties_resolve_to_lowest_accelerator(engine, oracle_mod):
    f = synth_fleet(6, 3, seed=6, max_batch_choices=(8,))
    for col in ("perf_alpha", "perf_beta", "perf_gamma", "perf_delta", "perf_acc_count"):
        getattr(f, col)[:, 1] = getattr(f, col)[:, 0]
        getattr(f, col)[:, 2] = getattr(f, col)[:, 0]
    f.acc_cost[:] = 40.0
    f.srv_cur_acc[:] = -1
    f.srv_cur_replicas[:] = 0
    f.srv_cur_cost[:] = 0
    cand_o, win_o = oracle_mod.solve(f)
    _, win_g = engine.solve(f)
    assert_allocs_equal(win_g, win_o, "tie winners")
    assert (np.asarray(win_g.acc)[np.asarray(win_g.feasible) == 1] == 0).all()


def test_reference_flow_from_kubernetes_objects(engine, oracle_mod):
    """SURVEY.md 8f ranks 1 + 3 around the CUDA path: ConfigMaps + VariantAutoscalings (the reference's
    optimizer_test.go fixture, with load on two variants) -> adapters -> fleet -> wva_solve -> AllocationSolution ->
    optimized allocs; identical to the same flow through the oracle."""
    from tests.test_adapters import ACC_CM, SC_CM, _va
    from workload_variant_autoscaler_b200 import Fleet, adapters
    sd = adapters.create_system_data(ACC_CM, SC_CM)
    vas = [_va(1), _va(2, arrival="600.0", replicas=2), _va(3, arrival="4200.5", replicas=1)]
    for va in vas[1:]:
        va["status"]["currentAlloc"]["load"].update(avgInputTokens="128", avgOutputTokens="256")
    for va in vas:
        _, cls = adapters.find_model_slo(SC_CM, va["spec"]["modelID"])
        for prof in va["spec"]["modelProfile"]["accelerators"]:
            adapters.add_model_accelerator_profile_to_system_data(sd, va["spec"]["modelID"], prof)
        adapters.add_server_info_to_system_data(sd, va, cls, environ={})
    fleet = Fleet.from_spec(sd["spec"])
    _, win_o = oracle_mod.solve(fleet)
    _, win_g = engine.solve(fleet)
    assert_allocs_equal(win_g, win_o, "winners")
    sol_g, sol_o = adapters.generate_solution(fleet, win_g), adapters.generate_solution(fleet, win_o)
    assert sol_g == sol_o and len(sol_g["spec"]) == 3
    opts = [adapters.create_optimized_alloc(v["metadata"]["name"], "default", sol_g) for v in vas]
    assert opts[0]["numReplicas"] == 1 and all(o["accelerator"] == "A100" for o in opts)
    assert opts[2]["numReplicas"] >= opts[1]["numReplicas"] >= 1


def test_grid_randomised_small_fleets(engine, oracle_mod):
    """Twenty seeded random fleets and grids (unsorted and repeated batch sizes / replica levels, keep-accelerator,
    zero-load and missing-profile servers, several queue ratios): cells and winners bit-exact against the oracle."""
    rng = np.random.default_rng(20260921)
    for case in range(20):
        S, A = int(rng.integers(1, 10)), int(rng.integers(1, 6))
        fleet = synth_fleet(S, A, seed=1000 + case, keep_accelerator=bool(case % 3 == 0), zero_load_frac=0.15,
                            tps_frac=0.3, server_batch=bool(case % 2))
        fleet.max_queue_to_batch_ratio = int(rng.choice([1, 4, 10, 17]))
        if case % 4 == 1 and S > 1:
            fleet.perf_present[int(rng.integers(0, fleet.n_models)), int(rng.integers(0, A))] = 0
        if case % 5 == 2:
            fleet.srv_min_replicas[:] = rng.integers(0, 4, S)
        nb, nr = int(rng.integers(1, 9)), int(rng.integers(1, 40))
        batch = rng.integers(1, 97, nb)          # unsorted, possibly repeated
        replicas = rng.integers(1, 70, nr)
        _grid_check(engine, oracle_mod, fleet, Grid(batch, replicas))


def test_size_randomised_fleets(engine, oracle_mod):
    """Twelve seeded random fleets through wva_solve (Size's two bisections + CreateAllocation + SolveUnlimited):
    candidates and winners bit-exact against the oracle, across batch-size ranges and queue ratios."""
    rng = np.random.default_rng(7)
    for case in range(12):
        S, A = int(rng.integers(2, 30)), int(rng.integers(1, 5))
        choices = [(1, 2, 3), (4, 8, 16, 32), (64, 128, 256), (5, 77, 300)][case % 4]
        fleet = synth_fleet(S, A, seed=500 + case, keep_accelerator=bool(case % 2), zero_load_frac=0.1, tps_frac=0.25,
                            server_batch=bool(case % 3), max_batch_choices=choices)
        fleet.max_queue_to_batch_ratio = int(rng.choice([2, 10, 25]))
        if case % 4 == 3:
            fleet.perf_at_tokens[:] = 64
        cand_o, win_o = oracle_mod.solve(fleet)
        cand_g, win_g = engine.solve(fleet)
        assert_allocs_equal(cand_g, cand_o, f"candidates, case {case}")
        assert_allocs_equal(win_g, win_o, f"winners, case {case}")


def test_grid_wide_replica_axis_and_long_tables(engine, oracle_mod):
    """R = 100 replica levels, ascending and then descending, and a 1700-entry table (longer than grid_rows'
    shared-memory staging; 18,700-state chains)."""
    fleet = synth_fleet(2, 2, seed=77)
    fleet.srv_arrival_rpm[:] = np.float32([900.0, 2500.0])
    _grid_check(engine, oracle_mod, fleet, Grid([3, 1700], np.arange(1, 101)))
    _grid_check(engine, oracle_mod, fleet, Grid([64, 7, 64], np.arange(100, 0, -1)))


@pytest.mark.parametrize("depth", ["1", "2", "3", "4", "5"])
def test_size_rounds_every_tree_depth(engine, oracle_mod, monkeypatch, depth):
    """The round-based size path resolves D reference iterations per round from a tree of 2^D - 1 speculative
    midpoints (wva_size.cuh); the results must not depend on D.  The small-fleet kernel is switched off here."""
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet = synth_fleet(40, 4, seed=101 + int(depth), max_batch_choices=(1, 2, 4, 8, 16, 32, 64, 128), zero_load_frac=0.1)
    fleet.srv_min_replicas[::6] = 0
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, f"size candidates (D = {depth})")
    assert_allocs_equal(win_g, win_o, f"winners (D = {depth})")


def test_size_small_fleet_kernel_on_a_larger_fleet(engine, oracle_mod, monkeypatch):
    """The warp-per-candidate kernel (small fleets) forced onto 1,200 candidates with batch sizes up to 256."""
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "100000")
    fleet = synth_fleet(300, 4, seed=107, max_batch_choices=(4, 8, 16, 32, 64, 128, 256))
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, "size candidates (warp per candidate)")
    assert_allocs_equal(win_g, win_o, "winners (warp per candidate)")


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


def test_adversarial_parameters_size_and_grid(engine, oracle_mod):
    """A hundred and fifty fleets from _adversarial_fleet through wva_solve and (every other one) wva_grid_solve: candidates,
    winners and cells bit-exact against the oracle.  A case the library reports as unsupported (the reference's
    rescale loop would not terminate) must be one the oracle cannot finish either — none occurs with finite inputs."""
    rng = np.random.default_rng(424242)
    feasible = 0
    for case in range(150):
        fleet = _adversarial_fleet(rng, case)
        cand_o, win_o = oracle_mod.solve(fleet)
        cand_g, win_g = engine.solve(fleet)
        assert_allocs_equal(cand_g, cand_o, f"candidates, adversarial case {case}")
        assert_allocs_equal(win_g, win_o, f"winners, adversarial case {case}")
        feasible += int(np.asarray(win_o["feasible"]).sum())
        if case % 2 == 0:
            _grid_check(engine, oracle_mod, fleet, Grid(rng.integers(1, 40, int(rng.integers(1, 6))),
                                                        rng.integers(1, 30, int(rng.integers(1, 12)))))
    assert feasible > 40, "the cases must include feasible servers"
