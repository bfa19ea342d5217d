"""Grid winners without a cell table, against the oracle bit for bit.

Without a cell table the cells that share their row's chain are evaluated only up to the row's first feasible one
(grid_shared), and rows that a smaller, non-shared batch size already decides are skipped.  The cell-table tests
never take that path, so this file runs the fleets of the small, randomised and adversarial grid tests through
grid_solve(want_cells=False), plus grids built to reach the walk's edge cases.
"""
import numpy as np
import pytest

from tests.test_gpu_parity import _adversarial_fleet
from tests.util import assert_allocs_equal
from workload_variant_autoscaler_b200 import Grid, synth_fleet

pytestmark = pytest.mark.gpu


def _winners_check(engine, oracle_mod, fleet, grid, what):
    _, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=False)
    _, win_g = engine.grid_solve(fleet, grid)
    assert_allocs_equal(win_g, win_o, what)
    return win_o


def test_winners_small_fleets(engine, oracle_mod):
    _winners_check(engine, oracle_mod, synth_fleet(8, 3, seed=1),
                   Grid([1, 2, 3, 4, 7, 8, 16, 33], [1, 2, 3, 5, 8, 13, 21, 34, 55, 64]), "small")
    fleet = synth_fleet(12, 4, seed=7, keep_accelerator=True, zero_load_frac=0.3)
    fleet.srv_min_replicas[::3] = 0
    _winners_check(engine, oracle_mod, fleet, Grid([1, 4, 16, 64], np.arange(1, 41)), "keep accelerator, zero load")
    fleet = synth_fleet(3, 2, seed=3)
    _winners_check(engine, oracle_mod, fleet, Grid([5], [3]), "one cell per pair")
    _winners_check(engine, oracle_mod, fleet, Grid([2, 9], np.arange(1, 34)), "R = 33")
    fleet = synth_fleet(10, 4, seed=11)
    fleet.perf_present[0, 1] = 0
    fleet.perf_present[3, :] = 0
    fleet.srv_has_target[5] = 0
    fleet.srv_model[6] = -1
    fleet.srv_arrival_rpm[8] = -1.0
    _winners_check(engine, oracle_mod, fleet, Grid([2, 8, 32], [1, 2, 4, 8, 16, 32]), "missing profiles and targets")


def test_winners_randomised_small_fleets(engine, oracle_mod):
    """The fleets and grids of test_grid_randomised_small_fleets (same seeds, same draws)."""
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
        batch = rng.integers(1, 97, nb)
        replicas = rng.integers(1, 70, nr)
        _winners_check(engine, oracle_mod, fleet, Grid(batch, replicas), f"randomised case {case}")


def test_winners_adversarial_fleets(engine, oracle_mod):
    """The grid cases of test_adversarial_parameters_size_and_grid (same seeds, same draws)."""
    rng = np.random.default_rng(424242)
    for case in range(150):
        fleet = _adversarial_fleet(rng, case)
        if case % 2 == 0:
            grid = Grid(rng.integers(1, 40, int(rng.integers(1, 6))), rng.integers(1, 30, int(rng.integers(1, 12))))
            _winners_check(engine, oracle_mod, fleet, grid, f"adversarial case {case}")


def test_winners_rows_decided_by_shared_cells_or_none(engine, oracle_mod):
    """Long, unsorted batch lists with repeated sizes and R = 70 replica levels (more than two per lane of a warp).
    Zero-load servers; TPS-limited servers, whose small batch sizes fail the stability limit, so their rows are
    decided by a shared cell at a larger size; servers with an unreachable ITL target, whose rows have no feasible
    cell and are walked to the end."""
    rng = np.random.default_rng(5)
    fleet = synth_fleet(10, 3, seed=313, zero_load_frac=0.2, tps_frac=0.4, max_batch_choices=(64, 128, 256))
    fleet.srv_slo_itl[[1, 6]] = 1e-4
    batch = rng.permutation(np.r_[np.arange(1, 121), [3, 40, 40, 120]])
    cells_o, win_o = oracle_mod.grid_solve(fleet, Grid(batch, np.arange(1, 71)))
    feas = ((cells_o["flags"] >> 1) & 1).reshape(fleet.n_servers, fleet.n_acc, batch.size, 70).any(axis=2)
    ok = (cells_o["flags"] & 1).reshape(fleet.n_servers, fleet.n_acc, batch.size, 70).any(axis=2)
    assert (ok & ~feas).sum() > 50, "the case must have analysable rows without a feasible cell"
    assert feas.sum() > 200
    _winners_check(engine, oracle_mod, fleet, Grid(batch, np.arange(1, 71)), "shared-decided rows")
    _winners_check(engine, oracle_mod, fleet, Grid(batch[::-1], np.arange(70, 0, -1)), "reversed lists")


def test_winners_with_cells_beyond_two_pow_23_states(engine, oracle_mod):
    """A queue ratio of 4000 puts K = N (1 + 4000) >= 2^23 at the two largest batch sizes, which grid_kernel
    evaluates, right after shared cells (N = 2000, K < 2^23) of the same rows."""
    fleet = synth_fleet(2, 1, seed=41, zero_load_frac=0.0, tps_frac=0.0, max_batch_choices=(64,))
    fleet.srv_arrival_rpm[:] = np.float32([30.0, 600.0])
    fleet.max_queue_to_batch_ratio = 4000
    grid = Grid([1, 2, 50, 2000, 2097, 2100], [1, 2, 3, 5])
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid)
    cells_g, win_g = engine.grid_solve(fleet, grid, want_cells=True)
    assert np.array_equal(cells_g["flags"], cells_o["flags"])
    assert (cells_o["flags"].reshape(2, 6, 4)[:, 3:] & 1).sum() > 0, "the largest batch sizes must be analysable"
    assert_allocs_equal(win_g, win_o, "winners with the cell table")
    _winners_check(engine, oracle_mod, fleet, grid, "K >= 2^23 next to shared cells")
