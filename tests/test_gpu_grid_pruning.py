"""Grid winners when the cells that cannot win are skipped (grid_solve without a cell table).

Without a cell table the rows of each server are ranked by (value, cost, replicas), the shared-chain cells give each
server a bound (the smallest key of a feasible cell), and grid_kernel only evaluates the cells at or below it, plus
the exact gates (TPS stability limit, alpha > slo_itl).  With a cell table every cell is evaluated.  The winners must
be the same bits either way, the same as the oracle's on small fleets, and the same as those of the build before the
pruning at the benchmark's size (tests/golden/grid_winners_config2.npz, written by that build).
"""
import os

import numpy as np
import pytest

from tests.grid_cases import _same_winners, check_pruning
from tests.util import ALLOC_FIELDS
from workload_variant_autoscaler_b200 import Grid, config2_grid, synth_fleet

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "grid_winners_config2.npz")
@pytest.mark.parametrize("seed", range(42, 50))
def test_pruned_winners_at_bench_size(engine, seed):
    fleet, grid = synth_fleet(100, 4, seed=seed), config2_grid()
    _, win_p = engine.grid_solve(fleet, grid)
    _, win_c = engine.grid_solve(fleet, grid, want_cells=True)
    _same_winners(win_p, win_c, f"seed {seed}")
    ref = np.load(GOLDEN)
    for f in ALLOC_FIELDS:
        want = ref[f"s{seed}_{f}"]
        got = np.asarray(getattr(win_p, f))
        assert np.array_equal(got.astype(want.dtype).view(np.uint8), want.view(np.uint8)), f"seed {seed}: field {f}"


def test_tied_rows_across_accelerators(engine, oracle_mod):
    """acc_cost x acc_count equal on every accelerator and no current allocation: the rows of one replica level tie
    in (value, cost, replicas), so the batch size and then the accelerator decide."""
    fleet = synth_fleet(12, 4, seed=17, zero_load_frac=0.0, tps_frac=0.0)
    fleet.acc_cost[:] = np.float32([80.0, 40.0, 20.0, 10.0])
    fleet.perf_acc_count[:] = np.int32([1, 2, 4, 8])
    fleet.srv_cur_acc[:] = -1
    fleet.srv_cur_replicas[:] = 0
    fleet.srv_cur_cost[:] = 0.0
    check_pruning(engine, oracle_mod, fleet, Grid([1, 2, 4, 8, 16, 32, 64, 128], np.arange(1, 25)), "tied rows")


def test_repeated_unsorted_batches_and_current_allocations(engine, oracle_mod):
    """Repeated, unsorted batch sizes; current allocations whose replica level gives value 0 and whose cost makes
    the other levels of that accelerator negative."""
    fleet = synth_fleet(16, 3, seed=23, zero_load_frac=0.1, tps_frac=0.2)
    fleet.srv_cur_acc[:] = np.arange(16) % 3
    fleet.srv_cur_replicas[:] = 1 + np.arange(16) % 5
    fleet.srv_cur_cost[:] = np.float32(5000.0)
    batch = np.array([64, 3, 17, 3, 128, 1, 64, 9, 255, 2, 17, 40])
    check_pruning(engine, oracle_mod, fleet, Grid(batch, np.arange(1, 31)), "repeated batches, value <= 0")
    check_pruning(engine, oracle_mod, fleet, Grid(batch[::-1], np.arange(30, 0, -1)), "reversed lists")


def test_no_feasible_shared_cell_tps_and_itl_gates(engine, oracle_mod):
    """Servers with an unreachable ITL target (alpha > slo_itl: nothing feasible, the bound stays open) next to TPS
    servers, whose small batch sizes fail the stability limit, and ordinary ones."""
    fleet = synth_fleet(14, 3, seed=29, zero_load_frac=0.1, tps_frac=0.5, max_batch_choices=(32, 64, 128, 256))
    fleet.srv_slo_itl[[0, 5, 9]] = 1.0
    cells_o, _ = oracle_mod.grid_solve(fleet, Grid(np.arange(1, 97), np.arange(1, 41)))
    feas = ((cells_o["flags"] >> 1) & 1).reshape(14, -1).any(axis=1)
    assert not feas[[0, 5, 9]].any() and feas.sum() >= 3
    check_pruning(engine, oracle_mod, fleet, Grid(np.arange(1, 97), np.arange(1, 41)), "ITL / TPS gates")


def test_cells_beyond_two_pow_23_next_to_shared_runs(engine, oracle_mod):
    """K = N (1 + 4000) >= 2^23 at the largest batch sizes, right after shared cells of the same rows."""
    fleet = synth_fleet(4, 2, seed=41, zero_load_frac=0.0, tps_frac=0.0, max_batch_choices=(64,))
    fleet.srv_arrival_rpm[:] = np.float32([30.0, 600.0, 120.0, 2400.0])
    fleet.max_queue_to_batch_ratio = 4000
    check_pruning(engine, oracle_mod, fleet, Grid([1, 2, 50, 2000, 2097, 2100], [1, 2, 3, 5]), "K >= 2^23")


def test_nan_value_turns_pruning_off(engine):
    """An infinite current cost makes the value of other accelerators NaN: that server is not pruned, and the
    winners match the fully evaluated grid."""
    fleet = synth_fleet(10, 3, seed=31, zero_load_frac=0.0)
    fleet.srv_cur_acc[[2, 7]] = 0
    fleet.srv_cur_replicas[[2, 7]] = 2
    fleet.srv_cur_cost[[2, 7]] = np.inf
    grid = Grid(np.arange(1, 65), np.arange(1, 33))
    _, win_p = engine.grid_solve(fleet, grid)
    _, win_c = engine.grid_solve(fleet, grid, want_cells=True)
    _same_winners(win_p, win_c, "NaN values")
