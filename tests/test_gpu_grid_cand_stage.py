"""grid_sort_cands on both sides of its shared-memory stage, bit for bit against the oracle.

Per chunk, ``grid_sort_cands`` stages the tables its candidates read (batch index and size by rank, the pair's
(table, batch) constants, the table's prefix log2 sums, the server's rate block and the pair's rows) in shared memory
while ``cand_stage_bytes = 24·B + 32·R + 4·Bmax <= kCandStageBytes = 16384``, and reads them from global memory
otherwise.  The two cases sit on the exact edge (16384 and 16408 bytes), built like ``test_gpu_grid_shapes``' cases and
run the same three ways: with the cell table, without it, and pruned winners against cell-table winners.  The
flagship shape (BASELINE config 2) must take the staged path.
"""
from __future__ import annotations

import functools

import pytest

from tests.grid_cases import STAGE_B, _batches, _three_ways, shape_fleet, winner_mix
from workload_variant_autoscaler_b200 import Grid, config2_grid

STAGE_CAP = 16384  # kCandStageBytes


def stage_bytes(grid):
    """cand_stage_bytes (wva_kernels.cuh) of a grid."""
    return 24 * int(grid.batch.size) + 32 * int(grid.replicas.size) + 4 * max(1, int(grid.batch.max()))


# name: (S, A, B batch sizes drawn from STAGE_B, replica list)
CASES = {
    "stage=16384": (4, 2, 668, [1, 4, 16]),
    "stage=16408": (4, 2, 669, [1, 4, 16]),
}


@functools.lru_cache(maxsize=None)
def stage_case(name):
    S, A, B, replicas = CASES[name]
    seed = 211 + list(CASES).index(name)
    return shape_fleet(S, A, seed), Grid(_batches(STAGE_B, B, seed), replicas)


@functools.lru_cache(maxsize=None)
def stage_oracle(name):
    import oracle
    return oracle.grid_solve(*stage_case(name), want_cells=True)


def test_stage_cases_sit_on_the_edge():
    assert [stage_bytes(stage_case(n)[1]) for n in CASES] == [STAGE_CAP, STAGE_CAP + 24]
    assert stage_bytes(config2_grid()) <= STAGE_CAP


@pytest.mark.parametrize("name", list(CASES))
def test_stage_case_has_winners_from_both_sources(oracle_mod, name):
    """Winners from shared-chain cells and from grid_kernel cells, so that the staged candidates decide some."""
    fleet, grid = stage_case(name)
    cells, win = stage_oracle(name)
    shared, kernel, _ = winner_mix(fleet, grid, cells, win)
    assert shared >= 1 and kernel >= 1, (shared, kernel)


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_grid_at_candidate_stage_edge(engine, oracle_mod, name):
    fleet, grid = stage_case(name)
    cells_o, win_o = stage_oracle(name)
    _three_ways(engine, fleet, grid, cells_o, win_o, name)
