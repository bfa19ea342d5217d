"""The cells handed to grid_kernel, at the edges of grid_order's rank intervals.

grid_order lists, per (server, accelerator, replica level) row, the cells left for grid_kernel as two rank intervals,
[0, min(lo, hi)) and [max(lo, kK), hi): lo is the row's first shared rank (b >= j + 2), kK the first rank with
K >= 2^23 and hi the first rank whose key (group, batch size, accelerator) lies above the server's bound (B with a
cell table).  Rows with no load and pairs without a table have none, nor, without a cell table, do pairs with
alpha > slo_itl; grid_sort_cands sorts them in chunks of at most 4096 candidates of one pair.  Every case here is
checked byte for byte against the oracle's winners and the winners of the cell-table path (which evaluates every
cell).

``wva_dbg_read_plan`` returns item_count[2·256 + 1 ..], so slots 15 and 16 are the candidates and chunks that
grid_order listed on the last call.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_grid_pruning import _check, _same_winners
from tests.test_gpu_grid_shapes import (INV_BATCH, INV_REPLICAS, _analyzer_of, _lambda, _three_ways, cell_shares_row,
                                        invariant_fleet, shape_fleet)
from tests.test_gpu_windows import chain_profile
from workload_variant_autoscaler_b200 import Grid, config2_grid, synth_fleet

CHUNK = 4096
f32 = np.float32


def _listed(engine):
    """(candidates, chunks) grid_order listed on the engine's last grid call."""
    plan = (C.c_uint32 * 31)()
    assert engine._L.wva_dbg_read_plan(engine._h, plan) == 0
    return int(plan[15]), int(plan[16])


# ---------------------------------------------------------------------------------------------------------------
# cases
# ---------------------------------------------------------------------------------------------------------------
def tied_repeated_case():
    """Rows of one replica level tie in (value, cost, replicas) on every accelerator, accelerator 1 has accelerator
    0's profile, and batch sizes repeat: a bound falls between repeated batch sizes of one row and between
    accelerators of equal group and batch size."""
    fleet = synth_fleet(12, 4, seed=67, zero_load_frac=0.0, tps_frac=0.0)
    fleet.acc_cost[:] = np.float32([80.0, 40.0, 20.0, 10.0])
    fleet.perf_acc_count[:] = np.int32([1, 2, 4, 8])
    for col in (fleet.perf_alpha, fleet.perf_beta, fleet.perf_gamma, fleet.perf_delta):
        col[:, 1] = col[:, 0]
    fleet.srv_cur_acc[:] = -1
    fleet.srv_cur_replicas[:] = 0
    fleet.srv_cur_cost[:] = 0.0
    batch = np.array([32, 8, 64, 8, 2, 128, 32, 16, 16, 1, 64, 4])
    return fleet, Grid(batch, np.arange(1, 21))


def gates_case():
    """Zero-load rows, a pair without a table, alpha > slo_itl on two servers (the pair is out), TPS servers whose
    small batch sizes fail the stability limit, and light to heavy loads: rows with a shared run (lo < B) next to
    rows without one (j = INT_MAX), each row's group above, equal to or below its server's bound group."""
    fleet = shape_fleet(14, 3, seed=71)
    fleet.srv_slo_tps[[5, 9]] = 800.0
    fleet.srv_slo_itl[[4, 11]] = 1.0
    return fleet, Grid([24, 2, 16, 64, 40, 16, 3, 8], np.arange(1, 41))


def k_limit_case():
    """K = N (1 + 4000) >= 2^23 from batch size 2097 on, right after the shared run of the same rows: the second
    interval [max(lo, kK), hi)."""
    fleet = synth_fleet(6, 2, seed=73, zero_load_frac=0.0, tps_frac=0.0, max_batch_choices=(64,))
    fleet.srv_arrival_rpm[:] = np.float32([30.0, 600.0, 120.0, 2400.0, 9.0, 60.0])
    fleet.max_queue_to_batch_ratio = 4000
    return fleet, Grid([1, 2, 50, 2000, 2097, 2097, 2100], [1, 2, 3, 5, 8])


def zero_candidates_case():
    """Short chains (invariant_fleet: the rows share their chains from a small batch size on), every other server
    without load and the others with alpha > slo_itl: grid_order lists nothing, and the winners come from the shared
    rows' walk and the zero-load rows alone."""
    fleet = invariant_fleet()
    fleet.srv_arrival_rpm[::2] = 0.0
    fleet.srv_slo_itl[1::2] = 0.5
    return fleet, Grid(INV_BATCH, INV_REPLICAS)


def nan_fleet(fleet):
    """An infinite current cost on accelerator 0 makes the value of the other accelerators NaN: no server is
    pruned, so every non-shared cell of a loaded row with a table is a candidate."""
    fleet.srv_cur_acc[:] = 0
    fleet.srv_cur_replicas[:] = 2
    fleet.srv_cur_cost[:] = np.inf
    return fleet


def one_server_case():
    """One server, two accelerators, nothing pruned (NaN values), 128 batch sizes x 120 replica levels: more than
    2 x 4096 candidates, so a pair takes more than one chunk."""
    fleet = synth_fleet(1, 2, seed=79, zero_load_frac=0.0, tps_frac=0.0, max_batch_choices=(128,))
    fleet.max_queue_to_batch_ratio = 1
    fleet.srv_arrival_rpm[:] = 6000.0
    fleet.srv_slo_ttft[:] = 0.0
    fleet.srv_slo_itl[:] = 0.0
    return nan_fleet(fleet), Grid(np.arange(1, 129), np.arange(1, 121))


# ---------------------------------------------------------------------------------------------------------------
# CPU: the cases hold what they are for
# ---------------------------------------------------------------------------------------------------------------
def test_zero_candidates_case_has_no_candidate_row():
    fleet, grid = zero_candidates_case()
    m = fleet.srv_model
    assert ((fleet.srv_arrival_rpm == 0) | (fleet.perf_alpha[m, 0] > fleet.srv_slo_itl)).all()
    assert (fleet.srv_arrival_rpm > 0).sum() >= 20 and (fleet.srv_arrival_rpm == 0).sum() >= 20


def test_one_server_case_has_more_than_two_chunks_of_candidates(oracle_mod):
    """Analysable cells that do not share their row's chain (cell_shares_row, a batch size at a time)."""
    fleet, grid = one_server_case()
    cells, _ = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    ok = (cells["flags"] & 1).reshape(2, grid.batch.size, grid.replicas.size).astype(bool)
    lams = [_lambda(fleet, 0, int(r)) for r in grid.replicas]
    n = 0
    for a in range(2):
        for bi, b in enumerate(grid.batch):
            qa = _analyzer_of(fleet, 0, a, int(b))
            P = chain_profile(qa.serv_rate(), qa.K, lams)
            shared = ~P["over"] & ~P["tail"] & (int(b) >= P["j"] + 2) & (qa.K < (1 << 23))
            n += int((ok[a, bi] & ~shared).sum())
    assert n > 2 * CHUNK, n


def test_gates_case_has_cells_only_grid_kernel_stores(oracle_mod):
    """Without a cell table grid_order drops the pairs with alpha > slo_itl and grid_sort_cands the TPS cells above
    the stability limit (lambda > RateRange.Max / 1000 · 0.9); with a cell table grid_kernel stores both as analysed
    and not feasible.  The case has cells of both kinds that do not share their row's chain."""
    fleet, grid = gates_case()
    cells, _ = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    S, A = fleet.n_servers, fleet.n_acc
    flags = cells["flags"].reshape(S, A, grid.batch.size, grid.replicas.size)
    m = fleet.srv_model
    found = {"itl": False, "tps": False}
    for s, a, bi, ri in zip(*np.nonzero(flags == 1)):
        s, a, b, r = int(s), int(a), int(grid.batch[bi]), int(grid.replicas[ri])
        itl = fleet.srv_slo_itl[s]
        if itl != 0 and fleet.perf_beta[m[s], a] >= 0 and fleet.perf_alpha[m[s], a] > itl:
            kind = "itl"
        elif fleet.srv_slo_tps[s] > 0:
            lim = f32(f32(f32(_analyzer_of(fleet, s, a, b).rate_range()[1]) / f32(1000)) * f32(f32(1) - f32(0.1)))
            kind = "tps" if _lambda(fleet, s, r) > lim else None
        else:
            kind = None
        if kind and not found[kind] and not cell_shares_row(fleet, s, a, b, r):
            found[kind] = True
    assert all(found.values()), found


# ---------------------------------------------------------------------------------------------------------------
# GPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("case", [tied_repeated_case, gates_case, k_limit_case], ids=lambda c: c.__name__)
def test_candidate_intervals_against_oracle(engine, oracle_mod, case):
    fleet, grid = case()
    _check(engine, oracle_mod, fleet, grid, case.__name__)


@pytest.mark.gpu
def test_zero_candidates(engine, oracle_mod):
    fleet, grid = zero_candidates_case()
    _, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=False)
    _, win_p = engine.grid_solve(fleet, grid)
    assert _listed(engine) == (0, 0)
    from tests.util import assert_allocs_equal
    assert_allocs_equal(win_p, win_o, "zero candidates")
    _, win_c = engine.grid_solve(fleet, grid, want_cells=True)
    _same_winners(win_p, win_c, "zero candidates: pruned vs cell table")


@pytest.mark.gpu
def test_one_server_several_chunks_per_pair(engine, oracle_mod):
    fleet, grid = one_server_case()
    _, win_p = engine.grid_solve(fleet, grid)
    n, chunks = _listed(engine)
    assert n > 2 * CHUNK and chunks >= 3, (n, chunks)  # two pairs: one of them has two chunks
    _check(engine, oracle_mod, fleet, grid, "one server, several chunks per pair")


@pytest.mark.gpu
@pytest.mark.parametrize("case", [one_server_case, gates_case], ids=lambda c: c.__name__)
def test_cell_table_against_oracle(engine, oracle_mod, case):
    """With a cell table grid_order lists every cell of a loaded row with a table that does not share its row's
    chain: one_server_case spans several chunks per pair, and gates_case has ITL-out pairs and TPS cells above the
    stability limit, which only grid_kernel stores."""
    fleet, grid = case()
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    if case is one_server_case:
        engine.grid_solve(fleet, grid, want_cells=True)
        n, chunks = _listed(engine)
        assert n > 2 * CHUNK and chunks >= 3, (n, chunks)
    _three_ways(engine, fleet, grid, cells_o, win_o, f"{case.__name__}, cell table")


@pytest.mark.gpu
def test_nan_servers_at_bench_shape(engine):
    fleet, grid = nan_fleet(synth_fleet(100, 4, seed=42)), config2_grid()
    _, win_p = engine.grid_solve(fleet, grid)
    n, chunks = _listed(engine)
    _, win_c = engine.grid_solve(fleet, grid, want_cells=True)
    _same_winners(win_p, win_c, "NaN values on every server")
    engine.grid_solve(synth_fleet(100, 4, seed=42), grid)
    n_pruned, _ = _listed(engine)
    assert n > 5 * n_pruned and chunks > n // CHUNK, (n, n_pruned, chunks)
