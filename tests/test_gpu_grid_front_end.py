"""The grid step's front end, bit for bit against the oracle (DESIGN.md 3.3).

``grid_order`` solves a server's rows itself, from the server's tables staged in shared memory while
``A·Bmax <= kOrderTabEntries = 4096`` and read from global memory above that.  ``FRONT_END`` puts one case on each side
of that threshold, with short tables (many accelerators) and with long ones, and one with ``A·R`` rows above the
ranking limit (``kOrderMaxRows = 2048``: pruning off) in which some pairs have no table.  Each runs with the cell table,
without it, and pruned against cell-table winners.

The step's kernels after ``build_pair_tables`` start while their predecessor drains and wait for it before reading
what the step wrote, and ``build_pair_tables`` zeroes the step's counters.  ``test_back_to_back_steps`` enqueues grid
steps on different grids and fleets without synchronising between them, interleaved with a load grid, a size grid and
a call with the cell table on the same handle: a counter left over from an earlier call, or a read that the wait does
not cover, gives a winner block that differs from its own oracle answer.
"""
from __future__ import annotations

import functools

import numpy as np
import pytest

from tests.grid_cases import _cells_equal, _three_ways, device_winners, shape_fleet
from tests.util import assert_allocs_equal
from workload_variant_autoscaler_b200 import Grid

f32 = np.float32
STAGED_ENTRIES = 4096  # kOrderTabEntries

# name: (S, A, batch list, replica list, staged)
FRONT_END = {
    "A*Bmax=4096 (A=16)": (4, 16, [40, 16, 256, 24], [1, 2, 3], True),
    "A*Bmax=4097 (A=17)": (4, 17, [40, 16, 241, 24], [1, 2, 3], False),
    "A*Bmax=4096 (A=2)": (5, 2, [24, 16, 2048, 48], [1, 2, 3, 5, 8, 13], True),
    "A*Bmax=4097 (A=1)": (5, 1, [24, 16, 4097, 48], [1, 2, 3, 5, 8, 13], False),
    "A*R=4096": (5, 4, [40, 16, 64], np.arange(1, 1025), True),
}


@functools.lru_cache(maxsize=None)
def front_end_case(name):
    S, A, batch, replicas, _ = FRONT_END[name]
    return shape_fleet(S, A, 301 + list(FRONT_END).index(name)), Grid(batch, replicas)


def test_front_end_cases_sit_on_their_sides():
    for name, (S, A, batch, replicas, staged) in FRONT_END.items():
        assert (A * max(batch) <= STAGED_ENTRIES) == staged, name
    fleet, grid = front_end_case("A*R=4096")
    assert fleet.n_acc * grid.replicas.size > 2048, "pruning is off above kOrderMaxRows rows"
    assert not fleet.perf_present[fleet.srv_model[3], fleet.n_acc - 1], "server 3 has a pair without a table"
    assert fleet.srv_arrival_rpm[0] == 0, "server 0 has no load: none of its pairs has a table"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FRONT_END))
def test_grid_front_end(engine, oracle_mod, name):
    fleet, grid = front_end_case(name)
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    _three_ways(engine, fleet, grid, cells_o, win_o, name)


class _Block:
    """A device winner block (10 columns of S words, see device_winners) read back as Allocs columns."""

    def __init__(self, blk, S):
        w = blk.cpu().numpy()
        self.n = S
        self.feasible = w.view(np.uint8)[:S]
        self.acc, self.replicas, self.batch = (w[k * S:(k + 1) * S] for k in (1, 2, 3))
        f = w.view(np.float32)
        for k, name in enumerate(("cost", "value", "itl", "ttft", "rho", "max_rate"), start=4):
            setattr(self, name, f[k * S:(k + 1) * S])

    def record(self, i):
        return {k: getattr(self, k)[i] for k in ("feasible", "acc", "replicas", "batch", "cost", "value")}


@pytest.mark.gpu
def test_back_to_back_steps(engine, oracle_mod):
    from workload_variant_autoscaler_b200 import synth_fleet
    f1 = synth_fleet(40, 4, seed=311)
    f2 = shape_fleet(30, 3, 312)
    S1, S2 = f1.n_servers, f2.n_servers
    g1 = Grid([4, 8, 16, 32, 64, 128], np.arange(1, 33))
    g2 = Grid([96, 8, 256, 2, 40], [1, 2, 3, 5, 8, 13, 21])
    g3 = Grid([16, 1536, 24], np.arange(1, 9))
    blocks = {k: device_winners(S1 if k < 3 else S2) for k in range(6)}
    want = {}

    engine.upload(f1)
    for k, g in ((0, g1), (1, g2), (2, g1)):  # three steps, no synchronisation in between
        engine.grid_solve_device(g, blocks[k][1])
        want[k] = (f1, g)
    levels = np.stack([f1.srv_arrival_rpm * f32(x) for x in (0.5, 2.0)])
    engine.load_grid(f1, levels)
    cells_g, win_c = engine.grid_solve(f2, g2, want_cells=True)  # f2 is resident from here on
    engine.grid_solve_device(g3, blocks[3][1])
    engine.grid_solve_device(g1, blocks[4][1])
    want[3], want[4] = (f2, g3), (f2, g1)
    engine.size_grid(f2, [8, 32])
    engine.upload(f2)
    engine.grid_solve_device(g2, blocks[5][1])
    want[5] = (f2, g2)
    engine.synchronize()

    cells_o, win_o = oracle_mod.grid_solve(f2, g2, want_cells=True)
    _cells_equal(cells_g, cells_o, "cell-table call between device steps")
    assert_allocs_equal(win_c, win_o, "cell-table call between device steps: winners")
    for k, (fleet, grid) in want.items():
        _, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=False)
        assert_allocs_equal(_Block(blocks[k][0], fleet.n_servers), win_o, f"device step {k}")
