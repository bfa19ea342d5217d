"""grid_kernel's one-pass exit and its exact fallback (DESIGN.md 3.2b), bit for bit against the oracle.

* Saturated fleets: every server's lambda lies between half and 0.999 of the tail rate of its batch size, with a queue
  of ten batches (K = 11 N), so the cells' chains run into the tail and go through ``grid_kernel``; nearly every warp
  takes the one-pass exit.
* The mixed warp: one pair, batch size 3 and 32 replica levels, so its 32 candidate cells are one full item with one
  pair table (the staged solve).  31 lanes are light loads that pass 1 decides; one lane's load is so small that its
  ``in_serv`` lies far below ``E_in``'s absolute term, and its one-pass ``in_serv`` rounds to a different float32 than
  the reference's (``tests.onepass.mix_replicas``), which the cell's ``rho`` (``in_serv / N``) would show.  So the warp must run pass 2, including its staged head from state 1,
  and every lane must come out with the reference's bits.
"""
from __future__ import annotations

import numpy as np
import pytest

from tests.grid_cases import _cells_equal, _fleet, _lam_grid, chain_profile
from tests.onepass import MIX_DELTA, MIX_N, MIX_RATIO, MIX_RPM, decided, mix_lane, mix_rates, mix_replicas
from tests.util import assert_allocs_equal
from workload_variant_autoscaler_b200 import Grid

f32 = np.float32
BATCHES = [4, 8, 16, 32, 64, 128, 256]
RATIO = 10


def saturated_case(seed):
    """alpha = gamma = 1 ms, beta = delta = 0: servRate[n-1] = n / 2 per ms; lambda near servRate[N-1] of a batch."""
    rng = np.random.default_rng(seed)
    S = 96
    N = rng.choice(BATCHES, S)
    frac = rng.uniform(0.5, 0.999, S)
    rpm = (N / 2.0 * frac * 60000.0).astype(np.float32)
    return _fleet(1.0, 1.0, rpm, 256, ratio=RATIO), Grid(BATCHES, [1, 2]), N


def mixed_case():
    return _fleet(1.0, 1.0, [MIX_RPM], MIX_N, delta=MIX_DELTA, ratio=MIX_RATIO), Grid([MIX_N], mix_replicas())


def test_saturated_case_reaches_the_tail():
    fleet, _, N = saturated_case(0)
    rates = [(np.arange(1, n + 1, dtype=np.float32) / f32(2)).astype(np.float32) for n in N]
    lam = np.array([_lam_grid(r, 1) for r in fleet.srv_arrival_rpm], np.float32)
    pr = chain_profile(rates, N * (1 + RATIO), lam)
    # each server's own batch size: the chain reaches state N - 1 without overflowing, so the cell does not share
    # its row's chain and grid_kernel solves it
    assert pr["tail"].all() and not pr["over"].any()


def test_mixed_warp_has_one_undecided_lane(oracle_mod):
    qa = oracle_mod.Analyzer(MIX_N, MIX_N * MIX_RATIO, 1.0, 0.0, 1.0, MIX_DELTA, 1, 2)
    assert np.array_equal(np.asarray(qa.serv_rate(), np.float32).view(np.uint32), mix_rates().view(np.uint32))
    assert qa.K == MIX_N * (1 + MIX_RATIO)
    reps = mix_replicas()
    assert len(reps) == 32
    lanes = [mix_lane(r) for r in reps]
    for r, L in zip(reps, lanes):
        # b = 3 < j + 2: no cell shares its row's chain, so all 32 are grid_kernel's
        assert L["m"] >= 2, r
    # 31 lanes decided with room to spare (the kernel's exit state may lie a block past the reference's)
    for r, L in zip(reps[:-1], lanes[:-1]):
        assert decided(L["A1"], 4 * L["E_acc"]) and decided(L["I1"], 4 * L["E_in"]), r
    last = lanes[-1]
    assert not decided(last["I1"], last["E_in"])
    assert f32(last["I1"]) != f32(last["in_serv"])


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(3))
def test_grid_onepass_cells_match_oracle(engine, oracle_mod, seed):
    fleet, grid, _ = saturated_case(seed)
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    cells_g, win_g = engine.grid_solve(fleet, grid, want_cells=True)
    _cells_equal(cells_g, cells_o, f"saturated case {seed}")
    assert_allocs_equal(win_g, win_o, f"saturated case {seed} winners (cell table)")
    _, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=False)
    _, win_g = engine.grid_solve(fleet, grid, want_cells=False)
    assert_allocs_equal(win_g, win_o, f"saturated case {seed} winners")


@pytest.mark.gpu
def test_grid_mixed_warp_falls_back_to_pass_2(engine, oracle_mod):
    fleet, grid = mixed_case()
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    assert np.all(cells_o["flags"] != 0)  # every cell analysed, every metric finite
    for k in ("ttft", "itl", "rho", "throughput"):
        assert np.all(np.isfinite(cells_o[k])), k
    cells_g, win_g = engine.grid_solve(fleet, grid, want_cells=True)
    _cells_equal(cells_g, cells_o, "mixed warp")
    assert_allocs_equal(win_g, win_o, "mixed warp winners (cell table)")
    _, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=False)
    _, win_g = engine.grid_solve(fleet, grid, want_cells=False)
    assert_allocs_equal(win_g, win_o, "mixed warp winners")
