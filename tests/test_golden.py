"""Committed golden fixtures (tests/golden/make_golden.py): the oracle must keep reproducing them
on CPU, and the CUDA path must reproduce them through the C ABI on the GPU box."""
import os
import sys

import numpy as np
import pytest


HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden as mg  # noqa: E402
from tests.util import assert_allocs_equal, assert_f32_bits_equal

GOLD = np.load(os.path.join(HERE, "golden", "golden_r01.npz"))


def _structs_equal(a, b):
    assert a.dtype == b.dtype and a.shape == b.shape
    for name in a.dtype.names:
        x, y = np.ascontiguousarray(a[name]).reshape(-1), np.ascontiguousarray(b[name]).reshape(-1)
        if x.dtype == np.float32:
            assert_f32_bits_equal(x, y, name)
        else:
            assert np.array_equal(x, y), name


def _synth():
    from workload_variant_autoscaler_b200 import Grid, synth_fleet
    f = synth_fleet(12, 3, seed=2024, max_batch_choices=(2, 4, 8, 16, 32), zero_load_frac=0.15)
    f.srv_min_replicas[::5] = 0
    return f, Grid([1, 2, 4, 8, 16, 31], [1, 2, 3, 4, 6, 8, 12, 16, 24, 33])


def test_oracle_reproduces_golden(oracle_mod):
    rows = []
    for it, ot in mg.CONFIG1_TOKENS:
        for rpm in mg.CONFIG1_LOADS:
            rows.append(oracle_mod.solve(mg.config1_fleet(rpm, it, ot))[1][0])
    _structs_equal(np.array(rows, dtype=oracle_mod.ALLOC_DTYPE), GOLD["config1_winners"])
    f, grid = _synth()
    cand, win = oracle_mod.solve(f)
    _structs_equal(cand, GOLD["synth_cand"])
    _structs_equal(win, GOLD["synth_win"])
    cells, gwin = oracle_mod.grid_solve(f, grid)
    _structs_equal(cells, GOLD["grid_cells"])
    _structs_equal(gwin, GOLD["grid_win"])
    sw = oracle_mod.sweep(f, 16)
    for k, v in sw.items():
        if v.dtype == np.float32:
            assert_f32_bits_equal(v, GOLD["sweep_" + k], k)
        else:
            assert np.array_equal(v, GOLD["sweep_" + k])


def test_config1_decisions_are_sane():
    """BASELINE configs[0] (single VA on A100, N=4): zero load keeps 1 replica; replicas grow with load."""
    w = GOLD["config1_winners"]
    n = len(mg.CONFIG1_LOADS)
    for block in (w[:n], w[n:]):
        assert block["feasible"].all() and (block["acc"] == 0).all() and (block["batch"] == 4).all()
        assert block["replicas"][0] == 1
        assert (np.diff(block["replicas"]) >= 0).all() and block["replicas"][-1] > 1
        assert (block["itl"][1:] <= 24.0 + 1e-3).all()


@pytest.mark.gpu
def test_cuda_reproduces_golden(engine):
    n = len(mg.CONFIG1_LOADS)
    k = 0
    for it, ot in mg.CONFIG1_TOKENS:
        for rpm in mg.CONFIG1_LOADS:
            _, win = engine.solve(mg.config1_fleet(rpm, it, ot))
            assert_allocs_equal(win, GOLD["config1_winners"][k:k + 1], f"config1 load {rpm} tokens {it}/{ot}")
            k += 1
    assert k == 2 * n
    f, grid = _synth()
    cand, win = engine.solve(f)
    assert_allocs_equal(cand, GOLD["synth_cand"], "golden size candidates")
    assert_allocs_equal(win, GOLD["synth_win"], "golden winners")
    cells, gwin = engine.grid_solve(f, grid, want_cells=True)
    assert np.array_equal(cells["flags"], GOLD["grid_cells"]["flags"])
    for key in ("ttft", "itl", "rho", "throughput"):
        assert_f32_bits_equal(cells[key], GOLD["grid_cells"][key], key)
    assert_allocs_equal(gwin, GOLD["grid_win"], "golden grid winners")
    sw = engine.sweep(f, 16)
    assert np.array_equal(sw["valid"], GOLD["sweep_valid"])
    for key in ("rate", "ttft", "itl", "throughput", "rho"):
        assert_f32_bits_equal(sw[key], GOLD["sweep_" + key], key)
