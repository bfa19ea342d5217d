"""The service-rate table caches on one handle.

Each path keeps its tables in a set of its own (the solve path, the size grid, the load grid, the grid), and the
sweep builds into the grid's.  These tests interleave every path on one handle and compare each result byte for
byte with the same call on a fresh handle, and pin, through the launch count, which calls rebuild their tables:
the solve path only when the token epoch changes, the grid on every call."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_load_grid import ALLOC_FIELDS, load_levels, mixed_fleet
from workload_variant_autoscaler_b200 import Engine, Grid, _abi, synth_fleet


def device_winners(S):
    """(tensor, AllocsC): a zeroed device winner block of S records and its columns."""
    import torch
    blk = torch.zeros(10 * S, dtype=torch.int32, device="cuda")
    cols = _abi.AllocsC()
    b = blk.data_ptr()
    cols.feasible = C.cast(b, _abi.u8p)
    for k, name in enumerate(("acc", "replicas", "batch"), start=1):
        setattr(cols, name, C.cast(b + 4 * S * k, _abi.i32p))
    for k, name in enumerate(("cost", "value", "itl", "ttft", "rho", "max_rate"), start=4):
        setattr(cols, name, C.cast(b + 4 * S * k, _abi.f32p))
    torch.cuda.synchronize()  # the zero fill runs on torch's stream, the engine on its own
    return blk, cols


def grid_device(eng, grid, S):
    """wva_grid_solve_device on the resident fleet -> the winner block's bytes."""
    blk, cols = device_winners(S)
    eng.grid_solve_device(grid, cols)
    eng.synchronize()
    return blk.cpu().numpy().view(np.uint8).copy()


def same(got, want, what):
    if isinstance(got, np.ndarray):
        assert np.array_equal(got, want), what
    elif isinstance(got, dict):
        for k in want:
            assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), f"{what}: {k}"
    else:
        for k in ALLOC_FIELDS:
            assert np.array_equal(getattr(got, k).view(np.uint8), getattr(want, k).view(np.uint8)), f"{what}: {k}"


def check(engine, call, fresh_call, what):
    """call(engine) against fresh_call(a new handle), every returned array byte for byte."""
    got = call(engine)
    eng = Engine(0)
    try:
        want = fresh_call(eng)
    finally:
        eng.close()
    if not isinstance(got, tuple):
        got, want = (got,), (want,)
    for x, y in zip(got, want):
        if y is not None:
            same(x, y, what)


@pytest.mark.gpu
def test_interleaving_on_one_handle(engine):
    fleet = mixed_fleet(30, 3, 67, True)
    rpm = load_levels(fleet, 4, 29)
    grid = Grid([1, 4, 16, 33], np.arange(1, 13))
    S = fleet.n_servers

    solve = lambda e: e.solve(fleet)  # noqa: E731
    size_grid = lambda e: e.size_grid(fleet, [4, 16, 64], want_candidates=True)  # noqa: E731
    load_grid = lambda e: e.load_grid(fleet, rpm, want_candidates=True)  # noqa: E731
    grid_cells = lambda e: e.grid_solve(fleet, grid, want_cells=True)  # noqa: E731
    sweep = lambda e: e.sweep(fleet, 8)  # noqa: E731
    resolve = lambda e: e.resolve(want_candidates=True)  # noqa: E731
    device = lambda e: grid_device(e, grid, S)  # noqa: E731

    def uploaded(call):  # a resident call on a fresh handle: wva_upload first
        def run(e):
            e.upload(fleet)
            return call(e)
        return run

    def sequence(tag):
        check(engine, solve, solve, f"{tag}: solve")
        check(engine, size_grid, size_grid, f"{tag}: size grid")
        check(engine, load_grid, load_grid, f"{tag}: load grid")
        check(engine, grid_cells, grid_cells, f"{tag}: grid with cells")
        check(engine, sweep, sweep, f"{tag}: sweep")
        check(engine, grid_cells, grid_cells, f"{tag}: grid after a sweep, same lists")
        check(engine, sweep, sweep, f"{tag}: another sweep")
        check(engine, device, uploaded(device), f"{tag}: grid_solve_device after a sweep")
        check(engine, device, uploaded(device), f"{tag}: grid_solve_device, cached lists")
        check(engine, solve, solve, f"{tag}: solve at the end")

    sequence("first pass")
    fleet.srv_out_tokens[:] = np.maximum(1, fleet.srv_out_tokens // 3)
    engine.update_load(out_tokens=fleet.srv_out_tokens)
    check(engine, resolve, uploaded(resolve), "resolve after a token change")
    check(engine, device, uploaded(device), "grid_solve_device after a token change")
    sequence("after a token change")
    z = int(np.flatnonzero(fleet.srv_arrival_rpm == 0)[0])
    fleet.srv_arrival_rpm[z] = 42.0  # zero load -> load: a pair-class change
    engine.update_load(arrival_rpm=fleet.srv_arrival_rpm)
    check(engine, resolve, uploaded(resolve), "resolve after a pair-class change")
    check(engine, device, uploaded(device), "grid_solve_device after a pair-class change")
    sequence("after a pair-class change")


@pytest.mark.gpu
def test_cache_semantics_through_launch_count(engine):
    fleet = synth_fleet(30, 4, seed=71, zero_load_frac=0.2)  # at most 120 candidates: the warp path
    S = fleet.n_servers

    def launches(call):
        n0 = engine.launch_count
        call()
        engine.synchronize()
        return engine.launch_count - n0

    engine.upload(fleet)
    first = launches(lambda: engine.resolve())
    cached = launches(lambda: engine.resolve())
    assert cached == first - 1, "a second resolve reuses the tables"
    _, cols = device_winners(S)
    assert launches(lambda: engine.resolve_device(cols)) == cached, "resolve_device reuses the tables too"
    rpm = fleet.srv_arrival_rpm * np.float32(1.5)  # zero stays zero, positive stays positive
    engine.update_load(arrival_rpm=rpm)
    assert launches(lambda: engine.resolve()) == cached, "a load change with the same pair classes keeps the tables"
    out = fleet.srv_out_tokens.copy()
    out[out > 1] -= 1
    assert not np.array_equal(out, fleet.srv_out_tokens)
    engine.update_load(out_tokens=out)
    assert launches(lambda: engine.resolve()) == cached + 1, "a token change rebuilds the tables"

    grid = Grid([2, 8, 32], np.arange(1, 17))
    engine.upload(fleet)
    _, cols = device_winners(S)
    step = launches(lambda: engine.grid_solve_device(grid, cols))
    assert launches(lambda: engine.grid_solve_device(grid, cols)) == step, "the grid rebuilds its tables every call"
    engine.sweep(fleet, 8)
    engine.upload(fleet)
    assert launches(lambda: engine.grid_solve_device(grid, cols)) == step, "after a sweep and an upload"
    assert launches(lambda: engine.grid_solve_device(grid, cols)) == step, "after a sweep and an upload, cached"
