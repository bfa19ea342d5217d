"""System.AllocateByType (pkg/core/system.go:271-300) and CreateAllocationDiff (pkg/core/allocation.go:353-380,
collected per server by pkg/solver/solver.go:51-58).

CPU: the oracle's restatement on the reference's own cases (allocation_test.go TestAllocationDiff_Content /
_NilHandling, system_test.go TestSystem_AllocateByType) and on hand-computed totals.
GPU: Engine.summarize() (summary_kernel, or the host loops after a greedy solve) equals the oracle bit for bit."""
import numpy as np
import pytest

from tests.grid_cases import check_summary
from tests.levels import limited_fleet
from workload_variant_autoscaler_b200 import Grid, synth_fleet
from workload_variant_autoscaler_b200._abi import ACC_ABSENT, ACC_NONE


def _winners(oracle_mod, rows):
    w = np.zeros(len(rows), oracle_mod.ALLOC_DTYPE)
    for i, (feas, acc, rep, cost) in enumerate(rows):
        w[i]["feasible"], w[i]["acc"], w[i]["replicas"], w[i]["cost"] = feas, acc, rep, cost
    return w


def test_allocation_diff_content_like_reference(oracle_mod):
    # allocation_test.go:462-492: (gpu-a, 2, 100) -> (gpu-b, 3, 150): costDiff 50
    f = synth_fleet(3, 2, seed=1)
    f.srv_cur_acc[:] = [0, 1, ACC_NONE]
    f.srv_cur_replicas[:] = [2, 1, 0]
    f.srv_cur_cost[:] = [100.0, 40.0, 0.0]
    win = _winners(oracle_mod, [(1, 1, 3, 150.0), (0, -1, 0, 0.0), (1, ACC_NONE, 0, 0.0)])
    d = oracle_mod.allocation_diffs(f, win)
    assert (d["old_acc"][0], d["new_acc"][0], d["old_replicas"][0], d["new_replicas"][0], d["cost_diff"][0]) == \
        (0, 1, 2, 3, np.float32(50.0))
    # allocation_test.go:523-559 "allocation to nil": new side reads "none", 0 replicas, cost 0
    assert (d["new_acc"][1], d["new_replicas"][1], d["cost_diff"][1]) == (ACC_ABSENT, 0, np.float32(-40.0))
    # a zero-replica allocation is an allocation with accelerator "" (allocation.go:259-288), not "none"
    assert (d["old_acc"][2], d["new_acc"][2], d["cost_diff"][2]) == (ACC_NONE, ACC_NONE, np.float32(0.0))


def test_allocate_by_type_hand_computed(oracle_mod):
    f = synth_fleet(5, 3, seed=2)
    f.acc_type[:] = [0, 1, 0]            # accelerators 0 and 2 share a type
    f.type_capacity[:] = [4, 9, 0]       # system_test.go:1404: limit = capacity of the type
    f.acc_multiplicity[:] = [1, 2, 4]
    f.perf_acc_count[:, :] = [[1, 2, 0]] * f.n_models  # AccCount 0 -> 1 instance (model.go:52-55)
    win = _winners(oracle_mod, [(1, 0, 3, 10.5), (1, 2, 2, 0.25), (1, 1, 5, 7.0), (0, -1, 0, 0.0),
                                (1, ACC_NONE, 0, 0.0)])
    t = oracle_mod.allocate_by_type(f, win)
    assert t["present"].tolist() == [1, 1, 0]
    assert t["count"].tolist() == [3 * 1 * 1 + 2 * 1 * 4, 5 * 2 * 2, 0]
    assert t["limit"].tolist() == [4, 9, 0]
    assert t["cost"][0] == np.float32(np.float32(10.5) + np.float32(0.25)) and t["cost"][1] == np.float32(7.0)
    # float32 accumulation in ascending server index
    f2 = synth_fleet(4, 1, seed=3)
    f2.acc_type[:] = [0]
    f2.type_capacity[:] = [1]
    w2 = _winners(oracle_mod, [(1, 0, 1, 1e8), (1, 0, 1, 1.0), (1, 0, 1, -1e8), (1, 0, 1, 1.0)])
    want = np.float32(np.float32(np.float32(np.float32(1e8) + np.float32(1.0)) + np.float32(-1e8)) + np.float32(1.0))
    assert oracle_mod.allocate_by_type(f2, w2)["cost"][0] == want == np.float32(1.0)


@pytest.mark.gpu
def test_summary_after_unlimited_solve(engine, oracle_mod):
    f = synth_fleet(1500, 5, seed=31, max_batch_choices=(2, 4, 8, 16), zero_load_frac=0.1)
    f.acc_type[:] = [0, 1, 0, 2, 1]
    f.type_capacity = np.array([7, 0, 100], np.int32)
    f.acc_multiplicity[:] = [1, 2, 1, 4, 1]
    f.srv_min_replicas[::7] = 0
    f.srv_has_target[5] = 0            # a server without any allocation ("none")
    _, win_o = oracle_mod.solve(f)
    engine.solve(f)
    t, d = check_summary(engine, oracle_mod, f, win_o)
    assert t["present"].sum() >= 2 and (d["new_acc"] == ACC_ABSENT).sum() >= 1 and (d["new_acc"] == ACC_NONE).sum() >= 1


@pytest.mark.gpu
def test_summary_after_greedy_solve(engine, oracle_mod):
    from workload_variant_autoscaler_b200._abi import SAT_PRIORITY_ROUND_ROBIN
    f = limited_fleet(17, 9, SAT_PRIORITY_ROUND_ROBIN, delayed=True)
    _, win_o = oracle_mod.solve(f)
    engine.solve(f)
    t, _ = check_summary(engine, oracle_mod, f, win_o)
    assert (t["count"] <= t["limit"]).all()


@pytest.mark.gpu
def test_summary_after_grid_solve_and_state_errors(engine, oracle_mod):
    from workload_variant_autoscaler_b200 import WvaError
    f = synth_fleet(9, 3, seed=37, max_batch_choices=(4, 8))
    grid = Grid([1, 2, 4, 8], [1, 2, 3, 4, 6, 8])
    _, win_o = oracle_mod.grid_solve(f, grid, want_cells=False)
    engine.grid_solve(f, grid)
    check_summary(engine, oracle_mod, f, win_o)
    engine.upload(f)                   # a new upload invalidates the previous solution
    with pytest.raises(WvaError):
        engine.summarize(f.n_types)
