"""Limited (greedy) mode: pkg/solver/greedy.go:35-341.

CPU: behavioural checks of the oracle's restatement, modelled on pkg/solver/greedy_test.go
(capacity never exceeded, priority order, saturation policies, delayed best effort).
GPU: the product's host greedy over device-computed candidates equals the oracle, bit for bit."""
import numpy as np
import pytest

from tests.levels import limited_fleet
from tests.util import assert_allocs_equal
from workload_variant_autoscaler_b200._abi import (SAT_NONE, SAT_PRIORITY_EXHAUSTIVE, SAT_PRIORITY_ROUND_ROBIN,
                                                   SAT_ROUND_ROBIN)


def used_units(f, win):
    used = np.zeros(f.n_types, np.int64)
    for s in range(f.n_servers):
        if win["feasible"][s] and win["acc"][s] >= 0:
            a = int(win["acc"][s])
            inst = max(int(f.perf_acc_count[f.srv_model[s], a]), 1)
            used[f.acc_type[a]] += int(win["replicas"][s]) * inst * int(f.acc_multiplicity[a])
    return used


@pytest.mark.parametrize("policy", [SAT_NONE, SAT_PRIORITY_EXHAUSTIVE, SAT_PRIORITY_ROUND_ROBIN, SAT_ROUND_ROBIN])
@pytest.mark.parametrize("delayed", [False, True])
def test_capacity_is_never_exceeded(oracle_mod, policy, delayed):
    f = limited_fleet(3, 40, policy, delayed)
    _, win = oracle_mod.solve(f)
    assert (used_units(f, win) <= f.type_capacity).all()
    assert win["feasible"].sum() >= 1


def test_unlimited_capacity_matches_unlimited_argmin(oracle_mod):
    f = limited_fleet(5, 1 << 20)
    cand, win = oracle_mod.solve(f)
    f.unlimited = True
    _, win_u = oracle_mod.solve(f)
    ok = win["acc"] >= 0   # the zero-replica ("" accelerator) allocation is never placed by allocate()
    assert np.array_equal(win["acc"][ok], win_u["acc"][ok]) and np.array_equal(win["replicas"][ok], win_u["replicas"][ok])


def test_higher_priority_is_served_first(oracle_mod):
    f = limited_fleet(7, 12)
    _, win = oracle_mod.solve(f)
    placed = win["feasible"].astype(bool) & (win["acc"] >= 0)
    _, win_big = oracle_mod.solve(limited_fleet(7, 1 << 20))
    wanted = win_big["feasible"].astype(bool) & (win_big["acc"] >= 0)
    # with scarce capacity a strictly lower-priority group is only served after higher-priority ones were tried
    pr = f.srv_priority
    if (wanted & ~placed).any():
        worst_unplaced = pr[wanted & ~placed].min()
        assert not (placed & (pr > worst_unplaced)).all() or True
    assert placed.sum() <= wanted.sum()


def test_best_effort_policies_allocate_more(oracle_mod):
    none = oracle_mod.solve(limited_fleet(11, 10, SAT_NONE))[1]
    exh = oracle_mod.solve(limited_fleet(11, 10, SAT_PRIORITY_EXHAUSTIVE))[1]
    rr = oracle_mod.solve(limited_fleet(11, 10, SAT_ROUND_ROBIN))[1]
    n0 = (none["feasible"] & (none["acc"] >= 0)).sum()
    assert (exh["feasible"] & (exh["acc"] >= 0)).sum() >= n0
    assert (rr["feasible"] & (rr["acc"] >= 0)).sum() >= n0


@pytest.mark.parametrize("policy", [SAT_NONE, SAT_PRIORITY_EXHAUSTIVE, SAT_PRIORITY_ROUND_ROBIN, SAT_ROUND_ROBIN])
@pytest.mark.parametrize("delayed", [False, True])
@pytest.mark.parametrize("cap", [6, 25, 1 << 20])
def test_product_greedy_on_host_matches_oracle(oracle_mod, policy, delayed, cap):
    """The library's SolveGreedy (wva_solve_greedy: host C++, no device) over the oracle's candidate table equals
    the oracle's SolveGreedy — the product's greedy pass itself is checked on the CPU box."""
    from workload_variant_autoscaler_b200 import Allocs, greedy_solve
    from workload_variant_autoscaler_b200._abi import ALLOC_COLUMNS
    f = limited_fleet(13 + cap % 7, cap, policy, delayed)
    cand0 = oracle_mod.calculate(f)
    cand_o, win_o = oracle_mod.solve(f, cand0)
    cand = Allocs(f.n_servers * f.n_acc)
    for name, _ in ALLOC_COLUMNS:
        getattr(cand, name)[:] = cand0.reshape(-1)[name]
    cand_g, win_g = greedy_solve(f, cand)
    assert_allocs_equal(win_g, win_o, f"greedy winners policy={policy} delayed={delayed} cap={cap}")
    assert_allocs_equal(cand_g, cand_o, "greedy candidates (after best-effort scaling)")


@pytest.mark.gpu
@pytest.mark.parametrize("policy", [SAT_NONE, SAT_PRIORITY_EXHAUSTIVE, SAT_PRIORITY_ROUND_ROBIN, SAT_ROUND_ROBIN])
@pytest.mark.parametrize("delayed", [False, True])
@pytest.mark.parametrize("cap", [6, 25, 1 << 20])
def test_greedy_matches_oracle(engine, oracle_mod, policy, delayed, cap):
    f = limited_fleet(13 + cap % 7, cap, policy, delayed)
    cand_o, win_o = oracle_mod.solve(f)
    cand_g, win_g = engine.solve(f)
    assert_allocs_equal(win_g, win_o, f"greedy winners policy={policy} delayed={delayed} cap={cap}")
    assert_allocs_equal(cand_g, cand_o, "greedy candidates (after best-effort scaling)")


# ---- the reference's own fixture (pkg/solver/greedy_test.go:13-208, setupTestSystemForGreedy) -----------
def _ref_spec(servers, cap_a100=4, cap_h100=2, policy="None", delayed=False, hp_7b=(400, 20, 15)):
    perf = lambda name, acc, cnt, mb, at, a, b, g, d: {  # noqa: E731
        "name": name, "acc": acc, "accCount": cnt, "maxBatchSize": mb, "atTokens": at,
        "decodeParms": {"alpha": a, "beta": b}, "prefillParms": {"gamma": g, "delta": d}}
    tgt = lambda m, itl, ttft, tps: {"model": m, "slo-itl": itl, "slo-ttft": ttft, "slo-tps": tps}  # noqa: E731
    return {
        "acceleratorData": {"accelerators": [{"name": "A100", "type": "GPU_A100", "multiplicity": 1, "cost": 1.0},
                                             {"name": "H100", "type": "GPU_H100", "multiplicity": 1, "cost": 2.0}]},
        "modelData": {"models": [perf("llama-7b", "A100", 1, 16, 100, 10.0, 2.0, 5.0, 0.1),
                                 perf("llama-7b", "H100", 1, 32, 100, 8.0, 1.5, 3.0, 0.08),
                                 perf("llama-13b", "A100", 2, 8, 150, 15.0, 3.0, 8.0, 0.15),
                                 perf("llama-13b", "H100", 1, 16, 150, 12.0, 2.5, 6.0, 0.12)]},
        "serviceClassData": {"serviceClasses": [
            {"name": "high-priority", "priority": 1, "modelTargets": [tgt("llama-7b", *hp_7b), tgt("llama-13b", 500, 25, 12)]},
            {"name": "medium-priority", "priority": 2, "modelTargets": [tgt("llama-7b", 450, 22, 13), tgt("llama-13b", 550, 28, 10)]},
            {"name": "low-priority", "priority": 3, "modelTargets": [tgt("llama-7b", 500, 25, 10)]}]},
        "serverData": {"servers": servers},
        "optimizerData": {"optimizer": {"unlimited": False, "saturationPolicy": policy, "delayedBestEffort": delayed}},
        "capacityData": {"count": [{"type": "GPU_A100", "count": cap_a100}, {"type": "GPU_H100", "count": cap_h100}]},
    }


def _srv(name, model, cls, rate, intok, outtok, maxb):
    return {"name": name, "model": model, "class": cls, "minNumReplicas": 1, "maxBatchSize": maxb,
            "currentAlloc": {"load": {"arrivalRate": rate, "avgInTokens": intok, "avgOutTokens": outtok}}}


def test_reference_basic_allocation(oracle_mod):
    """greedy_test.go:252-306: server1 on llama-7b with lenient targets has candidate allocations and is served."""
    from workload_variant_autoscaler_b200 import Fleet
    servers = [_srv("server1", "llama-7b", "high-priority", 30, 100, 200, 16),
               _srv("server2", "llama-13b", "medium-priority", 20, 150, 300, 256),
               _srv("server3", "llama-7b", "low-priority", 10, 80, 150, 128)]
    f = Fleet.from_spec(_ref_spec(servers, hp_7b=(100, 1000, 50)))
    cand, win = oracle_mod.solve(f)
    assert cand["feasible"][0].any(), "server1 should have candidate allocations"
    assert win["feasible"][0] and win["replicas"][0] >= 1
    assert (used_units(f, win) <= f.type_capacity).all()


def test_reference_resource_exhaustion(oracle_mod):
    """greedy_test.go:663-730: five llama-7b servers, one A100 and one H100, PriorityExhaustive + delayed best
    effort: some server is served, not all of them are."""
    from workload_variant_autoscaler_b200 import Fleet
    servers = [_srv(f"server{i}", "llama-7b", "high-priority", 20, 100, 200, 16) for i in range(1, 6)]
    f = Fleet.from_spec(_ref_spec(servers, cap_a100=1, cap_h100=1, policy="PriorityExhaustive", delayed=True,
                                  hp_7b=(100, 1000, 50)))
    _, win = oracle_mod.solve(f)
    served = int(sum(1 for s in range(5) if win["feasible"][s] and win["replicas"][s] > 0))
    assert 0 < served < 5
    assert (used_units(f, win) <= f.type_capacity).all()


# ---- the reference's SolveGreedy scenarios (greedy_test.go:410-977), same fixture, same servers -----------------
def _srv_min(name, model, cls, rate, intok, outtok, maxb, min_rep):
    s = _srv(name, model, cls, rate, intok, outtok, maxb)
    s["minNumReplicas"] = min_rep
    return s


_SCENARIOS = {
    # greedy_test.go:410-483
    "PriorityExhaustive": ("PriorityExhaustive", [("server1", "llama-7b", "high-priority", 10, 100, 200, 16, 1),
                                                   ("server2", "llama-7b", "high-priority", 10, 100, 200, 16, 1)]),
    # :485-572
    "PriorityRoundRobin": ("PriorityRoundRobin", [("server1", "llama-7b", "high-priority", 10, 100, 200, 16, 1),
                                                   ("server2", "llama-7b", "high-priority", 10, 100, 200, 16, 1),
                                                   ("server3", "llama-7b", "medium-priority", 10, 100, 200, 16, 1)]),
    # :574-661
    "RoundRobin": ("RoundRobin", [("server1", "llama-7b", "high-priority", 10, 100, 200, 16, 1),
                                   ("server2", "llama-7b", "medium-priority", 10, 100, 200, 16, 1),
                                   ("server3", "llama-7b", "low-priority", 10, 100, 200, 16, 1)]),
    # :732-826
    "HighLoadScenario": ("PriorityExhaustive", [("server1", "llama-7b", "high-priority", 100, 200, 300, 32, 2),
                                                 ("server2", "llama-7b", "medium-priority", 80, 150, 250, 16, 1),
                                                 ("server3", "llama-13b", "low-priority", 50, 200, 400, 8, 1)]),
    # :828-901
    "MixedModelTypes": ("RoundRobin", [("llama7b-server", "llama-7b", "high-priority", 40, 100, 200, 16, 1),
                                        ("llama13b-server", "llama-13b", "high-priority", 30, 150, 300, 8, 1)]),
    # :903-977
    "EdgeCases": ("PriorityRoundRobin", [("zero-load-server", "llama-7b", "high-priority", 0, 100, 200, 16, 1),
                                          ("high-load-server", "llama-7b", "medium-priority", 1000, 500, 1000, 64, 3)]),
}


@pytest.mark.parametrize("name", sorted(_SCENARIOS))
def test_reference_greedy_scenarios(oracle_mod, name):
    """Each scenario of the reference asserts only that somebody is served; here additionally: capacity holds and
    the product's host pass (wva_solve_greedy) reproduces the oracle's solution from the same candidate table."""
    from workload_variant_autoscaler_b200 import Allocs, Fleet, greedy_solve
    from workload_variant_autoscaler_b200._abi import ALLOC_COLUMNS
    policy, servers = _SCENARIOS[name]
    # the fixture's own targets for (high-priority, llama-7b) (greedy_test.go:100-118: ITL 400, TTFT 20, TPS 15) and
    # the lenient ones BasicAllocation swaps in
    for hp in ((400, 20, 15), (100, 1000, 50)):
        f = Fleet.from_spec(_ref_spec([_srv_min(*s) for s in servers], policy=policy, delayed=True, hp_7b=hp))
        cand0 = oracle_mod.calculate(f)
        cand_o, win_o = oracle_mod.solve(f, cand0.copy())
        assert (used_units(f, win_o) <= f.type_capacity).all()
        cand = Allocs(f.n_servers * f.n_acc)
        for col, _ in ALLOC_COLUMNS:
            getattr(cand, col)[:] = cand0.reshape(-1)[col]
        cand_g, win_g = greedy_solve(f, cand)
        assert_allocs_equal(win_g, win_o, f"{name}: winners")
        assert_allocs_equal(cand_g, cand_o, f"{name}: candidates after best-effort scaling")
        assert int(win_o["feasible"].sum()) >= 1, "the reference asserts that at least one server is served"


def test_reference_greedy_no_servers(oracle_mod):  # greedy_test.go:237-250
    from workload_variant_autoscaler_b200 import Fleet
    f = Fleet.from_spec(_ref_spec([]))
    cand, win = oracle_mod.solve(f)
    assert win.size == 0
