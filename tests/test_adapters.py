"""Input packer / output path (SURVEY.md 8f ranks 1 and 3): internal/utils/utils.go adapters restated on dicts.

The fixture is the reference's own (test/utils/unitutils.go:64-115 ConfigMaps, internal/optimizer/optimizer_test.go
VariantAutoscalings): three variants of meta/llama0-70b on A100, no load -> every variant is scaled to
minNumReplicas on its current accelerator (optimizer_test.go "scaled to %d without load")."""
import numpy as np
import pytest

from tests.levels import ACC_CM, SC_CM, _va
from workload_variant_autoscaler_b200 import Fleet, adapters
from workload_variant_autoscaler_b200.adapters import go_parse_float32

def test_parse_float32_is_go_strconv():
    f32 = np.float32
    assert go_parse_float32("40.00") == (f32(40.0), None)
    assert go_parse_float32("20.28")[0] == f32(20.28) and go_parse_float32("0.72")[0] == f32(0.72)
    assert go_parse_float32("1e-3")[0] == f32(1e-3) and go_parse_float32(".5")[0] == f32(0.5) and go_parse_float32("5.")[0] == f32(5)
    assert go_parse_float32("0x1p-2") == (f32(0.25), None)
    # a literal just above the midpoint of 1 and 1+2^-23: float64 rounds it ONTO the midpoint, and a second
    # rounding (ties to even) would give 1.0; ParseFloat(...,32) rounds once and gives the upper neighbour
    s = "1.000000059604644775390625000000000001"
    assert float(s) == 1.0 + 2.0 ** -24 and np.float32(float(s)) == f32(1.0)
    assert go_parse_float32(s)[0].view(np.uint32) == np.uint32(0x3F800001)
    assert go_parse_float32("1.0000000596046447753906250")[0] == f32(1.0)          # the exact tie goes to even
    v, err = go_parse_float32("1e39")
    assert np.isinf(v) and err == "range"
    assert go_parse_float32("3.4028235e38") == (np.finfo(np.float32).max, None)
    for bad in ("", "abc", "1e", "0x1", "+nan", "1.2.3", "e5", "1.5\n", " 1", "\u0661\u0662", "1_", "_1", "1__0", "1._5",
                "1_.5"):
        assert go_parse_float32(bad) == (f32(0.0), "syntax"), bad
    # Go's underscoreOK: underscores may separate digits (and follow a base prefix)
    assert go_parse_float32("1_000") == (f32(1000.0), None)
    assert go_parse_float32("0x_1p-2") == (f32(0.25), None) and go_parse_float32("1e1_0") == (f32(1e10), None)
    assert np.isinf(go_parse_float32("+Inf")[0]) and go_parse_float32("-infinity")[0] == f32("-inf")
    assert np.isnan(go_parse_float32("NaN")[0])
    assert np.signbit(go_parse_float32("-0")[0])


def test_parse_float32_huge_exponents_are_decided_in_linear_time():
    import time
    f32 = np.float32
    t0 = time.perf_counter()
    v, err = go_parse_float32("1e999999999")
    assert np.isposinf(v) and err == "range"
    v, err = go_parse_float32("-1e999999999999999999999")
    assert np.isneginf(v) and err == "range"
    v, err = go_parse_float32("1e-9999999")
    assert v == f32(0.0) and not np.signbit(v) and err is None
    v, err = go_parse_float32("-0.0000001e-999999999")
    assert v == f32(0.0) and np.signbit(v) and err is None
    assert go_parse_float32("0x1p-200000") == (f32(0.0), None)
    assert go_parse_float32("0x1p+99999999999")[1] == "range"
    assert go_parse_float32("0e999999999") == (f32(0.0), None)            # zero mantissa: exponent is irrelevant
    assert time.perf_counter() - t0 < 0.5
    # the boundaries themselves still round exactly
    assert go_parse_float32("1e-45")[0].view(np.uint32) == np.uint32(1) and go_parse_float32("1e-46")[0] == f32(0.0)
    assert go_parse_float32("0x1p-149")[0].view(np.uint32) == np.uint32(1)
    assert go_parse_float32("0x1.fffffep127") == (np.finfo(np.float32).max, None)
    assert go_parse_float32("0x1p128")[1] == "range" and go_parse_float32("3.4028236e38")[1] == "range"


def test_create_system_data_matches_reference_fixture():
    sd = adapters.create_system_data(ACC_CM, SC_CM)
    spec = sd["spec"]
    accs = {a["name"]: a for a in spec["acceleratorData"]["accelerators"]}
    assert {n: (a["type"], a["cost"], a["multiplicity"]) for n, a in accs.items()} == {
        "A100": ("NVIDIA-A100-PCIE-80GB", 40.0, 1), "MI300X": ("AMD-MI300X-192GB", 65.0, 1), "G2": ("Intel-Gaudi-2-96GB", 23.0, 1)}
    classes = {c["name"]: c for c in spec["serviceClassData"]["serviceClasses"]}
    assert classes["Premium"]["priority"] == 1 and classes["Freemium"]["priority"] == 10
    assert {"model": "meta/llama0-70b", "slo-itl": 80.0, "slo-ttft": 500.0} in classes["Premium"]["modelTargets"]
    assert spec["optimizerData"]["optimizer"] == {"unlimited": True} and spec["capacityData"]["count"] == []
    assert spec["modelData"]["models"] == [] and spec["serverData"]["servers"] == []
    # unparsable entries are skipped, not fatal (utils.go:127-130, :147-150)
    sd2 = adapters.create_system_data({**ACC_CM, "BAD": {"device": "x", "cost": "forty"}},
                                      {**SC_CM, "broken.yaml": "name: [unclosed", "float.yaml": "name: F\npriority: 2\ndata:\n  - model: m\n    slo-tpot: 1.5\n    slo-ttft: 2"})
    assert sorted(a["name"] for a in sd2["spec"]["acceleratorData"]["accelerators"]) == ["A100", "G2", "MI300X"]
    assert sorted(c["name"] for c in sd2["spec"]["serviceClassData"]["serviceClasses"]) == ["Freemium", "Premium"]
    entry, cls = adapters.find_model_slo(SC_CM, "meta/llama0-7b")
    assert (entry["slo-tpot"], entry["slo-ttft"], cls) == (150, 1500, "Freemium")
    with pytest.raises(adapters.AdapterError):
        adapters.find_model_slo(SC_CM, "nobody/nothing")


def test_profile_and_server_adapters():
    sd = adapters.create_system_data(ACC_CM, SC_CM)
    va = _va(1, arrival="123.9")
    adapters.add_model_accelerator_profile_to_system_data(sd, "meta/llama0-70b", va["spec"]["modelProfile"]["accelerators"][0])
    pd = sd["spec"]["modelData"]["models"][0]
    assert (pd["name"], pd["acc"], pd["accCount"], pd["maxBatchSize"]) == ("meta/llama0-70b", "A100", 1, 4)
    assert np.float32(pd["decodeParms"]["alpha"]) == np.float32(20.28) and pd["prefillParms"] == {"gamma": 0.0, "delta": 0.0}
    with pytest.raises(adapters.AdapterError):  # "length of decodeParms should be 2"
        adapters.add_model_accelerator_profile_to_system_data(sd, "m", {"acc": "A100", "perfParms": {"decodeParms": {"alpha": "1"}, "prefillParms": {"gamma": "0", "delta": "0"}}})
    with pytest.raises(adapters.AdapterError):  # ParseFloat error is returned
        adapters.add_model_accelerator_profile_to_system_data(sd, "m", {"acc": "A100", "perfParms": {"decodeParms": {"alpha": "x", "beta": "1"}, "prefillParms": {"gamma": "0", "delta": "0"}}})

    va["status"]["currentAlloc"]["load"].update(avgInputTokens="512.7", avgOutputTokens="NaN")
    va["status"]["currentAlloc"]["itlAverage"] = "+Inf"
    adapters.add_server_info_to_system_data(sd, va, "Premium", environ={})
    sv = sd["spec"]["serverData"]["servers"][0]
    assert sv["name"] == "test-variantautoscaling-1:default" and sv["class"] == "Premium" and sv["keepAccelerator"] is True
    assert sv["minNumReplicas"] == 1 and sv["maxBatchSize"] == 4
    cur = sv["currentAlloc"]
    assert cur["load"] == {"arrivalRate": float(np.float32(123.9)), "avgInTokens": 512, "avgOutTokens": 0}   # int() truncates; NaN -> 0
    assert cur["itlAverage"] == 0.0 and cur["cost"] == 40.0 and cur["accelerator"] == "A100"                   # Inf -> 0
    # scale to zero and a label that matches no profile: no maxBatchSize key, minNumReplicas 0
    va2 = _va(2)
    va2["metadata"]["labels"]["inference.optimization/acceleratorName"] = "H100"
    adapters.add_server_info_to_system_data(sd, va2, "Premium", environ={"WVA_SCALE_TO_ZERO": "true"})
    sv2 = sd["spec"]["serverData"]["servers"][1]
    assert sv2["minNumReplicas"] == 0 and "maxBatchSize" not in sv2


@pytest.mark.parametrize("scale_to_zero", [False, True])
def test_reference_flow_without_load_scales_to_min_replicas(oracle_mod, scale_to_zero):
    """optimizer_test.go:230-330 with the optimizer path = the oracle: ConfigMaps + 3 VariantAutoscalings ->
    SystemData -> fleet -> solve -> GenerateSolution -> CreateOptimizedAlloc."""
    env = {"WVA_SCALE_TO_ZERO": "true"} if scale_to_zero else {}
    sd = adapters.create_system_data(ACC_CM, SC_CM)
    vas = [_va(i) for i in (1, 2, 3)]
    for va in vas:
        _, cls = adapters.find_model_slo(SC_CM, va["spec"]["modelID"])
        for prof in va["spec"]["modelProfile"]["accelerators"]:
            adapters.add_model_accelerator_profile_to_system_data(sd, va["spec"]["modelID"], prof)
        adapters.add_server_info_to_system_data(sd, va, cls, environ=env)
    fleet = Fleet.from_spec(sd["spec"])
    assert fleet.unlimited and fleet.n_servers == 3 and fleet.n_acc == 3
    _, win = oracle_mod.solve(fleet)
    solution = adapters.generate_solution(fleet, win)
    want = 0 if scale_to_zero else 1
    for va in vas:
        opt = adapters.create_optimized_alloc(va["metadata"]["name"], va["metadata"]["namespace"], solution)
        # zeroLoadAllocation with minNumReplicas == 0 carries no accelerator (allocation.go:262-267)
        assert opt["accelerator"] == ("" if scale_to_zero else "A100") and opt["numReplicas"] == want and opt["lastRunTime"]
        m = adapters.replica_metrics(va["status"]["currentAlloc"]["numReplicas"], opt["numReplicas"])
        assert m["desired_ratio"] == float(want)
    with pytest.raises(adapters.AdapterError):
        adapters.create_optimized_alloc("missing", "default", solution)
    assert adapters.replica_metrics(0, 3)["desired_ratio"] == 3.0 and adapters.replica_metrics(2, 3)["desired_ratio"] == 1.5


def test_generate_solution_like_reference_system_test(oracle_mod):
    """pkg/core/system_test.go:1413-1519 (TestSystem_GenerateSolution): one A100, one model, one server under
    load -> the solution holds the server with an accelerator, a positive replica count and its load."""
    spec = {
        "acceleratorData": {"accelerators": [{"name": "A100", "type": "GPU_A100", "multiplicity": 1, "cost": 1.0}]},
        "modelData": {"models": [{"name": "test-model", "acc": "A100", "accCount": 1, "maxBatchSize": 16, "atTokens": 100,
                                  "decodeParms": {"alpha": 10.0, "beta": 2.0}, "prefillParms": {"gamma": 5.0, "delta": 0.1}}]},
        "serviceClassData": {"serviceClasses": [{"name": "default", "priority": 1, "modelTargets": [
            {"model": "test-model", "slo-itl": 100, "slo-ttft": 1000, "slo-tps": 50}]}]},
        "serverData": {"servers": [{"name": "test-server", "model": "test-model", "class": "default", "minNumReplicas": 1,
                                    "maxBatchSize": 16, "currentAlloc": {"accelerator": "A100", "numReplicas": 2, "load": {
                                        "arrivalRate": 30, "avgInTokens": 100, "avgOutTokens": 200}}}]},
        "optimizerData": {"optimizer": {"unlimited": True}},
        "capacityData": {"count": []},
    }
    fleet = Fleet.from_spec(spec)
    _, win = oracle_mod.solve(fleet)
    sol = adapters.generate_solution(fleet, win)["spec"]
    assert "test-server" in sol
    alloc = sol["test-server"]
    assert alloc["accelerator"] == "A100" and alloc["numReplicas"] > 0 and alloc["maxBatch"] == 16
    assert alloc["load"] == {"arrivalRate": 30.0, "avgInTokens": 100, "avgOutTokens": 200}
    assert alloc["cost"] == float(np.float32(1.0) * np.float32(alloc["numReplicas"]))   # accCost * instances * replicas


def test_parse_float32_round_trips_random_float32s():
    """Every finite float32 prints (shortest repr and 60 significant digits) to a literal that parses back to
    itself; the literal one float64-ulp above a float32 midpoint goes to the upper neighbour."""
    rng = np.random.default_rng(99)
    bits = rng.integers(0, 2 ** 32, 4000, dtype=np.uint64).astype(np.uint32)
    vals = bits.view(np.float32)
    vals = vals[np.isfinite(vals)]
    for v in vals[:3000]:
        for lit in (repr(float(v)), "%.60g" % float(v), "%.9e" % float(v)):
            got, err = go_parse_float32(lit)
            assert err is None and got.view(np.uint32) == v.view(np.uint32), (lit, got, v)
    for v in vals[:300]:
        if v <= 0 or not np.isfinite(np.nextafter(v, np.float32(np.inf))):
            continue
        up = np.nextafter(v, np.float32(np.inf))
        mid = (float(v) + float(up)) / 2.0                      # exact in float64
        above = np.nextafter(mid, np.inf)                       # one float64 ulp above the midpoint
        got, _ = go_parse_float32("%.60g" % above)
        assert got == up, (v, up, got)
        got, _ = go_parse_float32("%.60g" % np.nextafter(mid, -np.inf))
        assert got == v
