"""MM1KModel (closed form, pkg/analyzer/mm1kmodel.go): oracle restatement incl. Go's math.Pow, and the device
function behind wva_mm1k_solve bit for bit against it."""
import math

import numpy as np
import pytest
from tests.util import assert_f32_bits_equal



def test_go_pow_matches_libm_to_the_accuracy_of_binary_powering(oracle_mod):
    rng = np.random.default_rng(11)
    # exact cases
    assert oracle_mod.go_pow_uint(0.5, 10) == 2.0 ** -10
    assert oracle_mod.go_pow_uint(2.0, 1023) == 2.0 ** 1023
    assert oracle_mod.go_pow_uint(3.0, 0) == 1.0 and oracle_mod.go_pow_uint(1.0, 12345) == 1.0
    assert oracle_mod.go_pow_uint(0.0, 5) == 0.0 and oracle_mod.go_pow_uint(7.25, 1) == 7.25
    assert math.isnan(oracle_mod.go_pow_uint(float("nan"), 3))
    assert oracle_mod.go_pow_uint(0.5, 1074) == 2.0 ** -1074 and oracle_mod.go_pow_uint(0.5, 1075) == 0.0  # denormal edge
    assert oracle_mod.go_pow_uint(2.0, 1024) == math.inf
    # binary powering loses about one bit per squaring: within 2^(log2 n + 1) ulp of the correctly rounded power
    for _ in range(20000):
        x = float(rng.uniform(0.01, 3.0))
        n = int(rng.integers(0, 3000))
        a = oracle_mod.go_pow_uint(x, n)
        try:
            b = math.pow(x, n)
        except OverflowError:
            b = math.inf
        if b == 0.0 or math.isinf(b) or b < 1e-300:
            continue
        assert abs(a - b) <= 2.0 ** (math.ceil(math.log2(max(n, 2))) + 1) * math.ulp(b), (x, n, a, b)


def test_mm1k_closed_form_against_textbook_formulas(oracle_mod):  # mm1kmodel.go:51-92
    for K, lam, mu in ((10, 1.0, 2.0), (3, 1.5, 2.0), (50, 4.0, 5.0), (8, 2.0, 2.0), (20, 3.0, 1.0)):
        st = oracle_mod.mm1k_solve([K], [lam], [mu])
        rho = lam / mu
        if lam == mu:
            p = np.full(K + 1, 1.0 / (K + 1))
        else:
            p = (1 - rho) / (1 - rho ** (K + 1)) * rho ** np.arange(K + 1)
        L = float((np.arange(K + 1) * p).sum())
        thr = lam * (1 - p[K])
        assert st["is_valid"][0] == 1
        assert abs(st["sum_p"][0] - 1.0) < 1e-12
        assert st["avg_num_in_system"][0] == pytest.approx(L, rel=1e-6)
        assert st["throughput"][0] == pytest.approx(thr, rel=1e-6)
        assert st["avg_resp_time"][0] == pytest.approx(L / thr, rel=1e-6)  # Little's law
        assert st["avg_serv_time"][0] == pytest.approx(1 / mu, rel=1e-6)


def _cases():
    rng = np.random.default_rng(5)
    n = 4000
    K = rng.integers(0, 600, n).astype(np.int32)
    mu = rng.uniform(0.05, 20.0, n).astype(np.float32)
    lam = (mu * rng.uniform(0.0, 3.0, n)).astype(np.float32)
    # the reference's validity table (queuemodel_test.go:9-104) and the edges around it
    extra = [(10, 1.0, 2.0), (10, 0.0, 2.0), (10, -1.0, 2.0), (10, 1.0, 0.0), (10, 1.0, -1.0), (10, 9.9, 1.0),
             (10, 11.0, 1.0), (10, 10.0, 1.0), (3, 2.0, 2.0), (0, 0.0, 1.0), (1, 0.5, 1.0), (2816, 0.999, 1.0),
             (2816, 1.001, 1.0), (2816, 0.1, 1.0), (5, float("nan"), 1.0), (5, 1.0, float("inf"))]
    K = np.concatenate([K, np.array([e[0] for e in extra], np.int32)])
    lam = np.concatenate([lam, np.array([e[1] for e in extra], np.float32)])
    mu = np.concatenate([mu, np.array([e[2] for e in extra], np.float32)])
    lam[:200] = mu[:200]  # rho == 1 exactly
    K[200:600] = rng.integers(0, 3, 400)  # small K: rho >= K makes the model invalid (queuemodel.go:31)
    lam[600:700] = -lam[600:700]
    return K, lam, mu


@pytest.mark.gpu
def test_mm1k_device_function_bit_exact(engine, oracle_mod):
    K, lam, mu = _cases()
    got = engine.mm1k_solve(K, lam, mu)
    want = oracle_mod.mm1k_solve(K, lam, mu)
    assert (got["is_valid"] == want["is_valid"]).all()
    assert got["is_valid"].sum() > 1000 and (got["is_valid"] == 0).sum() > 100
    for name in ("rho", "avg_num_in_system", "throughput", "avg_resp_time", "avg_serv_time", "avg_wait_time",
                 "avg_queue_length"):
        assert_f32_bits_equal(got[name], want[name], name)
    gs, ws = got["sum_p"].view(np.uint64), want["sum_p"].view(np.uint64)
    nan = np.isnan(got["sum_p"]) & np.isnan(want["sum_p"])
    assert ((gs == ws) | nan).all(), "sum_p"


@pytest.mark.gpu
def test_mm1k_rejects_negative_and_oversized_K(engine):
    from workload_variant_autoscaler_b200 import WvaError
    with pytest.raises(WvaError):
        engine.mm1k_solve([-1], [1.0], [2.0])
    with pytest.raises(WvaError):
        engine.mm1k_solve([(1 << 20) + 1], [1.0], [2.0])
