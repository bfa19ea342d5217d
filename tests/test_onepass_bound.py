"""grid_kernel's one-pass decision (DESIGN.md 3.2b), restated on the CPU (``tests.onepass``).

On saturated chains the bounds must hold (``|reference - approximation| <= E``) and a decided output must round to the
reference's float32.  On light-load chains, whose ``in_serv`` sits far below ``E_in``'s absolute term and whose one-pass
``in_serv`` is then dominated by the rounding of ``1 - s1`` as the reference's is by ``1 - sumP``, the two values round
to different float32s for some lambdas: those must be undecided.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from tests.grid_cases import _lam_grid
from tests.onepass import decided, lane

f32 = np.float32


def _saturated(seed, count):
    """servRate[n-1] = n / c, lambda around servRate[N-1], K = 11 N."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(count):
        N = int(rng.integers(2, 257))
        c = f32(rng.uniform(0.5, 4.0))
        rates = (np.arange(1, N + 1, dtype=np.float32) / c).astype(np.float32)
        lam = f32(rates[-1] * f32(rng.uniform(0.85, 1.0)))
        out.append((rates, 11 * N, lam))
    return out


def _light(N, reps):
    """servRate[n-1] = n / 2 per ms, lambda = 3 req/min over r replicas (lambda / servRate[0] ~ 1e-4 / r), K = 11 N."""
    rates = (np.arange(1, N + 1, dtype=np.float32) / f32(2)).astype(np.float32)
    return [(rates, 11 * N, _lam_grid(3.0, r)) for r in reps]


def _check(L, what):
    assert abs(Fraction(L["acc"]) - Fraction(L["A1"])) <= L["E_acc"], what
    assert abs(Fraction(L["in_serv"]) - Fraction(L["I1"])) <= L["E_in"], what
    out = {}
    for name, ref, x, E in (("acc", L["acc"], L["A1"], L["E_acc"]), ("in_serv", L["in_serv"], L["I1"], L["E_in"])):
        out[name] = (decided(x, E), f32(ref) == f32(x))
        if out[name][0]:
            assert out[name][1], (name, what)
    return out


def test_onepass_bound_holds_on_saturated_chains():
    n_dec = {"acc": 0, "in_serv": 0}
    cases = _saturated(7, 24)
    for k, (rates, K, lam) in enumerate(cases):
        for name, (dec, _) in _check(lane(rates, K, lam), f"saturated chain {k}").items():
            n_dec[name] += dec
    # the bound decides nearly every output of these chains: pass 2 is the exception
    assert n_dec["acc"] >= len(cases) - 1 and n_dec["in_serv"] >= len(cases) - 2, n_dec


def test_onepass_refuses_the_lambdas_that_round_differently():
    differ = undecided = 0
    for N in (3, 8):
        for k, (rates, K, lam) in enumerate(_light(N, range(100000, 100200))):
            res = _check(lane(rates, K, lam), f"light chain N={N} #{k}")
            dec, same = res["in_serv"]
            undecided += not dec
            if not same:
                differ += 1
                assert not dec, (N, k)  # (also asserted inside _check)
    # the construction does reach both: one-pass values on the other side of a midpoint, and refusals
    assert differ >= 5 and undecided >= differ, (differ, undecided)


def test_decision_refuses_a_midpoint_inside_the_bound():
    # a value just below a midpoint, with a bound that reaches across it
    f = f32(1.5)
    mid = (float(f) + float(np.nextafter(f, f32(2)))) / 2
    x = mid - 2.0 ** -40
    assert not decided(x, Fraction(2) ** -39)
    assert decided(x, Fraction(2) ** -41)
    # below a power of two the lower midpoint is half as far away
    g = f32(2.0)
    lo_mid = (float(g) + float(np.nextafter(g, f32(0)))) / 2
    assert not decided(lo_mid + 2.0 ** -30, Fraction(2) ** -29)
    assert decided(2.0, Fraction(2) ** -27)
    # zero, subnormal, FLT_MAX and non-finite values are never decided
    for v in (0.0, 1e-40, float(np.finfo(np.float32).max), float("inf"), float("nan")):
        assert not decided(v, Fraction(0))
