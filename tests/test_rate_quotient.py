"""Division by a float32 service rate without Markstein's correction (DESIGN.md 3.1).

The recurrence divides by servRate[n], a float32 value, through ``div_rate`` and ``step_rate`` (wva_device.cuh):
``RN(a*yh + RN(a*yl))`` and ``RN(RN(p*lam)*yh + RN(p*RN(lam*yl)))`` around the double-word reciprocal
``yh = RN(1/b)``, ``yl = RN((1 - b*yh)/b)``.  Both are restated here in exact rational arithmetic (``float`` of a
``Fraction`` is the correctly rounded double) and compared with ``RN(a/b)``:

* on the hardest float32 divisors: ``b = M`` odd with 24 bits and ``a = A`` with ``A * 2^25 = M*O -+ 1`` for an odd
  54-bit ``O``, which puts ``a/b`` at the least distance from the rounding midpoint ``O * 2^-25`` that a quotient by a
  24-bit divisor can have (~2^-78 relative);
* on random float32 divisors, including ones just above and below a power of two, with ``p`` at the edges of the
  solver's exponent windows;
* and, as the negative control, on the same construction with odd 53-bit divisors, where the missing correction
  must show: the result depends on the divisor being a float32 value, and this test can see it when it is not.
"""
import math
import random
from fractions import Fraction

import numpy as np


def rn(x: Fraction) -> float:
    return float(x)  # int / int true division: correctly rounded


def make_recip(b: float):
    yh = rn(1 / Fraction(b))
    e = rn(1 - Fraction(b) * Fraction(yh))  # exact: yh is the correctly rounded reciprocal
    return yh, rn(Fraction(e) / Fraction(b))


def div_rate(a: float, r) -> float:
    yh, yl = r
    return rn(Fraction(a) * Fraction(yh) + Fraction(rn(Fraction(a) * Fraction(yl))))


def step_rate(p: float, lam: float, r) -> float:
    yh, yl = r
    c = rn(Fraction(lam) * Fraction(yl))
    a = rn(Fraction(p) * Fraction(lam))
    t = rn(Fraction(p) * Fraction(c))
    return rn(Fraction(a) * Fraction(yh) + Fraction(t))


def quotient(a: float, b: float) -> float:
    return rn(Fraction(a) / Fraction(b))


def is_f32(x: float) -> bool:
    return float(np.float32(x)) == x


def hardest(rng: random.Random, bits: int):
    """(A, M, O, shift): M odd with `bits` bits, O odd with 54 bits (a midpoint between doubles at its scale) and
    A * 2^shift = M*O -+ 1, shift = bits + 1, so that A has at most 53 bits."""
    shift = bits + 1
    while True:
        M = (1 << (bits - 1)) | rng.getrandbits(bits - 1) | 1
        inv = pow(M, -1, 1 << shift)
        plus = rng.random() < 0.5  # M*O + 1 (O = -M^-1) or M*O - 1 (O = M^-1)
        olo = (-inv if plus else inv) % (1 << shift)
        hi_bits = 54 - shift  # O = hi * 2^shift + olo in [2^53, 2^54)
        O = (((1 << (hi_bits - 1)) | rng.getrandbits(hi_bits - 1)) << shift | olo) if hi_bits else olo
        if O >> 53 == 1:
            break
    num = M * O + (1 if plus else -1)
    assert num % (1 << shift) == 0 and O % 2 == 1
    A = num >> shift
    assert A < 1 << 53
    return A, M, O, shift


def test_hardest_float32_divisors_round_correctly():
    rng = random.Random(0x5EED)
    bad = 0
    for k in range(3000):
        A, M, O, shift = hardest(rng, 24)
        eb = rng.randrange(-60, 60)
        b = math.ldexp(M, eb - 23)
        assert is_f32(b)
        ea = rng.randrange(-340, 941)
        a = math.ldexp(A, ea - 52)
        # a / b sits 2^-25 / M (scaled) from the midpoint O * 2^-25 (scaled): no closer case exists
        m = Fraction(O, 1 << shift) * Fraction(2) ** (ea - 52 - eb + 23)
        assert abs(Fraction(a) / Fraction(b) - m) == m / O / M
        r = make_recip(b)
        want = quotient(a, b)
        bad += div_rate(a, r) != want
        # the tail step with lambda a power of two, so that p * lambda = a exactly; p at the window edges too
        el = rng.randrange(-60, 61)
        ep = (-279, 599, 879)[k % 3] if k % 2 else ea - el
        if -279 <= ep <= 879:
            lam = math.ldexp(1.0, el)
            p = math.ldexp(A, ep - 52)
            a2 = p * lam  # exact
            bad += step_rate(p, lam, r) != quotient(a2, b)
    assert bad == 0


def test_random_float32_divisors_round_correctly():
    rng = random.Random(42)
    bad = 0
    for k in range(3000):
        kind = k % 4
        mant = rng.getrandbits(23)
        if kind == 1:
            mant = rng.getrandbits(6)  # just above a power of two
        elif kind == 2:
            mant = (1 << 23) - 1 - rng.getrandbits(6)  # just below a power of two
        b = math.ldexp((1 << 23) | mant, rng.randrange(-60, 61) - 23)
        lam = math.ldexp((1 << 23) | rng.getrandbits(23), rng.randrange(-60, 61) - 23)
        assert is_f32(b) and is_f32(lam)
        # p anywhere in [2^-280, 2^880), at the lower edge, at the narrow upper edge 2^600 or just below 2^880
        ep = (rng.randrange(-280, 880), -280, 599, 879)[k % 4]
        sig = rng.getrandbits(52)
        if k % 8 >= 6:
            sig = (1 << 52) - 1 - rng.getrandbits(4)
        p = math.ldexp((1 << 52) | sig, ep - 52)
        r = make_recip(b)
        a = rn(Fraction(p) * Fraction(lam))
        bad += step_rate(p, lam, r) != quotient(a, b)
        bad += div_rate(a, r) != quotient(a, b)
        bad += div_rate(p, r) != quotient(p, b)
    assert bad == 0


def test_53_bit_divisors_need_the_correction():
    """The same construction with odd 53-bit divisors: q0 without the correction is off by one ulp in some cases."""
    rng = random.Random(7)
    bad = 0
    for _ in range(600):
        A, M, _, _ = hardest(rng, 53)
        b = math.ldexp(M, -52)
        a = math.ldexp(A, rng.randrange(-200, 200))
        bad += div_rate(a, make_recip(b)) != quotient(a, b)
    assert bad >= 1
