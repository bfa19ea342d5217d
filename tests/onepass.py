"""grid_kernel's one-pass decision (DESIGN.md 3.2b) restated on the CPU, for the tests that check it.

Pass 1 of ``solve_shared_t`` (grid instantiation) also accumulates ``mom = sum(i*p[i])`` with one FMA per state and
keeps ``sum`` and ``mom`` at state ``min(N, m)``.  From those and ``zh = RN(1/sum)`` it forms ``A1 ~ acc`` and
``I1 ~ in_serv`` and skips pass 2 when the bounds ``E_acc`` / ``E_in`` put each value's float32 rounding beyond doubt.
Here the reference's pass 2 (exact quotients ``RN(p[i]/sum)``, its accumulations in its order) and the one-pass values
are computed from ``tests.grid_cases.chain_profile``'s ``p[i]`` (the reference's bits), the FMA exactly through
``fractions.Fraction`` and the bounds exactly (the kernel rounds them upwards, so it decides a subset of what is decided
here).
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np

from tests.grid_cases import _lam_grid, chain_profile

f32 = np.float32
U = Fraction(1, 1 << 53)
CU = U * (1 + Fraction(1, 1 << 16))
ABS = Fraction(1, 2) ** 1000


def reference(p, S, N, m):
    """Pass 2 of the reference: acc, in_serv (float64, its operations and order)."""
    zh = 1.0 / S
    acc, sum_p, acc_n = 0.0, zh, 0.0
    for i in range(1, m + 1):
        q = p[i] / S
        acc = acc + float(i) * q
        if i <= N:
            sum_p = sum_p + q
            acc_n = acc
    return acc, acc_n + (1.0 - sum_p) * float(N)


def onepass(p, S, N, m):
    """Pass 1's extra sums and the values and bounds formed from them: A1, I1, E_acc, E_in."""
    s, mom, s_n, mom_n = 1.0 + p[1], p[1], 1.0 + p[1], p[1]
    for i in range(2, m + 1):
        s = s + p[i]
        mom = float(Fraction(i) * Fraction(p[i]) + Fraction(mom))  # fma(i, p[i], mom): float(Fraction) is RN
        if i <= N:
            s_n, mom_n = s, mom
    assert s == S
    zh = 1.0 / S
    A1, AN, s1 = mom * zh, mom_n * zh, s_n * zh
    d1 = 1.0 - s1
    I1 = AN + d1 * float(N)
    m1 = min(N, m)
    E_acc = 2 * (m + 1) * CU * Fraction(A1) + ABS
    E_in = CU * (2 * (m1 + 1) * Fraction(AN) + N * (2 * m1 + 3) * Fraction(s1) + 4 * N * abs(Fraction(d1))
                 + 2 * abs(Fraction(I1))) + ABS
    return A1, I1, E_acc, E_in


def decided(x: float, E: Fraction) -> bool:
    """f32_decided: [x - E, x + E] strictly between the float32 midpoints next to RN32(x), a normal float32."""
    ax = abs(x)
    f = f32(ax)
    fb = int(np.array(f).view(np.uint32))
    if not (0x00800000 <= fb < 0x7F7FFFFF):
        return False
    up = np.array(fb + 1, np.uint32).view(np.float32)
    dn = np.array(fb - 1, np.uint32).view(np.float32)
    m_hi = (Fraction(float(f)) + Fraction(float(up))) / 2
    m_lo = (Fraction(float(f)) + Fraction(float(dn))) / 2
    return m_lo < Fraction(ax) - E and Fraction(ax) + E < m_hi


def chain(rates, K, lam):
    """The reference's p[0..K] and the states 1..m the solver accumulates (m = the exit state, or K), with the sum over
    them; that sum equals chain_profile's sum over all K states (the skipped states add nothing, DESIGN.md 3.2)."""
    pr = chain_profile(rates, K, lam, keep=True)
    assert not pr["over"][0]
    p = pr["p"][:, 0]
    j = int(pr["j"][0])
    m = K if j < 0 else j
    S = 1.0
    for i in range(1, m + 1):
        S = S + p[i]
    assert S == float(pr["sum"][0])
    return p, S, m


def lane(rates, K, lam):
    """Everything the tests compare for one solve: the reference's acc / in_serv, A1, I1 and their bounds."""
    N = rates.size
    p, S, m = chain(rates, K, lam)
    acc, ins = reference(p, S, N, m)
    A1, I1, E_acc, E_in = onepass(p, S, N, m)
    return {"acc": acc, "in_serv": ins, "A1": A1, "I1": I1, "E_acc": E_acc, "E_in": E_in, "m": m}


# ---------------------------------------------------------------------------------------------------------------
# the mixed warp: one pair, batch size 3, 32 replica levels -> its 32 candidate cells are one full, staged item
# ---------------------------------------------------------------------------------------------------------------
# alpha = gamma = 1 ms, delta = 0.5 ms per token (one input token; a nonzero delta keeps ITL and TTFT finite):
# servRate[n-1] = n / (2 + n / 2) per ms; lambda(1) ~ 4.2e-5 per ms ~ 1e-4 servRate[0]
MIX_N, MIX_RATIO, MIX_RPM, MIX_DELTA = 3, 10, 2.5, 0.5


def mix_rates():
    """servRate as BuildModel forms it (float32, its operations and order) for alpha = gamma = 1, beta = 0."""
    n = np.arange(1, MIX_N + 1, dtype=np.float32)
    prefill = (f32(1) + (f32(MIX_DELTA) * f32(1)) * n).astype(np.float32)
    decode = f32(1) * (f32(1) + f32(0) * n).astype(np.float32)
    return (n / (prefill + decode).astype(np.float32)).astype(np.float32)


def mix_lane(r):
    return lane(mix_rates(), MIX_N * (1 + MIX_RATIO), _lam_grid(MIX_RPM, r))


def mix_replicas():
    """Replica levels 1..31 (decided lanes) and one level R whose lambda ~ 1e-9 servRate[0] leaves in_serv far below
    E_in's absolute term, so that lane is undecided; R is the first level from 100000 on whose one-pass in_serv also
    rounds to a different float32 than the reference's (the cancellation in 1 - sumP dominates both values)."""
    for R in range(100000, 101000):
        L = mix_lane(R)
        if f32(L["I1"]) != f32(L["in_serv"]):
            return list(range(1, 32)) + [R]
    raise AssertionError("no replica level in [100000, 101000) rounds differently")
