"""The solvers' exponent windows at their edges, bit for bit against the oracle (DESIGN.md 3.1-3.2).

Every streaming solve divides with ``div_recip`` and keeps no ``p[0..K]`` vector; that is exact only while ``p``, the
running sum and the rates stay inside the windows of ``wva_device.cuh`` (``kHiPHi``, ``kHiSumHi``, ``kHiRowSumHi``,
``kHiRate*``, the pass-2 bound ``2^(E(sum) - 960)``).  Outside them a solve must bail out to the stored vector.  The
fleets here are steered onto those edges with beta = delta = 0: then ``servRate[n-1] = n / c`` and, with
``x = lambda * c``, ``p[n] ~ x^n / n!`` peaks near ``n = x`` at about ``2^(1.4427 x)``.  Which edge a case reaches is
decided by ``chain_profile`` (pass 1 of the reference in float64, same operations and order) and asserted by the CPU
tests below, so the GPU tests cannot silently drift off their edges.

Bands per path (E = binary exponent; each edge has cases at E = edge - 1 and E = edge):

* grid (``grid_kernel``, round-1 windows): E(max p) at 600, E(sum) at 620 for the cells that do not share their row;
  rows that share (``b >= j + 2``) with E(sum) at 620, and shared rows with p in [2^600, 2^620); chains that cross
  2^600 growing by 2^4 or more per step.
* size (``size_warp_kernel``, ``sz2_solve``) and sweep: E(max p) at 880, E(sum) at 680 and 900, the pass-2 IEEE path
  (sum in [2^882, 2^900), p < 2^880, states below 2^(E(sum) - 960) before termination), float64 overflow (the
  reference's rescale branch).  The sweep also has chains that cross 2^880 growing by 2^4 or more per step; the
  size path also has chains with K >= 2^23 (no early termination) whose pass 2 runs the IEEE path down to the
  smallest subnormal.
* every path: servRate[0] and servRate[N-1] at 2^-60 and 2^60, exactly on the boundary and just across it;
  lambda exactly at 2^-60 and one ulp below (grid, size).

Not reachable through the fleet interface, and so left out: a sum bail on its own (E(sum) 620 for unshared grid cells,
900 elsewhere) — the sum exceeds the peak by at most ~2^11 here, since Analyze keeps lambda below 0.999
servRate[N-1], so the cases at those sums have already crossed the p edge; on the size path no streaming solve sees p >= 2^880 after
its first one, because every later lambda of a candidate is at most the throughput of its first solve at lambda*
(0.9 RateRange.Max here) and a candidate whose first solve bails is re-run wholesale on the stored vector; steep
crossings on the size path, because lambda < servRate[N-1] keeps x below N and a crossing of 2^880 by 2^4 per step
needs x above 2600, where lambda* itself overflows; lambda alone at 2^60, because Analyze rejects lambda above
0.999 servRate[N-1], so lambda >= 2^60 always comes with servRate[N-1] above the window (the grid cases still put
lambda exactly on 2^60); exact lambda edges in the sweep, whose rates are spaced by the sweep itself.
"""
from __future__ import annotations

import numpy as np
import pytest

from tests.util import assert_allocs_equal, assert_f32_bits_equal
from workload_variant_autoscaler_b200 import Fleet, Grid, synth_fleet

f32 = np.float32
RATIO = 1          # queue ratio of every fleet here: K = 2 N (a long tail adds nothing at these edges)
SIZE_RATIO = 10
LONG_RATIO = 12400
SWEEP_RATES = 4096  # x = lambda * c steps by ~N / 4096: dense enough for the 2.5-wide pass-2 band near x = 612


# ---------------------------------------------------------------------------------------------------------------
# the reference's pass 1 (mm1modelstatedependent.go:93-105) in float64, vectorised over lambda
# ---------------------------------------------------------------------------------------------------------------
def _hi(v):
    """High 32 bits of float64 values (the solvers compare exponents on these)."""
    return (np.ascontiguousarray(v, np.float64).view(np.uint64) >> np.uint64(32)).astype(np.int64)


def _exp2(v):
    """Binary exponent floor(log2 v) of positive finite float64 values."""
    return np.frexp(v)[1].astype(np.int64) - 1


def _rate_below(lam32, m32):
    """wva_device.cuh rate_below: lambda at least 16 float32 ulps below m, both positive."""
    lb = lam32.view(np.uint32).astype(np.int64)
    mb = np.asarray(m32, np.float32).view(np.uint32).astype(np.int64)
    return (lb + 16 < mb) & (lam32 > 0) & (m32 > 0)


def chain_profile(serv_rate, K, lam, keep=False):
    """Pass 1 of the state-dependent model for every lambda of ``lam`` (float32).

    ``serv_rate`` is one rate vector for every lambda, or a list of them (one per lambda, each with its own ``K``).
    Returns a dict of arrays (one entry per lambda): ``emax`` = E(max p), ``esum`` = E(sum), ``j`` = the state at which
    DESIGN.md 3.2's early termination ends the chain (-1 if it never does), ``tail`` = the chain reaches state N - 1,
    ``over`` = p or the sum overflowed float64 (the reference's rescale branch; emax / esum are then meaningless),
    ``elive`` = smallest E(p) over states 1..j (where pass 2 divides by the sum), ``steep600`` / ``steep880`` = the
    step that first takes p to 2^600 / 2^880 multiplies it by 2^4 or more.  The operations and their order are the
    reference's, so until an overflow every p[n] and the sum are its bits; ``keep=True`` adds ``p`` [K+1, M] and
    ``sum``.
    """
    lam32 = np.atleast_1d(np.asarray(lam, np.float32))
    lam64 = lam32.astype(np.float64)
    M = lam32.size
    rates = list(serv_rate) if isinstance(serv_rate, (list, tuple)) else [serv_rate] * M
    rates = [np.ascontiguousarray(r, np.float32) for r in rates]
    Ks = np.broadcast_to(np.asarray(K, np.int64), (M,))
    Ns = np.array([r.size for r in rates])
    W = int(Ns.max())
    # rows padded with their last rate: column min(n, W - 1) is servRate[min(n, N - 1)], and the suffix minimum of
    # the padded row is min(servRate[min(n, N - 1)..N - 1])
    tab = np.stack([np.concatenate([r, np.full(W - r.size, r[-1], np.float32)]) for r in rates])
    sufmin = np.minimum.accumulate(tab[:, ::-1], axis=1)[:, ::-1]
    tab64 = tab.astype(np.float64)
    p = np.ones(M)
    s = np.ones(M)
    emax = np.zeros(M, np.int64)
    over = np.zeros(M, bool)
    j = np.full(M, -1, np.int64)
    elive = np.full(M, 1 << 20, np.int64)
    steep = {600: np.zeros(M, bool), 880: np.zeros(M, bool)}
    crossed = {600: np.zeros(M, bool), 880: np.zeros(M, bool)}
    thr_hi = None
    hist = [p.copy()] if keep else None
    with np.errstate(over="ignore", invalid="ignore"):
        for n in range(int(Ks.max())):
            act = n < Ks
            c = min(n, W - 1)
            r = tab64[:, c]
            p_prev = p
            p = np.where(act, (p * lam64) / r, p)              # p[n+1]
            s = np.where(act, s + p, s)
            m = n + 1
            if keep:
                hist.append(p.copy())
            over |= act & (~np.isfinite(p) | ~np.isfinite(s))
            ok = act & ~over & (p > 0)
            e = np.where(ok, _exp2(np.where(ok, p, 1.0)), -2000)
            emax = np.maximum(emax, np.where(over, 1 << 20, e))
            factor_e = np.log2(lam64 / r)
            for edge in (600, 880):
                first = act & ~crossed[edge] & ((e >= edge) | over)
                steep[edge] |= first & (factor_e >= 4)
                crossed[edge] |= first
            live = act & (j < 0)
            if m == 1:  # K >= 2^23: only an underflow to 0 ends the chain (the exit rule needs i < 2^23)
                thr_hi = np.where(Ks < (1 << 23), _hi(np.fmin(1.0, p) * 2.0 ** -78), 0)
            elive = np.where(live & ok, np.minimum(elive, e), elive)
            mn = sufmin[:, min(m, W - 1)]
            stop = live & (((_hi(np.where(over, 0.0, p)) < thr_hi) & _rate_below(lam32, mn)) | (p == 0))
            j = np.where(stop, m, j)
            if not keep and n >= W - 1 and np.all(~act | ((p == p_prev) & (s + p == s))):
                break  # past every head p is a fixed point (0, or stuck on the smallest subnormal) that adds nothing
    esum = np.where(over, 1 << 20, _exp2(np.where(over, 1.0, s)))
    out = {"emax": emax, "esum": esum, "j": j, "tail": (j < 0) | (j >= Ns - 1), "over": over, "elive": elive,
           "steep600": steep[600], "steep880": steep[880]}
    if keep:
        out["p"], out["sum"] = np.array(hist), s
    return out


# ---------------------------------------------------------------------------------------------------------------
# float32 lambdas exactly as the oracle forms them
# ---------------------------------------------------------------------------------------------------------------
def _lam_of_rate(rate):
    return f32(f32(rate) / f32(1000))


def _lam_grid(rpm, r):
    return _lam_of_rate(f32(f32(f32(rpm) / f32(60)) / f32(r)))


def _rpm_for_lambda(lam):
    """An arrival rate (requests per minute, float32) whose one-replica grid lambda is exactly ``lam``."""
    lam = f32(lam)
    base = f32(np.float64(lam) * 60000.0)
    for k in range(-64, 65):
        rpm = f32(base)
        for _ in range(abs(k)):
            rpm = np.nextafter(rpm, f32(np.inf if k > 0 else 0), dtype=np.float32)
        if _lam_grid(rpm, 1) == lam:
            return float(rpm)
    raise AssertionError(f"no arrival rate gives lambda {lam!r}")


def _sweep_lams(rmin, rmax, n):
    hi = f32(f32(rmax) * f32(0.999))
    span = f32(hi - f32(rmin))
    i = np.arange(n, dtype=np.float32)
    frac = (i / f32(n - 1)).astype(np.float32) if n > 1 else np.zeros(n, np.float32)
    rt = (f32(rmin) + (span * frac).astype(np.float32)).astype(np.float32)
    return (rt / f32(1000)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------
# fleets: one model and one accelerator per server, beta = delta = 0 unless given
# ---------------------------------------------------------------------------------------------------------------
def _fleet(alpha, gamma, rpm, batch, *, delta=0.0, tps=0.0, in_tok=1, out_tok=2, ratio=RATIO) -> Fleet:
    S = len(rpm)
    col = lambda v, dt=np.float32: np.broadcast_to(np.asarray(v, dt), (S,)).copy()  # noqa: E731
    return Fleet(
        acc_cost=[40.0], acc_multiplicity=[1], acc_type=[0], type_capacity=[1 << 20],
        perf_present=np.ones((S, 1)), perf_alpha=col(alpha).reshape(S, 1), perf_beta=np.zeros((S, 1)),
        perf_gamma=col(gamma).reshape(S, 1), perf_delta=col(delta).reshape(S, 1), perf_acc_count=np.ones((S, 1)),
        perf_max_batch=col(batch, np.int32).reshape(S, 1), perf_at_tokens=np.zeros((S, 1)),
        srv_model=np.arange(S), srv_priority=np.ones(S), srv_has_target=np.ones(S), srv_slo_itl=np.zeros(S),
        srv_slo_ttft=np.zeros(S), srv_slo_tps=col(tps), srv_keep_acc=np.zeros(S), srv_min_replicas=np.ones(S),
        srv_max_batch=col(batch, np.int32), srv_arrival_rpm=col(rpm), srv_in_tokens=col(in_tok, np.int32),
        srv_out_tokens=col(out_tok, np.int32), srv_cur_acc=np.full(S, -1), srv_cur_replicas=np.zeros(S),
        srv_cur_cost=np.zeros(S), unlimited=True, max_queue_to_batch_ratio=ratio)


def _concat(fleets) -> Fleet:
    kw = {}
    for n in Fleet.__dataclass_fields__:
        v = getattr(fleets[0], n)
        if isinstance(v, np.ndarray):
            kw[n] = np.concatenate([getattr(f, n) for f in fleets]) if (n.startswith(("srv_", "perf_"))) else v
        else:
            kw[n] = v
    kw["srv_model"] = np.arange(kw["srv_model"].size)
    return Fleet(**kw)


P60 = 2.0 ** 60
BELOW = lambda v: float(np.nextafter(f32(v), f32(0)))      # noqa: E731  one float32 ulp below
ABOVE = lambda v: float(np.nextafter(f32(v), f32(np.inf)))  # noqa: E731  one float32 ulp above


def _rate_edge_models(N):
    """(alpha, label) with out_tok = 2, gamma = 0, so c = alpha: servRate[0] = 1/c, servRate[N-1] = N/c."""
    return [(P60, "sr0 = 2^-60"), (ABOVE(P60), "sr0 < 2^-60"),
            (N / P60, "srN = 2^60"), (ABOVE(N / P60), "srN < 2^60")]


def grid_cases():
    """(fleet, grid) pairs of the grid path."""
    # 1) c = 1, lambda = x: x from 404 to 440 crosses E(max p) = 600 (x ~ 416) and E(sum) = 620 (x ~ 430).  b = 1024
    #    reaches its tail (grid_kernel); b = 2048 ends in its head (row sharing, up to E(sum) = 620).
    xs = np.arange(404.0, 440.0, 0.2)
    big = _fleet(1.0, 0.0, [_rpm_for_lambda(x) for x in xs], 1024)
    # 2) steep crossings of 2^600: x ~ 1800-2040 at b = 2048 crosses 2^600 near state 110 by x / 110 >= 2^4 per step
    steep = _fleet(1.0, 0.0, [_rpm_for_lambda(x) for x in np.linspace(1790.0, 2040.0, 6)], 1024)
    # 3) rate edges at b = 16: servRate[0] / servRate[15] on 2^-60 / 2^60, and lambda exactly on 2^-60 (c = 2^50,
    #    servRate[0] = 2^-50) and 2^60 (c = 2^-57, servRate[15] = 2^61)
    edges = []
    for alpha, _ in _rate_edge_models(16):
        c = np.float64(f32(alpha))
        for x in (0.5, 3.0, 9.0):
            edges.append((alpha, _rpm_for_lambda(x / c)))
    for lam in (2.0 ** -60, BELOW(2.0 ** -60)):
        for alpha in (2.0 ** 50, 2.0 ** 52, 2.0 ** 54):
            edges.append((alpha, _rpm_for_lambda(lam)))
    for lam in (P60, BELOW(P60)):
        for alpha in (2.0 ** -57, 2.0 ** -58, 2.0 ** -56):
            edges.append((alpha, _rpm_for_lambda(lam)))
    rate = _fleet([a for a, _ in edges], 0.0, [r for _, r in edges], 16)
    return [(big, Grid([1024, 2048], [1])), (steep, Grid([2048], [1])), (rate, Grid([4, 16], [1, 2]))]


def size_fleet():
    """Size candidates with TPS targets only: no bisection, so every lambda a candidate solves is known in advance:
    lambda* = 0.9 RateRange.Max, then the final Analyze at total / replicas (kept at one replica here).  Queue ratio
    10: the pass-2 IEEE band needs a chain that falls by ~960 binary orders after its peak, and past the head it
    falls by only about x / N = 0.9 per state."""
    rows = []
    # lambda* sweeps x* ~ 0.8991 N through the 680 / 880 / 900 bands and into float64 overflow (N >= 793); delta > 0
    # bends the profile a little so that neighbouring N do not skip exponents; the final lambda sits just below
    for N in range(440, 800):
        for d, frac in ((0.0, 0.999), (1e-5, 0.99)):
            rows.append((N, d, frac))
    tps = [float(f32(2.0 * float(_lam_star(_analyzer(N, 1.0, 0.0, d, ratio=SIZE_RATIO))) * 1000.0 * frac))
           for N, d, frac in rows]
    main = _fleet(1.0, 0.0, np.ones(len(rows)), [r[0] for r in rows], delta=[r[1] for r in rows], tps=tps,
                  ratio=SIZE_RATIO)
    # rate edges (N = 16): servRate[0] / servRate[15] on 2^-60 / 2^60; lambda_final exactly 2^-60 and one ulp below
    ea, et = [], []
    for a, _ in _rate_edge_models(16):
        for frac in (0.2, 0.5, 0.9):
            ea.append(a)
            et.append(float(f32(2.0 * float(_lam_star(_analyzer(16, a, 0.0, 0.0, ratio=SIZE_RATIO))) * 1000.0 * frac)))
    for lam in (2.0 ** -60, BELOW(2.0 ** -60)):
        for a in (2.0 ** 50, 2.0 ** 52, 2.0 ** 54):
            ea.append(a)
            et.append(float(f32(np.float64(f32(lam)) * 2000.0)))
    edge = _fleet(ea, 0.0, np.ones(len(ea)), 16, tps=et, ratio=SIZE_RATIO)
    return _concat([main, edge])


def long_queue_fleet():
    """K >= 2^23 (queue ratio 12400): no early termination, so after the peak the chain runs down to an underflow to 0
    and pass 2 divides states far below 2^(E(sum) - 960) by a sum in [2^882, 2^900).  Four candidates near
    N = 682, whose lambda* and final lambda (x ~ 610-613) put the sum in that band."""
    rows = [(N, frac) for N in (681, 682, 683, 684) for frac in (0.995,)]
    tps = [float(f32(2.0 * float(_lam_star(_analyzer(N, 1.0, 0.0, 0.0, ratio=LONG_RATIO))) * 1000.0 * frac))
           for N, frac in rows]
    return _fleet(1.0, 0.0, np.ones(len(rows)), [r[0] for r in rows], tps=tps, ratio=LONG_RATIO)


def overflow_search_fleet(slo_itl, slo_ttft):
    """The N = 1024 overflow fleet of the grid's stored-vector test with ITL (and TTFT) targets: the ITL bisection's
    end point lambda_max overflows float64, so the streaming solve bails in the search's first round and the
    stored-vector fallback bisects across overflowing midpoints."""
    fleet = synth_fleet(2, 1, seed=29, max_batch_choices=(1024,))
    fleet.perf_alpha[:] = 7.47
    fleet.perf_beta[:] = 0.0001
    fleet.perf_gamma[:] = 1.0
    fleet.perf_delta[:] = 0.00001
    fleet.srv_in_tokens[:] = 64
    fleet.srv_out_tokens[:] = 64
    fleet.srv_slo_tps[:] = 0
    fleet.srv_slo_itl[:] = slo_itl
    fleet.srv_slo_ttft[:] = slo_ttft
    fleet.srv_arrival_rpm[:] = [60.0 * 2100, 60.0 * 1900]
    return fleet


OVERFLOW_SEARCHES = [(7.55, 0.0, 1.6744), (7.56, 200.0, 1.8813)]  # slo_itl, slo_ttft, the candidates' max_rate


def sweep_fleet():
    """Sweep pairs: N = 1024 (x up to ~1022: 680, 880, 900, pass 2, overflow), N = 4096 (steep crossings of 2^880),
    and the rate edges at N = 16."""
    alpha = [1.0, 1.0] + [a for a, _ in _rate_edge_models(16)]
    batch = [1024, 4096] + [16] * 4
    return _fleet(alpha, 0.0, np.full(len(alpha), 600.0), batch)


def _analyzer(N, alpha, gamma, delta, in_tok=1, out_tok=2, ratio=RATIO):
    import oracle
    return oracle.Analyzer(int(N), int(N) * ratio, float(alpha), 0.0, float(gamma), float(delta), in_tok, out_tok)


def _lam_star(qa):
    lam_max = _lam_of_rate(qa.rate_range()[1])
    return _lam_of_rate(f32(f32(lam_max * f32(f32(1) - f32(0.1))) * f32(1000)))


def _fleet_model(fleet, s):
    return (float(fleet.perf_alpha[s, 0]), float(fleet.perf_gamma[s, 0]), float(fleet.perf_delta[s, 0]),
            int(fleet.srv_in_tokens[s]), int(fleet.srv_out_tokens[s]), int(fleet.max_queue_to_batch_ratio))


# ---------------------------------------------------------------------------------------------------------------
# the points each path evaluates, with their profiles
# ---------------------------------------------------------------------------------------------------------------
class _Lanes:
    """The (rates, K, lambda) of every point a path evaluates, profiled in one vectorised pass."""

    def __init__(self):
        self.sr, self.K, self.lam, self.N = [], [], [], []

    def add(self, qa, N, lams):
        sr = qa.serv_rate()
        for lam in lams:
            self.sr.append(sr)
            self.K.append(qa.K)
            self.lam.append(f32(lam))
            self.N.append(N)

    def profile(self):
        prof = chain_profile(self.sr, np.array(self.K), np.array(self.lam, np.float32))
        prof["lam"] = np.array(self.lam, np.float32)
        prof["sr0"] = np.array([r[0] for r in self.sr], np.float32)
        prof["srN"] = np.array([r[-1] for r in self.sr], np.float32)
        prof["N"] = np.array(self.N)
        return prof


def _cat(profs):
    return {k: np.concatenate([p[k] for p in profs]) for k in profs[0]}


def grid_points(fleet, grid, flags):
    """Profiles of the analysable cells (oracle flags bit 0) of a grid solve."""
    B, R = grid.batch.size, grid.replicas.size
    fl = flags.reshape(fleet.n_servers, 1, B, R)
    L = _Lanes()
    for s in range(fleet.n_servers):
        a, g, d, it, ot, ratio = _fleet_model(fleet, s)
        for bi, b in enumerate(grid.batch):
            lams = [_lam_grid(fleet.srv_arrival_rpm[s], r) for ri, r in enumerate(grid.replicas) if fl[s, 0, bi, ri] & 1]
            if lams:
                L.add(_analyzer(b, a, g, d, it, ot, ratio), int(b), lams)
    return L.profile()


def size_points(fleet, cand):
    """Profiles of the lambdas a size candidate is known to solve: lambda* (0.9 RateRange.Max) and the final
    Analyze at total / replicas with the oracle's replica count."""
    L = _Lanes()
    for s in range(fleet.n_servers):
        a, g, d, it, ot, ratio = _fleet_model(fleet, s)
        N = int(fleet.srv_max_batch[s])
        qa = _analyzer(N, a, g, d, it, ot, ratio)
        lams = [_lam_star(qa)]
        if cand["feasible"][s]:
            total = f32(f32(fleet.srv_slo_tps[s]) / f32(ot))
            lams.append(_lam_of_rate(f32(total / f32(cand["replicas"][s]))))
        L.add(qa, N, lams)
    return L.profile()


def sweep_points(fleet, n_rates, valid):
    v = valid.reshape(fleet.n_servers, n_rates)
    profs = []
    for s in range(fleet.n_servers):
        a, g, d, it, ot, ratio = _fleet_model(fleet, s)
        N = int(fleet.srv_max_batch[s])
        qa = _analyzer(N, a, g, d, it, ot, ratio)
        lo, hi = qa.rate_range()
        L = _Lanes()
        L.add(qa, N, _sweep_lams(lo, hi, n_rates)[v[s] == 1])
        profs.append(L.profile())
    return _cat(profs)


# ---------------------------------------------------------------------------------------------------------------
# bands
# ---------------------------------------------------------------------------------------------------------------
def _straddle(x, sel, edge):
    return int(np.sum(sel & (x == edge - 1))), int(np.sum(sel & (x == edge)))


def _rate_bands(P):
    """Counts for the rate edges: exactly on 2^-60 / 2^60 and just across (within 2^-20 relative)."""
    l, s0, sn = P["lam"], P["sr0"], P["srN"]
    lo, hi = f32(2.0 ** -60), f32(P60)
    below = lambda v, e: (v < e) & (v >= f32(e * (1 - 2.0 ** -20)))  # noqa: E731
    return {"sr0 == 2^-60": np.sum(s0 == lo), "sr0 just below 2^-60": np.sum(below(s0, lo)),
            "srN == 2^60": np.sum(sn == hi), "srN just below 2^60": np.sum(below(sn, hi)),
            "lam == 2^-60": np.sum(l == lo), "lam just below 2^-60": np.sum(below(l, lo))}


def grid_bands(P):
    ok = ~P["over"]
    shareable = ok & ~P["tail"] & (P["N"] >= P["j"] + 2)
    kernel = ok & ~shareable
    b = {}
    b["grid_kernel E(max p) 599 / 600"] = _straddle(P["emax"], kernel, 600)
    b["grid_kernel E(sum) 619 / 620"] = _straddle(P["esum"], kernel, 620)
    b["shared row E(sum) 619 / 620"] = _straddle(P["esum"], shareable, 620)
    in_band = shareable & (P["emax"] >= 600) & (P["esum"] < 620)
    b["shared row with p in [2^600, 2^620)"] = (int(in_band.sum()),) * 2
    b["steep crossing of 2^600"] = (int(P["steep600"].sum()),) * 2
    for k, v in _rate_bands(P).items():
        b[k] = (int(v),) * 2
    return b


def wide_bands(P, steep=True):
    ok = ~P["over"]
    b = {}
    b["E(max p) 879 / 880"] = _straddle(P["emax"], ok, 880)
    b["E(sum) 679 / 680"] = _straddle(P["esum"], ok, 680)
    b["E(sum) 899 / 900"] = _straddle(P["esum"], ok, 900)
    band = ok & (P["esum"] >= 882) & (P["esum"] < 900) & (P["emax"] < 880)
    ieee = band & (P["elive"] < P["esum"] - 960)
    b["pass-2 IEEE path"] = (int(ieee.sum()),) * 2
    b["float64 overflow"] = (int(P["over"].sum()),) * 2
    if steep:
        b["steep crossing of 2^880"] = (int(P["steep880"].sum()),) * 2
    return b


def _assert_bands(bands, skip=()):
    low = {k: v for k, v in bands.items() if k not in skip and min(v) < 3}
    assert not low, f"bands with fewer than 3 cases on a side: {low}"


# ---------------------------------------------------------------------------------------------------------------
# CPU: the helper is the reference's pass 1, and the cases reach their bands
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,x,delta", [(16, 3.0, 0.0), (64, 40.0, 1e-3), (512, 300.0, 0.0), (1024, 600.0, 0.0),
                                       (1024, 611.5, 0.0), (2048, 650.0, 2e-5)])
def test_chain_profile_matches_oracle_probs(oracle_mod, N, x, delta):
    """The helper's p[n] / sum equals the oracle's normalised vector bit for bit on non-overflowing chains."""
    qa = _analyzer(N, 1.0, 0.0, delta)
    lam = f32(x)
    prof = chain_profile(qa.serv_rate(), qa.K, [lam], keep=True)
    assert not prof["over"][0]
    st = qa.solve(float(lam))
    assert st["is_valid"]
    want = qa.probs()
    got = prof["p"][:, 0] / prof["sum"][0]
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))
    assert prof["emax"][0] == _exp2(prof["p"][:, 0].max())


def test_chain_profile_termination_rule_hand_checked():
    """N = 4, rates 1..4, lambda = 1/2: p = 1, 1/2, 1/8, 1/48, 1/384, and from state 4 on every step divides by 8
    (the tail rate 4), so p[n] = 2^-(3 (n - 4)) / 384.  p[1] = 1/2 puts the threshold at 2^-78 * 1/2 = 2^-79, and
    lambda is below every remaining rate from state 1 on.  p[27] = 2^-77.6 is above it, p[28] = 2^-80.6 below: j = 28,
    past the head (N - 1 = 3)."""
    sr = np.array([1, 2, 3, 4], np.float32)
    prof = chain_profile(sr, 40, [0.5], keep=True)
    p = prof["p"][:, 0]
    assert p[4] == 1.0 / 384 and p[27] > 2.0 ** -79 > p[28]
    assert prof["j"][0] == 28 and prof["tail"][0]
    # the same chain in a table of 40 rates 1..40 ends in its head: lambda = 1/2 is below all of them
    prof = chain_profile(np.arange(1, 41, dtype=np.float32), 80, [0.5])
    assert 0 < prof["j"][0] < 39 and not prof["tail"][0]
    # lambda not below the remaining rates: no termination however small p gets
    prof = chain_profile(sr, 40, [np.float32(3.99999)])
    assert prof["j"][0] == -1 and prof["tail"][0]


def test_grid_cases_reach_their_bands(oracle_mod):
    pts = []
    for fleet, grid in grid_cases():
        cells, _ = oracle_mod.grid_solve(fleet, grid, want_cells=True)
        pts.append(grid_points(fleet, grid, cells["flags"]))
    _assert_bands(grid_bands(_cat(pts)))


def test_size_cases_reach_their_bands(oracle_mod):
    fleet = size_fleet()
    cand, _ = oracle_mod.solve(fleet)
    P = size_points(fleet, cand.reshape(-1))
    _assert_bands(wide_bands(P, steep=False))
    _assert_bands({k: (int(v),) * 2 for k, v in _rate_bands(P).items()})


def test_long_queue_cases_reach_the_pass2_ieee_path(oracle_mod):
    fleet = long_queue_fleet()
    cand, _ = oracle_mod.solve(fleet)
    P = size_points(fleet, cand.reshape(-1))
    assert (P["N"] * (1 + LONG_RATIO) >= 1 << 23).all()
    ieee = ~P["over"] & (P["esum"] >= 882) & (P["esum"] < 900) & (P["emax"] < 880) & (P["elive"] < P["esum"] - 960)
    assert ieee.sum() >= 3, P["esum"]


def test_overflow_search_cases_bail_inside_the_search(oracle_mod):
    """The ITL bisection of overflow_search_fleet iterates (EvalITL crosses the targets between lambda_min and
    lambda_max), its end point lambda_max and 0.9 lambda_max overflow float64 while lambda_max / 2 does not, and the
    candidates are feasible."""
    import oracle
    f = overflow_search_fleet(7.55, 0.0)
    ratio = f.max_queue_to_batch_ratio
    qa = oracle.Analyzer(1024, 1024 * ratio, float(f.perf_alpha[0, 0]), float(f.perf_beta[0, 0]),
                         float(f.perf_gamma[0, 0]), float(f.perf_delta[0, 0]), int(f.srv_in_tokens[0]),
                         int(f.srv_out_tokens[0]))
    lo, hi = qa.rate_range()
    lmin, lmax = _lam_of_rate(lo), _lam_of_rate(hi)
    (e0, y0), (e1, y1) = qa.eval_itl(float(lmin)), qa.eval_itl(float(lmax))
    assert e0 == 0 and e1 == 0
    assert y0 < min(t for t, _, _ in OVERFLOW_SEARCHES) and y1 > max(t for t, _, _ in OVERFLOW_SEARCHES)
    P = chain_profile(qa.serv_rate(), qa.K, [lmax, f32(f32(0.9) * lmax), f32(lmax / f32(2))])
    assert P["over"].tolist() == [True, True, False]
    for slo_itl, slo_ttft, max_rate in OVERFLOW_SEARCHES:
        cand, _ = oracle_mod.solve(overflow_search_fleet(slo_itl, slo_ttft))
        assert (cand["feasible"] == 1).all() and (cand["replicas"] == 2).all()
        assert np.allclose(cand["max_rate"], max_rate, rtol=1e-4)


def test_sweep_cases_reach_their_bands(oracle_mod):
    fleet = sweep_fleet()
    o = oracle_mod.sweep(fleet, SWEEP_RATES)
    P = sweep_points(fleet, SWEEP_RATES, o["valid"])
    _assert_bands(wide_bands(P))
    _assert_bands({k: (int(v),) * 2 for k, v in _rate_bands(P).items() if not k.startswith("lam")})


# ---------------------------------------------------------------------------------------------------------------
# GPU: every path at these edges, bit for bit
# ---------------------------------------------------------------------------------------------------------------
def _cells_equal(cells_g, cells_o, what):
    assert np.array_equal(cells_g["flags"], cells_o["flags"]), f"{what}: cell flags differ"
    for k in ("ttft", "itl", "rho", "throughput"):
        assert_f32_bits_equal(cells_g[k], cells_o[k], f"{what}: cells.{k}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(3))
def test_grid_cells_at_window_edges(engine, oracle_mod, case):
    fleet, grid = grid_cases()[case]
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    cells_g, win_g = engine.grid_solve(fleet, grid, want_cells=True)
    _cells_equal(cells_g, cells_o, f"grid case {case}")
    assert_allocs_equal(win_g, win_o, f"grid case {case} winners (cell table)")


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(3))
def test_grid_winners_at_window_edges(engine, oracle_mod, case):
    """Without a cell table (grid_order pruning): the winners."""
    fleet, grid = grid_cases()[case]
    _, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=False)
    _, win_g = engine.grid_solve(fleet, grid, want_cells=False)
    assert_allocs_equal(win_g, win_o, f"grid case {case} winners")


@pytest.mark.gpu
def test_size_warp_kernel_at_window_edges(engine, oracle_mod):
    fleet = size_fleet()
    assert fleet.n_servers <= 1024  # size_warp_kernel's range
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, "size candidates (warp per candidate)")
    assert_allocs_equal(win_g, win_o, "winners (warp per candidate)")


@pytest.mark.gpu
@pytest.mark.parametrize("depth", ["1", "5"])
def test_size_rounds_at_window_edges(engine, oracle_mod, monkeypatch, depth):
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    fleet = size_fleet()
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, f"size candidates (rounds, D = {depth})")
    assert_allocs_equal(win_g, win_o, f"winners (rounds, D = {depth})")


@pytest.mark.gpu
@pytest.mark.parametrize("small_max", ["1024", "0"])
def test_size_long_queue_at_window_edges(engine, oracle_mod, monkeypatch, small_max):
    """Chains without early termination (K >= 2^23) whose pass 2 must take the exact IEEE path below 2^(E(sum) - 960)."""
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", small_max)
    fleet = long_queue_fleet()
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, f"long-queue size candidates (small max {small_max})")
    assert_allocs_equal(win_g, win_o, f"long-queue winners (small max {small_max})")


@pytest.mark.gpu
@pytest.mark.parametrize("small_max,depth", [("1024", "5"), ("0", "1"), ("0", "5")])
@pytest.mark.parametrize("case", range(len(OVERFLOW_SEARCHES)))
def test_size_search_bails_to_stored_vector(engine, oracle_mod, monkeypatch, small_max, depth, case):
    """A bisection whose streaming solves overflow float64 (the warp kernel and the rounds at depths 1 and 5): the
    candidate is re-run on the stored vector, whose search crosses overflowing midpoints."""
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", small_max)
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    slo_itl, slo_ttft, _ = OVERFLOW_SEARCHES[case]
    fleet = overflow_search_fleet(slo_itl, slo_ttft)
    cand_o, win_o = oracle_mod.solve(fleet)
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand_o, f"size candidates (overflowing search, small max {small_max}, D = {depth})")
    assert_allocs_equal(win_g, win_o, f"winners (overflowing search, small max {small_max}, D = {depth})")


def _sweep_equal(g, o, what):
    assert np.array_equal(g["valid"], o["valid"]), f"{what}: valid differs"
    for k in ("rate", "ttft", "itl", "throughput", "rho"):
        assert_f32_bits_equal(g[k], o[k], f"{what}: sweep.{k}")


@pytest.mark.gpu
def test_sweep_at_window_edges(engine, oracle_mod):
    """Points outside the streaming windows (including float64 overflow) are re-run on the stored vector."""
    fleet = sweep_fleet()
    o = oracle_mod.sweep(fleet, SWEEP_RATES)
    g = engine.sweep(fleet, SWEEP_RATES)
    _sweep_equal(g, o, "window-edge sweep")


@pytest.mark.gpu
def test_sweep_overflow_fleet_falls_back_to_stored_vector(engine, oracle_mod):
    """The N = 1024 fleet of the grid's overflow test, swept with 64 rates: the chains of the upper rates overflow
    float64, where the reference rescales its stored vector."""
    fleet = synth_fleet(2, 1, seed=29, max_batch_choices=(1024,))
    fleet.perf_alpha[:] = 7.47
    fleet.perf_beta[:] = 0.0001
    fleet.perf_gamma[:] = 1.0
    fleet.perf_delta[:] = 0.00001
    fleet.srv_in_tokens[:] = 64
    fleet.srv_out_tokens[:] = 64
    o = oracle_mod.sweep(fleet, 64)
    assert o["valid"].sum() == 128
    g = engine.sweep(fleet, 64)
    _sweep_equal(g, o, "overflow sweep")
