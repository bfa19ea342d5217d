"""The grid step's shared cases and checks: the fleets and batch lists at the shape thresholds and the streaming
solver's exponent windows, the chain profile that places a solve in its band, and the comparisons the grid, window
and pruning tests make against the oracle."""
from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from tests.levels import lam_range
from tests.util import ALLOC_FIELDS, assert_allocs_equal, assert_f32_bits_equal
from workload_variant_autoscaler_b200 import Fleet, Grid, _abi, synth_fleet

f32 = np.float32
RATIO = 1          # queue ratio of every fleet here: K = 2 N (a long tail adds nothing at these edges)
SIZE_RATIO = 10
LONG_RATIO = 12400
SWEEP_RATES = 4096  # x = lambda * c steps by ~N / 4096: dense enough for the 2.5-wide pass-2 band near x = 612


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


def _cells_equal(cells_g, cells_o, what):
    assert np.array_equal(cells_g["flags"], cells_o["flags"]), f"{what}: cell flags differ"
    for k in ("ttft", "itl", "rho", "throughput"):
        assert_f32_bits_equal(cells_g[k], cells_o[k], f"{what}: cells.{k}")


def _sweep_equal(g, o, what):
    assert np.array_equal(g["valid"], o["valid"]), f"{what}: valid differs"
    for k in ("rate", "ttft", "itl", "throughput", "rho"):
        assert_f32_bits_equal(g[k], o[k], f"{what}: sweep.{k}")


def shape_fleet(S, A, seed):
    """S servers x A accelerators with every pair class and exact ties across accelerators.

    Server 0 has no load, server 2 has a TPS target, server 3 has no profile on the last accelerator.  Cost per
    replica is 80 on every accelerator (acc_cost x acc_count) and nobody has a current allocation, so the rows of one
    replica level tie in (value, cost, replicas) on every accelerator; accelerator 1 has accelerator 0's profile, so
    their cells tie outright and the accelerator id decides.  Queue ratio 1 keeps the oracle cheap."""
    f = synth_fleet(S, A, seed=seed, zero_load_frac=0.0, tps_frac=0.0, max_batch_choices=(8,))
    f.max_queue_to_batch_ratio = 1
    counts = np.array([1, 2, 4, 8], np.int32)[np.arange(A) % 4]
    f.perf_acc_count[:] = counts[None, :]
    f.acc_cost[:] = (80.0 / counts).astype(np.float32)
    if A >= 2:
        for col in (f.perf_alpha, f.perf_beta, f.perf_gamma, f.perf_delta):
            col[:, 1] = col[:, 0]
    f.srv_cur_acc[:] = -1
    f.srv_cur_replicas[:] = 0
    f.srv_cur_cost[:] = 0.0
    f.srv_arrival_rpm[0] = 0.0
    f.perf_present[f.srv_model[3], A - 1] = 0
    f.srv_slo_tps[2] = 500.0
    f.srv_slo_itl[:] = 150.0  # above every alpha: each loaded server has a feasible cell
    f.srv_slo_ttft[:] = 1500.0
    # loads from light (shared chains at the smallest replica level) to heavy (long chains, grid_kernel)
    f.srv_arrival_rpm[1:] = np.geomspace(0.05, 3000.0, S - 1).astype(np.float32)
    return f


def _batches(values, B, seed):
    """B batch sizes drawn from ``values``, unsorted and repeated."""
    rng = np.random.default_rng(seed)
    b = rng.choice(np.asarray(values), B)
    b[: len(values)] = values
    rng.shuffle(b)
    return b


SMALL_B = [24, 16, 64, 40]  # unsorted; all above the lightest rows' jl + 2, below the heavy rows'
STAGE_B = [20, 16, 33, 40, 17, 64, 24, 48]  # ("draw", B): B batch sizes drawn from these
SHAPES = {
    "A=256": (4, 256, [40, 16], [1, 2, 4], {"prune": True}),
    "A=257": (4, 257, [40, 16], [1, 2, 4], {"prune": False}),
    "A*R=2048": (4, 4, [40, 16], np.arange(1, 513), {"prune": True, "order_q": 1}),
    "A*R=2049": (4, 3, [40, 16], np.arange(1, 684), {"prune": False}),
    "n=256": (5, 2, SMALL_B, np.arange(1, 129), {"prune": True, "order_q": 4, "order_passes": 1,
                                                  "finalize_keys": 1, "rows_threads": 128}),
    "n=257": (6, 1, SMALL_B, np.arange(1, 258), {"prune": True, "order_q": 2, "order_passes": 2,
                                                  "finalize_keys": 2}),
    "n=512": (5, 4, SMALL_B, np.arange(1, 129), {"prune": True, "order_q": 2, "order_passes": 2}),
    "n=513": (5, 3, SMALL_B, np.arange(1, 172), {"prune": True, "order_q": 1, "order_passes": 3,
                                                  "finalize_keys": 3}),
    "B=2048": (4, 2, ("draw", 2048), [1, 4, 16], {"stage_b": True, "stage_rmax": True}),
    "B=2049": (4, 2, ("draw", 2049), [1, 4, 16], {"stage_b": False, "stage_rmax": False}),
    "A*B=4096": (4, 16, ("draw", 256), [1, 3], {"stage_b": True, "stage_rmax": True}),
    "A*B=4097": (4, 17, ("draw", 241), [1, 3], {"stage_b": True, "stage_rmax": False}),
    "Bmax=1536": (5, 2, [24, 16, 1536, 48], [1, 2, 3, 5, 8, 13], {"rows_smem": True}),
    "Bmax=1537": (5, 2, [24, 16, 1537, 48], [1, 2, 3, 5, 8, 13], {"rows_smem": False}),
    "R=32": (5, 2, SMALL_B, np.arange(1, 33), {"rows_threads": 32}),
    "R=33": (5, 2, SMALL_B, np.arange(1, 34), {"rows_threads": 64}),
    "R=64": (5, 2, SMALL_B, np.arange(1, 65), {"rows_threads": 64}),
    "R=65": (5, 2, SMALL_B, np.arange(1, 66), {"rows_threads": 64}),
    "R=127": (5, 2, SMALL_B, np.arange(1, 128), {"rows_threads": 64}),
    "R=128": (5, 2, SMALL_B, np.arange(1, 129), {"rows_threads": 128}),
    "R=8193": (5, 1, [24], np.arange(1, 8194), {"prune": False}),
}


@functools.lru_cache(maxsize=None)
def shape_case(name):
    S, A, batch, replicas, _ = SHAPES[name]
    seed = 101 + list(SHAPES).index(name)
    if isinstance(batch, tuple):
        batch = _batches(STAGE_B, batch[1], seed)
    return shape_fleet(S, A, seed), Grid(batch, replicas)


@functools.lru_cache(maxsize=None)
def shape_oracle(name):
    import oracle
    fleet, grid = shape_case(name)
    return oracle.grid_solve(fleet, grid, want_cells=True)


def _lambda(fleet, s, r):
    """The grid's lambda of server s at r replicas (total_rate_of / r / 1000, float32)."""
    tps = f32(fleet.srv_slo_tps[s])
    total = f32(fleet.srv_arrival_rpm[s]) / f32(60) if tps == 0 else tps / f32(fleet.srv_out_tokens[s])
    return f32(f32(total / f32(r)) / f32(1000))


def _analyzer_of(fleet, s, a, b):
    import oracle
    m = int(fleet.srv_model[s])
    return oracle.Analyzer(int(b), int(b) * fleet.max_queue_to_batch_ratio, float(fleet.perf_alpha[m, a]),
                           float(fleet.perf_beta[m, a]), float(fleet.perf_gamma[m, a]), float(fleet.perf_delta[m, a]),
                           int(fleet.srv_in_tokens[s]), int(fleet.srv_out_tokens[s]))


def cell_shares_row(fleet, s, a, b, r):
    """The cell's chain ends in its head with b >= j + 2 (DESIGN.md 3.2a): a shared-chain cell, evaluated by
    grid_order / grid_shared; otherwise grid_kernel evaluates it."""
    qa = _analyzer_of(fleet, s, a, b)
    P = chain_profile(qa.serv_rate(), qa.K, [_lambda(fleet, s, r)])
    return bool(~P["over"][0] & ~P["tail"][0] & (b >= P["j"][0] + 2) & (qa.K < (1 << 23)))


def winner_mix(fleet, grid, cells, win):
    """(shared-chain winners, grid_kernel winners, servers whose winner ties with another accelerator's cell)."""
    S, A, B, R = fleet.n_servers, fleet.n_acc, grid.batch.size, grid.replicas.size
    feas = ((cells["flags"] >> 1) & 1).reshape(S, A, B, R)
    shared = kernel = ties = 0
    for s in range(S):
        w = win[s]
        if not w["feasible"] or fleet.srv_arrival_rpm[s] == 0:
            continue
        ri = int(np.nonzero(grid.replicas == w["replicas"])[0][0])
        bis = np.nonzero(grid.batch == w["batch"])[0]
        if cell_shares_row(fleet, s, int(w["acc"]), int(w["batch"]), int(w["replicas"])):
            shared += 1
        else:
            kernel += 1
        others = [a for a in range(A) if a != w["acc"] and feas[s, a, bis, ri].any()]
        ties += bool(others)
    return shared, kernel, ties


INV_BATCH = [8, 16, 32, 64, 128, 256]  # Bmax = 256
INV_REPLICAS = [1, 2, 3]


def invariant_fleet():
    """One accelerator, beta = gamma = 0, alpha = 1 and delta = 1/4, so the service rate of one busy server is 4/5
    and lambda of one replica sweeps 1e-7 .. 1e-5 (exact, by _rpm_for_lambda); the replica levels divide it further.
    Every row's chain ends within a few states: every cell of the grid shares its row.  delta > 0 makes the prefill
    time, and so the TTFT, follow the effective concurrency, which follows float32(in_serv) ulp by ulp."""
    return _fleet(1.0, 0.0, [_reachable_rpm(x) for x in np.geomspace(1e-7, 1e-5, 48)], 8, delta=0.25)


def _reachable_rpm(lam):
    """_rpm_for_lambda of the first float32 at or above lam that some arrival rate reaches exactly."""
    x = f32(lam)
    for _ in range(64):
        try:
            return _rpm_for_lambda(x)
        except AssertionError:
            x = np.nextafter(x, f32(np.inf))
    raise AssertionError(lam)


def tiny_acc_case():
    """The f0 guard of row_invariant: alpha = 2^-58 makes servRate[0] = 2^58 and lambda = 2^-60 (both inside
    solve_row's [2^-60, 2^60] windows), so acc ~ lambda / servRate[0] = 2^-118 < 1e-30 and the row takes the general
    branch however small 1 - sumP is.  Batch sizes 4 and 8 share the row (the chain ends at state 2)."""
    fleet = _fleet([2.0 ** -58, 2.0 ** -57, 1.0], 0.0, [_rpm_for_lambda(2.0 ** -60)] * 2 + [_rpm_for_lambda(1e-6)], 4)
    return fleet, Grid([1, 4, 8], [1])


def row_stats(fleet, grid):
    """Pass 2 of the reference (mm1modelstatedependent.go:44-55, 107-112) over chain_profile's pass-1 states, for
    every (server, replica level) row of a one-accelerator fleet at N = Bmax: p[n] / sum, then acc = sum of i p[i]
    and sumP = p[0] + ... + p[N] in that order.  Returns dict of arrays over rows (server-major)."""
    Bmax = int(grid.batch.max())
    out = {k: [] for k in ("s", "r", "lam", "acc", "m", "j", "shared_from", "q")}
    for s in range(fleet.n_servers):
        qa = _analyzer_of(fleet, s, 0, Bmax)
        lams = np.array([_lambda(fleet, s, int(r)) for r in grid.replicas], np.float32)
        P = chain_profile(qa.serv_rate(), qa.K, lams, keep=True)
        q = P["p"] / P["sum"][None, :]
        acc = np.zeros(lams.size)
        sump = q[0].copy()
        for i in range(1, Bmax + 1):
            acc = acc + np.float64(i) * q[i]
            sump = sump + q[i]
        for k, r in enumerate(grid.replicas):
            out["s"].append(s)
            out["r"].append(int(r))
            out["lam"].append(lams[k])
            out["acc"].append(acc[k])
            out["m"].append(1.0 - sump[k])
            out["j"].append(int(P["j"][k]) if not P["tail"][k] else -1)
            out["shared_from"].append(int(P["j"][k]) + 2 if not P["tail"][k] else 1 << 30)
            out["q"].append(q[:, k])
    return {k: (np.array(v) if k != "q" else v) for k, v in out.items()}


def row_invariant_np(acc, m, Nmax):
    """wva_kernels.cuh row_invariant's test in float64 numpy: (holds, d, bound); the guard gives d = bound = nan."""
    f0 = f32(acc)
    if not (f32(1e-30) < f0 < f32(1e30)):
        return False, np.nan, np.nan
    up, dn = np.nextafter(f0, f32(np.inf)), np.nextafter(f0, f32(0))
    hi_b = 0.5 * (np.float64(f0) + np.float64(up))
    lo_b = 0.5 * (np.float64(dn) + np.float64(f0))
    d = min(hi_b - acc, acc - lo_b)
    bound = 2.0 * (abs(m) * np.float64(Nmax)) + acc * 2.0 ** -50
    return bool(d > bound), d, bound


def row_classes(fleet, grid):
    """Class of every shared row: 'a' invariant, 'b' general with float32(in_serv) constant over the row's shared
    batch sizes, 'c' general with float32(in_serv) varying, 'guard' acc below the f0 guard; plus 'near-' / 'near+'
    for rows whose distance d lies in (0.5, 1] / (1, 2) times the bound."""
    st = row_stats(fleet, grid)
    Bmax = int(grid.batch.max())
    cls, near, vals = [], [], []
    for k in range(st["s"].size):
        bs = [int(b) for b in grid.batch if b >= st["shared_from"][k]]
        acc, m = st["acc"][k], st["m"][k]
        v = [f32(acc + m * np.float64(b)) for b in bs]
        vals.append(v)
        if not bs:
            cls.append(None)
            near.append(None)
            continue
        inv, d, bound = row_invariant_np(acc, m, Bmax)
        if np.isnan(d):
            cls.append("guard")
        else:
            cls.append("a" if inv else ("b" if len(set(v)) == 1 else "c"))
        ratio = d / bound if not np.isnan(d) else 0.0
        near.append("near-" if 0.5 < ratio <= 1 else ("near+" if 1 < ratio < 2 else None))
    st["cls"], st["near"], st["in_serv"] = cls, near, vals
    return st


def _winner_of(oracle_mod, fleet, s):
    _, w = oracle_mod.grid_solve(fleet.take_servers([s]), Grid(INV_BATCH, INV_REPLICAS), want_cells=False)
    return int(w[0]["feasible"]), int(w[0]["replicas"]), int(w[0]["batch"])


@functools.lru_cache(maxsize=None)
def invariant_case():
    """invariant_fleet with one server's slo_ttft set to the oracle's TTFT of a class-(c) cell that then wins: a
    one-ulp error in that cell flips its feasibility and the server's winner.  Returns (fleet, grid, server, cell)."""
    import oracle
    fleet, grid = invariant_fleet(), Grid(INV_BATCH, INV_REPLICAS)
    st = row_classes(fleet, grid)
    cells, _ = oracle.grid_solve(fleet, grid, want_cells=True)
    ttft = cells["ttft"].reshape(fleet.n_servers, 1, len(INV_BATCH), len(INV_REPLICAS))
    for k in np.nonzero(np.array([c == "c" for c in st["cls"]]))[0]:
        s, r = int(st["s"][k]), int(st["r"][k])
        ri = INV_REPLICAS.index(r)
        for bi, b in enumerate(INV_BATCH):
            t = f32(ttft[s, 0, bi, ri])
            if not t > 0:
                continue
            trial = fleet.take_servers(np.arange(fleet.n_servers))
            trial.srv_slo_ttft[s] = t
            if _winner_of(oracle, trial, s) != (1, r, b):
                continue
            trial.srv_slo_ttft[s] = np.nextafter(t, f32(0))
            if _winner_of(oracle, trial, s) == (1, r, b):
                continue
            trial.srv_slo_ttft[s] = t
            return trial, grid, s, (r, b)
    raise AssertionError("no class-(c) cell decides its server's winner")


def grid_fallback_case():
    """N = 1024, c = 1, x = lambda from 760 to 1000: the chains overflow float64, so grid_kernel bails and
    grid_fallback re-runs every cell on the stored vector."""
    xs = np.linspace(760.0, 1000.0, 300)
    return _fleet(1.0, 0.0, [_reachable_rpm(x) for x in xs], 1024), Grid([1024], [1])


def sweep_fallback_fleet():
    return _fleet(1.0, 0.0, [600.0], 1024)


SWEEP_FB_RATES = 1024


def size_fallback_fleet():
    """overflow_search_fleet's two servers, 130 times each: 260 candidates whose ITL bisection overflows float64
    (test_overflow_search_cases_bail_inside_the_search), each re-run by size_fallback."""
    return overflow_search_fleet(7.55, 0.0).take_servers(np.arange(260) % 2)


def _three_ways(engine, fleet, grid, cells_o, win_o, what):
    """With the cell table (cells and winners against the oracle), without it (winners against the oracle), and the
    pruned winners against the cell-table winners byte for byte."""
    cells_g, win_c = engine.grid_solve(fleet, grid, want_cells=True)
    _cells_equal(cells_g, cells_o, what)
    assert_allocs_equal(win_c, win_o, f"{what}: winners (cell table)")
    _, win_p = engine.grid_solve(fleet, grid)
    assert_allocs_equal(win_p, win_o, f"{what}: winners (pruned)")
    _same_winners(win_p, win_c, f"{what}: pruned vs cell table")


def _same_winners(a, b, what):
    for f in ALLOC_FIELDS:
        x, y = np.asarray(getattr(a, f)), np.asarray(getattr(b, f))
        assert x.dtype == y.dtype and np.array_equal(x.view(np.uint8), y.view(np.uint8)), f"{what}: field {f}"


def check_pruning(engine, oracle_mod, fleet, grid, what):
    _, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=False)
    _, win_p = engine.grid_solve(fleet, grid)
    _, win_c = engine.grid_solve(fleet, grid, want_cells=True)
    assert_allocs_equal(win_p, win_o, what + " (pruned)")
    _same_winners(win_p, win_c, what + ": pruned vs cell table")


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


def check_summary(engine, oracle_mod, f, win_o):
    got = engine.summarize(f.n_types)
    t = oracle_mod.allocate_by_type(f, win_o)
    d = oracle_mod.allocation_diffs(f, win_o)
    assert np.array_equal(got["by_type"]["present"], t["present"].astype(np.uint8))
    assert np.array_equal(got["by_type"]["count"], t["count"])
    assert np.array_equal(got["by_type"]["limit"], t["limit"])
    assert np.array_equal(got["by_type"]["cost"].view(np.uint32), np.ascontiguousarray(t["cost"]).view(np.uint32))
    for k_g, k_o in (("old_acc", "old_acc"), ("new_acc", "new_acc"), ("old_replicas", "old_replicas"),
                     ("new_replicas", "new_replicas")):
        assert np.array_equal(got["diff"][k_g], d[k_o]), k_g
    assert np.array_equal(got["diff"]["cost"].view(np.uint32), np.ascontiguousarray(d["cost_diff"]).view(np.uint32))
    return t, d


DELTA = 1e-5
XS = np.concatenate([np.arange(466.0, 482.0, 0.25), np.arange(604.0, 632.0, 0.125), np.arange(690.0, 740.0, 2.5)])
MAIN_N = (1024, 900)
LONG_XS = np.arange(612.0, 613.5, 0.5)  # the K >= 2^23 candidate's final solves, around the pass-2 IEEE band
EDGE_N = 16
EDGE_XS = (0.5, 3.0, 9.0)
LAM_EDGE_ALPHAS = (2.0 ** 50, 2.0 ** 52, 2.0 ** 54)


@functools.lru_cache(maxsize=None)
def _qa(N, alpha, delta, in_tok, out_tok, ratio):
    return _analyzer(N, alpha, 0.0, delta, in_tok, out_tok, ratio)


def _model(fleet, s, row=None):
    """(N, alpha, delta, in, out, ratio) of server s's only pair; row: (in, out) in place of the fleet's tokens."""
    it, ot = (int(fleet.srv_in_tokens[s]), int(fleet.srv_out_tokens[s])) if row is None else row
    return (int(fleet.srv_max_batch[s]), float(fleet.perf_alpha[s, 0]), float(fleet.perf_delta[s, 0]), it, ot,
            int(fleet.max_queue_to_batch_ratio))


def _main_fleet(n=MAIN_N, delta=DELTA):
    """One server per batch size, alpha = 1, no target, min_replicas 1, queue ratio 10."""
    return _fleet(1.0, 0.0, np.ones(len(n)), list(n), delta=delta, ratio=SIZE_RATIO)


def _x_rpm(xs):
    """Arrival rates whose one-replica lambda is exactly f32(x) (x = lambda at alpha = 1)."""
    return np.array([_rpm_for_lambda(f32(x)) for x in xs], np.float32)


def _edge_fleet():
    """N = 16, delta = 0: the four rate-edge models (one server each) and the three lambda-edge models."""
    alphas = [a for a, _ in _rate_edge_models(EDGE_N)] + list(LAM_EDGE_ALPHAS)
    return _fleet(alphas, 0.0, np.ones(len(alphas)), EDGE_N, ratio=SIZE_RATIO)


def _edge_rpm(fleet):
    """[3, S] rows of the edge fleet: x in EDGE_XS on the rate-edge servers; lambda on 2^-60, one ulp below, on
    2^-60 on the lambda-edge servers."""
    cols = []
    for s in range(fleet.n_servers):
        c = np.float64(f32(fleet.perf_alpha[s, 0]))
        if s < 4:
            cols.append([_rpm_for_lambda(x / c) for x in EDGE_XS])
        else:
            cols.append([_rpm_for_lambda(v) for v in (2.0 ** -60, BELOW(2.0 ** -60), 2.0 ** -60)])
    return np.array(cols, np.float32).T.copy()


def load_cases():
    """(fleet, rpm [L, S]) of the load grid: the main fleet at XS (both servers), the K >= 2^23 candidate at
    LONG_XS, the edge fleet."""
    main = _main_fleet()
    rpm = np.repeat(_x_rpm(XS)[:, None], main.n_servers, axis=1)
    long = _fleet(1.0, 0.0, [1.0], [682], delta=0.0, ratio=LONG_RATIO)
    edge = _edge_fleet()
    return [(main, rpm), (long, _x_rpm(LONG_XS)[:, None].copy()), (edge, _edge_rpm(edge))]


def profile_cases():
    """(fleet, rows): lambda fixed at 1 req/ms (rpm 60000), rows of perf_alpha = XS, so x = alpha; the edge models
    with their own rate and alpha fixed, and the lambda-edge models at lambda = 2^-60 with alpha 2^50 .. 2^54."""
    main = _main_fleet()
    main.srv_arrival_rpm[:] = f32(60000.0)
    alpha = np.repeat(XS.astype(np.float32)[:, None, None], main.n_servers, axis=1)
    out = [(main, {"perf_alpha": alpha})]
    # edge: one server per (rate-edge model, x) and per lambda edge; rows of alpha (3 rows)
    ea, erpm, rows = [], [], []
    for a, _ in _rate_edge_models(EDGE_N):
        c = np.float64(f32(a))
        for x in EDGE_XS:
            ea.append(a)
            erpm.append(_rpm_for_lambda(x / c))
            rows.append([a] * 3)
    for lam in (2.0 ** -60, BELOW(2.0 ** -60)):
        ea.append(LAM_EDGE_ALPHAS[0])
        erpm.append(_rpm_for_lambda(lam))
        rows.append(list(LAM_EDGE_ALPHAS))
    edge = _fleet(ea, 0.0, erpm, EDGE_N, ratio=SIZE_RATIO)
    out.append((edge, {"perf_alpha": np.array(rows, np.float32).T[:, :, None].copy()}))
    return out


def _ttft_targets(qa, xs):
    return [f32(qa.eval_ttft(float(f32(x)))[1]) for x in xs]


def slo_cases():
    """(fleet, (itl, ttft, tps) [L, S]): the main fleet at 60 req/min with TTFT rows whose searched lambda* lands on
    XS (all of its E(sum) 680 block, every other x above it), then TPS-only rows whose final rate is x = XS (lambda* =
    0.9 lambda_max overflows, so these items run in the stored re-run); the edge fleet with TPS-only rows; the
    K >= 2^23 candidates with one TPS row."""
    main = _main_fleet()
    main.srv_arrival_rpm[:] = 60.0
    S = main.n_servers
    qa = _qa(*_model(main, 0))
    ttft = np.array(_ttft_targets(qa, np.concatenate([XS[XS < 500], XS[XS > 500][::2]])), np.float32)
    L1 = ttft.size
    tps = (f32(2000) * XS.astype(np.float32)).astype(np.float32)
    L = L1 + tps.size
    itl_r = np.zeros((L, S), np.float32)
    ttft_r = np.zeros((L, S), np.float32)
    tps_r = np.zeros((L, S), np.float32)
    ttft_r[:L1] = ttft[:, None]
    tps_r[L1:] = tps[:, None]
    out = [(main, (itl_r, ttft_r, tps_r))]
    edge = _edge_fleet()
    et = np.zeros((3, edge.n_servers), np.float32)
    for s in range(edge.n_servers):
        a = float(edge.perf_alpha[s, 0])
        if s < 4:
            ls = float(_lam_star(_qa(EDGE_N, a, 0.0, 1, 2, SIZE_RATIO)))
            et[:, s] = [f32(2.0 * ls * 1000.0 * fr) for fr in (0.2, 0.5, 0.9)]
        else:
            et[:, s] = [f32(np.float64(f32(v)) * 2000.0) for v in (2.0 ** -60, BELOW(2.0 ** -60), 2.0 ** -60)]
    out.append((edge, (np.zeros_like(et), np.zeros_like(et), et)))
    lq = long_queue_fleet().take_servers(np.array([0, 1]))
    tp = lq.srv_slo_tps[None, :].copy()
    out.append((lq, (np.zeros_like(tp), np.zeros_like(tp), tp)))
    return out


def _alpha_for(N, which, edge, below):
    """A float32 alpha whose lambda_min (which 0) or lambda_max (which 1) is exactly edge, or with below, the
    nearest reachable float32 under it (delta = 0)."""
    a0 = int(np.array([0.001 / edge if which == 0 else N * 0.999 / edge], np.float32).view(np.uint32)[0])
    for k in sorted(range(-512, 513), key=abs):
        a = np.array([a0 + k], np.uint32).view(np.float32)[0]
        v = lam_range(_qa(N, float(a), 0.0, 1, 2, SIZE_RATIO))[which]
        if (v < f32(edge) and v >= f32(edge * (1 - 2.0 ** -20))) if below else v == f32(edge):
            return float(a)
    raise AssertionError(f"no alpha puts lambda {'min max'.split()[which]} on {edge!r} (below: {below})")


def bounds_cases():
    """Fleets of wva_slo_bounds: N from 465 to 481 (E(sum) 680 at lambda_max), 608 to 632 (E(max p) 880, E(sum) 900)
    and every other N from 700 to 740 (float64 overflow), each at delta 1e-5 .. 6e-5; the rate edges at N = 16, 24
    and 32; lambda_min on 2^-60 and just below, lambda_max on 2^60 and just below."""
    Ns = list(range(465, 481)) + list(range(608, 632)) + list(range(700, 740, 2))
    rows = [(N, d) for N in Ns for d in (1e-5, 2e-5, 3e-5, 4e-5, 5e-5, 6e-5)]
    main = _fleet(1.0, 0.0, np.full(len(rows), 600.0), [r[0] for r in rows], delta=[r[1] for r in rows],
                  ratio=SIZE_RATIO)
    ea, en = [], []
    for N in (16, 24, 32):
        for a, _ in _rate_edge_models(N):
            ea.append(a)
            en.append(N)
        for which, edge in ((0, 2.0 ** -60), (1, P60)):
            for below in (False, True):
                ea.append(_alpha_for(N, which, edge, below))
                en.append(N)
    edge = _fleet(ea, 0.0, np.full(len(ea), 600.0), en, ratio=SIZE_RATIO)
    return [main, edge]


# the solves a level call's tail runs, with their profiles (test_gpu_tail_windows, test_gpu_margin_edges)
class _Solves:
    """(rates, K, lambda, candidate) of every streaming solve a tail runs, profiled in one vectorised pass."""

    def __init__(self):
        self.sr, self.K, self.lam, self.cand = [], [], [], []

    def add(self, qa, lam, cand):
        self.sr.append(qa.serv_rate())
        self.K.append(qa.K)
        self.lam.append(f32(lam))
        self.cand.append(cand)

    def profile(self):
        P = chain_profile(self.sr, np.array(self.K), np.array(self.lam, np.float32))
        P["lam"] = np.array(self.lam, np.float32)
        P["sr0"] = np.array([r[0] for r in self.sr], np.float32)
        P["srN"] = np.array([r[-1] for r in self.sr], np.float32)
        P["K"] = np.array(self.K)
        P["cand"] = list(self.cand)
        return P


def _final_lam(rpm, tps, out_tok, replicas):
    """The final Analyze's lambda: totalRate / replicas in req/s, over 1000 (allocation.go:134-153)."""
    total = f32(f32(tps) / f32(out_tok)) if tps > 0 else f32(f32(rpm) / f32(60))
    return _lam_of_rate(f32(total / f32(replicas)))


def _bails(P):
    """The solves that leave the streaming windows: a rate or lambda outside [2^-60, 2^60), p at 2^880 or above, the
    sum at 2^900 or above, or a float64 overflow."""
    def inside(v):
        return (v >= f32(2.0 ** -60)) & (v < f32(P60))
    return P["over"] | (P["emax"] >= 880) | (P["esum"] >= 900) | ~inside(P["lam"]) | ~inside(P["sr0"]) | \
        ~inside(P["srN"])


def tail_bands(P):
    b = wide_bands(P, steep=False)
    for k, v in _rate_bands(P).items():
        b[k] = (int(v),) * 2
    return b


# ---- the load margins' records at the exponent windows (test_gpu_margin_edges) -------------------------------------
BELOW_NS = list(range(465, 482)) + list(range(608, 633)) + list(range(700, 741, 2))  # lambda ~ rateStar
ABOVE_NS = list(range(934, 966)) + list(range(1208, 1290)) + list(range(1380, 1481, 5))  # ~ rateStar / 2
MARGIN_DELTAS = (1e-5, 3e-5, 5e-5)
ABOVE_DELTAS = (1e-5, 2e-5, 3e-5, 4e-5, 5e-5, 6e-5)  # E(sum) 900 is narrow at rateStar / 2


def _rate_star(fleet, s):
    """rateStar (req/s) of server s's only pair: Size's throughput without a target."""
    err, _, met, _ = _qa(*_model(fleet, s)).size(0.0, 0.0, 0.0)
    assert err == 0
    return f32(met["throughput"])


def _step_rows(fleet, rows):
    """(rate, lo, hi) [L, S] from rows of (r, lo, hi) multiples of each server's first replica step 60 rateStar."""
    step = np.array([60.0 * float(_rate_star(fleet, s)) for s in range(fleet.n_servers)])
    m = np.asarray(rows, np.float64)
    return tuple((m[:, k:k + 1] * step[None, :]).astype(np.float32) for k in range(3))


def _grid_fleet(ns, deltas=MARGIN_DELTAS):
    rows = [(N, d) for N in ns for d in deltas]
    return _fleet(1.0, 0.0, np.ones(len(rows)), [r[0] for r in rows], delta=[r[1] for r in rows], ratio=SIZE_RATIO)


def margin_cases():
    """(name, fleet, rate, lo, hi) of wva_load_margins whose records' solves sit at the exponent windows.

    at: the load grid's main rows (load_cases), every other level with a one-point window and the others with a
        window of +-1 % holding no step; the edge fleet's rows with +-0.1 % windows.
    below: BELOW_NS x MARGIN_DELTAS at 1.5 steps (window [0.5, 1.5] steps: below is one replica at the float under
        the step, lambda just under rateStar) and at 99.5 steps (window [98.5, 100.5]: all three records within 1 %
        of rateStar).
    above: ABOVE_NS x ABOVE_DELTAS at half a step (window [0.5, 1.5] steps: above is two replicas at the step,
        lambda just over rateStar / 2).
    edge steps: the edge fleet at 1.5, 2.5 and 3.5 steps with windows down to the step below, and at 0.5, 1.5 and
        2.5 steps with windows up to the step above."""
    (main, rpm), _, (edge, erpm) = load_cases()
    lo, hi = rpm.copy(), rpm.copy()
    lo[1::2] = (rpm[1::2] * f32(0.99)).astype(np.float32)
    hi[1::2] = (rpm[1::2] * f32(1.01)).astype(np.float32)
    out = [("at main", main, rpm, lo, hi),
           ("at edge", edge, erpm, (erpm * f32(0.999)).astype(np.float32), (erpm * f32(1.001)).astype(np.float32))]
    fb = _grid_fleet(BELOW_NS)
    out.append(("below", fb) + _step_rows(fb, [(1.5, 0.5, 1.5), (99.5, 98.5, 100.5)]))
    fa = _grid_fleet(ABOVE_NS, ABOVE_DELTAS)
    out.append(("above", fa) + _step_rows(fa, [(0.5, 0.5, 1.5)]))
    out.append(("edge steps", edge) + _step_rows(edge, [(k + 1.5, k + 0.5, k + 1.5) for k in range(3)] +
                                                  [(k + 0.5, k + 0.5, k + 1.5) for k in range(3)]))
    return out


# ---- the bisection brackets of iv_advance and mg_start (test_gpu_margin_edges) -------------------------------------
BRACKET_RATIO = 1000  # K = 16000 at N = 16: the blocking at lambda_max is below float32's ulp, so rateStar = RateRange.Max
F32_MAX_BITS = 0x7F7FFFFF


def _alpha_for_rate_max(rmax):
    """A float32 alpha (N = 16, delta 0) whose RateRange.Max is near rmax (req/s)."""
    return float(f32(16 * 0.999 * 1000 / rmax))


def bracket_fleet():
    """N = 16, queue ratio 1000, one server per model: 0 and 2 with alpha 1 (rateStar = RateRange.Max ~ 16,000
    req/s), 1 with RateRange.Max ~ 3.2e29 req/s, so that counts past 2^24 lie just below float32's maximum and the
    bisections' estimates reach 3e38.  Server 2 has min_replicas 3."""
    f = _fleet([1.0, _alpha_for_rate_max(3.2e29), 1.0], 0.0, np.ones(3), 16, ratio=BRACKET_RATIO)
    f.srv_min_replicas[2] = 3
    return f


def _gate_points(fleet, s, start, gate, k):
    """The first k float32 rates at or above start whose pair state has the given gate (levels.pair_state)."""
    from tests.levels import from_bits, pair_state, u32_bits
    rs = _rate_star(fleet, s)
    rmax = f32(_qa(*_model(fleet, s)).rate_range()[1])
    out, b = [], u32_bits(f32(start))
    while len(out) < k and b <= F32_MAX_BITS:
        if pair_state(fleet, s, rs, rmax, from_bits(b))[1] == gate:
            out.append(b)
        b += 1
    assert len(out) == k, (s, gate)
    return out


def bracket_cases():
    """(fleet, rate, lo, hi) [4, 3] on bracket_fleet.  Servers 0 and 1: two rates of the gate-2 states past 2^24
    replicas (float32(total / float32(nrep)) rounds above RateRange.Max), a gate-1 rate among them, each with a
    window of +-100 floats, and one replica at half a step.  Server 2 (min_replicas 3): windows from the smallest
    positive rate, at 1.5 and 2.5 steps, and one from a quarter step."""
    from tests.levels import TINY, from_bits
    fleet = bracket_fleet()
    L, S = 4, fleet.n_servers
    rate, lo, hi = (np.zeros((L, S), np.float32) for _ in range(3))
    for s in (0, 1):
        step = 60.0 * float(_rate_star(fleet, s))
        first = step * (2 ** 24 + 1)
        g2 = _gate_points(fleet, s, first, 2, 2)
        g1 = [b + 10 for b in _gate_points(fleet, s, first, 1, 1)]
        for l, b in enumerate(g2 + g1):
            rate[l, s], lo[l, s], hi[l, s] = from_bits(b), from_bits(b - 100), from_bits(b + 100)
        rate[3, s], lo[3, s], hi[3, s] = f32(0.5 * step), f32(0.25 * step), f32(0.75 * step)
    step = 60.0 * float(_rate_star(fleet, 2))
    for l, (r, b, t) in enumerate(((1.5, None, 1.5), (2.5, None, 3.5), (0.5, 0.25, 0.5), (0.5, 0.25, 0.5))):
        rate[l, 2], hi[l, 2] = f32(r * step), f32(t * step)
        lo[l, 2] = TINY if b is None else f32(b * step)
    return fleet, rate, lo, hi
