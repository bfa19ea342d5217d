"""Second, independent restatement of the reference hot path in numpy and Python scalars (TEST ONLY).

Purpose: cross-check the C oracle (oracle/wva_oracle.c), because beyond the reference's own KATs nothing pins float
outputs under load (SURVEY.md §4, §8c).  This file is written against the Go sources directly and shares no code with
the C oracle: float32 arithmetic is done with ``np.float32`` scalars (each operation rounds to binary32, no fused
multiply-add), and the float64 recurrence of mm1modelstatedependent.go:70-116 is a plain loop over Python floats,
which round every operation to binary64 exactly as Go's float64 does (only a division by zero, which Python raises
on, is spelled out as the IEEE result).

Where Go would run into a limit, the restatement says so instead of guessing: ``Unsupported`` is raised for a queue
model outside the CUDA library's domain (N above 2^20, or 2^31 states or more) and for a rescale loop that would
never terminate (NaN rates), which the Go code would spin in forever.
"""
from __future__ import annotations

import math
import sys

import numpy as np

F = np.float32
EPS = F(0.001)                 # queueanalyzer.go:8
SSF = F(0.1)                   # queueanalyzer.go:11
TOL = F(1e-6)                  # utils.go:8
MAX_IT = 100                   # utils.go:9
INF = math.inf
MAX_F64 = sys.float_info.max   # math.MaxFloat64 (mm1modelstatedependent.go:74)
INT64_MIN = -(1 << 63)
MAX_BATCH = 1 << 20            # largest N the CUDA library builds a model for
MAX_STATES = 1 << 31           # K = N + MaxQueueSize must fit an int32
# Each pass of the rescale loop (mm1modelstatedependent.go:84-89) divides p[0..n] by MaxFloat64 / K >= 2^992, so a
# finite ratio lambda / servRate brings p[n+1] back within three passes; more than this many means it never will.
RESCALE_PASSES = 64


class Unsupported(RuntimeError):
    """The input is outside what can be restated.  ``reason`` is one of

    * ``"states"``: a queue model of N >= 2^31 or K >= 2^31 states (Go's 64-bit int; the C oracle refuses it too);
    * ``"batch"``: a batch size N above 2^20 with fewer states (the CUDA library refuses it, the C oracle does not);
    * ``"rescale"``: the rescale loop of mm1modelstatedependent.go:84-89 would not terminate (a NaN rate, e.g.
      Analyze at 0/0 replicas).
    """

    def __init__(self, reason, what):
        super().__init__(f"{reason}: {what}")
        self.reason = reason


def gmin(a, b):  # Go builtin min on floats: NaN if either is NaN, -0 < +0
    if np.isnan(a) or np.isnan(b):
        return F(np.nan)
    if a == 0 and b == 0:
        return a if np.signbit(a) else b
    return a if a < b else b


def gmax(a, b):
    if np.isnan(a) or np.isnan(b):
        return F(np.nan)
    if a == 0 and b == 0:
        return b if np.signbit(a) else a
    return a if a > b else b


def go_int(x):
    """int(x) for a float64 x, as Go compiles it on amd64 (CVTTSD2SQ): NaN, +-Inf and every value outside
    [-2^63, 2^63) give the "integer indefinite" MinInt64, the rest truncate toward zero."""
    x = float(x)
    if not (-9223372036854775808.0 <= x < 9223372036854775808.0):
        return INT64_MIN
    return int(x)


def _i64(x):
    """x wrapped to Go's 64-bit int."""
    return ((int(x) + (1 << 63)) % (1 << 64)) - (1 << 63)


def _f32i(x):
    """float32(x) for a Go int x: one rounding, straight from the 64-bit integer."""
    return np.array([x], np.int64).astype(np.float32)[0]


def _go_quo(x, y):
    """Go's integer division, truncating toward zero."""
    q = abs(x) // abs(y)
    return q if (x >= 0) == (y > 0) else -q


def _div0(a, b):
    """a / b for b == +-0 under IEEE rules (Python raises instead)."""
    if a != a or a == 0:
        return math.nan
    return math.copysign(INF, a) * math.copysign(1.0, b)


def queue_states(N, ratio):
    """K = N + N * MaxQueueToBatchRatio in Go's int (allocation.go:85-87, queueanalyzer.go:121) -> (max_queue, K),
    or Unsupported when the model is outside the domain restated here."""
    N, ratio = int(N), int(ratio)
    K = N + N * ratio
    if N >= MAX_STATES or K >= MAX_STATES:
        raise Unsupported("states", f"N = {N}, K = {K}")
    if N > MAX_BATCH:
        raise Unsupported("batch", f"N = {N}")
    return N * ratio, K


class QA:
    """QueueAnalyzer + MM1ModelStateDependent (queueanalyzer.go:14-131, mm1modelstatedependent.go)."""

    def __init__(self, N, Q, alpha, beta, gamma, delta, in_tok, out_tok):
        self.N, self.Q = N, Q
        self.a, self.b, self.g, self.d = F(alpha), F(beta), F(gamma), F(delta)
        self.it, self.ot = int(in_tok), int(out_tok)
        self.sr = np.zeros(N, np.float32)
        with np.errstate(all="ignore"):
            for n in range(1, N + 1):  # BuildModel :103-113
                pre = self.prefill(F(n))
                nd = self.ot - 1
                if self.it == 0 and self.ot == 1:
                    nd = 1
                dec = F(nd) * self.decode(F(n))
                self.sr[n - 1] = F(n) / (pre + dec)
            self.rmin = (self.sr[0] * EPS) * F(1000)
            self.rmax = (self.sr[N - 1] * (F(1) - EPS)) * F(1000)
        self._sr = [float(x) for x in self.sr]  # float64(servRate[n]): exact
        self.K = N + Q
        self._p = [0.0] * (self.K + 1)  # make([]float64, K+1) (mm1kmodel.go:22)
        self.valid = False

    @property
    def p(self):
        return np.array(self._p, np.float64)

    def reset(self):
        """A freshly built model (p all zero), as the sweep analyses every rate on."""
        self._p = [0.0] * (self.K + 1)

    def prefill(self, batch):  # :257-262
        if self.it == 0:
            return F(0)
        return self.g + (self.d * F(self.it)) * batch

    def decode(self, batch):  # :264-266
        return self.a + self.b * batch

    def effconc(self, serv):  # :296-302
        with np.errstate(all="ignore"):
            tok = F(self.ot - 1)
            num = serv - (self.g + self.a * tok)
            den = (self.d * F(self.it)) + (self.b * tok)
            n = num / den
        return gmin(gmax(n, F(0)), F(self.N))

    def solve(self, lam, mu=F(1)):  # queuemodel.go:27-37
        lam, mu = F(lam), F(mu)
        rho = F(1) - F(self._p[0])  # ComputeRho reads the previous solve's p[0] (mm1modelstatedependent.go:33-35)
        if rho < 0 or rho >= F(self.K) or lam < 0 or mu <= 0:
            self.valid = False
            return
        self.valid = True
        K, N, p, sr = self.K, self.N, self._p, self._sr
        lamd = float(lam)
        last = sr[N - 1]
        p[0] = 1.0
        scale = MAX_F64 / K
        for n in range(K):  # mm1modelstatedependent.go:77-90
            s = sr[n] if n < N else last
            try:
                x = p[n] * lamd / s
            except ZeroDivisionError:
                x = _div0(p[n] * lamd, s)
            passes = 0
            while not (0.0 <= x < INF):  # p < 0 || IsInf(p, 0) || IsNaN(p)
                passes += 1
                if passes > RESCALE_PASSES:
                    raise Unsupported("rescale", f"lambda = {lamd!r}, state {n + 1}, rate {s!r}")
                for i in range(n + 1):
                    p[i] /= scale
                try:
                    x = p[n] * lamd / s
                except ZeroDivisionError:
                    x = _div0(p[n] * lamd, s)
            p[n + 1] = x
        tot = 0.0
        for n in range(K + 1):  # :93-105
            tot += p[n]
            if tot < 0 or tot == INF or tot == -INF:
                tot = 0.0
                for i in range(K + 1):
                    p[i] /= scale
                    if i <= n:
                        tot += p[i]
        if tot == 0:  # :108-112
            p[:] = [_div0(v, tot) for v in p]
        else:
            p[:] = [v / tot for v in p]
        in_sys = 0.0
        sp = p[0]
        for i in range(1, N + 1):  # :47-55, up to and including i == num
            in_sys += i * p[i]
            sp += p[i]
        in_srv = in_sys + (1.0 - sp) * N
        for i in range(N + 1, K + 1):
            in_sys += i * p[i]
        with np.errstate(all="ignore"):
            self.num_serv = F(in_srv)
            num_sys = F(in_sys)
            self.tput = lam * (F(1) - F(p[K]))  # :59-66
            self.resp = num_sys / self.tput
            self.serv = self.num_serv / self.tput
            w = self.resp - self.serv
            self.wait = F(0) if w < 0 else w

    def analyze(self, rate):  # queueanalyzer.go:134-174
        rate = F(rate)
        if rate <= 0 or rate > self.rmax:
            return None
        with np.errstate(all="ignore"):
            self.solve(rate / F(1000))
            if not self.valid:
                return None
            e = self.effconc(self.serv)
            rho = gmin(gmax(self.num_serv / F(self.N), F(0)), F(1))
            return {"throughput": self.tput * F(1000), "wait": self.wait, "prefill": self.prefill(e),
                    "itl": self.decode(e), "rho": rho}

    def eval(self, which, x):  # :270-290
        self.solve(x)
        if not self.valid:
            raise ValueError
        e = self.effconc(self.serv)
        with np.errstate(all="ignore"):
            return self.wait + self.prefill(e) if which == "ttft" else self.decode(e)


def within(x, v, tol):  # utils.go:12-20
    if x == v:
        return True
    if v == 0 or tol < 0:
        return False
    with np.errstate(all="ignore"):
        return abs(float((x - v) / v)) <= float(tol)


def bsearch(xmin, xmax, target, fn):  # utils.go:26-70 -> (x, ind)
    xmin, xmax, target = F(xmin), F(xmax), F(target)
    if xmin > xmax:
        raise ValueError
    ys = []
    for x in (xmin, xmax):
        y = fn(x)
        ys.append(y)
        if within(y, target, TOL):
            return x, 0
    inc = ys[0] < ys[1]
    if (inc and target < ys[0]) or (not inc and target > ys[0]):
        return xmin, -1
    if (inc and target > ys[1]) or (not inc and target < ys[1]):
        return xmax, 1
    xs = F(0)
    for _ in range(MAX_IT):
        xs = F(0.5) * (xmin + xmax)
        y = fn(xs)
        if within(y, target, TOL):
            break
        if (inc and target < y) or (not inc and target > y):
            xmax = xs
        else:
            xmin = xs
    return xs, 0


def size(qa: QA, ttft, itl, tps):  # queueanalyzer.go:185-255 -> metrics dict or None
    ttft, itl, tps = F(ttft), F(itl), F(tps)
    if ttft < 0 or itl < 0 or tps < 0:
        return None
    lmin, lmax = qa.rmin / F(1000), qa.rmax / F(1000)
    try:
        l1 = lmax
        if ttft > 0:
            l1, ind = bsearch(lmin, lmax, ttft, lambda x: qa.eval("ttft", x))
            if ind < 0:
                return None
        l2 = lmax
        if itl > 0:
            l2, ind = bsearch(lmin, lmax, itl, lambda x: qa.eval("itl", x))
            if ind < 0:
                return None
    except ValueError:
        return None
    l3 = lmax * (F(1) - SSF) if tps > 0 else lmax
    lam = gmin(gmin(l1, l2), l3)
    return qa.analyze(lam * F(1000))


def _load_pair(f, s, a):
    """CreateAllocation's gates (allocation.go:42-70) -> model index, or None for a nil allocation."""
    if f.srv_arrival_rpm[s] < 0 or f.srv_in_tokens[s] < 0 or f.srv_out_tokens[s] < 0:
        return None
    m = int(f.srv_model[s])
    if m < 0 or not f.perf_present[m, a] or not f.srv_has_target[s]:
        return None
    return m


def _total_rate(f, s):  # allocation.go:134-139
    with np.errstate(all="ignore"):
        if F(f.srv_slo_tps[s]) == 0:
            return F(f.srv_arrival_rpm[s]) / F(60)
        return F(f.srv_slo_tps[s]) / F(int(f.srv_out_tokens[s]))


def _qa(f, s, a, m, N):
    """NewQueueAnalyzer for pair (s, a) at batch size N (allocation.go:87-114), or None when its checks refuse."""
    max_queue, _ = queue_states(N, f.max_queue_to_batch_ratio)
    if max_queue < 0:  # Configuration.check (queueanalyzer.go:305-311)
        return None
    return QA(int(N), max_queue, f.perf_alpha[m, a], f.perf_beta[m, a], f.perf_gamma[m, a], f.perf_delta[m, a],
              f.srv_in_tokens[s], f.srv_out_tokens[s])


def create_allocation(fleet, s, a):
    """allocation.go:27-163 on a Fleet -> dict (feasible, acc, replicas, batch, cost, itl, ttft, rho, max_rate)."""
    nil = {"feasible": 0}
    f = fleet
    m = _load_pair(f, s, a)
    if m is None:
        return nil
    ninst = int(f.perf_acc_count[m, a]) if f.perf_acc_count[m, a] > 0 else 1  # model.go:50-57
    if f.srv_arrival_rpm[s] == 0 or f.srv_out_tokens[s] == 0:  # zeroLoadAllocation :259-288
        nrep = int(f.srv_min_replicas[s])
        if nrep == 0:
            return {"feasible": 1, "acc": -1, "replicas": 0, "batch": 0, "cost": F(0), "itl": F(0), "ttft": F(0),
                    "rho": F(0), "max_rate": F(0)}
        mb = int(f.srv_max_batch[s]) if f.srv_max_batch[s] > 0 else int(f.perf_max_batch[m, a])
        al, be, ga, de = (F(f.perf_alpha[m, a]), F(f.perf_beta[m, a]), F(f.perf_gamma[m, a]), F(f.perf_delta[m, a]))
        with np.errstate(all="ignore"):
            pre = ga + de
            return {"feasible": 1, "acc": a, "replicas": nrep, "batch": mb,
                    "cost": F(f.acc_cost[a]) * _f32i(_i64(ninst * nrep)), "itl": al + be, "ttft": pre, "rho": F(0),
                    "max_rate": F(mb) / (pre + (al + be * F(mb)))}
    K = int(f.srv_out_tokens[s])
    N = int(f.srv_max_batch[s]) if f.srv_max_batch[s] > 0 else max(
        _go_quo(int(f.perf_max_batch[m, a]) * int(f.perf_at_tokens[m, a]), K), 1)
    qa = _qa(f, s, a, m, N)
    if qa is None:
        return nil
    met = size(qa, f.srv_slo_ttft[s], f.srv_slo_itl[s], f.srv_slo_tps[s])
    if met is None:
        return nil
    rate_star = met["throughput"]
    total = _total_rate(f, s)
    q = float(total) / float(rate_star) if rate_star != 0 else _div0(float(total), float(rate_star))
    nrep = go_int(math.ceil(q) if math.isfinite(q) else q)  # :140
    nrep = max(nrep, int(f.srv_min_replicas[s]))  # :141
    with np.errstate(all="ignore"):
        cost = F(f.acc_cost[a]) * _f32i(_i64(ninst * nrep))  # :144-145
        met2 = qa.analyze(total / _f32i(nrep))  # :148-149; 0 replicas give 0/0, whose rescale loop never ends
    if met2 is None:
        return nil
    return {"feasible": 1, "acc": a, "replicas": nrep, "batch": N, "cost": cost, "itl": met2["itl"],
            "ttft": met2["wait"] + met2["prefill"], "rho": met2["rho"], "max_rate": rate_star / F(1000)}


def grid_cell(fleet, s, a, b, r):
    """One cell of the candidate grid: Analyze (queueanalyzer.go:134-174) at totalRate / r (allocation.go:134-139,
    148) on the queue model with MaxBatchSize = b and MaxQueueSize = b * MaxQueueToBatchRatio, then the cell's SLO
    test: TTFT and ITL within their targets (a target of 0 is off), r at least the server's minimum replicas, and with
    a TPS target the per-replica lambda at most Size's stability limit lambdaMax * (1 - StabilitySafetyFraction)
    (queueanalyzer.go:231-234).  Pairs that Server.Calculate would not consider (server.go:70-82), CreateAllocation's
    nil gates and zero load (allocation.go:42-75) have no cell.

    -> dict(flags = analysed | feasible << 1, ttft, itl, rho, throughput), the floats 0 when not analysed."""
    f = fleet
    out = {"flags": 0, "ttft": F(0), "itl": F(0), "rho": F(0), "throughput": F(0)}
    if f.srv_keep_acc[s] and f.srv_cur_acc[s] != -1 and f.srv_cur_acc[s] != a:
        return out
    m = _load_pair(f, s, a)
    if m is None or f.srv_arrival_rpm[s] == 0 or f.srv_out_tokens[s] == 0:
        return out
    qa = _qa(f, s, a, m, b)
    if qa is None:
        return out
    with np.errstate(all="ignore"):
        rate = _total_rate(f, s) / F(r)
        met = qa.analyze(rate)
        if met is None:
            return out
        ttft, itl = met["wait"] + met["prefill"], met["itl"]
        slo_ttft, slo_itl = F(f.srv_slo_ttft[s]), F(f.srv_slo_itl[s])
        ok = ((slo_ttft == 0 or ttft <= slo_ttft) and (slo_itl == 0 or itl <= slo_itl)
              and r >= int(f.srv_min_replicas[s]))
        if F(f.srv_slo_tps[s]) > 0:
            ok = ok and rate / F(1000) <= (qa.rmax / F(1000)) * (F(1) - SSF)
    return {"flags": 1 | (2 if ok else 0), "ttft": ttft, "itl": itl, "rho": met["rho"],
            "throughput": met["throughput"]}
