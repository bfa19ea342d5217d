"""The level calls' tail kernels at the streaming solver's exponent windows, bit for bit against the oracle.

Six tail kernels run streaming solves of their own after phase 1 (DESIGN.md 3.2): load_kernel (wva_load_grid: the
final Analyze at totalRate / replicas), interval_tail (wva_load_intervals: the final Analyze at each interval start),
workload_kernel (wva_workload_grid / _trace, wva_profile_grid / _trace: the final Analyze), slo_kernel and
slo_trace_kernel (wva_slo_grid, wva_slo_trace: Analyze at lambda*, then the final Analyze) and bounds_tail
(wva_slo_bounds: Model.Solve at lambda_min and lambda_max, with no Analyze gate).  Each bails out of the windows of
``wva_device.cuh`` into its stored-vector re-run (``tail_item`` / ``tail_rerun`` in ``wva_size.cuh``).

test_gpu_windows explains why the size path cannot put its final Analyze on the 2^880 edge.  The tails can: with no
latency target lambda* = lambda_max, whose chain at alpha = 1 and queue ratio 10 leaves the p window from N ~ 620 on
(``_phase1_bails`` checks it for every candidate here), so phase 1 re-runs it on the stored vector and the tail's
solve at the caller's lambda is the first streaming solve there.  That lambda is placed exactly: by a level's or
tick's arrival rate (load, workload), by an interval's ``lo``, by a row of ``perf_alpha`` at a fixed rate (profile:
x = lambda * alpha), by a TTFT target whose bisection lands in a band or a TPS target that places the final rate
(SLO), and by N itself (bounds: lambda_max = 0.999 servRate[N-1]).

The fleets have beta = 0 and gamma = 0, so servRate[n-1] = n / (alpha + delta n) and x = lambda * alpha up to the
small bend of delta.  delta is 1e-5 rather than 0 on the fleets away from the rate edges: with beta = delta = 0 the
effective concurrency is 0 / 0 and every ITL and TTFT is NaN, which would leave the re-runs' latency columns unchecked
and gives the TTFT search nothing to bisect.  Which band a solve reaches is decided by ``chain_profile`` at the
float32 lambda the tail solves, formed from the oracle's records exactly as the oracle forms it; the CPU tests assert
at least three cases on each side of every edge, print the counts, and assert that each tail has a candidate with
items on both sides of an edge (some bail, some do not) and a call that bails on more than 128 items of different K
(the re-run kernels run 128 threads, so a thread re-runs several items on one scratch slot).

Bands per tail (E = binary exponent, "edge - 1 / edge"):

* load grid, load intervals, workload grid and trace, profile grid and trace: E(max p) 879 / 880, E(sum) 679 / 680
  and 899 / 900, the pass-2 IEEE path (sum in [2^882, 2^900), p < 2^880, states below 2^(E(sum) - 960) before
  termination), float64 overflow, servRate[0] and servRate[N-1] on 2^-60 / 2^60 and one ulp across, lambda on
  2^-60 and one ulp below.  The load grid also has a K >= 2^23 candidate whose final solve runs the pass-2 IEEE path.
* SLO grid and trace: the same, at the lambda* solve of TTFT rows (at 60 req/min, so the final Analyze is a small
  chain) and of TPS-only rows at the edge models.  slo_tail streams its final Analyze only after a lambda* solve that
  stayed inside the windows, so only those final solves are counted.  TPS-only rows on the main fleet (lambda* = 0.9
  lambda_max overflows float64) place the final rate on every band; there the whole item, final Analyze included,
  runs in slo_fallback's stored re-run.  The SLO grid also has two K >= 2^23 candidates (a TPS row on
  grid_cases.long_queue_fleet) whose lambda* solves run the pass-2 IEEE path.
* bounds: E(max p) 879 / 880, E(sum) 679 / 680 and 899 / 900 and float64 overflow at lambda_max; the rate edges and
  lambda_min exactly on 2^-60 and just below; lambda_max exactly on 2^60 and just below (the float32 values one ulp
  under a power of two are finer than the steps of lambda_min = 0.001 servRate[0] and lambda_max = 0.999
  servRate[N-1], so "just below" is the nearest one a float32 alpha reaches).

Not reachable, and so left out:
* a sum bail on its own: as on the size path the sum exceeds the peak by at most ~2^10 here, so the cases at
  E(sum) 900 have crossed the p edge already.
* the SLO tails' streaming final Analyze in the upper bands: it runs only after a lambda* solve inside the windows,
  at a lambda of at most that solve's throughput, so by the size path's argument (test_gpu_windows) it stays below
  where lambda* stayed.
* ITL rows that search: with beta = 0 ITL is alpha at every lambda, so an ITL search ends at a bound without
  bisecting; the SLO rows search TTFT.
* the pass-2 IEEE path on the bounds: lambda_max = 0.999 servRate[N-1] is the only large lambda they solve, and past
  state N its chain falls by only a factor 0.999 per state, so it reaches 2^(E(sum) - 960) only after ~6.6e5 states
  past the peak, at queue ratios above 1000, where each chain_profile and each oracle solve of the ~400 bounds
  candidates walks that whole chain.
* lambda exactly on 2^60 reaches the bounds' lambda_max (no Analyze gate) but, as on the size path, only with
  servRate[N-1] = lambda_max / 0.999 above the window: the solve bails on the rate whichever lambda edge it is at.
  Those cases are included; nothing separates the lambda window from the rate window there.
* steep crossings of 2^880: they need x above ~2600 at the crossing, where lambda_max of every candidate that has
  such a lambda overflows float64 already (as on the size path).
"""
from __future__ import annotations

import numpy as np
import pytest
from tests.grid_cases import (DELTA, MAIN_N, P60, SIZE_RATIO, XS, _concat, _edge_fleet, _edge_rpm, _fleet, _lam_of_rate,
                              _lam_star, _model, _qa, _rate_bands, _x_rpm, bounds_cases, chain_profile, f32, load_cases,
                              profile_cases, slo_cases, wide_bands)
from tests.levels import (LOAD, SLO, check_intervals, check_level_call, check_slo_bounds, lam_range, ref_grid,
                          ref_intervals, ref_slo_bounds, ref_trace)
from tests.util import assert_allocs_equal


FB_SLOTS = 128  # kFbBlocks * kFbThreads: the threads of every re-run kernel
# x = lambda * alpha of the levels: E(sum) 679 / 680 near x = 472; E(max p) 879 / 880, the pass-2 IEEE band and
# E(sum) 899 / 900 between 604 and 632; float64 overflow above ~705
# ---------------------------------------------------------------------------------------------------------------
# the solves a tail runs, with their profiles
# ---------------------------------------------------------------------------------------------------------------
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


def _add_finals(S, cand, fleet, rpm, tps, tokens, what):
    """The final solve of every feasible record of an [L, S] candidate block (A = 1)."""
    L = rpm.shape[0]
    c = cand.reshape(L, fleet.n_servers)
    for l in range(L):
        for s in range(fleet.n_servers):
            r = c[l, s]
            if not r["feasible"]:
                continue
            it, ot = tokens(l, s)
            S.add(_qa(*_model(fleet, s, (it, ot))), _final_lam(rpm[l, s], tps[l, s], ot, r["replicas"]),
                  (what, s, l))


def _phase1_bails(fleet, servers, tokens=lambda s: None):
    """Each given server's lambda* = lambda_max chain leaves the p window or overflows (on the chain's first 3 N
    states, which hold its peak): phase 1 re-runs it on the stored vector."""
    S = _Solves()
    for s in servers:
        m = _model(fleet, s, tokens(s))
        qa = _qa(*m)
        S.sr.append(qa.serv_rate())
        S.K.append(min(qa.K, 3 * m[0]))
        S.lam.append(_lam_star_max(qa))
        S.cand.append(s)
    P = S.profile()
    return bool(np.all(P["over"] | (P["emax"] >= 880)))


def _lam_star_max(qa):
    """lambda* without targets: lambda_max, solved by Analyze at lambda_max * 1000."""
    lam_max = _lam_of_rate(qa.rate_range()[1])
    return _lam_of_rate(f32(lam_max * f32(1000)))


# ---------------------------------------------------------------------------------------------------------------
# fleets and rows
# ---------------------------------------------------------------------------------------------------------------
def interval_cases():
    """(fleet, lo, hi, M): one server per x of XS (and more near E(sum) 680), N alternating 1024 / 900, with lo = hi
    (one interval, starting at lo); two N = 1024 servers from x = 400 to 3.5 and 2.5 rateStar, whose starts at 2, 3
    and 4 replicas (x ~ 506, ~ 675, ~ 759) sit below the p window, above it and past float64 overflow; the edge fleet
    with lo = hi on each of its rates."""
    xs = list(XS) + list(np.arange(466.125, 482.0, 0.25)) + [400.0, 400.0]
    main = _fleet(1.0, 0.0, np.ones(len(xs)), [MAIN_N[i % 2] for i in range(len(xs) - 2)] + [1024, 1024],
                  delta=DELTA, ratio=SIZE_RATIO)
    lo = _x_rpm(xs)
    hi = lo.copy()
    rate_star = 0.999 * 1013.6 * 1000  # req/s: lambda_max of N = 1024 (servRate[N-1] = 1013.6 at delta 1e-5)
    hi[-2] = f32(3.5 * rate_star * 60)
    hi[-1] = f32(2.5 * rate_star * 60)
    edge = _edge_fleet()
    erpm = _edge_rpm(edge)
    efl = _concat([edge.take_servers(np.arange(edge.n_servers)) for _ in range(3)])
    elo = erpm.reshape(-1)  # server s of copy l: row l
    return [(main, lo, hi, 8), (efl, elo, elo.copy(), 2)]


def _tokens_rows(L, S):
    """in_tokens alternating 1 / 2 over the levels (two token keys of one N), out_tokens 2."""
    it = np.where(np.arange(L)[:, None] % 2 == 0, 1, 2) * np.ones((1, S), np.int32)
    return it.astype(np.int32), np.full((L, S), 2, np.int32)


def workload_cases():
    """(fleet, (rpm, in, out)): the load grid's main and edge cases at a token mix that keeps N."""
    out = []
    cases = load_cases()
    for fleet, rpm in (cases[0], cases[2]):
        it, ot = _tokens_rows(*rpm.shape)
        out.append((fleet, (rpm, it, ot)))
    return out


def slo_trace_rows(fleet, rows):
    """The six row lists of wva_slo_trace for an SLO grid case: the fleet's own load at every tick."""
    itl, ttft, tps = rows
    L, S = itl.shape
    rep = lambda v: np.repeat(np.asarray(v)[None, :], L, 0).copy()  # noqa: E731
    return (rep(fleet.srv_arrival_rpm).astype(np.float32), rep(fleet.srv_in_tokens).astype(np.int32),
            rep(fleet.srv_out_tokens).astype(np.int32), itl, ttft, tps)


# ---------------------------------------------------------------------------------------------------------------
# the oracle's results and the solves behind them, once per module
# ---------------------------------------------------------------------------------------------------------------
def _load_solves(oracle_mod):
    S, calls = _Solves(), []
    for k, (fleet, rpm) in enumerate(load_cases()):
        cand, win = ref_grid(oracle_mod, fleet, {"arrival_rpm": rpm})
        calls.append((cand, win))
        _add_finals(S, cand, fleet, rpm, np.zeros_like(rpm), lambda l, s, f=fleet: (1, 2), ("load", k))
    return S.profile(), calls


def _interval_solves(oracle_mod):
    S, calls = _Solves(), []
    for k, (fleet, lo, hi, M) in enumerate(interval_cases()):
        out = ref_intervals(oracle_mod, fleet, lo, hi, M)
        count, _, start, rec, _ = out
        calls.append(out)
        for s in range(fleet.n_servers):
            for j in range(int(count[s])):
                r = rec[s * M + j]
                if r["feasible"]:
                    S.add(_qa(*_model(fleet, s)), _final_lam(start[s, j], 0, 2, r["replicas"]), (("iv", k), s, j))
    return S.profile(), calls


def _workload_solves(oracle_mod, trace):
    S, calls = _Solves(), []
    for k, (fleet, (rpm, it, ot)) in enumerate(workload_cases()):
        got = (ref_trace if trace else ref_grid)(oracle_mod, fleet, dict(zip(LOAD, (rpm, it, ot))))
        calls.append(got[:2])
        _add_finals(S, got[0], fleet, rpm, np.zeros_like(rpm), lambda l, s: (int(it[l, s]), int(ot[l, s])),
                    ("wl", k))
    return S.profile(), calls


def _profile_solves(oracle_mod, trace):
    S, calls = _Solves(), []
    for k, (fleet, rows) in enumerate(profile_cases()):
        if trace:
            got = ref_trace(oracle_mod, fleet, rows)
        else:
            got = ref_grid(oracle_mod, fleet, rows)
        calls.append(got[:2])
        L, Sn = rows["perf_alpha"].shape[:2]
        c = got[0].reshape(L, Sn)
        for l in range(L):
            for s in range(Sn):
                r = c[l, s]
                if not r["feasible"]:
                    continue
                m = list(_model(fleet, s))
                m[1] = float(rows["perf_alpha"][l, s, 0])
                S.add(_qa(*m), _final_lam(fleet.srv_arrival_rpm[s], 0, 2, r["replicas"]), (("pr", k), s, l))
    return S.profile(), calls


def _search_lam(oracle_mod, qa, ttft):
    """lambda* of Size with a TTFT target only (the ITL and TPS rules give lambda_max), as Analyze solves it."""
    lmin, lmax = lam_range(qa)

    def fn(x):
        err, y = qa.eval_ttft(x)
        if err:
            raise ValueError("invalid model")
        return y
    err, xs, ind = oracle_mod.binary_search(float(lmin), float(lmax), float(ttft), fn)
    assert err == 0 and ind >= 0
    return _lam_of_rate(f32(min(f32(xs), lmax) * f32(1000)))


def _slo_solves(oracle_mod, trace):
    S, calls = _Solves(), []
    for k, (fleet, rows) in enumerate(slo_cases()):
        itl, ttft, tps = rows
        if trace:
            got = ref_trace(oracle_mod, fleet, dict(zip(LOAD + SLO, slo_trace_rows(fleet, rows))))[:2]
        else:
            got = ref_grid(oracle_mod, fleet, dict(zip(SLO, rows)))
        calls.append(got)
        L, Sn = itl.shape
        c = got[0].reshape(L, Sn)
        for l in range(L):
            for s in range(Sn):
                r = c[l, s]
                if not r["feasible"]:
                    continue
                m = _model(fleet, s)
                qa = _qa(*m)
                if ttft[l, s] > 0:
                    lam_star = _search_lam(oracle_mod, qa, ttft[l, s])
                else:
                    lam_star = _lam_star(qa) if tps[l, s] > 0 else _lam_star_max(qa)
                S.add(qa, lam_star, (("slo", k), s, l, "star"))
                S.add(qa, _final_lam(fleet.srv_arrival_rpm[s], tps[l, s], m[4], r["replicas"]),
                      (("slo", k), s, l, "final"))
    return S.profile(), calls


def _bounds_solves(oracle_mod):
    S, calls = _Solves(), []
    for k, fleet in enumerate(bounds_cases()):
        calls.append(ref_slo_bounds(oracle_mod, fleet))
        for s in range(fleet.n_servers):
            qa = _qa(*_model(fleet, s))
            lmin, lmax = lam_range(qa)
            S.add(qa, lmin, (("bd", k), s, 0))
            S.add(qa, lmax, (("bd", k), s, 1))
    return S.profile(), calls


TAILS = {
    "load": _load_solves,
    "intervals": _interval_solves,
    "workload_grid": lambda o: _workload_solves(o, False),
    "workload_trace": lambda o: _workload_solves(o, True),
    "profile_grid": lambda o: _profile_solves(o, False),
    "profile_trace": lambda o: _profile_solves(o, True),
    "slo_grid": lambda o: _slo_solves(o, False),
    "slo_trace": lambda o: _slo_solves(o, True),
    "bounds": _bounds_solves,
}
# the bands each tail cannot reach (module docstring)
UNREACHABLE = {"bounds": ("pass-2 IEEE path",)}


@pytest.fixture(scope="module")
def tail_solves(oracle_mod):
    cache = {}

    def get(tail):
        if tail not in cache:
            cache[tail] = TAILS[tail](oracle_mod)
        return cache[tail]
    return get


# ---------------------------------------------------------------------------------------------------------------
# CPU: every tail reaches its bands, bails on both sides of an edge, and on more than 128 items of different K
# ---------------------------------------------------------------------------------------------------------------
def _bails(P):
    """The solves that leave the streaming windows: a rate or lambda outside [2^-60, 2^60), p at 2^880 or above, the
    sum at 2^900 or above, or a float64 overflow."""
    def inside(v):
        return (v >= f32(2.0 ** -60)) & (v < f32(P60))
    return P["over"] | (P["emax"] >= 880) | (P["esum"] >= 900) | ~inside(P["lam"]) | ~inside(P["sr0"]) | \
        ~inside(P["srN"])


def _items(P):
    """Each solve's item: (call, server, level / tick / start / end).  An SLO item holds two solves."""
    return [c[:3] for c in P["cand"]]


def _streamed(P):
    """The solves a tail runs as streaming solves: an item's solves in order, up to and including the first that
    bails (slo_tail returns at a bailed lambda* solve, and the re-run solves the whole item on the stored vector)."""
    bailed, out = set(), []
    for it, b in zip(_items(P), _bails(P)):
        out.append(it not in bailed)
        if b:
            bailed.add(it)
    return np.array(out)


def _take(P, m):
    return {k: (v[m] if isinstance(v, np.ndarray) else [x for x, t in zip(v, m) if t]) for k, v in P.items()}


def tail_bands(P):
    b = wide_bands(P, steep=False)
    for k, v in _rate_bands(P).items():
        b[k] = (int(v),) * 2
    return b


@pytest.mark.parametrize("tail", list(TAILS))
def test_tail_cases_reach_their_bands(tail_solves, tail):
    P, _ = tail_solves(tail)
    bands = tail_bands(_take(P, _streamed(P)))
    print(f"\n{tail}: " + ", ".join(f"{k} {v[0]} / {v[1]}" for k, v in bands.items()))
    skip = UNREACHABLE.get(tail, ())
    low = {k: v for k, v in bands.items() if k not in skip and min(v) < 3}
    assert not low, f"{tail}: bands with fewer than 3 cases on a side: {low}"


@pytest.mark.parametrize("tail", list(TAILS))
def test_tail_bails_on_both_sides_and_on_many_items(tail_solves, tail):
    P, _ = tail_solves(tail)
    items = {}  # item -> (bails, K): an item bails when any of its solves does
    for it, b, K in zip(_items(P), _bails(P), P["K"]):
        items[it] = (items.get(it, (False, K))[0] or bool(b), K)
    by_cand = {}
    for it, (b, _) in items.items():
        by_cand.setdefault(it[:2], set()).add(b)
    mixed = [c for c, v in by_cand.items() if v == {False, True}]
    assert mixed, f"{tail}: no candidate has items on both sides of an edge"
    by_call = {}
    for it, (b, K) in items.items():
        if b:
            by_call.setdefault(it[0], []).append(K)
    big = {k: v for k, v in by_call.items() if len(v) > FB_SLOTS and len(set(v)) > 1}
    print(f"\n{tail}: candidates with both sides {len(mixed)}, bailing items per call "
          f"{ {k: len(v) for k, v in by_call.items()} }")
    assert big, f"{tail}: no call bails on more than {FB_SLOTS} items of different K"


@pytest.mark.parametrize("tail", ["load", "slo_grid"])
def test_long_queue_tails_run_the_pass2_ieee_path(tail_solves, tail):
    """The K >= 2^23 candidates (no early termination) have streaming tail solves on the pass-2 IEEE path."""
    P, _ = tail_solves(tail)
    ieee = ~P["over"] & (P["esum"] >= 882) & (P["esum"] < 900) & (P["emax"] < 880) & (P["elive"] < P["esum"] - 960)
    assert (ieee & (P["K"] >= 1 << 23) & _streamed(P)).sum() >= 2


@pytest.mark.parametrize("case", ["load", "intervals", "workload", "profile"])
def test_phase1_bails_on_the_main_fleets(oracle_mod, case):
    """lambda* = lambda_max leaves the p window on every candidate of the main fleets, so the tail's solve is the
    first streaming solve at its lambda."""
    if case == "load":
        fleet = load_cases()[0][0]
        assert _phase1_bails(fleet, range(fleet.n_servers))
        fleet = load_cases()[1][0]
        assert _phase1_bails(fleet, range(fleet.n_servers))
    elif case == "intervals":
        fleet = interval_cases()[0][0]
        assert _phase1_bails(fleet, [0, 1])  # the two models of every server
    elif case == "workload":
        fleet = workload_cases()[0][0]
        for it in (1, 2):
            assert _phase1_bails(fleet, range(fleet.n_servers), lambda s: (it, 2))
    else:
        fleet, rows = profile_cases()[0]
        for a in XS[[0, -1]]:
            g = fleet.take_servers(np.arange(fleet.n_servers))
            g.perf_alpha[:] = a
            assert _phase1_bails(g, range(g.n_servers))


def test_bounds_reach_lambda_edges(oracle_mod):
    """lambda_min exactly on 2^-60 and just below it, lambda_max exactly on 2^60 and just below it, the latter with
    servRate[N-1] above 2^60."""
    edge = bounds_cases()[1]
    lmins, lmaxs, srn = [], [], []
    for s in range(edge.n_servers):
        qa = _qa(*_model(edge, s))
        lo, hi = lam_range(qa)
        lmins.append(lo)
        lmaxs.append(hi)
        srn.append(qa.serv_rate()[-1])
    lmins, lmaxs, srn = (np.array(v, np.float32) for v in (lmins, lmaxs, srn))
    near = lambda v, e: (v < f32(e)) & (v >= f32(e * (1 - 2.0 ** -20)))  # noqa: E731
    for sel in (lmins == f32(2.0 ** -60), near(lmins, 2.0 ** -60)):
        assert sel.sum() >= 3
    for sel in (lmaxs == f32(P60), near(lmaxs, P60)):
        assert sel.sum() >= 3 and (srn[sel] > f32(P60)).all()


# ---------------------------------------------------------------------------------------------------------------
# GPU: every tail at these edges, bit for bit
# ---------------------------------------------------------------------------------------------------------------
PHASE1 = [("warp", None, None), ("rounds-D1", "0", "1"), ("rounds-D5", "0", "5")]


def _variants(n_cases, long_case):
    """(case, phase-1 variant) pairs: every case on the warp kernel and the rounds, except the K >= 2^23 case (its
    phase 1 is one stored-vector solve of 8.5 M states, or none), which runs once."""
    return [pytest.param(c, p, id=f"{c}-{p[0]}") for c in range(n_cases) for p in PHASE1
            if c != long_case or p[1] is None]


def _phase1_env(monkeypatch, small_max, depth):
    """The phase-1 variant's settings, and the level step it runs at: the rounds, whose phase 1 differs from the warp
    kernel's and not the tail, run every third level of the long level lists."""
    if small_max is None:
        return 1
    monkeypatch.setenv("WVA_SIZE_SMALL_MAX", small_max)
    monkeypatch.setenv("WVA_SIZE_DEPTH", depth)
    return 3


def _thin(want, L, step):
    """Every step-th level of an oracle composition (its levels are independent)."""
    cand, win = want[0], want[1]
    return cand.reshape(L, -1)[::step].reshape(-1), win.reshape(L, -1)[::step].reshape(-1)


@pytest.fixture(scope="module")
def grid_refs(oracle_mod):
    """The oracle compositions of the load and SLO grid cases, once for the three phase-1 variants."""
    cache = {}

    def get(what, case):
        if (what, case) not in cache:
            if what == "load":
                fleet, rpm = load_cases()[case]
                cache[what, case] = fleet, rpm, ref_grid(oracle_mod, fleet, {"arrival_rpm": rpm})
            else:
                fleet, rows = slo_cases()[case]
                cache[what, case] = fleet, rows, ref_grid(oracle_mod, fleet, dict(zip(SLO, rows)))
        return cache[what, case]
    return get


def _same_allocs(got, want, what):
    assert_allocs_equal(got[0], want[0], f"{what}: candidates")
    assert_allocs_equal(got[1], want[1], f"{what}: winners")


@pytest.mark.gpu
@pytest.mark.parametrize("case,phase1", _variants(3, 1))
def test_load_grid_at_window_edges(engine, grid_refs, monkeypatch, case, phase1):
    step = _phase1_env(monkeypatch, *phase1[1:])
    fleet, rpm, want = grid_refs("load", case)
    step = step if rpm.shape[0] > 3 else 1
    _same_allocs(engine.load_grid(fleet, rpm[::step], want_candidates=True), _thin(want, rpm.shape[0], step),
                 f"load grid case {case}, {phase1[0]}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(2))
def test_load_intervals_at_window_edges(engine, oracle_mod, case):
    fleet, lo, hi, M = interval_cases()[case]
    count, _ = check_intervals(engine, oracle_mod, fleet, lo, hi, M, f"intervals case {case}")
    assert count.sum() >= fleet.n_servers


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
@pytest.mark.parametrize("case", range(2))
def test_workload_at_window_edges(engine, oracle_mod, case, trace):
    fleet, rows = workload_cases()[case]
    check_level_call(engine, oracle_mod, "workload_trace" if trace else "workload_grid", fleet, dict(zip(LOAD, rows)),
                     f"workload {'trace' if trace else 'grid'} case {case}")


@pytest.mark.gpu
@pytest.mark.parametrize("trace", [False, True])
@pytest.mark.parametrize("case", range(2))
def test_profile_at_window_edges(engine, oracle_mod, case, trace):
    fleet, rows = profile_cases()[case]
    if trace:
        check_level_call(engine, oracle_mod, "profile_trace", fleet, rows, f"profile trace case {case}")
    else:
        check_level_call(engine, oracle_mod, "profile_grid", fleet, rows, f"profile grid case {case}")


@pytest.mark.gpu
@pytest.mark.parametrize("case,phase1", _variants(3, 2))
def test_slo_grid_at_window_edges(engine, grid_refs, monkeypatch, case, phase1):
    step = _phase1_env(monkeypatch, *phase1[1:])
    fleet, rows, want = grid_refs("slo", case)
    L = rows[0].shape[0]
    step = step if L > 3 else 1
    _same_allocs(engine.slo_grid(fleet, *(r[::step] for r in rows), want_candidates=True), _thin(want, L, step),
                 f"SLO grid case {case}, {phase1[0]}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(2))
def test_slo_trace_at_window_edges(engine, oracle_mod, case):
    fleet, rows = slo_cases()[case]
    check_level_call(engine, oracle_mod, "slo_trace", fleet, dict(zip(LOAD + SLO, slo_trace_rows(fleet, rows))),
                     f"SLO trace case {case}")


@pytest.mark.gpu
@pytest.mark.parametrize("case", range(2))
def test_slo_bounds_at_window_edges(engine, oracle_mod, case):
    kind = check_slo_bounds(engine, oracle_mod, bounds_cases()[case], f"bounds case {case}")[0]
    assert (kind >= 2).any()
