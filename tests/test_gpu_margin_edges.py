"""wva_load_margins at its edges, bit for bit against the oracle: the records' tail at the streaming solver's exponent
windows, margin_kernel's and interval_kernel's warp layouts, the bisection brackets of iv_advance and mg_start, and
more than one pass of margin_tail's and interval_tail's grid-stride loops.

Records at the windows.  margin_tail runs the load grid's tail (DESIGN.md 3.19) at three rates per (level, server):
``at`` at the level's rate r, ``below`` at the float under lo (one replica fewer), ``above`` at hi (one more).  The
fleets have beta = gamma = 0, alpha = 1, no latency target and min_replicas 1 (grid_cases.margin_cases), so
rateStar is Size's throughput at lambda_max and each record's lambda is fixed by N, delta and its replica count.  As
in test_gpu_tail_windows, which band a solve reaches is decided by ``chain_profile`` at the float32 lambda MgTail
forms (total_rate_of at r, at nextafter(lo, 0) or at hi, over the record's replicas, over 1000), from the oracle
composition's records.  Bands per record kind (E = binary exponent, "edge - 1 / edge"):

* at: the load grid's main rows (x = lambda at XS) and the edge fleet: E(max p) 879 / 880, E(sum) 679 / 680 and
  899 / 900, the pass-2 IEEE path, float64 overflow, servRate[0] and servRate[N-1] on 2^-60 / 2^60 and one ulp
  across, lambda on 2^-60 and one ulp below.
* below: lambda just under rateStar, N in BELOW_NS (the bounds' lambda_max bands) x three deltas: E(max p)
  879 / 880, E(sum) 679 / 680 and 899 / 900, float64 overflow, and the rate edges on the edge fleet.
* above: lambda just over rateStar / 2, N in ABOVE_NS (twice the XS bands) x six deltas: the same bands as at,
  without the lambda edges.

Not reachable, and so left out:
* the pass-2 IEEE path on below: its lambda is within ulps of rateStar ~ 0.999 servRate[N-1], where the chain past
  state N falls by a factor ~0.999 per state; as for the bounds' lambda_max it reaches 2^(E(sum) - 960) only ~6.6e5
  states past the peak, at queue ratios above 1000.
* the lambda edges on below and above: their lambda is rateStar / (n - 1) or rateStar / n for the step's count n,
  and on the lambda-edge models (alpha 2^50 .. 2^54) rateStar / 1000 is ~1e-14, so lambda = 2^-60 needs a count of
  ~1e4 whose float32 quotient lands on 2^-60 exactly; only the at record places lambda directly.
* a sum bail on its own, and steep crossings of 2^880, for the reasons test_gpu_tail_windows gives.

Warp layouts.  Both kernels keep A IvAcc states (64 bytes, asserted in wva_size.cuh) per warp in dynamic shared
memory, margin_kernel also A stretch starts: 68 A and 64 A bytes per warp.  The host runs max(1, min(4, 48 KiB /
per-warp bytes)) warps per block, opts in above 48 KiB and refuses above the device's opt-in limit.  The tests run
each kernel on both sides of every layout threshold and at the first refused A.

Brackets.  iv_advance and mg_start bisect inside +-64 ulps of an estimate of the step when that bracket checks out,
otherwise over the whole range.  levels.iv_branch / mg_branch restate the choice; bracket_cases reach both branches
at gates 1 and 2: gate 2 (the rate check rejecting above RateRange.Max at a fixed count) exists only where float32
(total / float32(nrep)) rounds above RateRange.Max, which needs rateStar = RateRange.Max (queue ratio 1000) and a
count past 2^24; the whole range is searched when the estimate reaches 3e38 (RateRange.Max ~ 3.2e29) or when
min_replicas holds the count up above a window bottom where totalRate rounds to 0.
"""
from __future__ import annotations

import numpy as np
import pytest
from tests.grid_cases import (BELOW_NS, _final_lam, _model, _qa, _Solves, _bails, bracket_cases, margin_cases,
                              tail_bands)
from tests.levels import (F32, below, check_intervals, check_margins, iv_branch, load_pair, margin_record_rates,
                          mg_branch, ref_margins)
from tests.util import ALLOC_FIELDS, F32_MAX, WVA_ERR_UNSUPPORTED, same_bytes
from workload_variant_autoscaler_b200 import (MARGIN_HI_OPEN, MARGIN_LO_OPEN, MARGIN_TRUNCATED, Engine, WvaError,
                                              synth_fleet)

FB_SLOTS = 128  # kFbBlocks * kFbThreads: the threads of every re-run kernel
KINDS = ("at", "below", "above")


# ---------------------------------------------------------------------------------------------------------------
# the records' solves, with their profiles, once per module
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def margin_refs(oracle_mod):
    """{case name: (fleet, rate, lo, hi, ref_margins)} and the record solves' profile."""
    refs, S = {}, _Solves()
    for name, fleet, rate, lo, hi in margin_cases():
        ref = ref_margins(oracle_mod, fleet, rate, lo, hi)
        refs[name] = (fleet, rate, lo, hi, ref)
        xs = margin_record_rates(rate, *ref[:3])
        n_srv = fleet.n_servers
        for k, kind in enumerate(KINDS):
            rec = ref[3 + k]
            for i in range(rate.size):
                if not rec[i]["feasible"] or np.isnan(xs[kind][i]):
                    continue
                s = i % n_srv
                S.add(_qa(*_model(fleet, s)), _final_lam(xs[kind][i], 0, int(fleet.srv_out_tokens[s]),
                                                         int(rec[i]["replicas"])), (kind, name, i))
    return refs, S.profile()


def _kind(P, kind):
    m = np.array([c[0] == kind for c in P["cand"]])
    return {k: (v[m] if isinstance(v, np.ndarray) else [x for x, t in zip(v, m) if t]) for k, v in P.items()}


# the bands a record kind cannot reach (module docstring)
UNREACHABLE = {"below": ("pass-2 IEEE path", "lam == 2^-60", "lam just below 2^-60"),
               "above": ("lam == 2^-60", "lam just below 2^-60")}


# ---------------------------------------------------------------------------------------------------------------
# CPU: every record kind reaches its bands; records on both sides of an edge; a call bailing on > 128 records
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_records_reach_their_bands(margin_refs, kind):
    _, P = margin_refs
    bands = tail_bands(_kind(P, kind))
    print(f"\n{kind}: " + ", ".join(f"{k} {v[0]} / {v[1]}" for k, v in bands.items()))
    low = {k: v for k, v in bands.items() if k not in UNREACHABLE.get(kind, ()) and min(v) < 3}
    assert not low, f"{kind}: bands with fewer than 3 cases on a side: {low}"


def test_records_bail_on_both_sides_and_on_many_records(margin_refs):
    _, P = margin_refs
    items = {}  # (case, i) -> {kind: bails}
    calls = {}  # case -> [K of each bailing record]
    for (kind, name, i), b, K in zip(P["cand"], _bails(P), P["K"]):
        items.setdefault((name, i), {})[kind] = bool(b)
        if b:
            calls.setdefault(name, []).append(int(K))
    mixed = [it for it, v in items.items() if len(set(v.values())) == 2]
    all3 = [it for it, v in items.items() if len(v) == 3 and all(v.values())]
    big = {k: v for k, v in calls.items() if len(v) > FB_SLOTS and len(set(v)) > 1}
    print(f"\nitems with records on both sides {len(mixed)}, with three bailing records {len(all3)}, bailing records "
          f"per call { {k: len(v) for k, v in calls.items()} }")
    assert mixed, "no (level, server) has records on both sides of an edge"
    assert big, f"no call bails on more than {FB_SLOTS} records of different K"
    assert any(it[0] in big for it in all3), "no call with > 128 bailing records has an item whose three records bail"


def test_below_records_sit_under_rate_star(margin_refs):
    """The below records of the below fleet are one replica under the step at 1.5 steps, and at 99.5 steps all three
    records have 99, 100 and 101 replicas: the rates the docstring places."""
    refs, _ = margin_refs
    fleet, rate, lo, hi, ref = refs["below"]
    S = fleet.n_servers
    assert S == 3 * len(BELOW_NS)
    at, dn, up = ref[3].reshape(2, S), ref[4].reshape(2, S), ref[5].reshape(2, S)
    assert (dn[0]["replicas"] == 1).all() and (at[0]["replicas"] == 2).all()
    assert (dn[1]["replicas"] == 99).all() and (at[1]["replicas"] == 100).all() and (up[1]["replicas"] == 101).all()


# ---------------------------------------------------------------------------------------------------------------
# GPU: the records at the windows, bit for bit
# ---------------------------------------------------------------------------------------------------------------
def _keep(fleet):
    """keepAccelerator on, with a current allocation on the only accelerator (its transition penalty is the
    value)."""
    f = fleet.take_servers(np.arange(fleet.n_servers))
    f.srv_keep_acc[:] = 1
    f.srv_cur_acc[:] = 0
    f.srv_cur_replicas[:] = 2
    f.srv_cur_cost[:] = 80.0
    return f


@pytest.fixture(scope="module")
def keep_refs(oracle_mod, margin_refs):
    cache = {}

    def get(name):
        if name not in cache:
            fleet, rate, lo, hi, _ = margin_refs[0][name]
            f = _keep(fleet)
            cache[name] = (f, rate, lo, hi, ref_margins(oracle_mod, f, rate, lo, hi))
        return cache[name]
    return get


CASE_NAMES = ["at main", "at edge", "below", "above", "edge steps"]


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True], ids=["warp", "rounds"])
@pytest.mark.parametrize("keep", [False, True], ids=["nokeep", "keep"])
@pytest.mark.parametrize("case", CASE_NAMES)
def test_records_at_window_edges(engine, oracle_mod, margin_refs, keep_refs, monkeypatch, case, keep, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet, rate, lo, hi, ref = keep_refs(case) if keep else margin_refs[0][case]
    check_margins(engine, oracle_mod, fleet, rate, lo, hi, f"{case}, keep {keep}, rounds {rounds}", ref=ref)


# ---------------------------------------------------------------------------------------------------------------
# warp layouts, the shared-memory opt-in and the refusal
# ---------------------------------------------------------------------------------------------------------------
IVACC = 64
MARGIN_A = [180, 181, 240, 241, 361, 362, 722, 723]
INTERVAL_A = [192, 193, 256, 257, 384, 385, 768, 769]


def _wpb(per_warp):
    return max(1, min(4, (48 << 10) // per_warp))


def test_layout_thresholds():
    """The hard-coded A lie on both sides of every change of warps per block and of the 48 KiB opt-in."""
    for A_list, per in ((MARGIN_A, IVACC + 4), (INTERVAL_A, IVACC)):
        lay = [(_wpb(per * A), per * A * _wpb(per * A) > 48 << 10) for A in A_list]
        assert lay == [(4, False), (3, False), (3, False), (2, False), (2, False), (1, False), (1, False),
                       (1, True)], lay


def layout_fleet(A, S=None, seed=7):
    """S servers x A accelerators, small batches and queue ratio 1 (a cheap oracle); accelerator 0's profile and
    cost copied onto 32, 64, A // 2 + 1 and A - 1, so that its ties cross lane strides and warps.  S = 5 (not a
    multiple of 4, 3 or 2 warps per block: the last block has idle warps), 2 at one warp per block."""
    S = S or (5 if (IVACC + 4) * A <= (24 << 10) else 2)
    f = synth_fleet(S, A, seed=seed, zero_load_frac=0.0, tps_frac=0.0, max_batch_choices=(8,))
    f.max_queue_to_batch_ratio = 1
    for a in (32, 64, A // 2 + 1, A - 1):
        f.acc_cost[a] = f.acc_cost[0]
        for col in (f.perf_present, f.perf_alpha, f.perf_beta, f.perf_gamma, f.perf_delta, f.perf_acc_count):
            col[:, a] = col[:, 0]
    return f


def layout_rows(oracle_mod, fleet):
    """(rate, lo, hi) [1, S]: each server at 0.6 of its smallest first replica step over the accelerators, in the
    window [0.5, 6] times that: the steps of the pairs up to 3.6 times the smallest fall inside, and no more (the
    composition walks every step of every pair in the window)."""
    r = np.zeros((1, fleet.n_servers), np.float32)
    for s in range(fleet.n_servers):
        steps = [60.0 * float(p[0]) for p in (load_pair(oracle_mod, fleet, s, a) for a in range(fleet.n_acc)) if p]
        r[0, s] = F32(0.6 * min(steps))
    return r, (r * F32(0.5)).astype(np.float32), (r * F32(6)).astype(np.float32)


def _optin():
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


@pytest.mark.gpu
@pytest.mark.parametrize("A", MARGIN_A)
def test_margin_kernel_layouts(engine, oracle_mod, A):
    fleet = layout_fleet(A)
    _, _, flags, at, *_ = check_margins(engine, oracle_mod, fleet, *layout_rows(oracle_mod, fleet), f"A = {A}")
    assert (flags & MARGIN_HI_OPEN == 0).any() and at["feasible"].all()


@pytest.mark.gpu
@pytest.mark.parametrize("A", INTERVAL_A)
def test_interval_kernel_layouts(engine, oracle_mod, A):
    fleet = layout_fleet(A)
    _, lo, hi = layout_rows(oracle_mod, fleet)
    count, _ = check_intervals(engine, oracle_mod, fleet, lo[0], hi[0], 64, f"A = {A}")
    assert (count >= 2).any()


@pytest.mark.gpu
def test_refused_layouts_leave_the_handle_whole(engine):
    """The first A whose one warp exceeds the device's opt-in shared memory is refused by both calls, and the
    handle then gives what a fresh handle gives."""
    optin = _optin()
    for per, call in ((IVACC + 4, "margins"), (IVACC, "intervals")):
        A = optin // per + 1
        fleet = layout_fleet(A, S=2, seed=11)
        x = fleet.srv_arrival_rpm.astype(np.float32)
        with pytest.raises(WvaError) as e:
            if call == "margins":
                engine.load_margins(fleet, x[None, :], (x * F32(0.5))[None, :], (x * F32(2))[None, :])
            else:
                engine.load_intervals(fleet, x * F32(0.5), x * F32(2), 8)
        assert e.value.code == WVA_ERR_UNSUPPORTED and "shared memory" in str(e.value), (call, A, e.value)
    fleet = layout_fleet(241)
    x = fleet.srv_arrival_rpm.astype(np.float32)
    rate, lo, hi = x[None, :], (x * F32(0.5)).astype(np.float32)[None, :], (x * F32(2)).astype(np.float32)[None, :]
    fresh = Engine(0)
    try:
        for got, want in zip(engine.load_margins(fleet, rate, lo, hi), fresh.load_margins(fleet, rate, lo, hi)):
            _same(got, want, "margins after a refusal")
        for got, want in zip(engine.load_intervals(fleet, lo[0], hi[0], 16), fresh.load_intervals(fleet, lo[0], hi[0],
                                                                                                  16)):
            _same(got, want, "intervals after a refusal")
    finally:
        fresh.close()


def _same(x, y, what):
    if hasattr(x, "feasible"):
        for k in ALLOC_FIELDS:
            assert same_bytes(getattr(x, k), getattr(y, k)), f"{what}: {k}"
    else:
        assert same_bytes(np.asarray(x), np.asarray(y)), what


# ---------------------------------------------------------------------------------------------------------------
# the brackets of iv_advance and mg_start
# ---------------------------------------------------------------------------------------------------------------
def bracket_branches(oracle_mod, fleet, rate, lo, hi, ref):
    """{(search, gate, branch): count} over the searches the kernels run on bracket_cases: iv_advance at r and at
    hi (the up-walk's last step), mg_start at r and at the float under lo (the down-walk's last step)."""
    lo_e, hi_e, flags = ref[:3]
    L, S = rate.shape
    out = {}
    for s in range(S):
        rs, rmax, _, _ = load_pair(oracle_mod, fleet, s, 0)
        for l in range(L):
            r, f = F32(rate[l, s]), flags[l, s]
            bottom = F32(lo[l, s]) if lo[l, s] > 0 else np.nextafter(F32(0), F32(1))
            pts = [("iv", iv_branch(fleet, s, rs, rmax, r, hi[l, s])), ("mg", mg_branch(fleet, s, rs, rmax, r, bottom))]
            if not f & (MARGIN_HI_OPEN | MARGIN_TRUNCATED):
                pts.append(("iv", iv_branch(fleet, s, rs, rmax, hi_e[l, s], hi[l, s])))
            if not f & (MARGIN_LO_OPEN | MARGIN_TRUNCATED):
                pts.append(("mg", mg_branch(fleet, s, rs, rmax, below(lo_e[l, s]), bottom)))
            for what, (gate, branch) in pts:
                if branch is not None:
                    out[what, gate, branch] = out.get((what, gate, branch), 0) + 1
    return out


@pytest.fixture(scope="module")
def bracket_ref(oracle_mod):
    fleet, rate, lo, hi = bracket_cases()
    return fleet, rate, lo, hi, ref_margins(oracle_mod, fleet, rate, lo, hi)


def test_brackets_take_both_branches_at_both_gates(oracle_mod, bracket_ref):
    got = bracket_branches(oracle_mod, *bracket_ref)
    print("\n" + ", ".join(f"{k[0]} gate {k[1]} {k[2]}: {v}" for k, v in sorted(got.items())))
    missing = [(w, g, b) for w in ("iv", "mg") for g in (1, 2) for b in ("bracket", "whole") if (w, g, b) not in got]
    assert not missing, f"branches no case takes: {missing}"


def test_bracket_cases_sit_where_the_docstring_says(oracle_mod, bracket_ref):
    """Gate 2 past 2^24 replicas on servers 0 and 1 (rateStar = RateRange.Max), estimates at or above 3e38 on
    server 1, and min_replicas holding server 2's count."""
    fleet, rate, lo, hi, ref = bracket_ref
    at = ref[3].reshape(rate.shape)
    for s in (0, 1):
        rs, rmax, _, _ = load_pair(oracle_mod, fleet, s, 0)
        assert rs == rmax
        assert (at["feasible"][:2, s] == 0).all() and (at["feasible"][2:, s] == 1).all()
        assert at["replicas"][2, s] > 1 << 24
    assert float(rate[0, 1]) * 1.0 >= 3e38
    assert (at["replicas"][:, 2] >= 3).all()


@pytest.mark.gpu
@pytest.mark.parametrize("rounds", [False, True], ids=["warp", "rounds"])
def test_bracket_cases_margins(engine, oracle_mod, bracket_ref, monkeypatch, rounds):
    if rounds:
        monkeypatch.setenv("WVA_SIZE_SMALL_MAX", "0")
    fleet, rate, lo, hi, ref = bracket_ref
    check_margins(engine, oracle_mod, fleet, rate, lo, hi, "bracket cases", ref=ref)


@pytest.mark.gpu
@pytest.mark.parametrize("level", range(4))
def test_bracket_cases_intervals(engine, oracle_mod, bracket_ref, level):
    fleet, rate, lo, hi, _ = bracket_ref
    check_intervals(engine, oracle_mod, fleet, lo[level], hi[level], 256, f"bracket level {level}")


# ---------------------------------------------------------------------------------------------------------------
# more than one pass of margin_tail's and interval_tail's grid-stride loops, without the oracle
# ---------------------------------------------------------------------------------------------------------------
def _one_pass():
    import torch
    return 8 * torch.cuda.get_device_properties(0).multi_processor_count * 256


def _rows_equal(got, want, mask, what):
    """Records got [n] and want [n] byte for byte where mask holds."""
    for k in ALLOC_FIELDS:
        g, w = np.asarray(getattr(got, k)), np.asarray(getattr(want, k))
        bad = np.nonzero(mask & (g.view(np.uint8).reshape(g.size, -1) != w.view(np.uint8).reshape(w.size, -1)).any(1))
        assert bad[0].size == 0, f"{what}: {k} differs at {bad[0][:8]}"


@pytest.mark.gpu
def test_margin_tail_past_one_pass(engine):
    """3 L S records past two passes of margin_tail: wva_load_grid at r, below lo and hi reproduces them."""
    fleet = synth_fleet(1500, 8, seed=42)
    S, n_pass = fleet.n_servers, _one_pass()
    L = -(-2 * n_pass // (3 * S)) + 1
    x = fleet.srv_arrival_rpm.astype(np.float32)
    rate = (x[None, :] * np.random.default_rng(5).lognormal(0, 0.3, (L, S))).astype(np.float32)
    lo, hi = (rate * F32(0.5)).astype(np.float32), (rate * F32(2)).astype(np.float32)
    lo_m, hi_m, flags, at, dn, up = engine.load_margins(fleet, rate, lo, hi)
    closed_lo = ((flags & (MARGIN_LO_OPEN | MARGIN_TRUNCATED)) == 0).reshape(-1)
    closed_hi = ((flags & (MARGIN_HI_OPEN | MARGIN_TRUNCATED)) == 0).reshape(-1)
    loaded = ((rate > 0) & (fleet.srv_slo_tps == 0)[None, :]).reshape(-1)
    tails = (at.feasible.astype(bool) & loaded).sum() + (dn.feasible.astype(bool) & closed_lo & loaded).sum() + \
        (up.feasible.astype(bool) & closed_hi & loaded).sum()
    assert tails > n_pass, (tails, n_pass)
    r = rate.reshape(-1)
    rows = np.stack([r, np.where(closed_lo, below(lo_m.reshape(-1)), r), np.where(closed_hi, hi_m.reshape(-1), r)])
    _, win = engine.load_grid(fleet, rows.reshape(3 * L, S).astype(np.float32))
    n = L * S
    for k, (name, rec, mask) in enumerate((("at", at, np.ones(n, bool)), ("below", dn, closed_lo),
                                           ("above", up, closed_hi))):
        part = type(win)(n)
        for f in ALLOC_FIELDS:
            getattr(part, f)[:] = getattr(win, f)[k * n:(k + 1) * n]
        _rows_equal(part, rec, mask, name)


@pytest.mark.gpu
def test_interval_tail_past_one_pass(engine):
    """S M interval starts past one pass of interval_tail: wva_load_grid at each start reproduces its record."""
    fleet = synth_fleet(1500, 8, seed=43)
    S, n_pass = fleet.n_servers, _one_pass()
    M = 2 * n_pass // S + 1
    lo = np.maximum(fleet.srv_arrival_rpm.astype(np.float32), F32(1))
    hi = np.full(S, F32_MAX, np.float32)
    count, _, start, rec = engine.load_intervals(fleet, lo, hi, M)
    assert count.sum() > n_pass, (count.sum(), n_pass)
    j = np.arange(M)[:, None]
    valid = j < count[None, :]
    rows = np.where(valid, start.T, start[:, :1].T).astype(np.float32)  # (M, S)
    _, win = engine.load_grid(fleet, rows)
    want = type(win)(S * M)
    for f in ALLOC_FIELDS:  # rec is server-major (s * M + j); the grid's winners are level-major (j * S + s)
        getattr(want, f)[:] = np.asarray(getattr(rec, f)).reshape(S, M).T.reshape(-1)
    _rows_equal(win, want, valid.reshape(-1), "interval starts")
