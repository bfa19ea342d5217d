"""C oracle vs the independent numpy restatement (oracle/restate_np.py), bit for bit.

Float outputs under load are pinned by no reference test (SURVEY.md §8c), so two independently written restatements
agreeing is what stands in for the Go binary here.  The first three tests are small random cases.  The families after
them run the restatement on the inputs the GPU tests judge the kernels with, taken from those modules by import: the
exponent windows (test_gpu_windows), the grid's shape thresholds and stored-vector fallbacks (test_gpu_grid_shapes),
the adversarial fleets and the queue-size rule (test_gpu_adversarial_paths), the rows of the SLO, workload and
profile grids, and the rows that put the level calls' tails on the exponent windows (test_gpu_tail_windows).  A
kernel that matches the oracle bit for bit is only as right as the oracle, so a misreading of the Go code at one of
these edges would otherwise pass every GPU test.

Comparison: feasible, accelerator, replicas and batch size exactly; cost, ITL, TTFT, rho and max_rate (and a cell's
or sweep point's TTFT, ITL, rho and throughput) by their float32 bits, NaN equal to NaN; probability vectors by their
float64 bits.  Where the restatement raises Unsupported the oracle is held to its own rule: a model of 2^31 states or
more is refused by both.  A batch size above 2^20 with fewer states is refused by the CUDA library and by the
restatement only; the oracle would build it, and its Size there takes many seconds, so it is not asked.  A rescale
loop that would not terminate (a NaN rate) has no value in the reference, which never returns; the oracle finishes it
with NaN and the library refuses it, so there is nothing to agree on.

Sampling is deterministic.  Pairs whose batch size comes out above 4096 under the AtTokens rule are left out of the
adversarial and level-row samples (a Size there costs the restatement seconds); the windows family covers large N."""
import numpy as np
import pytest

from tests import grid_cases, levels
from tests.levels import (F, LOAD, SLO, TARGETS, TPS_TARGETS, Tally, _restated, at_row, cross_fleet, mixed_fleet,
                          pair_n, profile_fleet, profile_rows, same_f32, slo_levels, token_fleet, workload_levels)
from workload_variant_autoscaler_b200 import synth_fleet

CELL_FLOATS = ("ttft", "itl", "rho", "throughput")
SWEEP_FLOATS = ("ttft", "itl", "throughput", "rho")
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_create_allocation_cross(oracle_mod, seed):
    from oracle import restate_np as R
    f = synth_fleet(10, 3, seed=seed, max_batch_choices=(1, 2, 4, 8, 16), zero_load_frac=0.2)
    f.srv_min_replicas[::3] = 0
    n_feas = 0
    for s in range(f.n_servers):
        for a in range(f.n_acc):
            o = oracle_mod.create_allocation(f, s, a)
            r = R.create_allocation(f, s, a)
            assert o["feasible"] == r["feasible"], (s, a, o, r)
            if not o["feasible"]:
                continue
            n_feas += 1
            assert (o["acc"], o["replicas"], o["batch"]) == (r["acc"], r["replicas"], r["batch"]), (s, a, o, r)
            for k in ("cost", "itl", "ttft", "rho", "max_rate"):
                assert same_f32(o[k], r[k]), (s, a, k, o[k], r[k])
    assert n_feas >= 15


def test_analyze_and_solve_cross(oracle_mod):
    from oracle import restate_np as R
    rng = np.random.default_rng(7)
    for _ in range(12):
        N = int(rng.integers(1, 24))
        al, be = F(rng.uniform(5, 25)), F(rng.uniform(0.02, 0.8))
        ga, de = F(rng.uniform(0, 250)), F(np.exp(rng.uniform(np.log(1e-4), np.log(0.1))))
        it, ot = int(rng.integers(0, 2048)), int(rng.integers(1, 512))
        qa = oracle_mod.Analyzer(N, 10 * N, al, be, ga, de, it, ot)
        rq = R.QA(N, 10 * N, al, be, ga, de, it, ot)
        assert np.array_equal(qa.serv_rate().view(np.uint32), rq.sr.view(np.uint32))
        rmin, rmax = qa.rate_range()
        assert same_f32(rmin, rq.rmin) and same_f32(rmax, rq.rmax)
        for frac in (0.0, 0.3, 0.7, 1.0):
            rate = F(rmin + F(frac) * (rmax - rmin))
            err, m = qa.analyze(float(rate))
            mr = rq.analyze(rate)
            assert (err == 0) == (mr is not None)
            if mr is None:
                continue
            assert same_f32(m["throughput"], mr["throughput"]) and same_f32(m["avg_wait_time"], mr["wait"])
            assert same_f32(m["avg_prefill_time"], mr["prefill"]) and same_f32(m["avg_token_time"], mr["itl"])
            assert same_f32(m["rho"], mr["rho"])
            assert np.array_equal(qa.probs().view(np.uint64), rq.p.view(np.uint64))


def test_overflow_rescale_cross(oracle_mod):
    """N large enough that prod(lambda/servRate) overflows: both restatements must take the
    reference's rescale branches (mm1modelstatedependent.go:84-89) and agree."""
    from oracle import restate_np as R
    args = (800, 8000, 7.47, 0.0001, 1.0, 0.00001, 64, 64)
    qa, rq = oracle_mod.Analyzer(*args), R.QA(*args)
    rmin, rmax = qa.rate_range()
    rate = F(rmax) * F(0.98)
    err, m = qa.analyze(float(rate))
    mr = rq.analyze(rate)
    assert err == 0 and mr is not None
    assert np.array_equal(qa.probs().view(np.uint64), rq.p.view(np.uint64))
    assert same_f32(m["avg_wait_time"], mr["wait"]) and same_f32(m["rho"], mr["rho"])


# ---------------------------------------------------------------------------------------------------------------
# the comparison of one point
# ---------------------------------------------------------------------------------------------------------------
def _cell_index(fleet, grid, ci):
    R_, B = grid.replicas.size, grid.batch.size
    ri, bi = ci % R_, (ci // R_) % B
    a, s = (ci // (R_ * B)) % fleet.n_acc, ci // (R_ * B * fleet.n_acc)
    return int(s), int(a), int(grid.batch[bi]), int(grid.replicas[ri])


def cross_cell(oracle_mod, fleet, grid, ci, cell_o, tally, what="", probs=False):
    """Cell ci of the grid against the oracle's record cell_o; with probs, Analyze's probability vector too."""
    from oracle import restate_np as R
    s, a, b, r = _cell_index(fleet, grid, ci)
    c = _restated(lambda: R.grid_cell(fleet, s, a, b, r), oracle_mod,
                  lambda: oracle_mod.grid_cells(fleet, grid, ci, ci + 1), tally)
    if c is None:
        return
    assert int(cell_o["flags"]) == c["flags"], (what, (s, a, b, r), cell_o, c)
    tally.n[("feasible" if c["flags"] & 2 else "infeasible") if c["flags"] & 1 else "not analysed"] += 1
    for k in CELL_FLOATS:
        assert same_f32(cell_o[k], c[k]), (what, (s, a, b, r), k, cell_o[k], c[k])
    if probs and c["flags"] & 1:
        m = int(fleet.srv_model[s])
        args = (b, b * fleet.max_queue_to_batch_ratio, float(fleet.perf_alpha[m, a]), float(fleet.perf_beta[m, a]),
                float(fleet.perf_gamma[m, a]), float(fleet.perf_delta[m, a]), int(fleet.srv_in_tokens[s]),
                int(fleet.srv_out_tokens[s]))
        rate = R._total_rate(fleet, s) / F(r)
        qa, rq = oracle_mod.Analyzer(*args), R.QA(*args)
        assert qa.analyze(float(rate))[0] == 0 and rq.analyze(rate) is not None
        assert np.array_equal(qa.probs().view(np.uint64), rq.p.view(np.uint64)), (what, (s, a, b, r))
        tally.n["probability vectors"] += 1


def cross_sweep(oracle_mod, fleet, n_rates, o, points, tally, what="", probs=()):
    """Sweep points (flat indices into the oracle's sweep o) through the restatement's Analyze at the oracle's
    rates, each on a freshly built model."""
    from oracle import restate_np as R
    models = {}
    for i in points:
        s, a = divmod(int(i) // n_rates, fleet.n_acc)
        if (s, a) not in models:
            m = int(fleet.srv_model[s])
            N = pair_n(fleet, s, a)
            mq, _ = R.queue_states(N, fleet.max_queue_to_batch_ratio)
            models[s, a] = R.QA(N, mq, fleet.perf_alpha[m, a], fleet.perf_beta[m, a], fleet.perf_gamma[m, a],
                                fleet.perf_delta[m, a], fleet.srv_in_tokens[s], fleet.srv_out_tokens[s])
        rq = models[s, a]
        rq.reset()
        met = rq.analyze(F(o["rate"][i]))
        assert int(o["valid"][i]) == (met is not None), (what, int(i))
        tally.n["feasible" if met is not None else "infeasible"] += 1
        if met is None:
            continue
        got = {"ttft": met["wait"] + met["prefill"], "itl": met["itl"], "throughput": met["throughput"],
               "rho": met["rho"]}
        for k in SWEEP_FLOATS:
            assert same_f32(o[k][i], got[k]), (what, int(i), k, o[k][i], got[k])
        if i in probs:
            m = int(fleet.srv_model[s])
            qa = oracle_mod.Analyzer(rq.N, rq.Q, float(fleet.perf_alpha[m, a]), float(fleet.perf_beta[m, a]),
                                     float(fleet.perf_gamma[m, a]), float(fleet.perf_delta[m, a]),
                                     int(fleet.srv_in_tokens[s]), int(fleet.srv_out_tokens[s]))
            assert qa.analyze(float(o["rate"][i]))[0] == 0
            assert np.array_equal(qa.probs().view(np.uint64), rq.p.view(np.uint64)), (what, int(i))
            tally.n["probability vectors"] += 1


def _pick(rng, idx, k):
    idx = np.asarray(idx)
    return idx if idx.size <= k else np.sort(rng.choice(idx, k, replace=False))


# ---------------------------------------------------------------------------------------------------------------
# exponent windows (test_gpu_windows)
# ---------------------------------------------------------------------------------------------------------------
WINDOWS = ["grid-0", "grid-1", "grid-2", "size", "long-queue", "overflow-search-0", "overflow-search-1", "sweep"]


@pytest.mark.parametrize("case", WINDOWS)
def test_windows_cross(oracle_mod, case):
    """The cases test_gpu_windows steers onto every solver's exponent windows (their bands are asserted there):
    every analysable grid cell and a sample of the others, with a sample of probability vectors; every size
    candidate; one of the K >= 2^23 candidates (a chain of 8.5 M states costs the restatement seconds); the two
    overflowing-search fleets; and sweep points chosen per band from chain_profile, plus an even spread."""
    rng = np.random.default_rng(WINDOWS.index(case) + 11)
    t = Tally()
    if case.startswith("grid"):
        fleet, grid = grid_cases.grid_cases()[int(case[-1])]
        cells, _ = oracle_mod.grid_solve(fleet, grid, want_cells=True)
        ok = np.nonzero(cells["flags"] & 1)[0]
        rest = np.nonzero(~cells["flags"] & 1)[0]
        probs = set(_pick(rng, ok, 6).tolist())
        for ci in np.concatenate([ok, _pick(rng, rest, 16)]):
            cross_cell(oracle_mod, fleet, grid, int(ci), cells[ci], t, case, probs=int(ci) in probs)
        t.report(case, min_feasible=0 if case == "grid-1" else 3, min_infeasible=0,
                 **{"probability vectors": min(6, ok.size)})
        assert t.n["feasible"] + t.n["infeasible"] == ok.size >= 6
    elif case == "size":
        fleet = grid_cases.size_fleet()
        cross_fleet(oracle_mod, fleet, t, case)
        t.report(case, min_feasible=700, min_infeasible=0)
    elif case == "long-queue":
        fleet = grid_cases.long_queue_fleet()
        cross_fleet(oracle_mod, fleet, t, case, pairs=[(int(rng.integers(fleet.n_servers)), 0)])
        t.report(case, min_infeasible=0)
    elif case.startswith("overflow-search"):
        fleet = grid_cases.overflow_search_fleet(*grid_cases.OVERFLOW_SEARCHES[int(case[-1])][:2])
        cross_fleet(oracle_mod, fleet, t, case)
        t.report(case, min_feasible=2, min_infeasible=0)
    else:
        fleet, n = grid_cases.sweep_fleet(), grid_cases.SWEEP_RATES
        o = oracle_mod.sweep(fleet, n)
        valid = np.nonzero(o["valid"])[0]
        P = grid_cases.sweep_points(fleet, n, o["valid"])  # in the order of `valid`
        ok = ~P["over"]
        bands = [P["over"], P["steep880"], ok & (P["emax"] == 879), ok & (P["emax"] == 880),
                 ok & (P["esum"] == 679), ok & (P["esum"] == 680), ok & (P["esum"] == 899), ok & (P["esum"] == 900),
                 ok & (P["esum"] >= 882) & (P["esum"] < 900) & (P["emax"] < 880) & (P["elive"] < P["esum"] - 960)]
        pts, probs = set(), set()
        for k, band in enumerate(bands):
            assert band.any()
            got = valid[_pick(rng, np.nonzero(band)[0], 3)].tolist()
            pts.update(got)
            if k in (0, len(bands) - 1):  # float64 overflow and the pass-2 IEEE path
                probs.update(got[:2])
        pts.update(range(0, o["valid"].size, o["valid"].size // 48))
        cross_sweep(oracle_mod, fleet, n, o, sorted(pts), t, case, probs=probs)
        t.report(case, min_feasible=60, min_infeasible=0, **{"probability vectors": 4})


# ---------------------------------------------------------------------------------------------------------------
# grid shapes and stored-vector fallbacks (test_gpu_grid_shapes)
# ---------------------------------------------------------------------------------------------------------------
SHAPE_CASES = list(grid_cases.SHAPES) + ["tiny-acc", "invariant", "grid-fallback", "sweep-fallback", "size-fallback"]


def _sample_cells(rng, cells, k_feas=6, k_infeas=4, k_none=3):
    fl = cells["flags"]
    return np.concatenate([_pick(rng, np.nonzero(fl & 2)[0], k_feas),
                           _pick(rng, np.nonzero((fl & 1) & ~(fl >> 1) & 1)[0], k_infeas),
                           _pick(rng, np.nonzero(~fl & 1)[0], k_none)]).astype(np.int64)


@pytest.mark.parametrize("case", SHAPE_CASES)
def test_grid_shapes_cross(oracle_mod, case):
    """A deterministic sample of cells of every shape case (feasible, analysed and infeasible, not analysed), the
    tiny-acc and batch-invariant cases (with the cell whose TTFT is its server's target), the fallback cases past
    their 128 slots (cells, sweep points and size candidates)."""
    rng = np.random.default_rng(SHAPE_CASES.index(case) + 101)
    t = Tally()
    if case == "sweep-fallback":
        fleet, n = grid_cases.sweep_fallback_fleet(), grid_cases.SWEEP_FB_RATES
        o = oracle_mod.sweep(fleet, n)
        pts = sorted(set(range(0, n, n // 24)) | set(range(n - 8, n)))
        cross_sweep(oracle_mod, fleet, n, o, pts, t, case, probs={pts[-1], pts[len(pts) // 2]})
        t.report(case, min_feasible=20, min_infeasible=0, **{"probability vectors": 2})
        return
    if case == "size-fallback":
        fleet = grid_cases.size_fallback_fleet()
        cross_fleet(oracle_mod, fleet, t, case, pairs=[(0, 0), (1, 0), (fleet.n_servers - 1, 0)])
        t.report(case, min_feasible=3, min_infeasible=0)
        return
    if case == "tiny-acc":
        fleet, grid = grid_cases.tiny_acc_case()
        extra = ()
    elif case == "invariant":
        fleet, grid, s, (r, b) = grid_cases.invariant_case()
        B, R_ = grid.batch.size, grid.replicas.size
        extra = ((s * B + list(grid.batch).index(b)) * R_ + list(grid.replicas).index(r),)
    elif case == "grid-fallback":
        fleet, grid = grid_cases.grid_fallback_case()
        extra = ()
    else:
        fleet, grid = grid_cases.shape_case(case)
        extra = ()
    cells, _ = (oracle_mod.grid_solve(fleet, grid, want_cells=True) if case in ("tiny-acc", "invariant",
                                                                                   "grid-fallback")
                else grid_cases.shape_oracle(case))
    pick = np.unique(np.concatenate([_sample_cells(rng, cells), np.array(extra, np.int64)]))
    probs = set(_pick(rng, pick[(cells["flags"][pick] & 1) == 1], 2).tolist())
    for ci in pick:
        cross_cell(oracle_mod, fleet, grid, int(ci), cells[ci], t, case, probs=int(ci) in probs)
    t.report(case, min_feasible=1, min_infeasible=0, **{"probability vectors": 1})
    if case in grid_cases.SHAPES:  # zero load and a missing profile: cells that are not analysed
        assert t.n["not analysed"] >= 1


# ---------------------------------------------------------------------------------------------------------------
# adversarial fleets and the queue-size rule (test_gpu_adversarial_paths)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["size-grid", "load-levels", "queue-cases", "tiny-total", "replicas-past-int64"])
def test_adversarial_cross(oracle_mod, case):
    """size_grid_cases: every listed batch size is srv_max_batch of a copy of the fleet (as wva_size_grid defines
    its candidates), 8 sampled candidates per case; load_levels: 8 sampled (level, server, accelerator) per fleet;
    QUEUE_CASES: the restatement refuses exactly where the library does, and on queue_fleet the wrapped cases are
    refused by both restatements; TINY_TOTAL: rates at and below the smallest positive totalRate; and load levels
    whose totalRate / rateStar lies just past 2^63, where any replica count that kept the quotient's size would bring
    the per-replica rate back under RateRange.Max."""
    from oracle import restate_np as R
    t = Tally()
    if case == "size-grid":
        rng = np.random.default_rng(0x51CE + 1)
        for k, (fleet, batches, _) in enumerate(levels.size_grid_cases()):
            S, A = fleet.n_servers, fleet.n_acc
            for j in _pick(rng, np.arange(len(batches) * S * A), 8):
                bi, sa = divmod(int(j), S * A)
                f = fleet.take_servers(np.arange(S))
                f.srv_max_batch[:] = batches[bi]
                cross_fleet(oracle_mod, f, t, f"size grid case {k}, batch {batches[bi]}", pairs=[divmod(sa, A)])
        t.report(case, min_feasible=100, min_infeasible=50)
    elif case == "load-levels":
        rng = np.random.default_rng(0x10AD + 1)
        for k, (fleet, rpm) in enumerate(levels.load_grid_cases(oracle_mod)):
            S, A = fleet.n_servers, fleet.n_acc
            for j in _pick(rng, np.arange(rpm.shape[0] * S * A), 8):
                l, sa = divmod(int(j), S * A)
                f = fleet.take_servers(np.arange(S))
                f.srv_arrival_rpm[:] = rpm[l]
                cross_fleet(oracle_mod, f, t, f"load case {k}, level {l}", pairs=[divmod(sa, A)])
        t.report(case, min_feasible=100, min_infeasible=50)
    elif case == "queue-cases":
        for name, pmb, at, out, smb, ratio, refused in levels.QUEUE_CASES:
            N, _ = levels.go_queue(pmb, at, out, smb, ratio)
            try:
                R.queue_states(int(N), ratio)
                assert not refused, name
            except R.Unsupported:
                assert refused, name
            f = levels.queue_fleet(name)
            # server 0 carries the case; a model of N = 2^20 (K up to 2^31 - 2^20) is within both domains but far
            # too large to solve here, so only the other servers are compared for those two
            pairs = [(s, a) for s in range(f.n_servers) for a in range(f.n_acc)
                     if s > 0 or name in ("at_tokens_wrap", "ratio_wrap", "n_above_2p20")]
            cross_fleet(oracle_mod, f, t, name, pairs=pairs)
        t.report(case, min_feasible=5, min_infeasible=0, **{"refused (states)": 5, "refused (batch)": 2})
    elif case == "replicas-past-int64":
        # int(math.Ceil(q)) with q >= 2^63 is MinInt64 on amd64 (allocation.go:140), so the pair takes min_replicas
        # and Analyze refuses totalRate / min_replicas (queueanalyzer.go:140): nil, though q replicas would serve it
        f = synth_fleet(6, 2, seed=17, zero_load_frac=0.0, tps_frac=0.0, max_batch_choices=(4, 8, 16))
        for s in range(f.n_servers):
            for a in range(f.n_acc):
                own = oracle_mod.create_allocation(f, s, a)
                if not own["feasible"]:
                    continue
                for k in (1.25, 3.0):
                    g = f.take_servers(np.arange(f.n_servers))
                    g.srv_arrival_rpm[s] = F(60) * F(F(own["max_rate"]) * F(1000)) * F(k * 2.0 ** 63)
                    cross_fleet(oracle_mod, g, t, f"server {s}, {k} * 2^63 rateStar", pairs=[(s, a)])
        t.report(case, min_feasible=0, min_infeasible=12)
    else:
        f = synth_fleet(4, 2, seed=13, zero_load_frac=0.0, tps_frac=0.0, max_batch_choices=(4, 8))
        f.srv_min_replicas[:] = [0, 1, 0, 2]
        for rpm in (levels.TINY_TOTAL, np.nextafter(levels.TINY_TOTAL, F(0)), F(2.0 ** -149), F(1e-30)):
            g = f.take_servers(np.arange(4))
            g.srv_arrival_rpm[:] = rpm
            cross_fleet(oracle_mod, g, t, f"rate {rpm!r}")
        # below TINY_TOTAL totalRate is 0: 0 replicas and Analyze at 0/0 on min_replicas-0 servers
        t.report(case, min_feasible=4, min_infeasible=4, **{"refused (rescale)": 2})


# ---------------------------------------------------------------------------------------------------------------
# rows of the SLO, workload and profile grids
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["slo", "workload", "profile"])
def test_level_rows_cross(oracle_mod, case):
    """Each row applied to a copy of the fleet as the grid modules compose their references, then every
    (server, accelerator): SLO targets TARGETS x TARGETS and TPS_TARGETS (FLT_MAX among them) and the rows of
    slo_levels; workload rows with in_tokens 0, out_tokens 0 and 1 and a token mix that makes N = 1, and one that puts
    N at 2^21; profile rows with alpha..delta perturbed, perf_present toggled, AccCount 0 and negative, and a perf
    batch size that puts N at 2^21."""
    t = Tally()
    if case == "slo":
        f = synth_fleet(4, 2, seed=5, max_batch_choices=(1, 2, 4, 8, 16))
        for itl in TARGETS:
            for ttft in TARGETS:
                cross_fleet(oracle_mod, at_row(f, {"slo_itl": [itl], "slo_ttft": [ttft], "slo_tps": [0.0]}, 0), t, f"itl {itl}, ttft {ttft}")
        for tps in TPS_TARGETS:
            # FLT_MAX / out_tokens over rateStar leaves int64: int() is MinInt64, then min_replicas (allocation.go:140)
            cross_fleet(oracle_mod, at_row(f, {"slo_tps": [tps]}, 0), t, f"tps {tps}")
        g = mixed_fleet(12, 3, 47, False)
        rows = dict(zip(SLO, slo_levels(g, 4, 17)))
        for l in range(4):
            cross_fleet(oracle_mod, at_row(g, rows, l), t, f"slo_levels row {l}")
        t.report(case, min_feasible=150, min_infeasible=150)
    elif case == "workload":
        f = token_fleet(12, 3, 43, True)
        rpm, it, ot = workload_levels(f, 7, 13)
        assert {0, 1, 20000} <= set(ot.ravel().tolist()) and 0 in it
        # and a row of out_tokens 20000 everywhere at row 1's rates: N = 1 on the servers without a batch size
        rpm, it = np.concatenate([rpm, rpm[1:2]]), np.concatenate([it, it[1:2]])
        ot = np.concatenate([ot, np.full((1, f.n_servers), 20000, np.int32)])
        n1 = 0
        for l in range(rpm.shape[0]):
            fl = at_row(f, dict(zip(LOAD, (rpm, it, ot))), l)
            cross_fleet(oracle_mod, fl, t, f"workload row {l}")
            n1 += sum(fl.srv_max_batch[s] == 0 and fl.srv_arrival_rpm[s] > 0 and fl.srv_out_tokens[s] > 0 and
                      fl.srv_model[s] >= 0 and pair_n(fl, s, 0) == 1 for s in range(f.n_servers))
        assert n1 >= 2, n1
        # N = 512 * 2^12 / 1 = 2^21 on server 0: refused under load, zeroLoadAllocation at rate 0 or out_tokens 0
        g = synth_fleet(4, 2, seed=83, zero_load_frac=0.0)
        g.srv_max_batch[0] = 0
        g.perf_max_batch[:] = 512
        g.perf_at_tokens[:] = 1 << 12
        for rate, out in ((5.0, 1), (0.0, 1), (5.0, 0)):
            h = g.take_servers(np.arange(4))
            h.srv_out_tokens[:] = np.where(np.arange(4) == 0, out, 1 << 16)
            h.srv_arrival_rpm[0] = rate
            cross_fleet(oracle_mod, h, t, f"N = 2^21 server, rate {rate}, out {out}")
        t.report(case, min_feasible=100, min_infeasible=40, **{"refused (batch)": 2})
    else:
        f = profile_fleet(14, 3, 31, False)
        rows = profile_rows(f, 7, 3)
        rows["perf_acc_count"][3] = np.where(np.arange(f.n_acc) % 2, 0, -2)[None, :]
        for l in range(7):
            cross_fleet(oracle_mod, at_row(f, rows, l), t, f"profile row {l}")
        g = synth_fleet(4, 2, seed=83, zero_load_frac=0.0)
        g.srv_max_batch[0] = 0
        g.perf_at_tokens[:] = 1 << 12
        g.perf_max_batch[:] = 512
        g.srv_out_tokens[:] = 1 << 7
        mb = np.repeat(g.perf_max_batch[None], 2, axis=0).copy()
        mb[1, int(g.srv_model[0]), 0] = 1 << 16  # N = 2^16 * 2^12 / 2^7 = 2^21
        for l in range(2):
            cross_fleet(oracle_mod, at_row(g, {"perf_max_batch": mb}, l), t, f"perf batch row {l}")
        t.report(case, min_feasible=150, min_infeasible=40, **{"refused (batch)": 1})


# ---------------------------------------------------------------------------------------------------------------
# the level calls' tails at the exponent windows (test_gpu_tail_windows)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["load", "slo", "profile", "bounds"])
def test_tail_windows_cross(oracle_mod, case):
    """The rows test_gpu_tail_windows steers the tails' solves onto the exponent windows with (their bands are
    asserted there), each applied to a copy of the fleet as the level calls' compositions apply it: an even sample of
    the load levels and of the SLO grid's TTFT and TPS rows, every edge row, one level of the K >= 2^23 candidate,
    a sample of the perf_alpha rows, and a sample of the bounds' batch sizes at their own load (Size at lambda_max,
    then the final Analyze).  The bounds' rate-edge pairs are left out: at a load they need more than 2^31 replicas,
    which the record's int32 does not hold."""
    t = Tally()
    sample = lambda n, k: np.unique(np.linspace(0, n - 1, k).round().astype(int))  # noqa: E731
    if case == "load":
        (main, rpm), (long, lrpm), (edge, erpm) = grid_cases.load_cases()
        for l in sample(rpm.shape[0], 16):
            cross_fleet(oracle_mod, at_row(main, {"arrival_rpm": rpm}, l), t, f"load level {l}")
        cross_fleet(oracle_mod, at_row(long, {"arrival_rpm": lrpm}, len(lrpm) // 2), t, "K >= 2^23")
        for l in range(erpm.shape[0]):
            cross_fleet(oracle_mod, at_row(edge, {"arrival_rpm": erpm}, l), t, f"edge level {l}")
        t.report(case, min_feasible=40, min_infeasible=0)
    elif case == "slo":
        (main, (itl, ttft, tps)), (edge, erows) = grid_cases.slo_cases()[:2]
        L1 = int((ttft[:, 0] > 0).sum())
        for l in list(sample(L1, 6)) + list(L1 + sample(itl.shape[0] - L1, 6)):
            cross_fleet(oracle_mod, at_row(main, dict(zip(SLO, (itl, ttft, tps))), l), t, f"SLO row {l}")
        for l in range(erows[0].shape[0]):
            cross_fleet(oracle_mod, at_row(edge, dict(zip(SLO, erows)), l), t, f"edge row {l}")
        t.report(case, min_feasible=30, min_infeasible=0)
    elif case == "profile":
        for fleet, rows in grid_cases.profile_cases():
            L = rows["perf_alpha"].shape[0]
            for l in sample(L, 12):
                cross_fleet(oracle_mod, at_row(fleet, rows, l), t, f"perf_alpha row {l}")
        t.report(case, min_feasible=40, min_infeasible=0)
    else:
        main = grid_cases.bounds_cases()[0]
        cross_fleet(oracle_mod, main, t, "bounds", pairs=[(int(s), 0) for s in sample(main.n_servers, 24)])
        t.report(case, min_feasible=20, min_infeasible=0)


# ---------------------------------------------------------------------------------------------------------------
# the load margins' records at the exponent windows and the bracket cases (test_gpu_margin_edges)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["at main", "at edge", "below", "above", "edge steps", "brackets"])
def test_margin_edges_cross(oracle_mod, case):
    """The records test_gpu_margin_edges judges wva_load_margins on (their bands are asserted there): each record's
    rate (r, the float under lo, hi, from the oracle composition) applied to a copy of the fleet, on an even sample of
    the levels and servers of each record kind; every level and server of the bracket cases."""
    t = Tally()
    sample = lambda n, k: np.unique(np.linspace(0, n - 1, k).round().astype(int))  # noqa: E731
    if case == "brackets":
        fleet, rate, lo, hi = grid_cases.bracket_cases()
        levels_, servers = range(rate.shape[0]), range(fleet.n_servers)
    else:
        _, fleet, rate, lo, hi = next(c for c in grid_cases.margin_cases() if c[0] == case)
        levels_, servers = sample(rate.shape[0], 6), sample(fleet.n_servers, 12)
    L, S = rate.shape
    xs = levels.margin_record_rates(rate, *levels.ref_margins(oracle_mod, fleet, rate, lo, hi)[:3])
    for kind, x in xs.items():
        x = x.reshape(L, S)
        for l in levels_:
            pairs = [(int(s), 0) for s in servers if not np.isnan(x[l, s])]
            if pairs:
                row = np.where(np.isnan(x[l]), rate[l], x[l]).astype(np.float32)
                cross_fleet(oracle_mod, at_row(fleet, {"arrival_rpm": row[None, :]}, 0), t, f"{kind} level {l}",
                            pairs=pairs)
    t.report(case, min_feasible=8, min_infeasible=4 if case == "brackets" else 0)
