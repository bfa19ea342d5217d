"""The grid step at its shape thresholds and rounding edges, bit for bit against the oracle (DESIGN.md 3.3).

``wva_grid_solve`` takes different code paths depending on the shape of the call, and the thresholds are host rules:

* ``prepare_grid`` turns pruning off when ``A > 256`` or ``A·R > 2048`` (the accelerator fills 8 bits of a cell key,
  and ``grid_order`` ranks a server's rows in shared memory);
* ``enqueue_grid`` gives ``grid_rows`` 32 / 64 / 128 threads by ``R`` and keeps the pair's table in shared memory only
  while ``Bmax <= kRowsSmemEntries = 1536``;
* ``grid_order`` ranks with ``q`` threads per row (q doubles while ``2·q·n <= 1024``, ``n = A·R``), walks 256 rows
  per pass, and stages the batch sizes only while ``B <= 2048`` and ``RateRange.Max`` only while ``A·B <= 4096``;
* ``grid_finalize`` gives each of its 256 threads ``ceil(A·R / 256)`` keys.

``SHAPES`` puts one case on each side of each threshold, and ``test_shape_cases_sit_on_their_sides`` restates the
rules from the fleet and the grid alone.  The ``R=`` cases also set how many rows of a pair ``grid_sort_cands``
searches for a candidate's replica level, up to 8193.  Every case runs three ways on the GPU: with the cell table
(``grid_shared``), without it (``grid_order``, its bound and ``grid_finalize``'s re-evaluation), and pruned winners
against cell-table winners byte for byte.  ``key_order_case`` adds a winner that only a key ordering batch size before accelerator
keeps below grid_order's bound.

The second half is numeric.  ``grid_order`` and ``grid_shared`` evaluate a shared row through ``row_invariant`` when
they can prove ``(float)(acc + (1 - sumP)·N) == (float)acc`` for every batch size of the grid, and through the general
``shared_cell_metrics`` otherwise.  ``invariant_fleet`` sweeps lambda per replica from ~1e-7 to ~1e-5 of the service
rate, where rows fall on both branches; ``row_classes`` restates pass 2 of the reference in numpy and sorts the rows
into (a) invariant, (b) general with a constant ``float32(in_serv)``, (c) general with ``float32(in_serv)`` varying
with N, and (d) within 2x of the bound on either side.  The ``f0`` guard (``acc < 1e-30``) is reachable:
``tiny_acc_case`` puts lambda = 2^-60 on a service rate of 2^58, both inside ``solve_row``'s windows.

Last, the same kind of gap elsewhere: the stored-vector fallbacks (128 slots) with more than 256 entries each, the load
grid beyond 65,535 levels (``unlimited_kernel``'s ``grid.y``), and ``summary_kernel`` at 256 / 257 / 1024 types.
"""
from __future__ import annotations

import functools

import numpy as np
import pytest

from tests.test_gpu_windows import _fleet, _rpm_for_lambda, chain_profile, grid_points, overflow_search_fleet
from tests.util import assert_allocs_equal
from workload_variant_autoscaler_b200 import Grid, WvaError, _abi, synth_fleet

f32 = np.float32
COLUMNS = ("feasible", "acc", "replicas", "batch", "cost", "value", "itl", "ttft", "rho", "max_rate")


# ---------------------------------------------------------------------------------------------------------------
# the host rules, restated from the fleet and the grid
# ---------------------------------------------------------------------------------------------------------------
def host_plan(fleet, grid):
    """Which side of each shape threshold a call is on, by the rules of prepare_grid, enqueue_grid, grid_order and
    grid_finalize (wva_b200.cu, wva_kernels.cuh)."""
    A, B, R = fleet.n_acc, int(grid.batch.size), int(grid.replicas.size)
    Bmax = max(1, int(grid.batch.max()))
    n = A * R
    q = 1
    while q < 32 and 2 * q * n <= 1024:
        q *= 2
    return {
        "prune": A <= 256 and Bmax < (1 << 24) and A * R <= 2048,        # prepare_grid
        "rows_threads": 128 if R >= 128 else (64 if R > 32 else 32),     # enqueue_grid
        "rows_smem": Bmax <= 1536,                                        # enqueue_grid: kRowsSmemEntries
        "order_q": q,                                                     # grid_order: counting rank
        "order_passes": -(-n // 256),                                     # grid_order: 1024 / kOrderG rows a pass
        "stage_b": B <= 2048,                                             # grid_order: batch sizes staged
        "stage_rmax": A * B <= 4096,                                      # grid_order: RateRange.Max staged
        "finalize_keys": -(-n // 256),                                    # grid_finalize: keys per thread
    }


# ---------------------------------------------------------------------------------------------------------------
# fleets of the shape cases
# ---------------------------------------------------------------------------------------------------------------
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


# name: (S, A, batch list, replica list, the sides this case must be on)
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


# ---------------------------------------------------------------------------------------------------------------
# the batch-invariant row shortcut
# ---------------------------------------------------------------------------------------------------------------
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


# ---------------------------------------------------------------------------------------------------------------
# the stored-vector fallbacks past their 128 slots
# ---------------------------------------------------------------------------------------------------------------
FB_MIN = 257  # more than twice kFbSlots = 128: every slot takes three entries or more


def grid_fallback_case():
    """N = 1024, c = 1, x = lambda from 760 to 1000: the chains overflow float64, so grid_kernel bails and
    grid_fallback re-runs every cell on the stored vector."""
    xs = np.linspace(760.0, 1000.0, 300)
    return _fleet(1.0, 0.0, [_reachable_rpm(x) for x in xs], 1024), Grid([1024], [1])


def sweep_fallback_fleet():
    return _fleet(1.0, 0.0, [600.0], 1024)


SWEEP_FB_RATES = 1024


def load_fallback_levels(oracle_mod):
    """The overflow fleet of the load grid's stored-vector test, at 150 levels per server between 0.85 and 1 of
    rateStar (one replica): each level's Analyze overflows float64 and goes to load_fallback."""
    from tests.test_gpu_load_grid import overflow_fleet
    fleet = overflow_fleet()
    cols, lams = [], []
    for s in range(fleet.n_servers):
        qa = _analyzer_of(fleet, s, 0, int(fleet.srv_max_batch[s]))
        err, _, met, _ = qa.size(0.0, 0.0, 0.0)
        assert err == 0
        star = f32(met["throughput"])
        rpm = (f32(star * f32(60)) * np.linspace(0.85, 1.0, 150)).astype(np.float32)
        total = rpm / f32(60)
        nrep = np.maximum(np.ceil(total.astype(np.float64) / np.float64(star)), 1)
        lam = ((total / nrep.astype(np.float32)) / f32(1000)).astype(np.float32)
        cols.append(rpm)
        lams.append((qa, lam))
    return fleet, np.stack(cols, axis=1), lams


def size_fallback_fleet():
    """overflow_search_fleet's two servers, 130 times each: 260 candidates whose ITL bisection overflows float64
    (test_overflow_search_cases_bail_inside_the_search), each re-run by size_fallback."""
    return overflow_search_fleet(7.55, 0.0).take_servers(np.arange(260) % 2)


# ---------------------------------------------------------------------------------------------------------------
# CPU: every case on its side, every class populated, every fallback past its slots
# ---------------------------------------------------------------------------------------------------------------
def test_shape_cases_sit_on_their_sides():
    for name, (_, _, _, _, sides) in SHAPES.items():
        plan = host_plan(*shape_case(name))
        wrong = {k: plan[k] for k, v in sides.items() if plan[k] != v}
        assert not wrong, f"{name}: {wrong}"
    # and each threshold has a case on both of its sides
    plans = [host_plan(*shape_case(n)) for n in SHAPES]
    for key in ("prune", "rows_smem", "stage_b", "stage_rmax"):
        assert {p[key] for p in plans} == {True, False}, key
    for key, values in (("rows_threads", {32, 64, 128}), ("order_q", {1, 2, 4}), ("order_passes", {1, 2, 3}),
                        ("finalize_keys", {1, 2, 3})):
        assert values <= {p[key] for p in plans}, key
    # the exact edges: 2048 / 2049 and 256 / 257 on the two sides
    assert [shape_case(n)[0].n_acc * shape_case(n)[1].replicas.size for n in ("A*R=2048", "A*R=2049", "n=256", "n=257",
                                                                             "n=512", "n=513")] == \
        [2048, 2049, 256, 257, 512, 513]
    assert [shape_case(n)[1].batch.size for n in ("B=2048", "B=2049")] == [2048, 2049]
    assert [shape_case(n)[0].n_acc * shape_case(n)[1].batch.size for n in ("A*B=4096", "A*B=4097")] == [4096, 4097]
    assert [int(shape_case(n)[1].batch.max()) for n in ("Bmax=1536", "Bmax=1537")] == [1536, 1537]
    assert [shape_case(f"R={r}")[1].replicas.size for r in (32, 33, 64, 65, 127, 128, 8193)] == \
        [32, 33, 64, 65, 127, 128, 8193]


def test_repeated_unsorted_batches_at_the_staging_edges():
    for name in ("B=2048", "B=2049", "A*B=4096", "A*B=4097"):
        b = shape_case(name)[1].batch
        assert np.unique(b).size < b.size and not np.all(np.diff(b) >= 0), name


@pytest.mark.parametrize("name", list(SHAPES))
def test_shape_case_has_every_pair_class_winner_source_and_tie(oracle_mod, name):
    """Zero load, a missing profile and a TPS target in every case; winners from shared-chain cells and from
    grid_kernel cells; and (with two accelerators or more) a winner whose cell ties with another accelerator's."""
    fleet, grid = shape_case(name)
    cells, win = shape_oracle(name)
    assert fleet.srv_arrival_rpm[0] == 0 and win[0]["feasible"] == 1 and win[0]["replicas"] >= 1
    assert not fleet.perf_present[fleet.srv_model[3], fleet.n_acc - 1] and fleet.srv_slo_tps[2] > 0
    assert win["feasible"][1:].sum() >= 2
    shared, kernel, ties = winner_mix(fleet, grid, cells, win)
    assert shared >= 1 and kernel >= 1, (shared, kernel)
    if fleet.n_acc >= 2:
        assert ties >= 1


def test_row_stats_are_the_oracle_probabilities(oracle_mod):
    """The numpy pass 2 starts from the oracle's own normalised vector (a sample of rows, bit for bit)."""
    fleet, grid = invariant_fleet(), Grid(INV_BATCH, INV_REPLICAS)
    st = row_stats(fleet, grid)
    Bmax = int(grid.batch.max())
    for k in range(0, st["s"].size, 17):
        qa = _analyzer_of(fleet, int(st["s"][k]), 0, Bmax)
        assert qa.solve(float(st["lam"][k]))["is_valid"]
        want = qa.probs()
        assert np.array_equal(st["q"][k].view(np.uint64), want.view(np.uint64)), k


def test_row_classes_are_populated(oracle_mod):
    st = row_classes(invariant_fleet(), Grid(INV_BATCH, INV_REPLICAS))
    cls, near = list(st["cls"]), list(st["near"])
    assert None not in cls  # every row shares its chain
    counts = {c: cls.count(c) for c in ("a", "b", "c")} | {n: near.count(n) for n in ("near-", "near+")}
    assert min(counts.values()) >= 3, counts
    # rows whose float32(in_serv) varies with N are the ones the general branch exists for
    for k, c in enumerate(cls):
        if c == "c":
            assert len(set(st["in_serv"][k])) > 1
    guard = row_classes(*tiny_acc_case())
    assert guard["cls"][:2] == ["guard", "guard"] and (guard["acc"][:2] < 1e-30).all() and guard["cls"][2] == "a"


def test_invariant_case_slo_sits_on_a_class_c_cell(oracle_mod):
    fleet, grid, s, (r, b) = invariant_case()
    st = row_classes(fleet, grid)
    k = [i for i in range(st["s"].size) if st["s"][i] == s and st["r"][i] == r][0]
    assert st["cls"][k] == "c" and fleet.srv_slo_ttft[s] > 0


def test_fallback_cases_send_more_than_256_entries(oracle_mod):
    fleet, grid = grid_fallback_case()
    cells, _ = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    assert grid_points(fleet, grid, cells["flags"])["over"].sum() >= FB_MIN
    from tests.test_gpu_windows import sweep_points
    fleet = sweep_fallback_fleet()
    o = oracle_mod.sweep(fleet, SWEEP_FB_RATES)
    assert sweep_points(fleet, SWEEP_FB_RATES, o["valid"])["over"].sum() >= FB_MIN
    fleet, _, lams = load_fallback_levels(oracle_mod)
    assert sum(int(chain_profile(qa.serv_rate(), qa.K, lam)["over"].sum()) for qa, lam in lams) >= FB_MIN
    fleet = size_fallback_fleet()
    qa = _analyzer_of(fleet, 0, 0, 1024)
    lmax = f32(f32(qa.rate_range()[1]) / f32(1000))
    assert chain_profile(qa.serv_rate(), qa.K, [lmax])["over"][0]  # every candidate's search bails
    assert fleet.n_servers * fleet.n_acc >= FB_MIN and len({tuple(fleet.perf_alpha[m]) for m in fleet.srv_model}) == 1


# ---------------------------------------------------------------------------------------------------------------
# GPU: bit for bit
# ---------------------------------------------------------------------------------------------------------------
def _three_ways(engine, fleet, grid, cells_o, win_o, what):
    """With the cell table (cells and winners against the oracle), without it (winners against the oracle), and the
    pruned winners against the cell-table winners byte for byte."""
    from tests.test_gpu_grid_pruning import _same_winners
    from tests.test_gpu_windows import _cells_equal
    cells_g, win_c = engine.grid_solve(fleet, grid, want_cells=True)
    _cells_equal(cells_g, cells_o, what)
    assert_allocs_equal(win_c, win_o, f"{what}: winners (cell table)")
    _, win_p = engine.grid_solve(fleet, grid)
    assert_allocs_equal(win_p, win_o, f"{what}: winners (pruned)")
    _same_winners(win_p, win_c, f"{what}: pruned vs cell table")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(SHAPES))
def test_grid_at_shape_threshold(engine, oracle_mod, name):
    fleet, grid = shape_case(name)
    cells_o, win_o = shape_oracle(name)
    _three_ways(engine, fleet, grid, cells_o, win_o, name)


@pytest.mark.gpu
def test_grid_rows_on_both_branches_of_row_invariant(engine, oracle_mod):
    """Shared rows on the invariant and the general branch and near the bound, with one server's TTFT target on a
    class-(c) cell that wins."""
    fleet, grid, s, (r, b) = invariant_case()
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    assert (win_o[s]["replicas"], win_o[s]["batch"]) == (r, b)
    _three_ways(engine, fleet, grid, cells_o, win_o, "row_invariant branches")


@pytest.mark.gpu
def test_grid_rows_below_the_f0_guard(engine, oracle_mod):
    fleet, grid = tiny_acc_case()
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    _three_ways(engine, fleet, grid, cells_o, win_o, "acc < 1e-30")


@pytest.mark.gpu
def test_grid_fallback_past_its_slots(engine, oracle_mod):
    fleet, grid = grid_fallback_case()
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    _three_ways(engine, fleet, grid, cells_o, win_o, "grid_fallback, 300 cells")


@pytest.mark.gpu
def test_sweep_fallback_past_its_slots(engine, oracle_mod):
    from tests.test_gpu_windows import _sweep_equal
    fleet = sweep_fallback_fleet()
    o = oracle_mod.sweep(fleet, SWEEP_FB_RATES)
    _sweep_equal(engine.sweep(fleet, SWEEP_FB_RATES), o, "sweep_fallback")


@pytest.mark.gpu
def test_load_fallback_past_its_slots(engine, oracle_mod):
    from tests.test_gpu_load_grid import ref_load_grid
    fleet, rpm, _ = load_fallback_levels(oracle_mod)
    cand_o, win_o = ref_load_grid(oracle_mod, fleet, rpm)
    cand_g, win_g = engine.load_grid(fleet, rpm, want_candidates=True)
    assert_allocs_equal(cand_g, cand_o, "load_fallback: candidates")
    assert_allocs_equal(win_g, win_o, "load_fallback: winners")
    assert cand_o["feasible"].sum() >= FB_MIN


@pytest.mark.gpu
def test_size_fallback_past_its_slots(engine, oracle_mod):
    """The oracle sizes the two distinct servers; the 130 copies of each must come out the same."""
    fleet = size_fallback_fleet()
    cand2, win2 = oracle_mod.solve(overflow_search_fleet(7.55, 0.0))
    idx = np.arange(fleet.n_servers) % 2
    cand_g, win_g = engine.solve(fleet)
    assert_allocs_equal(cand_g, cand2.reshape(-1)[idx], "size_fallback: candidates")
    assert_allocs_equal(win_g, win2[idx], "size_fallback: winners")


class _Slice:
    """Records [i0, i1) of an Allocs, in the shape assert_allocs_equal reads."""

    def __init__(self, allocs, i0, i1):
        self.n = i1 - i0
        self._a, self._i0 = allocs, i0
        for f in COLUMNS:
            setattr(self, f, np.asarray(getattr(allocs, f))[i0:i1])

    def record(self, i):
        return self._a.record(self._i0 + i)


LOAD_PERIOD = [0.0, 30.0, 600.0, 1e-3, 4000.0, 120.0, 2500.0]


@pytest.mark.gpu
def test_load_grid_beyond_65535_levels(engine, oracle_mod):
    """unlimited_kernel runs grid.y = min(L, 65535) blocks of levels: at L = 65,537 levels that repeat with period
    P = 7, block l equals block l mod P byte for byte, and the first P blocks equal the oracle's composition."""
    from tests.test_gpu_load_grid import ref_load_grid
    fleet = synth_fleet(1, 2, seed=53, zero_load_frac=0.0, tps_frac=0.0)
    L, P, A = 65537, len(LOAD_PERIOD), 2
    rpm = np.tile(np.float32(LOAD_PERIOD), -(-L // P))[:L].reshape(L, 1)
    cand_g, win_g = engine.load_grid(fleet, rpm, want_candidates=True)
    cand_o, win_o = ref_load_grid(oracle_mod, fleet, rpm[:P])
    assert_allocs_equal(_Slice(cand_g, 0, P * A), cand_o, "first P candidate blocks")
    assert_allocs_equal(_Slice(win_g, 0, P), win_o, "first P winner blocks")
    assert win_o["feasible"].sum() >= P - 1
    lv = np.arange(L) % P
    for allocs, per in ((cand_g, A), (win_g, 1)):
        for f in COLUMNS:
            col = np.asarray(getattr(allocs, f)).reshape(L, per)
            assert np.array_equal(col.view(np.uint8), col[lv].view(np.uint8)), f


SUMMARY_TYPES = {256: [0, 255], 257: [0, 255, 256], 1024: [0, 255, 256, 511, 512, 767, 768, 1023]}


def _summary_fleet(T, types):
    f = synth_fleet(60, len(types), seed=59, max_batch_choices=(4, 8, 16), zero_load_frac=0.1)
    f.acc_cost[:] = 40.0  # every accelerator wins somewhere
    f.acc_type[:] = types
    f.type_capacity = np.full(T, 1 << 20, np.int32)
    return f


@pytest.mark.gpu
@pytest.mark.parametrize("T", sorted(SUMMARY_TYPES))
def test_summary_at_type_edges(engine, oracle_mod, T):
    """summary_kernel's thread t owns types t, t + 256, ...: accelerators on the first and last type each thread
    owns, at 256, 257 and kSumMaxTypes = 1024 types."""
    from tests.test_summary import _check
    f = _summary_fleet(T, SUMMARY_TYPES[T])
    _, win_o = oracle_mod.solve(f)
    engine.solve(f)
    t, _ = _check(engine, oracle_mod, f, win_o)
    assert t["present"][SUMMARY_TYPES[T]].all() and t["present"].sum() == len(SUMMARY_TYPES[T])


@pytest.mark.gpu
def test_summary_above_its_type_limit_is_unsupported(engine):
    f = _summary_fleet(1025, [0, 1024])
    engine.solve(f)
    with pytest.raises(WvaError) as e:
        engine.summarize(1025)
    assert e.value.code == _abi.WVA_ERR_UNSUPPORTED


def key_order_case():
    """A cell key orders batch size before accelerator.  One server, two accelerators with one cost per replica:
    on accelerator 0 (alpha = 20, x = lambda / servRate[0] = 20) batch size 16 is above RateRange.Max and 128 is a
    feasible shared-chain cell; on accelerator 1 (alpha = 8, x = 8) batch size 16 is a feasible grid_kernel cell.
    grid_order's bound is accelerator 0's cell at 128, and the winner, accelerator 1 at 16, lies below it only if the
    key compares the batch size first."""
    f = synth_fleet(1, 2, seed=61, zero_load_frac=0.0, tps_frac=0.0)
    f.max_queue_to_batch_ratio = 1
    f.acc_cost[:] = 80.0
    f.perf_acc_count[:] = 1
    f.perf_alpha[:] = [[20.0, 8.0]]
    f.perf_beta[:] = 0.01  # > 0: a finite effective concurrency
    f.perf_gamma[:] = f.perf_delta[:] = 0.0
    f.srv_in_tokens[:], f.srv_out_tokens[:] = 1, 2
    f.srv_slo_itl[:], f.srv_slo_ttft[:], f.srv_slo_tps[:] = 150.0, 1500.0, 0.0
    f.srv_cur_acc[:], f.srv_cur_replicas[:], f.srv_cur_cost[:] = -1, 0, 0.0
    f.srv_arrival_rpm[:] = _rpm_for_lambda(1.0)
    return f, Grid([128, 16], [1, 2])


def test_key_order_case_puts_the_winner_below_a_shared_cell_of_a_lower_accelerator(oracle_mod):
    fleet, grid = key_order_case()
    cells, win = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    fl = cells["flags"].reshape(2, 2, 2)  # [accelerator, batch index, replica index]; batch [128, 16]
    assert (win[0]["feasible"], win[0]["acc"], win[0]["replicas"], win[0]["batch"]) == (1, 1, 1, 16)
    assert not cell_shares_row(fleet, 0, 1, 16, 1)                          # the winner is grid_kernel's
    assert fl[0, 0, 0] == 3 and cell_shares_row(fleet, 0, 0, 128, 1)     # a feasible shared cell, same group
    assert fl[0, 1, 0] == 0                                                # accelerator 0 cannot analyse 16


@pytest.mark.gpu
def test_pruned_key_orders_batch_before_accelerator(engine, oracle_mod):
    fleet, grid = key_order_case()
    cells_o, win_o = oracle_mod.grid_solve(fleet, grid, want_cells=True)
    _three_ways(engine, fleet, grid, cells_o, win_o, "key order")
