"""Host-side mirror of the reference's optimizer interface over the C ABI.

``Engine`` plays the role of ``core.System`` + ``manager.Manager`` +
``solver.Optimizer`` for the hot path (pkg/manager/manager.go:13-27,
pkg/solver/optimizer.go:24-35, pkg/core/system.go:303-319): hand it the fleet
(``config.SystemSpec`` packed as a :class:`Fleet`), get candidate allocations
(``Server.Calculate``) and the per-server solution (``GenerateSolution``).  All compute
happens in the CUDA library; nothing here touches the oracle.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _abi, _lib
from ._abi import Allocs
from .fleet import Fleet, Grid


class WvaError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"wva error {code}: {msg}")
        self.code = code


def greedy_solve(fleet: Fleet, candidates: Allocs):
    """``Solver.SolveGreedy`` + best-effort policies (pkg/solver/greedy.go:35-341) over a candidate table the
    caller already holds (``wva_solve_greedy``: host only, no GPU).  ``candidates`` [S * A] carries
    ``value`` = transition penalty (what ``Engine.analyze`` returns); it is modified in place where the reference
    scales best-effort allocations.  Returns (candidates, winners [S])."""
    L = _lib.lib()
    if candidates.n != fleet.n_servers * fleet.n_acc:
        raise ValueError("candidates must hold n_servers * n_acc records")
    win = Allocs(fleet.n_servers)
    fc, cc, wc = fleet.as_c(), candidates.as_c(), win.as_c()
    rc = L.wva_solve_greedy(C.byref(fc), C.byref(cc), C.byref(wc))
    if rc != 0:
        raise WvaError(rc, L.wva_strerror(rc).decode())
    return candidates, win


def accelerator_demand(fleet: Fleet, threshold, candidates: Allocs, a: int):
    """The fleet's demand curve for accelerator ``a`` in unlimited mode, from ``Engine.price_thresholds``' output
    (host only, no GPU) -> (breakpoints, units).

    ``breakpoints`` are the ascending distinct thresholds of column ``a`` in (0, MaxFloat32].  They cut the prices
    [+0, MaxFloat32] into ``len(breakpoints) + 1`` stretches: [0, b_0), [b_0, b_1), ..., [b_last, MaxFloat32].
    ``units[j]`` (int64) is the number of ``a``'s units the unlimited winners use at every price of stretch ``j``,
    counted as ``System.AllocateByType`` counts them (pkg/core/system.go:271-300): replicas * NumInstances *
    multiplicity over the servers whose winner is ``a``'s candidate, i.e. whose threshold lies above the price.  A
    zero-replica candidate (accelerator "") uses no units."""
    return _demand(fleet, threshold, candidates, a, fleet.perf_acc_count)


def _demand(fleet: Fleet, threshold, candidates: Allocs, a: int, acc_count):
    """accelerator_demand with NumInstances read from acc_count (M, A) in place of the fleet's perf_acc_count."""
    S, A = fleet.n_servers, fleet.n_acc
    if not 0 <= a < A:
        raise ValueError(f"accelerator {a} out of range [0, {A})")
    th = np.ascontiguousarray(threshold, np.float32)
    if th.shape != (S, A) or candidates.n != S * A:
        raise ValueError("threshold must have shape (n_servers, n_acc) and candidates n_servers * n_acc records")
    col = th[:, a]
    idx = np.arange(S) * A + a
    m = fleet.srv_model
    on_a = candidates.acc[idx] == a  # a feasible record in column a is on a, or on "" with 0 replicas
    inst = np.maximum(acc_count[np.where(on_a, m, 0), a].astype(np.int64), 1)
    units = np.where(on_a, candidates.replicas[idx].astype(np.int64) * inst, 0) * int(fleet.acc_multiplicity[a])
    breakpoints = np.unique(col[(col > 0) & np.isfinite(col)])
    starts = np.concatenate([[np.float32(0.0)], breakpoints]).astype(np.float32)
    # server s wins on the stretches that start below threshold[s]: the first k[s] of them
    k = np.searchsorted(starts, col, side="left")
    per_k = np.zeros(starts.size + 1, np.int64)
    np.add.at(per_k, k, units)
    return breakpoints, np.cumsum(per_k[::-1])[::-1][1:]


def demand_by_level(fleet: Fleet, threshold, candidates: Allocs, a: int, *, perf_acc_count=None):
    """The demand curve for accelerator ``a`` at every row of ``Engine.price_threshold_grid``,
    ``price_threshold_trace``, ``profile_price_threshold_grid`` or ``profile_price_threshold_trace`` (host only, no
    GPU) -> (breakpoints, units (L, len(breakpoints) + 1) int64).

    ``breakpoints`` is the ascending union over the rows of column ``a``'s distinct thresholds in (0, MaxFloat32];
    it cuts the prices [+0, MaxFloat32] into stretches as ``accelerator_demand`` does.  ``units[l, j]`` is
    ``accelerator_demand``'s count for row ``l`` (threshold block ``l`` and candidate block ``l``, which for a trace
    is tick ``l``'s block, masked against its current allocation) on stretch ``j`` of the union.
    ``perf_acc_count`` (shape (L, M, A), the profile calls' AccCount rows; None: the fleet's own at every row) makes
    row ``l`` count NumInstances at that row's AccCount."""
    S, A = fleet.n_servers, fleet.n_acc
    th = np.ascontiguousarray(threshold, np.float32)
    if th.ndim != 3 or th.shape[1:] != (S, A) or candidates.n != th.shape[0] * S * A:
        raise ValueError("threshold must have shape (L, n_servers, n_acc) and candidates L * n_servers * n_acc "
                         "records")
    if perf_acc_count is not None:
        perf_acc_count = np.asarray(perf_acc_count)
        if perf_acc_count.shape != (th.shape[0], fleet.n_models, A):
            raise ValueError(f"perf_acc_count must have shape ({th.shape[0]}, {fleet.n_models}, {A}), got "
                             f"{perf_acc_count.shape}")
    n = S * A
    per_level = []
    for l in range(th.shape[0]):
        block = Allocs(n)
        for k in block.columns():
            getattr(block, k)[:] = getattr(candidates, k)[l * n:(l + 1) * n]
        per_level.append(_demand(fleet, th[l], block, a,
                                 fleet.perf_acc_count if perf_acc_count is None else perf_acc_count[l]))
    breakpoints = np.unique(np.concatenate([bp for bp, _ in per_level] + [np.zeros(0, np.float32)]))
    starts = np.concatenate([[np.float32(0.0)], breakpoints]).astype(np.float32)
    units = np.zeros((th.shape[0], starts.size), np.int64)
    for l, (bp, u) in enumerate(per_level):
        # the level's own stretch that holds each union stretch: the number of its breakpoints at or below the start
        units[l] = u[np.searchsorted(bp, starts, side="right")]
    return breakpoints, units


# The smallest positive float32 target, and the position past +Inf as a uint32 key (its float is a NaN): the SLO
# bounds order targets by their bit patterns, which are ordered like the positive values.
_MIN_TARGET = np.float32(np.finfo(np.float32).smallest_subnormal)
_PAST_INF = np.uint32(0x7F800001)


def _target_keys(x):
    """Bit patterns of positive float32 targets or NaN (past +Inf) as ordered uint32 keys."""
    x = np.ascontiguousarray(x, np.float32)
    return np.where(np.isnan(x), _PAST_INF, x.view(np.uint32)).astype(np.uint32)


def _key_targets(k):
    k = np.ascontiguousarray(k, np.uint32)
    return np.where(k == _PAST_INF, np.float32(np.nan), k.view(np.float32)).astype(np.float32)


def _zero_load_pairs(fleet: Fleet):
    """(S, A) bool: the pairs whose candidate is zeroLoadAllocation (pkg/core/allocation.go:42-75 with the
    keepAccelerator rule of server.go:70-82): feasible at every target, since neither search runs."""
    S, A = fleet.n_servers, fleet.n_acc
    acc = np.arange(A)[None, :]
    m = fleet.srv_model.astype(np.int64)
    known = (m >= 0) & (m < fleet.n_models)
    present = np.zeros((S, A), bool)
    present[known] = fleet.perf_present[m[known]] != 0
    cur = fleet.srv_cur_acc[:, None]
    masked = (fleet.srv_keep_acc[:, None] != 0) & (cur != -1) & (cur != acc)
    rpm, tin, tout = fleet.srv_arrival_rpm, fleet.srv_in_tokens, fleet.srv_out_tokens
    gated = (rpm < 0) | (tin < 0) | (tout < 0) | (fleet.srv_has_target == 0)
    zero = (rpm == 0) | (tout == 0)
    return present & ~masked & (~gated & zero)[:, None]


def slo_envelope(fleet: Fleet, bounds, which: int):
    """Per server, the targets of search ``which`` (0: TTFT, 1: ITL) between which its winner depends on that
    target, from ``Engine.slo_bounds``' output (host only, no GPU) -> (floor [S], ceiling [S]) float32.

    Both are exact statements about ``solve``'s unlimited winner of server ``s`` on the fleet with ``s``'s target
    of search ``which`` set to ``t`` (any positive float32 up to +Inf) and every other column unchanged:

    * ``floor[s]`` is the smallest positive target at which some candidate of ``s`` is not NIL (a zero-load
      candidate is never NIL).  At every target below it (``not t >= floor[s]``) every candidate is nil whatever
      the other targets are, so ``s``'s winner is nil.
    * ``ceiling[s]`` is the smallest target from which on every candidate of ``s`` that reads the target (kinds 1
      to 3) is FREE.  At every target ``t >= ceiling[s]`` each candidate, and so ``s``'s winner, is byte for byte
      the one with that target set to 0.  A server with no such candidate gets the smallest positive target.

    +Inf is itself a target, so where no target qualifies the value is NaN, as for the bounds' b1 and b2: the
    position past +Inf, which no comparison ``t >= x`` reaches."""
    kind, _, _, b1, b2 = (np.asarray(x) for x in bounds)
    S, A = fleet.n_servers, fleet.n_acc
    if which not in (0, 1):
        raise ValueError("which must be 0 (TTFT) or 1 (ITL)")
    if kind.shape != (S, A, 2):
        raise ValueError("bounds must have shape (n_servers, n_acc, 2)")
    k, k1, k2 = kind[..., which], _target_keys(b1[..., which]), _target_keys(b2[..., which])
    lo = _target_keys(_MIN_TARGET)
    # first target at which the candidate is not NIL: rising after its NIL stretch, falling from the start unless
    # its NIL stretch is everything
    not_nil = np.full((S, A), _PAST_INF, np.uint32)
    not_nil[k == 2] = k1[k == 2]
    not_nil[(k == 3) & (k2 > lo)] = lo
    not_nil[_zero_load_pairs(fleet)] = lo
    # first target from which on the candidate is FREE: rising from b2, falling only when FREE is every target
    free = np.full((S, A), lo, np.uint32)
    free[k == 1] = _PAST_INF
    free[k == 2] = k2[k == 2]
    free[k == 3] = np.where(k1[k == 3] == _PAST_INF, lo, _PAST_INF)
    floor = not_nil.min(axis=1) if A else np.full(S, _PAST_INF, np.uint32)
    ceiling = free.max(axis=1) if A else np.full(S, lo, np.uint32)
    return _key_targets(floor), _key_targets(ceiling)


def within_margins(lo, hi, flags, new_rpm, rpm_hi):
    """The (L, S) mask of servers whose new arrival rate lies inside the stretch ``Engine.load_margins`` returned
    for them (host only, no GPU).  For those servers ``load_grid`` at the new rate returns the decision key of
    ``at``, so a reconcile loop can skip their re-solve.

    The stretch is ``[lo, hi)``.  An open end is the window's edge, not a change: below ``rpm_lo`` (= ``lo`` with
    ``MARGIN_LO_OPEN``) and above ``rpm_hi`` (the window tops the margins were computed over, needed because ``hi``
    is +Inf with ``MARGIN_HI_OPEN``) nothing is known, so a rate there is outside.  A stretch truncated at the rate
    itself (``lo == hi``) holds nothing; NaN is never inside.

    It works unchanged on ``Engine.load_margin_trace``'s result: there the servers inside their stretch at tick t
    keep the decision the replayed reconcile makes at tick t.  On ``Engine.workload_margins`` and
    ``Engine.workload_margin_trace`` a new rate inside the stretch keeps the row's decision when the new tokens equal
    the row's; the mask does not look at tokens.  On ``Engine.profile_margins`` and ``Engine.profile_margin_trace``
    it holds when the tokens, prices and profiles also stay the row's, and on ``Engine.slo_margins`` and
    ``Engine.slo_margin_trace`` when the tokens and targets do."""
    lo, hi, top, x = (np.asarray(v, np.float32) for v in (lo, hi, rpm_hi, new_rpm))
    flags = np.asarray(flags, np.uint8)
    if not lo.shape == hi.shape == flags.shape == top.shape == x.shape:
        raise ValueError("lo, hi, flags, new_rpm and rpm_hi must have one shape")
    hi_open = (flags & _abi.MARGIN_HI_OPEN) != 0
    return (lo <= x) & np.where(hi_open, x <= top, x < hi)


# the fleet column each load or target row list replaces (every other row list is named after its column)
# (the load margins' window rows are rates, shaped and typed like the arrival rates)
_ROW_COLUMN = {"arrival_rpm": "srv_arrival_rpm", "in_tokens": "srv_in_tokens", "out_tokens": "srv_out_tokens",
               "slo_itl": "srv_slo_itl", "slo_ttft": "srv_slo_ttft", "slo_tps": "srv_slo_tps",
               "rpm_lo": "srv_arrival_rpm", "rpm_hi": "srv_arrival_rpm"}
_PROFILE_COLUMNS = ("acc_cost", "perf_present", "perf_alpha", "perf_beta", "perf_gamma", "perf_delta",
                    "perf_acc_count", "perf_max_batch", "perf_at_tokens")


def _row_lists(fleet: Fleet, given: dict):
    """The row lists of a grid or trace call, by argument name -> ({name: C-contiguous array of shape (L, *the
    column's shape) in the column's dtype}, L).  A list of None is left out; L is the lists' common first dimension,
    None when every list is None."""
    shape = {"S": (fleet.n_servers,), "A": (fleet.n_acc,), "MA": (fleet.n_models, fleet.n_acc)}
    cols = {name: (dt, shape.get(n)) for name, dt, n in _abi.FLEET_COLUMNS}
    rows, L = {}, None
    for name, x in given.items():
        if x is None:
            continue
        dt, tail = cols[_ROW_COLUMN.get(name, name)]
        r = np.ascontiguousarray(x, dt)
        if r.ndim != 1 + len(tail) or r.shape[1:] != tail or (L is not None and r.shape[0] != L):
            want = "L" if L is None else str(L)
            raise ValueError(f"{name} must have shape ({want}, {', '.join(map(str, tail))}), got {r.shape}")
        L = r.shape[0]
        rows[name] = r
    return rows, L


def _profile_rows_c(rows: dict):
    """wva_profile_rows over the profile columns in rows (NULL for the others)."""
    return _abi.ProfileRowsC(*[_abi.ptr(rows[k].reshape(-1)) if k in rows else None for k in _PROFILE_COLUMNS])


class Engine:
    """One engine per GPU (one process per GPU in multi-GPU runs)."""

    def __init__(self, device: int = 0):
        self._L = _lib.lib()
        h = C.c_void_p()
        rc = self._L.wva_create(C.byref(h), device)
        if rc != 0:
            raise WvaError(rc, self._L.wva_strerror(rc).decode() + " (the CUDA path has no CPU fallback)")
        self._h = h
        self._n_servers = self._n_acc = None  # shape of the fleet resident on the device

    def close(self):
        if getattr(self, "_h", None):
            self._L.wva_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int):
        if rc != 0:
            raise WvaError(rc, f"{self._L.wva_strerror(rc).decode()}: {self._L.wva_last_error(self._h).decode()}")

    # -- reference-shaped calls --------------------------------------------
    def analyze(self, fleet: Fleet) -> Allocs:
        """``Server.Calculate`` for every server -> candidates [S*A] (pkg/core/server.go:55-67)."""
        cand = Allocs(fleet.n_servers * fleet.n_acc)
        fc, cc = fleet.as_c(), cand.as_c()
        self._resident(fleet)
        self._check(self._L.wva_analyze(self._h, C.byref(fc), C.byref(cc)))
        return cand

    def solve(self, fleet: Fleet, want_candidates: bool = True):
        """``Manager.Optimize`` + ``GenerateSolution`` -> (candidates [S*A] | None, winners [S])."""
        cand = Allocs(fleet.n_servers * fleet.n_acc) if want_candidates else None
        win = Allocs(fleet.n_servers)
        fc, wc = fleet.as_c(), win.as_c()
        cc = cand.as_c() if cand is not None else None
        self._resident(fleet)
        self._check(self._L.wva_solve(self._h, C.byref(fc), C.byref(cc) if cc is not None else None, C.byref(wc)))
        return cand, win

    def grid_solve(self, fleet: Fleet, grid: Grid, want_cells: bool = False, out: Allocs | None = None):
        """Full (server x acc x batch x replica) grid -> (cells | None, winners [S]).

        ``out``: an ``Allocs`` of ``fleet.n_servers`` records to write the winners into (a reconcile
        loop reuses one instead of allocating ten columns per call)."""
        n = fleet.n_servers * fleet.n_acc * int(grid.batch.size) * int(grid.replicas.size)
        if out is not None and out.n != fleet.n_servers:
            raise ValueError("out must hold fleet.n_servers records")
        win = out if out is not None else Allocs(fleet.n_servers)
        cells = None
        cc = None
        if want_cells:
            cells = {"flags": np.zeros(n, np.uint8)}
            for k in ("ttft", "itl", "rho", "throughput"):
                cells[k] = np.zeros(n, np.float32)
            cc = _abi.CellsC(*[_abi.ptr(cells[k]) for k in ("flags", "ttft", "itl", "rho", "throughput")])
        fc, gc, wc = fleet.as_c(), grid.as_c(), win.as_c()
        self._resident(fleet)
        self._check(self._L.wva_grid_solve(self._h, C.byref(fc), C.byref(gc), C.byref(cc) if cc is not None else None,
                                           C.byref(wc)))
        return cells, win

    def size_grid(self, fleet: Fleet, batches, want_candidates: bool = False, out: Allocs | None = None):
        """The reference's ``Server.Calculate`` at every listed batch size -> (candidates [S*A*B] | None,
        winners [S]).

        Candidate ``(s*A + a)*B + bi`` is what ``analyze`` returns for ``(s, a)`` with every server's
        ``srv_max_batch`` set to ``batches[bi]``; ``winners[s]`` is the min-value candidate (ties: smaller batch
        size, then lower accelerator id; see ``wva_size_grid`` in include/wva_b200.h).  ``out``: an ``Allocs``
        of ``fleet.n_servers`` records to write the winners into."""
        b = np.ascontiguousarray(batches, np.int32).reshape(-1)
        if out is not None and out.n != fleet.n_servers:
            raise ValueError("out must hold fleet.n_servers records")
        win = out if out is not None else Allocs(fleet.n_servers)
        cand = Allocs(fleet.n_servers * fleet.n_acc * int(b.size)) if want_candidates else None
        fc, wc = fleet.as_c(), win.as_c()
        cc = cand.as_c() if cand is not None else None
        self._resident(fleet)
        self._check(self._L.wva_size_grid(self._h, C.byref(fc), int(b.size), _abi.ptr(b),
                                          C.byref(cc) if cc is not None else None, C.byref(wc)))
        return cand, win

    def load_grid(self, fleet: Fleet, arrival_rpm, want_candidates: bool = False, out: Allocs | None = None):
        """The reference's ``Server.Calculate`` and ``SolveUnlimited`` winner at each row of ``arrival_rpm``
        (shape (L, S), req/min) -> (candidates [L*S*A] | None, winners [L*S]), both level-major.

        Candidate block ``l`` is what ``analyze`` returns for the fleet with ``srv_arrival_rpm`` = row ``l``, and
        winner block ``l`` is ``solve``'s winners for it in unlimited mode (see ``wva_load_grid`` in
        include/wva_b200.h); ``fleet.srv_arrival_rpm`` is not read.  ``out``: an ``Allocs`` of ``L * S`` records
        to write the winners into."""
        rows, L = _row_lists(fleet, {"arrival_rpm": arrival_rpm})
        if L is None:
            raise ValueError("arrival_rpm is required")
        return self._level_call(self._L.wva_load_grid, fleet, L, [_abi.ptr(rows["arrival_rpm"].reshape(-1))],
                                want_candidates, out)

    def slo_grid(self, fleet: Fleet, slo_itl, slo_ttft, slo_tps, want_candidates: bool = False,
                 out: Allocs | None = None):
        """The reference's ``Server.Calculate`` and ``SolveUnlimited`` winner at each row of service-class targets
        (``slo_itl``, ``slo_ttft``, ``slo_tps``, each of shape (L, S), in the fleet columns' units) ->
        (candidates [L*S*A] | None, winners [L*S]), both level-major.

        Candidate block ``l`` is what ``analyze`` returns for the fleet with ``srv_slo_itl``, ``srv_slo_ttft`` and
        ``srv_slo_tps`` = row ``l``, and winner block ``l`` is ``solve``'s winners for it in unlimited mode; each
        distinct target of a server is searched once (see ``wva_slo_grid`` in include/wva_b200.h).  The fleet's own
        ``srv_slo_*`` are not read.  ``out``: an ``Allocs`` of ``L * S`` records to write the winners into."""
        names = ("slo_itl", "slo_ttft", "slo_tps")
        rows, L = _row_lists(fleet, dict(zip(names, (slo_itl, slo_ttft, slo_tps))))
        if len(rows) != len(names):
            raise ValueError("slo_itl, slo_ttft and slo_tps are required")
        return self._level_call(self._L.wva_slo_grid, fleet, L, [_abi.ptr(rows[k].reshape(-1)) for k in names],
                                want_candidates, out)

    def workload_grid(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None,
                      want_candidates: bool = False, out: Allocs | None = None):
        """The reference's ``Server.Calculate`` and ``SolveUnlimited`` winner at each row of (``arrival_rpm``
        req/min, ``in_tokens``, ``out_tokens``), each of shape (L, S) -> (candidates [L*S*A] | None,
        winners [L*S]), both level-major.

        Candidate block ``l`` is what ``analyze`` returns for the fleet with ``srv_arrival_rpm``,
        ``srv_in_tokens`` and ``srv_out_tokens`` = row ``l``, and winner block ``l`` is ``solve``'s winners for
        it in unlimited mode; each distinct (server, in, out) is sized once (see ``wva_workload_grid`` in
        include/wva_b200.h).  A token list of ``None`` is the fleet's own column at every level.  ``out``: an
        ``Allocs`` of ``L * S`` records to write the winners into."""
        return self._workload_rows(self._L.wva_workload_grid, fleet, arrival_rpm, in_tokens, out_tokens,
                                   want_candidates, out)

    def workload_trace(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None,
                       want_candidates: bool = False, out: Allocs | None = None):
        """The reference's reconcile replayed over the ticks of (``arrival_rpm`` req/min, ``in_tokens``,
        ``out_tokens``), each of shape (L, S): ``Server.Calculate``, ``SolveUnlimited`` and
        ``Server.ApplyDesiredAlloc`` per tick -> (candidates [L*S*A] | None, winners [L*S]), both tick-major.

        Tick ``t`` is ``workload_grid``'s level ``t`` on the fleet whose current allocation is the previous tick's
        feasible winner (the fleet's own ``srv_cur_*`` at tick 0, and unchanged after a nil winner), i.e. ``solve``
        on ``fleet.apply_winners`` of every earlier tick in turn (see ``wva_workload_trace`` in include/wva_b200.h).
        A token list of ``None`` is the fleet's own column at every tick.  ``out``: an ``Allocs`` of ``L * S``
        records to write the winners into."""
        return self._workload_rows(self._L.wva_workload_trace, fleet, arrival_rpm, in_tokens, out_tokens,
                                   want_candidates, out)

    def _workload_rows(self, call, fleet, arrival_rpm, in_tokens, out_tokens, want_candidates, out):
        """wva_workload_grid / wva_workload_trace over (L, S) rows; a token list of None is the fleet's own."""
        S = fleet.n_servers
        rows, L = _row_lists(fleet, {"arrival_rpm": arrival_rpm, "in_tokens": in_tokens, "out_tokens": out_tokens})
        if "arrival_rpm" not in rows:
            raise ValueError("arrival_rpm is required")
        for name, own in (("in_tokens", fleet.srv_in_tokens), ("out_tokens", fleet.srv_out_tokens)):
            if name not in rows:
                rows[name] = np.ascontiguousarray(np.broadcast_to(own, (L, S)), np.int32)
        return self._level_call(call, fleet, L,
                                [_abi.ptr(rows[k].reshape(-1)) for k in ("arrival_rpm", "in_tokens", "out_tokens")],
                                want_candidates, out)

    def _level_call(self, call, fleet, L, row_ptrs, want_candidates, out):
        """call(handle, fleet, L, *row_ptrs, candidates, winners) for an L-row call -> (candidates [L*S*A] | None,
        winners [L*S]); the winners go into ``out`` when given."""
        if out is not None and out.n != L * fleet.n_servers:
            raise ValueError("out must hold L * fleet.n_servers records")
        win = out if out is not None else Allocs(L * fleet.n_servers)
        cand = Allocs(L * fleet.n_servers * fleet.n_acc) if want_candidates else None
        fc, wc = fleet.as_c(), win.as_c()
        cc = cand.as_c() if cand is not None else None
        self._resident(fleet)
        self._check(call(self._h, C.byref(fc), L, *row_ptrs, C.byref(cc) if cc is not None else None, C.byref(wc)))
        return cand, win

    def profile_grid(self, fleet: Fleet, *, acc_cost=None, perf_present=None, perf_alpha=None, perf_beta=None,
                     perf_gamma=None, perf_delta=None, perf_acc_count=None, perf_max_batch=None, perf_at_tokens=None,
                     want_candidates: bool = False, out: Allocs | None = None):
        """The reference's ``Server.Calculate`` and ``SolveUnlimited`` winner at each row of accelerator costs
        (``acc_cost``, shape (L, A)) and performance profiles (``perf_*``, shape (L, M, A)) -> (candidates
        [L*S*A] | None, winners [L*S]), both level-major.

        Candidate block ``l`` is what ``analyze`` returns for the fleet with ``acc_cost`` and the ``perf_*`` columns
        = row ``l``, and winner block ``l`` is ``solve``'s winners for it in unlimited mode; each distinct (server,
        accelerator, alpha, beta, gamma, delta, batch size) is sized once (see ``wva_profile_grid`` in
        include/wva_b200.h).  A column of ``None`` is the fleet's own at every level; at least one must be given,
        and L is their row count.  ``srv_cur_cost`` is not re-priced.  ``out``: an ``Allocs`` of ``L * S`` records
        to write the winners into."""
        rows, L = _row_lists(fleet, {"acc_cost": acc_cost, "perf_present": perf_present, "perf_alpha": perf_alpha,
                                     "perf_beta": perf_beta, "perf_gamma": perf_gamma, "perf_delta": perf_delta,
                                     "perf_acc_count": perf_acc_count, "perf_max_batch": perf_max_batch,
                                     "perf_at_tokens": perf_at_tokens})
        if L is None:
            raise ValueError("profile_grid needs at least one row list")
        rc_ = _profile_rows_c(rows)
        return self._level_call(self._L.wva_profile_grid, fleet, L, [C.byref(rc_)], want_candidates, out)

    def profile_trace(self, fleet: Fleet, arrival_rpm=None, in_tokens=None, out_tokens=None, *, acc_cost=None,
                      perf_present=None, perf_alpha=None, perf_beta=None, perf_gamma=None, perf_delta=None,
                      perf_acc_count=None, perf_max_batch=None, perf_at_tokens=None, want_candidates: bool = False,
                      out: Allocs | None = None):
        """The reference's reconcile replayed over ticks of load (``arrival_rpm`` req/min, ``in_tokens``,
        ``out_tokens``, shape (L, S)), accelerator costs (``acc_cost``, shape (L, A)) and performance profiles
        (``perf_*``, shape (L, M, A)): ``Server.Calculate``, ``SolveUnlimited`` and ``Server.ApplyDesiredAlloc`` per
        tick -> (candidates [L*S*A] | None, winners [L*S]), both tick-major.

        Tick ``t`` is ``solve`` in unlimited mode on the fleet with every given column = row ``t`` and the current
        allocation advanced by ``fleet.apply_winners`` through ticks 0..t-1; the fleet's own ``srv_cur_cost`` is
        not re-priced (see ``wva_profile_trace`` in include/wva_b200.h).  A list of ``None`` is the fleet's own
        column at every tick; at least one must be given, and L is their common row count.  ``out``: an ``Allocs``
        of ``L * S`` records to write the winners into."""
        load = {"arrival_rpm": arrival_rpm, "in_tokens": in_tokens, "out_tokens": out_tokens}
        rows, L = _row_lists(fleet, {**load, "acc_cost": acc_cost, "perf_present": perf_present,
                                     "perf_alpha": perf_alpha, "perf_beta": perf_beta, "perf_gamma": perf_gamma,
                                     "perf_delta": perf_delta, "perf_acc_count": perf_acc_count,
                                     "perf_max_batch": perf_max_batch, "perf_at_tokens": perf_at_tokens})
        if L is None:
            raise ValueError("profile_trace needs at least one row list")
        rc_ = _profile_rows_c(rows)
        row_ptrs = [_abi.ptr(rows[k].reshape(-1)) if k in rows else None for k in load] + [C.byref(rc_)]
        return self._level_call(self._L.wva_profile_trace, fleet, L, row_ptrs, want_candidates, out)

    def slo_trace(self, fleet: Fleet, arrival_rpm=None, in_tokens=None, out_tokens=None, *, slo_itl=None,
                  slo_ttft=None, slo_tps=None, want_candidates: bool = False, out: Allocs | None = None):
        """The reference's reconcile replayed over ticks of load (``arrival_rpm`` req/min, ``in_tokens``,
        ``out_tokens``) and service-class targets (``slo_itl``, ``slo_ttft``, ``slo_tps``, in the fleet columns'
        units), each of shape (L, S): ``Server.Calculate``, ``SolveUnlimited`` and ``Server.ApplyDesiredAlloc`` per
        tick -> (candidates [L*S*A] | None, winners [L*S]), both tick-major.

        Tick ``t`` is ``solve`` in unlimited mode on the fleet with every given column = row ``t`` and the current
        allocation advanced by ``fleet.apply_winners`` through ticks 0..t-1; each distinct (server, tokens, search,
        target) is searched once (see ``wva_slo_trace`` in include/wva_b200.h).  A list of ``None`` is the fleet's
        own column at every tick; at least one must be given, and L is their common row count.  ``out``: an
        ``Allocs`` of ``L * S`` records to write the winners into."""
        names = ("arrival_rpm", "in_tokens", "out_tokens", "slo_itl", "slo_ttft", "slo_tps")
        rows, L = _row_lists(fleet, dict(zip(names, (arrival_rpm, in_tokens, out_tokens, slo_itl, slo_ttft,
                                                     slo_tps))))
        if L is None:
            raise ValueError("slo_trace needs at least one row list")
        row_ptrs = [_abi.ptr(rows[k].reshape(-1)) if k in rows else None for k in names]
        return self._level_call(self._L.wva_slo_trace, fleet, L, row_ptrs, want_candidates, out)

    def load_intervals(self, fleet: Fleet, rpm_lo, rpm_hi, max_per_server: int):
        """Where each server's ``load_grid`` winner changes its decision in ``[rpm_lo[s], rpm_hi[s]]`` (req/min)
        -> (count [S], truncated [S], start_rpm (S, M), records: ``Allocs`` of S * M).

        Interval ``j`` of server ``s`` starts at ``start_rpm[s, j]`` and ends where interval ``j + 1`` starts;
        record ``s * M + j`` is ``load_grid``'s winner for ``s`` at that rate.  ``truncated[s]`` is 1 when the
        decision changes again before ``rpm_hi[s]`` (see ``wva_load_intervals`` in include/wva_b200.h);
        ``fleet.srv_arrival_rpm`` is not read."""
        S, M = fleet.n_servers, int(max_per_server)
        lo = np.ascontiguousarray(rpm_lo, np.float32)
        hi = np.ascontiguousarray(rpm_hi, np.float32)
        for name, col in (("rpm_lo", lo), ("rpm_hi", hi)):
            if col.shape != (S,):
                raise ValueError(f"{name} must have shape ({S},), got {col.shape}")
        if M < 1:
            raise ValueError("max_per_server must be at least 1")
        count = np.zeros(S, np.int32)
        truncated = np.zeros(S, np.uint8)
        start = np.zeros((S, M), np.float32)
        rec = Allocs(S * M)
        oc = _abi.IntervalsC(M, _abi.ptr(count), _abi.ptr(truncated), _abi.ptr(start.reshape(-1)), rec.as_c())
        fc = fleet.as_c()
        self._resident(fleet)
        self._check(self._L.wva_load_intervals(self._h, C.byref(fc), _abi.ptr(lo), _abi.ptr(hi), C.byref(oc)))
        return count, truncated, start, rec

    def load_margins(self, fleet: Fleet, arrival_rpm=None, rpm_lo=None, rpm_hi=None):
        """The stretch of arrival rates around each level's rate on which ``load_grid``'s winner keeps its decision
        -> (lo (L, S), hi (L, S), flags (L, S), at, below, above), the records ``Allocs`` of L * S.

        Level ``l`` is ``load_grid``'s row ``l`` of ``arrival_rpm`` (shape (L, S), req/min; ``None``: one level at
        the fleet's own load).  ``[lo[l, s], hi[l, s])`` is the largest float32 stretch inside the window
        ``[rpm_lo, rpm_hi]`` (shape (L, S); by default ``[0, 2 * rate]``) that holds the rate and on which the
        winner's decision key does not change; ``at``, ``below`` and ``above`` are ``load_grid``'s winners at the
        rate, one float32 below ``lo`` and at ``hi``.  ``flags`` holds ``MARGIN_LO_OPEN`` (no change down to
        ``rpm_lo``), ``MARGIN_HI_OPEN`` (none up to ``rpm_hi``, ``hi`` = +Inf) and ``MARGIN_TRUNCATED`` (see
        ``wva_load_margins`` in include/wva_b200.h).  ``within_margins`` tests new rates against the result."""
        return self._margins(self._L.wva_load_margins, fleet, arrival_rpm, rpm_lo, rpm_hi)

    def load_margin_trace(self, fleet: Fleet, arrival_rpm, rpm_lo=None, rpm_hi=None):
        """``load_margins`` at every tick of ``workload_trace`` over the rates ``arrival_rpm`` (shape (L, S),
        req/min, required; the tokens are the fleet's own) -> the same tuple as ``load_margins``.

        Block ``t`` is ``load_margins`` with one level (row ``t`` of the rates and of the windows, by default
        ``[0, 2 * rate]``) on the fleet whose current allocation is the one the trace carries into tick ``t``
        (``fleet.apply_winners`` of every earlier tick's ``at`` in turn): the load moves at tick ``t`` only.  The
        ``at`` records are ``workload_trace``'s winners (see ``wva_load_margin_trace`` in include/wva_b200.h).
        ``within_margins`` tests new rates against the result as it does for ``load_margins``."""
        if arrival_rpm is None:
            raise ValueError("arrival_rpm is required")
        return self._margins(self._L.wva_load_margin_trace, fleet, arrival_rpm, rpm_lo, rpm_hi)

    def workload_margins(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None, rpm_lo=None,
                         rpm_hi=None):
        """``load_margins`` at rows that carry their own tokens: level ``l`` is ``workload_grid``'s row ``l`` of
        (``arrival_rpm`` req/min, required; ``in_tokens``, ``out_tokens``), each of shape (L, S) -> the same tuple as
        ``load_margins``.  A token list of ``None`` is the fleet's own column at every level.

        Block ``l`` is ``load_margins`` with one level (row ``l`` of the rates and of the windows, by default
        ``[0, 2 * rate]``) on the fleet with ``srv_in_tokens`` and ``srv_out_tokens`` = row ``l``, and the ``at``
        records are ``workload_grid``'s winners; each distinct (server, in, out) under a window top above 0 is sized
        once (see ``wva_workload_margins`` in include/wva_b200.h).  A new rate inside ``[lo, hi)`` keeps the row's
        decision when the new tokens equal the row's: ``within_margins`` tests the rate only."""
        if arrival_rpm is None:
            raise ValueError("arrival_rpm is required")
        return self._margins(self._L.wva_workload_margins, fleet, arrival_rpm, rpm_lo, rpm_hi, in_tokens, out_tokens)

    def workload_margin_trace(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None, rpm_lo=None,
                              rpm_hi=None):
        """``workload_margins`` at every tick of ``workload_trace`` over the same (rate, in, out) rows -> the same
        tuple as ``load_margins``.

        Block ``t`` is ``workload_margins`` with one level on the fleet whose current allocation is the one the trace
        carries into tick ``t`` (``fleet.apply_winners`` of every earlier tick's ``at`` in turn), and the ``at``
        records are ``workload_trace``'s winners (see ``wva_workload_margin_trace`` in include/wva_b200.h).  A new
        rate inside ``[lo, hi)`` keeps tick ``t``'s decision when the new tokens equal the row's."""
        if arrival_rpm is None:
            raise ValueError("arrival_rpm is required")
        return self._margins(self._L.wva_workload_margin_trace, fleet, arrival_rpm, rpm_lo, rpm_hi, in_tokens,
                             out_tokens)

    def profile_margins(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None, rpm_lo=None, rpm_hi=None,
                        *, acc_cost=None, perf_present=None, perf_alpha=None, perf_beta=None, perf_gamma=None,
                        perf_delta=None, perf_acc_count=None, perf_max_batch=None, perf_at_tokens=None):
        """``workload_margins`` at rows that also carry their own accelerator costs (``acc_cost``, shape (L, A)) and
        performance profiles (``perf_*``, shape (L, M, A)), as ``profile_trace`` takes them -> the same tuple as
        ``load_margins``.  A list of ``None`` is the fleet's own column at every level.

        Block ``l`` is ``load_margins`` with one level (row ``l`` of the rates and of the windows, by default
        ``[0, 2 * rate]``) on the fleet with every given column = row ``l``, and the ``at`` records are
        ``profile_trace``'s winner for each row alone; each distinct (server, accelerator, in, out, alpha .. delta,
        batch size) under a window top above 0 is sized once (see ``wva_profile_margins`` in include/wva_b200.h).
        ``srv_cur_cost`` is not re-priced.  A new rate inside ``[lo, hi)`` keeps the row's decision when the tokens,
        prices and profiles stay the row's."""
        if arrival_rpm is None:
            raise ValueError("arrival_rpm is required")
        profile = dict(zip(_PROFILE_COLUMNS, (acc_cost, perf_present, perf_alpha, perf_beta, perf_gamma, perf_delta,
                                              perf_acc_count, perf_max_batch, perf_at_tokens)))
        return self._margins(self._L.wva_profile_margins, fleet, arrival_rpm, rpm_lo, rpm_hi, in_tokens, out_tokens,
                             profile=profile)

    def profile_margin_trace(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None, rpm_lo=None,
                             rpm_hi=None, *, acc_cost=None, perf_present=None, perf_alpha=None, perf_beta=None,
                             perf_gamma=None, perf_delta=None, perf_acc_count=None, perf_max_batch=None,
                             perf_at_tokens=None):
        """``profile_margins`` at every tick of ``profile_trace`` over the same rows -> the same tuple as
        ``load_margins``.

        Block ``t`` is ``profile_margins`` with one level on the fleet whose current allocation is the one the trace
        carries into tick ``t`` (``fleet.apply_winners`` of every earlier tick's ``at`` in turn, each cost at its own
        tick's prices), and the ``at`` records are ``profile_trace``'s winners (see ``wva_profile_margin_trace`` in
        include/wva_b200.h)."""
        if arrival_rpm is None:
            raise ValueError("arrival_rpm is required")
        profile = dict(zip(_PROFILE_COLUMNS, (acc_cost, perf_present, perf_alpha, perf_beta, perf_gamma, perf_delta,
                                              perf_acc_count, perf_max_batch, perf_at_tokens)))
        return self._margins(self._L.wva_profile_margin_trace, fleet, arrival_rpm, rpm_lo, rpm_hi, in_tokens,
                             out_tokens, profile=profile)

    def slo_margins(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None, rpm_lo=None, rpm_hi=None, *,
                    slo_itl=None, slo_ttft=None, slo_tps=None):
        """``workload_margins`` at rows that also carry their own service-class targets (``slo_itl``, ``slo_ttft``,
        ``slo_tps``, shape (L, S), in the fleet columns' units), as ``slo_trace`` takes them -> the same tuple as
        ``load_margins``.  A list of ``None`` is the fleet's own column at every level.

        Block ``l`` is ``load_margins`` with one level (row ``l`` of the rates and of the windows, by default
        ``[0, 2 * rate]``) on the fleet with every given column = row ``l``, and the ``at`` records are
        ``slo_trace``'s winner for each row alone; each distinct (server, in, out, ITL, TTFT, TPS) under a window top
        above 0 is sized once (see ``wva_slo_margins`` in include/wva_b200.h).  A new rate inside ``[lo, hi)`` keeps
        the row's decision when the tokens and targets stay the row's."""
        if arrival_rpm is None:
            raise ValueError("arrival_rpm is required")
        return self._margins(self._L.wva_slo_margins, fleet, arrival_rpm, rpm_lo, rpm_hi, in_tokens, out_tokens,
                             slo={"slo_itl": slo_itl, "slo_ttft": slo_ttft, "slo_tps": slo_tps})

    def slo_margin_trace(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None, rpm_lo=None, rpm_hi=None,
                         *, slo_itl=None, slo_ttft=None, slo_tps=None):
        """``slo_margins`` at every tick of ``slo_trace`` over the same rows -> the same tuple as ``load_margins``.

        Block ``t`` is ``slo_margins`` with one level on the fleet whose current allocation is the one the trace
        carries into tick ``t`` (``fleet.apply_winners`` of every earlier tick's ``at`` in turn), and the ``at``
        records are ``slo_trace``'s winners (see ``wva_slo_margin_trace`` in include/wva_b200.h)."""
        if arrival_rpm is None:
            raise ValueError("arrival_rpm is required")
        return self._margins(self._L.wva_slo_margin_trace, fleet, arrival_rpm, rpm_lo, rpm_hi, in_tokens, out_tokens,
                             slo={"slo_itl": slo_itl, "slo_ttft": slo_ttft, "slo_tps": slo_tps})

    def _margins(self, call, fleet, arrival_rpm, rpm_lo, rpm_hi, *tokens, profile=None, slo=None):
        """wva_load_margins / wva_load_margin_trace over (L, S) rows and windows, or with `tokens` (in_tokens,
        out_tokens; None: the fleet's own) wva_workload_margins / wva_workload_margin_trace, and with `profile` as
        well ({column: rows or None}) wva_profile_margins / wva_profile_margin_trace, or with `slo` ({target: rows
        or None}) wva_slo_margins / wva_slo_margin_trace; the output arrays."""
        S = fleet.n_servers
        rows, L = _row_lists(fleet, {"arrival_rpm": arrival_rpm, "rpm_lo": rpm_lo, "rpm_hi": rpm_hi,
                                     **dict(zip(("in_tokens", "out_tokens"), tokens)), **(profile or {}),
                                     **(slo or {})})
        L = 1 if L is None else L
        rate = rows.get("arrival_rpm", np.ascontiguousarray(np.broadcast_to(fleet.srv_arrival_rpm, (L, S)), np.float32))
        lo = rows.get("rpm_lo", np.zeros((L, S), np.float32))
        hi = rows.get("rpm_hi", (rate * np.float32(2)).astype(np.float32))
        lo_out, hi_out = np.zeros((L, S), np.float32), np.zeros((L, S), np.float32)
        flags = np.zeros((L, S), np.uint8)
        at, below, above = Allocs(L * S), Allocs(L * S), Allocs(L * S)
        oc = _abi.MarginsC(_abi.ptr(lo_out.reshape(-1)), _abi.ptr(hi_out.reshape(-1)), _abi.ptr(flags.reshape(-1)),
                           at.as_c(), below.as_c(), above.as_c())
        fc = fleet.as_c()
        self._resident(fleet)
        token_rows = [_abi.ptr(rows[k].reshape(-1)) if k in rows else None
                      for k in ("in_tokens", "out_tokens")[:len(tokens)]]
        if profile is not None:
            rc_ = _profile_rows_c(rows)
            token_rows.append(C.byref(rc_))
        if slo is not None:
            token_rows += [_abi.ptr(rows[k].reshape(-1)) if k in rows else None for k in slo]
        self._check(call(self._h, C.byref(fc), L, _abi.ptr(rate.reshape(-1)), *token_rows, _abi.ptr(lo.reshape(-1)),
                         _abi.ptr(hi.reshape(-1)), C.byref(oc)))
        return lo_out, hi_out, flags, at, below, above

    def price_thresholds(self, fleet: Fleet, want_candidates: bool = False):
        """The exact price of each accelerator at which each server's unlimited winner leaves it -> (threshold
        (S, A) float32, above: ``Allocs`` of S * A, candidates [S*A] | None).

        ``threshold[s, a]`` is the smallest float32 price ``p`` in [+0, MaxFloat32] at which ``solve``'s winner for
        ``s`` on the fleet with ``acc_cost[a] = p`` is not ``a``'s candidate (+Inf when it is at every price; 0 when
        it never is).  Record ``s * A + a`` of ``above`` is ``profile_grid``'s winner for ``s`` at that price (zero
        bytes where the threshold is +Inf), and ``candidates`` is what ``analyze`` returns.  ``srv_cur_cost`` is not
        re-priced; ``fleet.unlimited`` and the capacities are not read (see ``wva_price_thresholds`` in
        include/wva_b200.h).  ``accelerator_demand`` turns a column into a demand curve."""
        S, A = fleet.n_servers, fleet.n_acc
        threshold = np.zeros((S, A), np.float32)
        above = Allocs(S * A)
        cand = Allocs(S * A) if want_candidates else None
        fc, ac = fleet.as_c(), above.as_c()
        cc = cand.as_c() if cand is not None else None
        self._resident(fleet)
        self._check(self._L.wva_price_thresholds(self._h, C.byref(fc), _abi.ptr(threshold.reshape(-1)), C.byref(ac),
                                                 C.byref(cc) if cc is not None else None))
        return threshold, above, cand

    def price_threshold_grid(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None,
                             want_candidates: bool = False):
        """``price_thresholds`` at every row of (``arrival_rpm`` req/min, ``in_tokens``, ``out_tokens``), each of
        shape (L, S) -> (threshold (L, S, A) float32, above: ``Allocs`` of L * S * A, candidates [L*S*A] | None,
        winners [L*S]).

        Block ``l`` of threshold, above and candidates is ``price_thresholds`` on the fleet with row ``l``, and
        winner block ``l`` is ``workload_grid``'s (see ``wva_price_threshold_grid`` in include/wva_b200.h).  A token
        list of ``None`` is the fleet's own column at every level.  ``demand_by_level`` turns a column into demand
        curves."""
        return self._price_rows(self._L.wva_price_threshold_grid, fleet, arrival_rpm, in_tokens, out_tokens,
                                want_candidates)

    def price_threshold_trace(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None,
                              want_candidates: bool = False):
        """``price_thresholds`` at every tick of ``workload_trace`` -> (threshold (L, S, A) float32, above:
        ``Allocs`` of L * S * A, candidates [L*S*A] | None, winners [L*S]).

        Block ``t`` is ``price_thresholds`` on the fleet with row ``t`` and the current allocation the trace carries
        into tick ``t`` (``fleet.apply_winners`` of every earlier tick in turn): the price changes at tick ``t``
        only.  Winners are ``workload_trace``'s (see ``wva_price_threshold_trace`` in include/wva_b200.h)."""
        return self._price_rows(self._L.wva_price_threshold_trace, fleet, arrival_rpm, in_tokens, out_tokens,
                                want_candidates)

    def profile_price_threshold_grid(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None, *,
                                     acc_cost=None, perf_present=None, perf_alpha=None, perf_beta=None,
                                     perf_gamma=None, perf_delta=None, perf_acc_count=None, perf_max_batch=None,
                                     perf_at_tokens=None, want_candidates: bool = False):
        """``price_threshold_grid`` at rows that also carry their own accelerator costs (``acc_cost``, shape (L, A))
        and performance profiles (``perf_*``, shape (L, M, A)), as ``profile_trace`` takes them -> (threshold (L, S,
        A) float32, above: ``Allocs`` of L * S * A, candidates [L*S*A] | None, winners [L*S]).

        Block ``l`` of threshold, above and candidates is ``price_thresholds`` on the fleet with every given column
        = row ``l``, and winner block ``l`` is ``solve``'s in unlimited mode on that fleet.  Column ``a`` of block
        ``l`` does not read row ``l``'s ``acc_cost[a]``.  A list of ``None`` is the fleet's own column at every
        level; ``srv_cur_cost`` is not re-priced (see ``wva_profile_price_threshold_grid`` in include/wva_b200.h).
        ``demand_by_level`` with ``perf_acc_count`` turns a column into demand curves."""
        profile = dict(zip(_PROFILE_COLUMNS, (acc_cost, perf_present, perf_alpha, perf_beta, perf_gamma, perf_delta,
                                              perf_acc_count, perf_max_batch, perf_at_tokens)))
        return self._price_rows(self._L.wva_profile_price_threshold_grid, fleet, arrival_rpm, in_tokens, out_tokens,
                                want_candidates, profile)

    def profile_price_threshold_trace(self, fleet: Fleet, arrival_rpm, in_tokens=None, out_tokens=None, *,
                                      acc_cost=None, perf_present=None, perf_alpha=None, perf_beta=None,
                                      perf_gamma=None, perf_delta=None, perf_acc_count=None, perf_max_batch=None,
                                      perf_at_tokens=None, want_candidates: bool = False):
        """``price_thresholds`` at every tick of ``profile_trace`` over the same rows -> the same tuple as
        ``profile_price_threshold_grid``.

        Block ``t`` is ``price_thresholds`` on the fleet with every given column = row ``t`` and the current
        allocation the trace carries into tick ``t`` (``fleet.apply_winners`` of every earlier tick in turn, each
        cost at its own tick's prices), and winners and candidates are ``profile_trace``'s (see
        ``wva_profile_price_threshold_trace`` in include/wva_b200.h)."""
        profile = dict(zip(_PROFILE_COLUMNS, (acc_cost, perf_present, perf_alpha, perf_beta, perf_gamma, perf_delta,
                                              perf_acc_count, perf_max_batch, perf_at_tokens)))
        return self._price_rows(self._L.wva_profile_price_threshold_trace, fleet, arrival_rpm, in_tokens, out_tokens,
                                want_candidates, profile)

    def _price_rows(self, call, fleet, arrival_rpm, in_tokens, out_tokens, want_candidates, profile=None):
        """wva_price_threshold_grid / _trace over (L, S) rows, or with `profile` ({column: rows or None})
        wva_profile_price_threshold_grid / _trace; the output arrays."""
        S, A = fleet.n_servers, fleet.n_acc
        rows, L = _row_lists(fleet, {"arrival_rpm": arrival_rpm, "in_tokens": in_tokens, "out_tokens": out_tokens,
                                     **(profile or {})})
        if "arrival_rpm" not in rows:
            raise ValueError("arrival_rpm is required")
        threshold = np.zeros((L, S, A), np.float32)
        above, win = Allocs(L * S * A), Allocs(L * S)
        cand = Allocs(L * S * A) if want_candidates else None
        fc, ac, wc = fleet.as_c(), above.as_c(), win.as_c()
        cc = cand.as_c() if cand is not None else None
        ptrs = [_abi.ptr(rows[k].reshape(-1)) if k in rows else None
                for k in ("arrival_rpm", "in_tokens", "out_tokens")]
        if profile is not None:
            rc_ = _profile_rows_c(rows)
            ptrs.append(C.byref(rc_))
        self._resident(fleet)
        self._check(call(self._h, C.byref(fc), L, *ptrs, _abi.ptr(threshold.reshape(-1)), C.byref(ac),
                         C.byref(cc) if cc is not None else None, C.byref(wc)))
        return threshold, above, cand, win

    def slo_bounds(self, fleet: Fleet):
        """Where each load pair's TTFT and ITL searches turn the candidate nil and stop binding -> (kind, y_lo, y_hi,
        b1, b2), each of shape (S, A, 2), index [s, a, w] with w = 0: TTFT, 1: ITL.

        ``kind`` (uint8): 0 the target is not read, 1 every positive target nil, 2 rising (stretches NIL,
        SEARCHED, FREE), 3 not rising (FREE, SEARCHED, NIL).  ``y_lo`` / ``y_hi`` are EvalTTFT / EvalITL at
        lambda_min / lambda_max.  A target ``t`` is in the first stretch when ``not t >= b1``, in the last when
        ``t >= b2``, else in the middle; NaN is past +Inf.  ``srv_slo_*``, ``fleet.unlimited`` and the capacities
        are not read (see ``wva_slo_bounds`` in include/wva_b200.h).  ``slo_envelope`` turns them into per-server
        statements."""
        S, A = fleet.n_servers, fleet.n_acc
        kind = np.zeros((S, A, 2), np.uint8)
        cols = [np.zeros((S, A, 2), np.float32) for _ in range(4)]
        oc = _abi.SloBoundsC(_abi.ptr(kind.reshape(-1)), *(_abi.ptr(c.reshape(-1)) for c in cols))
        fc = fleet.as_c()
        self._resident(fleet)
        self._check(self._L.wva_slo_bounds(self._h, C.byref(fc), C.byref(oc)))
        return (kind, *cols)

    def sweep(self, fleet: Fleet, n_rates: int) -> dict:
        n = fleet.n_servers * fleet.n_acc * n_rates
        out = {"valid": np.zeros(n, np.uint8)}
        for k in ("rate", "ttft", "itl", "throughput", "rho"):
            out[k] = np.zeros(n, np.float32)
        oc = _abi.SweepOutC(*[_abi.ptr(out[k]) for k in ("valid", "rate", "ttft", "itl", "throughput", "rho")])
        fc = fleet.as_c()
        self._resident(fleet)
        self._check(self._L.wva_sweep(self._h, C.byref(fc), n_rates, C.byref(oc)))
        return out

    # -- streaming reconcile ------------------------------------------------
    def _resident(self, fleet: Fleet):
        """Every call that takes a fleet makes it the handle's resident fleet (the C side re-uploads it);
        ``resolve`` / ``update_load`` size their buffers from these counts, not from an older upload."""
        self._n_servers, self._n_acc = fleet.n_servers, fleet.n_acc

    def upload(self, fleet: Fleet):
        fc = fleet.as_c()
        self._check(self._L.wva_upload(self._h, C.byref(fc)))
        self._resident(fleet)

    def update_load(self, arrival_rpm=None, in_tokens=None, out_tokens=None):
        if self._n_servers is None:
            raise WvaError(_abi.WVA_ERR_STATE, "no resident fleet (call upload or a solve first)")
        a = np.ascontiguousarray(arrival_rpm, np.float32) if arrival_rpm is not None else None
        i = np.ascontiguousarray(in_tokens, np.int32) if in_tokens is not None else None
        o = np.ascontiguousarray(out_tokens, np.int32) if out_tokens is not None else None
        for name, col in (("arrival_rpm", a), ("in_tokens", i), ("out_tokens", o)):
            if col is not None and col.shape != (self._n_servers,):  # the C side copies exactly S entries
                raise ValueError(f"{name} must have {self._n_servers} entries (one per resident server), "
                                 f"got shape {col.shape}")
        self._check(self._L.wva_update_load(self._h, _abi.ptr(a) if a is not None else None,
                                            _abi.ptr(i) if i is not None else None,
                                            _abi.ptr(o) if o is not None else None))

    def resolve(self, want_candidates: bool = False):
        if self._n_servers is None:
            raise WvaError(_abi.WVA_ERR_STATE, "no resident fleet (call upload or a solve first)")
        cand = Allocs(self._n_servers * self._n_acc) if want_candidates else None
        win = Allocs(self._n_servers)
        wc = win.as_c()
        cc = cand.as_c() if cand is not None else None
        self._check(self._L.wva_resolve(self._h, C.byref(cc) if cc is not None else None, C.byref(wc)))
        return cand, win

    def summarize(self, n_types: int) -> dict:
        """``System.AllocateByType`` (pkg/core/system.go:271-300) and ``CreateAllocationDiff`` per server
        (pkg/core/allocation.go:353-380) over the most recent solution of this engine.

        Returns ``{"by_type": {present,count,limit,cost} arrays [T], "diff": {old_acc,new_acc,old_replicas,
        new_replicas,cost} arrays [S]}``; accelerator ids use ``ACC_NONE`` for "" and ``ACC_ABSENT`` for
        "none"."""
        if self._n_servers is None:
            raise WvaError(_abi.WVA_ERR_STATE, "no resident fleet (solve first)")
        T, S = int(n_types), self._n_servers
        by_type = {"present": np.zeros(T, np.uint8), "count": np.zeros(T, np.int64), "limit": np.zeros(T, np.int32),
                   "cost": np.zeros(T, np.float32)}
        diff = {"old_acc": np.zeros(S, np.int32), "new_acc": np.zeros(S, np.int32),
                "old_replicas": np.zeros(S, np.int32), "new_replicas": np.zeros(S, np.int32),
                "cost": np.zeros(S, np.float32)}
        sc = _abi.SummaryC(_abi.ptr(by_type["present"]), _abi.ptr(by_type["count"]), _abi.ptr(by_type["limit"]),
                           _abi.ptr(by_type["cost"]), _abi.ptr(diff["old_acc"]), _abi.ptr(diff["new_acc"]),
                           _abi.ptr(diff["old_replicas"]), _abi.ptr(diff["new_replicas"]), _abi.ptr(diff["cost"]))
        self._check(self._L.wva_summarize(self._h, C.byref(sc)))
        return {"by_type": by_type, "diff": diff}

    def mm1k_solve(self, K, lam, mu) -> dict:
        """``MM1KModel.Solve`` (pkg/analyzer/mm1kmodel.go:19-92) for arrays of (K, lambda, mu) triples; returns the
        model statistics as numpy columns (``is_valid``, ``rho``, ``avg_num_in_system``, ``throughput``,
        ``avg_resp_time``, ``avg_serv_time``, ``avg_wait_time``, ``avg_queue_length``, ``sum_p``)."""
        K = np.ascontiguousarray(K, np.int32)
        lam = np.ascontiguousarray(lam, np.float32)
        mu = np.ascontiguousarray(mu, np.float32)
        if not (K.shape == lam.shape == mu.shape and K.ndim == 1):
            raise ValueError("K, lam, mu must be 1-D arrays of one length")
        n = K.size
        out = {"is_valid": np.zeros(n, np.uint8)}
        names = ("rho", "avg_num_in_system", "throughput", "avg_resp_time", "avg_serv_time", "avg_wait_time",
                 "avg_queue_length")
        for name in names:
            out[name] = np.zeros(n, np.float32)
        out["sum_p"] = np.zeros(n, np.float64)
        oc = _abi.Mm1kOutC(_abi.ptr(out["is_valid"]), *[_abi.ptr(out[name]) for name in names], _abi.ptr(out["sum_p"]))
        self._check(self._L.wva_mm1k_solve(self._h, n, _abi.ptr(K), _abi.ptr(lam), _abi.ptr(mu), C.byref(oc)))
        return out

    # -- device-resident variants (multi-GPU driver, bench) -------------------
    def grid_solve_device(self, grid: Grid, winners_dev: _abi.AllocsC):
        gc = grid.as_c()
        self._check(self._L.wva_grid_solve_device(self._h, C.byref(gc), C.byref(winners_dev)))

    def resolve_device(self, winners_dev: _abi.AllocsC):
        self._check(self._L.wva_resolve_device(self._h, C.byref(winners_dev)))

    def synchronize(self):
        self._check(self._L.wva_synchronize(self._h))

    @property
    def stream(self) -> int:
        return int(self._L.wva_stream(self._h) or 0)

    @property
    def launch_count(self) -> int:
        return int(self._L.wva_launch_count(self._h))

    @property
    def last_kernel_ms(self) -> float:
        return float(self._L.wva_last_kernel_ms(self._h))

    @property
    def last_device_ms(self) -> float:
        return float(self._L.wva_last_device_ms(self._h))
