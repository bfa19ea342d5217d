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


# the fleet column each load row list replaces (every other row list is named after its column)
_ROW_COLUMN = {"arrival_rpm": "srv_arrival_rpm", "in_tokens": "srv_in_tokens", "out_tokens": "srv_out_tokens"}
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
        rpm = np.ascontiguousarray(arrival_rpm, np.float32)
        if rpm.ndim != 2 or rpm.shape[1] != fleet.n_servers:
            raise ValueError(f"arrival_rpm must have shape (L, {fleet.n_servers}), got {rpm.shape}")
        L = rpm.shape[0]
        if out is not None and out.n != L * fleet.n_servers:
            raise ValueError("out must hold L * fleet.n_servers records")
        win = out if out is not None else Allocs(L * fleet.n_servers)
        cand = Allocs(L * fleet.n_servers * fleet.n_acc) if want_candidates else None
        fc, wc = fleet.as_c(), win.as_c()
        cc = cand.as_c() if cand is not None else None
        self._resident(fleet)
        self._check(self._L.wva_load_grid(self._h, C.byref(fc), L, _abi.ptr(rpm.reshape(-1)),
                                          C.byref(cc) if cc is not None else None, C.byref(wc)))
        return cand, win

    def slo_grid(self, fleet: Fleet, slo_itl, slo_ttft, slo_tps, want_candidates: bool = False,
                 out: Allocs | None = None):
        """The reference's ``Server.Calculate`` and ``SolveUnlimited`` winner at each row of service-class targets
        (``slo_itl``, ``slo_ttft``, ``slo_tps``, each of shape (L, S), in the fleet columns' units) ->
        (candidates [L*S*A] | None, winners [L*S]), both level-major.

        Candidate block ``l`` is what ``analyze`` returns for the fleet with ``srv_slo_itl``, ``srv_slo_ttft`` and
        ``srv_slo_tps`` = row ``l``, and winner block ``l`` is ``solve``'s winners for it in unlimited mode; each
        distinct target of a server is searched once (see ``wva_slo_grid`` in include/wva_b200.h).  The fleet's own
        ``srv_slo_*`` are not read.  ``out``: an ``Allocs`` of ``L * S`` records to write the winners into."""
        rows = []
        for name, x in (("slo_itl", slo_itl), ("slo_ttft", slo_ttft), ("slo_tps", slo_tps)):
            r = np.ascontiguousarray(x, np.float32)
            if r.ndim != 2 or r.shape[1] != fleet.n_servers:
                raise ValueError(f"{name} must have shape (L, {fleet.n_servers}), got {r.shape}")
            rows.append(r)
        L = rows[0].shape[0]
        if any(r.shape[0] != L for r in rows):
            raise ValueError(f"slo_itl, slo_ttft and slo_tps must have one row count, got {[r.shape for r in rows]}")
        if out is not None and out.n != L * fleet.n_servers:
            raise ValueError("out must hold L * fleet.n_servers records")
        win = out if out is not None else Allocs(L * fleet.n_servers)
        cand = Allocs(L * fleet.n_servers * fleet.n_acc) if want_candidates else None
        fc, wc = fleet.as_c(), win.as_c()
        cc = cand.as_c() if cand is not None else None
        self._resident(fleet)
        self._check(self._L.wva_slo_grid(self._h, C.byref(fc), L, *[_abi.ptr(r.reshape(-1)) for r in rows],
                                         C.byref(cc) if cc is not None else None, C.byref(wc)))
        return cand, win

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
        win, cand = self._row_outputs(fleet, L, want_candidates, out)
        fc, wc = fleet.as_c(), win.as_c()
        cc = cand.as_c() if cand is not None else None
        self._resident(fleet)
        self._check(call(self._h, C.byref(fc), L,
                         *[_abi.ptr(rows[k].reshape(-1)) for k in ("arrival_rpm", "in_tokens", "out_tokens")],
                         C.byref(cc) if cc is not None else None, C.byref(wc)))
        return cand, win

    @staticmethod
    def _row_outputs(fleet, L, want_candidates, out):
        """The winners (``out``, or new) and candidates (or None) of an L-row call."""
        if out is not None and out.n != L * fleet.n_servers:
            raise ValueError("out must hold L * fleet.n_servers records")
        win = out if out is not None else Allocs(L * fleet.n_servers)
        cand = Allocs(L * fleet.n_servers * fleet.n_acc) if want_candidates else None
        return win, cand

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
        win, cand = self._row_outputs(fleet, L, want_candidates, out)
        rc_ = _profile_rows_c(rows)
        fc, wc = fleet.as_c(), win.as_c()
        cc = cand.as_c() if cand is not None else None
        self._resident(fleet)
        self._check(self._L.wva_profile_grid(self._h, C.byref(fc), L, C.byref(rc_),
                                             C.byref(cc) if cc is not None else None, C.byref(wc)))
        return cand, win

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
        win, cand = self._row_outputs(fleet, L, want_candidates, out)
        rc_ = _profile_rows_c(rows)
        fc, wc = fleet.as_c(), win.as_c()
        cc = cand.as_c() if cand is not None else None
        self._resident(fleet)
        self._check(self._L.wva_profile_trace(self._h, C.byref(fc), L,
                                              *[_abi.ptr(rows[k].reshape(-1)) if k in rows else None for k in load],
                                              C.byref(rc_), C.byref(cc) if cc is not None else None, C.byref(wc)))
        return cand, win

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
