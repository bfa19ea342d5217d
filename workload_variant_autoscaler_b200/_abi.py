"""ctypes image of include/wva_b200.h (struct layouts only; no library is loaded here).

Shared by the product loader (``_lib.py``) and by the test-only oracle loader
(``oracle/__init__.py``), which consumes the same flat SoA ``wva_fleet``.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

WVA_OK = 0
WVA_ERR_BAD_ARG = -1
WVA_ERR_NO_DEVICE = -2
WVA_ERR_CUDA = -3
WVA_ERR_NOMEM = -4
WVA_ERR_STATE = -5
WVA_ERR_UNSUPPORTED = -6

ACC_NONE = -1      # accelerator name "" (pkg/core/allocation.go:264)
ACC_UNKNOWN = -2   # a name missing from the accelerator table
ACC_ABSENT = -3    # no allocation at all: CreateAllocationDiff's "none" (pkg/core/allocation.go:357-358)

MARGIN_LO_OPEN, MARGIN_HI_OPEN, MARGIN_TRUNCATED = 1, 2, 4  # wva_margins.flags

SAT_NONE, SAT_PRIORITY_EXHAUSTIVE, SAT_PRIORITY_ROUND_ROBIN, SAT_ROUND_ROBIN = 0, 1, 2, 3
SAT_BY_NAME = {  # pkg/config/config.go:28-41
    "None": SAT_NONE,
    "PriorityExhaustive": SAT_PRIORITY_EXHAUSTIVE,
    "PriorityRoundRobin": SAT_PRIORITY_ROUND_ROBIN,
    "RoundRobin": SAT_ROUND_ROBIN,
}

f32p = C.POINTER(C.c_float)
i32p = C.POINTER(C.c_int32)
i64p = C.POINTER(C.c_int64)
f64p = C.POINTER(C.c_double)
u8p = C.POINTER(C.c_uint8)


class Tunables(C.Structure):
    _fields_ = [("max_queue_to_batch_ratio", C.c_int32), ("accel_penalty_factor", C.c_float)]


class FleetC(C.Structure):
    _fields_ = [
        ("n_acc", C.c_int32),
        ("acc_cost", f32p),
        ("acc_multiplicity", i32p),
        ("acc_type", i32p),
        ("n_types", C.c_int32),
        ("type_capacity", i32p),
        ("n_models", C.c_int32),
        ("perf_present", u8p),
        ("perf_alpha", f32p),
        ("perf_beta", f32p),
        ("perf_gamma", f32p),
        ("perf_delta", f32p),
        ("perf_acc_count", i32p),
        ("perf_max_batch", i32p),
        ("perf_at_tokens", i32p),
        ("n_servers", C.c_int32),
        ("srv_model", i32p),
        ("srv_priority", i32p),
        ("srv_has_target", u8p),
        ("srv_slo_itl", f32p),
        ("srv_slo_ttft", f32p),
        ("srv_slo_tps", f32p),
        ("srv_keep_acc", u8p),
        ("srv_min_replicas", i32p),
        ("srv_max_batch", i32p),
        ("srv_arrival_rpm", f32p),
        ("srv_in_tokens", i32p),
        ("srv_out_tokens", i32p),
        ("srv_cur_acc", i32p),
        ("srv_cur_replicas", i32p),
        ("srv_cur_cost", f32p),
        ("unlimited", C.c_uint8),
        ("delayed_best_effort", C.c_uint8),
        ("saturation_policy", C.c_int32),
        ("tun", Tunables),
    ]


class AllocsC(C.Structure):
    _fields_ = [
        ("feasible", u8p),
        ("acc", i32p),
        ("replicas", i32p),
        ("batch", i32p),
        ("cost", f32p),
        ("value", f32p),
        ("itl", f32p),
        ("ttft", f32p),
        ("rho", f32p),
        ("max_rate", f32p),
    ]


class IntervalsC(C.Structure):
    _fields_ = [("max_per_server", C.c_int32), ("count", i32p), ("truncated", u8p), ("start_rpm", f32p),
                ("rec", AllocsC)]


class MarginsC(C.Structure):
    _fields_ = [("lo_rpm", f32p), ("hi_rpm", f32p), ("flags", u8p), ("at", AllocsC), ("below", AllocsC),
                ("above", AllocsC)]


class SloBoundsC(C.Structure):
    _fields_ = [("kind", u8p), ("y_lo", f32p), ("y_hi", f32p), ("b1", f32p), ("b2", f32p)]


class ProfileRowsC(C.Structure):
    _fields_ = [("acc_cost", f32p), ("perf_present", u8p), ("perf_alpha", f32p), ("perf_beta", f32p),
                ("perf_gamma", f32p), ("perf_delta", f32p), ("perf_acc_count", i32p), ("perf_max_batch", i32p),
                ("perf_at_tokens", i32p)]


class GridC(C.Structure):
    _fields_ = [("n_batch", C.c_int32), ("batch", i32p), ("n_replicas", C.c_int32), ("replicas", i32p)]


class CellsC(C.Structure):
    _fields_ = [("flags", u8p), ("ttft", f32p), ("itl", f32p), ("rho", f32p), ("throughput", f32p)]


class SweepOutC(C.Structure):
    _fields_ = [("valid", u8p), ("rate", f32p), ("ttft", f32p), ("itl", f32p), ("throughput", f32p), ("rho", f32p)]


class SummaryC(C.Structure):
    _fields_ = [("type_present", u8p), ("type_count", i64p), ("type_limit", i32p), ("type_cost", f32p),
                ("diff_old_acc", i32p), ("diff_new_acc", i32p), ("diff_old_replicas", i32p),
                ("diff_new_replicas", i32p), ("diff_cost", f32p)]


class Mm1kOutC(C.Structure):
    _fields_ = [("is_valid", u8p), ("rho", f32p), ("avg_num_in_system", f32p), ("throughput", f32p),
                ("avg_resp_time", f32p), ("avg_serv_time", f32p), ("avg_wait_time", f32p),
                ("avg_queue_length", f32p), ("sum_p", f64p)]


_CT = {np.dtype(np.float32): C.c_float, np.dtype(np.int32): C.c_int32, np.dtype(np.uint8): C.c_uint8,
       np.dtype(np.int64): C.c_int64, np.dtype(np.float64): C.c_double}


def ptr(a: np.ndarray):
    """ctypes pointer to a C-contiguous numpy array of f32 / i32 / i64 / u8."""
    assert a.flags["C_CONTIGUOUS"], "array must be C-contiguous"
    return a.ctypes.data_as(C.POINTER(_CT[a.dtype]))


# The array columns of wva_fleet: (name, dtype, length).  The length is "A" (accelerators), "T" (accelerator
# types), "MA" (models x accelerators, a row-major [M, A] table) or "S" (servers).
FLEET_COLUMNS = (
    ("acc_cost", np.float32, "A"),
    ("acc_multiplicity", np.int32, "A"),
    ("acc_type", np.int32, "A"),
    ("type_capacity", np.int32, "T"),
    ("perf_present", np.uint8, "MA"),
    ("perf_alpha", np.float32, "MA"),
    ("perf_beta", np.float32, "MA"),
    ("perf_gamma", np.float32, "MA"),
    ("perf_delta", np.float32, "MA"),
    ("perf_acc_count", np.int32, "MA"),
    ("perf_max_batch", np.int32, "MA"),
    ("perf_at_tokens", np.int32, "MA"),
    ("srv_model", np.int32, "S"),
    ("srv_priority", np.int32, "S"),
    ("srv_has_target", np.uint8, "S"),
    ("srv_slo_itl", np.float32, "S"),
    ("srv_slo_ttft", np.float32, "S"),
    ("srv_slo_tps", np.float32, "S"),
    ("srv_keep_acc", np.uint8, "S"),
    ("srv_min_replicas", np.int32, "S"),
    ("srv_max_batch", np.int32, "S"),
    ("srv_arrival_rpm", np.float32, "S"),
    ("srv_in_tokens", np.int32, "S"),
    ("srv_out_tokens", np.int32, "S"),
    ("srv_cur_acc", np.int32, "S"),
    ("srv_cur_replicas", np.int32, "S"),
    ("srv_cur_cost", np.float32, "S"),
)

ALLOC_COLUMNS = (
    ("feasible", np.uint8),
    ("acc", np.int32),
    ("replicas", np.int32),
    ("batch", np.int32),
    ("cost", np.float32),
    ("value", np.float32),
    ("itl", np.float32),
    ("ttft", np.float32),
    ("rho", np.float32),
    ("max_rate", np.float32),
)


class Allocs:
    """Host SoA of core.Allocation records (pkg/core/allocation.go:13-24)."""

    def __init__(self, n: int):
        self.n = n
        for name, dt in ALLOC_COLUMNS:
            setattr(self, name, np.zeros(n, dtype=dt))

    def as_c(self) -> AllocsC:
        c = self.__dict__.get("_c")
        if c is None:  # the columns are never re-attached: one struct per object
            c = self.__dict__["_c"] = AllocsC(*[ptr(getattr(self, name)) for name, _ in ALLOC_COLUMNS])
        return c

    def record(self, i: int) -> dict:
        return {name: getattr(self, name)[i].item() for name, _ in ALLOC_COLUMNS}

    def columns(self) -> dict:
        return {name: getattr(self, name) for name, _ in ALLOC_COLUMNS}
