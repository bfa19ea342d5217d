"""Bit-exact comparison helpers and the ABI constants shared by the parity tests."""
import numpy as np

ALLOC_FIELDS = ("feasible", "acc", "replicas", "batch", "cost", "value", "itl", "ttft", "rho", "max_rate")
FLOAT_FIELDS = ("cost", "value", "itl", "ttft", "rho", "max_rate")
F32_MAX = np.float32(np.finfo(np.float32).max)
# include/wva_b200.h, written out so that the tests pin the values rather than read them from _abi
WVA_ERR_BAD_ARG, WVA_ERR_STATE, WVA_ERR_UNSUPPORTED = -1, -5, -6
ACC_NONE, ACC_UNKNOWN = -1, -2


def same_bytes(a, b):
    return np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


def f32_bits(x):
    """The bits of float32(x), any NaN as the quiet NaN."""
    v = np.float32(x)
    return 0x7FC00000 if np.isnan(v) else int(np.array([v]).view(np.uint32)[0])


def error_code(fn):
    """(0, fn()) or (the WvaError's code, None)."""
    from workload_variant_autoscaler_b200 import WvaError
    try:
        return 0, fn()
    except WvaError as e:
        return e.code, None


def bits(a):
    a = np.ascontiguousarray(a, np.float32)
    b = a.view(np.uint32).copy()
    b[np.isnan(a)] = 0x7FC00000  # any NaN == any NaN (payload is not part of the contract)
    return b


def assert_f32_bits_equal(got, want, what=""):
    gb, wb = bits(got), bits(want)
    bad = np.nonzero(gb != wb)[0]
    if bad.size:
        i = int(bad[0])
        raise AssertionError(f"{what}: {bad.size} of {gb.size} float32 values differ; first at {i}: "
                             f"got {np.float32(got[i])!r} ({gb[i]:#010x}) want {np.float32(want[i])!r} ({wb[i]:#010x})")


def assert_allocs_equal(got, want_struct, what=""):
    """got: product Allocs (SoA); want_struct: oracle structured array (flattened)."""
    want = want_struct.reshape(-1)
    assert got.n == want.size, (got.n, want.size)
    for f in ("feasible", "acc", "replicas", "batch"):
        g = np.asarray(getattr(got, f)).astype(np.int64)
        w = want[f].astype(np.int64)
        bad = np.nonzero(g != w)[0]
        if bad.size:
            i = int(bad[0])
            raise AssertionError(f"{what}: field {f}: {bad.size} of {g.size} differ; first at {i}: got {g[i]} want {w[i]}"
                                 f"\n got  {got.record(i)}\n want {want[i]}")
    for f in FLOAT_FIELDS:
        assert_f32_bits_equal(getattr(got, f), want[f], f"{what}: field {f}")
