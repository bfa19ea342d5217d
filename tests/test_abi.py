"""The C-ABI shared library: builds in-tree for sm_90a, loads, and exports every entry point that
include/wva_b200.h declares.  No compute calls here (no GPU on the CPU box)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from workload_variant_autoscaler_b200 import _lib
    _lib.build()
    return _lib.lib()


def _declared_functions():
    src = open(os.path.join(ROOT, "include", "wva_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(wva_[a-z_0-9]+)\s*\(", src)))


def test_header_functions_are_exported(lib):
    from workload_variant_autoscaler_b200 import _lib
    declared = _declared_functions()
    assert len(declared) >= 18
    missing = [n for n in declared if not hasattr(lib, n)]
    assert not missing, f"declared in include/wva_b200.h but not exported: {missing}"
    assert sorted(_lib.EXPORTS) == declared, "python binding list and header disagree"


def test_abi_version_and_strerror(lib):
    assert lib.wva_abi_version() == 2
    assert lib.wva_strerror(0) == b"ok"
    for code in (-1, -2, -3, -4, -5, -6, -99):
        assert len(lib.wva_strerror(code)) > 0


def test_tunables_default_match_reference(lib):
    from workload_variant_autoscaler_b200 import _abi
    t = _abi.Tunables()
    lib.wva_tunables_default(C.byref(t))
    assert t.max_queue_to_batch_ratio == 10          # pkg/config/defaults.go:18
    assert abs(t.accel_penalty_factor - 0.1) < 1e-8  # pkg/config/defaults.go:21


def test_struct_layouts_match_header_sizes():
    """ctypes mirrors of the ABI structs: field counts and natural alignment (x86-64 SysV)."""
    from workload_variant_autoscaler_b200 import _abi
    assert C.sizeof(_abi.Tunables) == 8
    assert C.sizeof(_abi.AllocsC) == 10 * 8
    assert C.sizeof(_abi.GridC) == 32
    assert C.sizeof(_abi.CellsC) == 5 * 8
    assert C.sizeof(_abi.SweepOutC) == 6 * 8
    # wva_fleet: 4 sizes + 27 pointers + flags + tunables, padded as the C compiler pads it
    import subprocess
    import tempfile
    prog = ('#include <stdio.h>\n#include "wva_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n", sizeof(wva_fleet), '
            'sizeof(wva_allocs), sizeof(wva_grid), sizeof(wva_summary));return 0;}')
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(prog)
        subprocess.run(["gcc", "-I", os.path.join(ROOT, "include"), "-o", os.path.join(d, "t"),
                        os.path.join(d, "t.c")], check=True)
        out = subprocess.run([os.path.join(d, "t")], check=True, capture_output=True, text=True).stdout.split()
    assert [int(x) for x in out] == [C.sizeof(_abi.FleetC), C.sizeof(_abi.AllocsC), C.sizeof(_abi.GridC),
                                     C.sizeof(_abi.SummaryC)]
    # the column tables name the mirrors' array fields in order, with their element types
    import numpy as np
    for struct, table in ((_abi.FleetC, _abi.FLEET_COLUMNS), (_abi.AllocsC, _abi.ALLOC_COLUMNS)):
        arrays = [(n, t._type_) for n, t in struct._fields_ if issubclass(t, C._Pointer)]
        assert arrays == [(col[0], _abi._CT[np.dtype(col[1])]) for col in table]


def test_create_without_gpu_fails_loudly(lib):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    h = C.c_void_p()
    assert lib.wva_create(C.byref(h), 0) == -2  # WVA_ERR_NO_DEVICE: there is no CPU fallback
    assert not h.value
    from workload_variant_autoscaler_b200 import Engine, WvaError
    with pytest.raises(WvaError):
        Engine(0)


def test_product_never_imports_oracle():
    """The product package must not reference the test-only oracle."""
    pkg = os.path.join(ROOT, "workload_variant_autoscaler_b200")
    for dp, _, files in os.walk(pkg):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh", ".h", ".cc")):
                txt = open(os.path.join(dp, fn)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "wva_oracle" not in txt, fn
                assert "wvao_" not in txt, fn
