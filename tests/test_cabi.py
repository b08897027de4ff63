"""The C-ABI boundary without a GPU: libqk.so builds for sm_90a, loads, and exports exactly the entry
points include/qk.h declares; argument errors are reported through qk_last_error (no compute calls)."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared():
    src = open(os.path.join(ROOT, "include", "qk.h")).read()
    return sorted(set(re.findall(r"^QK_API [^(]*?(qk_[a-z_]+)\(", src, flags=re.M)))


def test_library_builds_loads_and_exports_every_declared_symbol():
    from quokka_b200 import build, _lib
    path = build.build()
    assert os.path.exists(path)
    lib = _lib.lib()
    names = declared()
    assert len(names) >= 27
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/qk.h but not exported"
    assert sorted(_lib.EXPORTS) == names, "quokka_b200/_lib.py signatures must cover include/qk.h exactly"
    out = subprocess.run(["nm", "-D", "--defined-only", path], capture_output=True, text=True).stdout
    exported = sorted(l.split()[-1] for l in out.splitlines() if " T " in l)
    assert exported == names, "only the extern \"C\" entry points may be exported"
    assert lib.qk_version() == 100


def test_sass_is_hopper_native():
    """sm_90a only, TMA-engine bulk copies + mbarrier transactions present in the hot kernels."""
    from quokka_b200 import _lib
    out = subprocess.run(["cuobjdump", "-lelf", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out and "sm_100" not in out and "sm_80" not in out
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert sass.count("UBLKCP") >= 10 and "SYNCS.ARRIVE.TRANS64" in sass


def test_argument_errors_are_reported_without_a_gpu():
    from quokka_b200 import _lib as L
    lib = L.lib()
    assert lib.qk_join_init(None, 1000, None) == -1                       # null table, capacity not a power of two
    assert b"power of two" in lib.qk_last_error()
    desc = L.qk_hashagg_desc()
    desc.capacity, desc.nkeys = 1024, 5
    assert lib.qk_hashagg_state_bytes(C.byref(desc)) > 0
    assert lib.qk_hashagg_init(C.byref(desc), None, None) == -1
    assert b"nkeys" in lib.qk_last_error()
    col = L.qk_column(None, None, 10, L.QK_F64, 0)
    assert lib.qk_partition_plan(C.byref(col), 8, 0, None, None, None, 0, None) == -1   # length 10 but no data
    col = L.qk_column(None, None, 0, 99, 0)
    assert lib.qk_partition_plan(C.byref(col), 8, 0, None, None, None, 0, None) == -1
    assert b"dtype" in lib.qk_last_error()


@pytest.mark.parametrize("variant", [2, 4, 5, 6, 8, -1])
def test_dense_agg_rejects_unknown_variants_first(variant):
    """qk_scan_filter_agg_dense takes variants 0, 1, 3 and 7; any other is refused before the other arguments are looked
    at (here ngroup_cols = -1 and null columns would be errors too)."""
    from quokka_b200 import _lib as L
    lib = L.lib()
    args = (None, 0, 0, None, None, None, -1, None, None, 0, None, None, None, 0)
    assert lib.qk_scan_filter_agg_dense(*args, variant, None) == -1
    assert b"variant" in lib.qk_last_error()
    assert lib.qk_scan_filter_agg_dense(*args, 0, None) == -1                # a known variant: the next check fails
    assert b"variant" not in lib.qk_last_error()


def test_no_cpu_fallback_in_ops():
    import torch
    from quokka_b200 import _lib as L, ops
    with pytest.raises(L.QkError, match="CUDA tensor"):
        ops.partition_plan(torch.zeros(4, dtype=torch.int64), 2)
    with pytest.raises(L.QkError, match="CUDA tensor"):
        ops.gather([torch.zeros(4)], torch.zeros(2, dtype=torch.int32))
