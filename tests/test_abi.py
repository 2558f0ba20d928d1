"""The C-ABI library builds for sm_90a, loads on a CPU-only box and exports every symbol that
include/kt_b200.h declares.  No compute calls: there is no GPU here and no CPU fallback to call."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions(header="kt_b200.h", prefix="kt_"):
    text = open(os.path.join(ROOT, "include", header)).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(" + prefix + r"[a-z_0-9]+)\s*\(", text)))


def test_header_exports_match_library(kt):
    L = kt.lib()
    names = header_functions()
    assert len(names) >= 20
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/kt_b200.h but not exported by libkt_b200.so"
    assert sorted(kt.EXPORTS) == names, "python binding and header disagree"


def test_host_header_exports_match_library(kt):
    """include/kt_host.h (the plugin surface: NewPlugin / PreFilter / Reserve / Unreserve) is exported too."""
    from kube_throttler_b200 import host

    L = kt.lib()
    names = header_functions("kt_host.h", "kth_")
    assert len(names) >= 12
    for n in names:
        assert hasattr(L, n), f"{n} declared in include/kt_host.h but not exported by libkt_b200.so"
    assert sorted(host.HOST_EXPORTS) == names, "python binding and kt_host.h disagree"


def test_struct_layouts(kt):
    from kube_throttler_b200 import abi

    assert C.sizeof(abi.Limits) == 16
    assert C.sizeof(abi.SelectorTable) == 16 + 8 * 8
    assert C.sizeof(abi.ThrottleCols) == 14 * 8
    assert C.sizeof(abi.StatusCols) == 8 * 8
    assert C.sizeof(abi.ReconcileOut) == 8 * 8
    assert C.sizeof(abi.Timing) == 24


def test_library_is_sm90a_cuda(kt):
    """The shipped .so carries sm_90a SASS for the three hot kernels (no PTX-JIT, no other arch)."""
    import shutil
    import subprocess

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-lelf", kt.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    sass = subprocess.run([cuobjdump, "-sass", kt.LIB_PATH], capture_output=True, text=True).stdout
    for k in ("k_reconcile", "k_finalize", "k_check"):
        assert k in sass


def test_no_gpu_means_error_not_fallback(kt):
    """On a box without a GPU kt_create must fail (KT_ERR_CUDA); with one, this test is vacuous."""
    from kube_throttler_b200 import abi

    try:
        eng = kt.Engine(4, 8, 4)
    except kt.KtError as e:
        assert e.code == abi.ERR_CUDA
    else:
        eng.close()


def test_product_never_imports_oracle():
    """Only tests/, __graft_entry__.smoke() and bench.py may touch oracle/."""
    pkg = os.path.join(ROOT, "kube_throttler_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".cc", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "oracle" not in text.replace("the oracle", "").replace("test-side oracle", "").replace("oracle wrapper", "") or \
                    not re.search(r"(import|include|dlopen|CDLL).{0,40}(oracle|ko_|libkt_oracle)", text), f"{f} references the oracle"
