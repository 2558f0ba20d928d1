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
    assert C.sizeof(abi.PassPlan) == 13 * 4
    assert [abi.PassPlan.__dict__[f].offset for f in ("threads_per_sm", "decide", "max_ctas", "grid", "capacity", "tile", "n_chk", "n_sub")] == \
        [0, 4, 8, 12, 16, 20, 36, 48]


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


def test_fused_pass_builds_and_their_register_budgets(kt):
    """The shipped SASS holds all 24 k_pass builds: the 12 kernel variants of dispatch_pass (fast family: TPC 1/2 x R <= 4/8 x
    128/256-row tiles; general family: TPC 1/2 x B 2/6) for 512 and for 768 resident threads per SM.  What the comment at
    kPassThreadsShallow claims holds: every 512-thread build fits 128 registers with no stack or local memory (no spills), every
    768-thread build fits 80 registers (a spill there is tolerated: those builds run the passes many rounds deep)."""
    import shutil
    import subprocess

    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-res-usage", kt.LIB_PATH], capture_output=True, text=True, check=True).stdout
    usage = {}
    for name, res in re.findall(r"Function (_ZN2kt6k_pass\S+):\s*\n\s*(.*)", out):
        m = re.fullmatch(r"_ZN2kt6k_passILi(\d)ELi(\d)ELi(\d)ELb([01])ELi(\d+)ELi(\d+)EEEvNS_8PassArgsE:?", name)
        assert m, name
        usage[tuple(int(x) for x in m.groups())] = {k: int(v) for k, v in re.findall(r"(\w+)(?:\[\d+\])?:(\d+)", res)}
    fast = [(tpc, 2, rt, 1, tile) for tpc in (1, 2) for rt in (4, 8) for tile in (128, 256)]
    general = [(tpc, b, 0, 0, 128) for tpc in (1, 2) for b in (2, 6)]
    want = {v + (threads,) for v in fast + general for threads in (512, 768)}
    assert set(usage) == want, sorted(set(usage) ^ want)
    for key, u in usage.items():
        if key[-1] == 512:
            assert u["REG"] <= 128 and u["STACK"] == 0 and u["LOCAL"] == 0, (key, u)
        else:
            assert u["REG"] <= 80, (key, u)


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
