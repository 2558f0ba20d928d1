import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a real H100 (run with -m gpu)")


@pytest.fixture(scope="session")
def oracle():
    from oracle import ko

    ko.build()
    return ko


@pytest.fixture(scope="session")
def kt():
    """The product binding.  GPU tests fail loudly if the CUDA library is missing -- no fallback."""
    import kube_throttler_b200 as kt

    if not os.path.exists(kt.LIB_PATH):
        kt.build()
    kt.lib()
    return kt


@pytest.fixture(scope="session")
def host_on_oracle(oracle):
    """kt_host.cc (the product's host layer) linked against tests/host_stub/engine_oracle.cc: a test double of the device engine
    that records the uploaded columns and lets the columnar ORACLE evaluate them.  Checks the host layer's packing, status
    bookkeeping, reservation cache and reason strings on the CPU; says nothing about the CUDA kernels (that is what `-m gpu`
    is for) and is never part of the product.  Returns a constructor with host.Plugin's signature."""
    import ctypes
    import functools
    import subprocess

    from kube_throttler_b200 import host

    out = os.path.join(ROOT, "tests", "_build", "libkt_hostoracle.so")
    srcs = [os.path.join(ROOT, "kube_throttler_b200", "csrc", "kt_host.cc"), os.path.join(ROOT, "tests", "host_stub", "engine_oracle.cc")]
    deps = srcs + [os.path.join(ROOT, "kube_throttler_b200", "csrc", f) for f in ("kt_json.h", "kt_quantity.h")] + \
        [os.path.join(ROOT, "include", f) for f in ("kt_b200.h", "kt_host.h")] + [os.path.join(ROOT, "oracle", "libkt_oracle.so")]
    if not os.path.exists(out) or os.path.getmtime(out) < max(os.path.getmtime(f) for f in deps):
        os.makedirs(os.path.dirname(out), exist_ok=True)
        subprocess.run(["g++", "-std=c++17", "-O1", "-shared", "-fPIC", "-o", out] + srcs +
                       ["-L", os.path.join(ROOT, "oracle"), "-lkt_oracle", "-Wl,-rpath," + os.path.join(ROOT, "oracle")], check=True)
    lib = ctypes.CDLL(out)
    return functools.partial(host.Plugin, library=lib)
