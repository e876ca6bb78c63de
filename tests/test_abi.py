"""`-m "not gpu"`: libacsfit.so builds (nvcc cross-compiles sm_90a without a GPU), loads, and exports
every symbol include/acsfit.h declares; the product refuses to run without CUDA."""
import ctypes
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    text = open(os.path.join(ROOT, "include", "acsfit.h")).read()
    return sorted(set(re.findall(r"ACSFIT_API[^;(]*?\b(acsfit_[a-z_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    from kubernetes_acs_engine_autoscaler_b200 import build as acs_build
    path = acs_build.build()
    lib = ctypes.CDLL(path)
    names = declared_symbols()
    assert len(names) >= 18
    for name in names:
        assert hasattr(lib, name), name
    lib.acsfit_abi_version.restype = ctypes.c_int
    assert lib.acsfit_abi_version() == 2  # 2: cluster-mode entry points
    # the python binding table covers the header too
    from kubernetes_acs_engine_autoscaler_b200 import _native
    assert set(names) <= set(_native.SIGNATURES)


def test_built_for_sm_90a_only():
    from kubernetes_acs_engine_autoscaler_b200 import build as acs_build
    cuobjdump = os.path.join(os.path.dirname(acs_build._nvcc()), "cuobjdump")
    out = subprocess.run([cuobjdump, "--list-elf", acs_build.build()], capture_output=True, text=True).stdout
    assert "sm_90a" in out
    assert not re.search(r"sm_(?!90a)\d+", out)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    with pytest.raises(RuntimeError):
        Engine()
    # the C ABI itself also refuses
    from kubernetes_acs_engine_autoscaler_b200 import _native
    lib = _native.load()
    ctx = ctypes.c_void_p()
    assert lib.acsfit_ctx_create(0, ctypes.byref(ctx)) == _native.E_CUDA


def test_threshold_property_on_host(tmp_path):
    """acsfit::node_threshold (csrc/acsfit_math.cuh) is exact: fits(thr) && !fits(nextup(thr))."""
    exe = os.path.join(str(tmp_path), "test_threshold")
    subprocess.check_call(["g++", "-O2", "-ffp-contract=off", "-x", "c++",
                           "-I", os.path.join(ROOT, "kubernetes_acs_engine_autoscaler_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "test_threshold.cpp"), "-o", exe])
    out = subprocess.run([exe, "1500000"], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout[-2000:]
