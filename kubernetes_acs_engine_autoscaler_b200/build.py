"""Build libacsfit.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m kubernetes_acs_engine_autoscaler_b200.build

The shared object is git-ignored but travels with the repo snapshot to the GPU box.
"""
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libacsfit.so")
SOURCES = ["acsfit.cu"]
HEADERS = ["acsfit_admit.cuh", "acsfit_kernels.cuh", "acsfit_math.cuh", "acsfit_rank.cuh", "acsfit_scan_plan.h", "acsfit_stream.cuh", "acsfit_stream_ff.cuh", os.path.join("..", "..", "include", "acsfit.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-fmad=false",  # 0.3*cap - util must stay a multiply followed by a subtract (scaler.py:86-87)
    "-Xcompiler", "-fPIC,-ffp-contract=off,-fvisibility=hidden",
    "-shared",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libacsfit.so (there is no CPU fallback)")


def needs_build():
    if not os.path.exists(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False, profile=False):
    """profile=True (or $ACSFIT_PROFILE=1) compiles the per-stage clock64 probe of tools/perf_probe.py into the
    pipeline kernel; the default build leaves it out (its accumulators cost registers in the placement loop)."""
    profile = profile or os.environ.get("ACSFIT_PROFILE") == "1"
    if not force and not profile and not needs_build():
        return LIB_PATH
    cmd = [_nvcc()] + NVCC_FLAGS + (["-DACSFIT_PROFILE=1"] if profile else []) + (["-Xptxas", "-v"] if verbose else []) + \
          ["-o", LIB_PATH] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s" % (res.stdout, res.stderr))
    if verbose:
        sys.stderr.write(res.stderr)
    return LIB_PATH


def hostfast_path():
    import sysconfig
    return os.path.join(PKG_DIR, "_hostfast" + (sysconfig.get_config_var("EXT_SUFFIX") or ".so"))


def build_hostfast(force=False):
    """the CPython helper module of the host-side ingestion (csrc/hostfast.c; gcc, no CUDA involved).  It is an
    accelerator only: kube.py / snapshot.py hold the same logic in Python and use it when the module is absent."""
    import sysconfig
    src, out = os.path.join(CSRC, "hostfast.c"), hostfast_path()
    if not force and os.path.exists(out) and os.path.getmtime(out) >= os.path.getmtime(src):
        return out
    cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
    if not cc:
        raise RuntimeError("no C compiler for _hostfast")
    cmd = [cc, "-O2", "-fPIC", "-shared", "-Wall", "-I" + sysconfig.get_paths()["include"], "-o", out, src]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("building _hostfast failed:\n%s\n%s" % (res.stdout, res.stderr))
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv, profile="--profile" in sys.argv))
    print(build_hostfast(force="--force" in sys.argv))
