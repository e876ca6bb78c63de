import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


@pytest.fixture(scope="session")
def oracle_mod():
    """the plain-C oracle (TEST INFRASTRUCTURE): built on demand with gcc."""
    import oracle
    oracle.build()
    return oracle


@pytest.fixture(scope="session", params=["ranks", "f64", "stream"])
def engine(request):
    """the product engine on cuda:0; GPU tests only.  Every test runs with both forms of the candidate scan --
    packed-rank integer compares (the default) and float64 compares (the fallback for huge request tables) -- and
    with the barrier-free streaming form of the pipeline kernel (csrc/acsfit_stream_ff.cuh)."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from kubernetes_acs_engine_autoscaler_b200 import build as acs_build
    acs_build.build()
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    eng = Engine(0, watchdog_ms=15000)
    eng.set_knob("ranks", 0 if request.param == "f64" else 1)
    eng.set_knob("stream", 1 if request.param == "stream" else 0)
    yield eng
    eng.close()
