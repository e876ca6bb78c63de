"""bench.py's timing harness with stand-ins for the CUDA pieces (no GPU): warm-up rules, GC handling, step list."""
import gc
import importlib.util
import os
import time

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def bench():
    spec = importlib.util.spec_from_file_location("bench_under_test", os.path.join(ROOT, "bench.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class FakeEvent(object):
    def __init__(self, enable_timing=False):
        self.t = None

    def record(self):
        self.t = time.perf_counter()

    def elapsed_time(self, other):
        return (other.t - self.t) * 1e3


class FakeFlush(object):
    def fill_(self, v):
        return self


@pytest.fixture
def fake_cuda(monkeypatch):
    monkeypatch.setattr(torch.cuda, "Event", FakeEvent)
    monkeypatch.setattr(torch.cuda, "synchronize", lambda *a, **k: None)


def test_timed_runs_w_warmups_and_exactly_k_steps(bench, fake_cuda):
    calls = []

    def step():
        calls.append(gc.isenabled())
        return {"decisions": 7}
    launches = iter([10, 25])
    res, total_ms, n = bench.timed(step, 5, 3, FakeFlush(), lambda: None, lambda: next(launches))
    assert res == {"decisions": 7} and n == 15
    assert len(calls) == 8                       # 3 warm-ups + 5 timed
    assert calls[3:] == [False] * 5              # cyclic GC paused over the timed steps ...
    assert gc.isenabled()                        # ... and back on afterwards
    assert len(bench.LAST_STEP_MS) == 5 and abs(sum(bench.LAST_STEP_MS) - total_ms) < 1e-9


def test_time_based_warm_up_only_extends_single_process_runs(bench, fake_cuda):
    calls = []

    def step():
        calls.append(1)
        time.sleep(0.01)
    bench.timed(step, 2, 1, FakeFlush(), lambda: None, lambda: 0, min_warm_seconds=0.08)
    assert len(calls) >= 2 + 6                   # ~8 warm-ups of 10 ms to fill 80 ms, then the 2 timed steps
    calls.clear()
    bench.timed(step, 2, 1, FakeFlush(), lambda: None, lambda: 0)   # the torchrun legs: count-based, deterministic
    assert len(calls) == 3
    calls.clear()
    bench.timed(step, 2, 0, FakeFlush(), lambda: None, lambda: 0, min_warm_seconds=0.08)   # W = 0 stays 0
    assert len(calls) == 2


def test_gc_is_restored_when_a_step_raises(bench, fake_cuda):
    def step():
        raise RuntimeError("tick failed")
    with pytest.raises(RuntimeError):
        bench.timed(step, 1, 0, FakeFlush(), lambda: None, lambda: 0)
    assert gc.isenabled()


def test_dump_outputs_writes_npy_and_caps_the_total(bench, tmp_path):
    import numpy as np
    a = {"placed": np.arange(5, dtype=np.float64) - 2, "used": np.ones((3, 4))}
    bench.dump_outputs(str(tmp_path / "out"), a)
    for k, v in a.items():
        np.testing.assert_array_equal(np.load(str(tmp_path / "out" / (k + ".npy"))), v)
    with pytest.raises(SystemExit):
        bench.dump_outputs(str(tmp_path / "big"), {"x": np.zeros(bench.DUMP_LIMIT_BYTES // 8 + 1)})
    assert not (tmp_path / "big").exists()


def test_clock_sampler_without_nvml_or_nvidia_smi_reports_nothing(bench):
    if torch.cuda.is_available():
        pytest.skip("a GPU is present: the sampler has something to report")
    with bench.ClockSampler(0) as c:
        time.sleep(0.05)
    s = c.summary()
    assert s["samples"] == 0 and s["sm_mhz"] is None and s["reasons"] == []
