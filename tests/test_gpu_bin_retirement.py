"""`-m gpu`: bin retirement in the bin-packing pipeline, against the plain-C oracle.

A bin pass with rank tables treats a bin as dead once its remaining amount S[d] is below the smallest request value
of the call in some dimension d: no pod of the pass can take it again.  Its resolver chain skips warps whose 32 bins
are all dead, and a stage whose warps are all dead forwards every later tile untouched.  None of this may change an
answer, so every case here is compared exactly with the oracle (bins, pools, credited evaluations), with retirement
on (the default) and off (knob "retire" = 0).  Each case also checks, from the oracle's own placements, that it
builds the situation it is named after.  Stages are 256 bins wide (min_stages = 1) unless a case says otherwise."""
import numpy as np
import pytest
import torch

from test_gpu_parity import to_np

pytestmark = pytest.mark.gpu

BIG = 1 << 30


def remaining(req, bin_of, unit):
    """each bin's remaining amounts after the pass, subtracted in pod order as the reference does"""
    nb = int(bin_of.max()) + 1
    S = np.tile(np.asarray(unit, np.float64), (nb, 1))
    for i in np.nonzero(bin_of >= 0)[0]:
        S[bin_of[i]] = S[bin_of[i]] - req[i]
    return S


def dead_bins(req, bin_of, unit):
    """[bins, D]: dimension d retires the bin (S[d] < the smallest request of d)"""
    return remaining(req, bin_of, unit) < req.min(axis=0)


def pack(engine, oracle_mod, req, unit, knobs=None):
    """one pool, no size limit: the oracle's answer, and the engine's with retirement on and off"""
    req = np.ascontiguousarray(req, np.float64)
    unit = np.asarray(unit, np.float64).reshape(1, -1)
    args = (np.zeros(1, np.int32), np.array([BIG], np.int32), np.zeros(1, np.uint8), 0)
    o = oracle_mod.fulfill_pending(req, len(req), unit, *args)
    knobs = {"min_stages": 1, **(knobs or {})}
    try:
        for k, v in knobs.items():
            engine.set_knob(k, v)
        for retire in (1, 0):
            engine.set_knob("retire", retire)
            g = engine.fulfill_pending(engine.dev(req, torch.float64), len(req), unit, *args)
            torch.cuda.synchronize()
            for k in ("new_size", "units_needed", "bins_opened"):
                np.testing.assert_array_equal(g[k], o[k], err_msg="%s (retire=%d)" % (k, retire))
            np.testing.assert_array_equal(to_np(g["acc_pool"]), o["acc_pool"], err_msg="retire=%d" % retire)
            np.testing.assert_array_equal(to_np(g["bin_of"]), o["bin_of"], err_msg="retire=%d" % retire)
            assert g["num_unaccounted"] == o["num_unaccounted"]
            assert g["evals"] == o["evals"], retire
    finally:
        engine.set_knob("retire", 1)
        engine.set_knob("min_stages", 0)
        engine.set_knob("bin_pass_stages", 0)
    return o


def one_heavy_dim(rng, P, D, heavy, light):
    """every pod is heavy in one random dimension and light in the others"""
    req = rng.choice(light, size=(P, D)).astype(np.float64)
    k = rng.integers(0, D, size=P)
    req[np.arange(P), k] = rng.choice(heavy, size=P)
    return req


@pytest.mark.parametrize("D", [2, 4, 8, 16])
def test_retires_through_every_dimension(engine, oracle_mod, D):
    rng = np.random.default_rng(100 + D)
    req = one_heavy_dim(rng, 20000, D, [5.0, 6.0, 7.0], [1.0, 2.0])
    o = pack(engine, oracle_mod, req, np.full(D, 16.0))
    dead = dead_bins(req, o["bin_of"], np.full(D, 16.0))
    assert dead.any(axis=0).all(), dead.sum(axis=0)  # every dimension retires some bin
    assert o["bins_opened"][0] > 3 * 256              # several stages of 256 bins


def test_retires_through_the_pods_column(engine, oracle_mod):
    """dimension 1 is the pods column (110 per node, 1 per pod): every bin dies by count, with room left in the
    other dimension; the first stages retire while the last one is still open"""
    rng = np.random.default_rng(7)
    P = 110 * 600 + 37
    req = np.stack([rng.choice([1.0, 2.0, 3.0], size=P), np.ones(P)], axis=1)
    unit = [1000.0, 110.0]
    o = pack(engine, oracle_mod, req, unit)
    S = remaining(req, o["bin_of"], unit)
    assert o["bins_opened"][0] == 601
    assert (S[:600, 1] == 0).all() and (S[:600, 0] > 0).all() and S[600, 1] > 0


def test_whole_stage_retires_while_a_later_stage_is_open(engine, oracle_mod):
    """requests of 3 and 4 in a unit of 10: a bin dies with its second or third pod, so stage 0 (bins 0-255) is
    all dead long before the last pod while the newest stage still has open bins"""
    rng = np.random.default_rng(11)
    P = 3000
    req = np.stack([rng.choice([3.0, 4.0], size=P), np.ones(P)], axis=1)
    unit = [10.0, 110.0]
    o = pack(engine, oracle_mod, req, unit)
    bin_of = o["bin_of"]
    dead = dead_bins(req, bin_of, unit).any(axis=1)
    first_pod_of_stage2 = int(np.argmax(bin_of >= 512))
    dead_early = dead_bins(req[:first_pod_of_stage2], bin_of[:first_pod_of_stage2], unit).any(axis=1)
    assert dead_early[:256].all()      # stage 0 retired before stage 2 opened a bin
    assert not dead[-8:].all()         # the last stage stays live


@pytest.mark.parametrize("layout", ["whole_stage", "one_warp"])
def test_bin_left_with_exactly_the_minimum_is_live(engine, oracle_mod, layout):
    """bins 0-31 keep exactly the smallest request (3 of 10) in dimension 0: they are live, and the pods of 3 of the
    next tile must go there.  "whole_stage": every other bin of stage 0 is dead (2 left); "one_warp": warps 1-4 are
    dead and warps 5-7 untouched.  Retiring on S <= min instead of S < min breaks both."""
    if layout == "whole_stage":
        first = [7.0] * 32 + [8.0] * 224
    else:
        first = [7.0] * 32 + [8.0] * 32 + [5.0] * 192
    col0 = np.array(first + [3.0] * 64 + [4.0] * 16)
    req = np.stack([col0, np.ones(len(col0))], axis=1)
    unit = [10.0, 110.0]
    o = pack(engine, oracle_mod, req, unit)
    assert (o["bin_of"][256:288] == np.arange(32)).all()
    S = remaining(req[:256], o["bin_of"][:256], unit)
    assert (S[:32, 0] == 3.0).all() and req[:, 0].min() == 3.0


def test_zero_minimum_retires_nothing(engine, oracle_mod):
    """one all-zero request row makes every dimension's minimum 0: no bin ever dies, answers stay exact"""
    rng = np.random.default_rng(5)
    req = one_heavy_dim(rng, 6000, 4, [5.0, 6.0, 7.0], [1.0, 2.0])
    req[1234] = 0.0
    o = pack(engine, oracle_mod, req, np.full(4, 16.0))
    assert not dead_bins(req, o["bin_of"], np.full(4, 16.0)).any()


def test_float64_scan_and_default_stages(engine, oracle_mod, request):
    """the same retiring workload with the float64 scan (no rank tables: nothing retires) and with the library's own
    stage plan, several passes included"""
    rng = np.random.default_rng(9)
    req = one_heavy_dim(rng, 12000, 4, [5.0, 6.0, 7.0], [1.0, 2.0])
    try:
        engine.set_knob("ranks", 0)
        pack(engine, oracle_mod, req, np.full(4, 16.0))
    finally:
        engine.set_knob("ranks", 0 if request.node.callspec.params["engine"] == "f64" else 1)
    pack(engine, oracle_mod, req, np.full(4, 16.0), {"min_stages": 0})
    pack(engine, oracle_mod, req, np.full(4, 16.0), {"bin_pass_stages": 2})
