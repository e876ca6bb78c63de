"""`-m gpu`: every instantiation of the first-fit kernels against the plain-C oracle, with proof that it ran.

The host picks `firstfit_pipeline_kernel<D, BINS, NT, PRUNE, RW>` or `firstfit_stream_kernel<D, BINS, RW>` at run
time from D, the pass, the packed-rank word count RW of the tick's request table and the schedule.  Each case here
forces one rank layout (tests/variant_cases.py), runs the fused scale-up tick under one schedule and compares it
with the oracle exactly; then the library's launch records (Engine.last_launches) must show that the node pass and
the bin passes ran the intended variant -- a silent fall-back from ranks to the float64 scan, from the streaming
form to the barrier kernel or from a chained to an unchained pass fails the case even when the answer is right.
The last tests pack bins across the real 1024-stage pass limit, with answers in closed form."""
import functools

import numpy as np
import pytest
import torch

import variant_cases as vc
from kubernetes_acs_engine_autoscaler_b200 import synthetic as syn
from test_gpu_parity import bits, oracle_scale_up, to_np
from test_rank_math_cpu import layout

pytestmark = pytest.mark.gpu

# knob settings of each schedule, applied on top of the engine fixture's mode; DEFAULT_KNOBS restores the ctx
SCHEDULES = {
    "default": {},
    "waves": {"min_stages": 1 << 20},                 # the narrowest stages: more stage CTAs than the GPU holds
    "waves_noprune": {"min_stages": 1 << 20, "prune": 0},
    "unchained": {"overlap": 0},
    # several bin passes per pool; min_stages = 32 leaves room beside the node stages for a chained first pass
    "multipass_chained": {"bin_pass_stages": 2, "min_stages": 32},
    "multipass_unchained": {"bin_pass_stages": 2, "overlap": 0},
}
DEFAULT_KNOBS = {"min_stages": 0, "prune": -1, "overlap": 1, "bin_pass_stages": 0}


def mode_of(request):
    """the scan form the session's `engine` fixture runs this test with ("ranks", "f64" or "stream")"""
    return request.node.callspec.params["engine"]


@functools.lru_cache(maxsize=None)
def case_and_oracle(name):
    """the tick of one layout and the oracle's answer; neither depends on the schedule or the scan form"""
    import oracle
    c = vc.case(name)
    used0 = syn.initial_used(c)
    used_o = used0.copy()
    return c, used0, oracle_scale_up(oracle, c, used_o), used_o


def run_tick(engine, c, used0, knobs):
    f64, i32 = torch.float64, torch.int32
    try:
        for k, v in knobs.items():
            engine.set_knob(k, v)
        d_used = engine.dev(used0, f64)
        g = engine.scale_up(engine.dev(c["req"], f64), c["unit_all"], c["unit_ordered"], c["pool_actual"],
                            c["pool_max"], c["pool_ignored"], c["over_provision"], engine.dev(c["cap_type"], f64),
                            engine.dev(c["node_type"], i32), d_used)
        torch.cuda.synchronize()
        return g, to_np(d_used), engine.last_launches()
    finally:
        for k, v in DEFAULT_KNOBS.items():
            engine.set_knob(k, v)


def check_records(recs, mode, D, rw, schedule, o):
    nodes = [r for r in recs if r["pass"] == 0]
    bins = [r for r in recs if r["pass"] == 1]
    assert len(nodes) == 1, recs
    assert bins, recs
    for r in recs:
        assert r["D"] == D and r["RW"] == rw, r
        # the streaming form wherever its conditions hold, the barrier kernel everywhere else
        stream_ok = mode == "stream" and D <= 8 and rw > 0 and r["Tn"] >= 32 and r["Tn"] % 32 == 0 and not r["prune"]
        assert r["form"] == int(stream_ok), r
        if not r["form"]:
            assert r["publish_every"] == (4 if r["stages"] > r["resident"] else 1), r
        assert (r["pool"] >= 0) == bool(r["pass"]), r
    if mode == "stream" and D <= 8 and rw > 0:
        assert all(r["form"] == 1 for r in recs), recs  # its stages are planned >= 32 wide: never the barrier kernel
    # every pool that opened bins has bin-pass records, in increasing pass order, each starting where the last ended
    for t in np.nonzero(o["bins_opened"])[0]:
        passes = [r for r in bins if r["pool"] == t]
        assert passes, (t, recs)
        assert passes[0]["bin_base"] == 0
        for a, b in zip(passes, passes[1:]):
            assert b["bin_base"] == a["bin_base"] + a["stages"] * a["Tn"], (a, b)

    chained = [r for r in recs if r["chained"]]
    if chained:  # node pass + first bin pass of pool 0, launched together: every stage CTA of both must be resident
        assert [r["pass"] for r in chained] == [0, 1] and chained[1]["pool"] == 0 and chained[1] is bins[0], recs
        assert chained[0]["stages"] + chained[1]["stages"] <= min(r["resident"] for r in chained), chained

    if schedule.startswith("waves"):
        for r in (nodes[0], bins[0]):
            if r["form"]:
                assert r["Tn"] == 32, r                 # the narrowest streaming stage
            else:
                assert r["stages"] > r["resident"], r   # several waves of stage CTAs
        if not nodes[0]["form"]:
            assert nodes[0]["prune"] == (1 if schedule == "waves" else 0), nodes[0]
    if schedule in ("unchained", "multipass_unchained"):
        assert not any(r["chained"] for r in recs)
    if schedule.startswith("multipass"):
        assert all(r["stages"] <= 2 for r in bins), bins
        pool0 = [r for r in bins if r["pool"] == 0]
        assert len(pool0) >= 2, pool0
    if schedule == "multipass_chained":
        assert nodes[0]["chained"] == 1 and bins[0]["chained"] == 1 and bins[0]["pool"] == 0, recs
        assert not any(r["chained"] for r in bins[1:]), recs


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sorted(vc.LAYOUTS))
def test_variant_matches_oracle(request, engine, oracle_mod, name, schedule):
    c, used0, o, used_o = case_and_oracle(name)
    D, U, _ = vc.LAYOUTS[name]
    mode = mode_of(request)
    rw = 0 if mode == "f64" else vc.expected_rw(U, layout)
    g, used, recs = run_tick(engine, c, used0, SCHEDULES[schedule])
    for k in ("feasible", "placed", "acc_pool"):
        np.testing.assert_array_equal(to_np(g[k]), o[k], err_msg=k)
    for k in ("new_size", "units_needed", "bins_opened"):
        np.testing.assert_array_equal(g[k], o[k], err_msg=k)
    for k in ("n_to_schedule", "n_pending", "num_unaccounted", "decisions"):
        assert g[k] == o[k], k
    np.testing.assert_array_equal(bits(used), bits(used_o))
    check_records(recs, mode, D, rw, schedule, o)


@pytest.mark.parametrize("D", [4, 16])
def test_bin_passes_at_full_size_closed_form(engine, D):
    """fulfill_pending across the real pass limit (1024 stages of the widest stage): every pod requests the
    pool's unit in dimension 0 and nothing else, so it opens its own bin after failing every earlier one; pool 0's
    size limit cuts it inside the second pass and pool 1 packs the rest the same way."""
    tn = 256 if D <= 8 else 128                       # max_stage_nodes(D): the widest stage, kept at this size
    M = 1024 * tn + 5000
    take = 1024 * tn + 2000
    unit = np.resize(np.array([1.5, 7096762368.0, 110.0, 8.0]), D)
    req = np.zeros((M, D))
    req[:, 0] = unit[0]
    actual = np.array([3, 1], np.int32)
    pmax = np.array([3 + take, 1 << 30], np.int32)
    g = engine.fulfill_pending(engine.dev(req, torch.float64), M, np.stack([unit, unit]), actual, pmax,
                               np.zeros(2, np.uint8), 0)
    torch.cuda.synchronize()
    recs = engine.last_launches()
    j = np.arange(M)
    rest = M - take
    np.testing.assert_array_equal(to_np(g["bin_of"]), np.where(j < take, j, j - take))
    np.testing.assert_array_equal(to_np(g["acc_pool"]), np.where(j < take, 0, 1))
    np.testing.assert_array_equal(g["bins_opened"], [M, rest])
    np.testing.assert_array_equal(g["units_needed"], [M, rest])
    np.testing.assert_array_equal(g["new_size"], [3 + take, 1 + rest])
    assert g["num_unaccounted"] == 0
    assert g["evals"] == M + M * (M - 1) // 2 + rest + rest * (rest - 1) // 2
    pool0 = [r for r in recs if r["pass"] == 1 and r["pool"] == 0]
    assert len(pool0) == 2, recs
    assert (pool0[0]["bin_base"], pool0[0]["stages"], pool0[0]["Tn"]) == (0, 1024, tn), pool0
    assert pool0[1]["bin_base"] == 1024 * tn, pool0
    assert pool0[0]["stages"] > pool0[0]["resident"], pool0  # the first pass runs in waves


def test_rank_path_on_two_devices_in_one_process(oracle_mod):
    """function attributes are per device: a second ctx on another device of the same process must get the
    rank-table sort's shared-memory size too"""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    c, used0, _, _ = case_and_oracle("d8_rw2")
    engines = [Engine(0), Engine(1)]
    try:
        used_o = used0.copy()
        placed_o, calls_o = oracle_mod.first_fit_nodes(c["req"], c["cap_type"], c["node_type"], used_o)
        for eng in engines:
            d_used = eng.dev(used0, torch.float64)
            placed, dec = eng.first_fit_nodes(eng.dev(c["req"], torch.float64), None,
                                              eng.dev(c["cap_type"], torch.float64),
                                              eng.dev(c["node_type"], torch.int32), d_used)
            torch.cuda.synchronize(eng.device)
            np.testing.assert_array_equal(to_np(placed), placed_o)
            np.testing.assert_array_equal(bits(to_np(d_used)), bits(used_o))
            assert int(to_np(dec)[0]) == calls_o
            assert [r["RW"] for r in eng.last_launches()] == [2]
    finally:
        for eng in engines:
            eng.close()
