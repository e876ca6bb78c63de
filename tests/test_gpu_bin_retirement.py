"""`-m gpu`: bin retirement in the bin-packing pipeline, against the plain-C oracle.

A bin pass with rank tables treats a bin as dead once its remaining amount S[d] is below the smallest request value
of the call in some dimension d: no pod of the pass can take it again.  Its resolver chain skips warps whose 32 bins
are all dead, and a stage whose warps are all dead forwards every later tile untouched.  None of this may change an
answer, so every case here is compared exactly with the oracle (bins, pools, credited evaluations), with retirement
on (the default) and off (knob "retire" = 0).  Each case also checks, from the oracle's own placements, that it
builds the situation it is named after.  Stages are 256 bins wide (min_stages = 1) unless a case says otherwise.

Every case also checks the library's report of what retirement marked (Engine.last_bin_retirement: dead warps and
retired stages of the call's bin passes) against the model of tests/bin_chain_cases.py, computed from the oracle's
final bins and the call's launch records; with retirement off the report is (0, 0).  The cases of that file build
dead-warp patterns on purpose (holes in the chain, a last live warp that moves, every 8-warp pattern, narrow stages)
and run through every entry point that packs bins."""
import os

import numpy as np
import pytest
import torch

import aa_oracle
import bin_chain_cases as bcc
import sel_oracle
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


# knob values every case leaves behind (the engine fixture lives for the session; "overlap": a chain-timeout redo turns
# chaining off for the ctx, and its default follows ACSFIT_OVERLAP)
RESTORE = {"retire": 1, "min_stages": 0, "bin_pass_stages": 0, "inject_chain_timeout": 0,
           "overlap": int(int(os.environ.get("ACSFIT_OVERLAP", "1")) != 0)}


def check_passes(recs, S_by_pool, redone=False):
    """the bin passes of every pool: the first starts at bin 0 (a chained first pass included), each next one where the
    previous ended, and together they cover every bin the oracle opened in that pool"""
    bins = [r for r in recs if r["pass"] == 1 and not (redone and r["chained"])]
    assert {r["pool"] for r in bins} == {t for t, S in S_by_pool.items() if len(S)}, (bins, list(S_by_pool))
    for t in {r["pool"] for r in bins}:
        passes = [r for r in bins if r["pool"] == t]
        assert passes[0]["bin_base"] == 0 and all(r["chained"] == 0 for r in passes[1:]), passes
        for a, b in zip(passes, passes[1:]):
            assert b["bin_base"] == a["bin_base"] + a["stages"] * a["Tn"], (a, b)
        end = passes[-1]["bin_base"] + passes[-1]["stages"] * passes[-1]["Tn"]
        assert passes[-1]["bin_base"] < len(S_by_pool[t]) <= end, (passes, len(S_by_pool[t]))


def check_report(engine, S_by_pool, req, retire, label, redone=False):
    """the call's launch records and the hook's (dead warps, retired stages) against the model; returns both.
    redone: the chained launch of the records was discarded and redone unchained; only the redo counts"""
    recs = engine.last_launches()
    bins = [r for r in recs if r["pass"] == 1]
    assert bins, label
    for r in bins:
        assert r["Tn"] > 0 and r["stages"] > 0 and r["bin_base"] >= 0, (label, r)
    got = engine.last_bin_retirement()
    check_passes(recs, S_by_pool, redone)
    kept = [r for r in recs if not (redone and r["chained"])]
    want = bcc.retirement(kept, S_by_pool, bcc.minreq(req)) if retire else (0, 0)
    assert got == want, "%s: hook (dead warps, retired stages) %s, model %s; records %s" % (label, got, want, bins)
    return recs, got


def run_both(engine, call, check, knobs=None):
    """call() under each retire setting with the knobs set, check(g, retire) after each; knobs restored after.
    Returns [(records, hook) for retire = 1, 0]"""
    out = []
    try:
        for k, v in {"min_stages": 1, **(knobs or {})}.items():
            engine.set_knob(k, v)
        for retire in (1, 0):
            engine.set_knob("retire", retire)
            g = call()
            torch.cuda.synchronize()
            out.append(check(g, retire))
    finally:
        for k, v in RESTORE.items():
            engine.set_knob(k, v)
    return out


def assert_fulfill_equal(g, o, label):
    for k in ("new_size", "units_needed", "bins_opened"):
        np.testing.assert_array_equal(g[k], o[k], err_msg="%s: %s" % (label, k))
    np.testing.assert_array_equal(to_np(g["acc_pool"]), o["acc_pool"], err_msg=label + ": acc_pool")
    np.testing.assert_array_equal(to_np(g["bin_of"]), o["bin_of"], err_msg=label + ": bin_of")
    assert g["num_unaccounted"] == o["num_unaccounted"], label
    assert g["evals"] == o["evals"], label


def pack(engine, oracle_mod, req, unit, knobs=None):
    """one pool, no size limit: the oracle's answer, and the engine's with retirement on and off (answers, launch
    records and the retirement report).  Returns the oracle's answer and the (records, report) of retire = 1."""
    req = np.ascontiguousarray(req, np.float64)
    unit = np.asarray(unit, np.float64).reshape(1, -1)
    args = (np.zeros(1, np.int32), np.array([BIG], np.int32), np.zeros(1, np.uint8), 0)
    o = oracle_mod.fulfill_pending(req, len(req), unit, *args)
    S = {0: bcc.remaining(req, o["bin_of"], unit[0])}

    def check(g, retire):
        assert_fulfill_equal(g, o, "retire=%d" % retire)
        return check_report(engine, S, req, retire, "retire=%d" % retire)
    rep = run_both(engine, lambda: engine.fulfill_pending(engine.dev(req, torch.float64), len(req), unit, *args),
                   check, knobs)
    o["report"] = rep[0]
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


# ---------------------------------------------------------------------------------------------------------------------
# dead-warp patterns built on purpose (tests/bin_chain_cases.py), through every entry point that packs bins
# ---------------------------------------------------------------------------------------------------------------------
CHAIN = bcc.cases()


def mode_of(request):
    return request.node.callspec.params["engine"]


def expected_tn(c, mode, D):
    """the stage width the plan must give the case: the streaming form (packed-rank scan, D <= 8) never plans stages
    narrower than 32 bins"""
    return max(c["Tn"], 32) if mode == "stream" and D <= 8 else c["Tn"]


@pytest.mark.parametrize("name", sorted(CHAIN))
def test_chain_case(engine, oracle_mod, request, name):
    c = CHAIN[name]
    D = c["req"].shape[1]
    o = pack(engine, oracle_mod, c["req"], c["unit"], c["knobs"])
    recs, (warps, stages) = o["report"]
    first = [r for r in recs if r["pass"] == 1][0]
    assert first["Tn"] == expected_tn(c, mode_of(request), D) and first["bin_base"] == 0, first
    if first["RW"] > 0 and first["form"] == 0 and first["Tn"] == c["Tn"]:
        want = sum(bin(m).count("1") for m in c["expect"].values())
        assert warps >= want, (warps, want)  # the patterned stages' dead warps are in the report


def multi_pool_inputs(c):
    """three pools in visiting order: pool 0 the case's unit clipped by its max size, pool 1 ignored, pool 2 a wider
    unit that takes what pool 0 could not; duplicates in num_listed, over_provision 1"""
    u = c["unit"]
    units = np.stack([u, u, u * np.where(np.arange(len(u)) == 0, 2.0, 1.0)])
    actual = np.array([3, 0, 1], np.int32)
    pool_max = np.array([3 + 300, 50, BIG], np.int32)
    ignored = np.array([0, 1, 0], np.uint8)
    return units, actual, pool_max, ignored, 1


@pytest.mark.parametrize("name", ["hole_LDL", "retired_then_placing", "width_16"])
def test_chain_case_several_pools_and_passes(engine, oracle_mod, name):
    """fulfill_pending with several pools (pool 0 clipped, an ignored pool between two packing pools, over_provision,
    duplicates in num_listed) and at most 2 stages per bin pass, so that later passes start at bin_base > 0"""
    c = CHAIN[name]
    req = c["req"]
    units, actual, pool_max, ignored, over = multi_pool_inputs(c)
    listed = len(req) + 17
    o = oracle_mod.fulfill_pending(req, listed, units, actual, pool_max, ignored, over)
    assert o["acc_pool"].max() == 2 and (o["acc_pool"] == 0).any()  # pool 0 clipped, pool 2 takes the rest

    def one(t, idx):
        return oracle_mod.fulfill_pending(req[idx], len(idx), units[t:t + 1], np.zeros(1, np.int32),
                                          np.array([BIG], np.int32), np.zeros(1, np.uint8), 0)["bin_of"]
    S = bcc.pool_bins(one, req, o["acc_pool"], units, ignored)

    def check(g, retire):
        assert_fulfill_equal(g, o, "retire=%d" % retire)
        recs, rep = check_report(engine, S, req, retire, "retire=%d" % retire)
        bins = [r for r in recs if r["pass"] == 1]
        assert {r["pool"] for r in bins} == {0, 2} and all(r["stages"] <= 2 for r in bins)
        assert any(r["bin_base"] > 0 for r in bins if r["pool"] == 0)
        return recs, rep
    run_both(engine, lambda: engine.fulfill_pending(engine.dev(req, torch.float64), listed, units, actual, pool_max,
                                                    ignored, over), check, {"bin_pass_stages": 2})


def test_chain_case_selector_gate(engine):
    """fulfill_pending_sel: pool 0 admits class 0 only, pool 1 every class.  Pool 0's pass sees a subset of the call's
    rows (the minimum still comes from every row); pool 1 packs the rest"""
    c = CHAIN["hole_LDL"]
    req = c["req"]
    P = len(req)
    pod_class = (np.arange(P) % 7 == 3).astype(np.uint8)  # one pod in seven is class 1
    units = np.stack([c["unit"], c["unit"]])
    actual, pool_max, ignored = np.zeros(2, np.int32), np.full(2, BIG, np.int32), np.zeros(2, np.uint8)
    pool_match = np.array([1, 3], np.uint64)
    o = sel_oracle.fulfill_pending_sel(req, P, units, actual, pool_max, ignored, 0, pool_match, pod_class)
    assert (o["acc_pool"] == 1).sum() == (pod_class == 1).sum()

    def one(t, idx):
        return sel_oracle.fulfill_pending_sel(req[idx], len(idx), units[t:t + 1], actual[:1], pool_max[:1],
                                              ignored[:1], 0, pool_match[t:t + 1], pod_class[idx])["bin_of"]
    S = bcc.pool_bins(one, req, o["acc_pool"], units)

    def check(g, retire):
        assert_fulfill_equal(g, o, "retire=%d" % retire)
        return check_report(engine, S, req, retire, "retire=%d" % retire)
    run_both(engine, lambda: engine.fulfill_pending_sel(engine.dev(req, torch.float64), P, units, actual, pool_max,
                                                        ignored, 0, engine.dev(pod_class, torch.uint8), pool_match, 2),
             check)


def _u64_dev(engine, a):
    return engine.dev(np.ascontiguousarray(a, np.uint64).view(np.int64), torch.int64)


@pytest.mark.parametrize("name,blocked", [("hole_LDL", False), ("last_live_dies_first", False),
                                          ("hole_LDL", True), ("only_warp7_live", True)])
def test_chain_case_anti_affinity(engine, oracle_mod, name, blocked):
    """fulfill_pending_aa (the AA bin kernels, whose shared memory puts the retirement minimum after the AA arrays).
    Zero masks: the same answer and the same report as the plain path.  Blocked: the openers of every second live
    bin carry term 0 and every probe matches it, so those live bins refuse the probes, which the chain passes on
    through them to later live bins"""
    c = CHAIN[name]
    req = c["req"]
    P = len(req)
    carries = np.zeros(P, np.uint64)
    if blocked:
        opened = np.nonzero(req[:, 0] == bcc.LIVE)[0]
        carries[opened[::2]] = 1
        carries[req[:, 0] == bcc.PROBE] = 1
    matches = carries.copy()
    args = (np.zeros(1, np.int32), np.array([BIG], np.int32), np.zeros(1, np.uint8), 0)
    unit = c["unit"].reshape(1, -1)
    o = aa_oracle.fulfill_pending_aa(req, P, unit, *args, carries, matches)
    if not blocked:
        np.testing.assert_array_equal(o["bin_of"], oracle_mod.fulfill_pending(req, P, unit, *args)["bin_of"])
    S = {0: bcc.remaining(req, o["bin_of"], c["unit"])}

    def check(g, retire):
        assert_fulfill_equal(g, o, "retire=%d" % retire)
        return check_report(engine, S, req, retire, "retire=%d" % retire)
    rep = run_both(engine, lambda: engine.fulfill_pending_aa(engine.dev(req, torch.float64), P, unit, *args,
                                                             _u64_dev(engine, carries), _u64_dev(engine, matches)),
                   check, c["knobs"])
    assert all(r["form"] == 0 for r in rep[0][0] if r["pass"] == 1)
    if not blocked:  # the plain path reports the same (its form may differ in the streaming mode)
        plain = pack(engine, oracle_mod, req, c["unit"], c["knobs"])["report"]
        if all(r["form"] == 0 for r in plain[0]):
            assert plain[1] == rep[0][1]


# ---------------------------------------------------------------------------------------------------------------------
# scale_up: nodes take the first pods, the rest is packed by the chained first bin pass
# ---------------------------------------------------------------------------------------------------------------------
def scale_up_inputs(c, node_min=None):
    """4 nodes of 30 in the pattern dimension take 12 pods of 10 placed in front of the case's pods (node_min: one
    more node of that size takes one pod of node_min, which then is the call's minimum of that dimension); an
    infeasible pod (more pods than a bin holds) sits among them"""
    D = c["req"].shape[1]
    head = bcc.rows([10.0] * 12, D)
    caps = [np.where(np.arange(D) == 0, 30.0, 1000.0)]
    n_type = [0] * 4
    if node_min is not None:
        head = np.concatenate([head, bcc.rows([node_min], D)])
        caps.append(np.where(np.arange(D) == 0, node_min, 1000.0))
        n_type.append(1)
    bad = bcc.rows([5.0], D)
    bad[0, bcc.PODS_COL] = 500.0
    req = np.concatenate([head, bad, c["req"]])
    unit = c["unit"].reshape(1, -1)
    N = len(n_type)
    return {"req": req, "P": len(req), "unit_all": unit, "unit_ordered": unit, "pool_actual": np.zeros(1, np.int32),
            "pool_max": np.array([BIG], np.int32), "pool_ignored": np.zeros(1, np.uint8), "over_provision": 0,
            "cap_type": np.stack(caps), "node_type": np.array(n_type, np.int32), "used0": np.zeros((N, D))}


def oracle_scale_up_bins(oracle_mod, s):
    from test_gpu_parity import oracle_scale_up
    used = s["used0"].copy()
    o = oracle_scale_up(oracle_mod, s, used)
    pend = np.nonzero(o["placed"] == -1)[0]
    f = oracle_mod.fulfill_pending(s["req"][pend], len(pend), s["unit_ordered"], s["pool_actual"], s["pool_max"],
                                   s["pool_ignored"], 0)
    return o, used, {0: bcc.remaining(s["req"][pend], f["bin_of"], s["unit_ordered"][0])}


def assert_tick_equal(g, o, used, used_o, label):
    for k in ("feasible", "placed", "acc_pool"):
        v = g[k] if isinstance(g[k], np.ndarray) else to_np(g[k])
        np.testing.assert_array_equal(v, o[k], err_msg="%s: %s" % (label, k))
    for k in ("new_size", "units_needed", "bins_opened"):
        np.testing.assert_array_equal(g[k], o[k], err_msg="%s: %s" % (label, k))
    for k in ("n_to_schedule", "n_pending", "num_unaccounted", "decisions"):
        assert g[k] == o[k], (label, k)
    np.testing.assert_array_equal(used, used_o, err_msg=label + ": used")


@pytest.mark.parametrize("name,node_min", [("hole_LDL", None), ("last_live_dies_first", None),
                                           ("retired_then_placing", None), ("min_from_infeasible_row", None),
                                           ("only_warp0_live", 2.0)])
def test_chain_case_scale_up(engine, oracle_mod, request, name, node_min):
    """scale_up, scale_up_host, scale_up_sel and scale_up_sel_host (trivial selectors); the device entry chains the
    first bin pass behind the node pass (record chained == 1), and once more with an injected chain timeout, whose
    unchained redo must give the same answer and the same report.  node_min: the call's minimum of the pattern
    dimension comes from a pod a node takes, which the bin pass never sees: fewer bins die, answers stay exact"""
    c = CHAIN[name]
    s = scale_up_inputs(c, node_min)
    o, used_o, S = oracle_scale_up_bins(oracle_mod, s)
    assert (o["placed"] >= 0).sum() == 12 + (node_min is not None)
    assert (o["feasible"] == 0).sum() == 1 + (name == "min_from_infeasible_row")
    req, D = s["req"], s["req"].shape[1]
    args = (s["unit_all"], s["unit_ordered"], s["pool_actual"], s["pool_max"], s["pool_ignored"], 0)
    P, N = s["P"], len(s["node_type"])
    sel = (np.zeros(P, np.uint8), np.full(N, np.iinfo(np.uint64).max, np.uint64), np.ones(1, np.uint64),
           np.ones(1, np.uint64), 1)
    dev_used = {}

    def dev_call(kind):
        def call():
            dev_used["u"] = engine.dev(s["used0"], torch.float64)
            a = (engine.dev(req, torch.float64),) + args + (engine.dev(s["cap_type"], torch.float64),
                                                            engine.dev(s["node_type"], torch.int32), dev_used["u"])
            if kind == "sel":
                return engine.scale_up_sel(*a, engine.dev(sel[0], torch.uint8), _u64_dev(engine, sel[1]), *sel[2:])
            return engine.scale_up(*a)
        return call

    def host_call(kind):
        def call():
            dev_used["u"] = s["used0"].copy()
            a = (req,) + args + (s["cap_type"], s["node_type"], dev_used["u"])
            if kind == "sel":
                return engine.scale_up_sel_host(*a, *sel)
            return engine.scale_up_host(*a)
        return call

    for label, call, knobs in (("scale_up", dev_call("plain"), {}),
                               ("scale_up redo", dev_call("plain"), {"inject_chain_timeout": 1}),
                               ("scale_up_sel", dev_call("sel"), {}),
                               ("scale_up_host", host_call("plain"), {}),
                               ("scale_up_sel_host", host_call("sel"), {})):

        def check(g, retire, label=label):
            u = dev_used["u"] if isinstance(dev_used["u"], np.ndarray) else to_np(dev_used["u"])
            assert_tick_equal(g, o, u, used_o, "%s retire=%d" % (label, retire))
            return check_report(engine, S, req, retire, "%s retire=%d" % (label, retire), redone="redo" in label)
        rep = run_both(engine, call, check, {**c["knobs"], **knobs})
        recs = rep[0][0]
        if label == "scale_up":
            assert [r["chained"] for r in recs if r["pass"] == 1][0] == 1, recs
            chained_rep = rep[0][1]
        if label == "scale_up redo":
            assert [r["chained"] for r in recs if r["pass"] == 1][:2] == [1, 0], recs
            assert rep[0][1] == chained_rep, (rep[0][1], chained_rep)
