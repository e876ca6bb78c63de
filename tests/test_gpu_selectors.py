"""`-m gpu`: the node-selector entry points (acsfit_*_sel) against the plain-C selector oracle (tests/sel_oracle.c),
exactly, on the adversarial ticks of tests/selector_cases.py, under the engine fixture's three scan modes and
several pipeline schedules; the chained node + first-bin-pass launch and its watchdog redo; and the host layer's
promise that the mode changes nothing for pods without selectors."""
import functools
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import sel_oracle
import selector_cases as sc

pytestmark = pytest.mark.gpu

SCHEDULES = {
    "default": {},
    "waves": {"min_stages": 1 << 20},                 # more stage CTAs than the GPU holds: the PRUNE form
    "waves_noprune": {"min_stages": 1 << 20, "prune": 0},
    "unchained": {"overlap": 0},
    "multipass": {"bin_pass_stages": 2, "min_stages": 32},
}
DEFAULT_KNOBS = {"min_stages": 0, "prune": -1, "overlap": 1, "bin_pass_stages": 0, "inject_chain_timeout": 0}
F64, I32, U8 = torch.float64, torch.int32, torch.uint8


def to_np(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


@functools.lru_cache(maxsize=None)
def case_and_oracle(kind, D):
    c = sc.make_case(kind, D)
    used_o = c["used0"].copy()
    return c, sel_oracle.scale_up_sel(c, used_o), used_o


def eligible_for_first_pool(c, o):
    """count_ineligible == 0: every pod to schedule matches the first pool visited and fits its unit"""
    t0 = 0
    f = np.nonzero(o["feasible"])[0]
    match = (c["pool_match_ordered"][t0] >> c["pod_class"][f].astype(np.uint64)) & np.uint64(1)
    fits = (c["unit_ordered"][t0][None, :] - c["req"][f] >= 0).all(axis=1)
    return bool(len(f)) and bool(match.all()) and bool(fits.all())


def run_sel(engine, c, knobs):
    try:
        for k, v in knobs.items():
            engine.set_knob(k, v)
        d_used = engine.dev(c["used0"], F64)
        g = engine.scale_up_sel(engine.dev(c["req"], F64), c["unit_all"], c["unit_ordered"], c["pool_actual"],
                                c["pool_max"], c["pool_ignored"], c["over_provision"], engine.dev(c["cap_type"], F64),
                                engine.dev(c["node_type"], I32), d_used, engine.dev(c["pod_class"], U8),
                                engine.dev(c["node_match"].view(np.int64), torch.int64), c["pool_match_all"],
                                c["pool_match_ordered"], c["classes"])
        torch.cuda.synchronize()
        g["sel_hits"] = engine.last_sel_hits()
        return g, to_np(d_used), engine.last_launches()
    finally:
        for k, v in DEFAULT_KNOBS.items():
            engine.set_knob(k, v)


def assert_tick_equal(g, o, used, used_o):
    for k in ("feasible", "placed", "acc_pool", "new_size", "units_needed", "bins_opened"):
        np.testing.assert_array_equal(to_np(g[k]), np.asarray(o[k]), err_msg=k)
    for k in ("n_to_schedule", "n_pending", "num_unaccounted", "decisions"):
        assert g[k] == o[k], k
    np.testing.assert_array_equal(used.view(np.uint64), used_o.view(np.uint64))


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("D", sc.DIMS)
@pytest.mark.parametrize("kind", sc.KINDS)
def test_scale_up_sel_matches_oracle(request, engine, kind, D, schedule):
    c, o, used_o = case_and_oracle(kind, D)
    g, used, recs = run_sel(engine, c, SCHEDULES[schedule])
    assert_tick_equal(g, o, used, used_o)
    # the scans' match filter: a pod placed on a node was a scan hit in that node's stage, and a pod that matches no
    # node is never one (the resolver's own match test would still place every pod right without the filter)
    assert g["sel_hits"] >= int((o["placed"] >= 0).sum())
    if kind == "all_mismatched":
        assert g["sel_hits"] == 0
    nodes = [r for r in recs if r["pass"] == 0]
    assert nodes and all(r["form"] == 0 for r in nodes)  # selector node passes run the barrier form, "stream" or not
    for r in nodes:  # automatic pruning: exactly when the pass has more stages than the GPU holds at once
        assert r["prune"] == (0 if schedule == "waves_noprune" else int(r["stages"] > r["resident"]))
    chained = any(r["chained"] for r in recs)
    elig = eligible_for_first_pool(c, o)
    if chained:
        assert elig and schedule != "unchained"
    if elig and schedule == "default" and D <= 4:  # two stage CTAs per SM leave room for the chained bin stages
        assert chained


@pytest.mark.parametrize("D", sc.DIMS)
@pytest.mark.parametrize("kind", sc.KINDS)
def test_entry_points_match_oracle(engine, kind, D):
    c, o, used_o = case_and_oracle(kind, D)
    req = engine.dev(c["req"], F64)
    pc = engine.dev(c["pod_class"], U8)
    # feasibility
    m, ev = engine.feasible_mask_sel(req, engine.dev(c["unit_all"], F64), pc, c["pool_match_all"], c["classes"])
    mo, evo = sel_oracle.feasible_mask_sel(c["req"], c["unit_all"], c["pool_match_all"], c["pod_class"])
    np.testing.assert_array_equal(to_np(m), mo)
    assert int(to_np(ev)[0]) == evo
    # first fit over the feasible pods, through pod_idx (pod_class stays indexed by req row)
    idx = np.nonzero(mo)[0].astype(np.int32)
    d_used = engine.dev(c["used0"], F64)
    p, dec = engine.first_fit_nodes_sel(req, engine.dev(idx, I32), engine.dev(c["cap_type"], F64),
                                        engine.dev(c["node_type"], I32), d_used, pc,
                                        engine.dev(c["node_match"].view(np.int64), torch.int64), c["classes"])
    u = c["used0"].copy()
    po, deco = sel_oracle.first_fit_nodes_sel(c["req"][idx], c["cap_type"], c["node_type"], u, c["node_match"],
                                              c["pod_class"][idx])
    np.testing.assert_array_equal(to_np(p), po)
    assert int(to_np(dec)[0]) == deco
    np.testing.assert_array_equal(to_np(d_used).view(np.uint64), u.view(np.uint64))
    # bin packing of the pending pods
    pend = idx[po < 0]
    if len(pend):
        f = engine.fulfill_pending_sel(engine.dev(c["req"][pend], F64), len(pend), c["unit_ordered"], c["pool_actual"],
                                       c["pool_max"], c["pool_ignored"], 1, engine.dev(c["pod_class"][pend], U8),
                                       c["pool_match_ordered"], c["classes"])
        fo = sel_oracle.fulfill_pending_sel(c["req"][pend], len(pend), c["unit_ordered"], c["pool_actual"],
                                            c["pool_max"], c["pool_ignored"], 1, c["pool_match_ordered"],
                                            c["pod_class"][pend])
        for k in fo:
            np.testing.assert_array_equal(to_np(f[k]), np.asarray(fo[k]), err_msg=k)
    # the host-buffer form of the whole tick
    used_h = c["used0"].copy()
    h = engine.scale_up_sel_host(c["req"], c["unit_all"], c["unit_ordered"], c["pool_actual"], c["pool_max"],
                                 c["pool_ignored"], c["over_provision"], c["cap_type"], c["node_type"], used_h,
                                 c["pod_class"], c["node_match"], c["pool_match_all"], c["pool_match_ordered"],
                                 c["classes"])
    assert_tick_equal(h, o, used_h, used_o)
    # selector-sensitive: the plain tick answers differently (except for the case without selectors)
    used_p = c["used0"].copy()
    plain = engine.scale_up_host(c["req"], c["unit_all"], c["unit_ordered"], c["pool_actual"], c["pool_max"],
                                 c["pool_ignored"], c["over_provision"], c["cap_type"], c["node_type"], used_p)
    same = all(np.array_equal(np.asarray(plain[k]), np.asarray(o[k])) for k in ("feasible", "placed", "acc_pool", "new_size"))
    assert same == (kind not in sc.SENSITIVE)


@pytest.mark.parametrize("D", (2, 4))
def test_chain_timeout_redo(engine, D):
    c, o, used_o = case_and_oracle("first_pool", D)
    assert eligible_for_first_pool(c, o)
    g, used, recs = run_sel(engine, c, {"inject_chain_timeout": 1})
    assert_tick_equal(g, o, used, used_o)
    assert any(r["chained"] for r in recs)  # the chained launch ran, was treated as timed out ...
    assert recs[-1]["chained"] == 0 and any(r["pass"] == 0 and not r["chained"] for r in recs)  # ... and was redone


def test_refusals(engine):
    c, o, _ = case_and_oracle("two_classes", 4)
    req = engine.dev(c["req"], F64)
    from kubernetes_acs_engine_autoscaler_b200._native import AcsfitError
    bad = c["pod_class"].copy()
    bad[7] = c["classes"]  # a class number >= classes
    with pytest.raises(AcsfitError):
        engine.feasible_mask_sel(req, engine.dev(c["unit_all"], F64), engine.dev(bad, U8), c["pool_match_all"],
                                 c["classes"])
    with pytest.raises(AcsfitError):  # class 0 must match every pool
        engine.feasible_mask_sel(req, engine.dev(c["unit_all"], F64), engine.dev(c["pod_class"], U8),
                                 c["pool_match_all"] & ~np.uint64(1), c["classes"])
    with pytest.raises(AcsfitError):
        engine.feasible_mask_sel(req, engine.dev(c["unit_all"], F64), engine.dev(c["pod_class"], U8),
                                 c["pool_match_all"], 65)
    d_used = engine.dev(c["used0"], F64)
    with pytest.raises(AcsfitError):  # class 0 must match every node too (checked on the device)
        engine.first_fit_nodes_sel(req, None, engine.dev(c["cap_type"], F64), engine.dev(c["node_type"], I32), d_used,
                                   engine.dev(c["pod_class"], U8),
                                   engine.dev((c["node_match"] & ~np.uint64(1)).view(np.int64), torch.int64),
                                   c["classes"])


# ---------------------------------------------------------------- host layer: the mode changes nothing without selectors
def _objects(c):
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeResource

    def res(row):
        r = KubeResource()
        r.raw = {"k%d" % d: float(v) for d, v in enumerate(row)}
        return r
    caps = [res(r) for r in c["cap_type"]]
    nodes = [SimpleNamespace(selectors=n.selectors, capacity=caps[c["node_type"][i]], used_capacity=res(c["used0"][i]))
             for i, n in enumerate(c["nodes"])]
    pods = [SimpleNamespace(selectors={}, resources=res(r)) for r in c["req"]]
    return pods, nodes


def test_mode_on_without_selectors_launches_the_plain_path(engine):
    from kubernetes_acs_engine_autoscaler_b200 import snapshot
    c, _, _ = case_and_oracle("no_selectors", 4)
    prev = snapshot._engine
    snapshot.set_engine(engine)
    try:
        runs = []
        for on in (False, True):
            pods, nodes = _objects(c)
            cls = snapshot.selector_classes(pods, nodes, c["pools"]) if on else None
            assert cls is None or cls.trivial
            n0 = engine.launch_count
            placed = snapshot.first_fit_nodes(pods, nodes, classes=cls)
            runs.append((placed, [dict(n.used_capacity.raw) for n in nodes], engine.launch_count - n0,
                         engine.last_launches()))
        assert np.array_equal(runs[0][0], runs[1][0])
        assert runs[0][1] == runs[1][1] and runs[0][2] == runs[1][2] and runs[0][3] == runs[1][3]
    finally:
        snapshot.set_engine(prev)
