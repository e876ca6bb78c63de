"""`-m gpu`: the pod-affinity entry points (acsfit_first_fit_nodes_pa, acsfit_fulfill_pending_pa) against the plain-C
oracle (tests/pa_oracle.c), exactly -- placements, used bits, node masks, pool sizes, units, bins opened, accounted
pool, bin of each pod, counters and the flips the reruns fixed -- on the ticks of tests/aa_cases.py and the rank-layout
ticks of tests/variant_cases.py with affinity masks added, under both candidate scans and several pipeline schedules; the refusals; and the host layer end to end (Cluster.loop_logic) with the switch off and on."""
import functools

import numpy as np
import pytest
import torch

import aa_cases as ac
import pa_oracle
import variant_cases as vc

pytestmark = pytest.mark.gpu

SCHEDULES = {
    "default": {},
    "waves_prune": {"min_stages": 1 << 20, "prune": 1},
    "waves_noprune": {"min_stages": 1 << 20, "prune": 0},
    "multipass": {"bin_pass_stages": 2, "min_stages": 32},
    "no_retire": {"retire": 0},
}
DEFAULT_KNOBS = {"min_stages": 0, "prune": -1, "overlap": 1, "bin_pass_stages": 0, "retire": 1}
F64, I32, U8, I64 = torch.float64, torch.int32, torch.uint8, torch.int64
U64 = np.uint64
# affinity overlays: (signatures, share of pods with one, self-affine share, signatures present on the nodes)
PA_KINDS = {
    "none": (0, 0.0, 0.0, "none"),        # every affinity mask 0
    "sig1": (1, 0.3, 0.8, "none"),        # one self-affine group, absent at first: one flip
    "sig2": (2, 0.3, 0.8, "none"),        # two: two flips in turn
    "present": (8, 0.3, 0.8, "all"),      # every signature on some node already: no rerun
    "mixed": (8, 0.3, 0.6, "even"),       # half present, half bootstrapped; other pods match too
    "blocked": (4, 0.2, 0.0, "none"),     # nobody matches: every pod with a signature is blocked everywhere
    "bits64": (64, 0.5, 0.7, "even"),     # 64 signatures
}


def to_np(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def i64(a):
    return np.ascontiguousarray(a, dtype=U64).view(np.int64)


def pa_overlay(c, kind, seed=0):
    c = dict(c)
    S, share, selfish, present = PA_KINDS[kind]
    rng = np.random.default_rng(seed + 17)
    P, N = len(c["req"]), len(c["node_type"])
    req, match, has = np.zeros(P, U64), np.zeros(P, U64), np.zeros(N, U64)
    if S:
        who = np.nonzero(rng.random(P) < share)[0]
        g = rng.integers(0, S, size=len(who)).astype(U64)
        req[who] = U64(1) << g
        own = rng.random(len(who)) < selfish
        match[who[own]] |= U64(1) << g[own]
        if kind != "blocked":  # some pods without a signature match one (they can end a bootstrap early)
            other = np.nonzero(rng.random(P) < 0.05)[0]
            match[other] |= U64(1) << rng.integers(0, S, size=len(other)).astype(U64)
        sigs = {"all": range(S), "even": range(0, S, 2), "none": ()}[present]
        for s in sigs:
            has[int(rng.integers(N))] |= U64(1) << U64(s)
    c.update(pa_requires=req, pa_matches=match, pa_self=req & match, node_has0=has)
    return c


@functools.lru_cache(maxsize=None)
def case(base, pa_kind, D):
    c = ac.make_case(base, D) if D else ac.overlay(__import__("cluster_cases")._with_used(vc.case(base)), seed=3)
    return pa_overlay(c, pa_kind)


@functools.lru_cache(maxsize=None)
def oracle_of(base, pa_kind, D):
    return oracle_of_case(case(base, pa_kind, D))


def oracle_of_case(c, pod_idx=None):
    """the oracle over the req rows `pod_idx` in that order (None: every row); placements and flips are in list
    positions, and "pend" holds the req rows of the pods left pending, in list order"""
    used, nc, nx, has = c["used0"].copy(), c["node_carries0"].copy(), c["node_matches0"].copy(), c["node_has0"].copy()
    rows = np.arange(len(c["req"])) if pod_idx is None else np.asarray(pod_idx)
    placed, calls, flips = pa_oracle.first_fit_nodes_pa(
        c["req"][rows], c["cap_type"], c["node_type"], used, c["pa_requires"][rows], c["pa_self"][rows],
        c["pa_matches"][rows], has, c["pod_carries"][rows], c["pod_matches"][rows], nc, nx, c.get("node_match"),
        None if "pod_class" not in c else c["pod_class"][rows])
    pend = rows[placed < 0]
    present = int(np.bitwise_or.reduce(has)) if len(has) else 0
    f = pa_oracle.fulfill_pending_pa(c["req"][pend], len(pend) + 3, c["unit"], c["pool_actual"], c["pool_max"],
                                     c["pool_ignored"], c["over_provision"], c["pa_requires"][pend],
                                     c["pa_self"][pend], c["pa_matches"][pend], present, c["pod_carries"][pend],
                                     c["pod_matches"][pend], c.get("pool_match"),
                                     None if "pod_class" not in c else c["pod_class"][pend])
    return {"placed": placed, "decisions": calls, "used": used, "nc": nc, "nx": nx, "has": has, "flips": flips,
            "pend": pend, "present": present, "fulfill": f}


def run(engine, c, pend, present, knobs, with_aa=True, pod_idx=None):
    """the node pass over the req rows `pod_idx` (None: every row), then the bin pass over the rows `pend`"""
    try:
        for k, v in knobs.items():
            engine.set_knob(k, v)
        sel = "pod_class" in c
        d_used = engine.dev(c["used0"], F64)
        d_nc, d_nx = engine.dev(i64(c["node_carries0"]), I64), engine.dev(i64(c["node_matches0"]), I64)
        d_has = engine.dev(i64(c["node_has0"]), I64)
        aa = (engine.dev(i64(c["pod_carries"]), I64), engine.dev(i64(c["pod_matches"]), I64), d_nc, d_nx) \
            if with_aa else ()
        p, dec = engine.first_fit_nodes_pa(
            engine.dev(c["req"], F64), None if pod_idx is None else engine.dev(pod_idx, I32),
            engine.dev(c["cap_type"], F64), engine.dev(c["node_type"], I32), d_used,
            engine.dev(i64(c["pa_requires"]), I64), engine.dev(i64(c["pa_self"]), I64),
            engine.dev(i64(c["pa_matches"]), I64), d_has, *aa,
            **(dict(pod_class=engine.dev(c["pod_class"], U8), node_match=engine.dev(i64(c["node_match"]), I64),
                    classes=c["classes"]) if sel else {}))
        node_flips = engine.last_affinity_reruns()
        aa_b = (engine.dev(i64(c["pod_carries"][pend]), I64), engine.dev(i64(c["pod_matches"][pend]), I64)) \
            if with_aa else (None, None)
        f = engine.fulfill_pending_pa(
            engine.dev(c["req"][pend], F64), len(pend) + 3, c["unit"], c["pool_actual"], c["pool_max"],
            c["pool_ignored"], c["over_provision"], engine.dev(i64(c["pa_requires"][pend]), I64),
            engine.dev(i64(c["pa_self"][pend]), I64), engine.dev(i64(c["pa_matches"][pend]), I64), present, *aa_b,
            *((engine.dev(c["pod_class"][pend], U8), c["pool_match"], c["classes"]) if sel else ()))
        torch.cuda.synchronize()
        bin_flips = engine.last_affinity_reruns()
        return {"placed": to_np(p), "decisions": int(to_np(dec)[0]), "used": to_np(d_used),
                "nc": to_np(d_nc).view(U64), "nx": to_np(d_nx).view(U64), "has": to_np(d_has).view(U64),
                "flips": node_flips,
                "fulfill": dict({k: to_np(v) if isinstance(v, torch.Tensor) else v for k, v in f.items()},
                                flips=bin_flips)}
    finally:
        for k, v in DEFAULT_KNOBS.items():
            engine.set_knob(k, v)


def assert_equal(g, o, with_aa=True):
    np.testing.assert_array_equal(g["placed"], o["placed"])
    assert g["decisions"] == o["decisions"]
    np.testing.assert_array_equal(g["used"].view(U64), o["used"].view(U64))
    np.testing.assert_array_equal(g["has"], o["has"])
    if with_aa:
        np.testing.assert_array_equal(g["nc"], o["nc"])
        np.testing.assert_array_equal(g["nx"], o["nx"])
    assert g["flips"] == o["flips"]
    for k, v in o["fulfill"].items():
        np.testing.assert_array_equal(np.asarray(g["fulfill"][k]), np.asarray(v), err_msg=k)


@pytest.fixture(scope="module")
def eng():
    """one engine for the module; each case runs under both candidate scans (packed ranks and float64) inside the
    test.  The pod-affinity entry points ignore the streaming knob (barrier form only), so it is not varied."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from kubernetes_acs_engine_autoscaler_b200 import build as acs_build
    acs_build.build()
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    e = Engine(0, watchdog_ms=15000)
    e.set_knob("stream", 0)
    yield e
    e.close()


def check(eng, base, pa_kind, D, schedules=("default",), scans=(1, 0)):
    c, o = case(base, pa_kind, D), oracle_of(base, pa_kind, D)
    try:
        for ranks in scans:
            eng.set_knob("ranks", ranks)
            for schedule in schedules:
                assert_equal(run(eng, c, o["pend"], o["present"], SCHEDULES[schedule]), o)
    finally:
        eng.set_knob("ranks", 1)
    return c, o


@pytest.mark.parametrize("D", ac.DIMS)
@pytest.mark.parametrize("pa_kind", sorted(PA_KINDS))
def test_pa_matches_oracle(eng, pa_kind, D):
    _, o = check(eng, "with_sel" if pa_kind in ("mixed", "bits64") else "replicas", pa_kind, D)
    if pa_kind == "present":
        assert o["flips"] == [] and o["fulfill"]["flips"] == []  # no bootstrap signature: nothing rerun
    if pa_kind in ("sig1", "sig2"):
        assert len(o["flips"]) == int(pa_kind[-1])  # one rerun per self-affine group, in turn


@pytest.mark.parametrize("pa_kind", ["sig2", "mixed", "blocked"])
def test_pa_schedules(eng, pa_kind):
    check(eng, "with_sel" if pa_kind == "mixed" else "replicas", pa_kind, 4,
          schedules=sorted(set(SCHEDULES) - {"default"}), scans=(1,))


@pytest.mark.parametrize("base,pa_kind", [("zero", "sig2"), ("edges", "mixed"), ("all_blocked", "sig2"),
                                          ("all_blocked", "mixed"), ("symmetric", "blocked")])
def test_pa_with_and_without_anti_affinity(eng, base, pa_kind):
    c, o = check(eng, base, pa_kind, 4)
    if base == "all_blocked":  # the node pass places nothing, so the bootstraps happen in the bins
        assert o["flips"] == [] and len(o["fulfill"]["flips"]) >= 2
    if base == "zero":  # all anti-affinity masks 0: the call without `aa` gives the same
        assert_equal(run(eng, c, o["pend"], o["present"], {}, with_aa=False), o, with_aa=False)


@pytest.mark.parametrize("name", ["d2_rw1_u8192", "d4_rw1_guard31", "d8_rw3_padded", "d16_f64_width"])
def test_pa_layouts_match_oracle(eng, name):
    check(eng, name, "mixed", 0, schedules=("default", "multipass"), scans=(1,))


def test_none_equals_anti_affinity_entry_points(eng):
    c, o = case("replicas", "none", 4), oracle_of("replicas", "none", 4)
    g = run(eng, c, o["pend"], 0, {})
    assert g["flips"] == [] and g["fulfill"]["flips"] == []
    d_used = eng.dev(c["used0"], F64)
    d_nc, d_nx = eng.dev(i64(c["node_carries0"]), I64), eng.dev(i64(c["node_matches0"]), I64)
    p, dec = eng.first_fit_nodes_aa(eng.dev(c["req"], F64), None, eng.dev(c["cap_type"], F64),
                                    eng.dev(c["node_type"], I32), d_used, eng.dev(i64(c["pod_carries"]), I64),
                                    eng.dev(i64(c["pod_matches"]), I64), d_nc, d_nx)
    np.testing.assert_array_equal(to_np(p), g["placed"])
    assert int(to_np(dec)[0]) == g["decisions"]
    np.testing.assert_array_equal(to_np(d_used).view(U64), g["used"].view(U64))


def test_flips_and_blocked_pods_through_many_bin_passes(eng):
    # every other pod requires a signature nobody matches: blocked in every bin; with one stage per bin pass the
    # blocked pods ride through pass after pass until one places nothing, and the call returns cleanly
    c = pa_overlay(ac.make_case("replicas", 2), "blocked")
    o = oracle_of("replicas", "blocked", 2)
    g = run(eng, c, o["pend"], o["present"], {"bin_pass_stages": 1, "min_stages": 32})
    assert_equal(g, o)
    assert o["fulfill"]["num_unaccounted"] > 3
    assert_equal(run(eng, c, o["pend"], o["present"], {}), o)  # the next call still matches


def test_refusals(eng):
    from kubernetes_acs_engine_autoscaler_b200._native import AcsfitError, E_INVALID
    c, o = case("replicas", "sig1", 4), oracle_of("replicas", "sig1", 4)
    req, cap, nt = eng.dev(c["req"], F64), eng.dev(c["cap_type"], F64), eng.dev(c["node_type"], I32)
    r, s, m = (eng.dev(i64(c[k]), I64) for k in ("pa_requires", "pa_self", "pa_matches"))
    has = eng.dev(i64(c["node_has0"]), I64)
    two_bits = eng.dev(i64(c["pa_requires"] | U64(6)), I64)
    bad_calls = [
        lambda: eng.first_fit_nodes_pa(req, None, cap, nt, eng.dev(c["used0"], F64), None, s, m, has),
        lambda: eng.first_fit_nodes_pa(req, None, cap, nt, eng.dev(c["used0"], F64), r, s, m, None),
        lambda: eng.first_fit_nodes_pa(req, None, cap, nt, eng.dev(c["used0"], F64), two_bits, s, m, has),
        lambda: eng.fulfill_pending_pa(req, len(c["req"]), c["unit"], c["pool_actual"], c["pool_max"],
                                       c["pool_ignored"], 1, r, None, m),
    ]
    for call in bad_calls:
        with pytest.raises(AcsfitError) as e:
            call()
        assert e.value.status == E_INVALID
    assert_equal(run(eng, c, o["pend"], o["present"], {}), o)  # the next call still matches the oracle


# ---------------------------------------------------------------- through Cluster.loop_logic
import golden_util as gu  # noqa: E402

# a few of the recorded reference ticks (the anti-affinity and selector tests replay all of them)
TICKS = [s for s in gu.load_json("ticks.json.gz")
         if s["name"] in ("config1_16x4_dry_run", "random_1000", "crowded_2001", "duplicate_uids", "no_nodes")]


@pytest.fixture()
def host(tmp_path, monkeypatch, eng):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", eng)
    return monkeypatch


def tick(state, engine, on):
    from test_gpu_selector_states import tick as tick2
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_POD_AFFINITY", on)
        return tick2(state, engine, "0", "0")


@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_switch_without_terms_is_the_reference_tick(host, eng, state):
    off = tick(state, eng, "0")
    on = tick(state, eng, "1")
    gu.assert_tick_matches(off, state["expected"])
    gu.assert_tick_matches(on, state["expected"])
    assert on["launches"] == off["launches"]


def affinity_state(full, cache_running):
    """pool `agentpool1` (Standard_D2_v2): one node, full (`full`) or with room for three 0.3-cpu pods.  Three pending
    `web` pods, each needing a pod labelled app=cache on its node (required affinity, hostname topology);
    `cache_running` puts such a pod on the node, otherwise the web pods are labelled app=cache themselves
    (self-affine replicas)."""
    name = "k8s-agentpool1-16334397-0"
    node = {"metadata": {"name": name, "creationTimestamp": "2016-08-25T05:13:16Z",
                         "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2", "agentpool": "agentpool1",
                                    "failure-domain.beta.kubernetes.io/region": "southcentralus",
                                    "kubernetes.io/hostname": name}}, "spec": {}}
    aff = {"podAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
        {"topologyKey": "kubernetes.io/hostname", "labelSelector": {"matchLabels": {"app": "cache"}}}]}}

    def pod(n, cpu, labels, phase="Pending", node_name=None, affinity=None):
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": cpu}}}]}
        if node_name:
            spec["nodeName"] = node_name
        if affinity:
            spec["affinity"] = affinity
        return {"metadata": {"name": n, "namespace": "default", "uid": "uid-" + n, "labels": labels,
                             "creationTimestamp": "2026-09-20T07:00:00Z"}, "spec": spec, "status": {"phase": phase}}
    pods = [pod("web-%d" % i, "300m", {"app": "web" if cache_running else "cache"}, affinity=aff) for i in range(3)]
    pods.append(pod("cache", "1900m" if full else "100m", {"app": "cache" if cache_running else "other"},
                    "Running", name))
    return {"name": "pod_affinity", "now": "2026-09-21T12:00:00Z", "nodes": [node], "pods": pods,
            "arm_parameters": {"masterVMSize": {"value": "Standard_D2_v2"}, "firstConsecutiveStaticIP": {"value": "10.0.0.1"},
                               "agentpool1VMSize": {"value": "Standard_D2_v2"}},
            "settings": {"idle_threshold": 1800, "spare_agents": 0, "over_provision": 1, "dry_run": True,
                         "ignore_pools": ""}}


def test_web_beside_a_cache_on_a_full_node_scales_nothing(host, eng, monkeypatch):
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    monkeypatch.setattr(Scaler, "REFERENCE_RAISE_ON_INSUFFICIENT", False)  # notify and scale the rest
    s = affinity_state(full=True, cache_running=True)
    off = tick(s, eng, "0")
    on = tick(s, eng, "1")
    assert off["exception"] is None and on["exception"] is None
    # off: the web pods look placeable in a new node; on: no node or new node holds a cache pod
    assert off["scale_pools_calls"] == [{"agentpool1": 1 + 1 + 1}]
    assert on["scale_pools_calls"] in ([], [{"agentpool1": 1 + 1}])
    assert any("required pod affinity" in m for _, _, m in on["log"])


def test_self_affine_replicas_share_the_node(host, eng):
    s = affinity_state(full=False, cache_running=False)
    node = s["nodes"][0]["metadata"]["name"]
    on = tick(s, eng, "1")
    assert on["exception"] is None
    assert float.fromhex(on["used"][node]["pods"]) == 4.0 and on["scale_pools_calls"] == []
