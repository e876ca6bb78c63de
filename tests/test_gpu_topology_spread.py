"""`-m gpu`: the topology-spread entry points (acsfit_first_fit_nodes_ts, acsfit_fulfill_pending_ts) against the
plain-C oracle (tests/ts_oracle.c), exactly -- placements, used bits, node counts and masks, pool sizes, units, bins
opened, accounted pool, bin of each pod, counters, and the rises and flips the reruns fixed -- on the ticks of
tests/aa_cases.py and the rank-layout ticks of tests/variant_cases.py with spread keys (and pod-affinity masks) added,
under both candidate scans and several pipeline schedules; a rise at a 256-pod tile edge; the refusals; and the host
layer end to end (Cluster.loop_logic) with the switch off and on."""
import functools

import numpy as np
import pytest
import torch

import aa_cases as ac
import ts_oracle
import variant_cases as vc
from test_gpu_pod_affinity import DEFAULT_KNOBS, SCHEDULES, i64, pa_overlay, to_np

pytestmark = pytest.mark.gpu

F64, I32, U8, I64 = torch.float64, torch.int32, torch.uint8, torch.int64
U64 = np.uint64
INT32_MAX = 2 ** 31 - 1
MAX_SPREAD_RISES = 4096  # the rises one node pass follows (kMaxSpreadRises in csrc/acsfit.cu)
# spread overlays: (keys, share of pods with a key, domain nodes per key (0: all), start counts, floor)
TS_KINDS = {
    "none": (0, 0.0, 0, "zero", "max"),        # no key: the pod-affinity results
    "flat": (6, 0.1, 0, "zero", "zero"),       # 10 % of the pods in groups, a master holds every minimum at 0
    "rise1": (1, 0.4, 3, "zero", "one"),       # one key over 3 nodes whose floor allows one rise
    "rises": (1, 0.4, 3, "zero", "max"),       # ... and no floor: several rises
    "pinned": (3, 0.3, 4, "one", "max"),       # three keys, every domain already at 1: the minimums start at 1
    "keys64": (64, 0.6, 0, "some", "mixed"),   # 64 keys over every node
}


def ts_overlay(c, kind, seed=0):
    c = dict(c)
    K, share, dom, start, floor = TS_KINDS[kind]
    rng = np.random.default_rng(seed + 29)
    P, N = len(c["req"]), len(c["node_type"])
    key, skew, match = np.full(P, 0xFF, np.uint8), np.zeros(P, np.int32), np.zeros(P, U64)
    count, domain = np.zeros((K, N), np.int32), np.zeros(N, U64)
    if K:
        who = np.nonzero(rng.random(P) < share)[0]
        g = rng.integers(0, K, size=len(who))
        key[who] = g
        own = rng.random(len(who)) < 0.85  # most pods select themselves
        match[who[own]] |= U64(1) << g[own].astype(U64)
        other = np.nonzero(rng.random(P) < 0.03)[0]  # some pods without a key are selected too
        match[other] |= U64(1) << rng.integers(0, K, size=len(other)).astype(U64)
        skew[who] = rng.integers(1, 3, size=len(who)) - own
        # a small domain set is taken where the group's pods land without the rule, so that its minimum can rise
        free = _placed_without_spread(c)
        for k in range(K):
            if dom:
                landed = np.bincount(free[who[(g == k) & (free[who] >= 0)]], minlength=N)
                nodes = np.argsort(-landed, kind="stable")[:dom]
            else:
                nodes = np.arange(N)
            domain[nodes] |= U64(1) << U64(k)
            if start == "one":
                count[k, nodes] = 1
            elif start == "some":
                count[k, rng.integers(0, N, size=N // 4)] = rng.integers(1, 3, size=N // 4)
        fl = {"zero": 0, "one": 1, "max": INT32_MAX}
        c["ts_floor"] = np.asarray([fl[floor] if floor in fl else (0, 1, INT32_MAX)[k % 3] for k in range(K)],
                                   np.int32)
    else:
        c["ts_floor"] = np.zeros(0, np.int32)
    c.update(ts_keys=K, ts_key=key, ts_skew=skew, ts_matches=match, ts_count0=count, ts_domain=domain)
    return c


def _placed_without_spread(c):
    P, N = len(c["req"]), len(c["node_type"])
    z = np.zeros(P, U64)
    placed, _, _, _ = ts_oracle.first_fit_nodes_ts(
        c["req"], c["cap_type"], c["node_type"], c["used0"].copy(), 0, np.full(P, 0xFF, np.uint8),
        np.zeros(P, np.int32), z, np.zeros((0, N), np.int32), np.zeros(N, U64), np.zeros(0, np.int32),
        c["pa_requires"], c["pa_self"], c["pa_matches"], c["node_has0"].copy(), c["pod_carries"], c["pod_matches"],
        c["node_carries0"].copy(), c["node_matches0"].copy(), c.get("node_match"), c.get("pod_class"))
    return placed


@functools.lru_cache(maxsize=None)
def case(base, ts_kind, pa_kind, D):
    c = ac.make_case(base, D) if D else ac.overlay(__import__("cluster_cases")._with_used(vc.case(base)), seed=3)
    return ts_overlay(pa_overlay(c, pa_kind), ts_kind)


def oracle_of_case(c, pod_idx=None):
    """the oracle over the req rows `pod_idx` in that order (None: every row); placements, flips and rises are in list
    positions, and "pend" holds the req rows of the pods left pending, in list order"""
    used, nc, nx, has = c["used0"].copy(), c["node_carries0"].copy(), c["node_matches0"].copy(), c["node_has0"].copy()
    count = c["ts_count0"].copy()
    rows = np.arange(len(c["req"])) if pod_idx is None else np.asarray(pod_idx)
    placed, calls, flips, rises = ts_oracle.first_fit_nodes_ts(
        c["req"][rows], c["cap_type"], c["node_type"], used, c["ts_keys"], c["ts_key"][rows], c["ts_skew"][rows],
        c["ts_matches"][rows], count, c["ts_domain"], c["ts_floor"], c["pa_requires"][rows], c["pa_self"][rows],
        c["pa_matches"][rows], has, c["pod_carries"][rows], c["pod_matches"][rows], nc, nx, c.get("node_match"),
        None if "pod_class" not in c else c["pod_class"][rows], follow=MAX_SPREAD_RISES)
    pend = rows[placed < 0]
    present = int(np.bitwise_or.reduce(has)) if len(has) else 0
    f = ts_oracle.fulfill_pending_ts(c["req"][pend], len(pend) + 3, c["unit"], c["pool_actual"], c["pool_max"],
                                     c["pool_ignored"], c["over_provision"], c["ts_keys"], c["ts_key"][pend],
                                     c["ts_skew"][pend], c["ts_matches"][pend], c["pa_requires"][pend],
                                     c["pa_self"][pend], c["pa_matches"][pend], present, c["pod_carries"][pend],
                                     c["pod_matches"][pend], c.get("pool_match"),
                                     None if "pod_class" not in c else c["pod_class"][pend])
    return {"placed": placed, "decisions": calls, "used": used, "nc": nc, "nx": nx, "has": has, "count": count,
            "flips": flips, "rises": rises, "pend": pend, "present": present, "fulfill": f}


@functools.lru_cache(maxsize=None)
def oracle_of(base, ts_kind, pa_kind, D):
    return oracle_of_case(case(base, ts_kind, pa_kind, D))


def run(engine, c, pend, present, knobs, with_aa=True, with_pa=True, pod_idx=None):
    """the node pass over the req rows `pod_idx` (None: every row), then the bin pass over the rows `pend`"""
    try:
        for k, v in knobs.items():
            engine.set_knob(k, v)
        sel = "pod_class" in c
        d_used = engine.dev(c["used0"], F64)
        d_nc, d_nx = engine.dev(i64(c["node_carries0"]), I64), engine.dev(i64(c["node_matches0"]), I64)
        d_has = engine.dev(i64(c["node_has0"]), I64)
        d_cnt = engine.dev(np.ascontiguousarray(c["ts_count0"]), I32)
        aa = (engine.dev(i64(c["pod_carries"]), I64), engine.dev(i64(c["pod_matches"]), I64), d_nc, d_nx) \
            if with_aa else None
        pa = tuple(engine.dev(i64(c[k]), I64) for k in ("pa_requires", "pa_self", "pa_matches")) + (d_has,) \
            if with_pa else None
        p, dec = engine.first_fit_nodes_ts(
            engine.dev(c["req"], F64), None if pod_idx is None else engine.dev(pod_idx, I32),
            engine.dev(c["cap_type"], F64), engine.dev(c["node_type"], I32), d_used, c["ts_keys"],
            engine.dev(c["ts_key"], U8), engine.dev(c["ts_skew"], I32), engine.dev(i64(c["ts_matches"]), I64), d_cnt,
            engine.dev(i64(c["ts_domain"]), I64), c["ts_floor"],
            pa=pa, aa=aa,
            **(dict(pod_class=engine.dev(c["pod_class"], U8), node_match=engine.dev(i64(c["node_match"]), I64),
                    classes=c["classes"]) if sel else {}))
        node_flips, node_rises = engine.last_affinity_reruns(), engine.last_spread_rises()
        f = engine.fulfill_pending_ts(
            engine.dev(c["req"][pend], F64), len(pend) + 3, c["unit"], c["pool_actual"], c["pool_max"],
            c["pool_ignored"], c["over_provision"], c["ts_keys"], engine.dev(c["ts_key"][pend], U8),
            engine.dev(c["ts_skew"][pend], I32), engine.dev(i64(c["ts_matches"][pend]), I64),
            pa=tuple(engine.dev(i64(c[k][pend]), I64) for k in ("pa_requires", "pa_self", "pa_matches"))
            if with_pa else None, present=present,
            aa=(engine.dev(i64(c["pod_carries"][pend]), I64), engine.dev(i64(c["pod_matches"][pend]), I64))
            if with_aa else None,
            **(dict(pod_class=engine.dev(c["pod_class"][pend], U8), pool_match=c["pool_match"],
                    classes=c["classes"]) if sel else {}))
        torch.cuda.synchronize()
        bin_flips = engine.last_affinity_reruns()
        return {"placed": to_np(p), "decisions": int(to_np(dec)[0]), "used": to_np(d_used),
                "nc": to_np(d_nc).view(U64), "nx": to_np(d_nx).view(U64), "has": to_np(d_has).view(U64),
                "count": to_np(d_cnt), "flips": node_flips, "rises": node_rises,
                "fulfill": dict({k: to_np(v) if isinstance(v, torch.Tensor) else v for k, v in f.items()},
                                flips=bin_flips)}
    finally:
        for k, v in DEFAULT_KNOBS.items():
            engine.set_knob(k, v)


def assert_equal(g, o, with_aa=True, with_pa=True):
    np.testing.assert_array_equal(g["placed"], o["placed"])
    assert g["decisions"] == o["decisions"]
    np.testing.assert_array_equal(g["used"].view(U64), o["used"].view(U64))
    np.testing.assert_array_equal(g["count"], o["count"])
    if with_pa:
        np.testing.assert_array_equal(g["has"], o["has"])
    if with_aa:
        np.testing.assert_array_equal(g["nc"], o["nc"])
        np.testing.assert_array_equal(g["nx"], o["nx"])
    assert g["rises"] == o["rises"]
    assert g["flips"] == o["flips"]
    for k, v in o["fulfill"].items():
        np.testing.assert_array_equal(np.asarray(g["fulfill"][k]), np.asarray(v), err_msg=k)


@pytest.fixture(scope="module")
def eng():
    """one engine for the module; each case runs under both candidate scans (packed ranks and float64)"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from kubernetes_acs_engine_autoscaler_b200 import build as acs_build
    acs_build.build()
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    e = Engine(0, watchdog_ms=15000)
    e.set_knob("stream", 0)
    yield e
    e.close()


def check(eng, base, ts_kind, pa_kind, D, schedules=("default",), scans=(1, 0)):
    c, o = case(base, ts_kind, pa_kind, D), oracle_of(base, ts_kind, pa_kind, D)
    try:
        for ranks in scans:
            eng.set_knob("ranks", ranks)
            for schedule in schedules:
                assert_equal(run(eng, c, o["pend"], o["present"], SCHEDULES[schedule]), o)
    finally:
        eng.set_knob("ranks", 1)
    return c, o


@pytest.mark.parametrize("D", ac.DIMS)
@pytest.mark.parametrize("ts_kind", sorted(TS_KINDS))
def test_ts_matches_oracle(eng, ts_kind, D):
    _, o = check(eng, "with_sel" if ts_kind in ("flat", "keys64") else "replicas", ts_kind, "none", D)
    if ts_kind in ("none", "flat"):
        assert o["rises"] == []  # no key, or every minimum held at 0 by the floor: one pass
    if ts_kind == "rise1":
        assert len(o["rises"]) <= 1  # the floor allows one rise
    if ts_kind == "pinned":
        assert len(o["rises"]) >= 2


@pytest.mark.parametrize("ts_kind,pa_kind", [("rises", "sig2"), ("pinned", "mixed"), ("flat", "sig1")])
def test_rises_and_flips_in_one_pass(eng, ts_kind, pa_kind):
    _, o = check(eng, "with_sel", ts_kind, pa_kind, 4)
    if ts_kind != "flat":
        assert o["rises"] and o["flips"]


@pytest.mark.parametrize("ts_kind", ["rises", "pinned"])
def test_ts_schedules(eng, ts_kind):
    # waves with forced pruning (the rises happen inside a multi-wave pass), two-stage bin passes, retirement off
    check(eng, "replicas", ts_kind, "sig1", 4, schedules=sorted(set(SCHEDULES) - {"default"}), scans=(1,))


@pytest.mark.parametrize("base,ts_kind", [("zero", "rises"), ("edges", "pinned"), ("all_blocked", "flat")])
def test_ts_with_and_without_sel_aa_pa(eng, base, ts_kind):
    c, o = check(eng, base, ts_kind, "none", 4)
    if base == "zero":  # every anti-affinity and pod-affinity mask 0: the calls without `aa` and `pa` give the same
        assert_equal(run(eng, c, o["pend"], o["present"], {}, with_aa=False, with_pa=False), o, False, False)


@pytest.mark.parametrize("name", ["d2_rw1_u8192", "d4_rw1_guard31", "d8_rw3_padded", "d16_f64_width"])
def test_ts_layouts_match_oracle(eng, name):
    check(eng, name, "rises", "mixed", 0, schedules=("default", "multipass"), scans=(1,))


def tile_edge_case(P=300, cap=1000.0):
    """P replicas of one group (maxSkew 1) over two roomy nodes: the minimum rises after every second pod, at
    positions 1, 3, ..., 255 (the last pod of the first 256-pod tile), 257, ...; a new node of the pool takes one"""
    N, D = 2, 2
    c = {"req": np.ones((P, D)), "cap_type": np.full((N, D), cap), "node_type": np.arange(N, dtype=np.int32),
         "used0": np.zeros((N, D)), "unit": np.full((1, D), 4.0), "pool_actual": np.zeros(1, np.int32),
         "pool_max": np.full(1, 1000, np.int32), "pool_ignored": np.zeros(1, np.uint8), "over_provision": 0,
         "pod_carries": np.zeros(P, U64), "pod_matches": np.zeros(P, U64), "node_carries0": np.zeros(N, U64),
         "node_matches0": np.zeros(N, U64), "pa_requires": np.zeros(P, U64), "pa_self": np.zeros(P, U64),
         "pa_matches": np.zeros(P, U64), "node_has0": np.zeros(N, U64)}
    c.update(ts_keys=1, ts_key=np.zeros(P, np.uint8), ts_skew=np.zeros(P, np.int32), ts_matches=np.ones(P, U64),
             ts_count0=np.zeros((1, N), np.int32), ts_domain=np.ones(N, U64), ts_floor=np.full(1, INT32_MAX, np.int32))
    return c


def test_rise_at_a_tile_edge(eng):
    c = tile_edge_case()
    o = oracle_of_case(c)
    assert (0, 255) in o["rises"] and (0, 257) in o["rises"] and len(o["rises"]) == 150
    assert o["placed"].tolist() == [0, 1] * 150
    assert_equal(run(eng, c, o["pend"], o["present"], {}), o)


def test_refusals(eng):
    from kubernetes_acs_engine_autoscaler_b200._native import AcsfitError, E_INVALID
    c, o = case("replicas", "rises", "none", 4), oracle_of("replicas", "rises", "none", 4)
    req, cap, nt = eng.dev(c["req"], F64), eng.dev(c["cap_type"], F64), eng.dev(c["node_type"], I32)
    key, skew, m = eng.dev(c["ts_key"], U8), eng.dev(c["ts_skew"], I32), eng.dev(i64(c["ts_matches"]), I64)
    dom = eng.dev(i64(c["ts_domain"]), I64)

    def nodes(**kw):
        a = dict(keys=c["ts_keys"], pod_key=key, pod_skew=skew, pod_matches=m,
                 node_count=eng.dev(c["ts_count0"], I32), node_domain=dom, floor=c["ts_floor"])
        a.update(kw)
        return eng.first_fit_nodes_ts(req, None, cap, nt, eng.dev(c["used0"], F64), a.pop("keys"), a.pop("pod_key"),
                                      a.pop("pod_skew"), a.pop("pod_matches"), a.pop("node_count"),
                                      a.pop("node_domain"), a.pop("floor"))
    big_key = eng.dev(np.where(c["ts_key"] == 0, 1, c["ts_key"]).astype(np.uint8), U8)  # key 1 >= keys = 1
    bad_calls = [
        lambda: nodes(pod_key=None),
        lambda: nodes(node_count=None),
        lambda: nodes(node_domain=None),
        lambda: nodes(pod_key=big_key),
        lambda: nodes(pod_skew=eng.dev(np.full(len(c["req"]), -1, np.int32), I32)),
        lambda: nodes(floor=np.full(1, -1, np.int32)),
        lambda: nodes(node_count=eng.dev(np.full_like(c["ts_count0"], -1), I32)),
        lambda: nodes(keys=65),
        lambda: nodes(pod_matches=eng.dev(i64(c["ts_matches"] | U64(2)), I64)),  # key 1 >= keys = 1
        lambda: nodes(keys=0, pod_key=eng.dev(np.full(len(c["req"]), 0xFF, np.uint8), U8),
                      node_count=eng.dev(np.zeros((0, len(c["node_type"])), np.int32), I32),
                      floor=np.zeros(0, np.int32)),  # matches with a bit while there is no key at all
        lambda: eng.fulfill_pending_ts(req, len(c["req"]), c["unit"], c["pool_actual"], c["pool_max"],
                                       c["pool_ignored"], 1, 1, key, skew, eng.dev(i64(c["ts_matches"] | U64(1 << 63)),
                                                                                   I64)),
        lambda: eng.fulfill_pending_ts(req, len(c["req"]), c["unit"], c["pool_actual"], c["pool_max"],
                                       c["pool_ignored"], 1, 1, key, None, m),
    ]
    for call in bad_calls:
        with pytest.raises(AcsfitError) as e:
            call()
        assert e.value.status == E_INVALID
    assert_equal(run(eng, c, o["pend"], o["present"], {}), o)  # the next call still matches the oracle


# ---------------------------------------------------------------- through Cluster.loop_logic
import golden_util as gu  # noqa: E402

TICKS = gu.load_json("ticks.json.gz")


@pytest.fixture()
def host(tmp_path, monkeypatch, eng):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", eng)
    return monkeypatch


def tick(state, engine, on):
    from test_gpu_selector_states import tick as tick2
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_TOPOLOGY_SPREAD", on)
        return tick2(state, engine, "0", "0")


@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_switch_without_constraints_is_the_reference_tick(host, eng, state):
    off = tick(state, eng, "0")
    on = tick(state, eng, "1")
    gu.assert_tick_matches(off, state["expected"])
    gu.assert_tick_matches(on, state["expected"])
    assert on["launches"] == off["launches"]


def spread_state(running_per_node, n_nodes, replicas, master_replica=False, skew=1):
    """pool `agentpool1` (Standard_D2_v2) of `n_nodes` nodes, each running `running_per_node` replicas of `web`
    (0.1 cpu), plus `replicas` pending ones spread with maxSkew `skew` over kubernetes.io/hostname; the master runs
    a replica when `master_replica`"""
    def node(name, pool=True):
        labels = {"beta.kubernetes.io/instance-type": "Standard_D2_v2", "kubernetes.io/hostname": name,
                  "failure-domain.beta.kubernetes.io/region": "southcentralus"}
        if pool:
            labels["agentpool"] = "agentpool1"
        return {"metadata": {"name": name, "creationTimestamp": "2016-08-25T05:13:16Z", "labels": labels}, "spec": {}}
    names = ["k8s-agentpool1-16334397-%d" % i for i in range(n_nodes)]
    nodes = [node(n) for n in names] + [node("k8s-master-16334397-0", pool=False)]
    spread = [{"maxSkew": skew, "topologyKey": "kubernetes.io/hostname", "whenUnsatisfiable": "DoNotSchedule",
               "labelSelector": {"matchLabels": {"app": "web"}}}]

    def pod(n, node_name=None, phase="Pending"):
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "100m"}}}],
                "topologySpreadConstraints": spread}
        if node_name:
            spec["nodeName"] = node_name
        return {"metadata": {"name": n, "namespace": "default", "uid": "uid-" + n, "labels": {"app": "web"},
                             "creationTimestamp": "2026-09-20T07:00:00Z"}, "spec": spec, "status": {"phase": phase}}
    pods = [pod("run-%d-%d" % (i, j), names[i], "Running") for i in range(n_nodes) for j in range(running_per_node)]
    if master_replica:
        pods.append(pod("run-master", "k8s-master-16334397-0", "Running"))
    pods += [pod("web-%d" % i) for i in range(replicas)]
    return {"name": "topology_spread", "now": "2026-09-21T12:00:00Z", "nodes": nodes, "pods": pods,
            "arm_parameters": {"masterVMSize": {"value": "Standard_D2_v2"},
                               "firstConsecutiveStaticIP": {"value": "10.0.0.1"},
                               "agentpool1VMSize": {"value": "Standard_D2_v2"}},
            "settings": {"idle_threshold": 1800, "spare_agents": 0, "over_provision": 0, "dry_run": True,
                         "ignore_pools": ""}}


def test_stacked_replicas_scale_up(host, eng):
    # three pending replicas "fit" the one roomy node; with the master (no replica) holding the minimum at 0 the
    # scheduler takes one there and needs new nodes for the other two, one each
    s = spread_state(0, 1, 3)
    off = tick(s, eng, "0")
    on = tick(s, eng, "1")
    assert off["exception"] is None and on["exception"] is None
    assert off["scale_pools_calls"] == []
    assert on["scale_pools_calls"] == [{"agentpool1": 1 + 2}]


def test_pinned_pool_does_not_scale(host, eng):
    # three nodes already run one replica each and so does the master: the minimum is 1, and a fourth replica lands
    # on a node with room -- nothing scales.  A rule that took the minimum as 0 would ask for a node.
    s = spread_state(1, 3, 1, master_replica=True)
    on = tick(s, eng, "1")
    assert on["exception"] is None and on["scale_pools_calls"] == []
    # without the master's replica the master holds the minimum at 0: the fourth replica needs a new node
    s = spread_state(1, 3, 1, master_replica=False)
    on = tick(s, eng, "1")
    assert on["exception"] is None and on["scale_pools_calls"] == [{"agentpool1": 3 + 1}]
