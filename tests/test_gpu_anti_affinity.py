"""`-m gpu`: the pod anti-affinity entry points (acsfit_first_fit_nodes_aa, acsfit_fulfill_pending_aa) against the
plain-C oracle (tests/aa_oracle.c), exactly, on the ticks of tests/aa_cases.py and on the rank-layout ticks of
tests/variant_cases.py, under the engine fixture's three scan modes and several pipeline schedules; the refusals;
and the host layer end to end (Cluster.loop_logic) with the switch on."""
import functools

import numpy as np
import pytest
import torch

import aa_cases as ac
import aa_oracle
import sel_oracle
import variant_cases as vc

pytestmark = pytest.mark.gpu

SCHEDULES = {
    "default": {},
    "waves_prune": {"min_stages": 1 << 20, "prune": 1},
    "waves_noprune": {"min_stages": 1 << 20, "prune": 0},
    "multipass": {"bin_pass_stages": 2, "min_stages": 32},
}
DEFAULT_KNOBS = {"min_stages": 0, "prune": -1, "overlap": 1, "bin_pass_stages": 0}
F64, I32, U8, I64 = torch.float64, torch.int32, torch.uint8, torch.int64


def to_np(t):
    return t.cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def i64(a):
    return np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)


@functools.lru_cache(maxsize=None)
def case(kind, D):
    return ac.make_case(kind, D)


@functools.lru_cache(maxsize=None)
def layout_case(name):
    import cluster_cases as cc
    return ac.overlay(cc._with_used(vc.case(name)), seed=3)


@functools.lru_cache(maxsize=None)
def oracle_of(key):
    return oracle_of_case(case(*key) if isinstance(key, tuple) else layout_case(key))


def oracle_of_case(c, pod_idx=None):
    """the oracle over the req rows `pod_idx` in that order (None: every row); placements are in list positions, and
    "pend" holds the req rows of the pods left pending, in list order"""
    used, nc, nx = c["used0"].copy(), c["node_carries0"].copy(), c["node_matches0"].copy()
    rows = np.arange(len(c["req"])) if pod_idx is None else np.asarray(pod_idx)
    placed, calls = aa_oracle.first_fit_nodes_aa(c["req"][rows], c["cap_type"], c["node_type"], used,
                                                 c["pod_carries"][rows], c["pod_matches"][rows], nc, nx,
                                                 c.get("node_match"),
                                                 None if "pod_class" not in c else c["pod_class"][rows])
    pend = rows[placed < 0]
    f = aa_oracle.fulfill_pending_aa(c["req"][pend], len(pend) + 3, c["unit"], c["pool_actual"], c["pool_max"],
                                     c["pool_ignored"], c["over_provision"], c["pod_carries"][pend],
                                     c["pod_matches"][pend], c.get("pool_match"),
                                     None if "pod_class" not in c else c["pod_class"][pend])
    return {"placed": placed, "decisions": calls, "used": used, "nc": nc, "nx": nx, "pend": pend, "fulfill": f}


def run(engine, c, pend, knobs, pod_idx=None):
    """node pass over the req rows `pod_idx` (None: every row), then the bin pass over the rows `pend`; returns
    outputs and launch records of both"""
    try:
        for k, v in knobs.items():
            engine.set_knob(k, v)
        sel = "pod_class" in c
        d_used = engine.dev(c["used0"], F64)
        d_nc, d_nx = engine.dev(i64(c["node_carries0"]), I64), engine.dev(i64(c["node_matches0"]), I64)
        p, dec = engine.first_fit_nodes_aa(
            engine.dev(c["req"], F64), None if pod_idx is None else engine.dev(pod_idx, I32),
            engine.dev(c["cap_type"], F64), engine.dev(c["node_type"], I32), d_used,
            engine.dev(i64(c["pod_carries"]), I64), engine.dev(i64(c["pod_matches"]), I64), d_nc, d_nx,
            *((engine.dev(c["pod_class"], U8), engine.dev(i64(c["node_match"]), I64), c["classes"]) if sel else ()))
        node_recs = engine.last_launches()
        f = engine.fulfill_pending_aa(
            engine.dev(c["req"][pend], F64), len(pend) + 3, c["unit"], c["pool_actual"], c["pool_max"],
            c["pool_ignored"], c["over_provision"], engine.dev(i64(c["pod_carries"][pend]), I64),
            engine.dev(i64(c["pod_matches"][pend]), I64),
            *((engine.dev(c["pod_class"][pend], U8), c["pool_match"], c["classes"]) if sel else ()))
        torch.cuda.synchronize()
        out = {"placed": to_np(p), "decisions": int(to_np(dec)[0]), "used": to_np(d_used),
               "nc": to_np(d_nc).view(np.uint64), "nx": to_np(d_nx).view(np.uint64),
               "fulfill": {k: to_np(v) if isinstance(v, torch.Tensor) else v for k, v in f.items()}}
        return out, node_recs, engine.last_launches()
    finally:
        for k, v in DEFAULT_KNOBS.items():
            engine.set_knob(k, v)


def assert_equal(g, o):
    np.testing.assert_array_equal(g["placed"], o["placed"])
    assert g["decisions"] == o["decisions"]
    np.testing.assert_array_equal(g["used"].view(np.uint64), o["used"].view(np.uint64))
    np.testing.assert_array_equal(g["nc"], o["nc"])
    np.testing.assert_array_equal(g["nx"], o["nx"])
    for k, v in o["fulfill"].items():
        np.testing.assert_array_equal(np.asarray(g["fulfill"][k]), np.asarray(v), err_msg=k)


def check_records(node_recs, bin_recs, schedule):
    nodes = [r for r in node_recs if r["pass"] == 0]
    bins = [r for r in bin_recs if r["pass"] == 1]
    assert nodes and all(r["pass"] == 0 for r in node_recs)
    for r in nodes + bins:
        assert r["form"] == 0 and r["chained"] == 0, r
    for r in nodes:
        assert r["prune"] == {"waves_prune": 1, "waves_noprune": 0}.get(schedule, int(r["stages"] > r["resident"]))
    if schedule == "multipass" and bins:
        assert len(bins) >= 2 or bins[0]["stages"] <= 2


def mode_rw_ok(request, recs):
    mode = request.node.callspec.params["engine"]
    return all(r["RW"] == 0 for r in recs) if mode == "f64" else True


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("D", ac.DIMS)
@pytest.mark.parametrize("kind", ac.KINDS)
def test_aa_matches_oracle(request, engine, kind, D, schedule):
    c, o = case(kind, D), oracle_of((kind, D))
    g, nrec, brec = run(engine, c, o["pend"], SCHEDULES[schedule])
    assert_equal(g, o)
    check_records(nrec, brec, schedule)
    assert mode_rw_ok(request, nrec + brec)
    if kind == "all_blocked":
        assert (o["placed"] < 0).all()
    if kind == "replicas":  # one replica of a deployment per node and per bin
        assert (o["placed"] >= 0).sum() <= 3 * c["node_type"].shape[0]


@pytest.mark.parametrize("schedule", sorted(SCHEDULES))
@pytest.mark.parametrize("name", sorted(vc.LAYOUTS))
def test_aa_layouts_match_oracle(request, engine, name, schedule):
    c, o = layout_case(name), oracle_of(name)
    g, nrec, brec = run(engine, c, o["pend"], SCHEDULES[schedule])
    assert_equal(g, o)
    check_records(nrec, brec, schedule)
    assert mode_rw_ok(request, nrec + brec)


@pytest.mark.parametrize("D", ac.DIMS)
def test_zero_masks_equal_sel_and_plain(engine, D):
    c = case("zero", D)
    o = oracle_of(("zero", D))
    # the oracle with zero masks is the selector oracle
    used = c["used0"].copy()
    po, calls = sel_oracle.first_fit_nodes_sel(c["req"], c["cap_type"], c["node_type"], used,
                                               np.ones(len(c["node_type"]), np.uint64), np.zeros(len(c["req"]), np.uint8))
    np.testing.assert_array_equal(po, o["placed"])
    assert calls == o["decisions"]
    np.testing.assert_array_equal(used.view(np.uint64), o["used"].view(np.uint64))
    # the plain and the _sel entry points give what the AA entry point gives
    g, _, _ = run(engine, c, o["pend"], {})
    d_used = engine.dev(c["used0"], F64)
    p, dec = engine.first_fit_nodes(engine.dev(c["req"], F64), None, engine.dev(c["cap_type"], F64),
                                    engine.dev(c["node_type"], I32), d_used)
    np.testing.assert_array_equal(to_np(p), g["placed"])
    assert int(to_np(dec)[0]) == g["decisions"]
    np.testing.assert_array_equal(to_np(d_used).view(np.uint64), g["used"].view(np.uint64))
    d_used = engine.dev(c["used0"], F64)
    p, _ = engine.first_fit_nodes_sel(engine.dev(c["req"], F64), None, engine.dev(c["cap_type"], F64),
                                      engine.dev(c["node_type"], I32), d_used,
                                      engine.dev(np.zeros(len(c["req"]), np.uint8), U8),
                                      engine.dev(i64(np.ones(len(c["node_type"]), np.uint64)), I64), 1)
    np.testing.assert_array_equal(to_np(p), g["placed"])
    pend = o["pend"]
    f = engine.fulfill_pending(engine.dev(c["req"][pend], F64), len(pend) + 3, c["unit"], c["pool_actual"],
                               c["pool_max"], c["pool_ignored"], c["over_provision"])
    for k in ("new_size", "units_needed", "bins_opened", "acc_pool", "bin_of", "num_unaccounted", "evals"):
        np.testing.assert_array_equal(to_np(f[k]), np.asarray(g["fulfill"][k]), err_msg=k)


def test_refusals(engine):
    from kubernetes_acs_engine_autoscaler_b200._native import AcsfitError, E_INVALID
    c, o = case("with_sel", 4), oracle_of(("with_sel", 4))
    req, cap, nt = engine.dev(c["req"], F64), engine.dev(c["cap_type"], F64), engine.dev(c["node_type"], I32)
    pc, px = engine.dev(i64(c["pod_carries"]), I64), engine.dev(i64(c["pod_matches"]), I64)
    nc, nx = engine.dev(i64(c["node_carries0"]), I64), engine.dev(i64(c["node_matches0"]), I64)
    cls, nm = engine.dev(c["pod_class"], U8), engine.dev(i64(c["node_match"]), I64)
    bad_calls = [
        lambda: engine.first_fit_nodes_aa(req, None, cap, nt, engine.dev(c["used0"], F64), None, px, nc, nx),
        lambda: engine.first_fit_nodes_aa(req, None, cap, nt, engine.dev(c["used0"], F64), pc, px, None, nx),
        lambda: engine.first_fit_nodes_aa(req, None, cap, nt, engine.dev(c["used0"], F64), pc, px, nc, nx, cls, nm, 2),
        lambda: engine.first_fit_nodes_aa(req, None, cap, nt, engine.dev(c["used0"], F64), pc, px, nc, nx, cls,
                                          engine.dev(i64(c["node_match"] & ~np.uint64(1)), I64), 3),
        lambda: engine.fulfill_pending_aa(req, len(c["req"]), c["unit"], c["pool_actual"], c["pool_max"],
                                          c["pool_ignored"], 1, pc, None),
        lambda: engine.fulfill_pending_aa(req, len(c["req"]), c["unit"], c["pool_actual"], c["pool_max"],
                                          c["pool_ignored"], 1, pc, px, cls, c["pool_match"] & ~np.uint64(1), 3),
    ]
    for call in bad_calls:
        with pytest.raises(AcsfitError) as e:
            call()
        assert e.value.status == E_INVALID
    g, _, _ = run(engine, c, o["pend"], {})  # the next call still matches the oracle
    assert_equal(g, o)


def _cluster_refusal_worker(rank, world, port, q):
    import os
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    try:
        dist.init_process_group("gloo", rank=rank, world_size=world)
        from kubernetes_acs_engine_autoscaler_b200.engine import Engine
        from kubernetes_acs_engine_autoscaler_b200._native import AcsfitError
        eng = Engine(0)
        eng.cluster_connect(4096, 1024)
        c = ac.make_case("replicas", 4)
        statuses = []
        for call in ("nodes", "bins"):
            try:
                if call == "nodes":
                    eng.first_fit_nodes_aa(eng.dev(c["req"], F64), None, eng.dev(c["cap_type"], F64),
                                           eng.dev(c["node_type"], I32), eng.dev(c["used0"], F64),
                                           eng.dev(i64(c["pod_carries"]), I64), eng.dev(i64(c["pod_matches"]), I64),
                                           eng.dev(i64(c["node_carries0"]), I64), eng.dev(i64(c["node_matches0"]), I64))
                else:
                    eng.fulfill_pending_aa(eng.dev(c["req"], F64), len(c["req"]), c["unit"], c["pool_actual"],
                                           c["pool_max"], c["pool_ignored"], 1, eng.dev(i64(c["pod_carries"]), I64),
                                           eng.dev(i64(c["pod_matches"]), I64))
                statuses.append(0)
            except AcsfitError as e:
                statuses.append(e.status)
        dist.barrier()
        eng.close()
        dist.destroy_process_group()
        q.put((rank, statuses))
    except Exception as e:  # reported to the parent, which fails the test
        q.put((rank, repr(e)))


def test_cluster_mode_refuses(tmp_path):
    import multiprocessing as mp
    import socket
    from kubernetes_acs_engine_autoscaler_b200._native import E_INVALID
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_cluster_refusal_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        results = dict(q.get(timeout=240) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=60)
            if p.is_alive():
                p.terminate()
                p.join()
    assert results == {0: [E_INVALID, E_INVALID], 1: [E_INVALID, E_INVALID]}, results


# ---------------------------------------------------------------- through Cluster.loop_logic
import golden_util as gu  # noqa: E402

TICKS = gu.load_json("ticks.json.gz")


@pytest.fixture()
def host(tmp_path, monkeypatch, engine):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", engine)
    return monkeypatch


def tick(state, engine, on):
    from test_gpu_selector_states import tick as tick2
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_POD_ANTI_AFFINITY", on)
        return tick2(state, engine, "0", "0")


@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_switch_on_without_terms_is_the_reference_tick(host, engine, state):
    off = tick(state, engine, "0")
    on = tick(state, engine, "1")
    gu.assert_tick_matches(on, state["expected"])
    assert on["launches"] == off["launches"]


def replicas_state(over_provision):
    """pool `agentpool1` (Standard_D2_v2): one idle node with room for three 0.3-cpu pods.  Three pending replicas of
    one deployment, each avoiding the others on a node (required anti-affinity, hostname topology)."""
    name = "k8s-agentpool1-16334397-0"
    node = {"metadata": {"name": name, "creationTimestamp": "2016-08-25T05:13:16Z",
                         "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2", "agentpool": "agentpool1",
                                    "failure-domain.beta.kubernetes.io/region": "southcentralus",
                                    "kubernetes.io/hostname": name}}, "spec": {}}
    aff = {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
        {"topologyKey": "kubernetes.io/hostname", "labelSelector": {"matchLabels": {"app": "ha"}}}]}}

    def pod(i):
        return {"metadata": {"name": "ha-%d" % i, "namespace": "default", "uid": "uid-ha-%d" % i,
                             "labels": {"app": "ha"}, "creationTimestamp": "2026-09-20T07:00:00Z"},
                "spec": {"containers": [{"name": "c", "resources": {"requests": {"cpu": "300m"}}}], "affinity": aff},
                "status": {"phase": "Pending"}}
    return {"name": "ha_replicas", "now": "2026-09-21T12:00:00Z", "nodes": [node], "pods": [pod(i) for i in range(3)],
            "arm_parameters": {"masterVMSize": {"value": "Standard_D2_v2"}, "firstConsecutiveStaticIP": {"value": "10.0.0.1"},
                               "agentpool1VMSize": {"value": "Standard_D2_v2"}},
            "settings": {"idle_threshold": 1800, "spare_agents": 0, "over_provision": over_provision, "dry_run": True,
                         "ignore_pools": ""}}


@pytest.mark.parametrize("over_provision", [0, 2])
def test_replicas_that_avoid_each_other_grow_the_pool(host, engine, over_provision):
    s = replicas_state(over_provision)
    node = s["nodes"][0]["metadata"]["name"]
    off = tick(s, engine, "0")
    on = tick(s, engine, "1")
    for got in (off, on):
        assert got["exception"] is None and "Pods to schedule: 3" in [m for _, _, m in got["log"]]
    # off: all three "fit" the node, nothing is pending and the pool stays
    assert off["scale_pools_calls"] == [] and float.fromhex(off["used"][node]["pods"]) == 3.0
    # on: one replica lands on the node, the other two need new nodes
    assert float.fromhex(on["used"][node]["pods"]) == 1.0
    assert on["scale_pools_calls"] == [{"agentpool1": 1 + 2 + over_provision}]


# ---------------------------------------------------------------- recorded ticks with terms, against a restatement
AA_KEY = "aa-group"


def _term(selector, namespaces=None):
    t = {"topologyKey": "kubernetes.io/hostname", "labelSelector": selector}
    if namespaces is not None:
        t["namespaces"] = namespaces
    return t


def with_anti_affinity(state, variant):
    """the recorded tick with every pod in one of three groups (label aa-group), and required hostname anti-affinity
    terms on some pods: running or assigned pods that avoid group g0 (their terms block pending pods), pending replicas
    that avoid their own group, and pending pods that avoid group g1 (their terms select running pods)"""
    import copy
    s = copy.deepcopy(state)
    for i, p in enumerate(s["pods"]):
        meta, spec = p["metadata"], p["spec"]
        g = (i + variant) % 3
        meta["labels"] = dict(meta.get("labels") or {}, **{AA_KEY: "g%d" % g})
        assigned = p["status"]["phase"] != "Pending" or spec.get("nodeName")
        if assigned:
            terms = [_term({"matchLabels": {AA_KEY: "g0"}})] if i % 4 == variant % 4 else []
        elif g == 0:
            terms = [_term({"matchLabels": {AA_KEY: "g0"}})]
        elif g == 1:
            terms = [_term({"matchExpressions": [{"key": AA_KEY, "operator": "In", "values": ["g1"]}]},
                           [meta["namespace"], "elsewhere"])]
        else:
            terms = [_term({"matchExpressions": [{"key": AA_KEY, "operator": "NotIn", "values": ["g0", "g1"]}]})] \
                if i % 2 else []
        if terms:
            spec["affinity"] = {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": terms}}
    return s


def restate_aa(state, seen):
    """the scale-up half of the tick with the anti-affinity rule, pair by pair, in plain Python on the product's kube
    types.  Returns (exception name or None, scale_pools calls, used, warnings).  `seen` counts the node rejections by
    direction: a running pod's term that selects the pending pod, and the pending pod's term that selects a running pod."""
    from kubernetes_acs_engine_autoscaler_b200 import capacity, kube
    from kubernetes_acs_engine_autoscaler_b200.kube import KubePodStatus, KubeResource
    from test_gpu_selectors_host import NO_FIT
    from test_gpu_taints import _kube
    st = state["settings"]
    if not state["nodes"]:
        return None, [], {}, ["Failed to list nodes. Please check kube configuration. Terminating scale loop."]
    nodes, pods, pools = _kube(state)
    running = [p for p in pods if p.status in (KubePodStatus.RUNNING, KubePodStatus.CONTAINER_CREATING)
               or (p.status == KubePodStatus.PENDING and p.node_name)]
    used = [KubeResource() for _ in nodes]
    on_node = [[] for _ in nodes]  # (pod, is running)
    for p in running:
        for k, n in enumerate(nodes):
            if n.name == p.node_name:
                used[k] = used[k] + p.resources
                on_node[k].append((p, True))

    def selects(owner, q):
        return any(q.namespace in ns and kube.selector_matches(sel, q.labels) for ns, sel in owner.anti_affinity_terms)

    def blocked(p, there, count=False):
        for q, is_running in there:
            mine, theirs = selects(p, q), selects(q, p)
            if count and is_running:
                seen["pending_term_selects_running"] += mine
                seen["running_term_blocks_pending"] += theirs
            if mine or theirs:
                return True
        return False

    def fits_unit(pool, pod):
        return (capacity.RESOURCE_SPEC[pool.instance_type] - pod.resources).possible

    warnings, to_schedule = [], []
    for p in pods:
        if p.status != KubePodStatus.PENDING or p.node_name:
            continue
        if any(fits_unit(pool, p) for pool in pools):
            to_schedule.append(p)
        else:
            warnings.append(NO_FIT % p.name)
    pending = []
    for p in to_schedule:
        for k, n in enumerate(nodes):
            if not blocked(p, on_node[k], count=True) and (n.capacity - (used[k] + p.resources)).possible:
                used[k] = used[k] + p.resources
                on_node[k].append((p, False))
                break
        else:
            pending.append(p)
    calls, exc = [], None
    if pending:
        unique = list(dict((p, False) for p in pending).keys())
        ignored = set(st["ignore_pools"].split(","))
        acc, sizes, left = set(), {}, len(pending)
        for pool in capacity.order_by_cost_asc(pools):
            sizes[pool.name] = pool.actual_capacity
            if pool.name in ignored or not left:
                continue
            unit = capacity.RESOURCE_SPEC[pool.instance_type]
            bins, members, bin_of = [], [], {}
            for p in unique:
                if p in acc or not (unit - p.resources).possible:
                    continue
                for b, rem in enumerate(bins):
                    if not blocked(p, members[b]) and (rem - p.resources).possible:
                        break
                else:
                    bins.append(unit)
                    members.append([])
                    b = len(bins) - 1
                bins[b] = bins[b] - p.resources
                members[b].append((p, False))
                bin_of[p] = b
            needed = len(bins) + st["over_provision"]
            requested = needed - max(0, needed - (pool.max_size - pool.actual_capacity))
            sizes[pool.name] = pool.actual_capacity + requested
            for p, b in bin_of.items():
                if b < min(len(bins), requested):
                    acc.add(p)
                    left -= 1
        if left:
            warnings.append("Failed to scale sufficiently.")
            exc = "NameError" if st.get("notifier") == "recording" else "AttributeError"
        else:
            calls.append(sizes)
    used_hex = {n.name: {k: float(v).hex() for k, v in used[i].raw.items()} for i, n in enumerate(nodes)}
    return exc, calls, used_hex, warnings


@pytest.mark.parametrize("variant", (0, 1, 2))
def test_ticks_with_terms_match_restatement(host, engine, variant):
    import collections
    seen = collections.Counter()
    differs = 0
    for state in TICKS:
        s = with_anti_affinity(state, variant)
        got = tick(s, engine, "1")
        exc, calls, used, warnings = restate_aa(s, seen)
        if not s["settings"].get("scale_up", True):
            exc = None
        else:
            assert got["scale_pools_calls"] == calls, s["name"]
            assert got["used"] == used, s["name"]
        assert (got["exception"] or [None])[0] == exc, s["name"]
        warn = [m for lvl, _, m in got["log"] if lvl == "WARNING"]
        if s["settings"].get("scale_up", True):
            assert warn == warnings, s["name"]
        else:
            assert warn == [w for w in warnings if w != "Failed to scale sufficiently."], s["name"]
        off = tick(s, engine, "0")
        differs += (off["scale_pools_calls"], off["used"], off["exception"]) != \
            (got["scale_pools_calls"], got["used"], got["exception"])
    # both directions through the pods already on the nodes occur, and the rule changes outcomes
    assert seen["running_term_blocks_pending"] > 0 and seen["pending_term_selects_running"] > 0, seen
    assert differs >= 3, differs
