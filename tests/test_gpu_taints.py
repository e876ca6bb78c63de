"""`-m gpu`: node taints and pod tolerations with node selectors (Cluster(node_taints=True)) on the real CUDA engine.

* Engine level: the ticks of tests/taint_cases.py, whose match classes come from snapshot.selector_classes(...,
  taints=True), through scale_up_sel, feasible_mask_sel, first_fit_nodes_sel and fulfill_pending_sel, exactly equal to
  the plain-C selector oracle (tests/sel_oracle.c) for D in {2, 4, 8, 16} under the engine fixture's modes; the scan
  hits are bounded as in tests/test_gpu_selectors.py, and a first pool most pods may not use runs no chained bin pass.
* The recorded reference ticks with all three switches on and no taint: the reference's tick, same launches, same node
  flags sent to the GPU.
* The recorded ticks with a tainted pool, tolerating and intolerant pods, selectors, and lifecycle / PreferNoSchedule
  taints as noise: exception, scale_pools arguments, used_capacity, warnings, and (with selector_node_states) node
  states, the maintain journal and dry-run lines equal a plain-Python restatement of the rules.
* The tick that motivates the switch: a full CPU pool, an idle GPU node tainted sku=gpu:NoSchedule, one pending CPU pod."""
import copy
import functools

import numpy as np
import pytest
import torch

import golden_util as gu
import sel_oracle
import taint_cases as tc
from test_gpu_selector_states import DRY_MAINTAIN, restate_maintain, tick as tick2
from test_gpu_selectors import assert_tick_equal, eligible_for_first_pool, run_sel, to_np
from test_gpu_selectors_host import NO_FIT, NO_POOL, pool_of, with_selectors
from test_taints_cpu import UNTOLERATED, restated_blocking, restated_tolerates

pytestmark = pytest.mark.gpu

F64, I32, U8 = torch.float64, torch.int32, torch.uint8


@functools.lru_cache(maxsize=None)
def case_and_oracle(kind, D):
    c = tc.make_case(kind, D)
    used_o = c["used0"].copy()
    return c, sel_oracle.scale_up_sel(c, used_o), used_o


@pytest.mark.parametrize("D", tc.DIMS)
@pytest.mark.parametrize("kind", tc.KINDS)
def test_taint_classes_through_the_sel_kernels(engine, kind, D):
    c, o, used_o = case_and_oracle(kind, D)
    g, used, recs = run_sel(engine, c, {})
    assert_tick_equal(g, o, used, used_o)
    assert g["sel_hits"] >= int((o["placed"] >= 0).sum())
    if kind == "all_intolerant":  # no pod matches any node: the scans hand nothing to the resolver
        assert g["sel_hits"] == 0 and not (o["placed"] >= 0).any()
    chained = any(r["chained"] for r in recs)
    if chained:
        assert eligible_for_first_pool(c, o)
    if kind == "first_tainted":   # most pods may not use the first pool visited: no chained first bin pass
        assert not eligible_for_first_pool(c, o) and not chained
    if kind in ("class0_empty", "all_intolerant"):
        assert c["pod_class"].all()
    # the entry points one by one
    req = engine.dev(c["req"], F64)
    pc = engine.dev(c["pod_class"], U8)
    m, ev = engine.feasible_mask_sel(req, engine.dev(c["unit_all"], F64), pc, c["pool_match_all"], c["classes"])
    mo, evo = sel_oracle.feasible_mask_sel(c["req"], c["unit_all"], c["pool_match_all"], c["pod_class"])
    np.testing.assert_array_equal(to_np(m), mo)
    assert int(to_np(ev)[0]) == evo
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
    # taint-sensitive: the selector classes alone answer differently (except where no taint blocks)
    from kubernetes_acs_engine_autoscaler_b200 import snapshot
    alone = snapshot.selector_classes(c["pods"], c["nodes"], c["pools"])
    sc = dict(c, pod_class=alone.pod_class, node_match=alone.node_match, pool_match_all=alone.pool_match,
              pool_match_ordered=alone.pool_match[c["order"]], classes=alone.classes)
    oa = sel_oracle.scale_up_sel(sc, c["used0"].copy())
    same = all(np.array_equal(np.asarray(oa[k]), np.asarray(o[k])) for k in ("feasible", "placed", "acc_pool", "new_size"))
    assert same == (kind == "noise_only")


# ---------------------------------------------------------------- through Cluster.loop_logic
TICKS = gu.load_json("ticks.json.gz")
GPU_TAINT = {"key": "sku", "value": "gpu", "effect": "NoSchedule"}
NOISE = ([{"key": "node.kubernetes.io/not-ready", "effect": "NoExecute"}],
         [{"key": "soft", "value": "1", "effect": "PreferNoSchedule"}],
         [{"key": "node.kubernetes.io/unreachable", "effect": "NoSchedule"}], [])
TOLERATIONS = ([], [{"key": "sku", "operator": "Equal", "value": "gpu"}], [{"operator": "Exists"}],
               [{"key": "sku", "operator": "Equal", "value": "cpu"}], [{"key": "sku", "operator": "Exists",
                                                                        "effect": "NoSchedule"}])


@pytest.fixture()
def host(tmp_path, monkeypatch, engine):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", engine)
    return monkeypatch


def tick(state, engine, selectors, states_on, taints):
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_NODE_TAINTS", taints)
        return tick2(state, engine, selectors, states_on)


@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_switches_on_without_taints_is_the_reference_tick(host, engine, state):
    off = tick(state, engine, "0", "0", "0")
    on = tick(state, engine, "1", "1", "1")
    gu.assert_tick_matches(on, state["expected"])
    assert on["launches"] == off["launches"]
    assert on["node_flags_sent"] == off["node_flags_sent"]


def with_taints(state, variant):
    """the recorded tick with selectors (with_selectors), one pool tainted sku=gpu:NoSchedule, noise taints on every
    node, and tolerations on the unassigned pending pods"""
    s = with_selectors(state, variant)
    pools = [k[:-len("VMSize")] for k in s["arm_parameters"] if k.endswith("VMSize") and k != "masterVMSize"]
    tainted = pools[variant % len(pools)]
    for i, n in enumerate(s["nodes"]):
        taints = ([GPU_TAINT] if pool_of(n["metadata"]["name"]) == tainted else []) + NOISE[(i + variant) % len(NOISE)]
        if taints:
            n.setdefault("spec", {})["taints"] = copy.deepcopy(taints)
    for i, p in enumerate(s["pods"]):
        if p["status"]["phase"] == "Pending" and not p["spec"].get("nodeName"):
            tol = TOLERATIONS[(i + 2 * variant) % len(TOLERATIONS)]
            if tol:
                p["spec"]["tolerations"] = copy.deepcopy(tol)
    return s


def _kube(state):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, utils
    from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod
    st = state["settings"]
    journal = []
    nodes = []
    for o in state["nodes"]:
        n = KubeNode(gu.FakeKubeObject(o, journal, "node"))
        n.capacity = capacity.get_capacity_for_instance_type(n.instance_type)
        if utils.is_agent(n):
            nodes.append(n)
    pods = [KubePod(gu.FakeKubeObject(o, journal, "pod")) for o in state["pods"]]
    buckets = {}
    for param, spec in state["arm_parameters"].items():
        if param.endswith("VMSize") and param != "masterVMSize":
            buckets.setdefault(param[:-len("VMSize")], (spec["value"], []))
    for n in nodes:
        buckets[utils.get_pool_name(n)][1].append(n)
    pools = []
    for name, (vm, members) in buckets.items():
        pool = AgentPool(name, vm, members)
        pool.max_size = st.get("pool_max_size", {}).get(name, pool.max_size)
        pools.append(pool)
    return nodes, pods, pools


def tolerated(pod, taints):
    return all(restated_tolerates(pod.tolerations, t) for t in taints)


def node_ok(node, pod):
    """the selector matches (KubeNode.is_match) and the pod tolerates the node's blocking taints (restated)"""
    return all(node.selectors.get(k) == v for k, v in pod.selectors.items()) and \
        tolerated(pod, restated_blocking(node.taints))


def restate(state):
    """the scale-up half of the tick with the selector and taint rules, in plain Python on the product's kube types.
    Returns (exception name or None, scale_pools calls, used, warnings, names of the pods to schedule)."""
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.kube import KubePodStatus, KubeResource
    st = state["settings"]
    if not state["nodes"]:
        return None, [], {}, ["Failed to list nodes. Please check kube configuration. Terminating scale loop."], set()
    nodes, pods, pools = _kube(state)
    running = [p for p in pods if p.status in (KubePodStatus.RUNNING, KubePodStatus.CONTAINER_CREATING)
               or (p.status == KubePodStatus.PENDING and p.node_name)]
    used = [KubeResource() for _ in nodes]
    for p in running:
        for k, n in enumerate(nodes):
            if n.name == p.node_name:
                used[k] = used[k] + p.resources
    pool_taints = {}
    for pool in pools:
        sets = [restated_blocking(n.taints) for n in pool.nodes]
        pool_taints[pool.name] = set.intersection(*sets) if sets else set()

    def selected(pool, pod):
        return all(pool.labels.get(k) == v for k, v in pod.selectors.items())

    def pool_ok(pool, pod):
        return selected(pool, pod) and tolerated(pod, pool_taints[pool.name])

    def fits_unit(pool, pod):
        return (capacity.RESOURCE_SPEC[pool.instance_type] - pod.resources).possible

    warnings, to_schedule = [], []
    for p in pods:
        if p.status != KubePodStatus.PENDING or p.node_name:
            continue
        if any(pool_ok(pool, p) and fits_unit(pool, p) for pool in pools):
            to_schedule.append(p)
        elif any(selected(pool, p) and fits_unit(pool, p) for pool in pools):
            warnings.append(UNTOLERATED % p.name)
        elif p.selectors and any(fits_unit(pool, p) for pool in pools):
            warnings.append(NO_POOL % (p.name, p.selectors))
        else:
            warnings.append(NO_FIT % p.name)
    pending = []
    for p in to_schedule:
        for k, n in enumerate(nodes):
            if node_ok(n, p) and (n.capacity - (used[k] + p.resources)).possible:
                used[k] = used[k] + p.resources
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
            bins, bin_of = [], {}
            for p in unique:
                if p in acc or not (pool_ok(pool, p) and (unit - p.resources).possible):
                    continue
                for b, rem in enumerate(bins):
                    if (rem - p.resources).possible:
                        bins[b] = rem - p.resources
                        bin_of[p] = b
                        break
                else:
                    bins.append(unit - p.resources)
                    bin_of[p] = len(bins) - 1
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
    return exc, calls, used_hex, warnings, {p.name for p in to_schedule}


def assert_maintain_restated(s, got, exc, names):
    """node states, maintain journal, node and dry-run lines: upstream get_node_state / maintain with the taint-aware
    match as `pending_list`"""
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode
    st = s["settings"]
    if exc is not None or not st.get("maintainance", True) or not s["nodes"]:
        assert got["maintain_journal"] is None and got["state_calls"] == [], s["name"]
        return
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(KubeNode, "is_match", node_ok)
        calls, journal, node_lines, dry_lines, deleted = restate_maintain(s, names)
    assert got["state_calls"] == calls, s["name"]
    assert got["maintain_journal"] == journal, s["name"]
    assert [m for _, _, m in got["log"] if m.startswith("node: ")] == node_lines, s["name"]
    assert [m for _, _, m in got["log"] if DRY_MAINTAIN.match(m)] == dry_lines, s["name"]
    assert got["deleted_nodes"] == deleted, s["name"]


@pytest.mark.parametrize("states_on", ("0", "1"))
@pytest.mark.parametrize("variant", (0, 1, 2))
def test_ticks_with_taints_match_restatement(host, engine, variant, states_on):
    differs = ran = 0
    for state in TICKS:
        s = with_taints(state, variant)
        got = tick(s, engine, "1", states_on, "1")
        exc, calls, used, warnings, names = restate(s)
        if not s["settings"].get("scale_up", True):
            exc = None
        else:
            assert got["scale_pools_calls"] == calls, s["name"]
            assert got["used"] == used, s["name"]
        assert (got["exception"] or [None])[0] == exc, s["name"]
        warn = [m for lvl, _, m in got["log"] if lvl == "WARNING"]
        if s["settings"].get("scale_up", True):
            assert warn == warnings, s["name"]
        else:  # maintain only: just the feasibility warnings
            assert warn == [w for w in warnings if w != "Failed to scale sufficiently."], s["name"]
        if states_on == "1":
            assert_maintain_restated(s, got, exc, names)
            ran += got["maintain_journal"] is not None
        off = tick(s, engine, "1", states_on, "0")
        differs += (off["scale_pools_calls"], off["used"], off["exception"], off["state_calls"]) != \
            (got["scale_pools_calls"], got["used"], got["exception"], got["state_calls"])
    assert differs >= 3, differs
    assert states_on == "0" or ran >= 5, ran


# ---------------------------------------------------------------- the motivating tick
def gpu_taint_state(dry_run):
    """pool `agentpool1` (Standard_D2_v2, the cheap one): two nodes, each busy with a 1.5-cpu pod.  Pool `gpupool`
    (Standard_NC6): one old idle node tainted sku=gpu:NoSchedule.  One pending 1-cpu pod without tolerations."""
    def node(pool, i, itype, taints=None):
        name = "k8s-%s-16334397-%d" % (pool, i)
        spec = {"taints": taints} if taints else {}
        return {"metadata": {"name": name, "creationTimestamp": "2016-08-25T05:13:16Z",
                             "labels": {"beta.kubernetes.io/instance-type": itype, "agentpool": pool,
                                        "failure-domain.beta.kubernetes.io/region": "southcentralus",
                                        "kubernetes.io/hostname": name}}, "spec": spec}

    def pod(name, cpu, phase, node_name=None):
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": cpu}}}]}
        if node_name:
            spec["nodeName"] = node_name
        status = {"phase": phase}
        if phase == "Running":
            status["startTime"] = "2026-09-20T07:00:00Z"
        return {"metadata": {"name": name, "namespace": "default", "uid": "uid-" + name,
                             "creationTimestamp": "2026-09-20T07:00:00Z"}, "spec": spec, "status": status}
    nodes = [node("agentpool1", i, "Standard_D2_v2") for i in range(2)] + \
        [node("gpupool", 0, "Standard_NC6", [dict(GPU_TAINT)])]
    pods = [pod("web-%d" % i, "1500m", "Running", nodes[i]["metadata"]["name"]) for i in range(2)] + \
        [pod("worker", "1", "Pending")]
    return {"name": "gpu_taint_%s" % ("dry" if dry_run else "live"), "now": "2026-09-21T12:00:00Z",
            "nodes": nodes, "pods": pods,
            "arm_parameters": {"masterVMSize": {"value": "Standard_D2_v2"}, "firstConsecutiveStaticIP": {"value": "10.0.0.1"},
                               "agentpool1VMSize": {"value": "Standard_D2_v2"}, "gpupoolVMSize": {"value": "Standard_NC6"}},
            "settings": {"idle_threshold": 1800, "spare_agents": 0, "over_provision": 0, "dry_run": dry_run,
                         "ignore_pools": ""}}


@pytest.mark.parametrize("dry_run", [True, False])
def test_tainted_gpu_pool_no_longer_absorbs_the_cpu_pod(host, engine, dry_run):
    s = gpu_taint_state(dry_run)
    gpu_node = s["nodes"][2]["metadata"]["name"]
    alone = tick(s, engine, "1", "1", "0")
    taints = tick(s, engine, "1", "0", "1")
    both = tick(s, engine, "1", "1", "1")
    for got in (alone, taints, both):
        assert got["exception"] is None and "Pods to schedule: 1" in [m for _, _, m in got["log"]]
    # selectors alone: the pod "fits" the idle GPU node, nothing grows, and the GPU node waits for it
    assert alone["scale_pools_calls"] == [] and alone["used"][gpu_node] == {"cpu": float(1).hex(), "pods": float(1).hex()}
    # taints on: the CPU pool grows by one; the GPU node stays empty
    for got in (taints, both):
        assert got["scale_pools_calls"] == [{"agentpool1": 3, "gpupool": 1}]
        assert got["used"][gpu_node] == {}
    # node states: pod-pending unless both switches are on
    assert [st for n, st in taints["state_calls"] if n == gpu_node] == ["pod-pending"]
    assert [st for n, st in both["state_calls"] if n == gpu_node] == ["under-utilized-drainable"]
    exc, calls, used, warnings, names = restate(s)
    assert (exc, [calls, used]) == (None, [both["scale_pools_calls"], both["used"]]) and names == {"worker"}
    assert_maintain_restated(s, both, None, names)
