"""`-m gpu`: required node affinity with node selectors (Cluster(node_affinity=True)) on the real CUDA engine.

* Engine level: the ticks of tests/node_affinity_cases.py, whose match classes come from
  snapshot.selector_classes(..., taints=True, affinity=True), through scale_up_sel, feasible_mask_sel,
  first_fit_nodes_sel and fulfill_pending_sel, exactly equal to the plain-C selector oracle (tests/sel_oracle.c) for
  D in {2, 4, 8, 16} under the engine fixture's modes; the scan hits are bounded, and a first pool most pods may not
  use runs no chained bin pass.
* The recorded reference ticks with every switch on and no affinity: the reference's tick, same launches, same node
  flags sent to the GPU.
* The recorded ticks with node affinity added (pool targeting, NotIn, Gt on a numeric label, DaemonSet-style
  matchFields, hostname NotIn) on top of selectors, taints and (in two variants) pod anti-affinity: exception,
  scale_pools arguments, used_capacity, warnings, and (with selector_node_states) node states, the maintain journal and
  dry-run lines equal a plain-Python restatement of the rules.
* The tick that motivates the switch: a CPU node with room, an empty GPU pool, one pod with `agentpool In [gpupool]`.
* DaemonSet-style pending pods pinned to existing nodes leave the pods to schedule with the affinity warning."""
import functools

import numpy as np
import pytest
import torch

import golden_util as gu
import node_affinity_cases as nc
import sel_oracle
from test_gpu_anti_affinity import with_anti_affinity
from test_gpu_selector_states import tick as tick2
from test_gpu_selectors import assert_tick_equal, eligible_for_first_pool, run_sel, to_np
from test_gpu_selectors_host import NO_FIT, NO_POOL
from test_gpu_taints import _kube, assert_maintain_restated, with_taints
from test_node_affinity_cpu import AFFINITY, r_affinity, r_pool_affinity
from test_taints_cpu import UNTOLERATED, restated_blocking, restated_tolerates

pytestmark = pytest.mark.gpu

F64, I32, U8 = torch.float64, torch.int32, torch.uint8


@functools.lru_cache(maxsize=None)
def case_and_oracle(kind, D):
    c = nc.make_case(kind, D)
    used_o = c["used0"].copy()
    return c, sel_oracle.scale_up_sel(c, used_o), used_o


@pytest.mark.parametrize("D", nc.DIMS)
@pytest.mark.parametrize("kind", nc.KINDS)
def test_affinity_classes_through_the_sel_kernels(engine, kind, D):
    c, o, used_o = case_and_oracle(kind, D)
    g, used, recs = run_sel(engine, c, {})
    assert_tick_equal(g, o, used, used_o)
    assert g["sel_hits"] >= int((o["placed"] >= 0).sum())
    chained = any(r["chained"] for r in recs)
    if chained:
        assert eligible_for_first_pool(c, o)
    if kind == "first_avoided":   # most pods may not use the first pool visited: no chained first bin pass
        assert not eligible_for_first_pool(c, o) and not chained
    req = engine.dev(c["req"], F64)
    pc = engine.dev(c["pod_class"], U8)
    m, ev = engine.feasible_mask_sel(req, engine.dev(c["unit_all"], F64), pc, c["pool_match_all"], c["classes"])
    mo, evo = sel_oracle.feasible_mask_sel(c["req"], c["unit_all"], c["pool_match_all"], c["pod_class"])
    np.testing.assert_array_equal(to_np(m), mo)
    assert int(to_np(ev)[0]) == evo
    if kind == "daemonset":       # pinned to existing nodes: no pool, so not feasible
        pinned = np.asarray([p.node_affinity is not None for p in c["pods"]])
        assert pinned.any() and not mo[pinned].any()
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
    # affinity-sensitive: the classes of selectors and taints alone answer differently (except without affinity)
    from kubernetes_acs_engine_autoscaler_b200 import snapshot
    alone = snapshot.selector_classes(c["pods"], c["nodes"], c["pools"], taints=True)
    sc = dict(c, pod_class=alone.pod_class, node_match=alone.node_match, pool_match_all=alone.pool_match,
              pool_match_ordered=alone.pool_match[c["order"]], classes=alone.classes)
    oa = sel_oracle.scale_up_sel(sc, c["used0"].copy())
    same = all(np.array_equal(np.asarray(oa[k]), np.asarray(o[k])) for k in ("feasible", "placed", "acc_pool", "new_size"))
    assert same == (kind == "no_affinity")


# ---------------------------------------------------------------- through Cluster.loop_logic
TICKS = gu.load_json("ticks.json.gz")


@pytest.fixture()
def host(tmp_path, monkeypatch, engine):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", engine)
    return monkeypatch


def tick(state, engine, selectors="1", states_on="1", taints="1", anti="0", affinity="1"):
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_NODE_TAINTS", taints)
        mp.setenv("ACSFIT_POD_ANTI_AFFINITY", anti)
        mp.setenv("ACSFIT_NODE_AFFINITY", affinity)
        return tick2(state, engine, selectors, states_on)


@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_switches_on_without_affinity_is_the_reference_tick(host, engine, state):
    off = tick(state, engine, "0", "0", "0", "0", "0")
    on = tick(state, engine, "1", "1", "1", "1", "1")
    gu.assert_tick_matches(on, state["expected"])
    assert on["launches"] == off["launches"]
    assert on["node_flags_sent"] == off["node_flags_sent"]


def with_affinity(state, variant, anti):
    """the recorded tick with selectors and taints (with_taints), a numeric node label `gen`, optionally pod
    anti-affinity terms (with_anti_affinity), and required node affinity on some unassigned pending pods"""
    s = with_taints(state, variant)
    if anti:
        s = with_anti_affinity(s, variant)
    pools = [k[:-len("VMSize")] for k in s["arm_parameters"] if k.endswith("VMSize") and k != "masterVMSize"]
    types_ = [s["arm_parameters"][p + "VMSize"]["value"] for p in pools]
    names = [n["metadata"]["name"] for n in s["nodes"]]
    for i, n in enumerate(s["nodes"]):
        gen = ("0", "3", "+5", "x", None, "007")[(i + variant) % 6]
        if gen is not None:
            n["metadata"].setdefault("labels", {})["gen"] = gen

    def expr(*reqs):
        return {"matchExpressions": [dict(zip(("key", "operator", "values"), r)) for r in reqs]}
    choices = [
        lambda i: None,
        lambda i: [expr(("agentpool", "In", [pools[i % len(pools)]]))],
        lambda i: [expr(("agentpool", "NotIn", [pools[(i + 1) % len(pools)]]))],
        lambda i: [expr(("gen", "Gt", ["2"]))],
        lambda i: [expr(("gen", "Lt", ["4"]), ("agentpool", "Exists", None))],
        lambda i: [{"matchFields": [{"key": "metadata.name", "operator": "In", "values": [names[i % len(names)]]}]}]
        if names else None,
        lambda i: [expr(("kubernetes.io/hostname", "NotIn", [names[i % len(names)]]))] if names else None,
        lambda i: [expr(("agentpool", "In", ["gpupool"])), expr(("beta.kubernetes.io/instance-type", "In",
                                                                  [types_[(i + variant) % len(types_)]]))],
    ]
    for i, p in enumerate(s["pods"]):
        if p["status"]["phase"] == "Pending" and not p["spec"].get("nodeName"):
            terms = choices[(i + variant) % len(choices)](i)
            if terms is not None:
                for t in terms:  # drop the absent values of Exists
                    for e in t.get("matchExpressions", ()):
                        if e["values"] is None:
                            del e["values"]
                p["spec"].setdefault("affinity", {})["nodeAffinity"] = {
                    "requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": terms}}
    return s


def raw_affinity(pod):
    return pod.original.obj["spec"].get("affinity")


def tolerated(pod, taints):
    return all(restated_tolerates(pod.tolerations, t) for t in taints)


def node_ok(node, pod):
    """selector, node affinity and tolerations all admit the node (restated)"""
    return all(node.selectors.get(k) == v for k, v in pod.selectors.items()) and \
        r_affinity(raw_affinity(pod), node.selectors, node.name) and tolerated(pod, restated_blocking(node.taints))


def restate(state, anti):
    """the scale-up half of the tick with the selector, node-affinity, taint and (with `anti`) pod anti-affinity rules,
    pair by pair, in plain Python on the product's kube types.  Returns (exception name or None, scale_pools calls,
    used, warnings, names of the pods to schedule)."""
    from kubernetes_acs_engine_autoscaler_b200 import capacity, kube
    from kubernetes_acs_engine_autoscaler_b200.kube import KubePodStatus, KubeResource
    st = state["settings"]
    if not state["nodes"]:
        return None, [], {}, ["Failed to list nodes. Please check kube configuration. Terminating scale loop."], set()
    nodes, pods, pools = _kube(state)
    running = [p for p in pods if p.status in (KubePodStatus.RUNNING, KubePodStatus.CONTAINER_CREATING)
               or (p.status == KubePodStatus.PENDING and p.node_name)]
    used = [KubeResource() for _ in nodes]
    on_node = [[] for _ in nodes]
    for p in running:
        for k, n in enumerate(nodes):
            if n.name == p.node_name:
                used[k] = used[k] + p.resources
                on_node[k].append(p)
    pool_taints = {}
    for pool in pools:
        sets = [restated_blocking(n.taints) for n in pool.nodes]
        pool_taints[pool.name] = set.intersection(*sets) if sets else set()

    def selected(pool, pod):
        return all(pool.labels.get(k) == v for k, v in pod.selectors.items())

    def affine(pool, pod):
        return r_pool_affinity(raw_affinity(pod), pool.labels)

    def pool_ok(pool, pod):
        return selected(pool, pod) and affine(pool, pod) and tolerated(pod, pool_taints[pool.name])

    def fits_unit(pool, pod):
        return (capacity.RESOURCE_SPEC[pool.instance_type] - pod.resources).possible

    def selects(owner, q):
        return any(q.namespace in ns and kube.selector_matches(sel, q.labels) for ns, sel in owner.anti_affinity_terms)

    def blocked(p, there):
        return anti and any(selects(p, q) or selects(q, p) for q in there)

    warnings, to_schedule = [], []
    for p in pods:
        if p.status != KubePodStatus.PENDING or p.node_name:
            continue
        if any(pool_ok(pool, p) and fits_unit(pool, p) for pool in pools):
            to_schedule.append(p)
        elif any(selected(pool, p) and affine(pool, p) and fits_unit(pool, p) for pool in pools):
            warnings.append(UNTOLERATED % p.name)
        elif any(selected(pool, p) and fits_unit(pool, p) for pool in pools):
            warnings.append(AFFINITY % p.name)
        elif p.selectors and any(fits_unit(pool, p) for pool in pools):
            warnings.append(NO_POOL % (p.name, p.selectors))
        else:
            warnings.append(NO_FIT % p.name)
    pending = []
    for p in to_schedule:
        for k, n in enumerate(nodes):
            if node_ok(n, p) and not blocked(p, on_node[k]) and (n.capacity - (used[k] + p.resources)).possible:
                used[k] = used[k] + p.resources
                on_node[k].append(p)
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
                if p in acc or not (pool_ok(pool, p) and (unit - p.resources).possible):
                    continue
                for b, rem in enumerate(bins):
                    if not blocked(p, members[b]) and (rem - p.resources).possible:
                        break
                else:
                    bins.append(unit)
                    members.append([])
                    b = len(bins) - 1
                bins[b] = bins[b] - p.resources
                members[b].append(p)
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
    return exc, calls, used_hex, warnings, {p.name for p in to_schedule}


def assert_maintain(s, got, exc, names):
    """node states and the maintain journal with the affinity-aware match (assert_maintain_restated of the taint
    tests, with this module's node_ok as KubeNode.is_match)"""
    import test_gpu_taints
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(test_gpu_taints, "node_ok", node_ok)
        assert_maintain_restated(s, got, exc, names)


@pytest.mark.parametrize("states_on", ("0", "1"))
@pytest.mark.parametrize("variant", (0, 1, 2))
def test_ticks_with_affinity_match_restatement(host, engine, variant, states_on):
    anti = variant > 0 and states_on == "0"
    differs = ran = affinity_warnings = 0
    for state in TICKS:
        s = with_affinity(state, variant, anti)
        got = tick(s, engine, "1", states_on, "1", "1" if anti else "0", "1")
        exc, calls, used, warnings, names = restate(s, anti)
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
        affinity_warnings += sum(w.endswith("required node affinity. Scheduling skipped.") for w in warn)
        if states_on == "1":
            assert_maintain(s, got, exc, names)
            ran += got["maintain_journal"] is not None
        off = tick(s, engine, "1", states_on, "1", "1" if anti else "0", "0")
        differs += (off["scale_pools_calls"], off["used"], off["exception"], off["state_calls"]) != \
            (got["scale_pools_calls"], got["used"], got["exception"], got["state_calls"])
    assert differs >= 3, differs
    assert affinity_warnings >= 3, affinity_warnings
    assert states_on == "0" or ran >= 5, ran


# ---------------------------------------------------------------- the motivating tick and the DaemonSet tick
def _node(pool, i, itype):
    name = "k8s-%s-16334397-%d" % (pool, i)
    return {"metadata": {"name": name, "creationTimestamp": "2016-08-25T05:13:16Z",
                         "labels": {"beta.kubernetes.io/instance-type": itype, "agentpool": pool,
                                    "failure-domain.beta.kubernetes.io/region": "southcentralus",
                                    "kubernetes.io/hostname": name}}, "spec": {}}


def _pod(name, cpu, phase, node_name=None, affinity_terms=None, kind=None):
    spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": cpu}}}]}
    if node_name:
        spec["nodeName"] = node_name
    if affinity_terms:
        spec["affinity"] = {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {
            "nodeSelectorTerms": affinity_terms}}}
    status = {"phase": phase}
    if phase == "Running":
        status["startTime"] = "2026-09-20T07:00:00Z"
    meta = {"name": name, "namespace": "default", "uid": "uid-" + name, "creationTimestamp": "2026-09-20T07:00:00Z"}
    if kind:
        meta["annotations"] = {"kubernetes.io/created-by": '{"reference": {"kind": "%s"}}' % kind}
    return {"metadata": meta, "spec": spec, "status": status}


def _state(name, nodes, pods, pools, dry_run):
    params = {"masterVMSize": {"value": "Standard_D2_v2"}, "firstConsecutiveStaticIP": {"value": "10.0.0.1"}}
    for pool, itype in pools:
        params[pool + "VMSize"] = {"value": itype}
    return {"name": name, "now": "2026-09-21T12:00:00Z", "nodes": nodes, "pods": pods, "arm_parameters": params,
            "settings": {"idle_threshold": 1800, "spare_agents": 0, "over_provision": 0, "dry_run": dry_run,
                         "ignore_pools": ""}}


@pytest.mark.parametrize("dry_run", [True, False])
def test_pod_pinned_to_the_empty_gpu_pool_grows_it(host, engine, dry_run):
    """pool `agentpool1` (Standard_D2_v2): one old idle node with room.  Pool `gpupool` (Standard_NC6): no node.  One
    pending 1-cpu pod with `agentpool In [gpupool]`."""
    nodes = [_node("agentpool1", 0, "Standard_D2_v2")]
    cpu_node = nodes[0]["metadata"]["name"]
    pods = [_pod("trainer", "1", "Pending",
                 affinity_terms=[{"matchExpressions": [{"key": "agentpool", "operator": "In", "values": ["gpupool"]}]}])]
    s = _state("gpu_affinity", nodes, pods, (("agentpool1", "Standard_D2_v2"), ("gpupool", "Standard_NC6")), dry_run)
    off = tick(s, engine, affinity="0")
    on = tick(s, engine, affinity="1")
    for got in (off, on):
        assert got["exception"] is None and "Pods to schedule: 1" in [m for _, _, m in got["log"]]
    # off: the pod "fits" the CPU node, nothing grows, and the CPU node waits for it
    assert off["scale_pools_calls"] == [] and off["used"][cpu_node] == {"cpu": float(1).hex(), "pods": float(1).hex()}
    # on: the GPU pool grows by one; the CPU node stays empty and is no longer held by the pod
    assert on["scale_pools_calls"] == [{"agentpool1": 1, "gpupool": 1}]
    assert on["used"][cpu_node] == {}
    assert [st for n, st in off["state_calls"] if n == cpu_node] == ["pod-pending"]
    assert [st for n, st in on["state_calls"] if n == cpu_node] == ["under-utilized-drainable"]
    exc, calls, used, warnings, names = restate(s, False)
    assert (exc, calls, used, warnings, names) == (None, on["scale_pools_calls"], on["used"], [], {"trainer"})
    assert_maintain(s, on, None, names)


def test_daemonset_pods_pinned_to_existing_nodes_are_skipped(host, engine):
    """two nodes, each busy with a 1.5-cpu pod; pending DaemonSet pods, each pinned to one node by matchFields (as the
    DaemonSet controller writes them), and one pending 1-cpu pod that fits no node"""
    nodes = [_node("agentpool1", i, "Standard_D2_v2") for i in range(2)]
    names = [n["metadata"]["name"] for n in nodes]
    pods = [_pod("web-%d" % i, "1500m", "Running", names[i]) for i in range(2)]
    pods += [_pod("ds-%d" % i, "100m", "Pending", kind="DaemonSet", affinity_terms=[
        {"matchFields": [{"key": "metadata.name", "operator": "In", "values": [names[i]]}]}]) for i in range(2)]
    pods.append(_pod("app", "1", "Pending"))
    s = _state("daemonset_affinity", nodes, pods, (("agentpool1", "Standard_D2_v2"),), True)
    off = tick(s, engine, affinity="0")
    on = tick(s, engine, affinity="1")
    assert "Pods to schedule: 3" in [m for _, _, m in off["log"]]
    assert "Pods to schedule: 1" in [m for _, _, m in on["log"]]
    warn = [m for lvl, _, m in on["log"] if lvl == "WARNING"]
    assert warn == [AFFINITY % "ds-0", AFFINITY % "ds-1"]
    # off, the DaemonSet pods take room on the first node in the simulation; on, they take none, and the pool grows
    # for the one pod that fits no node only
    running = {"cpu": float(1.5).hex(), "pods": float(1).hex()}
    assert off["used"][names[0]] != running
    assert on["used"] == {names[0]: running, names[1]: running}
    assert on["scale_pools_calls"] == [{"agentpool1": 3}]
    exc, calls, used, warnings, names_ = restate(s, False)
    assert (exc, calls, used, warnings, names_) == (None, on["scale_pools_calls"], on["used"], warn, {"app"})
