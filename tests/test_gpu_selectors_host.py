"""`-m gpu`: the node-selector mode through the public surface -- `Cluster.loop_logic` in dry run on kube-style dicts
with the REAL CUDA engine.

* With the mode on ($ACSFIT_NODE_SELECTORS=1) and no selector anywhere, every recorded reference tick still matches
  the reference exactly (scale_pools arguments, used_capacity bits, node states, adapter calls, the whole log) and
  makes the same kernel launches as with the mode off.
* With selectors added to the recorded ticks (nodes labelled `agentpool` as acs-engine does; pods pinned to pools,
  instance types, hosts, or to nothing), the tick equals a plain-Python restatement of the upstream rules on
  KubeNode.is_match / KubeResource: exception, scale_pools arguments, used_capacity key sets and bits, warnings.
* Scaler.fulfill_pending in the non-raising insufficient-scale mode tells the notifier once per selector."""
import copy
import types

import pytest

import golden_util as gu

pytestmark = pytest.mark.gpu

TICKS = gu.load_json("ticks.json.gz")
NO_POOL = "Pending pod %s cannot fit: no agent pool matches its node selector %s. Scheduling skipped."
NO_FIT = ("Pending pod %s cannot fit. Please check that requested resource amount is consistent with node size."
          "Scheduling skipped.")


@pytest.fixture()
def host(tmp_path, monkeypatch, engine):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", engine)
    return monkeypatch


@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_mode_on_without_selectors_is_the_reference_tick(host, engine, state):
    runs = []
    for on in ("0", "1"):
        n0 = engine.launch_count
        got = tick(state, on)
        runs.append(engine.launch_count - n0)
        gu.assert_tick_matches(got, state["expected"])
    assert runs[0] == runs[1], runs


def tick(state, mode):
    """one recorded tick through gu.run_tick with $ACSFIT_NODE_SELECTORS = mode, in its own monkeypatch scope (run_tick
    wraps EngineScaler methods: wrappers must not pile up over the ticks of one test)"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_NODE_SELECTORS", mode)
        return gu.run_tick(state, mp)


def pool_of(node_name):
    return node_name.split("-")[1]


def with_selectors(state, variant):
    """the recorded tick with `agentpool` node labels and nodeSelectors on the unassigned pending pods"""
    s = copy.deepcopy(state)
    pools = [k[:-len("VMSize")] for k in s["arm_parameters"] if k.endswith("VMSize") and k != "masterVMSize"]
    types_ = [s["arm_parameters"][p + "VMSize"]["value"] for p in pools]
    hosts = []
    for n in s["nodes"]:
        n["metadata"].setdefault("labels", {})["agentpool"] = pool_of(n["metadata"]["name"])
        hosts.append(n["metadata"]["name"])
    choices = [lambda i: {}, lambda i: {"agentpool": pools[i % len(pools)]},
               lambda i: {"agentpool": pools[-1 - i % len(pools)], "beta.kubernetes.io/instance-type": types_[-1 - i % len(pools)]},
               lambda i: {"beta.kubernetes.io/instance-type": types_[(i + variant) % len(types_)]},
               lambda i: {"kubernetes.io/hostname": hosts[i % len(hosts)]} if hosts else {},
               lambda i: {"agentpool": "gpupool"}]
    for i, p in enumerate(s["pods"]):
        if p["status"]["phase"] == "Pending" and not p["spec"].get("nodeName"):
            sel = choices[(i + variant) % len(choices)](i)
            if sel:
                p["spec"]["nodeSelector"] = sel
    return s


def restate(state):
    """the scale-up half of the tick with the upstream selector rules, in plain Python on the product's kube types
    (whose parsing the recorded ticks pin).  Returns (exception name or None, scale_pools calls, used, warnings)."""
    from kubernetes_acs_engine_autoscaler_b200 import capacity, utils
    from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod, KubePodStatus, KubeResource
    st = state["settings"]
    if not state["nodes"]:  # loop_logic stops before anything else when the node list is empty
        return None, [], {}, ["Failed to list nodes. Please check kube configuration. Terminating scale loop."]
    journal = []
    nodes = []
    for o in state["nodes"]:
        n = KubeNode(gu.FakeKubeObject(o, journal, "node"))
        n.capacity = capacity.get_capacity_for_instance_type(n.instance_type)
        if utils.is_agent(n):
            nodes.append(n)
    pods = [KubePod(gu.FakeKubeObject(o, journal, "pod")) for o in state["pods"]]
    running = [p for p in pods if p.status in (KubePodStatus.RUNNING, KubePodStatus.CONTAINER_CREATING)
               or (p.status == KubePodStatus.PENDING and p.node_name)]
    used = [KubeResource() for _ in nodes]
    for p in running:
        for k, n in enumerate(nodes):
            if n.name == p.node_name:
                used[k] = used[k] + p.resources
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

    def matches(labels, pod):
        return all(labels.get(k) == v for k, v in pod.selectors.items())

    def fits_unit(pool, pod):
        return (capacity.RESOURCE_SPEC[pool.instance_type] - pod.resources).possible

    warnings, to_schedule = [], []
    for p in pods:
        if p.status != KubePodStatus.PENDING or p.node_name:
            continue
        if any(matches(pool.labels, p) and fits_unit(pool, p) for pool in pools):
            to_schedule.append(p)
        elif p.selectors and any(fits_unit(pool, p) for pool in pools):
            warnings.append(NO_POOL % (p.name, p.selectors))
        else:
            warnings.append(NO_FIT % p.name)
    pending = []
    for p in to_schedule:
        for k, n in enumerate(nodes):
            if KubeNode.is_match(n, p) and (n.capacity - (used[k] + p.resources)).possible:
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
                if p in acc or not (matches(pool.labels, p) and (unit - p.resources).possible):
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
        if left:  # the reference's undefined-name raise: AttributeError first when there is no notifier
            warnings.append("Failed to scale sufficiently.")
            exc = "NameError" if st.get("notifier") == "recording" else "AttributeError"
        else:
            calls.append(sizes)
    used_hex = {n.name: {k: float(v).hex() for k, v in used[i].raw.items()} for i, n in enumerate(nodes)}
    return exc, calls, used_hex, warnings


@pytest.mark.parametrize("variant", (0, 1, 2))
def test_loop_logic_with_selectors_matches_restatement(host, variant):
    differs = 0
    for state in TICKS:
        if not state["settings"].get("scale_up", True):
            continue
        s = with_selectors(state, variant)
        got = tick(s, "1")
        exc, calls, used, warnings = restate(s)
        assert (got["exception"] or [None])[0] == exc, s["name"]
        assert got["scale_pools_calls"] == calls, s["name"]
        assert got["used"] == used, s["name"]
        assert [m for lvl, _, m in got["log"] if lvl == "WARNING"] == warnings, s["name"]
        # the same tick with the mode off ignores the selectors: most ticks must come out differently
        off = tick(s, "0")
        differs += (off["scale_pools_calls"], off["used"], off["exception"]) != (got["scale_pools_calls"], got["used"], got["exception"])
    assert differs >= len(TICKS) // 3


def test_failed_to_scale_is_reported_per_selector(host):
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.engine_scaler import EngineScaler
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod
    j = []
    node = {"metadata": {"name": "k8s-agentpool1-16334397-0", "creationTimestamp": "2026-09-20T07:00:00Z",
                         "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2", "agentpool": "agentpool1",
                                    "failure-domain.beta.kubernetes.io/region": "southcentralus"}}, "spec": {}}
    n = KubeNode(gu.FakeKubeObject(node, j, "node"))
    n.capacity = capacity.get_capacity_for_instance_type(n.instance_type)
    sels = [{}, {"agentpool": "agentpool1"}, {}, {"agentpool": "agentpool1"}, {}, {"agentpool": "agentpool2"},
            {"agentpool": "agentpool2"}, {}]
    pods = []
    for i, sel in enumerate(sels):
        o = {"metadata": {"name": "p%d" % i, "namespace": "ns", "uid": "u%d" % i, "creationTimestamp": "2026-09-21T07:00:00Z"},
             "spec": {"containers": [{"name": "c", "resources": {"requests": {"cpu": "1500m"}}}], "nodeSelector": sel},
             "status": {"phase": "Pending"}}
        pods.append(KubePod(gu.FakeKubeObject(o, j, "pod")))
    params = {"agentpool1VMSize": {"value": "Standard_D2_v2"}, "agentpool2VMSize": {"value": "Standard_D2_v2"},
              "masterVMSize": {"value": "Standard_D2_v2"}}
    failed = []
    notifier = types.SimpleNamespace(notify_failed_to_scale=lambda sel, left: failed.append((sel, [p.name for p in left])),
                                     notify_scale=lambda *a: None)
    s = EngineScaler("rg", [n], 0, 1, 1800, True, None, {}, dict(params), "", notifier, node_selectors=True)
    for pool in s.agent_pools:
        pool.max_size = {"agentpool1": 2, "agentpool2": 1}[pool.name]  # one more instance each
    s.REFERENCE_RAISE_ON_INSUFFICIENT = False
    calls = []
    s.scale_pools = lambda sizes: calls.append(dict(sizes))
    s.fulfill_pending(pods)
    # one 1.5-cpu pod per Standard_D2_v2 bin, one new instance per pool: agentpool1 (visited first) accounts p0,
    # agentpool2 (which only its own pins and the unpinned pods match) accounts p2; the rest is reported per selector
    assert calls == [{"agentpool1": 2, "agentpool2": 1}]
    assert failed == [({"agentpool": "agentpool1"}, ["p1", "p3"]), ({}, ["p4", "p7"]),
                      ({"agentpool": "agentpool2"}, ["p5", "p6"])]
