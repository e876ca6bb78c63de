"""`-m gpu`: Cluster(topology_spread=True) end to end on the recorded reference ticks with spread constraints overlaid,
against a plain-Python restatement of the scale-up half of the tick (PodTopologySpread's filter, pod by pod and node
by node, on the product's kube types): the scale_pools calls, every node's used capacity and the exception.  The
overlay adds a master node (with pods of the groups on it), group labels and a `rev` label on every pod, and on the
pending pods constraints that vary maxSkew, the selector (null included), matchLabelKeys, minDomains, both policies and
ScheduleAnyway entries.  Only the topology-spread switch is on, so the pods land by resources and the rule alone."""
import copy

import pytest

import golden_util as gu
from test_gpu_taints import _kube

pytestmark = pytest.mark.gpu

TICKS = [s for s in gu.load_json("ticks.json.gz") if s["nodes"]]
HOST = "kubernetes.io/hostname"


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from kubernetes_acs_engine_autoscaler_b200 import build as acs_build
    acs_build.build()
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    e = Engine(0, watchdog_ms=15000)
    yield e
    e.close()


@pytest.fixture()
def host(tmp_path, monkeypatch, engine):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", engine)
    return monkeypatch


def tick(state, engine, on):
    from test_gpu_selector_states import tick as tick2
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_TOPOLOGY_SPREAD", on)
        return tick2(state, engine, "0", "0")


def with_spread(state, variant):
    s = copy.deepcopy(state)
    first = s["nodes"][0]
    master_name = "k8s-master-%s-0" % first["metadata"]["name"].split("-")[2]
    labels = dict(first["metadata"].get("labels", {}))
    labels[HOST] = master_name
    s["nodes"].append({"metadata": {"name": master_name, "creationTimestamp": first["metadata"]["creationTimestamp"],
                                    "labels": labels},
                       "spec": {"taints": [{"key": "node-role.kubernetes.io/master", "effect": "NoSchedule"}]}})
    for i, n in enumerate(s["nodes"][:-1]):
        if (i + variant) % 4 == 0:
            n["metadata"].setdefault("labels", {})["zone"] = "a"
    for i, p in enumerate(s["pods"]):
        p["metadata"]["labels"] = dict(p["metadata"].get("labels") or {}, app="g%d" % ((i + variant) % 3),
                                       rev="r%d" % (i % 2))
    ns = s["pods"][0]["metadata"]["namespace"] if s["pods"] else "default"
    for j in range(variant + 1):  # pods of the groups on the master: it bounds the minimum
        s["pods"].append({"metadata": {"name": "on-master-%d" % j, "namespace": ns, "uid": "uid-on-master-%d" % j,
                                       "labels": {"app": "g%d" % j, "rev": "r0"},
                                       "creationTimestamp": "2016-08-25T05:13:16Z"},
                          "spec": {"nodeName": master_name, "containers": [
                              {"name": "c", "resources": {"requests": {"cpu": "10m"}}}]},
                          "status": {"phase": "Running"}})

    def sel(g):
        return {"matchLabels": {"app": "g%d" % g}}

    def c(**kw):
        out = {"maxSkew": 1, "topologyKey": HOST, "whenUnsatisfiable": "DoNotSchedule"}
        out.update(kw)
        return out
    choices = [
        lambda i: None,
        lambda i: [c(labelSelector=sel(i % 3))],
        lambda i: [c(maxSkew=2, labelSelector=sel(i % 3))],
        lambda i: [c(labelSelector=sel(i % 3), matchLabelKeys=["rev"])],
        lambda i: [c(labelSelector=sel(i % 3), nodeTaintsPolicy="Honor")],
        lambda i: [c(labelSelector=sel(i % 3), minDomains=1000)],
        lambda i: [c(labelSelector=None)],
        lambda i: [c(labelSelector={"matchExpressions": [{"key": "app", "operator": "In", "values": ["g0", "g1"]}]},
                     nodeAffinityPolicy="Ignore"),
                   c(labelSelector=sel(0), topologyKey="zone", maxSkew=1)],
        lambda i: [c(labelSelector=sel(i % 3), whenUnsatisfiable="ScheduleAnyway")],
    ]
    for i, p in enumerate(s["pods"]):
        if p["status"]["phase"] == "Pending" and not p["spec"].get("nodeName"):
            cons = choices[(i + variant) % len(choices)](i)
            if cons is not None:
                p["spec"]["topologySpreadConstraints"] = cons
            if (i + variant) % 5 == 0:
                p["spec"]["nodeSelector"] = {"zone": "a"}  # no landing rule here; a domain rule with Honor
    return s


def restate(state):
    """(exception name or None, scale_pools calls, used) of the scale-up half with hostname topology spread"""
    from kubernetes_acs_engine_autoscaler_b200 import capacity, kube, utils
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePodStatus, KubeResource
    st = state["settings"]
    nodes, pods, pools = _kube(state)
    listed = [KubeNode(gu.FakeKubeObject(o, [], "node")) for o in state["nodes"]]
    masters = [n for n in listed if not utils.is_agent(n)]
    every = nodes + masters
    running = [p for p in pods if p.status in (KubePodStatus.RUNNING, KubePodStatus.CONTAINER_CREATING)
               or (p.status == KubePodStatus.PENDING and p.node_name)]
    used = [KubeResource() for _ in nodes]
    on_node = [[] for _ in every]
    for p in running:
        for k, n in enumerate(every):
            if n.name == p.node_name:
                if k < len(nodes):
                    used[k] = used[k] + p.resources
                on_node[k].append(p)

    def raw(p):
        return p.original.obj["spec"].get("topologySpreadConstraints") or []

    def constraint(p):
        """(maxSkew, selector or None, minDomains, honor affinity, honor taints) of the hostname DoNotSchedule entry"""
        for e in raw(p):
            if e["topologyKey"] == HOST and e["whenUnsatisfiable"] == "DoNotSchedule":
                sel = e.get("labelSelector")
                selector = None
                if sel is not None:
                    selector = kube.label_selector(sel, "t")
                    extra = tuple((k, "In", (p.labels[k],)) for k in e.get("matchLabelKeys", ()) if k in p.labels)
                    selector = (selector[0], tuple(sorted(selector[1] + extra)))
                return (e["maxSkew"], selector, e.get("minDomains", 1),
                        e.get("nodeAffinityPolicy", "Honor") == "Honor", e.get("nodeTaintsPolicy", "Ignore") == "Honor")
        return None

    def selects(p, c, q):
        return c[1] is not None and q.namespace == p.namespace and kube.selector_matches(c[1], q.labels)

    def domain(p, c, n):
        if c[3] and not all(n.selectors.get(k) == v for k, v in p.selectors.items()):
            return False
        if c[3] and p.node_affinity is not None and not kube.node_affinity_matches(p.node_affinity, n.selectors, n.name):
            return False
        return not c[4] or kube.tolerates_all(p.tolerations, kube.blocking_taints(n.taints))

    def spread_ok(p, k):
        c = constraint(p)
        if c is None:
            return True
        cnt = [sum(selects(p, c, q) for q in there) for there in on_node]
        doms = [m for m, n in enumerate(every) if domain(p, c, n)]
        low = 0 if len(doms) < c[2] else min(cnt[m] for m in doms)
        return cnt[k] + int(selects(p, c, p)) - low <= c[0]

    to_schedule = [p for p in pods if p.status == KubePodStatus.PENDING and not p.node_name and
                   any((capacity.RESOURCE_SPEC[pool.instance_type] - p.resources).possible for pool in pools)]
    pending = []
    for p in to_schedule:
        for k, n in enumerate(nodes):
            if (n.capacity - (used[k] + p.resources)).possible and spread_ok(p, k):
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
                if p in acc or not (unit - p.resources).possible:
                    continue
                c = constraint(p)
                for b, rem in enumerate(bins):  # a new node: count from 0, minimum taken as 0
                    if (rem - p.resources).possible and \
                            (c is None or sum(selects(p, c, q) for q in members[b]) + selects(p, c, p) <= c[0]):
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
            exc = "NameError" if st.get("notifier") == "recording" else "AttributeError"
        else:
            calls.append(sizes)
    used_hex = {n.name: {k: float(v).hex() for k, v in used[i].raw.items()} for i, n in enumerate(nodes)}
    return exc, calls, used_hex


@pytest.mark.parametrize("variant", (0, 1, 2))
def test_ticks_with_spread_match_restatement(host, engine, variant):
    differs = 0
    for state in TICKS:
        s = with_spread(state, variant)
        got = tick(s, engine, "1")
        exc, calls, used = restate(s)
        if s["settings"].get("scale_up", True):
            assert got["scale_pools_calls"] == calls, s["name"]
            assert got["used"] == used, s["name"]
            assert (got["exception"] or [None])[0] == exc, s["name"]
        off = tick(s, engine, "0")
        differs += (off["scale_pools_calls"], off["used"], off["exception"]) != \
            (got["scale_pools_calls"], got["used"], got["exception"])
    assert differs >= 5, differs  # the rule changes the outcome of many ticks
