"""`-m "not gpu"`: the host side of Cluster(topology_spread=True) -- topologySpreadConstraints with topologyKey
kubernetes.io/hostname and whenUnsatisfiable DoNotSchedule.

* kube.topology_spread_constraint: the honoured constraint, matchLabelKeys, the policies, and every validation rule
  (ValueError naming the pod).
* snapshot.topology_spread bit for bit against a per-(pod, node) plain-Python restatement: keys, selectors with
  matchLabelKeys, namespaces, null selectors, pods that do not select themselves, both policies, the master as a
  domain, minDomains, and 64 keys accepted, a 65th refused.
* The plain-C oracle (tests/ts_oracle.c): equal to tests/pa_oracle.c without keys, and hand-worked ticks: stacked
  replicas, a pinned pool whose minimum rises, a master that holds the minimum at 0, and the bins.
* The switch (environment and pass-through)."""
from types import SimpleNamespace

import numpy as np
import pytest

import aa_cases as ac
import golden_util as gu
import pa_oracle
import ts_oracle
from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot

HOST = "kubernetes.io/hostname"
INT32_MAX = 2 ** 31 - 1
WEB = {"matchLabels": {"app": "web"}}


def tsc(selector=WEB, skew=1, when="DoNotSchedule", topology=HOST, **extra):
    c = {"maxSkew": skew, "whenUnsatisfiable": when, "topologyKey": topology}
    if selector is not None:
        c["labelSelector"] = selector
    c.update(extra)
    return c


def pod_obj(name, labels=None, constraints=None, namespace="ns"):
    spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "1"}}}]}
    if constraints is not None:
        spec["topologySpreadConstraints"] = constraints
    return {"metadata": {"name": name, "namespace": namespace, "uid": "u-" + name, "labels": dict(labels or {}),
                         "creationTimestamp": "2026-09-21T07:00:00Z"}, "spec": spec, "status": {"phase": "Pending"}}


def parse(constraints, labels=None):
    return kube.topology_spread_constraint(constraints, labels or {}, "pod p")


# ---------------------------------------------------------------- parsing
def test_honoured_constraint_and_defaults():
    c = parse([tsc(skew=2, topology="topology.kubernetes.io/zone"), tsc(when="ScheduleAnyway"), tsc(skew=3)])
    assert c == (3, ((("app", "web"),), ()), 1, True, False)
    assert (c.max_skew, c.min_domains, c.honor_affinity, c.honor_taints) == (3, 1, True, False)
    assert parse(None) is None and parse([]) is None
    assert parse([tsc(topology="zone"), tsc(when="ScheduleAnyway")]) is None
    c = parse([tsc(minDomains=3, nodeAffinityPolicy="Ignore", nodeTaintsPolicy="Honor")])
    assert (c.min_domains, c.honor_affinity, c.honor_taints) == (3, False, True)
    assert parse([tsc(selector=None)]).selector is None


def test_match_label_keys_add_the_pods_own_values():
    c = parse([tsc(matchLabelKeys=["rev", "absent"])], {"app": "web", "rev": "7"})
    assert c.selector == ((("app", "web"),), (("rev", "In", ("7",)),))
    sel = {"matchLabels": {"app": "web"}, "matchExpressions": [{"key": "tier", "operator": "Exists"}]}
    c = parse([tsc(selector=sel, matchLabelKeys=["rev"])], {"rev": "1"})
    assert c.selector == ((("app", "web"),), (("rev", "In", ("1",)), ("tier", "Exists", ())))
    assert parse([tsc(matchLabelKeys=["rev"])], {}).selector == ((("app", "web"),), ())


@pytest.mark.parametrize("bad", [
    {"x": 1},
    [tsc(skew=0)], [tsc(skew=-1)], [tsc(skew=1.0)], [tsc(skew=True)], [tsc(skew="1")], [{"whenUnsatisfiable": "DoNotSchedule", "topologyKey": HOST}],
    [tsc(when="Never")], [tsc(when=None)],
    [tsc(topology="")], [tsc(topology=None)],
    [tsc(), tsc(skew=2)], [tsc(when="ScheduleAnyway"), tsc(skew=2, when="ScheduleAnyway")],
    [tsc(minDomains=0)], [tsc(minDomains=2, when="ScheduleAnyway")], [tsc(minDomains="2")],
    [tsc(matchLabelKeys=["app"])], [tsc(selector={"matchExpressions": [{"key": "rev", "operator": "Exists"}]},
                                        matchLabelKeys=["rev"])],
    [tsc(selector=None, matchLabelKeys=["rev"])], [tsc(matchLabelKeys="rev")],
    [tsc(nodeAffinityPolicy="honor")], [tsc(nodeTaintsPolicy="Always")],
    [tsc(selector={"matchExpressions": [{"key": "app", "operator": "In"}]})],
    [tsc(topology="zone", skew=0)],  # other constraints are validated too
])
def test_malformed_constraints_raise_naming_the_pod(bad):
    p = kube.KubePod(gu.FakeKubeObject(pod_obj("broken", {"app": "web"}, bad), [], "pod"))
    with pytest.raises(ValueError, match="broken"):
        p.topology_spread


def test_property_on_kube_pods():
    p = kube.KubePod(gu.FakeKubeObject(pod_obj("a", {"app": "web", "rev": "2"}, [tsc(matchLabelKeys=["rev"])]), [],
                                       "pod"))
    assert p.topology_spread == (1, ((("app", "web"),), (("rev", "In", ("2",)),)), 1, True, False)
    assert kube.KubePod(gu.FakeKubeObject(pod_obj("b"), [], "pod")).topology_spread is None


# ---------------------------------------------------------------- the builder
def fake_pod(name, ns, labels, constraints=None, node=None, selectors=None, tolerations=(), node_affinity=None):
    return SimpleNamespace(name=name, namespace=ns, labels=labels, node_name=node, selectors=selectors or {},
                           tolerations=list(tolerations), node_affinity=node_affinity,
                           topology_spread=kube.topology_spread_constraint(constraints, labels, "pod " + name))


def fake_node(name, labels=None, taints=()):
    return SimpleNamespace(name=name, selectors=dict(labels or {}), taints=list(taints))


NO_SCHED = {"key": "dedicated", "value": "gpu", "effect": "NoSchedule"}
TOLERATE = {"key": "dedicated", "operator": "Exists"}
AFF_POOL_A = (((("pool", "In", ("a",)),), ()),)  # kube.node_affinity_terms' canonical form


def generated(seed, n_sched=90, n_run=300, n_nodes=30, n_other=2):
    rng = np.random.default_rng(seed)
    apps, nss = ["a%d" % i for i in range(4)], ["n0", "n1"]
    sels = [{"matchLabels": {"app": a}} for a in apps] + \
        [{"matchExpressions": [{"key": "tier", "operator": "In", "values": ["t0", "t1"]}]},
         {"matchExpressions": [{"key": "app", "operator": "NotIn", "values": ["a0"]}]}, None]

    def mk(i, node=None):
        labels = {"app": apps[int(rng.integers(len(apps)))]}
        if rng.random() < 0.5:
            labels["tier"] = "t%d" % rng.integers(3)
        if rng.random() < 0.5:
            labels["rev"] = "r%d" % rng.integers(2)
        constraints = None
        if rng.random() < 0.6:
            extra = {}
            if rng.random() < 0.3:
                extra["nodeAffinityPolicy"] = "Ignore"
            if rng.random() < 0.3:
                extra["nodeTaintsPolicy"] = "Honor"
            if rng.random() < 0.2:
                extra["minDomains"] = int(rng.integers(1, 60))
            sel = sels[int(rng.integers(len(sels)))]
            if sel is not None and "matchLabels" in sel and rng.random() < 0.4:
                extra["matchLabelKeys"] = ["rev"]
            constraints = [tsc(selector=sel, skew=int(rng.integers(1, 3)), **extra)]
            if rng.random() < 0.2:
                constraints.append(tsc(selector=sel, topology="zone"))
        selectors = {"pool": "a"} if rng.random() < 0.2 else None
        tol = [TOLERATE] if rng.random() < 0.3 else []
        aff = AFF_POOL_A if rng.random() < 0.15 else None
        return fake_pod("p%d" % i, nss[int(rng.integers(2))], labels, constraints, node, selectors, tol, aff)
    nodes = [fake_node("node%d" % n, {"pool": "ab"[n % 2]}, [NO_SCHED] if n % 5 == 0 else []) for n in range(n_nodes)]
    other = [fake_node("master%d" % n, {"pool": "m"}, [{"key": "master", "effect": "NoSchedule"}])
             for n in range(n_other)]
    names = [n.name for n in nodes + other] + ["gone0", "gone1"]
    sched = [mk(i) for i in range(n_sched)]
    running = [mk(n_sched + i, names[int(rng.integers(len(names)))]) for i in range(n_run)]
    return sched, nodes, other, running


def restated(sched, nodes, other, running):
    """per (pod, node): the keys, skews, matches, counts, domains and floors, straight from the definitions"""
    every = nodes + other

    def selects(ns, sel, q):
        return sel is not None and q.namespace == ns and kube.selector_matches(sel, q.labels)

    def domain(p, c, n):
        ok = True
        if c.honor_affinity:
            ok = all(n.selectors.get(k) == v for k, v in p.selectors.items()) and \
                kube.node_affinity_matches(p.node_affinity, n.selectors, n.name) if p.node_affinity is not None else \
                all(n.selectors.get(k) == v for k, v in p.selectors.items())
        if c.honor_taints:
            ok = ok and kube.tolerates_all(p.tolerations, kube.blocking_taints(n.taints))
        return ok
    keys, key_of = [], []
    for p in sched:
        c = p.topology_spread
        if c is None:
            key_of.append(0xFF)
            continue
        k = (p.namespace, c.selector, tuple(domain(p, c, n) for n in every), c.min_domains)
        if k not in keys:
            keys.append(k)
        key_of.append(keys.index(k))
    matches = [sum(1 << k for k, (ns, sel, _, _) in enumerate(keys) if selects(ns, sel, q)) for q in sched]
    skew = [0 if k == 0xFF else p.topology_spread.max_skew - ((m >> k) & 1) for p, k, m in zip(sched, key_of, matches)]
    counts = [[sum(1 for q in running if q.node_name == n.name and selects(ns, sel, q)) for n in every]
              for ns, sel, _, _ in keys]
    domain_bits = [sum(1 << k for k, key in enumerate(keys) if key[2][i]) for i in range(len(nodes))]
    floor = []
    for k, (_, _, dom, md) in enumerate(keys):
        outside = [counts[k][len(nodes) + j] for j in range(len(other)) if dom[len(nodes) + j]]
        floor.append(0 if sum(dom) < md else min(outside) if outside else INT32_MAX)
    return keys, key_of, skew, matches, [row[:len(nodes)] for row in counts], domain_bits, floor


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_builder_matches_restatement(seed):
    sched, nodes, other, running = generated(seed)
    ts = snapshot.topology_spread(sched, nodes, running, other)
    keys, key_of, skew, matches, counts, domain_bits, floor = restated(sched, nodes, other, running)
    assert [(ns, sel, dom, md) for ns, sel, dom, md in ts.keys] == \
        [(ns, sel, np.asarray(dom, bool).tobytes(), md) for ns, sel, dom, md in keys]
    assert len(keys) > 5 and 0 in floor
    assert ts.pod_key.tolist() == key_of
    assert ts.pod_skew.tolist() == skew
    assert ts.pod_matches.tolist() == matches
    assert ts.node_count.tolist() == counts
    assert ts.node_domain.tolist() == domain_bits
    assert ts.floor.tolist() == floor
    assert not ts.trivial and snapshot.topology_spread([p for p in sched if p.topology_spread is None], nodes,
                                                       running, other).trivial


def test_builder_corner_cases():
    nodes = [fake_node("n0"), fake_node("n1")]
    master = [fake_node("m", taints=[{"key": "master", "effect": "NoSchedule"}])]
    running = [fake_pod("r0", "ns", {"app": "web"}, node="n0"), fake_pod("r1", "other", {"app": "web"}, node="n1"),
               fake_pod("r2", "ns", {"app": "web"}, node="m")]
    sched = [fake_pod("a", "ns", {"app": "web"}, [tsc()]),                      # selects itself
             fake_pod("b", "ns", {"app": "db"}, [tsc(skew=2)]),                 # does not: skew stays 2
             fake_pod("c", "ns", {"app": "web"}, [tsc(selector=None)]),         # null selector: selects nobody
             fake_pod("d", "ns", {"app": "web"}, [tsc(nodeTaintsPolicy="Honor")]),  # the master is no domain
             fake_pod("e", "ns", {"app": "web"}, [tsc(minDomains=4)])]           # 3 domains < 4: floor 0
    ts = snapshot.topology_spread(sched, nodes, running, master)
    assert len(ts.keys) == 4 and ts.pod_key.tolist() == [0, 0, 1, 2, 3]  # a and b share their key
    assert ts.pod_skew.tolist() == [0, 2, 1, 0, 0]
    assert ts.pod_matches.tolist() == [0b1101, 0, 0b1101, 0b1101, 0b1101]
    assert ts.node_count.tolist() == [[1, 0], [0, 0], [1, 0], [1, 0]]  # r1 is in another namespace
    assert ts.floor.tolist() == [1, 0, INT32_MAX, 0]  # the master's count, a null selector's, no master, minDomains
    assert ts.node_domain.tolist() == [0b1111, 0b1111]
    # without running pods and nodes (the bins): keys by namespace, selector and minDomains, counts of size 0
    ts = snapshot.topology_spread(sched)
    assert ts.node_count.shape == (3, 0) and ts.pod_key.tolist() == [0, 0, 1, 0, 2]
    assert ts.pod_skew.tolist() == [0, 2, 1, 0, 0]


def test_64_keys_accepted_65th_refused():
    def pods(n):
        return [fake_pod("p%d" % i, "ns", {"app": "a%d" % i}, [tsc(selector={"matchLabels": {"app": "a%d" % i}})])
                for i in range(n)] + [fake_pod("dup", "ns", {}, [tsc(selector={"matchLabels": {"app": "a0"}})])]
    ts = snapshot.topology_spread(pods(64))
    assert len(ts.keys) == 64 and ts.pod_key[63] == 63 and ts.pod_key[64] == 0
    assert ts.pod_matches[63] == np.uint64(1) << np.uint64(63)
    with pytest.raises(ValueError, match="64"):
        snapshot.topology_spread(pods(65))


# ---------------------------------------------------------------- the oracle
def no_keys(P, N):
    return dict(keys=0, pod_key=np.full(P, 0xFF, np.uint8), pod_skew=np.zeros(P, np.int32),
                ts_matches=np.zeros(P, np.uint64), node_count=np.zeros((0, N), np.int32),
                node_domain=np.zeros(N, np.uint64), floor=np.zeros(0, np.int32))


def test_oracle_without_keys_is_the_pod_affinity_oracle():
    for kind in ("zero", "with_sel", "replicas"):
        c = ac.make_case(kind, 4)
        P, N = len(c["req"]), len(c["node_type"])
        nm = c.get("node_match", np.ones(N, np.uint64))
        cls = c.get("pod_class", np.zeros(P, np.uint8))
        pc, px = c.get("pod_carries", np.zeros(P, np.uint64)), c.get("pod_matches", np.zeros(P, np.uint64))
        nc0, nx0 = c.get("node_carries", np.zeros(N, np.uint64)), c.get("node_matches", np.zeros(N, np.uint64))
        rq = np.where(np.arange(P) % 7 == 0, 1, 0).astype(np.uint64)  # some self-affine pods: flips happen
        u1, u2 = c["used0"].copy(), c["used0"].copy()
        nh1, nh2 = np.zeros(N, np.uint64), np.zeros(N, np.uint64)
        nc1, nx1, nc2, nx2 = nc0.copy(), nx0.copy(), nc0.copy(), nx0.copy()
        a = ts_oracle.first_fit_nodes_ts(c["req"], c["cap_type"], c["node_type"], u1, **no_keys(P, N),
                                         pod_requires=rq, pod_self=rq, pod_aff_matches=rq, node_has=nh1,
                                         pod_carries=pc, pod_matches=px, node_carries=nc1, node_matches=nx1,
                                         node_match=nm, pod_class=cls)
        b = pa_oracle.first_fit_nodes_pa(c["req"], c["cap_type"], c["node_type"], u2, rq, rq, rq, nh2, pc, px, nc2,
                                         nx2, nm, cls)
        assert a[0].tolist() == b[0].tolist() and a[1] == b[1] and a[2] == b[2] and a[3] == []
        assert np.array_equal(u1, u2) and np.array_equal(nh1, nh2) and np.array_equal(nc1, nc2)
        pend = np.nonzero(a[0] < 0)[0]
        args = (c["req"][pend], len(pend) + 2, c["unit"], c["pool_actual"], c["pool_max"], c["pool_ignored"], 1)
        k = no_keys(len(pend), 0)
        fa = ts_oracle.fulfill_pending_ts(*args, 0, k["pod_key"], k["pod_skew"], k["ts_matches"], rq[pend], rq[pend],
                                          rq[pend], 0, pc[pend], px[pend], c.get("pool_match", np.ones(3, np.uint64)),
                                          cls[pend])
        fb = pa_oracle.fulfill_pending_pa(*args, rq[pend], rq[pend], rq[pend], 0, pc[pend], px[pend],
                                          c.get("pool_match", np.ones(3, np.uint64)), cls[pend])
        for key in fb:
            assert np.array_equal(np.asarray(fa[key]), np.asarray(fb[key])), key


def nodes_tick(caps, used):
    cap = np.asarray(caps, np.float64)
    return cap, np.arange(len(caps), dtype=np.int32), np.asarray(used, np.float64)


def one_key(P, skew, count, domain=None, floor=INT32_MAX, selects=True):
    """every pod has key 0 with maxSkew `skew` and (selects) selects itself"""
    count = np.asarray(count, np.int32).reshape(1, -1)
    N = count.shape[1]
    return dict(keys=1, pod_key=np.zeros(P, np.uint8), pod_skew=np.full(P, skew - int(selects), np.int32),
                ts_matches=np.full(P, int(selects), np.uint64), node_count=count,
                node_domain=np.ones(N, np.uint64) if domain is None else np.asarray(domain, np.uint64),
                floor=np.asarray([floor], np.int32))


def test_stacked_replicas_spread_over_nodes_and_bins():
    # three replicas fit node 0 alone; maxSkew 1 over two empty nodes: one per node, the third waits for a new node
    cap, nt, used = nodes_tick([[8, 8], [8, 8]], [[0, 0], [0, 0]])
    req = np.ones((3, 2), np.float64)
    k = one_key(3, 1, [[0, 0]])
    placed, _, _, rises = ts_oracle.first_fit_nodes_ts(req, cap, nt, used, **k)
    # after pod 0 the minimum is still 0; pod 1 raises it to 1, so pod 2 may land on node 0 again
    assert placed.tolist() == [0, 1, 0] and rises == [(0, 1)] and k["node_count"].tolist() == [[2, 1]]
    # with a master holding the minimum at 0 the third replica stays pending
    k = one_key(3, 1, [[0, 0]], floor=0)
    placed, _, _, rises = ts_oracle.first_fit_nodes_ts(req, cap, nt, used.copy() * 0, **k)
    assert placed.tolist() == [0, 1, -1] and rises == []
    # the bins: a new node takes at most maxSkew self-selecting replicas
    b = one_key(4, 1, [[]])
    f = ts_oracle.fulfill_pending_ts(req[[0, 0, 0, 0]], 4, np.asarray([[8, 8]], np.float64), [0], [10], [0], 0, 1,
                                     b["pod_key"], b["pod_skew"], b["ts_matches"])
    assert f["bin_of"].tolist() == [0, 1, 2, 3] and f["bins_opened"].tolist() == [4]
    b = one_key(4, 2, [[]])
    f = ts_oracle.fulfill_pending_ts(req[[0, 0, 0, 0]], 4, np.asarray([[8, 8]], np.float64), [0], [10], [0], 0, 1,
                                     b["pod_key"], b["pod_skew"], b["ts_matches"])
    assert f["bin_of"].tolist() == [0, 0, 1, 1]
    # a pod that does not select itself is not limited by its own placements
    b = one_key(4, 1, [[]], selects=False)
    f = ts_oracle.fulfill_pending_ts(req[[0, 0, 0, 0]], 4, np.asarray([[8, 8]], np.float64), [0], [10], [0], 0, 1,
                                     b["pod_key"], b["pod_skew"], b["ts_matches"])
    assert f["bin_of"].tolist() == [0, 0, 0, 0]


def test_pinned_pool_minimum_rises():
    # three GPU nodes already run one replica each: the minimum is 1, so a fourth replica may land on any of them
    cap, nt, used = nodes_tick([[8, 8]] * 3, [[1, 1]] * 3)
    req = np.ones((7, 2), np.float64)
    k = one_key(7, 1, [[1, 1, 1]])
    placed, _, _, rises = ts_oracle.first_fit_nodes_ts(req, cap, nt, used, **k)
    assert placed.tolist() == [0, 1, 2, 0, 1, 2, 0] and rises == [(0, 2), (0, 5)]
    # a rule that took the minimum as 0 would refuse every one of them
    k = one_key(7, 1, [[1, 1, 1]], floor=0)
    placed, _, _, rises = ts_oracle.first_fit_nodes_ts(req, cap, nt, used.copy() * 0 + 1, **k)
    assert placed.tolist() == [-1] * 7 and rises == []


def test_master_holds_the_minimum_at_zero():
    # the master (no pod of the group, floor 0) keeps the minimum at 0: each agent node takes one replica
    cap, nt, used = nodes_tick([[8, 8]] * 2, [[0, 0]] * 2)
    req = np.ones((4, 2), np.float64)
    k = one_key(4, 1, [[0, 0]], floor=0)
    placed, _, _, rises = ts_oracle.first_fit_nodes_ts(req, cap, nt, used, **k)
    assert placed.tolist() == [0, 1, -1, -1] and rises == []
    # a node outside the domain set (node affinity policy) does not count for the minimum
    k = one_key(4, 1, [[0, 5]], domain=[1, 0])
    placed, _, _, rises = ts_oracle.first_fit_nodes_ts(req, cap, nt, used * 0, **k)
    assert placed.tolist() == [0, 0, 0, 0] and rises == [(0, 0), (0, 1), (0, 2), (0, 3)]


# ---------------------------------------------------------------- the switch
def _cluster(**kw):
    from kubernetes_acs_engine_autoscaler_b200.cluster import Cluster
    return Cluster(kubeconfig=None, idle_threshold=60, spare_agents=1, service_principal_app_id="x",
                   service_principal_secret="x", service_principal_tenant_id="x", subscription_id="x",
                   client_private_key="x", ca_private_key="x", instance_init_time=600, resource_group="rg",
                   notifier=None, ignore_pools="", **kw)


def test_switch_reads_the_environment(monkeypatch):
    for value, want in ((None, False), ("", False), ("0", False), ("1", True)):
        if value is None:
            monkeypatch.delenv("ACSFIT_TOPOLOGY_SPREAD", raising=False)
        else:
            monkeypatch.setenv("ACSFIT_TOPOLOGY_SPREAD", value)
        assert _cluster().topology_spread is want, value
        assert _cluster(node_selectors=True, pod_affinity=True).topology_spread is want
    monkeypatch.setenv("ACSFIT_TOPOLOGY_SPREAD", "0")
    assert _cluster(topology_spread=True).topology_spread is True
    assert _cluster(topology_spread=True).pod_affinity is False
    monkeypatch.setenv("ACSFIT_TOPOLOGY_SPREAD", "1")
    assert _cluster(topology_spread=False).topology_spread is False


class _Stop(Exception):
    pass


@pytest.mark.parametrize("on", [False, True])
def test_switch_reaches_engine_scaler_and_scaler(monkeypatch, on):
    from kubernetes_acs_engine_autoscaler_b200 import cluster, engine_scaler
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    assert Scaler("rg", [], 0, 1, 60, True, None, None).topology_spread is False
    seen = []

    class Rec(engine_scaler.EngineScaler):
        def __init__(self, **kw):
            engine_scaler.EngineScaler.__init__(self, **kw)
            seen.append((self.topology_spread, [n.name for n in cl.other_nodes]))
            raise _Stop()
    monkeypatch.setattr(cluster, "EngineScaler", Rec)
    cl = _cluster(topology_spread=on)
    node = {"metadata": {"name": "k8s-cpu-1-0", "creationTimestamp": "2026-09-20T07:00:00Z",
                         "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2"}}, "spec": {}}
    master = {"metadata": {"name": "k8s-master-1-0", "creationTimestamp": "2026-09-20T07:00:00Z",
                           "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2"}}, "spec": {}}
    cl.list_nodes = lambda: [SimpleNamespace(obj=node), SimpleNamespace(obj=master)]
    cl.create_kube_node = lambda n: SimpleNamespace(name=n.obj["metadata"]["name"], selectors=n.obj["metadata"]["labels"],
                                                    unschedulable=False)
    cl.arm_parameters, cl.arm_template = {"cpuVMSize": {"value": "Standard_D2_v2"}}, {}
    with pytest.raises(_Stop):
        cl.loop_logic()
    assert seen == [(on, ["k8s-master-1-0"] if on else [])]
