"""`-m "not gpu"`: the host side of Cluster(pod_anti_affinity=True) -- required pod anti-affinity with topologyKey
kubernetes.io/hostname.

* kube.label_selector / kube.selector_matches against a table of the selector operators; null vs {} selectors,
  namespace defaulting, ignored topology keys and namespaceSelector terms, malformed input (ValueError naming the pod),
  and KubePod.anti_affinity_terms through both pod construction routes.
* snapshot.anti_affinity bit for bit against a per-pod plain-Python restatement on generated clusters (the symmetric
  direction through running pods, dropped irrelevant terms), 64 terms accepted and a 65th refused.
* The plain-C oracle (tests/aa_oracle.c) against a per-(pod, node) Python restatement, and equal to the selector oracle
  when every mask is 0.
* The switch (environment and pass-through)."""
from types import SimpleNamespace

import numpy as np
import pytest

import aa_cases as ac
import aa_oracle
import golden_util as gu
import sel_oracle
from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot

HOST = "kubernetes.io/hostname"


def term(selector, namespaces=None, topology=HOST, **extra):
    t = {"topologyKey": topology}
    if selector is not None:
        t["labelSelector"] = selector
    if namespaces is not None:
        t["namespaces"] = namespaces
    t.update(extra)
    return t


def affinity(*terms):
    return {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": list(terms)}}


def pod_obj(name, labels=None, aff=None, namespace="ns", phase="Pending", node=None):
    spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "1"}}}]}
    if aff is not None:
        spec["affinity"] = aff
    if node:
        spec["nodeName"] = node
    return {"metadata": {"name": name, "namespace": namespace, "uid": "u-" + name, "labels": dict(labels or {}),
                         "creationTimestamp": "2026-09-21T07:00:00Z"}, "spec": spec, "status": {"phase": phase}}


# ---------------------------------------------------------------- selectors
LABELS = {"app": "web", "tier": "front"}
OPERATOR_TABLE = [
    ({"matchLabels": {"app": "web"}}, True),
    ({"matchLabels": {"app": "db"}}, False),
    ({"matchLabels": {"app": "web", "tier": "back"}}, False),
    ({"matchExpressions": [{"key": "app", "operator": "In", "values": ["db", "web"]}]}, True),
    ({"matchExpressions": [{"key": "app", "operator": "In", "values": ["db"]}]}, False),
    ({"matchExpressions": [{"key": "zone", "operator": "In", "values": ["a"]}]}, False),
    ({"matchExpressions": [{"key": "app", "operator": "NotIn", "values": ["db"]}]}, True),
    ({"matchExpressions": [{"key": "app", "operator": "NotIn", "values": ["web"]}]}, False),
    ({"matchExpressions": [{"key": "zone", "operator": "NotIn", "values": ["a"]}]}, True),  # absent key: NotIn holds
    ({"matchExpressions": [{"key": "tier", "operator": "Exists"}]}, True),
    ({"matchExpressions": [{"key": "zone", "operator": "Exists"}]}, False),
    ({"matchExpressions": [{"key": "zone", "operator": "DoesNotExist"}]}, True),
    ({"matchExpressions": [{"key": "app", "operator": "DoesNotExist"}]}, False),
    ({"matchLabels": {"app": "web"}, "matchExpressions": [{"key": "tier", "operator": "In", "values": ["back"]}]}, False),
    ({}, True),                                                                              # {} selects every pod
    ({"matchLabels": None, "matchExpressions": None}, True),
]


@pytest.mark.parametrize("selector,want", OPERATOR_TABLE)
def test_selector_operators(selector, want):
    canon = kube.label_selector(selector, "pod x")
    assert kube.selector_matches(canon, LABELS) is want
    assert kube.selector_matches(canon, {}) is (not selector.get("matchLabels")
                                                and all(e["operator"] in ("NotIn", "DoesNotExist")
                                                        for e in selector.get("matchExpressions") or ()))


def test_terms_null_vs_empty_namespaces_and_ignored_terms():
    terms = kube.anti_affinity_terms(affinity(
        term({}),                                                       # every pod of the pod's namespace
        term(None),                                                     # null selector: selects no pod, dropped
        term({"matchLabels": {"app": "web"}}, namespaces=["a", "b"]),
        term({"matchLabels": {"app": "web"}}, topology="topology.kubernetes.io/zone"),   # not the hostname: ignored
        term({"matchLabels": {"app": "web"}}, namespaceSelector={"matchLabels": {"team": "x"}}),  # not honoured
        term({"matchLabels": {"app": "web"}}, namespaceSelector=None),  # null namespaceSelector: as absent
        term({}),                                                       # duplicate
    ), "home", "pod p")
    web = ((("app", "web"),), ())
    assert terms == ((frozenset(["home"]), ((), ())), (frozenset(["a", "b"]), web), (frozenset(["home"]), web))
    assert kube.anti_affinity_terms(None, "home", "pod p") == ()
    assert kube.anti_affinity_terms({"nodeAffinity": {}}, "home", "pod p") == ()
    assert kube.anti_affinity_terms({"podAntiAffinity": {"preferredDuringSchedulingIgnoredDuringExecution": [
        {"weight": 1, "podAffinityTerm": term({})}]}}, "home", "pod p") == ()  # preferred terms: out of scope
    # equal selectors written differently are one term
    a = kube.label_selector({"matchExpressions": [{"key": "k", "operator": "In", "values": ["b", "a", "a"]},
                                                  {"key": "j", "operator": "Exists"}]}, "pod p")
    b = kube.label_selector({"matchExpressions": [{"key": "j", "operator": "Exists", "values": []},
                                                  {"key": "k", "operator": "In", "values": ["a", "b"]}]}, "pod p")
    assert a == b


MALFORMED = [
    "required",
    {"podAntiAffinity": []},
    {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"topologyKey": HOST}}},
    {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [None]}},
    affinity({"labelSelector": {}}),                                                   # no topologyKey
    affinity(term("app=web")),
    affinity(term({"matchLabels": ["app"]})),
    affinity(term({"matchLabels": {"app": 1}})),
    affinity(term({"matchExpressions": [{"key": "app", "operator": "Equals", "values": ["web"]}]})),
    affinity(term({"matchExpressions": [{"key": "app", "operator": "In", "values": []}]})),
    affinity(term({"matchExpressions": [{"key": "app", "operator": "Exists", "values": ["web"]}]})),
    affinity(term({"matchExpressions": [{"key": "app", "operator": "In", "values": "web"}]})),
    affinity(term({"matchExpressions": [{"operator": "Exists"}]})),
    affinity(term({}, namespaces="ns")),
]


@pytest.mark.parametrize("bad", MALFORMED)
def test_malformed_affinity_raises_naming_the_pod(bad):
    p = kube.KubePod(gu.FakeKubeObject(pod_obj("broken", aff=bad), [], "pod"))
    with pytest.raises(ValueError, match="broken"):
        p.anti_affinity_terms


def test_property_through_both_routes(monkeypatch):
    aff = affinity(term({"matchLabels": {"app": "web"}}))
    raw = [gu.FakeKubeObject(o, [], "pod") for o in (pod_obj("a", {"app": "web"}, aff, "x"), pod_obj("b"))]
    routes = [kube.make_pods(raw), [kube.KubePod(o) for o in raw]]
    if kube._hostfast is not None:
        monkeypatch.setattr(kube, "_hostfast", None)
        routes.append(kube.make_pods(raw))
    for pods in routes:
        assert [p.anti_affinity_terms for p in pods] == [((frozenset(["x"]), ((("app", "web"),), ())),), ()]


# ---------------------------------------------------------------- the mask builder
def fake_pod(name, ns, labels, terms, node=None):
    return SimpleNamespace(name=name, namespace=ns, labels=labels, node_name=node,
                           anti_affinity_terms=kube.anti_affinity_terms(affinity(*terms), ns, "pod " + name))


def generated(seed, n_sched=120, n_run=300, n_nodes=40, n_terms=12):
    rng = np.random.default_rng(seed)
    apps, nss = ["a%d" % i for i in range(6)], ["n0", "n1", "n2"]
    pool = []
    for k in range(n_terms):
        kind = k % 4
        app = apps[int(rng.integers(len(apps)))]
        if kind == 0:
            sel = {"matchLabels": {"app": app}}
        elif kind == 1:
            sel = {"matchExpressions": [{"key": "app", "operator": "In", "values": [app, apps[(k + 1) % 6]]}]}
        elif kind == 2:
            sel = {"matchExpressions": [{"key": "tier", "operator": "NotIn", "values": ["t0"]},
                                        {"key": "app", "operator": "Exists"}]}
        else:
            sel = {"matchExpressions": [{"key": "canary", "operator": "DoesNotExist"}], "matchLabels": {"app": app}}
        pool.append(term(sel, namespaces=[nss[k % 3]] if k % 5 == 0 else None))

    def mk(i, node=None):
        labels = {"app": apps[int(rng.integers(len(apps)))]}
        if rng.random() < 0.5:
            labels["tier"] = "t%d" % rng.integers(3)
        if rng.random() < 0.1:
            labels["canary"] = "1"
        terms = [pool[int(j)] for j in rng.choice(n_terms, size=int(rng.integers(0, 3)), replace=False)] \
            if rng.random() < 0.5 else []
        return fake_pod("p%d" % i, nss[int(rng.integers(3))], labels, terms, node)
    nodes = [SimpleNamespace(name="node%d" % n) for n in range(n_nodes)]
    sched = [mk(i) for i in range(n_sched)]
    running = [mk(n_sched + i, "node%d" % rng.integers(n_nodes + 5)) for i in range(n_run)]  # some on unlisted nodes
    return sched, nodes, running


def restated(sched, nodes, running, symmetric=True):
    """per pod: the relevant terms in first-occurrence order, then carries / matches / node masks, pair by pair"""
    on_nodes = {n.name for n in nodes}
    run = [p for p in running if p.node_name in on_nodes]
    everyone = sched + run
    order = list(dict.fromkeys(t for p in everyone for t in p.anti_affinity_terms))

    def selects(t, q):
        return q.namespace in t[0] and kube.selector_matches(t[1], q.labels)

    def relevant(t):
        """some pod to place and some OTHER pod (by list position), one carrying t and t selecting the other"""
        carriers = [i for i, p in enumerate(everyone) if t in p.anti_affinity_terms]
        chosen = [i for i, q in enumerate(everyone) if selects(t, q)]
        return any(i != j and (i < len(sched) or (symmetric and j < len(sched))) for i in carriers for j in chosen)
    terms = [t for t in order if relevant(t)]

    def masks(p):
        c = sum(1 << k for k, t in enumerate(terms) if t in p.anti_affinity_terms)
        m = sum(1 << k for k, t in enumerate(terms) if selects(t, p))
        return c, m
    pc = [masks(p) for p in sched]
    nc, nx = [], []
    for n in nodes:
        c = m = 0
        for p in running:
            if p.node_name == n.name:
                a, b = masks(p)
                c, m = c | a, m | b
        nc.append(c)
        nx.append(m)
    return terms, [a for a, _ in pc], [b for _, b in pc], nc, nx


@pytest.mark.parametrize("seed", range(6))
def test_builder_matches_restatement(seed):
    sched, nodes, running = generated(seed)
    aa = snapshot.anti_affinity(sched, nodes, running)
    terms, pc, pm, nc, nx = restated(sched, nodes, running)
    assert aa.terms == terms
    assert aa.pod_carries.tolist() == pc and aa.pod_matches.tolist() == pm
    assert aa.node_carries.tolist() == nc and aa.node_matches.tolist() == nx
    assert aa.pod_carries.dtype == np.uint64 and aa.node_matches.dtype == np.uint64
    # the bin pass: the pending pods alone
    b = snapshot.anti_affinity(sched)
    terms_b, pc_b, pm_b, _, _ = restated(sched, [], [])
    assert b.terms == terms_b and b.pod_carries.tolist() == pc_b and b.pod_matches.tolist() == pm_b
    assert len(b.node_carries) == 0


def test_symmetric_block_and_dropped_terms():
    web = term({"matchLabels": {"app": "web"}})
    db = term({"matchLabels": {"app": "db"}})
    nodes = [SimpleNamespace(name="n0"), SimpleNamespace(name="n1")]
    running = [fake_pod("r0", "ns", {"app": "cache"}, [web], "n0"),    # a running pod's term selects the pending pod
               fake_pod("r1", "ns", {"app": "db"}, [db], "n1")]        # carried and selected by running pods only
    sched = [fake_pod("s0", "ns", {"app": "web"}, [])]
    aa = snapshot.anti_affinity(sched, nodes, running)
    assert len(aa.terms) == 1                                          # the db term cannot block s0: dropped
    assert aa.pod_carries.tolist() == [0] and aa.pod_matches.tolist() == [1]
    assert aa.node_carries.tolist() == [1, 0] and aa.node_matches.tolist() == [0, 0]
    # a term of another namespace does not select the pod
    other = [fake_pod("r0", "other", {"app": "cache"}, [web], "n0")]
    assert snapshot.anti_affinity(sched, nodes, other).trivial
    # nothing blocks anything: trivial, zero masks
    assert snapshot.anti_affinity([fake_pod("s", "ns", {}, [])], nodes, []).trivial


def test_64_terms_accepted_65th_refused():
    def replicas(n):
        return [fake_pod("s%d" % i, "ns", {"app": "a%d" % i}, [term({"matchLabels": {"app": "a%d" % i}})])
                for i in range(n)] * 2
    aa = snapshot.anti_affinity(replicas(64))
    assert len(aa.terms) == 64
    assert sorted(aa.pod_carries[:64].tolist()) == [1 << k for k in range(64)]
    assert (aa.pod_carries == aa.pod_matches).all()
    with pytest.raises(ValueError, match="64"):
        snapshot.anti_affinity(replicas(65))


def test_lone_replicas_block_nothing_and_are_dropped():
    """a pod to place whose term selects only itself, with no other pod carrying or selected: the term can block
    nothing, so it neither takes a bit nor counts against the 64-term limit"""
    lone = [fake_pod("s%d" % i, "ns", {"app": "a%d" % i}, [term({"matchLabels": {"app": "a%d" % i}})])
            for i in range(100)]
    aa = snapshot.anti_affinity(lone)
    assert aa.trivial and not aa.pod_carries.any() and not aa.pod_matches.any()
    # the same replica with a second replica already on a node: kept (the running one selects and carries it)
    nodes = [SimpleNamespace(name="n0")]
    second = fake_pod("r0", "ns", {"app": "a7"}, [term({"matchLabels": {"app": "a7"}})], "n0")
    aa = snapshot.anti_affinity(lone, nodes, [second])
    assert len(aa.terms) == 1 and aa.pod_carries[7] == 1 and aa.pod_matches[7] == 1
    assert aa.node_carries.tolist() == [1] and aa.node_matches.tolist() == [1]
    # a lone pod to place that carries a term selecting only itself, but is selected by another pod's term: only the
    # other term is kept
    other = fake_pod("r1", "ns", {"app": "x"},
                     [term({"matchExpressions": [{"key": "app", "operator": "In", "values": ["a3"]}]})], "n0")
    aa = snapshot.anti_affinity(lone, nodes, [other])
    assert aa.terms == [(frozenset(["ns"]), ((), (("app", "In", ("a3",)),)))]
    assert aa.pod_matches.tolist() == [1 if i == 3 else 0 for i in range(100)] and not aa.pod_carries.any()


# ---------------------------------------------------------------- the oracle
def py_first_fit(c):
    used, nc, nx = c["used0"].copy(), c["node_carries0"].astype(object), c["node_matches0"].astype(object)
    placed, calls = [], 0
    for p in range(len(c["req"])):
        hit = -1
        for n in range(len(used)):
            calls += 1
            blocked = (int(c["pod_carries"][p]) & int(nx[n])) | (int(c["pod_matches"][p]) & int(nc[n]))
            if not blocked and all(c["cap_type"][c["node_type"][n], d] - (used[n, d] + c["req"][p, d]) >= 0
                                   for d in range(used.shape[1])):
                hit = n
                break
        placed.append(hit)
        if hit >= 0:
            used[hit] = used[hit] + c["req"][p]
            nc[hit] = int(nc[hit]) | int(c["pod_carries"][p])
            nx[hit] = int(nx[hit]) | int(c["pod_matches"][p])
    return np.array(placed), calls, used, [int(v) for v in nc], [int(v) for v in nx]


def py_bins(req, unit, pc, pm):
    bins, placed = [], []
    for p in range(len(req)):
        hit = -1
        for i, (left, c, m) in enumerate(bins):
            if not ((int(pc[p]) & m) | (int(pm[p]) & c)) and (left - req[p] >= 0).all():
                hit = i
                break
        if hit < 0:
            hit = len(bins)
            bins.append((unit.copy(), 0, 0))
        left, c, m = bins[hit]
        bins[hit] = (left - req[p], c | int(pc[p]), m | int(pm[p]))
        placed.append(hit)
    return placed


@pytest.mark.parametrize("kind", ["replicas", "symmetric", "cross_ns", "bits64", "all_blocked"])
def test_oracle_matches_python_restatement(kind):
    c = ac.make_case(kind, 2)
    c = dict(c, req=c["req"][:200], pod_carries=c["pod_carries"][:200], pod_matches=c["pod_matches"][:200],
             node_type=c["node_type"][:60], used0=c["used0"][:60].copy(), node_carries0=c["node_carries0"][:60].copy(),
             node_matches0=c["node_matches0"][:60].copy())
    used, nc, nx = c["used0"].copy(), c["node_carries0"].copy(), c["node_matches0"].copy()
    placed, calls = aa_oracle.first_fit_nodes_aa(c["req"], c["cap_type"], c["node_type"], used, c["pod_carries"],
                                                 c["pod_matches"], nc, nx)
    pp, pcalls, pused, pnc, pnx = py_first_fit(c)
    assert placed.tolist() == pp.tolist() and calls == pcalls
    assert np.array_equal(used.view(np.uint64), pused.view(np.uint64))
    assert nc.tolist() == pnc and nx.tolist() == pnx
    pend = np.nonzero(placed < 0)[0]
    unit = c["unit"][:1]
    f = aa_oracle.fulfill_pending_aa(c["req"][pend], len(pend), unit, [0], [1 << 20], [0], 0, c["pod_carries"][pend],
                                     c["pod_matches"][pend])
    assert f["bin_of"].tolist() == py_bins(c["req"][pend], unit[0], c["pod_carries"][pend], c["pod_matches"][pend])


def test_oracle_with_zero_masks_is_the_selector_oracle():
    for kind in ("zero", "with_sel"):
        c = ac.make_case(kind, 4)
        P, N = len(c["req"]), len(c["node_type"])
        nm = c.get("node_match", np.ones(N, np.uint64))
        cls = c.get("pod_class", np.zeros(P, np.uint8))
        pool_match = c.get("pool_match", np.ones(3, np.uint64))
        z, zn = np.zeros(P, np.uint64), np.zeros(N, np.uint64)
        u1, u2 = c["used0"].copy(), c["used0"].copy()
        a = aa_oracle.first_fit_nodes_aa(c["req"], c["cap_type"], c["node_type"], u1, z, z, zn.copy(), zn.copy(), nm, cls)
        b = sel_oracle.first_fit_nodes_sel(c["req"], c["cap_type"], c["node_type"], u2, nm, cls)
        assert a[0].tolist() == b[0].tolist() and a[1] == b[1] and np.array_equal(u1, u2)
        pend = np.nonzero(a[0] < 0)[0]
        args = (c["req"][pend], len(pend) + 2, c["unit"], c["pool_actual"], c["pool_max"], c["pool_ignored"], 1)
        fa = aa_oracle.fulfill_pending_aa(*args, z[pend], z[pend], pool_match, cls[pend])
        fb = sel_oracle.fulfill_pending_sel(*args, pool_match, cls[pend])
        for k in fb:
            assert np.array_equal(np.asarray(fa[k]), np.asarray(fb[k])), k


# ---------------------------------------------------------------- the switch
def _cluster(**kw):
    from kubernetes_acs_engine_autoscaler_b200.cluster import Cluster
    return Cluster(kubeconfig=None, idle_threshold=60, spare_agents=1, service_principal_app_id="x",
                   service_principal_secret="x", service_principal_tenant_id="x", subscription_id="x",
                   client_private_key="x", ca_private_key="x", instance_init_time=600, resource_group="rg",
                   notifier=None, ignore_pools="", **kw)


def test_switch_reads_the_environment(monkeypatch):
    monkeypatch.delenv("ACSFIT_NODE_SELECTORS", raising=False)
    for value, want in ((None, False), ("", False), ("0", False), ("1", True), ("yes", True)):
        if value is None:
            monkeypatch.delenv("ACSFIT_POD_ANTI_AFFINITY", raising=False)
        else:
            monkeypatch.setenv("ACSFIT_POD_ANTI_AFFINITY", value)
        assert _cluster().pod_anti_affinity is want, value
        assert _cluster(node_selectors=True).pod_anti_affinity is want   # independent of node selectors
    monkeypatch.setenv("ACSFIT_POD_ANTI_AFFINITY", "0")
    assert _cluster(pod_anti_affinity=True).pod_anti_affinity is True
    assert _cluster(pod_anti_affinity=True).node_selectors is False
    monkeypatch.setenv("ACSFIT_POD_ANTI_AFFINITY", "1")
    assert _cluster(pod_anti_affinity=False).pod_anti_affinity is False


class _Stop(Exception):
    pass


@pytest.mark.parametrize("on", [False, True])
def test_switch_reaches_engine_scaler_and_scaler(monkeypatch, on):
    from kubernetes_acs_engine_autoscaler_b200 import cluster, engine_scaler
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    assert Scaler("rg", [], 0, 1, 60, True, None, None).pod_anti_affinity is False
    seen = []

    class Rec(engine_scaler.EngineScaler):
        def __init__(self, **kw):
            engine_scaler.EngineScaler.__init__(self, **kw)
            seen.append(self.pod_anti_affinity)
            raise _Stop()
    monkeypatch.setattr(cluster, "EngineScaler", Rec)
    cl = _cluster(pod_anti_affinity=on)
    node = {"metadata": {"name": "k8s-cpu-1-0", "creationTimestamp": "2026-09-20T07:00:00Z",
                         "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2"}}, "spec": {}}
    cl.list_nodes = lambda: [SimpleNamespace(obj=node)]
    cl.create_kube_node = lambda n: SimpleNamespace(name=n.obj["metadata"]["name"], selectors=n.obj["metadata"]["labels"],
                                                    unschedulable=False)
    cl.arm_parameters, cl.arm_template = {"cpuVMSize": {"value": "Standard_D2_v2"}}, {}
    with pytest.raises(_Stop):
        cl.loop_logic()
    assert seen == [on]
