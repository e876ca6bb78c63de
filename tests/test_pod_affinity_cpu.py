"""`-m "not gpu"`: the host side of Cluster(pod_affinity=True) -- required pod affinity with topologyKey
kubernetes.io/hostname.

* kube.affinity_terms: hostname terms kept, zone and namespaceSelector terms dropped, a null labelSelector kept (it
  selects no pod), malformed input raises ValueError naming the pod; anti_affinity_terms still drops null selectors.
* snapshot.pod_affinity bit for bit against a per-pod plain-Python restatement of the scheduler's satisfyPodAffinity
  (every term must select the pod on the node); signature numbering, 64 accepted and a 65th refused.
* The plain-C oracle (tests/pa_oracle.c): equal to tests/aa_oracle.c when every affinity mask is 0, and hand-worked
  ticks: a web pod beside a cache pod on a full node, three self-affine replicas, the bootstrap exception taken by
  another matching pod, two bootstrap signatures, and signatures carried from the node pass and from pool to pool.
* The switch (environment and pass-through)."""
from types import SimpleNamespace

import numpy as np
import pytest

import aa_cases as ac
import aa_oracle
import golden_util as gu
import pa_oracle
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
    return {"podAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": list(terms)}}


def pod_obj(name, labels=None, aff=None, namespace="ns"):
    spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "1"}}}]}
    if aff is not None:
        spec["affinity"] = aff
    return {"metadata": {"name": name, "namespace": namespace, "uid": "u-" + name, "labels": dict(labels or {}),
                         "creationTimestamp": "2026-09-21T07:00:00Z"}, "spec": spec, "status": {"phase": "Pending"}}


WEB = {"matchLabels": {"app": "web"}}
CANON_WEB = ((("app", "web"),), ())


# ---------------------------------------------------------------- parsing
def test_terms_kept_and_dropped():
    got = kube.affinity_terms(affinity(term(WEB), term(WEB, topology="topology.kubernetes.io/zone"),
                                       term(WEB, namespaceSelector={}), term(None), term(WEB, namespaces=["a", "b"])),
                              "ns", "pod p")
    assert got == ((frozenset(["ns"]), CANON_WEB), (frozenset(["ns"]), None), (frozenset(["a", "b"]), CANON_WEB))
    assert kube.affinity_terms(None, "ns", "pod p") == ()
    assert kube.affinity_terms({"podAntiAffinity": {}}, "ns", "pod p") == ()
    # the anti-affinity parser shares the code and still leaves null selectors out; neither reads the other's block
    both = {"podAffinity": affinity(term(WEB))["podAffinity"],
            "podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [term(None), term(WEB)]}}
    assert kube.anti_affinity_terms(both, "ns", "pod p") == ((frozenset(["ns"]), CANON_WEB),)
    assert kube.affinity_terms(both, "ns", "pod p") == ((frozenset(["ns"]), CANON_WEB),)


@pytest.mark.parametrize("bad", [
    {"podAffinity": []},
    {"podAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {}}},
    affinity({"labelSelector": WEB}),
    affinity(term(WEB, namespaces="ns")),
    affinity(term({"matchExpressions": [{"key": "app", "operator": "In"}]})),
    affinity(term({"matchExpressions": [{"key": "app", "operator": "Near", "values": ["x"]}]})),
])
def test_malformed_affinity_raises_naming_the_pod(bad):
    p = kube.KubePod(gu.FakeKubeObject(pod_obj("broken", aff=bad), [], "pod"))
    with pytest.raises(ValueError, match="broken"):
        p.affinity_terms


def test_property_on_kube_pods():
    raw = [gu.FakeKubeObject(o, [], "pod") for o in (pod_obj("a", {"app": "web"}, affinity(term(WEB)), "x"),
                                                     pod_obj("b"))]
    for pods in (kube.make_pods(raw), [kube.KubePod(o) for o in raw]):
        assert [p.affinity_terms for p in pods] == [((frozenset(["x"]), CANON_WEB),), ()]


# ---------------------------------------------------------------- the mask builder
def fake_pod(name, ns, labels, terms, node=None):
    return SimpleNamespace(name=name, namespace=ns, labels=labels, node_name=node,
                           affinity_terms=kube.affinity_terms(affinity(*terms), ns, "pod " + name))


def generated(seed, n_sched=120, n_run=300, n_nodes=40):
    rng = np.random.default_rng(seed)
    apps, nss = ["a%d" % i for i in range(5)], ["n0", "n1"]
    pool = [term({"matchLabels": {"app": a}}) for a in apps] + \
        [term({"matchExpressions": [{"key": "tier", "operator": "In", "values": ["t0", "t1"]}]}),
         term({"matchExpressions": [{"key": "canary", "operator": "DoesNotExist"}]}, namespaces=["n0", "n1"]),
         term({"matchExpressions": [{"key": "app", "operator": "NotIn", "values": ["a0"]}]}),
         term(None)]

    def mk(i, node=None):
        labels = {"app": apps[int(rng.integers(len(apps)))]}
        if rng.random() < 0.5:
            labels["tier"] = "t%d" % rng.integers(3)
        if rng.random() < 0.2:
            labels["canary"] = "1"
        k = int(rng.integers(0, 3)) if rng.random() < 0.6 else 0
        terms = [pool[int(j)] for j in rng.choice(len(pool) - (0 if rng.random() < 0.05 else 1), size=k, replace=False)]
        return fake_pod("p%d" % i, nss[int(rng.integers(2))], labels, terms, node)
    nodes = [SimpleNamespace(name="node%d" % n) for n in range(n_nodes)]
    sched = [mk(i) for i in range(n_sched)]
    running = [mk(n_sched + i, "node%d" % rng.integers(n_nodes + 5)) for i in range(n_run)]  # some on unlisted nodes
    return sched, nodes, running


def satisfies(sig, q):
    """satisfyPodAffinity's per-pod test for topologyKey hostname: q counts when every term selects it"""
    return all(t[1] is not None and q.namespace in t[0] and kube.selector_matches(t[1], q.labels) for t in sig)


def restated(sched, nodes, running):
    sigs = list(dict.fromkeys(frozenset(p.affinity_terms) for p in sched if p.affinity_terms))
    bit = {s: 1 << k for k, s in enumerate(sigs)}
    requires = [bit[frozenset(p.affinity_terms)] if p.affinity_terms else 0 for p in sched]
    matches = [sum(bit[s] for s in sigs if satisfies(s, q)) for q in sched]
    has = [sum(bit[s] for s in sigs if any(q.node_name == n.name and satisfies(s, q) for q in running))
           for n in nodes]
    return sigs, requires, matches, has


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_builder_matches_restatement(seed):
    sched, nodes, running = generated(seed)
    pa = snapshot.pod_affinity(sched, nodes, running)
    sigs, requires, matches, has = restated(sched, nodes, running)
    assert pa.signatures == sigs and len(sigs) > 3
    assert pa.pod_requires.tolist() == requires
    assert pa.pod_matches.tolist() == matches
    assert pa.pod_self.tolist() == [r & m for r, m in zip(requires, matches)]
    assert pa.node_has.tolist() == has
    assert pa.present == int(np.bitwise_or.reduce(np.asarray(has, np.uint64)))
    assert pa.present_signatures() == {s for k, s in enumerate(sigs) if (pa.present >> k) & 1}
    assert not pa.trivial and snapshot.pod_affinity([p for p in sched if not p.affinity_terms]).trivial


def test_null_selector_signature_matches_nobody():
    pods = [fake_pod("x", "ns", {"app": "web"}, [term(None)]), fake_pod("y", "ns", {"app": "web"}, [term(WEB)])]
    pa = snapshot.pod_affinity(pods)
    assert pa.pod_requires.tolist() == [1, 2] and pa.pod_matches.tolist() == [2, 2] and pa.pod_self.tolist() == [0, 2]


def test_64_signatures_accepted_65th_refused():
    def pods(n):
        return [fake_pod("p%d" % i, "ns", {"app": "a%d" % i}, [term({"matchLabels": {"app": "a%d" % i}})])
                for i in range(n)] + [fake_pod("dup", "ns", {}, [term({"matchLabels": {"app": "a0"}})])]
    pa = snapshot.pod_affinity(pods(64))
    assert len(pa.signatures) == 64 and pa.pod_requires[63] == np.uint64(1) << np.uint64(63)
    assert pa.pod_requires[64] == 1  # the same signature, the same bit
    with pytest.raises(ValueError, match="64"):
        snapshot.pod_affinity(pods(65))


# ---------------------------------------------------------------- the oracle
def test_oracle_with_zero_masks_is_the_anti_affinity_oracle():
    for kind in ("zero", "with_sel", "replicas"):
        c = ac.make_case(kind, 4)
        P, N = len(c["req"]), len(c["node_type"])
        nm = c.get("node_match", np.ones(N, np.uint64))
        cls = c.get("pod_class", np.zeros(P, np.uint8))
        pool_match = c.get("pool_match", np.ones(3, np.uint64))
        pc, px = c.get("pod_carries", np.zeros(P, np.uint64)), c.get("pod_matches", np.zeros(P, np.uint64))
        nc0, nx0 = c.get("node_carries", np.zeros(N, np.uint64)), c.get("node_matches", np.zeros(N, np.uint64))
        z, zn = np.zeros(P, np.uint64), np.zeros(N, np.uint64)
        u1, u2 = c["used0"].copy(), c["used0"].copy()
        nc1, nx1, nc2, nx2 = nc0.copy(), nx0.copy(), nc0.copy(), nx0.copy()
        a = pa_oracle.first_fit_nodes_pa(c["req"], c["cap_type"], c["node_type"], u1, z, z, z, zn.copy(), pc, px,
                                         nc1, nx1, nm, cls)
        b = aa_oracle.first_fit_nodes_aa(c["req"], c["cap_type"], c["node_type"], u2, pc, px, nc2, nx2, nm, cls)
        assert a[0].tolist() == b[0].tolist() and a[1] == b[1] and a[2] == []
        assert np.array_equal(u1, u2) and np.array_equal(nc1, nc2) and np.array_equal(nx1, nx2)
        pend = np.nonzero(a[0] < 0)[0]
        args = (c["req"][pend], len(pend) + 2, c["unit"], c["pool_actual"], c["pool_max"], c["pool_ignored"], 1)
        fa = pa_oracle.fulfill_pending_pa(*args, z[pend], z[pend], z[pend], 0, pc[pend], px[pend], pool_match,
                                          cls[pend])
        fb = aa_oracle.fulfill_pending_aa(*args, pc[pend], px[pend], pool_match, cls[pend])
        for k in fb:
            assert np.array_equal(np.asarray(fa[k]), np.asarray(fb[k])), k


def nodes_tick(caps, used):
    """D = 2 nodes, one type per node"""
    cap = np.asarray(caps, np.float64)
    return cap, np.arange(len(caps), dtype=np.int32), np.asarray(used, np.float64)


def masks(rows):
    """rows of (requires, matches) -> (requires, self, matches) uint64 arrays"""
    r = np.asarray([x[0] for x in rows], np.uint64)
    m = np.asarray([x[1] for x in rows], np.uint64)
    return r, r & m, m


def test_web_beside_cache_on_a_full_node():
    # node 0 is full and runs the cache pod (signature 0 present there); node 1 has room but no cache pod
    cap, nt, used = nodes_tick([[4, 4], [8, 8]], [[4, 4], [0, 0]])
    req = np.asarray([[1, 1]], np.float64)
    r, s, m = masks([(1, 0)])  # the web pod requires signature 0 and does not match it itself
    has = np.asarray([1, 0], np.uint64)
    placed, calls, flips = pa_oracle.first_fit_nodes_pa(req, cap, nt, used, r, s, m, has)
    assert placed.tolist() == [-1] and calls == 2 and flips == []
    # the bins: the cache signature is present (on node 0), but no new node holds a cache pod -> no bin, no growth
    f = pa_oracle.fulfill_pending_pa(req, 1, np.asarray([[8, 8]], np.float64), [1], [10], [0], 0, r, s, m, present=1)
    assert f["bins_opened"].tolist() == [0] and f["new_size"].tolist() == [1] and f["num_unaccounted"] == 1
    assert f["acc_pool"].tolist() == [-1] and f["bin_of"].tolist() == [-1] and f["evals"] == 1
    # without the affinity the pod takes node 1
    placed, _, _ = pa_oracle.first_fit_nodes_pa(req, cap, nt, used.copy(), r * 0, s * 0, m * 0, has.copy())
    assert placed.tolist() == [1]


def test_three_self_affine_replicas_share_one_node_and_one_bin():
    cap, nt, used = nodes_tick([[2, 2], [8, 8], [8, 8]], [[0, 0]] * 3)
    req = np.ones((3, 2), np.float64)
    r, s, m = masks([(1, 1)] * 3)
    has = np.zeros(3, np.uint64)
    placed, _, flips = pa_oracle.first_fit_nodes_pa(req, cap, nt, used, r, s, m, has)
    # the first replica bootstraps on node 0; the others must join it -- node 0 has room for one more only
    assert placed.tolist() == [0, 0, -1] and flips == [(0, 0)] and has.tolist() == [1, 0, 0]
    f = pa_oracle.fulfill_pending_pa(req, 3, np.asarray([[8, 8]], np.float64), [0], [10], [0], 0, r, s, m)
    assert f["bins_opened"].tolist() == [1] and f["bin_of"].tolist() == [0, 0, 0] and f["flips"] == [(0, 0)]
    # once the signature is present elsewhere (the node pass placed two), the last replica opens no new bin
    f = pa_oracle.fulfill_pending_pa(req[2:], 1, np.asarray([[8, 8]], np.float64), [0], [10], [0], 0, r[2:], s[2:],
                                     m[2:], present=1)
    assert f["bins_opened"].tolist() == [0] and f["num_unaccounted"] == 1 and f["flips"] == []


def test_bootstrap_taken_by_another_matching_pod():
    # pod 0 matches signature 0 but has no affinity; pod 1 is self-affine.  Pod 0 lands first, so pod 1 may not
    # bootstrap: it must join pod 0's node (node 1, as node 0 is too small for pod 0)
    cap, nt, used = nodes_tick([[1, 1], [4, 4]], [[0, 0]] * 2)
    req = np.asarray([[2, 2], [1, 1]], np.float64)
    r, s, m = masks([(0, 1), (1, 1)])
    has = np.zeros(2, np.uint64)
    placed, _, flips = pa_oracle.first_fit_nodes_pa(req, cap, nt, used, r, s, m, has)
    assert placed.tolist() == [1, 1] and flips == [(0, 0)]


def test_two_bootstrap_signatures_flip_in_turn():
    cap, nt, used = nodes_tick([[8, 8], [8, 8]], [[0, 0]] * 2)
    req = np.ones((4, 2), np.float64)
    # pod 0: no affinity, matches nothing; pod 1: self-affine on 1; pod 2: self-affine on 0; pod 3: requires 1
    r, s, m = masks([(0, 0), (2, 2), (1, 1), (2, 0)])
    has = np.zeros(2, np.uint64)
    placed, _, flips = pa_oracle.first_fit_nodes_pa(req, cap, nt, used, r, s, m, has)
    assert placed.tolist() == [0, 0, 0, 0] and flips == [(1, 1), (0, 2)]


def test_flip_in_the_node_pass_is_seen_by_the_bins():
    cap, nt, used = nodes_tick([[1, 1]], [[0, 0]])
    req = np.ones((2, 2), np.float64)
    r, s, m = masks([(1, 1), (1, 1)])
    has = np.zeros(1, np.uint64)
    placed, _, flips = pa_oracle.first_fit_nodes_pa(req, cap, nt, used, r, s, m, has)
    assert placed.tolist() == [0, -1] and flips == [(0, 0)]
    present = int(np.bitwise_or.reduce(has))
    unit = np.asarray([[8, 8]], np.float64)
    f = pa_oracle.fulfill_pending_pa(req[1:], 1, unit, [0], [10], [0], 0, r[1:], s[1:], m[1:], present=present)
    assert f["bins_opened"].tolist() == [0] and f["num_unaccounted"] == 1
    f = pa_oracle.fulfill_pending_pa(req[1:], 1, unit, [0], [10], [0], 0, r[1:], s[1:], m[1:])  # without it
    assert f["bins_opened"].tolist() == [1] and f["num_unaccounted"] == 0 and f["flips"] == [(0, 0)]


def test_flip_in_pool_0_is_seen_by_pool_1():
    # pool 0 (visited first) packs pod 0 into a bin -- its bootstrap -- but cannot grow (max reached).  A pod counts from
    # the moment it is placed, so signature 0 is present from then on: in pool 1 neither pod may bootstrap, no bin
    # holds a matching pod, and pool 1 does not grow.  (Pod 1 does not fit pool 0's unit.)
    req = np.asarray([[1, 1], [4, 4]], np.float64)
    r, s, m = masks([(1, 1), (1, 1)])
    unit = np.asarray([[2, 2], [8, 8]], np.float64)
    f = pa_oracle.fulfill_pending_pa(req, 2, unit, [1, 1], [1, 10], [0, 0], 0, r, s, m)
    assert f["flips"] == [(0, 0)]
    assert f["bins_opened"].tolist() == [1, 0] and f["bin_of"].tolist() == [0, -1]
    assert f["acc_pool"].tolist() == [-1, -1] and f["num_unaccounted"] == 2 and f["new_size"].tolist() == [1, 1]
    # with room in pool 0, pod 0 is accounted there and pod 1 is blocked in pool 1 all the same
    f = pa_oracle.fulfill_pending_pa(req, 2, unit, [1, 1], [5, 10], [0, 0], 0, r, s, m)
    assert f["acc_pool"].tolist() == [0, -1] and f["bins_opened"].tolist() == [1, 0] and f["num_unaccounted"] == 1


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
            monkeypatch.delenv("ACSFIT_POD_AFFINITY", raising=False)
        else:
            monkeypatch.setenv("ACSFIT_POD_AFFINITY", value)
        assert _cluster().pod_affinity is want, value
        assert _cluster(node_selectors=True, pod_anti_affinity=True).pod_affinity is want
    monkeypatch.setenv("ACSFIT_POD_AFFINITY", "0")
    assert _cluster(pod_affinity=True).pod_affinity is True
    assert _cluster(pod_affinity=True).pod_anti_affinity is False
    monkeypatch.setenv("ACSFIT_POD_AFFINITY", "1")
    assert _cluster(pod_affinity=False).pod_affinity is False


class _Stop(Exception):
    pass


@pytest.mark.parametrize("on", [False, True])
def test_switch_reaches_engine_scaler_and_scaler(monkeypatch, on):
    from kubernetes_acs_engine_autoscaler_b200 import cluster, engine_scaler
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    assert Scaler("rg", [], 0, 1, 60, True, None, None).pod_affinity is False
    seen = []

    class Rec(engine_scaler.EngineScaler):
        def __init__(self, **kw):
            engine_scaler.EngineScaler.__init__(self, **kw)
            seen.append(self.pod_affinity)
            raise _Stop()
    monkeypatch.setattr(cluster, "EngineScaler", Rec)
    cl = _cluster(pod_affinity=on)
    node = {"metadata": {"name": "k8s-cpu-1-0", "creationTimestamp": "2026-09-20T07:00:00Z",
                         "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2"}}, "spec": {}}
    cl.list_nodes = lambda: [SimpleNamespace(obj=node)]
    cl.create_kube_node = lambda n: SimpleNamespace(name=n.obj["metadata"]["name"], selectors=n.obj["metadata"]["labels"],
                                                    unschedulable=False)
    cl.arm_parameters, cl.arm_template = {"cpuVMSize": {"value": "Standard_D2_v2"}}, {}
    with pytest.raises(_Stop):
        cl.loop_logic()
    assert seen == [on]
