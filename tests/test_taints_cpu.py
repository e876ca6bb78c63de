"""`-m "not gpu"`: the host side of Cluster(node_taints=True) -- node taints and pod tolerations with node selectors.

* kube.tolerates against a table of Kubernetes' ToleratesTaint cases; kube.blocking_taints (effects, lifecycle keys).
* KubeNode.taints, KubePod.tolerations through both pod construction routes, AgentPool.taints, malformed input.
* snapshot.selector_classes(..., taints=True) and snapshot.pending_match(..., taints=True) bit for bit against a
  per-(pod, node) plain-Python restatement of the rule on generated clusters (labels, selectors, hostname pins, taint
  and toleration sets, `Exists`-all, class 0 left empty, 64 signatures and a refused 65th); without a blocking taint
  anywhere the answers equal taints=False, and taints=False equals the per-pair restatement of the selector rule.
* The switch (environment, ValueError, pass-through) and the warnings of get_pods_to_schedule with their precedence
  (the plain-C oracles stand in for the GPU)."""
import logging
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import golden_util as gu
from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot
from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool

HOST, POOL, ITYPE = "kubernetes.io/hostname", "agentpool", "beta.kubernetes.io/instance-type"
LIFECYCLE = ("node.kubernetes.io/not-ready", "node.alpha.kubernetes.io/unreachable",
             "node.cloudprovider.kubernetes.io/uninitialized", "node.kubernetes.io/unschedulable")


def T(key, value=None, effect="NoSchedule"):
    t = {"key": key, "effect": effect}
    if value is not None:
        t["value"] = value
    return t


def Tol(key=None, operator=None, value=None, effect=None, seconds=None):
    t = {}
    for k, v in (("key", key), ("operator", operator), ("value", value), ("effect", effect),
                 ("tolerationSeconds", seconds)):
        if v is not None:
            t[k] = v
    return t


# ---------------------------------------------------------------- the matching rule
TOLERATES = [
    # (tolerations, taint, tolerated)
    ([], T("sku", "gpu"), False),
    ([Tol("sku", "Equal", "gpu", "NoSchedule")], T("sku", "gpu"), True),
    ([Tol("sku", "Equal", "gpu", "NoExecute")], T("sku", "gpu"), False),          # effect differs
    ([Tol("sku", "Equal", "gpu")], T("sku", "gpu", "NoExecute"), True),            # empty effect: every effect
    ([Tol("sku", "Equal", "gpu", "")], T("sku", "gpu"), True),
    ([Tol("other", "Equal", "gpu")], T("sku", "gpu"), False),                      # key differs
    ([Tol("sku", "Equal", "cpu")], T("sku", "gpu"), False),                        # value differs
    ([Tol("sku", None, "gpu")], T("sku", "gpu"), True),                            # empty operator = Equal
    ([Tol("sku", "", "gpu")], T("sku", "gpu"), True),
    ([Tol("sku", "Exists")], T("sku", "gpu"), True),                               # Exists: any value
    ([Tol("sku", "Exists", "cpu")], T("sku", "gpu"), True),
    ([Tol(None, "Exists")], T("sku", "gpu"), True),                                # empty key + Exists: everything
    ([Tol(None, "Exists", effect="NoExecute")], T("sku", "gpu"), False),
    ([Tol(None, "Exists", effect="NoExecute")], T("sku", "gpu", "NoExecute"), True),
    ([Tol(None, "Equal", "gpu")], T("any", "gpu"), True),                          # empty key matches every key
    ([Tol(None, "Equal", "cpu")], T("any", "gpu"), False),
    ([Tol("sku", "Equal")], T("sku"), True),                                       # missing values read as ""
    ([Tol("sku", "Equal", "")], T("sku"), True),
    ([Tol("sku")], T("sku", ""), True),
    ([Tol("sku", "Equal")], T("sku", "gpu"), False),
    ([Tol("sku", "Equal", "gpu")], T("sku"), False),
    ([Tol("sku", "Gt", "gpu")], T("sku", "gpu"), False),                           # unknown operator: nothing
    ([Tol(None, "exists")], T("sku", "gpu"), False),
    ([Tol("sku", "Exists", seconds=30)], T("sku", "gpu", "NoExecute"), True),      # tolerationSeconds ignored
    ([Tol("a", "Exists"), Tol("sku", "Equal", "gpu")], T("sku", "gpu"), True),     # any toleration may match
    ([Tol("a", "Exists"), Tol("b", "Exists")], T("sku", "gpu"), False),
    ([Tol("sku", "Exists", effect="PreferNoSchedule")], T("sku", "gpu", "PreferNoSchedule"), True),
]


@pytest.mark.parametrize("case", range(len(TOLERATES)))
def test_tolerates_table(case):
    tolerations, taint, want = TOLERATES[case]
    assert kube.tolerates(tolerations, taint) is want
    assert kube.tolerates(tolerations, (taint["key"], taint.get("value", ""), taint["effect"])) is want


def test_blocking_taints():
    taints = [T("sku", "gpu"), T("x", None, "NoExecute"), T("soft", "1", "PreferNoSchedule"), T("odd", "1", "Bogus"),
              T("sku", "gpu")] + [T(k) for k in LIFECYCLE] + [T(k, effect="NoExecute") for k in LIFECYCLE]
    assert kube.blocking_taints(taints) == {("sku", "gpu", "NoSchedule"), ("x", "", "NoExecute")}
    assert kube.blocking_taints([T("node.kubernetes.iox/a"), T("kubernetes.io/a")]) == \
        {("node.kubernetes.iox/a", "", "NoSchedule"), ("kubernetes.io/a", "", "NoSchedule")}
    assert kube.blocking_taints([]) == frozenset()
    assert kube.tolerates_all([], kube.blocking_taints([T(k) for k in LIFECYCLE] + [T("s", "1", "PreferNoSchedule")]))


# ---------------------------------------------------------------- kube types
def node_obj(name, labels=None, taints=None):
    spec = {} if taints is None else {"taints": taints}
    return {"metadata": {"name": name, "creationTimestamp": "2026-09-20T07:00:00Z", "labels": dict(labels or {})},
            "spec": spec}


def pod_obj(name, tolerations=None, selector=None, cpu="1", phase="Pending"):
    spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": cpu}}}]}
    if tolerations is not None:
        spec["tolerations"] = tolerations
    if selector:
        spec["nodeSelector"] = selector
    return {"metadata": {"name": name, "namespace": "ns", "uid": "u-" + name, "creationTimestamp": "2026-09-21T07:00:00Z"},
            "spec": spec, "status": {"phase": phase}}


def test_node_taints_and_pod_tolerations_through_both_routes(monkeypatch):
    j = []
    taints = [T("sku", "gpu"), T("soft", "1", "PreferNoSchedule")]
    n = kube.KubeNode(gu.FakeKubeObject(node_obj("k8s-gpu-1-0", taints=taints), j, "node"))
    assert n.taints == taints
    assert kube.KubeNode(gu.FakeKubeObject(node_obj("k8s-gpu-1-1"), j, "node")).taints == []
    tols = [Tol("sku", "Equal", "gpu", "NoSchedule")]
    raw = [gu.FakeKubeObject(o, j, "pod") for o in (pod_obj("a", tols), pod_obj("b"), pod_obj("c", []))]
    routes = [kube.make_pods(raw), [kube.KubePod(o) for o in raw]]
    if kube._hostfast is not None:  # the C route builds plain pods attribute by attribute: the property still reads them
        monkeypatch.setattr(kube, "_hostfast", None)
        routes.append(kube.make_pods(raw))
    for pods in routes:
        assert [p.tolerations for p in pods] == [tols, [], []]


@pytest.mark.parametrize("bad", ["sku=gpu:NoSchedule", {"key": "sku"}, [["sku"]], ["x"], [T("a"), None]])
def test_malformed_taints_and_tolerations_raise(bad):
    j = []
    n = kube.KubeNode(gu.FakeKubeObject(node_obj("k8s-gpu-1-0", taints=bad), j, "node"))
    with pytest.raises(ValueError, match="k8s-gpu-1-0"):
        n.taints
    p = kube.KubePod(gu.FakeKubeObject(pod_obj("broken", bad), j, "pod"))
    with pytest.raises(ValueError, match="broken"):
        p.tolerations
    # read only when the switch is on: the selector builder without taints never touches them
    pod = SimpleNamespace(selectors={POOL: "gpu"}, tolerations=None)
    cls = snapshot.selector_classes([p, pod], [n], [AgentPool("gpu", "t", [n])])
    assert cls.pod_class.tolist() == [0, 1]
    with pytest.raises(ValueError, match="broken"):
        snapshot.selector_classes([p], [], [], taints=True)
    with pytest.raises(ValueError, match="k8s-gpu-1-0"):
        snapshot.pending_match([pod], [n], taints=True)


def test_pool_taints():
    j = []
    mk = lambda i, taints: kube.KubeNode(gu.FakeKubeObject(node_obj("k8s-gpu-1-%d" % i, taints=taints), j, "node"))  # noqa: E731
    shared, other = T("sku", "gpu"), T("team", "a", "NoExecute")
    nodes = [mk(0, [shared, other, T(LIFECYCLE[0])]), mk(1, [T("soft", "1", "PreferNoSchedule"), shared, other]),
             mk(2, [shared, T("team", "b", "NoExecute"), T(LIFECYCLE[1], effect="NoExecute")])]
    assert AgentPool("gpu", "t", nodes).taints == [("sku", "gpu", "NoSchedule")]
    assert AgentPool("gpu", "t", nodes[:2]).taints == [("sku", "gpu", "NoSchedule"), ("team", "a", "NoExecute")]
    assert AgentPool("gpu", "t", []).taints == []                                   # an empty pool has none
    assert AgentPool("gpu", "t", [mk(3, [T(k) for k in LIFECYCLE])]).taints == []
    assert AgentPool("gpu", "t", [mk(4, None), nodes[0]]).taints == []


# ---------------------------------------------------------------- the class builder against a per-pair restatement
def restated_blocking(taints):
    return {(t.get("key") or "", t.get("value") or "", t.get("effect") or "") for t in taints
            if t.get("effect") in ("NoSchedule", "NoExecute")
            and not any((t.get("key") or "").startswith(p) for p in ("node.kubernetes.io/", "node.alpha.kubernetes.io/",
                                                                     "node.cloudprovider.kubernetes.io/"))}


def restated_tolerates(tolerations, taint):
    key, value, effect = taint
    for t in tolerations:
        if t.get("effect") and t["effect"] != effect:
            continue
        if t.get("key") and t["key"] != key:
            continue
        op = t.get("operator") or ""
        if op == "Exists" or (op in ("", "Equal") and (t.get("value") or "") == value):
            return True
    return False


def restated_ok(pod, labels, taints, use_taints):
    if not all(labels.get(k) == v for k, v in pod.selectors.items()):
        return False
    return not use_taints or all(restated_tolerates(pod.tolerations, t) for t in taints)


def restated_pool_taints(pool):
    sets = [restated_blocking(n.taints) for n in pool.nodes]
    return set.intersection(*sets) if sets else set()


def restate_classes(pods, nodes, pools, use_taints):
    node_taints = [restated_blocking(n.taints) if use_taints else set() for n in nodes]
    pool_taints = [restated_pool_taints(p) if use_taints else set() for p in pools]
    every = (tuple([True] * len(nodes)), tuple([True] * len(pools)))
    sigs = [every]
    pod_class = []
    for pod in pods:
        sig = (tuple(restated_ok(pod, n.selectors, t, use_taints) for n, t in zip(nodes, node_taints)),
               tuple(restated_ok(pod, p.labels, t, use_taints) for p, t in zip(pools, pool_taints)))
        if sig not in sigs:
            sigs.append(sig)
        pod_class.append(sigs.index(sig))
    if len(sigs) > 64:
        return None
    node_match = [sum(1 << c for c, s in enumerate(sigs) if s[0][i]) for i in range(len(nodes))]
    pool_match = [sum(1 << c for c, s in enumerate(sigs) if s[1][i]) for i in range(len(pools))]
    return pod_class, node_match, pool_match, len(sigs)


def restate_pending(pods, nodes, use_taints):
    return [any(restated_ok(p, n.selectors, restated_blocking(n.taints) if use_taints else set(), use_taints)
                for p in pods) for n in nodes]


POOLS = ("cpu", "gpu", "mem", "spot")
TAINT_SETS = [[], [], [], [T("sku", "gpu")], [T("sku", "gpu"), T("team", "ml", "NoExecute")],
              [T("spot", None, "NoSchedule")], [T("soft", "1", "PreferNoSchedule")], [T(LIFECYCLE[0])],
              [T(LIFECYCLE[2]), T("sku", "gpu")], [T("team", "web", "NoExecute")]]
TOLERATION_SETS = [[], [], [Tol("sku", "Equal", "gpu")], [Tol("sku", "Exists", effect="NoSchedule")],
                   [Tol(None, "Exists")], [Tol("team", "Equal", "ml"), Tol("sku", "Exists")], [Tol("spot", "Exists")],
                   [Tol("team", "Exists", effect="NoExecute")], [Tol("sku", "Equal", "cpu")],
                   [Tol("sku", "Gt", "gpu")]]


def gen_cluster(rng, N, n_sel, P, taint_prob=0.5, taint_sets=TAINT_SETS, toleration_sets=TOLERATION_SETS,
                pool_tainted=None):
    """nodes of four pools (pool `gpu` uniformly tainted when pool_tainted is given), pods mixing selectors, hostname
    pins and toleration sets"""
    nodes = []
    for i in range(N):
        pool = POOLS[rng.integers(len(POOLS))]
        labels = {POOL: pool, HOST: "node-%d" % i, ITYPE: "type-%s" % pool}
        if rng.random() < 0.3:
            labels["zone"] = str(rng.integers(3))
        if pool_tainted is not None and pool == "gpu":
            taints = list(pool_tainted)
        else:
            taints = list(taint_sets[rng.integers(len(taint_sets))]) if rng.random() < taint_prob else []
        nodes.append(SimpleNamespace(selectors=labels, taints=taints, unschedulable=False))
    pools = [AgentPool(p, "type-" + p, [n for n in nodes if n.selectors[POOL] == p]) for p in POOLS]
    kinds = [lambda: {}, lambda: {}, lambda: {POOL: POOLS[rng.integers(len(POOLS))]},
             lambda: {HOST: "node-%d" % rng.integers(max(N, 1))}, lambda: {"zone": str(rng.integers(3))},
             lambda: {POOL: "gpu", ITYPE: "type-gpu"}, lambda: {"missing": "x"}]
    selectors = [kinds[rng.integers(len(kinds))]() for _ in range(n_sel)]
    pods = [SimpleNamespace(selectors=dict(selectors[rng.integers(n_sel)]),
                            tolerations=list(toleration_sets[rng.integers(len(toleration_sets))])) for _ in range(P)]
    return pods, nodes, pools


def check_classes(pods, nodes, pools, use_taints):
    want = restate_classes(pods, nodes, pools, use_taints)
    if want is None:
        with pytest.raises(ValueError, match="64"):
            snapshot.selector_classes(pods, nodes, pools, taints=use_taints)
        return None
    got = snapshot.selector_classes(pods, nodes, pools, taints=use_taints)
    assert got.pod_class.dtype == np.uint8 and got.node_match.dtype == np.uint64 and got.pool_match.dtype == np.uint64
    assert got.pod_class.tolist() == want[0]
    assert got.node_match.tolist() == want[1]
    assert got.pool_match.tolist() == want[2]
    assert got.classes == want[3]
    return got


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("shape", [(1, 1, 1), (40, 3, 30), (200, 8, 120), (300, 20, 200)])
def test_classes_and_pending_match_equal_per_pair_restatement(seed, shape):
    N, n_sel, P = shape
    rng = np.random.default_rng([seed, N])
    pods, nodes, pools = gen_cluster(rng, N, n_sel, P)
    for use_taints in (True, False):
        check_classes(pods, nodes, pools, use_taints)
        check_classes(pods, [], pools, use_taints)
        check_classes(pods, nodes, [], use_taints)
        for sub in (pods, pods[:3], pods[::7], []):
            assert snapshot.pending_match(sub, nodes, taints=use_taints).tolist() == \
                restate_pending(sub, nodes, use_taints)


@pytest.mark.parametrize("seed", range(4))
def test_class_zero_left_empty(seed):
    """pool `gpu` is tainted on every node, and no pod tolerates it (nor carries an Exists-all toleration): no pod
    matches everything, so class 0 has no pod and bit 0 still marks every node and pool"""
    rng = np.random.default_rng([seed, 99])
    tols = [s for s in TOLERATION_SETS if not restated_tolerates(s, ("sku", "gpu", "NoSchedule"))]
    pods, nodes, pools = gen_cluster(rng, 150, 6, 100, taint_prob=0.0, toleration_sets=tols,
                                     pool_tainted=[T("sku", "gpu")])
    got = check_classes(pods, nodes, pools, True)
    assert got.pod_class.all() and (got.node_match & np.uint64(1)).all() and (got.pool_match & np.uint64(1)).all()
    assert not got.trivial


@pytest.mark.parametrize("pins", [62, 63])
def test_64_signatures_and_the_65th(pins):
    """pool `gpu` tainted, no toleration: the pods without a selector share one signature that is not class 0; each
    hostname pin into pool `cpu` adds one.  1 + 1 + 62 = 64 classes are accepted, one more pin is refused"""
    nodes = [SimpleNamespace(selectors={POOL: "cpu", HOST: "c%d" % i}, taints=[T(LIFECYCLE[0])], unschedulable=False) for i in range(70)]
    nodes += [SimpleNamespace(selectors={POOL: "gpu", HOST: "g%d" % i}, taints=[T("sku", "gpu")], unschedulable=False) for i in range(5)]
    pools = [AgentPool("cpu", "t", nodes[:70]), AgentPool("gpu", "t", nodes[70:])]
    pods = [SimpleNamespace(selectors={}, tolerations=[])]
    pods += [SimpleNamespace(selectors={HOST: "c%d" % i}, tolerations=[Tol("sku", "Equal", "cpu")]) for i in range(pins)]
    if pins == 62:
        got = check_classes(pods, nodes, pools, True)
        assert got.classes == 64 and not (got.pod_class == 0).any()
    else:
        with pytest.raises(ValueError, match="64"):
            snapshot.selector_classes(pods, nodes, pools, taints=True)
    # the selector mode alone sees 1 + pins signatures: no refusal there
    assert snapshot.selector_classes(pods, nodes, pools).classes == pins + 1


@pytest.mark.parametrize("seed", range(4))
def test_no_blocking_taint_anywhere_equals_selectors_alone(seed):
    rng = np.random.default_rng([seed, 7])
    noise = [[], [T("soft", "1", "PreferNoSchedule")], [T(LIFECYCLE[0])], [T(LIFECYCLE[3], effect="NoExecute")]]
    pods, nodes, pools = gen_cluster(rng, 200, 10, 150, taint_prob=0.6, taint_sets=noise)
    a = snapshot.selector_classes(pods, nodes, pools, taints=True)
    b = snapshot.selector_classes(pods, nodes, pools)
    for k in ("pod_class", "node_match", "pool_match"):
        assert getattr(a, k).tolist() == getattr(b, k).tolist(), k
    assert a.classes == b.classes
    assert snapshot.pending_match(pods, nodes, taints=True).tolist() == snapshot.pending_match(pods, nodes).tolist()
    plain = [SimpleNamespace(selectors={}, tolerations=p.tolerations) for p in pods]
    assert snapshot.selector_classes(plain, nodes, pools, taints=True).trivial


def test_selectors_without_taint_attributes():
    """taints=False reads neither .taints nor .tolerations (objects with only .selectors work, as before)"""
    nodes = [SimpleNamespace(selectors={POOL: p}) for p in ("a", "b", "a")]
    pods = [SimpleNamespace(selectors=s) for s in ({}, {POOL: "b"}, {POOL: "a"}, {POOL: "b"})]
    cls = snapshot.selector_classes(pods, nodes, [])
    assert cls.pod_class.tolist() == [0, 1, 2, 1] and cls.node_match.tolist() == [5, 3, 5] and cls.classes == 3
    assert snapshot.pending_match(pods[1:2], nodes).tolist() == [False, True, False]


def test_pending_match_at_scale():
    """20 k nodes with hostname pins, a few taint sets: same answer as the per-pair evaluation"""
    rng = np.random.default_rng(5)
    pods, nodes, pools = gen_cluster(rng, 20000, 40, 120)
    assert snapshot.pending_match(pods, nodes, taints=True).tolist() == restate_pending(pods, nodes, True)


# ---------------------------------------------------------------- the switch
def _cluster(**kw):
    from kubernetes_acs_engine_autoscaler_b200.cluster import Cluster
    return Cluster(kubeconfig=None, idle_threshold=60, spare_agents=1, service_principal_app_id="x",
                   service_principal_secret="x", service_principal_tenant_id="x", subscription_id="x",
                   client_private_key="x", ca_private_key="x", instance_init_time=600, resource_group="rg",
                   notifier=None, ignore_pools="", **kw)


def test_switch_reads_the_environment_and_needs_node_selectors(monkeypatch):
    monkeypatch.delenv("ACSFIT_NODE_SELECTORS", raising=False)
    for value, want in ((None, False), ("", False), ("0", False), ("1", True), ("yes", True)):
        if value is None:
            monkeypatch.delenv("ACSFIT_NODE_TAINTS", raising=False)
        else:
            monkeypatch.setenv("ACSFIT_NODE_TAINTS", value)
        assert _cluster(node_selectors=True).node_taints is want, value
        assert _cluster(node_selectors=False).node_taints is False   # no effect without node selectors
        assert _cluster().node_taints is False
    monkeypatch.setenv("ACSFIT_NODE_TAINTS", "0")
    assert _cluster(node_selectors=True, node_taints=True).node_taints is True
    assert _cluster(node_selectors=True, node_taints=False).node_taints is False
    assert _cluster(node_selectors=False, node_taints=False).node_taints is False
    with pytest.raises(ValueError):
        _cluster(node_selectors=False, node_taints=True)
    with pytest.raises(ValueError):
        _cluster(node_taints=True)                                   # $ACSFIT_NODE_SELECTORS unset: off
    monkeypatch.setenv("ACSFIT_NODE_SELECTORS", "1")
    assert _cluster(node_taints=True).node_taints is True
    # independent of selector_node_states
    assert _cluster(node_taints=True, selector_node_states=False).selector_node_states is False


class _Stop(Exception):
    pass


@pytest.mark.parametrize("on", [False, True])
def test_switch_reaches_engine_scaler_and_scaler(monkeypatch, on):
    from kubernetes_acs_engine_autoscaler_b200 import cluster, engine_scaler
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    assert Scaler("rg", [], 0, 1, 60, True, None, None).node_taints is False
    seen = []

    class Rec(engine_scaler.EngineScaler):
        def __init__(self, **kw):
            engine_scaler.EngineScaler.__init__(self, **kw)
            seen.append(self.node_taints)
            raise _Stop()
    monkeypatch.setattr(cluster, "EngineScaler", Rec)
    monkeypatch.delenv("ACSFIT_NODE_TAINTS", raising=False)
    cl = _cluster(node_selectors=True, node_taints=on)
    cl.list_nodes = lambda: [SimpleNamespace(obj=node_obj("k8s-cpu-1-0", {ITYPE: "Standard_D2_v2"}))]
    cl.create_kube_node = lambda n: SimpleNamespace(name=n.obj["metadata"]["name"], selectors=n.obj["metadata"]["labels"],
                                                    unschedulable=False)
    cl.arm_parameters, cl.arm_template = {"cpuVMSize": {"value": "Standard_D2_v2"}}, {}
    with pytest.raises(_Stop):
        cl.loop_logic()
    assert seen == [on]


def test_scaler_passes_the_switch_to_pending_match(monkeypatch):
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    s = Scaler("rg", [], 0, 1, 60, True, None, None)
    s.selector_node_states = True
    nodes = [SimpleNamespace(selectors={POOL: "gpu"}, taints=[T("sku", "gpu")])]
    pods = [SimpleNamespace(selectors={}, tolerations=[])]
    assert s.no_pending_match(nodes, pods).tolist() == [False]
    s.node_taints = True
    assert s.no_pending_match(nodes, pods).tolist() == [True]
    pods[0].tolerations = [Tol("sku", "Exists")]
    assert s.no_pending_match(nodes, pods).tolist() == [False]


# ---------------------------------------------------------------- warnings of get_pods_to_schedule
NO_POOL = "Pending pod %s cannot fit: no agent pool matches its node selector %s. Scheduling skipped."
NO_FIT = ("Pending pod %s cannot fit. Please check that requested resource amount is consistent with node size."
          "Scheduling skipped.")
UNTOLERATED = ("Pending pod %s cannot fit: every agent pool that would fit it and matches its node selector has a taint "
               "it does not tolerate. Scheduling skipped.")


class SelOracleEngine(object):
    """the plain-C oracles on CPU tensors for K0, plain and with selector classes"""

    def __init__(self):
        from oracle_engine import OracleEngine
        self.base = OracleEngine()

    def __getattr__(self, name):
        return getattr(self.base, name)

    def feasible_mask_sel(self, req, unit, pod_class, pool_match, classes):
        import sel_oracle
        mask, evals = sel_oracle.feasible_mask_sel(req.numpy(), unit.numpy(), pool_match, pod_class.numpy())
        return torch.from_numpy(mask), torch.tensor([evals], dtype=torch.int64)


def test_warnings_and_their_precedence(tmp_path, monkeypatch, oracle_mod):
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", SelOracleEngine())
    j = []
    gpu_taint = T("sku", "gpu")

    def node(pool, itype, taints=None):
        o = node_obj("k8s-%s-1-0" % pool, {POOL: pool, ITYPE: itype, "failure-domain.beta.kubernetes.io/region": "r"},
                     taints)
        return KubeNode(gu.FakeKubeObject(o, j, "node"))
    # cpu: 2 cores, untainted; gpu: 6 cores, tainted sku=gpu:NoSchedule (plus noise)
    nodes = [node("cpu", "Standard_D2_v2"), node("gpu", "Standard_NC6", [gpu_taint, T("soft", "1", "PreferNoSchedule")])]
    pools = [AgentPool("cpu", "Standard_D2_v2", nodes[:1]), AgentPool("gpu", "Standard_NC6", nodes[1:])]
    specs = [  # name, cpu, selector, tolerations, warning with taints on, warning with selectors alone
        ("small", "1", None, None, None, None),
        ("big", "5", None, None, UNTOLERATED, None),                        # fits only the tainted pool
        ("big-tol", "5", None, [Tol("sku", "Equal", "gpu")], None, None),
        ("pinned-gpu", "1", {POOL: "gpu"}, None, UNTOLERATED, None),
        ("pinned-gpu-tol", "1", {POOL: "gpu"}, [Tol(None, "Exists")], None, None),
        ("pinned-cpu-big", "5", {POOL: "cpu"}, None, NO_POOL, NO_POOL),      # the selector rules it out first
        ("pinned-cpu-big-tol", "5", {POOL: "cpu"}, [Tol("sku", "Exists")], NO_POOL, NO_POOL),
        ("pinned-nowhere", "1", {POOL: "nosuch"}, None, NO_POOL, NO_POOL),
        ("huge", "64", None, None, NO_FIT, NO_FIT),                          # fits no pool at all
        ("huge-pinned", "64", {POOL: "gpu"}, None, NO_FIT, NO_FIT),
        ("gpu-soft-only", "5", None, [Tol("soft", "Exists")], UNTOLERATED, None),
    ]
    pods = [KubePod(gu.FakeKubeObject(pod_obj(name, tols, sel, cpu), j, "pod")) for name, cpu, sel, tols, _, _ in specs]

    def expected(k):
        out = []
        for (name, _, sel, _, on, off), pod in zip(specs, pods):
            w = (on, off)[k]
            if w is not None:
                out.append(w % ((name, pod.selectors) if w == NO_POOL else name))
        return out
    log = logging.getLogger("autoscaler.cluster")
    for k, taints in enumerate((True, False)):
        monkeypatch.setenv("ACSFIT_NODE_TAINTS", "0")
        cl = _cluster(node_selectors=True, node_taints=taints)
        handler = gu.ListHandler()
        log.addHandler(handler)
        try:
            got = cl.get_pods_to_schedule(pods, pools)
        finally:
            log.removeHandler(handler)
        want_names = [s[0] for s in specs if (s[4], s[5])[k] is None]
        assert [p.name for p in got] == want_names
        assert [m for lvl, _, m in handler.records if lvl == "WARNING"] == expected(k)
