"""`-m "not gpu"`: the host side of Cluster(pod_affinity_node_states=True) -- a node is pod-pending only when some pod to
schedule could land on it given its required pod affinity (and, when those modes are on, anti-affinity and selectors).

* snapshot.pod_affinity_rows bit for bit against a pair-by-pair restatement with kube's term predicates; its numbering
  is snapshot.pod_affinity(pods, agent_nodes, running)'s.
* The plain-C oracle (tests/pa_states_oracle.c) over the host's deduplicated table against a restatement of the rule per
  (pod to schedule, node), alone and with anti-affinity and selectors; with every need 0 it is tests/aa_states_oracle.c.
* The bootstrap folding, hand-worked: a self-affine group with no member running, a member on an ignored pool's node, a
  member only on the master, a pod that does not match its own terms, a null labelSelector.
* The 65-signature and 65-class refusals, the switch rules, and the flags maintain sends (the oracle stands in for the
  GPU); with the switch off the pod-affinity builder is never called."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import aa_states_oracle
import golden_util as gu
import pa_states_oracle
from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot
from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode
from test_aa_states_cpu import AdmitOracleEngine, by_node, csr, edge_case, with_selectors
from test_anti_affinity_cpu import affinity as anti_affinity
from test_pod_affinity_cpu import WEB, affinity, generated, satisfies, term

NO_MATCH = 2  # ACSFIT_NODEF_NO_PENDING_MATCH
U64 = np.uint64


def with_anti_affinity(seed, pods):
    """gives every pod an anti_affinity_terms attribute: about a fifth of them avoid one of three apps"""
    rng = np.random.default_rng([seed, 11])
    for p in pods:
        k = int(rng.integers(0, 3)) if rng.random() < 0.2 else None
        aff = anti_affinity(term({"matchLabels": {"app": "a%d" % k}})) if k is not None else None
        p.anti_affinity_terms = kube.anti_affinity_terms(aff, p.namespace, "pod " + p.name)


def restated_affine(sched, lists, agent_pods):
    """bool[N][P]: the pod-affinity rule pair by pair (satisfyPodAffinity with the first-pod exception)"""
    out = []
    for lst in lists:
        row = []
        for p in sched:
            sig = frozenset(p.affinity_terms)
            if not sig or any(satisfies(sig, q) for q in lst):
                row.append(True)
            else:
                row.append(not any(satisfies(sig, q) for q in agent_pods) and satisfies(sig, p))
        out.append(row)
    return out


def anti_selects(owner, q):
    return any(q.namespace in ns and kube.selector_matches(sel, q.labels) for ns, sel in owner.anti_affinity_terms)


def restated_admits(sched, nodes, lists, agent_pods, anti, selectors):
    affine = restated_affine(sched, lists, agent_pods)
    return np.array([any((not selectors or KubeNode.is_match(n, p)) and affine[i][j] and
                         (not anti or not any(anti_selects(p, q) or anti_selects(q, p) for q in lst))
                         for j, p in enumerate(sched))
                     for i, (n, lst) in enumerate(zip(nodes, lists))], dtype=bool)


def oracle_flags(adm, lists):
    zeros = np.zeros(len(lists), np.uint8)
    if adm.row_has is None:
        return aa_states_oracle.pending_admit(csr(lists), adm.row_carries, adm.row_matches, adm.node_match,
                                              adm.sig_class, adm.sig_carries, adm.sig_matches, zeros)
    return pa_states_oracle.pending_admit_pa(csr(lists), adm.row_carries, adm.row_matches, adm.row_has,
                                             adm.node_match, adm.sig_class, adm.sig_carries, adm.sig_matches,
                                             adm.sig_need, zeros)


def check(sched, nodes, running, lists, agent_nodes, anti=False, selectors=False):
    """the host table through the oracle equals the restatement; returns the flags (None: no table)"""
    names = None if agent_nodes is None else {n.name for n in agent_nodes}
    agent_pods = [q for lst in lists for q in lst] if names is None else [q for q in running if q.node_name in names]
    want = restated_admits(sched, nodes, lists, agent_pods, anti, selectors)
    adm = snapshot.pending_admit(sched, running, nodes, lists, selectors=selectors, anti_affinity=anti,
                                 pod_affinity=True, agent_nodes=agent_nodes)
    if adm is None:  # nothing can exclude a pod to schedule: the selector rule alone decides
        base = snapshot.pending_match(sched, nodes) if selectors else np.ones(len(nodes), bool)
        np.testing.assert_array_equal(base, want)
        return None
    assert (adm.row_carries is not None) == (adm.sig_carries is not None)
    assert (adm.row_has is not None) == (adm.sig_need is not None)
    flags = oracle_flags(adm, lists)
    np.testing.assert_array_equal((flags & NO_MATCH) == 0, want)
    # the table is the distinct signatures of the pods: the same answer per pod, without deduplication
    if adm.row_has is not None:
        req, own, _, _, present, _ = snapshot.pod_affinity_rows(sched, running, lists, nodes=agent_nodes)
        need = np.where((req & U64(present)) == 0, np.where(own != 0, U64(0), req), req)
        assert set(adm.sig_need.tolist()) == set(need.tolist())
        cls = snapshot.selector_classes(sched, nodes, []) if selectors else None
        pod_class = cls.pod_class if cls is not None and not cls.trivial else np.zeros(len(sched), np.uint8)
        pc = pm = None
        if adm.row_carries is not None:
            pc, pm, _, _, _ = snapshot.anti_affinity_rows(sched, running, lists)
        per_pod = pa_states_oracle.pending_admit_pa(csr(lists), adm.row_carries, adm.row_matches, adm.row_has,
                                                    adm.node_match, pod_class, pc, pm, need,
                                                    np.zeros(len(nodes), np.uint8))
        np.testing.assert_array_equal(per_pod, flags)
        cols = [adm.sig_class.astype(U64)] + ([adm.sig_carries, adm.sig_matches] if pc is not None else []) + \
            [adm.sig_need]
        assert len(set(zip(*[c.tolist() for c in cols]))) == len(adm.sig_class)
    return flags


# ---------------------------------------------------------------- the row masks
@pytest.mark.parametrize("seed", range(4))
def test_rows_match_pairwise_restatement(seed):
    sched, nodes, running = generated(seed)
    agent = nodes + [SimpleNamespace(name="node%d" % (len(nodes) + 1))]  # an agent node outside the table
    table = nodes[:30] + [SimpleNamespace(name="empty")]                  # the scalable pools' nodes
    lists = by_node(table, running)
    req, own, mat, has, present, sigs = snapshot.pod_affinity_rows(sched, running, lists, nodes=agent)
    pa = snapshot.pod_affinity(sched, agent, running)
    assert sigs == pa.signatures and len(sigs) > 3
    bit = {s: 1 << k for k, s in enumerate(sigs)}
    assert req.tolist() == [bit[frozenset(p.affinity_terms)] if p.affinity_terms else 0 for p in sched]
    assert mat.tolist() == [sum(b for s, b in bit.items() if satisfies(s, q)) for q in sched]
    assert own.tolist() == (req & mat).tolist()
    flat = [q for lst in lists for q in lst]
    assert has.tolist() == [sum(b for s, b in bit.items() if satisfies(s, q)) for q in flat]
    names = {n.name for n in agent}
    assert present == sum(b for s, b in bit.items() if any(satisfies(s, q) for q in running if q.node_name in names))
    assert present == pa.present
    # without agent nodes the table's own rows decide
    _, _, _, has2, present2, _ = snapshot.pod_affinity_rows(sched, running, lists)
    assert has2.tolist() == has.tolist() and present2 == int(np.bitwise_or.reduce(has)) if len(has) else 0
    with pytest.raises(ValueError):
        snapshot.pod_affinity_rows(sched, running[1:], [[running[0]]])


def test_existing_builder_is_unchanged_by_the_shared_masks():
    sched, nodes, running = generated(5)
    pa = snapshot.pod_affinity(sched, nodes, running)
    req, own, mat, _, present, sigs = snapshot.pod_affinity_rows(sched, running, by_node(nodes, running), nodes=nodes)
    assert (pa.pod_requires.tolist(), pa.pod_self.tolist(), pa.pod_matches.tolist(), pa.present, pa.signatures) == \
        (req.tolist(), own.tolist(), mat.tolist(), present, sigs)


# ---------------------------------------------------------------- the rule through the host table and the oracle
@pytest.mark.parametrize("selectors", [False, True])
@pytest.mark.parametrize("anti", [False, True])
@pytest.mark.parametrize("seed", range(4))
def test_admission_matches_pairwise_restatement(seed, anti, selectors):
    sched, nodes, running = generated(seed, n_sched=30, n_run=200, n_nodes=40)
    with_anti_affinity(seed, sched + running)
    for p in sched + running:
        p.selectors = {}
    table = nodes[:25] + [SimpleNamespace(name="empty-%d" % i) for i in range(3)]
    if selectors:
        with_selectors(seed, sched, table, running)
    for n in table:
        n.selectors = getattr(n, "selectors", {})
    lists = by_node(table, running)
    flags = check(sched, table, running, lists, nodes, anti=anti, selectors=selectors)
    assert flags is not None
    # a few pods: still the restatement; the table's own rows as the agent pods
    check(sched[:4], table, running, lists, None, anti=anti, selectors=selectors)


@pytest.mark.parametrize("with_match", [False, True])
@pytest.mark.parametrize("kind", ["random", "offset", "bit63", "last_admits", "none", "u0"])
def test_oracle_with_zero_need_is_the_anti_affinity_oracle(kind, with_match):
    rng = np.random.default_rng(len(kind) + 100)
    row_ptr, rc, rm, node_match, cls, car, mat, flags = edge_case(kind, rng)
    nm = node_match if with_match else None
    has = rng.integers(0, 1 << 63, size=len(rc), dtype=U64)
    got = pa_states_oracle.pending_admit_pa(row_ptr, rc, rm, has, nm, cls, car, mat, np.zeros(len(cls), U64), flags)
    np.testing.assert_array_equal(got, aa_states_oracle.pending_admit(row_ptr, rc, rm, nm, cls, car, mat, flags))
    # without the anti-affinity masks the oracle is the class test alone
    got = pa_states_oracle.pending_admit_pa(row_ptr, None, None, has, nm, cls, None, None, np.zeros(len(cls), U64),
                                            flags)
    zero = np.zeros(len(rc), U64)
    np.testing.assert_array_equal(got, aa_states_oracle.pending_admit(row_ptr, zero, zero, nm, cls, 0 * car, 0 * mat,
                                                                      flags))


# ---------------------------------------------------------------- the bootstrap, hand-worked
def pod(name, app, node=None, terms=(), ns="ns"):
    return SimpleNamespace(name=name, namespace=ns, labels={"app": app}, node_name=node, selectors={},
                           affinity_terms=kube.affinity_terms(affinity(*terms) if terms else None, ns, "pod " + name),
                           anti_affinity_terms=())


def cluster_of(n=4):
    return [SimpleNamespace(name="n%d" % i, selectors={}) for i in range(n)]


def flagged(sched, nodes, running, agent_nodes):
    lists = by_node(nodes, running)
    flags = check(sched, nodes, running, lists, agent_nodes)
    return None if flags is None else ((flags & NO_MATCH) != 0).tolist()


def test_self_affine_group_with_no_member_running_bootstraps_everywhere():
    nodes = cluster_of()
    running = [pod("db", "db", "n0")]
    web = [pod("web-%d" % i, "web", terms=[term(WEB)]) for i in range(3)]
    assert flagged(web, nodes, running, nodes) is None  # every need folds to 0: nothing can exclude a pod
    # one replica running on n1: only n1 admits the rest
    running.append(pod("web-r", "web", "n1", terms=[term(WEB)]))
    assert flagged(web, nodes, running, nodes) == [True, False, True, True]


def test_member_on_an_ignored_pools_node_cancels_the_bootstrap():
    nodes = cluster_of()                       # the scalable pools' nodes, maintain's table
    ignored = SimpleNamespace(name="ign0", selectors={})
    running = [pod("web-r", "web", "ign0", terms=[term(WEB)])]
    web = [pod("web-0", "web", terms=[term(WEB)])]
    assert flagged(web, nodes, running, nodes + [ignored]) == [True] * 4
    # only the table's pods as agent pods (the single-node path): the group bootstraps
    assert flagged(web, nodes, running, None) is None


def test_member_only_on_the_master_does_not_cancel_the_bootstrap():
    nodes = cluster_of()
    running = [pod("web-r", "web", "k8s-master-0", terms=[term(WEB)])]
    web = [pod("web-0", "web", terms=[term(WEB)])]
    assert flagged(web, nodes, running, nodes) is None


def test_pod_that_does_not_match_its_own_terms_needs_a_match():
    nodes = cluster_of()
    web = [pod("web-0", "web", terms=[term({"matchLabels": {"app": "cache"}})])]
    assert flagged(web, nodes, [pod("db", "db", "n0")], nodes) == [True] * 4     # no cache anywhere: no node
    assert flagged(web, nodes, [pod("cache", "cache", "n2")], nodes) == [True, True, False, True]
    # beside a pod without terms, a node stays pod-pending for that pod
    plain = pod("plain", "x")
    assert flagged(web + [plain], nodes, [pod("cache", "cache", "n2")], nodes) == [False] * 4


def test_null_label_selector_admits_no_node():
    nodes = cluster_of()
    odd = [pod("odd", "web", terms=[term(None)])]
    assert flagged(odd, nodes, [pod("web-r", "web", "n1", terms=[term(WEB)])], nodes) == [True] * 4
    adm = snapshot.pending_admit(odd, [], nodes, [[]] * 4, anti_affinity=False, pod_affinity=True, agent_nodes=nodes)
    assert adm.sig_need.tolist() == [1] and adm.row_carries is None and adm.sig_carries is None


# ---------------------------------------------------------------- refusals
def test_65_signatures_and_65_classes_are_refused():
    nodes = cluster_of(80)
    sigs = [pod("p%d" % i, "b%d" % i, terms=[term({"matchLabels": {"app": "a%d" % i}})]) for i in range(65)]
    running = [pod("r", "x", "n0")]
    lists = by_node(nodes, running)
    with pytest.raises(ValueError, match="64"):
        snapshot.pending_admit(sigs, running, nodes, lists, anti_affinity=False, pod_affinity=True)
    assert snapshot.pending_admit(sigs[:64], running, nodes, lists, anti_affinity=False, pod_affinity=True) is not None
    for i, n in enumerate(nodes):
        n.selectors = {"host": "h%d" % i}
    many = [pod("q%d" % i, "b", terms=[term(WEB)]) for i in range(80)]
    for i, p in enumerate(many):
        p.selectors = {"host": "h%d" % i}                                    # 80 node sets: 80 classes besides 0
    assert snapshot.pending_admit(many, running, nodes, lists, anti_affinity=False, pod_affinity=True) is not None
    with pytest.raises(ValueError):
        snapshot.pending_admit(many, running, nodes, lists, selectors=True, anti_affinity=False, pod_affinity=True)


# ---------------------------------------------------------------- the switch
def _cluster(**kw):
    from kubernetes_acs_engine_autoscaler_b200.cluster import Cluster
    return Cluster(kubeconfig=None, idle_threshold=60, spare_agents=1, service_principal_app_id="x",
                   service_principal_secret="x", service_principal_tenant_id="x", subscription_id="x",
                   client_private_key="x", ca_private_key="x", instance_init_time=600, resource_group="rg",
                   notifier=None, ignore_pools="", **kw)


def test_switch_reads_the_environment_and_needs_pod_affinity(monkeypatch):
    monkeypatch.delenv("ACSFIT_POD_AFFINITY", raising=False)
    for value, want in ((None, False), ("", False), ("0", False), ("1", True)):
        if value is None:
            monkeypatch.delenv("ACSFIT_POD_AFFINITY_NODE_STATES", raising=False)
        else:
            monkeypatch.setenv("ACSFIT_POD_AFFINITY_NODE_STATES", value)
        assert _cluster(pod_affinity=True).pod_affinity_node_states is want, value
        assert _cluster(pod_affinity=False).pod_affinity_node_states is False
        assert _cluster().pod_affinity_node_states is False
    monkeypatch.setenv("ACSFIT_POD_AFFINITY_NODE_STATES", "0")
    assert _cluster(pod_affinity=True, pod_affinity_node_states=True).pod_affinity_node_states is True
    assert _cluster(pod_affinity=True, pod_affinity_node_states=False).pod_affinity_node_states is False
    with pytest.raises(ValueError):
        _cluster(pod_affinity=False, pod_affinity_node_states=True)
    with pytest.raises(ValueError):
        _cluster(pod_affinity_node_states=True)                          # $ACSFIT_POD_AFFINITY unset: off
    monkeypatch.setenv("ACSFIT_POD_AFFINITY", "1")
    c = _cluster(pod_affinity_node_states=True)
    assert c.pod_affinity_node_states is True
    # independent of the other states switches
    assert (c.anti_affinity_node_states, c.selector_node_states) == (False, False)
    c = _cluster(pod_anti_affinity=True, anti_affinity_node_states=True, node_selectors=True,
                 selector_node_states=True, pod_affinity_node_states=True)
    assert (c.pod_affinity_node_states, c.anti_affinity_node_states, c.selector_node_states) == (True, True, True)


class _Stop(Exception):
    pass


@pytest.mark.parametrize("on", [False, True])
def test_switch_reaches_engine_scaler_and_scaler(monkeypatch, on):
    from kubernetes_acs_engine_autoscaler_b200 import cluster, engine_scaler
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    assert Scaler("rg", [], 0, 1, 60, True, None, None).pod_affinity_node_states is False
    seen = []

    class Rec(engine_scaler.EngineScaler):
        def __init__(self, **kw):
            engine_scaler.EngineScaler.__init__(self, **kw)
            seen.append(self.pod_affinity_node_states)
            raise _Stop()
    monkeypatch.setattr(cluster, "EngineScaler", Rec)
    cl = _cluster(pod_affinity=True, pod_affinity_node_states=on)
    node = {"metadata": {"name": "k8s-cpu-1-0", "creationTimestamp": "2026-09-20T07:00:00Z",
                         "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2"}}, "spec": {}}
    cl.list_nodes = lambda: [SimpleNamespace(obj=node)]
    cl.create_kube_node = lambda n: SimpleNamespace(name=n.obj["metadata"]["name"], selectors=n.obj["metadata"]["labels"],
                                                    unschedulable=False)
    cl.arm_parameters, cl.arm_template = {"cpuVMSize": {"value": "Standard_D2_v2"}}, {}
    with pytest.raises(_Stop):
        cl.loop_logic()
    assert seen == [on]


class PaOracleEngine(AdmitOracleEngine):
    """AdmitOracleEngine with acsfit_pending_admit_pa answered by tests/pa_states_oracle.c"""

    def __init__(self):
        AdmitOracleEngine.__init__(self)
        self.pa_admits = 0

    def pending_admit_pa(self, row_ptr, rc, rm, rh, node_match, sig_class, sig_carries, sig_matches, sig_need,
                         node_flags):
        self.pa_admits += 1
        u64 = lambda t: None if t is None else t.numpy().view(U64)  # noqa: E731
        out = pa_states_oracle.pending_admit_pa(row_ptr.numpy(), u64(rc), u64(rm), u64(rh), u64(node_match),
                                                sig_class, sig_carries, sig_matches, sig_need, node_flags.numpy())
        node_flags.copy_(torch.from_numpy(out))
        return node_flags


def web_cache_objects():
    """pools `cpu` (four old Standard_D2_v2 nodes) and `ign` (one node, ignored): a cache pod on cpu node 0, a db pod
    on cpu node 1; web-0 is pending and requires a cache pod on its node; replica-0 of a self-affine group runs on the
    ignored node and replica-1 is pending"""
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.kube import KubePod
    j = []
    nodes = []
    for name, pool in [("k8s-cpu-1-%d" % i, "cpu") for i in range(4)] + [("k8s-ign-1-0", "ign")]:
        o = {"metadata": {"name": name, "creationTimestamp": "2016-08-25T05:13:16Z",
                          "labels": {"agentpool": pool, "beta.kubernetes.io/instance-type": "Standard_D2_v2",
                                     "failure-domain.beta.kubernetes.io/region": "r"}},
             "spec": {}}
        n = KubeNode(gu.FakeKubeObject(o, j, "node"))
        n.capacity = capacity.get_capacity_for_instance_type(n.instance_type)
        nodes.append(n)

    def mk(name, app, node=None, needs=None):
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "100m"}}}]}
        if needs:
            spec["affinity"] = affinity(term({"matchLabels": {"app": needs}}))
        status = {"phase": "Pending"}
        if node:
            spec["nodeName"] = node
            status = {"phase": "Running", "startTime": "2016-08-25T05:13:16Z"}
        o = {"metadata": {"name": name, "namespace": "ns", "uid": "u-" + name, "labels": {"app": app},
                          "creationTimestamp": "2016-08-25T05:13:16Z"}, "spec": spec, "status": status}
        return KubePod(gu.FakeKubeObject(o, j, "pod"))
    running = [mk("cache", "cache", nodes[0].name), mk("db", "db", nodes[1].name),
               mk("replica-0", "rep", nodes[4].name, needs="rep")]
    return nodes, running, [mk("web-0", "web", needs="cache"), mk("replica-1", "rep", needs="rep")], j


@pytest.mark.parametrize("anti", [False, True])
@pytest.mark.parametrize("on", [False, True])
def test_maintain_sends_the_flag_only_when_on(tmp_path, monkeypatch, on, anti):
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.engine_scaler import EngineScaler
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    eng = PaOracleEngine()
    monkeypatch.setattr(snapshot, "_engine", eng)
    if not on:  # off: the pod-affinity builder is never reached, nor are the pods' affinity terms read for maintain
        def boom(*a, **k):
            raise AssertionError("pod affinity read with pod_affinity_node_states off")
        monkeypatch.setattr(snapshot, "pod_affinity_rows", boom)
        monkeypatch.setattr(snapshot, "_pod_affinity_masks", boom)
    nodes, running, pending, journal = web_cache_objects()
    params = {"cpuVMSize": {"value": "Standard_D2_v2"}, "ignVMSize": {"value": "Standard_D2_v2"},
              "masterVMSize": {"value": "Standard_D2_v2"}}
    s = EngineScaler("rg", nodes, 0, 0, 1800, True, None, {}, params, "ign", None, pod_affinity=True,
                     pod_anti_affinity=anti, anti_affinity_node_states=anti, pod_affinity_node_states=on)
    cpu = nodes[:4]
    lists = [[p for p in running if p.node_name == n.name] for n in cpu]
    states = [s.get_node_state(n, lst, pending) for n, lst in zip(cpu, lists)]
    s.maintain(pending, running)
    flags = eng.sent[-1]
    if on:
        # web-0 lands only beside the cache (cpu node 0); replica-1's group has a member on the ignored node, so it
        # may land only there, which maintain does not classify
        assert flags.tolist() == [0, 2, 2, 2] and eng.pa_admits == 5 and eng.admits == 0
        # get_node_state sees only the node's pods: replica-1 bootstraps on every node it is asked about
        assert states == ["pod-pending"] * 4
    else:
        assert flags.tolist() == [0, 0, 0, 0] and eng.pa_admits == 0 and eng.admits == 0
        assert states == ["pod-pending"] * 4
    assert journal == []  # dry run
    # nothing to schedule: no admission call
    n0 = eng.pa_admits
    s.maintain([], running)
    assert eng.sent[-1].tolist() == [0, 0, 0, 0] and eng.pa_admits == n0
    # only web-0 pending: get_node_state agrees with maintain
    eng.sent.clear()
    states = [s.get_node_state(n, lst, pending[:1]) for n, lst in zip(cpu, lists)]
    idle = ["under-utilized-undrainable"] + ["under-utilized-drainable"] * 2  # the db pod has no controller
    assert states == (["pod-pending"] + idle if on else ["pod-pending"] * 4)
