"""`-m "not gpu"`: the host side of Cluster(topology_spread_node_states=True) -- a node is pod-pending only when some pod
to schedule could land on it given its hostname topology spread constraint (and, when those modes are on,
anti-affinity, pod affinity and selectors).

* The plain-C oracle (tests/ts_states_oracle.c) with every key 0xFF is tests/pa_states_oracle.c.
* snapshot.pending_admit's table through the oracle against a per-(pod to schedule, node) restatement built from the
  pod and node objects (tests/test_topology_spread_cpu.py's `restated`); the table is deduplicated over (class, carries,
  matches, need, key, skew) and, without a constraint, is the table of the other switches.
* Hand-worked: the A/B/C/D example, the master and an ignored pool's node holding the minimum at 0, minDomains above
  the domain count, a key with no domain, a pod its own selector does not select, and the one-node get_node_state.
* The 65-key refusal, the switch rules, and the flags maintain sends (the oracle stands in for the GPU); with the
  switch off no constraint is read."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import golden_util as gu
import pa_states_oracle
import ts_states_oracle
from kubernetes_acs_engine_autoscaler_b200 import snapshot
from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode
from test_aa_states_cpu import AdmitOracleEngine, by_node, csr, edge_case
from test_topology_spread_cpu import INT32_MAX, fake_node, fake_pod, generated, restated, tsc

NO_MATCH = 2  # ACSFIT_NODEF_NO_PENDING_MATCH
U64 = np.uint64


def oracle_flags(adm, lists):
    """the table through tests/ts_states_oracle.c (keys) or tests/pa_states_oracle.c"""
    zeros = np.zeros(len(lists), np.uint8)
    if adm.sig_key is None:
        return pa_states_oracle.pending_admit_pa(csr(lists), adm.row_carries, adm.row_matches, adm.row_has,
                                                 adm.node_match, adm.sig_class, adm.sig_carries, adm.sig_matches,
                                                 adm.sig_need, zeros)
    return ts_states_oracle.pending_admit_ts(csr(lists), adm.row_carries, adm.row_matches, adm.row_has,
                                             adm.node_match, adm.sig_class, adm.sig_carries, adm.sig_matches,
                                             adm.sig_need, adm.sig_key, adm.sig_skew, adm.node_count,
                                             adm.node_domain, adm.floor, zeros)


def restated_admits(sched, nodes, other, running, selectors=False):
    """bool[N]: some pod to schedule passes the spread test (and the selector match) on the node -- per (pod, node),
    each minimum recomputed from the restated counts, domains and floors"""
    _, key_of, skew, _, counts, domain_bits, floor = restated(sched, nodes, other, running)

    def key_min(k):
        return min([floor[k]] + [counts[k][m] for m in range(len(nodes)) if (domain_bits[m] >> k) & 1])

    def spread(j, n):
        k = key_of[j]
        return k == 0xFF or counts[k][n] <= skew[j] + key_min(k)
    return np.array([any((not selectors or KubeNode.is_match(nodes[n], p)) and spread(j, n)
                         for j, p in enumerate(sched)) for n in range(len(nodes))], dtype=bool)


def flagged(sched, nodes, running, other=(), **kw):
    """the flags of the host table through the oracle, as a list of bools (None: no table)"""
    lists = by_node(nodes, running)
    adm = snapshot.pending_admit(sched, running, nodes, lists, anti_affinity=False, topology_spread=True,
                                 other_nodes=other, **kw)
    if adm is None:
        return None
    want = restated_admits(sched, nodes, list(other), running, kw.get("selectors", False))
    flags = (oracle_flags(adm, lists) & NO_MATCH) != 0
    np.testing.assert_array_equal(~flags, want)
    return flags.tolist()


# ---------------------------------------------------------------- the oracle
@pytest.mark.parametrize("with_match", [False, True])
@pytest.mark.parametrize("kind", ["random", "offset", "bit63", "last_admits", "none", "u0"])
def test_oracle_without_keys_is_the_pod_affinity_oracle(kind, with_match):
    rng = np.random.default_rng(len(kind) + 200)
    row_ptr, rc, rm, node_match, cls, car, mat, flags = edge_case(kind, rng)
    nm = node_match if with_match else None
    N, U = len(flags), len(cls)
    has = rng.integers(0, 1 << 63, size=len(rc), dtype=U64)
    need = np.where(rng.random(U) < 0.5, U64(0), U64(1) << rng.integers(0, 64, size=U).astype(U64))
    no_key = dict(pod_key=np.full(U, 0xFF, np.uint8), pod_skew=np.zeros(U, np.int32),
                  node_count=np.zeros((0, N), np.int32), node_domain=np.zeros(N, U64), floor=np.zeros(0, np.int32))
    for aa in (False, True):
        a = (rc, rm, car, mat) if aa else (None,) * 4
        got = ts_states_oracle.pending_admit_ts(row_ptr, a[0], a[1], has, nm, cls, a[2], a[3], need, **no_key,
                                                node_flags=flags)
        np.testing.assert_array_equal(got, pa_states_oracle.pending_admit_pa(row_ptr, a[0], a[1], has, nm, cls, a[2],
                                                                             a[3], need, flags))


def test_oracle_limit_is_computed_in_64_bits():
    """floor INT32_MAX and a positive skew: the limit does not wrap, every count passes"""
    row_ptr = np.zeros(3, np.int64)
    got = ts_states_oracle.pending_admit_ts(row_ptr, None, None, None, None, [0], None, None, None, [0], [5],
                                            [[INT32_MAX, 7]], [0, 0], [INT32_MAX], np.zeros(2, np.uint8))
    assert got.tolist() == [0, 0]
    got = ts_states_oracle.pending_admit_ts(row_ptr, None, None, None, None, [0], None, None, None, [0], [5],
                                            [[INT32_MAX, 7]], [1, 1], [INT32_MAX], np.zeros(2, np.uint8))
    assert got.tolist() == [NO_MATCH, 0]  # the minimum is 7 now: INT32_MAX > 12


# ---------------------------------------------------------------- the table against the restatement
@pytest.mark.parametrize("selectors", [False, True])
@pytest.mark.parametrize("seed", range(4))
def test_admission_matches_pairwise_restatement(seed, selectors):
    sched, nodes, other, running = generated(seed, n_sched=40, n_run=300, n_nodes=30)
    table, outside = nodes[:22], nodes[22:] + other  # maintain's nodes; an ignored pool's nodes and the masters
    lists = by_node(table, running)
    # a few pods with constraints (some nodes admit none of them), then every pod
    few = [p for p in sched if p.topology_spread is not None][:3]
    adm = snapshot.pending_admit(few, running, table, lists, selectors=selectors, anti_affinity=False,
                                 topology_spread=True, other_nodes=outside)
    want = restated_admits(few, table, outside, running, selectors)
    np.testing.assert_array_equal((oracle_flags(adm, lists) & NO_MATCH) == 0, want)
    adm = snapshot.pending_admit(sched, running, table, lists, selectors=selectors, anti_affinity=False,
                                 topology_spread=True, other_nodes=outside)
    assert adm is not None and adm.sig_key is not None and adm.row_carries is None and adm.row_has is None
    want = restated_admits(sched, table, outside, running, selectors)
    flags = oracle_flags(adm, lists)
    np.testing.assert_array_equal((flags & NO_MATCH) == 0, want)
    # the table is the distinct (class, key, skew) of the pods: the same answer per pod, without deduplication
    ts = snapshot.topology_spread(sched, table, running, outside)
    cls = snapshot.selector_classes(sched, table, []) if selectors else None
    pod_class = cls.pod_class if cls is not None and not cls.trivial else np.zeros(len(sched), np.uint8)
    per_pod = ts_states_oracle.pending_admit_ts(csr(lists), None, None, None, adm.node_match, pod_class, None, None,
                                                None, ts.pod_key, ts.pod_skew, ts.node_count, ts.node_domain, ts.floor,
                                                np.zeros(len(table), np.uint8))
    np.testing.assert_array_equal(per_pod, flags)
    rows = set(zip(adm.sig_class.tolist(), adm.sig_key.tolist(), adm.sig_skew.tolist()))
    assert len(rows) == len(adm.sig_class)
    assert rows == set(zip(pod_class.tolist(), ts.pod_key.tolist(), ts.pod_skew.tolist()))
    assert (adm.node_count.tolist(), adm.node_domain.tolist(), adm.floor.tolist()) == \
        (ts.node_count.tolist(), ts.node_domain.tolist(), ts.floor.tolist())


def test_without_a_constraint_the_table_is_the_other_switches_one():
    sched, nodes, other, running = generated(7, n_sched=30)
    plain = [p for p in sched if p.topology_spread is None]
    for p in plain + running:
        p.anti_affinity_terms = ()
    lists = by_node(nodes, running)
    assert snapshot.pending_admit(plain, running, nodes, lists, anti_affinity=False, topology_spread=True,
                                  other_nodes=other) is None
    # a pod with a constraint adds the key and skew columns, nothing else
    adm = snapshot.pending_admit(sched, running, nodes, lists, anti_affinity=False, topology_spread=True)
    assert adm.row_carries is adm.row_has is adm.sig_carries is adm.sig_need is None and adm.node_match is None


# ---------------------------------------------------------------- hand-worked
def web(name, node=None, **constraint):
    return fake_pod(name, "ns", {"app": "web"}, None if node else [tsc(**constraint)], node)


def four():
    return [fake_node(n) for n in "ABCD"]


def test_pending_replica_holds_only_the_nodes_it_may_land_on():
    # A and B run one replica each, C and D none: the pending replica (maxSkew 1, selects itself) may land where the
    # count is at most 0 + min = 0
    running = [web("r0", "A"), web("r1", "B")]
    assert flagged([web("p")], four(), running) == [True, True, False, False]
    # maxSkew 2: every node
    assert flagged([web("p", skew=2)], four(), running) == [False] * 4
    # a replica on every node: the minimum is 1 and every node admits the pod again
    running += [web("r2", "C"), web("r3", "D")]
    assert flagged([web("p")], four(), running) == [False] * 4


def test_the_master_holds_the_minimum_at_zero():
    running = [web("r%d" % i, n) for i, n in enumerate("ABCD")]
    master = [fake_node("m", taints=[{"key": "node-role.kubernetes.io/master", "effect": "NoSchedule"}])]
    assert flagged([web("p")], four(), running, master) == [True] * 4
    # nodeTaintsPolicy Honor: the tainted master is no domain
    assert flagged([web("p", nodeTaintsPolicy="Honor")], four(), running, master) == [False] * 4


def test_an_ignored_pools_node_holds_the_minimum():
    running = [web("r%d" % i, n) for i, n in enumerate("ABCD")] + [web("i0", "ign0")]
    assert flagged([web("p")], four(), running, [fake_node("ign1")]) == [True] * 4
    assert flagged([web("p")], four(), running, [fake_node("ign0")]) == [False] * 4


def test_min_domains_above_the_domain_count_sets_the_floor_to_zero():
    running = [web("r%d" % i, n) for i, n in enumerate("ABCD")]
    assert flagged([web("p", minDomains=5)], four(), running) == [True] * 4
    assert flagged([web("p", minDomains=4)], four(), running) == [False] * 4


def test_a_key_with_no_domain_admits_every_node():
    # in the arrays: no node_domain bit and floor INT32_MAX give min = INT32_MAX, and the limit clamps to INT32_MAX
    got = ts_states_oracle.pending_admit_ts(np.zeros(5, np.int64), None, None, None, None, [0], None, None, None, [0],
                                            [1], [[5, 0, 7, INT32_MAX]], [0] * 4, [INT32_MAX], np.zeros(4, np.uint8))
    assert got.tolist() == [0] * 4
    # from the pods, a key without a domain has fewer domains than its minDomains (at least 1): floor 0, min 0
    running = [web("r%d" % i, "A") for i in range(5)]
    p = fake_pod("p", "ns", {"app": "web"}, [tsc()], selectors={"pool": "none"})
    assert flagged([p], four(), running) == [True, False, False, False]
    adm = snapshot.pending_admit([p], running, four(), by_node(four(), running), anti_affinity=False,
                                 topology_spread=True)
    assert adm.node_domain.tolist() == [0] * 4 and adm.floor.tolist() == [0]


def test_pod_its_own_selector_does_not_select_keeps_max_skew():
    # the pending db pod spreads over web pods: pod_skew = maxSkew = 1, so a count of min + 1 still admits it
    running = [web("r0", "A"), web("r1", "B"), web("r2", "C"), web("r3", "C"), web("r4", "D"), web("r5", "D"),
               web("r6", "D")]
    db = fake_pod("db", "ns", {"app": "db"}, [tsc()])
    assert flagged([db], four(), running) == [False, False, False, True]
    assert flagged([web("p")], four(), running) == [False, False, True, True]
    adm = snapshot.pending_admit([db], running, four(), by_node(four(), running), anti_affinity=False,
                                 topology_spread=True)
    assert adm.sig_skew.tolist() == [1]


def test_65_keys_are_refused():
    nodes = four()
    pods = [fake_pod("p%d" % i, "ns", {"app": "a%d" % i}, [tsc(selector={"matchLabels": {"app": "a%d" % i}})])
            for i in range(65)]
    assert snapshot.pending_admit(pods[:64], [], nodes, [[]] * 4, anti_affinity=False,
                                  topology_spread=True).sig_key.max() == 63
    with pytest.raises(ValueError, match="64"):
        snapshot.pending_admit(pods, [], nodes, [[]] * 4, anti_affinity=False, topology_spread=True)


# ---------------------------------------------------------------- the switch
def _cluster(**kw):
    from kubernetes_acs_engine_autoscaler_b200.cluster import Cluster
    return Cluster(kubeconfig=None, idle_threshold=60, spare_agents=1, service_principal_app_id="x",
                   service_principal_secret="x", service_principal_tenant_id="x", subscription_id="x",
                   client_private_key="x", ca_private_key="x", instance_init_time=600, resource_group="rg",
                   notifier=None, ignore_pools="", **kw)


def test_switch_reads_the_environment_and_needs_topology_spread(monkeypatch):
    monkeypatch.delenv("ACSFIT_TOPOLOGY_SPREAD", raising=False)
    for value, want in ((None, False), ("", False), ("0", False), ("1", True)):
        if value is None:
            monkeypatch.delenv("ACSFIT_TOPOLOGY_SPREAD_NODE_STATES", raising=False)
        else:
            monkeypatch.setenv("ACSFIT_TOPOLOGY_SPREAD_NODE_STATES", value)
        assert _cluster(topology_spread=True).topology_spread_node_states is want, value
        assert _cluster(topology_spread=False).topology_spread_node_states is False
        assert _cluster().topology_spread_node_states is False
    monkeypatch.setenv("ACSFIT_TOPOLOGY_SPREAD_NODE_STATES", "0")
    assert _cluster(topology_spread=True, topology_spread_node_states=True).topology_spread_node_states is True
    assert _cluster(topology_spread=True, topology_spread_node_states=False).topology_spread_node_states is False
    with pytest.raises(ValueError):
        _cluster(topology_spread=False, topology_spread_node_states=True)
    with pytest.raises(ValueError):
        _cluster(topology_spread_node_states=True)                       # $ACSFIT_TOPOLOGY_SPREAD unset: off
    monkeypatch.setenv("ACSFIT_TOPOLOGY_SPREAD", "1")
    c = _cluster(topology_spread_node_states=True)
    assert (c.topology_spread_node_states, c.pod_affinity_node_states, c.anti_affinity_node_states,
            c.selector_node_states) == (True, False, False, False)
    c = _cluster(pod_anti_affinity=True, anti_affinity_node_states=True, node_selectors=True,
                 selector_node_states=True, pod_affinity=True, pod_affinity_node_states=True,
                 topology_spread_node_states=True)
    assert (c.topology_spread_node_states, c.pod_affinity_node_states, c.anti_affinity_node_states,
            c.selector_node_states) == (True, True, True, True)


class _Stop(Exception):
    pass


@pytest.mark.parametrize("on", [False, True])
def test_switch_reaches_engine_scaler_and_scaler(monkeypatch, on):
    from kubernetes_acs_engine_autoscaler_b200 import cluster, engine_scaler
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    s = Scaler("rg", [], 0, 1, 60, True, None, None)
    assert s.topology_spread_node_states is False and s.other_nodes == []
    seen = []

    class Rec(engine_scaler.EngineScaler):
        def __init__(self, **kw):
            engine_scaler.EngineScaler.__init__(self, **kw)
            seen.append((self.topology_spread_node_states, [n.name for n in self.other_nodes]))
            raise _Stop()
    monkeypatch.setattr(cluster, "EngineScaler", Rec)
    cl = _cluster(topology_spread=True, topology_spread_node_states=on)
    meta = lambda name: {"metadata": {"name": name, "creationTimestamp": "2026-09-20T07:00:00Z",  # noqa: E731
                                      "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2"}}, "spec": {}}
    cl.list_nodes = lambda: [SimpleNamespace(obj=meta("k8s-cpu-1-0")), SimpleNamespace(obj=meta("k8s-master-1-0"))]
    cl.create_kube_node = lambda n: SimpleNamespace(name=n.obj["metadata"]["name"], selectors=n.obj["metadata"]["labels"],
                                                    unschedulable=False)
    cl.arm_parameters, cl.arm_template = {"cpuVMSize": {"value": "Standard_D2_v2"}}, {}
    with pytest.raises(_Stop):
        cl.loop_logic()
    assert seen == [(on, ["k8s-master-1-0"])]


class TsOracleEngine(AdmitOracleEngine):
    """AdmitOracleEngine with acsfit_pending_admit_ts answered by tests/ts_states_oracle.c"""

    def __init__(self):
        AdmitOracleEngine.__init__(self)
        self.ts_admits = 0

    def pending_admit_ts(self, row_ptr, rc, rm, rh, node_match, sig_class, sig_carries, sig_matches, sig_need,
                         sig_key, sig_skew, keys, node_count, node_domain, floor, node_flags):
        self.ts_admits += 1
        u64 = lambda t: None if t is None else t.numpy().view(U64)  # noqa: E731
        assert node_count.shape == (keys, len(node_flags))
        out = ts_states_oracle.pending_admit_ts(row_ptr.numpy(), u64(rc), u64(rm), u64(rh), u64(node_match),
                                                sig_class, sig_carries, sig_matches, sig_need, sig_key, sig_skew,
                                                node_count.numpy(), u64(node_domain), floor, node_flags.numpy())
        node_flags.copy_(torch.from_numpy(out))
        return node_flags


def spread_objects():
    """pools `cpu` (four old Standard_D2_v2 nodes) and `ign` (one node, ignored): one web replica runs on each cpu node
    and none on the ignored node; replica web-p is pending (maxSkew 1)"""
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

    def mk(name, node=None):
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "100m"}}}],
                "topologySpreadConstraints": [tsc()]}
        status = {"phase": "Pending"}
        if node:
            spec["nodeName"] = node
            status = {"phase": "Running", "startTime": "2016-08-25T05:13:16Z"}
        o = {"metadata": {"name": name, "namespace": "ns", "uid": "u-" + name, "labels": {"app": "web"},
                          "creationTimestamp": "2016-08-25T05:13:16Z"}, "spec": spec, "status": status}
        return KubePod(gu.FakeKubeObject(o, j, "pod"))
    running = [mk("web-%d" % i, nodes[i].name) for i in range(4)]
    return nodes, running, [mk("web-p")], j


@pytest.mark.parametrize("anti", [False, True])
@pytest.mark.parametrize("on", [False, True])
def test_maintain_sends_the_flag_only_when_on(tmp_path, monkeypatch, on, anti):
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.engine_scaler import EngineScaler
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    eng = TsOracleEngine()
    monkeypatch.setattr(snapshot, "_engine", eng)
    if not on:  # off: the spread builder is never reached, nor are the pods' constraints read for maintain
        def boom(*a, **k):
            raise AssertionError("topology spread read with topology_spread_node_states off")
        monkeypatch.setattr(snapshot, "topology_spread", boom)
        monkeypatch.setattr(snapshot, "_topology_spread", boom)
    nodes, running, pending, journal = spread_objects()
    params = {"cpuVMSize": {"value": "Standard_D2_v2"}, "ignVMSize": {"value": "Standard_D2_v2"},
              "masterVMSize": {"value": "Standard_D2_v2"}}
    s = EngineScaler("rg", nodes, 0, 0, 1800, True, None, {}, params, "ign", None, topology_spread=True,
                     topology_spread_node_states=on, pod_anti_affinity=anti, anti_affinity_node_states=anti)
    cpu = nodes[:4]
    lists = [[p for p in running if p.node_name == n.name] for n in cpu]
    states = [s.get_node_state(n, lst, pending) for n, lst in zip(cpu, lists)]
    s.maintain(pending, running)
    flags = eng.sent[-1]
    if on:
        # the ignored pool's empty node holds the minimum at 0, so no cpu node (count 1) admits web-p
        assert flags.tolist() == [2, 2, 2, 2] and eng.ts_admits == 5 and eng.admits == 0
        # get_node_state sees only the node: its own count is the minimum, so web-p may land there
        assert states == ["pod-pending"] * 4
    else:
        assert flags.tolist() == [0, 0, 0, 0] and eng.ts_admits == 0 and eng.admits == 0
        assert states == ["pod-pending"] * 4
    assert journal == []  # dry run
    # nothing to schedule: no admission call
    n0 = eng.ts_admits
    s.maintain([], running)
    assert eng.sent[-1].tolist() == [0, 0, 0, 0] and eng.ts_admits == n0
    if on:  # one-node get_node_state with minDomains 2: one domain < 2, floor 0, the node's count 1 is too many
        pending[0].original.obj["spec"]["topologySpreadConstraints"] = [tsc(minDomains=2)]
        pending[0].__dict__.pop("topology_spread", None)
        assert s.get_node_state(cpu[0], lists[0], pending) != "pod-pending"
        assert s.get_node_state(nodes[4], [], pending) == "pod-pending"
