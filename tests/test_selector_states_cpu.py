"""`-m "not gpu"`: the host side of the selector-aware node states (Cluster(selector_node_states=True)).

* snapshot.pending_match against `any(KubeNode.is_match(node, pod) for pod in pods)` on generated nodes and pods:
  pods without selectors mixed in, selector keys no node carries, nodes without labels, hostname pins, the
  autoscaler's cordon label, several pods sharing one selector.
* The expected K6 answer with ACSFIT_NODEF_NO_PENDING_MATCH needs no new C code: it is
  np.where(match, states(any_pending=1), states(any_pending=0)) from two calls of the pinned oracle.  That
  construction reproduces a plain-Python restatement of the upstream get_node_state, whose POD_PENDING branch asks
  for a pending pod that matches the node.
* The switch: its environment variable, its dependence on node_selectors, and the node flags maintain sends (the
  oracle stands in for the GPU, with the construction above for bit 1)."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import golden_util as gu
import idle_cases as ic
from kubernetes_acs_engine_autoscaler_b200 import snapshot
from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode

HOST, CORDON, POOL, ITYPE = "kubernetes.io/hostname", "openai/cordoned-by-autoscaler", "agentpool", \
    "beta.kubernetes.io/instance-type"
POOLS, TYPES = ("cpu", "gpu", "mem"), ("Standard_D2_v2", "Standard_NC6")


def gen_nodes(rng, N):
    nodes = []
    for i in range(N):
        if rng.random() < 0.1:
            labels = {}                                                     # a node without labels
        else:
            labels = {POOL: POOLS[rng.integers(len(POOLS))], HOST: "node-%d" % i, ITYPE: TYPES[rng.integers(2)]}
            if rng.random() < 0.2:
                labels[CORDON] = "true"
            if rng.random() < 0.3:
                labels["zone"] = str(rng.integers(3))
        nodes.append(SimpleNamespace(selectors=labels))
    return nodes


def gen_selectors(rng, N, k):
    """k distinct selectors of every kind (some of them repeated by the pods)"""
    kinds = [
        lambda: {POOL: POOLS[rng.integers(len(POOLS))]},
        lambda: {HOST: "node-%d" % rng.integers(max(N, 1))},                # hostname pin
        lambda: {POOL: POOLS[rng.integers(len(POOLS))], ITYPE: TYPES[rng.integers(2)]},
        lambda: {"no-node-has-this": "x"},                                  # a key no node carries
        lambda: {POOL: "gpu", "no-node-has-this": "x"},
        lambda: {CORDON: "true"},                                           # the autoscaler's cordon label
        lambda: {"zone": str(rng.integers(3)), POOL: POOLS[rng.integers(len(POOLS))]},
        lambda: {POOL: "nosuchpool"},
    ]
    return [kinds[i % len(kinds)]() for i in range(k)]


def pods_for(rng, selectors, P, unselected=0):
    pods = [SimpleNamespace(selectors=dict(selectors[rng.integers(len(selectors))])) for _ in range(P)]
    for _ in range(unselected):
        pods.insert(int(rng.integers(len(pods) + 1)), SimpleNamespace(selectors={}))
    return pods


def plain_match(pods, nodes):
    return np.array([any(KubeNode.is_match(n, p) for p in pods) for n in nodes], dtype=bool)


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("k", [1, 3, 8, 20])
def test_pending_match_equals_is_match(seed, k):
    rng = np.random.default_rng([seed, k])
    N = int(rng.integers(1, 400))
    nodes = gen_nodes(rng, N)
    sels = gen_selectors(rng, N, k)
    pods = pods_for(rng, sels, 3 * k)                                       # several pods share each selector
    got = snapshot.pending_match(pods, nodes)
    assert got.dtype == bool and got.shape == (N,)
    np.testing.assert_array_equal(got, plain_match(pods, nodes))
    # a pod without a selector matches every node
    mixed = pods_for(rng, sels, k, unselected=1)
    assert snapshot.pending_match(mixed, nodes).all() and plain_match(mixed, nodes).all()


def test_pending_match_edges():
    nodes = [SimpleNamespace(selectors=l) for l in ({}, {"a": "1"}, {"a": "2", "b": "1"}, {"b": "1"})]
    P = lambda *sels: [SimpleNamespace(selectors=s) for s in sels]  # noqa: E731
    for pods in (P(), P({"c": "1"}), P({"a": "1"}, {"a": "1"}), P({"a": "2", "b": "1"}, {"b": "1"}),
                 P({"b": "1", "a": "3"}), P({"a": None}),                  # None matches a missing label, as in is_match
                 P({"a": "1"}, {"b": "1"}, {"c": "9"})):
        np.testing.assert_array_equal(snapshot.pending_match(pods, nodes), plain_match(pods, nodes), err_msg=str(pods))
    assert snapshot.pending_match(P({"a": "1"}), []).shape == (0,)
    assert not snapshot.pending_match(P(), nodes).any()


def test_pending_match_sees_the_cordon_label():
    """KubeNode.cordon() writes the cordon label into the node's labels: a pod pinned to it then matches"""
    j = []
    objs = [{"metadata": {"name": "k8s-agentpool1-1-%d" % i, "creationTimestamp": "2026-09-20T07:00:00Z",
                          "labels": {POOL: "agentpool1", HOST: "k8s-agentpool1-1-%d" % i}}, "spec": {}} for i in range(3)]
    nodes = [KubeNode(gu.FakeKubeObject(o, j, "node")) for o in objs]
    pods = [SimpleNamespace(selectors={CORDON: "true"})]
    assert not snapshot.pending_match(pods, nodes).any()
    nodes[1].cordon()
    np.testing.assert_array_equal(snapshot.pending_match(pods, nodes), [False, True, False])
    np.testing.assert_array_equal(snapshot.pending_match(pods, nodes), plain_match(pods, nodes))


def test_pending_match_at_scale_groups_nodes():
    """20 k nodes of a few label projections plus hostname pins: same answer as the per-node evaluation"""
    rng = np.random.default_rng(11)
    nodes = gen_nodes(rng, 20000)
    sels = gen_selectors(rng, 20000, 64)
    pods = pods_for(rng, sels, 200)
    np.testing.assert_array_equal(snapshot.pending_match(pods, nodes), plain_match(pods, nodes))


# ---------------------------------------------------------------- the oracle construction vs upstream get_node_state
STATE = {name: code for code, name in enumerate(
    ["instance-terminated", "pod-pending", "grace-period", "spare-agent", "idle-schedulable", "idle-unschedulable",
     "busy-unschedulable", "busy", "under-utilized-drainable", "under-utilized-undrainable"])}


def upstream_states(c, nodes, pods):
    """get_node_state of the upstream ec2 autoscaler on one CSR case, node by node in plain Python: POD_PENDING needs
    a pending pod that matches the node (pending_list)"""
    S, N, D = c["S"], c["N"], c["D"]
    out = np.zeros((S, N), dtype=np.uint8)
    rp, req, flags = c["row_ptr"], c["req_run"], c["flags_run"]
    for n in range(N):
        busy = undrainable = False
        util = [0.0] * D
        for k in range(int(rp[n]), int(rp[n + 1])):
            f = int(flags[k])
            undrainable = undrainable or bool(f & ic.PODF_UNDRAINABLE)
            if f & ic.PODF_BUSY:
                busy = True
                util = [u + float(r) for u, r in zip(util, req[k])]
        cap = c["cap_type"][c["node_type"][n]]
        under = all(float(cap[d]) * 0.3 - util[d] >= 0 for d in range(D))
        unsched = bool(c["node_flags"][n] & ic.NODEF_UNSCHEDULABLE)
        pending_list = [p for p in pods if KubeNode.is_match(nodes[n], p)]
        for s in range(S):
            if busy and not under:
                st = "busy-unschedulable" if unsched else "busy"
            elif pending_list and not unsched:
                st = "pod-pending"
            elif c["node_age"][n] <= c["thr"][s] and not unsched:
                st = "grace-period"
            elif under and (busy or not unsched):
                st = "under-utilized-undrainable" if undrainable else "under-utilized-drainable"
            else:
                st = "idle-unschedulable" if unsched else "idle-schedulable"
            out[s, n] = STATE[st]
    return out


def construction(oracle_mod, c, match):
    idx = ic.identity_idx(c)
    st = {ap: oracle_mod.node_states(c["row_ptr"], idx, c["req_run"], c["flags_run"], c["cap_type"], c["node_type"],
                                     c["node_flags"], c["node_age"], ap, c["thr"]) for ap in (False, True)}
    return np.where(match, st[True], st[False]), st


@pytest.mark.parametrize("name", [n for n in ic.NAMES if ic.CASES[n][0] < 10000])
def test_oracle_construction_is_upstream_get_node_state(oracle_mod, name):
    c = ic.case(name, 4)
    rng = np.random.default_rng(len(name))
    nodes = gen_nodes(rng, c["N"])
    sels = gen_selectors(rng, c["N"], 8)
    decided = False
    for pods in (pods_for(rng, sels, 12), pods_for(rng, sels[:2], 4), [], pods_for(rng, sels, 3, unselected=1)):
        match = snapshot.pending_match(pods, nodes)
        want, st = construction(oracle_mod, c, match)
        np.testing.assert_array_equal(want, upstream_states(c, nodes, pods))
        decided |= bool((want != st[True]).any() and (want != st[False]).any())  # both rules appear
    assert decided or c["N"] < 100


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
            monkeypatch.delenv("ACSFIT_SELECTOR_NODE_STATES", raising=False)
        else:
            monkeypatch.setenv("ACSFIT_SELECTOR_NODE_STATES", value)
        assert _cluster(node_selectors=True).selector_node_states is want, value
        assert _cluster(node_selectors=False).selector_node_states is False   # no effect without node selectors
        assert _cluster().selector_node_states is False
    monkeypatch.setenv("ACSFIT_SELECTOR_NODE_STATES", "0")
    assert _cluster(node_selectors=True, selector_node_states=True).selector_node_states is True
    assert _cluster(node_selectors=True, selector_node_states=False).selector_node_states is False
    assert _cluster(node_selectors=False, selector_node_states=False).selector_node_states is False
    with pytest.raises(ValueError):
        _cluster(node_selectors=False, selector_node_states=True)
    with pytest.raises(ValueError):
        _cluster(selector_node_states=True)                                  # $ACSFIT_NODE_SELECTORS unset: off
    monkeypatch.setenv("ACSFIT_NODE_SELECTORS", "1")
    assert _cluster(selector_node_states=True).selector_node_states is True


class FlagOracleEngine(object):
    """the oracle engine, with ACSFIT_NODEF_NO_PENDING_MATCH applied by the construction above; records the node
    flags it is sent"""

    def __init__(self):
        from oracle_engine import OracleEngine
        self.base = OracleEngine()
        self.sent = []

    def __getattr__(self, name):
        return getattr(self.base, name)

    def node_states(self, row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags, node_age,
                    any_pending, thr):
        flags = node_flags.numpy().copy()
        self.sent.append((flags, bool(any_pending)))
        st = {ap: self.base.node_states(row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags,
                                        node_age, ap, thr).numpy() for ap in (False, any_pending)}
        return torch.from_numpy(np.where(flags & 2, st[False], st[any_pending]))


def _tick_objects():
    """three idle, old, schedulable nodes in pool `cpu`, one in pool `gpu`; one pending pod pinned to `gpu`"""
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.kube import KubePod
    j = []
    nodes = []
    for pool, i in (("cpu", 0), ("cpu", 1), ("cpu", 2), ("gpu", 0)):
        o = {"metadata": {"name": "k8s-%s-1-%d" % (pool, i), "creationTimestamp": "2016-08-25T05:13:16Z",
                          "labels": {POOL: pool, ITYPE: "Standard_D2_v2", "failure-domain.beta.kubernetes.io/region": "r"}},
             "spec": {}}
        n = KubeNode(gu.FakeKubeObject(o, j, "node"))
        n.capacity = capacity.get_capacity_for_instance_type(n.instance_type)
        nodes.append(n)
    pod = {"metadata": {"name": "p", "namespace": "ns", "uid": "u", "creationTimestamp": "2026-09-21T07:00:00Z"},
           "spec": {"containers": [{"name": "c", "resources": {"requests": {"cpu": "1"}}}], "nodeSelector": {POOL: "gpu"}},
           "status": {"phase": "Pending"}}
    return nodes, [KubePod(gu.FakeKubeObject(pod, j, "pod"))], j


@pytest.mark.parametrize("on", [False, True])
def test_maintain_sends_the_flag_only_when_on(tmp_path, monkeypatch, oracle_mod, on):
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.engine_scaler import EngineScaler
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    eng = FlagOracleEngine()
    monkeypatch.setattr(snapshot, "_engine", eng)
    nodes, pods, journal = _tick_objects()
    params = {"cpuVMSize": {"value": "Standard_D2_v2"}, "gpuVMSize": {"value": "Standard_D2_v2"},
              "masterVMSize": {"value": "Standard_D2_v2"}}
    s = EngineScaler("rg", nodes, 0, 1, 1800, False, None, {}, params, "", None, node_selectors=True,
                     selector_node_states=on)
    states = [s.get_node_state(n, [], pods) for n in nodes]
    s.maintain(pods, [])
    flags, any_pending = eng.sent[-1]
    assert any_pending
    if on:
        assert states == ["under-utilized-drainable"] * 3 + ["pod-pending"]
        assert flags.tolist() == [2, 2, 2, 0]
        # budget: 3 nodes - 1 spare: two are cordoned and drained, the third is a spare agent
        assert [e for e in journal if e[0] == "node.update"] == [["node.update", "k8s-cpu-1-0", True, "true"],
                                                                 ["node.update", "k8s-cpu-1-1", True, "true"]]
    else:
        assert states == ["pod-pending"] * 4
        assert flags.tolist() == [0, 0, 0, 0]
        assert journal == []
    # nothing to schedule: the flag is not computed, and the states are the reference's
    eng.sent.clear()
    s.maintain([], [])
    assert eng.sent[-1][0].tolist() == [int(n.unschedulable) for n in nodes] and not eng.sent[-1][1]


def test_no_pending_match_is_none_when_it_cannot_matter():
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    s = Scaler("rg", [], 0, 1, 60, True, None, None)
    nodes = [SimpleNamespace(selectors={POOL: "a"})]
    pinned = [SimpleNamespace(selectors={POOL: "b"})]
    assert s.selector_node_states is False and s.no_pending_match(nodes, pinned) is None
    s.selector_node_states = True
    assert s.no_pending_match(nodes, []) is None
    assert s.no_pending_match(nodes, pinned).tolist() == [True]
    assert s.no_pending_match(nodes, [SimpleNamespace(selectors={})]).tolist() == [False]
