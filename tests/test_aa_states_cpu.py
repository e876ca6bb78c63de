"""`-m "not gpu"`: the host side of Cluster(anti_affinity_node_states=True) -- a node is pod-pending only when some pod
to schedule could land on it given the pods already there (required pod anti-affinity, both directions).

* The plain-C oracle (tests/aa_states_oracle.c) and the host masks (snapshot.pending_admit / anti_affinity_rows)
  against a plain-Python restatement that applies kube's anti-affinity predicates per (pod to schedule, node), with and
  without node selectors, on generated clusters: nodes without pods, pods on unlisted nodes, one node holding every pod.
* The oracle against a numpy restatement on the kernel's edge shapes: row_ptr[0] > 0, class 63 and term bit 63, the
  only admitting signature last, no signature admitting, U = 0.
* The switch: its environment variable, its ValueError, and the node flags maintain sends with it on and off (the
  oracle stands in for the GPU)."""
import itertools
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import aa_states_oracle
import golden_util as gu
from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot
from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode
from test_anti_affinity_cpu import affinity, generated, term

NO_MATCH = 2  # ACSFIT_NODEF_NO_PENDING_MATCH
POOLS = ("p0", "p1", "p2")


def selects(owner, q):
    """a term of `owner` selects pod q (kube's predicates, hostname topology)"""
    return any(q.namespace in ns and kube.selector_matches(sel, q.labels) for ns, sel in owner.anti_affinity_terms)


def restated_admits(sched, nodes, lists, selectors):
    """bool[N]: some pod to schedule matches the node (KubeNode.is_match, with selectors) and neither blocks a pod of
    the node nor is blocked by one -- pair by pair"""
    return np.array([any((not selectors or KubeNode.is_match(n, p)) and
                         not any(selects(p, q) or selects(q, p) for q in lst) for p in sched)
                     for n, lst in zip(nodes, lists)], dtype=bool)


def by_node(nodes, running):
    groups = {}
    for p in running:
        groups.setdefault(p.node_name, []).append(p)
    return [groups.get(n.name, []) for n in nodes]


def csr(lists, base=0):
    return base + np.concatenate([[0], np.cumsum([len(l) for l in lists])]).astype(np.int64)


def with_selectors(seed, sched, nodes, running):
    rng = np.random.default_rng([seed, 7])
    for n in nodes:
        n.selectors = {"pool": POOLS[int(rng.integers(3))]} if rng.random() < 0.9 else {}
    for p in itertools.chain(sched, running):
        p.selectors = {"pool": POOLS[int(rng.integers(3))]} if rng.random() < 0.7 else {}


def check_host_and_oracle(sched, nodes, running, lists, selectors):
    want = restated_admits(sched, nodes, lists, selectors)
    adm = snapshot.pending_admit(sched, running, nodes, lists, selectors=selectors)
    row_ptr = csr(lists)
    zeros = np.zeros(len(nodes), np.uint8)
    if adm is None:  # no term can block a pod to schedule: the selector rule alone decides
        assert snapshot.anti_affinity(sched, nodes, running).trivial
        base = snapshot.pending_match(sched, nodes) if selectors else np.ones(len(nodes), bool)
        np.testing.assert_array_equal(base, want)
        return None
    flags = aa_states_oracle.pending_admit(row_ptr, adm.row_carries, adm.row_matches, adm.node_match, adm.sig_class,
                                           adm.sig_carries, adm.sig_matches, zeros)
    np.testing.assert_array_equal((flags & NO_MATCH) == 0, want)
    assert not (flags & ~np.uint8(NO_MATCH)).any()
    # the signatures are the distinct (class, carries, matches) of the pods: the oracle over every pod agrees
    pc, pm, rc, rm, terms = snapshot.anti_affinity_rows(sched, running, lists)
    cls = snapshot.selector_classes(sched, nodes, []) if selectors else None
    pod_class = cls.pod_class if cls is not None and not cls.trivial else np.zeros(len(sched), np.uint8)
    node_match = cls.node_match if cls is not None and not cls.trivial else None
    per_pod = aa_states_oracle.pending_admit(row_ptr, rc, rm, node_match, pod_class, pc, pm, zeros)
    np.testing.assert_array_equal(per_pod, flags)
    sigs = set(zip(adm.sig_class.tolist(), adm.sig_carries.tolist(), adm.sig_matches.tolist()))
    assert len(sigs) == len(adm.sig_class) == len(set(zip(pod_class.tolist(), pc.tolist(), pm.tolist())))
    # same term numbering and dropping as anti_affinity, whose node masks are the OR of the rows
    aa = snapshot.anti_affinity(sched, nodes, running)
    assert terms == aa.terms
    node_of = np.repeat(np.arange(len(nodes)), np.diff(row_ptr))
    for mask, node_mask in ((rc, aa.node_carries), (rm, aa.node_matches)):
        ored = np.zeros(len(nodes), np.uint64)
        np.bitwise_or.at(ored, node_of, mask)
        np.testing.assert_array_equal(ored, node_mask)
    return flags


@pytest.mark.parametrize("selectors", [False, True])
@pytest.mark.parametrize("seed", range(6))
def test_admission_matches_pairwise_restatement(seed, selectors):
    sched, nodes, running = generated(seed, n_sched=40, n_run=300, n_nodes=50)
    nodes[5:5] = [SimpleNamespace(name="empty-%d" % i) for i in range(3)]  # nodes without pods
    if selectors:
        with_selectors(seed, sched, nodes, running)
    lists = by_node(nodes, running)
    assert any(not l for l in lists)
    flags = check_host_and_oracle(sched, nodes, running, lists, selectors)
    assert flags is not None
    # a subset of the pods to schedule: fewer admitted nodes, and some node both ways
    few = check_host_and_oracle(sched[:3], nodes, running, lists, selectors)
    if few is not None:
        assert ((few & NO_MATCH) >= (flags & NO_MATCH)).all()


def test_replicas_spread_one_per_node():
    """the motivating shape: a self-anti-affine deployment, one replica per node on some nodes, one replica pending"""
    web = term({"matchLabels": {"app": "web"}})
    mk = lambda name, node=None, app="web", terms=(web,): SimpleNamespace(  # noqa: E731
        name=name, namespace="ns", labels={"app": app}, node_name=node, selectors={},
        anti_affinity_terms=kube.anti_affinity_terms(affinity(*terms), "ns", "pod " + name))
    nodes = [SimpleNamespace(name="n%d" % i, selectors={}) for i in range(6)]
    running = [mk("web-%d" % i, "n%d" % i) for i in range(3)] + [mk("db", "n3", app="db", terms=())]
    pending = [mk("web-9")]
    lists = by_node(nodes, running)
    flags = check_host_and_oracle(pending, nodes, running, lists, False)
    assert ((flags & NO_MATCH) != 0).tolist() == [True, True, True, False, False, False]
    # one node holding every pod
    everything = [SimpleNamespace(**dict(vars(p), node_name="n5")) for p in running]
    flags = check_host_and_oracle(pending, nodes, everything, by_node(nodes, everything), False)
    assert ((flags & NO_MATCH) != 0).tolist() == [False] * 5 + [True]
    # a pod to schedule that carries no term but is selected by a running pod's term is blocked there too
    plain = mk("web-plain", terms=())
    flags = check_host_and_oracle([plain], nodes, running, lists, False)
    assert ((flags & NO_MATCH) != 0).tolist() == [True, True, True, False, False, False]


def test_rows_refuse_a_pod_that_is_not_running():
    sched, nodes, running = generated(1)
    with pytest.raises(ValueError):
        snapshot.anti_affinity_rows(sched, running[1:], [[running[0]]])


# ---------------------------------------------------------------- the oracle on the kernel's edge shapes
def py_admit(row_ptr, rc, rm, node_match, cls, car, mat, flags):
    out = flags.copy()
    for n in range(len(flags)):
        nc = nx = 0
        for k in range(int(row_ptr[n]), int(row_ptr[n + 1])):
            nc |= int(rc[k])
            nx |= int(rm[k])
        ok = any((node_match is None or (int(node_match[n]) >> int(c)) & 1) and (int(a) & nx | int(b) & nc) == 0
                 for c, a, b in zip(cls, car, mat))
        if not ok:
            out[n] |= NO_MATCH
    return out


def edge_case(kind, rng):
    N = 37
    lens = rng.integers(0, 5, size=N)
    lens[::7] = 0
    base = 11 if kind == "offset" else 0
    row_ptr = csr([[None] * int(k) for k in lens], base)
    R = int(row_ptr[-1])
    rc = rng.integers(0, 1 << 63, size=R, dtype=np.uint64) & rng.integers(0, 1 << 63, size=R, dtype=np.uint64)
    rm = rc ^ rng.integers(0, 1 << 63, size=R, dtype=np.uint64) & np.uint64(0xF0F0)
    rc[base:] |= np.uint64(1) << np.uint64(63)
    node_match = rng.integers(0, 1 << 63, size=N, dtype=np.uint64) | np.uint64(1)
    node_match[::3] |= np.uint64(1) << np.uint64(63)
    U = 9
    cls = rng.integers(0, 64, size=U).astype(np.uint8)
    car = rng.integers(0, 1 << 63, size=U, dtype=np.uint64) & np.uint64(0xFF)
    mat = np.zeros(U, np.uint64)
    if kind == "bit63":
        cls[:] = 63
        mat[:] = np.uint64(1) << np.uint64(63)
        mat[-1] = 0
    elif kind == "last_admits":
        cls[:] = 0
        mat[:] = np.uint64(1) << np.uint64(63)  # every node has a carrier of bit 63 ... except the empty ones
        mat[-1] = 0
        car[-1] = 0
    elif kind == "none":  # every node with a pod blocks every signature; a node without pods blocks nothing
        cls[:] = 0
        car[:] = ~np.uint64(0)
        mat[:] = ~np.uint64(0)
    elif kind == "u0":
        cls, car, mat = cls[:0], car[:0], mat[:0]
    flags = (rng.random(N) < 0.3).astype(np.uint8) | np.uint8(4)
    return row_ptr, rc, rm, node_match, cls, car, mat, flags


@pytest.mark.parametrize("with_match", [False, True])
@pytest.mark.parametrize("kind", ["random", "offset", "bit63", "last_admits", "none", "u0"])
def test_oracle_edges(kind, with_match):
    rng = np.random.default_rng(len(kind))
    row_ptr, rc, rm, node_match, cls, car, mat, flags = edge_case(kind, rng)
    nm = node_match if with_match else None
    got = aa_states_oracle.pending_admit(row_ptr, rc, rm, nm, cls, car, mat, flags)
    np.testing.assert_array_equal(got, py_admit(row_ptr, rc, rm, nm, cls, car, mat, flags))
    assert ((got & ~np.uint8(NO_MATCH)) == (flags & ~np.uint8(NO_MATCH))).all()  # no other bit changes
    if kind == "none":
        np.testing.assert_array_equal((got & NO_MATCH) != 0, np.diff(row_ptr) > 0)
    if kind == "u0":
        assert (got & NO_MATCH).all()
    if kind == "last_admits" and not with_match:
        assert not (got & NO_MATCH).any()


# ---------------------------------------------------------------- the switch
def _cluster(**kw):
    from kubernetes_acs_engine_autoscaler_b200.cluster import Cluster
    return Cluster(kubeconfig=None, idle_threshold=60, spare_agents=1, service_principal_app_id="x",
                   service_principal_secret="x", service_principal_tenant_id="x", subscription_id="x",
                   client_private_key="x", ca_private_key="x", instance_init_time=600, resource_group="rg",
                   notifier=None, ignore_pools="", **kw)


def test_switch_reads_the_environment_and_needs_pod_anti_affinity(monkeypatch):
    monkeypatch.delenv("ACSFIT_POD_ANTI_AFFINITY", raising=False)
    for value, want in ((None, False), ("", False), ("0", False), ("1", True), ("yes", True)):
        if value is None:
            monkeypatch.delenv("ACSFIT_ANTI_AFFINITY_NODE_STATES", raising=False)
        else:
            monkeypatch.setenv("ACSFIT_ANTI_AFFINITY_NODE_STATES", value)
        assert _cluster(pod_anti_affinity=True).anti_affinity_node_states is want, value
        assert _cluster(pod_anti_affinity=False).anti_affinity_node_states is False
        assert _cluster().anti_affinity_node_states is False
    monkeypatch.setenv("ACSFIT_ANTI_AFFINITY_NODE_STATES", "0")
    assert _cluster(pod_anti_affinity=True, anti_affinity_node_states=True).anti_affinity_node_states is True
    assert _cluster(pod_anti_affinity=True, anti_affinity_node_states=False).anti_affinity_node_states is False
    assert _cluster(pod_anti_affinity=False, anti_affinity_node_states=False).anti_affinity_node_states is False
    with pytest.raises(ValueError):
        _cluster(pod_anti_affinity=False, anti_affinity_node_states=True)
    with pytest.raises(ValueError):
        _cluster(anti_affinity_node_states=True)                      # $ACSFIT_POD_ANTI_AFFINITY unset: off
    monkeypatch.setenv("ACSFIT_POD_ANTI_AFFINITY", "1")
    assert _cluster(anti_affinity_node_states=True).anti_affinity_node_states is True


def test_combined_mode_refuses_65_selector_classes():
    sched, nodes, running = generated(2, n_nodes=80)
    for i, n in enumerate(nodes):
        n.selectors = {"host": "h%d" % i}
    for i, p in enumerate(sched):
        p.selectors = {"host": "h%d" % (i % 80)}                         # 80 node sets: 80 classes besides class 0
    lists = by_node(nodes, running)
    assert snapshot.pending_admit(sched, running, nodes, lists) is not None
    with pytest.raises(ValueError):
        snapshot.pending_admit(sched, running, nodes, lists, selectors=True)


class AdmitOracleEngine(object):
    """the oracle engine with acsfit_pending_admit answered by tests/aa_states_oracle.c and
    ACSFIT_NODEF_NO_PENDING_MATCH applied to K6 as np.where(flag, states(any_pending=0), states(any_pending)); records
    the node flags K6 is sent and the admission calls"""

    def __init__(self):
        from oracle_engine import OracleEngine
        self.base = OracleEngine()
        self.sent, self.admits = [], 0

    def __getattr__(self, name):
        return getattr(self.base, name)

    def pending_admit(self, row_ptr, rc, rm, node_match, sig_class, sig_carries, sig_matches, node_flags):
        self.admits += 1
        out = aa_states_oracle.pending_admit(row_ptr.numpy(), rc.numpy().view(np.uint64), rm.numpy().view(np.uint64),
                                             None if node_match is None else node_match.numpy().view(np.uint64),
                                             sig_class, sig_carries, sig_matches, node_flags.numpy())
        node_flags.copy_(torch.from_numpy(out))
        return node_flags

    def node_states(self, row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags, node_age,
                    any_pending, thr):
        flags = node_flags.numpy().copy()
        self.sent.append(flags)
        st = {ap: self.base.node_states(row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags,
                                        node_age, ap, thr).numpy() for ap in (False, any_pending)}
        return torch.from_numpy(np.where(flags & NO_MATCH, st[False], st[any_pending]))


CREATED_BY = '{"kind":"SerializedReference","reference":{"kind":"ReplicaSet","name":"web-1"}}'


def replica_objects():
    """pool `cpu`: four old, schedulable Standard_D2_v2 nodes; replicas web-0 and web-1 (one per node, each avoiding
    app=web on its node) run on the first two, a db pod on the third; replica web-2 is pending"""
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.kube import KubePod
    j = []
    nodes = []
    for i in range(4):
        o = {"metadata": {"name": "k8s-cpu-1-%d" % i, "creationTimestamp": "2016-08-25T05:13:16Z",
                          "labels": {"agentpool": "cpu", "beta.kubernetes.io/instance-type": "Standard_D2_v2",
                                     "failure-domain.beta.kubernetes.io/region": "r"}},
             "spec": {}}
        n = KubeNode(gu.FakeKubeObject(o, j, "node"))
        n.capacity = capacity.get_capacity_for_instance_type(n.instance_type)
        nodes.append(n)
    aff = affinity(term({"matchLabels": {"app": "web"}}))

    def pod(name, app, node=None):
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "100m"}}}]}
        if app == "web":
            spec["affinity"] = aff
        status = {"phase": "Pending"}
        if node:
            spec["nodeName"] = node
            status = {"phase": "Running", "startTime": "2016-08-25T05:13:16Z"}
        o = {"metadata": {"name": name, "namespace": "ns", "uid": "u-" + name, "labels": {"app": app},
                          "annotations": {"kubernetes.io/created-by": CREATED_BY},
                          "creationTimestamp": "2016-08-25T05:13:16Z"}, "spec": spec, "status": status}
        return KubePod(gu.FakeKubeObject(o, j, "pod"))
    running = [pod("web-0", "web", nodes[0].name), pod("web-1", "web", nodes[1].name), pod("db", "db", nodes[2].name)]
    return nodes, running, [pod("web-2", "web")], j


@pytest.mark.parametrize("on", [False, True])
def test_maintain_sends_the_flag_only_when_on(tmp_path, monkeypatch, on):
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.engine_scaler import EngineScaler
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    eng = AdmitOracleEngine()
    monkeypatch.setattr(snapshot, "_engine", eng)
    if not on:  # off: no host work and no launch beyond the reference's
        monkeypatch.setattr(snapshot, "pending_admit", None)
    nodes, running, pending, journal = replica_objects()
    params = {"cpuVMSize": {"value": "Standard_D2_v2"}, "masterVMSize": {"value": "Standard_D2_v2"}}
    s = EngineScaler("rg", nodes, 0, 0, 1800, True, None, {}, params, "", None, pod_anti_affinity=True,
                     anti_affinity_node_states=on)
    lists = [[p for p in running if p.node_name == n.name] for n in nodes]
    states = [s.get_node_state(n, lst, pending) for n, lst in zip(nodes, lists)]
    s.maintain(pending, running)
    flags = eng.sent[-1]
    if on:
        # get_node_state of the db node and of the empty node keeps no term (web-2 meets no other web pod): no call
        assert flags.tolist() == [2, 2, 0, 0] and eng.admits == 3
        assert states == ["under-utilized-drainable"] * 2 + ["pod-pending"] * 2
    else:
        assert flags.tolist() == [0, 0, 0, 0] and eng.admits == 0
        assert states == ["pod-pending"] * 4
    assert journal == []  # dry run
    # nothing to schedule: no admission call, the reference's states
    eng.sent.clear()
    n0 = eng.admits
    s.maintain([], running)
    assert eng.sent[-1].tolist() == [0, 0, 0, 0] and eng.admits == n0
