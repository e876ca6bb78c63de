"""`-m gpu`: node states with pod anti-affinity -- acsfit_pending_admit and Cluster(anti_affinity_node_states=True).

* The kernel equals the plain-C oracle (tests/aa_states_oracle.c, per signature, no deduplication) exactly on
  N in {1, 31, 33, 2000, about 10^6}, U in {1, 255, 256, 257, 4000} (one shared-memory tile holds 256 signatures), with
  and without node_match, on: random masks and classes, nodes without pods, one node holding every pod,
  row_ptr[0] > 0, nodes admitted in the first tile beside nodes admitted only by the last signature (either direction
  of the block test), the only admitting signature last, no signature admitting, class 63 and term bit 63.  Every
  call's launch record must show kernel 3 with the expected grid and U.
* Views at an element offset are read correctly; misaligned arrays, NULL arrays that are read, class 64, U < 0, N < 0
  and a decreasing row_ptr are refused with ACSFIT_E_INVALID, leaving the flags untouched.
* The recorded reference ticks with every switch on and no anti-affinity term: the reference's tick, the same node
  flags sent to K6.
* The motivating tick: one replica per node plus one pending replica.  Nodes that run a sibling are no longer
  pod-pending, the others still are, and the dry-run journal equals a plain-Python restatement of maintain with the
  rule."""
import ctypes

import numpy as np
import pytest
import torch

import aa_states_oracle
import golden_util as gu
from kubernetes_acs_engine_autoscaler_b200 import _native, kube
from test_gpu_selector_states import DRY_MAINTAIN, restate_maintain
from test_gpu_selector_states import tick as tick2

pytestmark = pytest.mark.gpu

NO_MATCH = 2  # ACSFIT_NODEF_NO_PENDING_MATCH
TILE = 256    # signatures per shared-memory tile = threads per CTA (csrc/acsfit_admit.cuh)
U64 = np.uint64
KINDS = ("random", "empty", "one_node", "mixed_carries", "mixed_matches", "last_admits", "none", "bit63")


@pytest.fixture(scope="module")
def eng():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from kubernetes_acs_engine_autoscaler_b200 import build as acs_build
    acs_build.build()
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    e = Engine(0)
    yield e
    e.close()


def bit(k):
    return U64(1) << U64(k)


def make(kind, N, U, seed=0, base=0):
    """(row_ptr [N+1] with rows from `base`, run_carries, run_matches (rows below base are all ones and must not be
    read), node_match [N], sig_class, sig_carries, sig_matches [U], node_flags [N])"""
    rng = np.random.default_rng([seed, N, U, KINDS.index(kind)])
    lens = rng.integers(0, 8, size=N)
    if kind == "empty":
        lens[rng.random(N) < 0.5] = 0
    elif kind == "one_node":
        lens[:] = 0
        lens[N // 2] = 3 * N + 5
    elif kind in ("mixed_carries", "mixed_matches"):
        lens = np.where(np.arange(N) % 2 == 0, 0, np.maximum(lens, 1))  # empty nodes beside nodes with pods
    elif kind in ("last_admits", "none"):
        lens = np.maximum(lens, 1)
    row_ptr = (base + np.concatenate([[0], np.cumsum(lens)])).astype(np.int64)
    R = int(row_ptr[-1])
    rc = np.where(rng.random(R) < 0.4, U64(1) << rng.integers(0, 64, size=R).astype(U64), U64(0))
    rm = np.where(rng.random(R) < 0.6, U64(1) << rng.integers(0, 64, size=R).astype(U64), U64(0))
    rc[:base], rm[:base] = ~U64(0), ~U64(0)
    node_match = rng.integers(0, 1 << 63, size=N, dtype=U64) | U64(1)
    node_match[rng.random(N) < 0.5] |= bit(63)
    cls = rng.integers(0, 64, size=U).astype(np.uint8)
    car = np.where(rng.random(U) < 0.5, U64(1) << rng.integers(0, 64, size=U).astype(U64), U64(0))
    mat = np.where(rng.random(U) < 0.5, U64(1) << rng.integers(0, 64, size=U).astype(U64), U64(0))
    if kind in ("mixed_carries", "mixed_matches", "last_admits", "none"):
        cls[:] = 0
        car[:], mat[:] = 0, 0
        if kind == "mixed_carries":      # blocked through the pod's carries and the node's matches
            rm[base:] |= bit(0)
            car[:-1] = bit(0)
        elif kind == "mixed_matches":    # blocked through the pod's matches and the node's carries
            rc[base:] |= bit(1)
            mat[:-1] = bit(1)
        else:
            rm[base:] |= bit(0)
            rc[base:] |= bit(1)
            car[0::2], mat[1::2] = bit(0), bit(1)
            if kind == "last_admits":    # the only admitting signature is the last one (class 63)
                car[-1], mat[-1], cls[-1] = 0, 0, 63
    elif kind == "bit63":
        rc[base:][rng.random(R - base) < 0.5] |= bit(63)
        cls[:] = 63
        mat[:] = bit(63)
        car[:] = 0
    flags = (rng.random(N) < 0.3).astype(np.uint8) | np.uint8(4)
    return row_ptr, rc, rm, node_match, cls, car, mat, flags


def dev64(eng, a):
    return eng.dev(np.ascontiguousarray(a).view(np.int64), torch.int64)


def run_case(eng, c, with_match):
    row_ptr, rc, rm, node_match, cls, car, mat, flags = c
    nm = node_match if with_match else None
    d_flags = eng.dev(flags, torch.uint8)
    eng.pending_admit(eng.dev(row_ptr, torch.int64), dev64(eng, rc), dev64(eng, rm),
                      None if nm is None else dev64(eng, nm), cls, car, mat, d_flags)
    got = d_flags.cpu().numpy()
    want = aa_states_oracle.pending_admit(row_ptr, rc, rm, nm, cls, car, mat, flags)
    np.testing.assert_array_equal(got, want)
    check_record(eng.last_scan_launch(), len(flags), len(cls))
    return got


def check_record(rec, N, U):
    assert rec == {"kernel": 3, "form": 0, "D": 0, "bytes": TILE * 17, "warps": TILE // 32, "chunk": TILE,
                   "grid": (N + TILE - 1) // TILE, "S": U}, rec


@pytest.mark.parametrize("with_match", [False, True])
@pytest.mark.parametrize("U", [1, 255, 256, 257, 4000])
@pytest.mark.parametrize("N", [1, 31, 33, 2000])
@pytest.mark.parametrize("kind", KINDS)
def test_kernel_equals_oracle(eng, kind, N, U, with_match):
    base = 5 if (N + U) % 2 else 0  # row_ptr[0] > 0 in half of the cases
    got = run_case(eng, make(kind, N, U, base=base), with_match)
    flagged = (got & NO_MATCH) != 0
    if kind in ("mixed_carries", "mixed_matches") and N > 1:
        assert not flagged.any()  # the empty nodes are admitted by signature 0, the others only by the last one
    if kind == "none":
        assert flagged.all()
    if kind == "last_admits" and N > 30:  # node_match has bit 63 on about half of the nodes
        assert flagged.any() == with_match and not flagged.all()


@pytest.mark.parametrize("with_match", [False, True])
@pytest.mark.parametrize("kind,U", [("random", 1), ("random", 64), ("mixed_carries", 257), ("mixed_matches", 4000),
                                    ("last_admits", 257), ("empty", 64)])
def test_kernel_equals_oracle_at_a_million_nodes(eng, kind, U, with_match):
    run_case(eng, make(kind, 1_000_003, U, base=7), with_match)


def test_offset_views_are_read_correctly(eng):
    """views one element into larger tensors (8-byte but not 16-byte aligned) give the answer of fresh arrays"""
    row_ptr, rc, rm, node_match, cls, car, mat, flags = make("random", 777, 300, seed=3)
    N = len(flags)
    pad = lambda a: np.concatenate([a[:1], a])  # noqa: E731
    d_rp = eng.dev(pad(row_ptr), torch.int64)[1:]
    d_rc, d_rm, d_nm = dev64(eng, pad(rc))[1:], dev64(eng, pad(rm))[1:], dev64(eng, pad(node_match))[1:]
    d_flags = eng.dev(pad(flags), torch.uint8)[1:]
    assert d_rc.data_ptr() % 16 == 8 and d_flags.data_ptr() % 2 == 1
    eng.pending_admit(d_rp, d_rc, d_rm, d_nm, cls, car, mat, d_flags)
    np.testing.assert_array_equal(d_flags.cpu().numpy(),
                                  aa_states_oracle.pending_admit(row_ptr, rc, rm, node_match, cls, car, mat, flags))
    check_record(eng.last_scan_launch(), N, len(cls))


def _p(t, off=0):
    return None if t is None else ctypes.c_void_p(t.data_ptr() + off)


def test_refusals(eng):
    row_ptr, rc, rm, node_match, cls, car, mat, flags = make("random", 100, 10, seed=5)
    N = len(flags)
    d_rp, d_rc, d_rm, d_nm = eng.dev(row_ptr, torch.int64), dev64(eng, rc), dev64(eng, rm), dev64(eng, node_match)
    d_flags = eng.dev(flags, torch.uint8)

    def call(rp=d_rp, rcp=d_rc, rmp=d_rm, n=N, nm=d_nm, c=cls, a=car, m=mat, u=len(cls), fl=d_flags, offs=(0, 0, 0, 0)):
        ptr = lambda x: x.ctypes.data_as(ctypes.c_void_p) if isinstance(x, np.ndarray) else x  # noqa: E731
        return eng._lib.acsfit_pending_admit(
            eng._ctx, _p(rp, offs[0]) if isinstance(rp, torch.Tensor) else rp,
            _p(rcp, offs[1]) if isinstance(rcp, torch.Tensor) else rcp, _p(rmp) if isinstance(rmp, torch.Tensor) else rmp,
            n, _p(nm, offs[2]) if isinstance(nm, torch.Tensor) else nm, ptr(c), ptr(a), ptr(m), u,
            _p(fl, offs[3]) if isinstance(fl, torch.Tensor) else fl, eng._stream())
    bad_class = cls.copy()
    bad_class[3] = 64
    refused = {
        "class 64": call(c=bad_class),
        "U < 0": call(u=-1),
        "N < 0": call(n=-1),
        "NULL sig_class": call(c=None),
        "NULL sig_carries": call(a=None),
        "NULL sig_matches": call(m=None),
        "NULL run_carries": call(rcp=None),
        "NULL run_matches": call(rmp=None),
        "NULL row_ptr": call(rp=None),
        "NULL node_flags": call(fl=None),
        "misaligned row_ptr": call(offs=(4, 0, 0, 0)),
        "misaligned run_carries": call(offs=(0, 4, 0, 0)),
        "misaligned node_match": call(offs=(0, 0, 4, 0)),
        "decreasing row_ptr": call(rp=eng.dev(row_ptr[::-1].copy(), torch.int64)),
    }
    for what, status in refused.items():
        assert status == _native.E_INVALID, what
    np.testing.assert_array_equal(d_flags.cpu().numpy(), flags)  # nothing was launched
    # arrays that are not read may be NULL: no rows, or nothing to test
    empty_rp = eng.dev(np.full(N + 1, 9, np.int64), torch.int64)
    assert call(rp=empty_rp, rcp=None, rmp=None, nm=None) == _native.OK
    want = aa_states_oracle.pending_admit(np.full(N + 1, 9), rc, rm, None, cls, car, mat, flags)
    np.testing.assert_array_equal(d_flags.cpu().numpy(), want)
    check_record(eng.last_scan_launch(), N, len(cls))
    d_flags = eng.dev(flags, torch.uint8)
    assert call(c=None, a=None, m=None, u=0, fl=d_flags) == _native.OK  # U = 0: no node is admitted
    np.testing.assert_array_equal(d_flags.cpu().numpy(), flags | NO_MATCH)
    check_record(eng.last_scan_launch(), N, 0)
    assert call(n=0, rp=None, fl=None) == _native.OK
    assert eng.last_scan_launch()["kernel"] == 0


# ---------------------------------------------------------------- through Cluster.loop_logic
TICKS = gu.load_json("ticks.json.gz")


@pytest.fixture()
def host(tmp_path, monkeypatch, engine):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", engine)
    return monkeypatch


def tick(state, engine, on, every="1"):
    """one tick with pod anti-affinity on and $ACSFIT_ANTI_AFFINITY_NODE_STATES = on; `every` sets node selectors,
    selector node states, taints and node affinity"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_POD_ANTI_AFFINITY", "1")
        mp.setenv("ACSFIT_ANTI_AFFINITY_NODE_STATES", on)
        mp.setenv("ACSFIT_NODE_TAINTS", every)
        mp.setenv("ACSFIT_NODE_AFFINITY", every)
        return tick2(state, engine, every, every)


@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_every_switch_on_without_terms_is_the_reference_tick(host, engine, state):
    off = tick(state, engine, "0", every="0")
    on = tick(state, engine, "1")
    gu.assert_tick_matches(on, state["expected"])
    assert on["node_flags_sent"] == off["node_flags_sent"]


def replicas_state():
    """pool `agentpool1`: five old, schedulable Standard_D2_v2 nodes.  Replicas web-0 .. web-2 of a deployment that
    spreads one replica per node (required anti-affinity on app=web, hostname topology) run on nodes 0 .. 2, a db pod
    on node 3, nothing on node 4.  Replica web-3 is pending."""
    def node(i):
        name = "k8s-agentpool1-16334397-%d" % i
        return {"metadata": {"name": name, "creationTimestamp": "2016-08-25T05:13:16Z",
                             "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2", "agentpool": "agentpool1",
                                        "failure-domain.beta.kubernetes.io/region": "southcentralus",
                                        "kubernetes.io/hostname": name}}, "spec": {}}
    aff = {"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
        {"topologyKey": "kubernetes.io/hostname", "labelSelector": {"matchLabels": {"app": "web"}}}]}}
    created_by = '{"kind":"SerializedReference","reference":{"kind":"ReplicaSet","name":"r"}}'

    def pod(name, app, node_name=None):
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "100m"}}}]}
        if app == "web":
            spec["affinity"] = aff
        status = {"phase": "Pending"}
        if node_name:
            spec["nodeName"] = node_name
            status = {"phase": "Running", "startTime": "2026-09-20T07:00:00Z"}
        return {"metadata": {"name": name, "namespace": "default", "uid": "uid-" + name, "labels": {"app": app},
                             "annotations": {"kubernetes.io/created-by": created_by},
                             "creationTimestamp": "2026-09-20T07:00:00Z"}, "spec": spec, "status": status}
    nodes = [node(i) for i in range(5)]
    names = [n["metadata"]["name"] for n in nodes]
    pods = [pod("web-%d" % i, "web", names[i]) for i in range(3)] + [pod("db", "db", names[3]), pod("web-3", "web")]
    return {"name": "spread_replicas", "now": "2026-09-21T12:00:00Z", "nodes": nodes, "pods": pods,
            "arm_parameters": {"masterVMSize": {"value": "Standard_D2_v2"}, "firstConsecutiveStaticIP": {"value": "10.0.0.1"},
                               "agentpool1VMSize": {"value": "Standard_D2_v2"}},
            "settings": {"idle_threshold": 1800, "spare_agents": 0, "over_provision": 0, "dry_run": True,
                         "ignore_pools": ""}}


def restate_with_rule(state, to_schedule):
    """restate_maintain with the rule folded into its match: a pod to schedule matches a node only when no pod on the
    node avoids it and it avoids none of them (kube's predicates, pair by pair)"""
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod, KubePodStatus
    pods = [KubePod(gu.FakeKubeObject(o, [], "pod")) for o in state["pods"]]
    on_node = {}
    for p in pods:
        if p.status in (KubePodStatus.RUNNING, KubePodStatus.CONTAINER_CREATING) or \
                (p.status == KubePodStatus.PENDING and p.node_name):
            on_node.setdefault(p.node_name, []).append(p)

    def selects(owner, q):
        return any(q.namespace in ns and kube.selector_matches(sel, q.labels) for ns, sel in owner.anti_affinity_terms)
    orig = KubeNode.is_match
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(KubeNode, "is_match", lambda node, pod: orig(node, pod) and not any(
            selects(pod, q) or selects(q, pod) for q in on_node.get(node.name, [])))
        return restate_maintain(state, to_schedule)


def test_pending_replica_no_longer_holds_its_siblings_nodes(host, engine):
    s = replicas_state()
    names = [n["metadata"]["name"] for n in s["nodes"]]
    off = tick(s, engine, "0", every="0")
    on = tick(s, engine, "1", every="0")
    for got in (off, on):
        assert got["exception"] is None and "Pods to schedule: 1" in [m for _, _, m in got["log"]]
    assert off["state_calls"] == [[n, "pod-pending"] for n in names]
    assert not [m for _, _, m in off["log"] if DRY_MAINTAIN.match(m)]
    # on: the nodes that run a sibling follow the idle rules; the db node and the empty node still wait for web-3
    assert on["state_calls"] == [[n, "under-utilized-drainable"] for n in names[:3]] + \
        [[n, "pod-pending"] for n in names[3:]]
    assert [m for _, _, m in on["log"] if DRY_MAINTAIN.match(m)] == \
        ["[Dry run] Would have drained and cordoned %s" % n for n in names[:3]]
    # get_node_state node by node (the single-node path follows the rule), then maintain's one call for every node
    assert on["node_flags_sent"] == [[NO_MATCH]] * 3 + [[0]] * 2 + [[NO_MATCH] * 3 + [0, 0]]
    calls, journal, node_lines, dry_lines, deleted = restate_with_rule(s, {"web-3"})
    assert on["state_calls"] == calls
    assert on["maintain_journal"] == journal
    assert [m for _, _, m in on["log"] if m.startswith("node: ")] == node_lines
    assert [m for _, _, m in on["log"] if DRY_MAINTAIN.match(m)] == dry_lines
    assert on["deleted_nodes"] == deleted
    for key in ("exception", "scale_pools_calls", "used"):
        assert on[key] == off[key], key
