"""`-m gpu`: node states with pod affinity -- acsfit_pending_admit_pa and Cluster(pod_affinity_node_states=True).

* Both forms of the kernel (affinity alone, and with anti-affinity) equal the plain-C oracle (tests/pa_states_oracle.c,
  per signature, no deduplication) exactly on N in {1, 31, 33, 2000}, U in {1, 255, 256, 257, 4000}, and about 10^6
  nodes with U up to 257, with
  and without node_match, row_ptr[0] > 0 in half of the cases, on: random masks, nodes without pods, one node holding
  every pod, need = 0 beside need != 0, a node admitted only by the last signature through its has mask, nodes that has
  admits but anti-affinity blocks, no signature admitting, and bit 63.  Every call's launch record must show kernel 4,
  its form, shared bytes, grid and U.
* Views at an element offset are read correctly; every refusal leaves the flags untouched.
* The recorded reference ticks with every switch on and no affinity term: the reference's tick, the same node flags
  sent to K6 and the same launch count.
* The motivating ticks: a web pod that requires a cache pod, and a self-affine group (bootstrap, then one replica
  running), alone and with the anti-affinity and selector states.  Idle nodes are no longer pod-pending, the node
  holding the cache (or the replica) still is, and the dry-run journal equals a plain-Python restatement of maintain
  with the rule.  The ticks run with one form of the candidate scan: the admission test does not depend on it.
The cases are chosen so that the module adds well under a minute to the suite."""
import ctypes

import numpy as np
import pytest
import torch

import golden_util as gu
import pa_states_oracle
from kubernetes_acs_engine_autoscaler_b200 import _native, kube
from test_gpu_aa_states import dev64, make
from test_gpu_selector_states import DRY_MAINTAIN, restate_maintain
from test_gpu_selector_states import tick as tick2

pytestmark = pytest.mark.gpu

NO_MATCH = 2  # ACSFIT_NODEF_NO_PENDING_MATCH
TILE = 256    # signatures per shared-memory tile = threads per CTA (csrc/acsfit_admit.cuh)
U64 = np.uint64
KINDS = ("random", "empty", "one_node", "need_mix", "last_has", "aa_blocks", "none", "bit63")
BASE_KIND = {"random": "random", "empty": "empty", "one_node": "one_node", "need_mix": "random",
             "last_has": "random", "aa_blocks": "random", "none": "random", "bit63": "random"}


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


def make_pa(kind, N, U, seed=0, base=0):
    """make()'s table plus run_has (rows below base all ones: never read) and sig_need"""
    row_ptr, rc, rm, node_match, cls, car, mat, flags = make(BASE_KIND[kind], N, U, seed=seed, base=base)
    rng = np.random.default_rng([seed, N, U, KINDS.index(kind), 1])
    R = len(rc)
    has = np.where(rng.random(R) < 0.5, U64(1) << rng.integers(0, 64, size=R).astype(U64), U64(0))
    need = np.where(rng.random(U) < 0.3, U64(0), U64(1) << rng.integers(0, 64, size=U).astype(U64))
    if kind == "need_mix":  # need = 0 on every other signature of a class many nodes lack
        need[::2] = 0
        cls[::2] = 63
    elif kind in ("last_has", "aa_blocks", "none", "bit63"):
        cls[:] = 0
        car[:], mat[:] = 0, 0
        lens = np.diff(row_ptr)
        hit = np.repeat(rng.random(N) < 0.5, lens)  # the rows of about half of the nodes
        if kind == "last_has":   # only the last signature's need (bit 2) is ever held
            need[:] = bit(1)
            need[-1] = bit(2)
            has[base:] &= ~(bit(1) | bit(2))
            has[base:][hit] |= bit(2)
        elif kind == "aa_blocks":  # has admits every node with pods, anti-affinity blocks every one of them
            need[:] = bit(3)
            has[base:] |= bit(3)
            rm[base:] |= bit(0)
            car[:] = bit(0)
        elif kind == "none":     # nobody holds bit 5
            need[:] = bit(5)
            has[base:] &= ~bit(5)
        else:
            need[:] = bit(63)
            has[base:] &= ~bit(63)
            has[base:][hit] |= bit(63)
    has[:base] = ~U64(0)
    return row_ptr, rc, rm, has, node_match, cls, car, mat, need, flags


def check_record(rec, N, U, aa):
    assert rec == {"kernel": 4, "form": 1 if aa else 0, "D": 0, "bytes": TILE * (25 if aa else 9),
                   "warps": TILE // 32, "chunk": TILE, "grid": (N + TILE - 1) // TILE, "S": U}, rec


def run_case(eng, c, with_match, aa):
    row_ptr, rc, rm, has, node_match, cls, car, mat, need, flags = c
    nm = node_match if with_match else None
    if not aa:
        rc = rm = car = mat = None
    d_flags = eng.dev(flags, torch.uint8)
    eng.pending_admit_pa(eng.dev(row_ptr, torch.int64), None if rc is None else dev64(eng, rc),
                         None if rm is None else dev64(eng, rm), dev64(eng, has),
                         None if nm is None else dev64(eng, nm), cls, car, mat, need, d_flags)
    got = d_flags.cpu().numpy()
    want = pa_states_oracle.pending_admit_pa(row_ptr, rc, rm, has, nm, cls, car, mat, need, flags)
    np.testing.assert_array_equal(got, want)
    check_record(eng.last_scan_launch(), len(flags), len(cls), aa)
    return got


@pytest.mark.parametrize("U", [1, 255, 256, 257, 4000])
@pytest.mark.parametrize("N", [1, 31, 33, 2000])
@pytest.mark.parametrize("kind", KINDS)
def test_kernel_equals_oracle(eng, kind, N, U):
    """both forms, with and without node_match, on one table (four launches per case)"""
    base = 5 if (N + U) % 2 else 0  # row_ptr[0] > 0 in half of the cases
    c = make_pa(kind, N, U, base=base)
    with_pods = np.diff(c[0]) > 0
    for aa in (False, True):
        for with_match in (False, True):
            flagged = (run_case(eng, c, with_match, aa) & NO_MATCH) != 0
            if kind == "none":
                assert flagged.all()
            if kind == "aa_blocks":
                assert flagged[~with_pods].all()   # nobody holds the need
                assert flagged[with_pods].all() == aa or not with_pods.any()
            if kind == "last_has" and N >= 31 and not with_match:
                assert flagged.any() and not flagged.all()


# each kind once, the form alternating; U stays small here because the C oracle walks every signature per node
@pytest.mark.parametrize("kind,U,aa", [("random", 1, False), ("need_mix", 64, True), ("last_has", 257, False),
                                       ("aa_blocks", 257, True), ("bit63", 64, False), ("empty", 64, True)])
def test_kernel_equals_oracle_at_a_million_nodes(eng, kind, U, aa):
    run_case(eng, make_pa(kind, 1_000_003, U, base=7), True, aa)


@pytest.mark.parametrize("aa", [False, True])
def test_offset_views_are_read_correctly(eng, aa):
    """views one element into larger tensors (8-byte but not 16-byte aligned) give the answer of fresh arrays"""
    row_ptr, rc, rm, has, node_match, cls, car, mat, need, flags = make_pa("random", 777, 300, seed=3)
    pad = lambda a: np.concatenate([a[:1], a])  # noqa: E731
    d_rp = eng.dev(pad(row_ptr), torch.int64)[1:]
    d_rc, d_rm, d_rh = dev64(eng, pad(rc))[1:], dev64(eng, pad(rm))[1:], dev64(eng, pad(has))[1:]
    d_nm = dev64(eng, pad(node_match))[1:]
    d_flags = eng.dev(pad(flags), torch.uint8)[1:]
    assert d_rh.data_ptr() % 16 == 8 and d_flags.data_ptr() % 2 == 1
    if not aa:
        rc = rm = car = mat = d_rc = d_rm = None
    eng.pending_admit_pa(d_rp, d_rc, d_rm, d_rh, d_nm, cls, car, mat, need, d_flags)
    np.testing.assert_array_equal(d_flags.cpu().numpy(), pa_states_oracle.pending_admit_pa(
        row_ptr, rc, rm, has, node_match, cls, car, mat, need, flags))
    check_record(eng.last_scan_launch(), len(flags), len(cls), aa)


def _p(t, off=0):
    return None if t is None else ctypes.c_void_p(t.data_ptr() + off)


def test_refusals(eng):
    row_ptr, rc, rm, has, node_match, cls, car, mat, need, flags = make_pa("random", 100, 10, seed=5)
    N = len(flags)
    d_rp, d_rc, d_rm, d_rh = eng.dev(row_ptr, torch.int64), dev64(eng, rc), dev64(eng, rm), dev64(eng, has)
    d_nm = dev64(eng, node_match)
    d_flags = eng.dev(flags, torch.uint8)
    ptr = lambda x: x.ctypes.data_as(ctypes.c_void_p) if isinstance(x, np.ndarray) else x  # noqa: E731
    dptr = lambda x, off=0: _p(x, off) if isinstance(x, torch.Tensor) else x  # noqa: E731

    def call(rp=d_rp, rcp=d_rc, rmp=d_rm, rhp=d_rh, n=N, nm=d_nm, c=cls, a=car, m=mat, nd=need, u=len(cls),
             fl=d_flags, offs=(0, 0, 0, 0, 0)):
        return eng._lib.acsfit_pending_admit_pa(
            eng._ctx, dptr(rp, offs[0]), dptr(rcp, offs[1]), dptr(rmp), dptr(rhp, offs[4]), n, dptr(nm, offs[2]),
            ptr(c), ptr(a), ptr(m), ptr(nd), u, dptr(fl, offs[3]), eng._stream())
    bad_class = cls.copy()
    bad_class[3] = 64
    refused = {
        "class 64": call(c=bad_class),
        "U < 0": call(u=-1),
        "N < 0": call(n=-1),
        "NULL sig_class": call(c=None),
        "NULL sig_need": call(nd=None),
        "NULL sig_need, no anti-affinity": call(nd=None, rcp=None, rmp=None, a=None, m=None),
        "NULL run_has": call(rhp=None),
        "NULL run_has, no anti-affinity": call(rhp=None, rcp=None, rmp=None, a=None, m=None),
        "NULL run_carries only": call(rcp=None),
        "NULL run_matches only": call(rmp=None),
        "NULL sig_carries only": call(a=None),
        "NULL sig_matches only": call(m=None),
        "only run_carries given": call(rmp=None, a=None, m=None),
        "NULL row_ptr": call(rp=None),
        "NULL node_flags": call(fl=None),
        "misaligned row_ptr": call(offs=(4, 0, 0, 0, 0)),
        "misaligned run_carries": call(offs=(0, 4, 0, 0, 0)),
        "misaligned node_match": call(offs=(0, 0, 4, 0, 0)),
        "misaligned run_has": call(offs=(0, 0, 0, 0, 4)),
        "misaligned run_has, no anti-affinity": call(offs=(0, 0, 0, 0, 4), rcp=None, rmp=None, a=None, m=None),
        "decreasing row_ptr": call(rp=eng.dev(row_ptr[::-1].copy(), torch.int64)),
    }
    for what, status in refused.items():
        assert status == _native.E_INVALID, what
    np.testing.assert_array_equal(d_flags.cpu().numpy(), flags)  # nothing was launched
    # arrays that are not read may be NULL: no rows, or nothing to test
    empty_rp = eng.dev(np.full(N + 1, 9, np.int64), torch.int64)
    assert call(rp=empty_rp, rcp=None, rmp=None, rhp=None, nm=None, a=None, m=None) == _native.OK
    want = pa_states_oracle.pending_admit_pa(np.full(N + 1, 9), None, None, has, None, cls, None, None, need, flags)
    np.testing.assert_array_equal(d_flags.cpu().numpy(), want)
    check_record(eng.last_scan_launch(), N, len(cls), False)
    # ... and with the anti-affinity test: no rows, the signature pair given
    d_flags = eng.dev(flags, torch.uint8)
    assert call(rp=empty_rp, rcp=None, rmp=None, rhp=None, nm=None, fl=d_flags) == _native.OK
    want = pa_states_oracle.pending_admit_pa(np.full(N + 1, 9), rc, rm, has, None, cls, car, mat, need, flags)
    np.testing.assert_array_equal(d_flags.cpu().numpy(), want)
    check_record(eng.last_scan_launch(), N, len(cls), True)
    d_flags = eng.dev(flags, torch.uint8)
    assert call(c=None, nd=None, u=0, fl=d_flags, rcp=None, rmp=None, a=None, m=None) == _native.OK  # U = 0
    np.testing.assert_array_equal(d_flags.cpu().numpy(), flags | NO_MATCH)
    check_record(eng.last_scan_launch(), N, 0, False)
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


def tick(state, engine, on, anti="0", selectors="0"):
    """one tick with pod affinity on and $ACSFIT_POD_AFFINITY_NODE_STATES = on; `anti` turns pod anti-affinity and its
    states on, `selectors` node selectors, their states, taints and node affinity"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_POD_AFFINITY", "1")
        mp.setenv("ACSFIT_POD_AFFINITY_NODE_STATES", on)
        mp.setenv("ACSFIT_POD_ANTI_AFFINITY", anti)
        mp.setenv("ACSFIT_ANTI_AFFINITY_NODE_STATES", anti)
        mp.setenv("ACSFIT_NODE_TAINTS", selectors)
        mp.setenv("ACSFIT_NODE_AFFINITY", selectors)
        return tick2(state, engine, selectors, selectors)


# The admission test runs beside the scan, whose form the engine fixture varies; one form suffices for the ticks.
ONE_FORM = pytest.mark.parametrize("engine", ["ranks"], indirect=True)


@ONE_FORM
@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_every_switch_on_without_terms_is_the_reference_tick(host, engine, state):
    off = tick(state, engine, "0")
    on = tick(state, engine, "1", anti="1", selectors="1")
    gu.assert_tick_matches(on, state["expected"])
    assert on["node_flags_sent"] == off["node_flags_sent"]
    assert on["launches"] == off["launches"]


def cluster_state(name, pods):
    """pool `agentpool1`: five old, schedulable Standard_D2_v2 nodes; `pods`: (name, app, node index or None,
    app its required pod affinity selects or None)"""
    def node(i):
        n = "k8s-agentpool1-16334397-%d" % i
        return {"metadata": {"name": n, "creationTimestamp": "2016-08-25T05:13:16Z",
                             "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2", "agentpool": "agentpool1",
                                        "failure-domain.beta.kubernetes.io/region": "southcentralus",
                                        "kubernetes.io/hostname": n}}, "spec": {}}
    created_by = '{"kind":"SerializedReference","reference":{"kind":"ReplicaSet","name":"r"}}'
    nodes = [node(i) for i in range(5)]
    names = [n["metadata"]["name"] for n in nodes]

    def pod(pname, app, at, needs):
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "100m"}}}]}
        if needs:
            spec["affinity"] = {"podAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
                {"topologyKey": "kubernetes.io/hostname", "labelSelector": {"matchLabels": {"app": needs}}}]}}
        status = {"phase": "Pending"}
        if at is not None:
            spec["nodeName"] = names[at]
            status = {"phase": "Running", "startTime": "2026-09-20T07:00:00Z"}
        return {"metadata": {"name": pname, "namespace": "default", "uid": "uid-" + pname, "labels": {"app": app},
                             "annotations": {"kubernetes.io/created-by": created_by},
                             "creationTimestamp": "2026-09-20T07:00:00Z"}, "spec": spec, "status": status}
    return {"name": name, "now": "2026-09-21T12:00:00Z", "nodes": nodes, "pods": [pod(*p) for p in pods],
            "arm_parameters": {"masterVMSize": {"value": "Standard_D2_v2"}, "firstConsecutiveStaticIP": {"value": "10.0.0.1"},
                               "agentpool1VMSize": {"value": "Standard_D2_v2"}},
            "settings": {"idle_threshold": 1800, "spare_agents": 0, "over_provision": 0, "dry_run": True,
                         "ignore_pools": ""}}


SCENARIOS = {
    # web needs a cache pod on its node: only node 2 holds one
    "web_cache": ([("cache", "cache", 2, None), ("db", "db", 0, None), ("web", "web", None, "cache")], {"web"}, [2]),
    # a self-affine group with no member running: its first pod may land anywhere
    "self_affine_bootstrap": ([("db", "db", 0, None), ("rep-0", "rep", None, "rep"), ("rep-1", "rep", None, "rep")],
                              {"rep-0", "rep-1"}, [0, 1, 2, 3, 4]),
    # one replica runs on node 3: its pending sibling may land only there
    "self_affine_running": ([("db", "db", 0, None), ("rep-0", "rep", 3, "rep"), ("rep-1", "rep", None, "rep")],
                            {"rep-1"}, [3]),
}


def restate_with_rule(state, to_schedule, per_node):
    """restate_maintain with the rule folded into its match: a pod to schedule matches a node only when it has no
    signature, or a pod on the node satisfies every term of it, or no pod in the cluster (per_node: on that node) does
    and it satisfies its terms itself -- kube's predicates, pair by pair"""
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod, KubePodStatus
    pods = [KubePod(gu.FakeKubeObject(o, [], "pod")) for o in state["pods"]]
    on_node = {}
    for p in pods:
        if p.status in (KubePodStatus.RUNNING, KubePodStatus.CONTAINER_CREATING) or \
                (p.status == KubePodStatus.PENDING and p.node_name):
            on_node.setdefault(p.node_name, []).append(p)
    everyone = [q for lst in on_node.values() for q in lst]

    def satisfies(terms, q):
        return all(sel is not None and q.namespace in ns and kube.selector_matches(sel, q.labels) for ns, sel in terms)

    def affine(node, pod):
        terms = pod.affinity_terms
        here = on_node.get(node.name, [])
        if not terms or any(satisfies(terms, q) for q in here):
            return True
        seen = here if per_node else everyone
        return not any(satisfies(terms, q) for q in seen) and satisfies(terms, pod)
    orig = KubeNode.is_match
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(KubeNode, "is_match", lambda node, pod: orig(node, pod) and affine(node, pod))
        return restate_maintain(state, to_schedule)


@ONE_FORM
@pytest.mark.parametrize("anti,selectors", [("0", "0"), ("1", "0"), ("0", "1"), ("1", "1")])
@pytest.mark.parametrize("scenario", sorted(SCENARIOS))
def test_pod_affinity_no_longer_holds_idle_nodes(host, engine, scenario, anti, selectors):
    pods, to_schedule, pending_nodes = SCENARIOS[scenario]
    s = cluster_state(scenario, pods)
    names = [n["metadata"]["name"] for n in s["nodes"]]
    off = tick(s, engine, "0", anti=anti, selectors=selectors)
    on = tick(s, engine, "1", anti=anti, selectors=selectors)
    for got in (off, on):
        assert got["exception"] is None
        assert "Pods to schedule: %d" % len(to_schedule) in [m for _, _, m in got["log"]]
    assert [st for _, st in off["state_calls"]] == ["pod-pending"] * 5
    # maintain: the nodes the pods to schedule may land on stay pod-pending, the others follow the idle rules
    maintain_states = [m.rsplit("state: ", 1)[1] for _, _, m in on["log"] if m.startswith("node: ")]
    assert [i for i, st in enumerate(maintain_states) if st == "pod-pending"] == pending_nodes
    assert on["node_flags_sent"][-1] == [0 if i in pending_nodes else NO_MATCH for i in range(5)]
    calls, journal, node_lines, dry_lines, deleted = restate_with_rule(s, to_schedule, per_node=False)
    assert on["maintain_journal"] == journal
    assert [m for _, _, m in on["log"] if m.startswith("node: ")] == node_lines
    assert [m for _, _, m in on["log"] if DRY_MAINTAIN.match(m)] == dry_lines
    assert on["deleted_nodes"] == deleted
    if len(pending_nodes) < 5:
        assert dry_lines  # some idle node is now drained or cordoned
    # get_node_state applies the rule to the pods it is given: a group may bootstrap on a node without a member
    per_node_calls = restate_with_rule(s, to_schedule, per_node=True)[0]
    assert on["state_calls"] == per_node_calls
    if scenario.startswith("self"):
        assert on["state_calls"] == [[n, "pod-pending"] for n in names]
    else:
        assert on["state_calls"] == calls
    for key in ("exception", "scale_pools_calls", "used"):
        assert on[key] == off[key], key
