"""`-m gpu`: node states with hostname topology spread -- acsfit_pending_admit_ts and
Cluster(topology_spread_node_states=True).

* All four forms of the kernel (spread alone, with anti-affinity, with pod affinity, with both) equal the plain-C oracle
  (tests/ts_states_oracle.c, per pod, no deduplication, minimums recomputed) exactly on N in {1, 31, 33, 2000} and
  about 10^6, U in {1, 255, 256, 257, 4000}, keys in {0, 1, 64} with bit 63, with and without node_match, and
  row_ptr[0] > 0 in half of the cases; and on: counts exactly at the limit and one above, a node admitted only by the
  last signature of the last tile, floor INT32_MAX plus a positive skew (the clamp), and nodes the spread test admits
  but anti-affinity or affinity rejects.  Every call's launch record must show kernel 5, its form, shared bytes, grid
  and U.
* Views at an element offset are read correctly; every refusal leaves the flags untouched.
* The recorded reference ticks with every switch on and no constraint: the reference's tick, the same node flags sent
  to K6 and the same launch count.
* The motivating ticks (replicas stacked on some nodes), alone and with the other node-states switches, and the
  recorded ticks with spread constraints overlaid: the dry-run journal equals a plain-Python restatement of maintain
  with the rule.
The cases are chosen so that the module adds well under a minute to the suite."""
import ctypes

import numpy as np
import pytest
import torch

import golden_util as gu
import ts_states_oracle
from kubernetes_acs_engine_autoscaler_b200 import _native, kube
from test_gpu_aa_states import dev64
from test_gpu_pa_states import make_pa
from test_gpu_selector_states import DRY_MAINTAIN, restate_maintain
from test_gpu_selector_states import tick as tick2
from test_gpu_taints import _kube
from test_gpu_topology_spread_ticks import HOST, with_spread

pytestmark = pytest.mark.gpu

NO_MATCH = 2  # ACSFIT_NODEF_NO_PENDING_MATCH
TILE = 256    # signatures per shared-memory tile = threads per CTA (csrc/acsfit_admit.cuh)
U64 = np.uint64
INT32_MAX = 2 ** 31 - 1
FORMS = [(False, False), (True, False), (False, True), (True, True)]  # (anti-affinity, pod affinity)


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


def make_ts(kind, N, U, keys, seed=0, base=0):
    """make_pa()'s table (AA and PA arrays) plus sig_key, sig_skew, node_count [keys, N], node_domain, floor"""
    pa_kind = "aa_blocks" if kind == "others_reject" else "random"
    row_ptr, rc, rm, has, node_match, cls, car, mat, need, flags = make_pa(pa_kind, N, U, seed=seed, base=base)
    rng = np.random.default_rng([seed, N, U, keys, len(kind)])
    count = rng.integers(0, 5, size=(keys, N)).astype(np.int32)
    domain = rng.integers(0, 1 << 63, size=N, dtype=U64) | (U64(1) << U64(63))
    domain &= U64(0xFFFFFFFFFFFFFFFF) if keys == 64 else U64((1 << keys) - 1)
    floor = np.where(rng.random(keys) < 0.3, INT32_MAX, rng.integers(0, 4, size=keys)).astype(np.int32)
    key = np.where(rng.random(U) < 0.2, 0xFF, rng.integers(0, max(keys, 1), size=U)).astype(np.uint8)
    if keys == 0:
        key[:] = 0xFF
    skew = rng.integers(0, 3, size=U).astype(np.int32)
    if kind != "random":
        cls[:] = 0
        if kind != "others_reject":
            car[:], mat[:], need[:] = 0, 0, 0
    if kind == "at_limit":         # min 1, skew 1: count 2 is at the limit, 3 above it
        count[:] = rng.integers(1, 4, size=(keys, N))
        count[:, 0] = 1
        domain[:], floor[:] = U64((1 << keys) - 1) if keys < 64 else ~U64(0), INT32_MAX
        key[:], skew[:] = rng.integers(0, keys, size=U), 1
    elif kind == "last_sig":       # key 0 admits only empty nodes; the last signature (key 1) admits the rest it can
        count[0] = np.where(rng.random(N) < 0.5, 0, 3)
        count[1] = np.where(rng.random(N) < 0.5, 0, 3)
        domain[:], floor[:] = U64(3), 0
        key[:], skew[:] = 0, 0
        key[-1] = 1
    elif kind == "clamp":          # min INT32_MAX (no domain, floor INT32_MAX) and skew 5: the limit clamps
        count[:] = np.where(rng.random((keys, N)) < 0.5, INT32_MAX, 7)
        domain[:], floor[:] = 0, INT32_MAX
        key[:], skew[:] = 0, 5
    elif kind == "others_reject":  # the spread test admits every node
        floor[:], skew[:] = INT32_MAX, 0
        domain[:] = 0
    return row_ptr, rc, rm, has, node_match, cls, car, mat, need, key, skew, count, domain, floor, flags


def check_record(rec, N, U, aa, pa):
    assert rec == {"kernel": 5, "form": int(aa) | 2 * int(pa), "D": 0, "bytes": TILE * (16 * aa + 8 * pa + 6),
                   "warps": TILE // 32, "chunk": TILE, "grid": (N + TILE - 1) // TILE, "S": U}, rec


def run_case(eng, c, with_match, aa, pa, d_count=None, d_domain=None):
    row_ptr, rc, rm, has, node_match, cls, car, mat, need, key, skew, count, domain, floor, flags = c
    nm = node_match if with_match else None
    if not aa:
        rc = rm = car = mat = None
    if not pa:
        has = need = None
    d_flags = eng.dev(flags, torch.uint8)
    if d_count is None:
        d_count, d_domain = eng.dev(count, torch.int32), dev64(eng, domain)
    eng.pending_admit_ts(eng.dev(row_ptr, torch.int64), None if rc is None else dev64(eng, rc),
                         None if rm is None else dev64(eng, rm), None if has is None else dev64(eng, has),
                         None if nm is None else dev64(eng, nm), cls, car, mat, need, key, skew, len(floor), d_count,
                         d_domain, floor, d_flags)
    got = d_flags.cpu().numpy()
    want = ts_states_oracle.pending_admit_ts(row_ptr, rc, rm, has, nm, cls, car, mat, need, key, skew, count, domain,
                                             floor, flags)
    np.testing.assert_array_equal(got, want)
    check_record(eng.last_scan_launch(), len(flags), len(cls), aa, pa)
    return (got & NO_MATCH) != 0


@pytest.mark.parametrize("keys", [0, 1, 64])
@pytest.mark.parametrize("U", [1, 255, 256, 257, 4000])
@pytest.mark.parametrize("N", [1, 31, 33, 2000])
def test_kernel_equals_oracle(eng, N, U, keys):
    """the four forms, with and without node_match, on one random table (eight launches per case)"""
    base = 5 if (N + U + keys) % 2 else 0
    c = make_ts("random", N, U, keys, base=base)
    for aa, pa in FORMS:
        for with_match in (False, True):
            run_case(eng, c, with_match, aa, pa)


@pytest.mark.parametrize("kind,keys", [("at_limit", 1), ("at_limit", 64), ("last_sig", 2), ("clamp", 1),
                                       ("others_reject", 1)])
@pytest.mark.parametrize("N,U", [(33, 257), (2000, 4000)])
def test_kernel_edges_equal_oracle(eng, kind, keys, N, U):
    c = make_ts(kind, N, U, keys, base=3)
    with_pods = np.diff(c[0]) > 0
    for aa, pa in FORMS:
        for with_match in (False, True):
            flagged = run_case(eng, c, with_match, aa, pa)
            if kind == "at_limit" and not (aa or pa):
                count = c[11]
                assert (count == 2).any() and (count == 3).any()
                if keys == 1:  # exactly at the limit: admitted; one above: flagged
                    np.testing.assert_array_equal(flagged, count[0] > 2)
            if kind == "clamp":
                assert not flagged.any()
            if kind == "last_sig" and not with_match and not (aa or pa):
                np.testing.assert_array_equal(flagged, (c[11][0] > 0) & (c[11][1] > 0))
            if kind == "others_reject":  # anti-affinity rejects every node with pods, affinity every node without
                assert flagged[with_pods].all() == aa or not with_pods.any()
                assert flagged[~with_pods].all() == pa or with_pods.all()


@pytest.mark.parametrize("keys,U,form", [(64, 257, 0), (1, 64, 1), (64, 1, 2), (0, 257, 3)])
def test_kernel_equals_oracle_at_a_million_nodes(eng, keys, U, form):
    aa, pa = FORMS[form]
    run_case(eng, make_ts("random", 1_000_003, U, keys, base=7), True, aa, pa)


@pytest.mark.parametrize("form", range(4))
def test_offset_views_are_read_correctly(eng, form):
    """node_count one int32 and node_domain one element into larger tensors give the answer of fresh arrays"""
    aa, pa = FORMS[form]
    c = make_ts("random", 777, 300, 5, seed=3)
    count, domain = c[11], c[12]
    big = eng.dev(np.concatenate([np.zeros(1, np.int32), count.reshape(-1)]), torch.int32)
    d_count = big[1:]
    d_domain = dev64(eng, np.concatenate([domain[:1], domain]))[1:]
    assert d_count.data_ptr() % 8 == 4 and d_domain.data_ptr() % 16 == 8
    run_case(eng, c, True, aa, pa, d_count=d_count, d_domain=d_domain)


def _p(t, off=0):
    return None if t is None else ctypes.c_void_p(t.data_ptr() + off)


def test_refusals(eng):
    row_ptr, rc, rm, has, node_match, cls, car, mat, need, key, skew, count, domain, floor, flags = \
        make_ts("random", 100, 10, 3, seed=5)
    N = len(flags)
    d_rp, d_rc, d_rm, d_rh = eng.dev(row_ptr, torch.int64), dev64(eng, rc), dev64(eng, rm), dev64(eng, has)
    d_nm, d_count, d_domain = dev64(eng, node_match), eng.dev(count, torch.int32), dev64(eng, domain)
    d_flags = eng.dev(flags, torch.uint8)
    ptr = lambda x: x.ctypes.data_as(ctypes.c_void_p) if isinstance(x, np.ndarray) else x  # noqa: E731
    dptr = lambda x, off=0: _p(x, off) if isinstance(x, torch.Tensor) else x  # noqa: E731

    def call(rp=d_rp, rcp=d_rc, rmp=d_rm, rhp=d_rh, n=N, nm=d_nm, c=cls, a=car, m=mat, nd=need, k=key, s=skew,
             u=len(cls), ts="default", nc=d_count, dom=d_domain, fl_=floor, keys=len(floor), fl=d_flags,
             offs=(0, 0, 0, 0)):
        if ts == "default":
            ts = _native.TopologySpread(None, None, None, None if nc is None else nc.data_ptr() + offs[2],
                                        None if dom is None else dom.data_ptr() + offs[3],
                                        None if fl_ is None else fl_.ctypes.data, keys)
        return eng._lib.acsfit_pending_admit_ts(
            eng._ctx, dptr(rp, offs[0]), dptr(rcp, offs[1]), dptr(rmp), dptr(rhp), n, dptr(nm), ptr(c), ptr(a),
            ptr(m), ptr(nd), ptr(k), ptr(s), u, None if ts is None else ctypes.cast(ctypes.byref(ts), ctypes.c_void_p),
            dptr(fl), eng._stream())
    bad_key, bad_skew, bad_floor, neg = key.copy(), skew.copy(), floor.copy(), count.copy()
    bad_key[3], bad_skew[4], bad_floor[1], neg[2, 50] = 3, -1, -1, -1
    bad_class = cls.copy()
    bad_class[3] = 64
    refused = {
        "class 64": call(c=bad_class),
        "U < 0": call(u=-1),
        "N < 0": call(n=-1),
        "NULL sig_class": call(c=None),
        "NULL row_ptr": call(rp=None),
        "NULL node_flags": call(fl=None),
        "NULL run_carries only": call(rcp=None),
        "NULL sig_matches only": call(m=None),
        "NULL run_has only": call(rhp=None),
        "NULL sig_need only": call(nd=None),
        "misaligned row_ptr": call(offs=(4, 0, 0, 0)),
        "misaligned run_carries": call(offs=(0, 4, 0, 0)),
        "decreasing row_ptr": call(rp=eng.dev(row_ptr[::-1].copy(), torch.int64)),
        "NULL ts": call(ts=None),
        "keys -1": call(keys=-1),
        "keys 65": call(keys=65),
        "NULL node_count": call(nc=None),
        "NULL node_domain": call(dom=None),
        "NULL floor": call(fl_=None),
        "NULL sig_key": call(k=None),
        "NULL sig_skew": call(s=None),
        "key >= keys": call(k=bad_key),
        "key >= keys (0 keys)": call(keys=0),
        "negative skew": call(s=bad_skew),
        "negative floor": call(fl_=bad_floor),
        "negative count": call(nc=eng.dev(neg, torch.int32)),
        "misaligned node_count": call(offs=(0, 0, 2, 0)),
        "misaligned node_domain": call(offs=(0, 0, 0, 4)),
    }
    for what, status in refused.items():
        assert status == _native.E_INVALID, what
    np.testing.assert_array_equal(d_flags.cpu().numpy(), flags)  # nothing was launched
    # arrays that are not read may be NULL: no rows and no key
    empty_rp = eng.dev(np.full(N + 1, 9, np.int64), torch.int64)
    no_key = np.full(len(cls), 0xFF, np.uint8)
    assert call(rp=empty_rp, rcp=None, rmp=None, rhp=None, nm=None, a=None, m=None, nd=None, k=no_key, nc=None,
                dom=None, fl_=None, keys=0) == _native.OK
    want = ts_states_oracle.pending_admit_ts(np.full(N + 1, 9), None, None, None, None, cls, None, None, None, no_key,
                                             skew, np.zeros((0, N), np.int32), np.zeros(N, U64), np.zeros(0, np.int32),
                                             flags)
    np.testing.assert_array_equal(d_flags.cpu().numpy(), want)
    check_record(eng.last_scan_launch(), N, len(cls), False, False)
    d_flags = eng.dev(flags, torch.uint8)
    assert call(c=None, k=None, s=None, nd=None, u=0, fl=d_flags, rcp=None, rmp=None, rhp=None, a=None,
                m=None) == _native.OK  # U = 0
    np.testing.assert_array_equal(d_flags.cpu().numpy(), flags | NO_MATCH)
    check_record(eng.last_scan_launch(), N, 0, False, False)
    assert call(n=0, rp=None, fl=None, nc=None, dom=None) == _native.OK
    assert eng.last_scan_launch()["kernel"] == 0


# ---------------------------------------------------------------- through Cluster.loop_logic
TICKS = gu.load_json("ticks.json.gz")


@pytest.fixture()
def host(tmp_path, monkeypatch, engine):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", engine)
    return monkeypatch


def tick(state, engine, on, others="0"):
    """one tick with topology spread on and $ACSFIT_TOPOLOGY_SPREAD_NODE_STATES = on; `others` sets every other switch
    (node selectors, taints, node affinity, pod anti-affinity, pod affinity and their node states)"""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_TOPOLOGY_SPREAD", "1")
        mp.setenv("ACSFIT_TOPOLOGY_SPREAD_NODE_STATES", on)
        for name in ("POD_ANTI_AFFINITY", "ANTI_AFFINITY_NODE_STATES", "POD_AFFINITY", "POD_AFFINITY_NODE_STATES",
                     "NODE_TAINTS", "NODE_AFFINITY"):
            mp.setenv("ACSFIT_" + name, others)
        return tick2(state, engine, others, others)


# The admission test runs beside the scan, whose form the engine fixture varies; one form suffices for the ticks.
ONE_FORM = pytest.mark.parametrize("engine", ["ranks"], indirect=True)


@ONE_FORM
@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_every_switch_on_without_constraints_is_the_reference_tick(host, engine, state):
    off = tick(state, engine, "0")
    on = tick(state, engine, "1", others="1")
    gu.assert_tick_matches(on, state["expected"])
    assert on["node_flags_sent"] == off["node_flags_sent"]
    assert on["launches"] == off["launches"]


def cluster_state(name, pods):
    """pool `agentpool1`: five old, schedulable Standard_D2_v2 nodes; `pods`: (name, app, node index or None, maxSkew of
    a hostname constraint over app=web or None)"""
    def node(i):
        n = "k8s-agentpool1-16334397-%d" % i
        return {"metadata": {"name": n, "creationTimestamp": "2016-08-25T05:13:16Z",
                             "labels": {"beta.kubernetes.io/instance-type": "Standard_D2_v2", "agentpool": "agentpool1",
                                        "failure-domain.beta.kubernetes.io/region": "southcentralus",
                                        HOST: n}}, "spec": {}}
    created_by = '{"kind":"SerializedReference","reference":{"kind":"ReplicaSet","name":"r"}}'
    nodes = [node(i) for i in range(5)]
    names = [n["metadata"]["name"] for n in nodes]

    def pod(pname, app, at, skew):
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "100m"}}}]}
        if skew:
            spec["topologySpreadConstraints"] = [{"maxSkew": skew, "topologyKey": HOST,
                                                  "whenUnsatisfiable": "DoNotSchedule",
                                                  "labelSelector": {"matchLabels": {"app": "web"}}}]
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
    # web replicas run on nodes 0 and 1: the pending replica may land only where none runs
    "stacked": ([("web-0", "web", 0, 1), ("web-1", "web", 1, 1), ("db", "db", 2, None), ("web-2", "web", None, 1)],
                {"web-2"}, [2, 3, 4]),
    # one replica on each of nodes 0-3, two on node 4: with maxSkew 1 the minimum is 1, node 4 is above it
    "one_each": ([("web-%d" % i, "web", i, 1) for i in range(4)] + [("web-4", "web", 4, 1), ("web-5", "web", 4, 1),
                                                                   ("web-6", "web", None, 1)], {"web-6"}, [0, 1, 2, 3]),
    # a db pod spreads over the web pods: it does not select itself, so maxSkew 1 admits min + 1
    "not_self": ([("web-0", "web", 0, None), ("web-1", "web", 1, None), ("web-2", "web", 1, None),
                  ("web-3", "web", 1, None), ("db", "db", None, 1)], {"db"}, [0, 2, 3, 4]),
}


def restate_with_rule(state, to_schedule, per_node, selectors=True):
    """restate_maintain with the rule folded into its match (without `selectors` the match is the rule alone, as with
    node selectors off): a pod to schedule matches a node only when its
    DoNotSchedule hostname constraint allows it there -- the selected pods on the node, plus the pod when it selects
    itself, at most maxSkew above the smallest count over the constraint's domains (every listed node; per_node: the
    node alone), 0 with fewer domains than minDomains"""
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod, KubePodStatus
    pods = [KubePod(gu.FakeKubeObject(o, [], "pod")) for o in state["pods"]]
    listed = [KubeNode(gu.FakeKubeObject(o, [], "node")) for o in state["nodes"]]
    on_node = {}
    for p in pods:
        if p.status in (KubePodStatus.RUNNING, KubePodStatus.CONTAINER_CREATING) or \
                (p.status == KubePodStatus.PENDING and p.node_name):
            on_node.setdefault(p.node_name, []).append(p)

    def constraint(p):
        for e in p.original.obj["spec"].get("topologySpreadConstraints") or []:
            if e["topologyKey"] == HOST and e["whenUnsatisfiable"] == "DoNotSchedule":
                sel = e.get("labelSelector")
                selector = None
                if sel is not None:
                    selector = kube.label_selector(sel, "t")
                    extra = tuple((k, "In", (p.labels[k],)) for k in e.get("matchLabelKeys", ()) if k in p.labels)
                    selector = (selector[0], tuple(sorted(selector[1] + extra)))
                return (e["maxSkew"], selector, e.get("minDomains", 1),
                        e.get("nodeAffinityPolicy", "Honor") == "Honor", e.get("nodeTaintsPolicy", "Ignore") == "Honor")
        return None

    def selects(p, c, q):
        return c[1] is not None and q.namespace == p.namespace and kube.selector_matches(c[1], q.labels)

    def domain(p, c, n):
        if c[3] and not all(n.selectors.get(k) == v for k, v in p.selectors.items()):
            return False
        if c[3] and p.node_affinity is not None and not kube.node_affinity_matches(p.node_affinity, n.selectors, n.name):
            return False
        return not c[4] or kube.tolerates_all(p.tolerations, kube.blocking_taints(n.taints))

    def spread(node, p):
        c = constraint(p)
        if c is None:
            return True
        count = lambda n: sum(selects(p, c, q) for q in on_node.get(n.name, []))  # noqa: E731
        doms = [n for n in ([node] if per_node else listed) if domain(p, c, n)]
        low = 0 if len(doms) < c[2] else min(count(n) for n in doms)
        return count(node) + int(selects(p, c, p)) - low <= c[0]
    orig = KubeNode.is_match
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(KubeNode, "is_match", lambda node, pod: (not selectors or orig(node, pod)) and spread(node, pod))
        return restate_maintain(state, to_schedule)


def to_schedule_of(state):
    """names of the pending, unassigned pods some pool fits (no selector rule: only topology spread is on)"""
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.kube import KubePodStatus
    _, pods, pools = _kube(state)
    return {p.name for p in pods if p.status == KubePodStatus.PENDING and not p.node_name and
            any((capacity.RESOURCE_SPEC[pool.instance_type] - p.resources).possible for pool in pools)}


@ONE_FORM
@pytest.mark.parametrize("others", ["0", "1"])
@pytest.mark.parametrize("scenario", sorted(SCENARIOS))
def test_spread_no_longer_holds_every_node(host, engine, scenario, others):
    pods, to_schedule, pending_nodes = SCENARIOS[scenario]
    s = cluster_state(scenario, pods)
    off = tick(s, engine, "0", others=others)
    on = tick(s, engine, "1", others=others)
    for got in (off, on):
        assert got["exception"] is None
        assert "Pods to schedule: %d" % len(to_schedule) in [m for _, _, m in got["log"]]
    assert [st for _, st in off["state_calls"]] == ["pod-pending"] * 5
    maintain_states = [m.rsplit("state: ", 1)[1] for _, _, m in on["log"] if m.startswith("node: ")]
    assert [i for i, st in enumerate(maintain_states) if st == "pod-pending"] == pending_nodes
    assert on["node_flags_sent"][-1] == [0 if i in pending_nodes else NO_MATCH for i in range(5)]
    calls, journal, node_lines, dry_lines, deleted = restate_with_rule(s, to_schedule, per_node=False)
    assert on["maintain_journal"] == journal
    assert [m for _, _, m in on["log"] if m.startswith("node: ")] == node_lines
    assert [m for _, _, m in on["log"] if DRY_MAINTAIN.match(m)] == dry_lines
    assert on["deleted_nodes"] == deleted
    assert dry_lines  # some node the pending pod may not land on is now drained or cordoned
    # get_node_state sees one node: its own count is the minimum
    assert on["state_calls"] == restate_with_rule(s, to_schedule, per_node=True)[0]
    for key in ("exception", "scale_pools_calls", "used"):
        assert on[key] == off[key], key


SPREAD_TICKS = [st for st in TICKS if st["nodes"]]


@ONE_FORM
@pytest.mark.parametrize("variant", (0, 1, 2))
def test_ticks_with_spread_match_restatement(host, engine, variant):
    differs = 0
    for state in SPREAD_TICKS:
        s = with_spread(state, variant)
        got = tick(s, engine, "1")
        if got["maintain_journal"] is None:
            continue
        names = to_schedule_of(s)
        calls, journal, node_lines, dry_lines, deleted = restate_with_rule(s, names, False, selectors=False)
        assert got["maintain_journal"] == journal, s["name"]
        assert [m for _, _, m in got["log"] if m.startswith("node: ")] == node_lines, s["name"]
        assert [m for _, _, m in got["log"] if DRY_MAINTAIN.match(m)] == dry_lines, s["name"]
        assert got["deleted_nodes"] == deleted, s["name"]
        assert got["state_calls"] == restate_with_rule(s, names, True, selectors=False)[0], s["name"]
        off = tick(s, engine, "0")
        differs += off["node_flags_sent"] != got["node_flags_sent"]
    assert differs >= 1, differs  # the rule changes which nodes stay pod-pending in some tick
