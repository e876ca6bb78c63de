"""`-m "not gpu"`: the host side of Cluster(node_affinity=True) -- required node affinity with node selectors.

* kube.node_affinity_terms / kube.node_affinity_matches against a table of cases for every operator (absent, empty and
  non-integer labels, Go's ParseInt rule, the int64 bounds, ORed terms, the empty term, preferred-only affinity), and
  every malformed shape refused with a ValueError naming the pod.
* The pool rule: a new node's name and kubernetes.io/hostname are set, to a value no current node has.
* KubePod.node_affinity through both pod construction routes.
* snapshot.selector_classes(..., affinity=True) and snapshot.pending_match(..., affinity=True) bit for bit against a
  per-(pod, node) plain-Python restatement on generated clusters, with and without taints, with hostname NotIn terms
  (one projection per node), 64 signatures and a refused 65th; nodeSelector {k: v} and affinity `k In [v]` give the same
  arrays.
* The switch (environment, ValueError, pass-through, never read when off) and the warnings of get_pods_to_schedule with
  their precedence (the plain-C oracles stand in for the GPU)."""
import logging
from types import SimpleNamespace

import numpy as np
import pytest

import golden_util as gu
from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot
from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool
from test_taints_cpu import (NO_FIT, NO_POOL, TAINT_SETS, TOLERATION_SETS, UNTOLERATED, SelOracleEngine, T, Tol,
                             _cluster, node_obj, restated_blocking, restated_tolerates)

HOST, POOL, ITYPE = "kubernetes.io/hostname", "agentpool", "beta.kubernetes.io/instance-type"
AFFINITY = "Pending pod %s cannot fit: no agent pool that would fit it matches its required node affinity. " \
    "Scheduling skipped."
INT64_MAX, INT64_MIN = 2 ** 63 - 1, -2 ** 63


def R(key, op, *values):
    r = {"key": key, "operator": op}
    if values:
        r["values"] = list(values)
    return r


def F(op, value, key="metadata.name"):
    return {"key": key, "operator": op, "values": [value]}


def term(exprs=None, fields=None):
    t = {}
    if exprs is not None:
        t["matchExpressions"] = exprs
    if fields is not None:
        t["matchFields"] = fields
    return t


def aff(*terms, preferred=None):
    node = {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": list(terms)}}
    if preferred is not None:
        node["preferredDuringSchedulingIgnoredDuringExecution"] = preferred
    return {"nodeAffinity": node}


# ---------------------------------------------------------------- a plain restatement of the rule, on the raw spec
NEW = object()  # a new node's name / hostname: set, and equal to nothing


def r_int(s):
    """strconv.ParseInt(s, 10, 64)"""
    if not isinstance(s, str) or not s:
        return None
    body = s[1:] if s[0] in "+-" else s
    if not body or any(ch not in "0123456789" for ch in body):
        return None
    v = int(s)
    return v if INT64_MIN <= v <= INT64_MAX else None


def r_req(req, have):
    op, vals = req["operator"], req.get("values") or []
    if op == "In":
        return have is not None and have in vals
    if op == "NotIn":
        return have is None or have not in vals
    if op == "Exists":
        return have is not None
    if op == "DoesNotExist":
        return have is None
    a = r_int(have) if isinstance(have, str) else None
    return a is not None and (a > r_int(vals[0]) if op == "Gt" else a < r_int(vals[0]))


def r_affinity(raw, labels, name):
    node = (raw or {}).get("nodeAffinity") or {}
    required = node.get("requiredDuringSchedulingIgnoredDuringExecution")
    if required is None:
        return True
    for t in required["nodeSelectorTerms"]:
        ex, fl = t.get("matchExpressions") or [], t.get("matchFields") or []
        if (ex or fl) and all(r_req(e, labels.get(e["key"])) for e in ex) and all(r_req(f, name) for f in fl):
            return True
    return False


def r_pool_affinity(raw, labels):
    return r_affinity(raw, dict(labels, **{HOST: NEW}), NEW)


# ---------------------------------------------------------------- the matching rule
NUM = "num"
OPERATORS = [
    # (requirement, node labels, matches)
    (R(POOL, "In", "gpu"), {POOL: "gpu"}, True),
    (R(POOL, "In", "gpu", "gpu2"), {POOL: "gpu2"}, True),
    (R(POOL, "In", "gpu"), {POOL: "cpu"}, False),
    (R(POOL, "In", "gpu"), {}, False),                                  # absent
    (R(POOL, "In", ""), {POOL: ""}, True),                              # empty label value
    (R(POOL, "In", "gpu"), {POOL: ""}, False),
    (R(POOL, "NotIn", "gpu"), {POOL: "cpu"}, True),
    (R(POOL, "NotIn", "gpu"), {POOL: "gpu"}, False),
    (R(POOL, "NotIn", "gpu"), {}, True),                                # NotIn holds when the key is absent
    (R(POOL, "NotIn", "gpu"), {POOL: ""}, True),
    (R(POOL, "Exists"), {POOL: ""}, True),
    (R(POOL, "Exists"), {}, False),
    (R(POOL, "DoesNotExist"), {}, True),
    (R(POOL, "DoesNotExist"), {POOL: "x"}, False),
    (R(NUM, "Gt", "3"), {NUM: "4"}, True),
    (R(NUM, "Gt", "3"), {NUM: "3"}, False),
    (R(NUM, "Lt", "3"), {NUM: "2"}, True),
    (R(NUM, "Lt", "3"), {NUM: "3"}, False),
    (R(NUM, "Gt", "3"), {}, False),                                     # absent label: false
    (R(NUM, "Lt", "3"), {}, False),
    (R(NUM, "Gt", "-1"), {NUM: ""}, False),                             # empty label: not an integer
    (R(NUM, "Lt", "9"), {NUM: "x"}, False),
    (R(NUM, "Gt", "4"), {NUM: "+5"}, True),                             # Go's ParseInt: a sign, then digits
    (R(NUM, "Lt", "-2"), {NUM: "-3"}, True),
    (R(NUM, "Gt", "6"), {NUM: "007"}, True),
    (R(NUM, "Lt", "8"), {NUM: "007"}, True),
    (R(NUM, "Gt", "0"), {NUM: "1_0"}, False),                           # no underscores ...
    (R(NUM, "Lt", "99"), {NUM: "1_0"}, False),
    (R(NUM, "Gt", "0"), {NUM: " 5"}, False),                            # ... no spaces
    (R(NUM, "Lt", "99"), {NUM: "5 "}, False),
    (R(NUM, "Lt", "99"), {NUM: "5\n"}, False),
    (R(NUM, "Gt", "0"), {NUM: "+"}, False),
    (R(NUM, "Gt", "-9"), {NUM: "-0"}, True),
    (R(NUM, "Gt", "0"), {NUM: "٥"}, False),                        # a non-ASCII digit
    (R(NUM, "Gt", "0"), {NUM: "5.0"}, False),
    (R(NUM, "Gt", "9223372036854775806"), {NUM: "9223372036854775807"}, True),    # the int64 bounds ...
    (R(NUM, "Gt", "0"), {NUM: "9223372036854775808"}, False),                     # ... and one past each
    (R(NUM, "Lt", "-9223372036854775807"), {NUM: "-9223372036854775808"}, True),
    (R(NUM, "Lt", "0"), {NUM: "-9223372036854775809"}, False),
    (R(NUM, "Lt", "9223372036854775807"), {NUM: "5"}, True),
    (R(NUM, "Gt", "-9223372036854775808"), {NUM: "5"}, True),
    (R(NUM, "Gt", "+3"), {NUM: "4"}, True),
    (R(NUM, "Lt", "007"), {NUM: "6"}, True),
]


@pytest.mark.parametrize("case", range(len(OPERATORS)))
def test_operator_table(case):
    req, labels, want = OPERATORS[case]
    terms = kube.node_affinity_terms(aff(term([req])), "pod p")
    assert kube.node_affinity_matches(terms, labels, "n0") is want
    assert r_affinity(aff(term([req])), labels, "n0") is want
    # the vectorised matcher on one node
    node = SimpleNamespace(selectors=labels, name="n0")
    pod = SimpleNamespace(selectors={}, node_affinity=terms)
    assert snapshot.pending_match([pod], [node], affinity=True).tolist() == [want]


@pytest.mark.parametrize("text,want", [("0", 0), ("-0", 0), ("+5", 5), ("-3", -3), ("007", 7), ("1_0", None),
                                       (" 5", None), ("5 ", None), ("", None), ("+", None), ("-", None), ("+-1", None),
                                       ("0x10", None), ("1e3", None), (str(INT64_MAX), INT64_MAX),
                                       (str(INT64_MAX + 1), None), (str(INT64_MIN), INT64_MIN),
                                       (str(INT64_MIN - 1), None), (None, None), (5, None)])
def test_parse_int64(text, want):
    assert kube.parse_int64(text) == want


def test_terms_fields_and_canonical_form():
    labels = {POOL: "gpu", HOST: "n1", "zone": "z1"}
    m = lambda a, name="n1": kube.node_affinity_matches(kube.node_affinity_terms(a, "pod p"), labels, name)  # noqa: E731
    assert m(aff(term([R(POOL, "In", "cpu")]), term([R("zone", "In", "z1")])))          # ORed terms
    assert not m(aff(term([R(POOL, "In", "cpu")]), term([R("zone", "In", "z2")])))
    assert not m(aff(term([R(POOL, "In", "gpu"), R("zone", "In", "z2")])))              # ANDed requirements
    assert not m(aff(term()))                                                            # the empty term: nothing
    assert not m(aff(term([], [])))
    assert m(aff(term(), term([R(POOL, "Exists")])))
    assert m(aff(term(fields=[F("In", "n1")])))
    assert not m(aff(term(fields=[F("In", "n1")])), "n2")
    assert m(aff(term(fields=[F("NotIn", "n2")])))
    assert not m(aff(term([R(POOL, "In", "gpu")], [F("In", "n2")])))                   # expressions AND fields
    assert m(aff(term([R(POOL, "In", "gpu")], [F("In", "n1")])))
    # no constraint: None; preferred-only is ignored; a term list that can match nothing: ()
    assert kube.node_affinity_terms(None, "p") is None
    assert kube.node_affinity_terms({}, "p") is None
    assert kube.node_affinity_terms({"nodeAffinity": None}, "p") is None
    assert kube.node_affinity_terms({"nodeAffinity": {}}, "p") is None
    assert kube.node_affinity_terms({"podAntiAffinity": {}}, "p") is None
    pref = [{"weight": 1, "preference": {"matchExpressions": [R(POOL, "In", "cpu")]}}]
    assert kube.node_affinity_terms({"nodeAffinity": {"preferredDuringSchedulingIgnoredDuringExecution": pref}}, "p") \
        is None
    assert kube.node_affinity_terms({"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": None}}, "p") \
        is None
    assert kube.node_affinity_terms(aff(term()), "p") == ()
    assert kube.node_affinity_terms(aff(term([R(POOL, "In", "a")]), preferred=pref), "p") == \
        kube.node_affinity_terms(aff(term([R(POOL, "In", "a")])), "p")
    # equal forms: order and duplicates of terms, requirements and values do not matter
    a = aff(term([R(POOL, "In", "b", "a", "a"), R("zone", "Exists")]), term([R(NUM, "Gt", "+3")]), term())
    b = aff(term([R(NUM, "Gt", "3")]), term([R("zone", "Exists"), R(POOL, "In", "a", "b")]),
            term([R(POOL, "In", "a", "b"), R("zone", "Exists")]))
    assert kube.node_affinity_terms(a, "p") == kube.node_affinity_terms(b, "p")
    hash(kube.node_affinity_terms(a, "p"))


def test_pool_rule_for_hostname_and_node_name():
    """a new node's hostname label and name are set, to a value no current node has"""
    labels = {POOL: "gpu", ITYPE: "t"}
    cases = [(R(HOST, "Exists"), True), (R(HOST, "DoesNotExist"), False), (R(HOST, "In", "n1"), False),
             (R(HOST, "NotIn", "n1"), True), (R(HOST, "Gt", "0"), False), (R(HOST, "Lt", "0"), False),
             (F("In", "n1"), False), (F("NotIn", "n1"), True)]
    for req, want in cases:
        a = aff(term(fields=[req])) if req["key"] == "metadata.name" else aff(term([req]))
        terms = kube.node_affinity_terms(a, "p")
        assert kube.pool_affinity_matches(terms, labels) is want, req
        assert r_pool_affinity(a, labels) is want, req
    # a numeric hostname on every node does not leak into the pool
    node = SimpleNamespace(selectors={POOL: "gpu", HOST: "7", ITYPE: "t"}, taints=[], name="7", unschedulable=False)
    pool = AgentPool("gpu", "t", [node])
    pods = [SimpleNamespace(selectors={}, node_affinity=kube.node_affinity_terms(aff(term([R(HOST, "Gt", "5")])), "p"))]
    cls = snapshot.selector_classes(pods, [node], [pool], affinity=True)
    assert cls.node_match.tolist() == [3] and cls.pool_match.tolist() == [1]
    # nodeSelector hostname: x still matches no pool
    assert snapshot.selector_classes([SimpleNamespace(selectors={HOST: "7"})], [node], [pool]).pool_match.tolist() == [1]


# ---------------------------------------------------------------- malformed input
BAD = [
    {"nodeAffinity": "x"},
    {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": "x"}},
    {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {}}},                   # no nodeSelectorTerms
    {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": None}}},
    aff(),                                                                                         # empty
    {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": {"a": 1}}}},
    aff("x"),                                                                                      # not mappings
    aff(None),
    aff(term("x")),
    aff(term(["x"])),
    aff(term(fields=[None])),
    aff(term([R(POOL, "in", "a")])),                                                               # unknown operator
    aff(term([R(POOL, "Matches", "a")])),
    aff(term([{"key": POOL, "values": ["a"]}])),
    aff(term([R(POOL, "In")])),                                                                    # value counts
    aff(term([R(POOL, "NotIn")])),
    aff(term([R(POOL, "Exists", "a")])),
    aff(term([R(POOL, "DoesNotExist", "a")])),
    aff(term([R(NUM, "Gt")])),
    aff(term([R(NUM, "Lt", "1", "2")])),
    aff(term([R(NUM, "Gt", "x")])),                                                                # not integers
    aff(term([R(NUM, "Gt", "1_0")])),
    aff(term([R(NUM, "Lt", " 5")])),
    aff(term([R(NUM, "Gt", "9223372036854775808")])),
    aff(term([R(NUM, "Gt", 5)])),
    aff(term([R(POOL, "In", 5)])),
    aff(term([{"key": POOL, "operator": "In", "values": "a"}])),
    aff(term([{"key": 5, "operator": "Exists"}])),
    aff(term(fields=[F("In", "n1", key="metadata.namespace")])),                                   # matchFields
    aff(term(fields=[F("In", "n1", key="spec.nodeName")])),
    aff(term(fields=[R("metadata.name", "Exists")])),
    aff(term(fields=[F("Gt", "1")])),
    aff(term(fields=[R("metadata.name", "In", "a", "b")])),
    aff(term(fields=[R("metadata.name", "In")])),
]


def pod_obj(name, affinity=None, selector=None, cpu="1", tolerations=None, phase="Pending"):
    spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": cpu}}}]}
    if affinity is not None:
        spec["affinity"] = affinity
    if selector:
        spec["nodeSelector"] = selector
    if tolerations is not None:
        spec["tolerations"] = tolerations
    return {"metadata": {"name": name, "namespace": "ns", "uid": "u-" + name, "creationTimestamp": "2026-09-21T07:00:00Z"},
            "spec": spec, "status": {"phase": phase}}


@pytest.mark.parametrize("case", range(len(BAD)))
def test_malformed_affinity_raises_naming_the_pod(case):
    j = []
    p = kube.KubePod(gu.FakeKubeObject(pod_obj("broken-%d" % case, BAD[case]), j, "pod"))
    with pytest.raises(ValueError, match="broken-%d" % case):
        p.node_affinity
    with pytest.raises(ValueError, match="broken-%d" % case):
        kube.node_affinity_terms(BAD[case], "pod broken-%d" % case)
    with pytest.raises(ValueError, match="broken-%d" % case):
        snapshot.selector_classes([p], [], [], affinity=True)
    with pytest.raises(ValueError, match="broken-%d" % case):
        snapshot.pending_match([p], [SimpleNamespace(selectors={}, name="n")], affinity=True)


def test_switch_off_never_reads_the_affinity(tmp_path, monkeypatch, oracle_mod):
    """without `affinity`, the builders read no node_affinity (a malformed one raises nothing), and a tick with the
    switch off is the tick of the other switches"""
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", SelOracleEngine())
    j = []
    n = kube.KubeNode(gu.FakeKubeObject(node_obj("k8s-cpu-1-0", {POOL: "cpu", ITYPE: "Standard_D2_v2"}), j, "node"))
    pools = [AgentPool("cpu", "Standard_D2_v2", [n])]
    pods = [kube.KubePod(gu.FakeKubeObject(pod_obj("broken-%d" % i, b), j, "pod")) for i, b in enumerate(BAD)]
    pods.append(kube.KubePod(gu.FakeKubeObject(pod_obj("pinned", selector={POOL: "cpu"}), j, "pod")))
    for taints in (False, True):
        cls = snapshot.selector_classes(pods, [n], pools, taints=taints)
        assert cls.pod_class.tolist() == [0] * len(BAD) + [0]
        assert snapshot.pending_match(pods, [n], taints=taints).tolist() == [True]
        cl = _cluster(node_selectors=True, node_taints=taints, node_affinity=False)
        assert len(cl.get_pods_to_schedule(pods, pools)) == len(pods)


# ---------------------------------------------------------------- kube types
def test_node_affinity_through_both_routes(monkeypatch):
    j = []
    a = aff(term([R(POOL, "In", "gpu")]), term(fields=[F("In", "n1")]))
    raw = [gu.FakeKubeObject(o, j, "pod") for o in (pod_obj("a", a), pod_obj("b"), pod_obj("c", {}),
                                                    pod_obj("d", aff(term())))]
    want = [kube.node_affinity_terms(a, "p"), None, None, ()]
    assert want[0] == (((), (("metadata.name", "In", ("n1",)),)), (((POOL, "In", ("gpu",)),), ()))
    routes = [kube.make_pods(raw), [kube.KubePod(o) for o in raw]]
    if kube._hostfast is not None:  # the C route builds plain pods attribute by attribute: the property still reads them
        monkeypatch.setattr(kube, "_hostfast", None)
        routes.append(kube.make_pods(raw))
    for pods in routes:
        assert [p.node_affinity for p in pods] == want


# ---------------------------------------------------------------- the class builder against a per-pair restatement
POOLS = ("cpu", "gpu", "mem", "spot")
NUMS = ["0", "1", "5", "007", "+4", "-3", "x", "1_0", " 5", "", None]


def affinity_kinds(N):
    """raw affinities (None: no field): pool targeting, NotIn, Exists / DoesNotExist, Gt / Lt on a numeric label,
    ORed terms, matchFields pins (DaemonSet-style), hostname NotIn, the empty term, preferred-only"""
    host = lambda i: "node-%d" % (i % max(N, 1))  # noqa: E731
    return [
        lambda i: None, lambda i: None, lambda i: {},
        lambda i: aff(term([R(POOL, "In", POOLS[i % 4])])),
        lambda i: aff(term([R(POOL, "In", "gpu", "mem")])),
        lambda i: aff(term([R(POOL, "NotIn", "cpu", "gpu")])),
        lambda i: aff(term([R("zone", "Exists")])),
        lambda i: aff(term([R("zone", "DoesNotExist")])),
        lambda i: aff(term([R(NUM, "Gt", "3")])),
        lambda i: aff(term([R(NUM, "Lt", str(i % 3 - 1))])),
        lambda i: aff(term([R(POOL, "In", "cpu")]), term([R(NUM, "Gt", "0"), R("zone", "In", "1")])),
        lambda i: aff(term(fields=[F("In", host(i))])),
        lambda i: aff(term(fields=[F("NotIn", host(i))])),
        lambda i: aff(term([R(HOST, "NotIn", host(i))])),
        lambda i: aff(term([R(HOST, "Exists"), R(POOL, "In", "spot")])),
        lambda i: aff(term()),
        lambda i: aff(term(), term([R(POOL, "NotIn", "mem")])),
        lambda i: aff(term([R(POOL, "In", "cpu")], [F("NotIn", host(i))])),
        lambda i: {"nodeAffinity": {"preferredDuringSchedulingIgnoredDuringExecution": [
            {"weight": 1, "preference": {"matchExpressions": [R(POOL, "In", "gpu")]}}]}},
    ]


def gen_cluster(rng, N, n_sig, P, taint_prob=0.3, kinds=None):
    """nodes of four pools (some without a hostname label, a numeric label `num` of any shape), pods mixing
    selectors, toleration sets and node affinities"""
    nodes = []
    for i in range(N):
        pool = POOLS[rng.integers(len(POOLS))]
        labels = {POOL: pool, ITYPE: "type-%s" % pool}
        if rng.random() < 0.9:
            labels[HOST] = "node-%d" % i
        if rng.random() < 0.4:
            labels["zone"] = str(rng.integers(3))
        num = NUMS[rng.integers(len(NUMS))]
        if num is not None:
            labels[NUM] = num
        taints = list(TAINT_SETS[rng.integers(len(TAINT_SETS))]) if rng.random() < taint_prob else []
        nodes.append(SimpleNamespace(selectors=labels, taints=taints, unschedulable=False, name="node-%d" % i))
    pools = [AgentPool(p, "type-" + p, [n for n in nodes if n.selectors[POOL] == p]) for p in POOLS]
    kinds = kinds or affinity_kinds(N)
    sel_kinds = [lambda: {}, lambda: {}, lambda: {}, lambda: {POOL: POOLS[rng.integers(len(POOLS))]},
                 lambda: {"zone": str(rng.integers(3))}]
    sigs = [(sel_kinds[rng.integers(len(sel_kinds))](), kinds[rng.integers(len(kinds))](int(rng.integers(1 << 20))),
             list(TOLERATION_SETS[rng.integers(len(TOLERATION_SETS))])) for _ in range(n_sig)]
    pods = []
    for _ in range(P):
        sel, raw, tol = sigs[rng.integers(n_sig)]
        pods.append(SimpleNamespace(selectors=dict(sel), tolerations=list(tol), raw_affinity=raw,
                                    node_affinity=kube.node_affinity_terms(raw, "pod")))
    return pods, nodes, pools


def restated_ok(pod, labels, name, taints, use_taints, use_affinity, pool=False):
    if not all(labels.get(k) == v for k, v in pod.selectors.items()):
        return False
    if use_taints and not all(restated_tolerates(pod.tolerations, t) for t in taints):
        return False
    if not use_affinity:
        return True
    return r_pool_affinity(pod.raw_affinity, labels) if pool else r_affinity(pod.raw_affinity, labels, name)


def restate_classes(pods, nodes, pools, use_taints, use_affinity):
    node_taints = [restated_blocking(n.taints) if use_taints else set() for n in nodes]
    pool_taints = []
    for p in pools:
        sets = [restated_blocking(n.taints) for n in p.nodes] if use_taints else []
        pool_taints.append(set.intersection(*sets) if sets else set())
    sigs = [(tuple([True] * len(nodes)), tuple([True] * len(pools)))]
    pod_class = []
    for pod in pods:
        sig = (tuple(restated_ok(pod, n.selectors, n.name, t, use_taints, use_affinity) for n, t in zip(nodes, node_taints)),
               tuple(restated_ok(pod, p.labels, None, t, use_taints, use_affinity, pool=True)
                     for p, t in zip(pools, pool_taints)))
        if sig not in sigs:
            sigs.append(sig)
        pod_class.append(sigs.index(sig))
    if len(sigs) > 64:
        return None
    node_match = [sum(1 << c for c, s in enumerate(sigs) if s[0][i]) for i in range(len(nodes))]
    pool_match = [sum(1 << c for c, s in enumerate(sigs) if s[1][i]) for i in range(len(pools))]
    return pod_class, node_match, pool_match, len(sigs)


def restate_pending(pods, nodes, use_taints, use_affinity):
    return [any(restated_ok(p, n.selectors, n.name, restated_blocking(n.taints), use_taints, use_affinity) for p in pods)
            for n in nodes]


def check_classes(pods, nodes, pools, use_taints, use_affinity=True):
    want = restate_classes(pods, nodes, pools, use_taints, use_affinity)
    if want is None:
        with pytest.raises(ValueError, match="64"):
            snapshot.selector_classes(pods, nodes, pools, taints=use_taints, affinity=use_affinity)
        return None
    got = snapshot.selector_classes(pods, nodes, pools, taints=use_taints, affinity=use_affinity)
    assert got.pod_class.dtype == np.uint8 and got.node_match.dtype == np.uint64 and got.pool_match.dtype == np.uint64
    assert got.pod_class.tolist() == want[0]
    assert got.node_match.tolist() == want[1]
    assert got.pool_match.tolist() == want[2]
    assert got.classes == want[3]
    return got


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("shape", [(1, 1, 1), (40, 3, 30), (150, 8, 100), (250, 14, 200)])
def test_classes_and_pending_match_equal_per_pair_restatement(seed, shape):
    N, n_sig, P = shape
    rng = np.random.default_rng([seed, N, 11])
    pods, nodes, pools = gen_cluster(rng, N, n_sig, P)
    for use_taints in (False, True):
        check_classes(pods, nodes, pools, use_taints)
        check_classes(pods, [], pools, use_taints)
        check_classes(pods, nodes, [], use_taints)
        for sub in (pods, pods[:3], pods[::7], []):
            assert snapshot.pending_match(sub, nodes, taints=use_taints, affinity=True).tolist() == \
                restate_pending(sub, nodes, use_taints, True)
    # affinity=False reads no affinity: the answer of the other switches
    check_classes(pods, nodes, pools, True, use_affinity=False)


@pytest.mark.parametrize("seed", range(3))
def test_hostname_not_in_gives_one_projection_per_node(seed):
    """every pod avoids one node by hostname (or by name): each node is its own projection"""
    rng = np.random.default_rng([seed, 3])
    N = 300
    kinds = [lambda i: aff(term([R(HOST, "NotIn", "node-%d" % (i % N))])),
             lambda i: aff(term([R(POOL, "In", "cpu", "mem"), R(HOST, "NotIn", "node-%d" % (i % N))])),
             lambda i: aff(term(fields=[F("NotIn", "node-%d" % (i % N))]))]
    pods, nodes, pools = gen_cluster(rng, N, 20, 200, kinds=kinds)
    for use_taints in (False, True):
        check_classes(pods, nodes, pools, use_taints)
        assert snapshot.pending_match(pods, nodes, taints=use_taints, affinity=True).tolist() == \
            restate_pending(pods, nodes, use_taints, True)
    proj = snapshot._projection(nodes, snapshot._match_keys(pods, False, True)[0], False)
    assert len(proj.proj) == N


@pytest.mark.parametrize("pins", [63, 64])
def test_64_signatures_and_the_65th(pins):
    """each `hostname NotIn [c_i]` pod is one signature; with the pods without affinity (class 0), 1 + 63 = 64 classes
    are accepted and one more is refused"""
    nodes = [SimpleNamespace(selectors={POOL: "cpu", HOST: "c%d" % i}, taints=[], name="c%d" % i, unschedulable=False) for i in range(70)]
    pools = [AgentPool("cpu", "t", nodes)]
    pods = [SimpleNamespace(selectors={}, tolerations=[], node_affinity=None, raw_affinity=None)]
    for i in range(pins):
        raw = aff(term([R(HOST, "NotIn", "c%d" % i)]))
        pods.append(SimpleNamespace(selectors={}, tolerations=[], raw_affinity=raw,
                                    node_affinity=kube.node_affinity_terms(raw, "p")))
    if pins == 63:
        got = check_classes(pods, nodes, pools, False)
        assert got.classes == 64 and got.pod_class[0] == 0 and got.pod_class[1:].all()
    else:
        with pytest.raises(ValueError, match="64"):
            snapshot.selector_classes(pods, nodes, pools, affinity=True)
    assert snapshot.selector_classes(pods, nodes, pools).trivial     # without the switch: no signature at all


@pytest.mark.parametrize("seed", range(4))
def test_node_selector_and_in_affinity_give_identical_classes(seed):
    """pods written with nodeSelector {k: v, ...} and the same pods written as `k In [v]` affinity produce identical
    SelectorClasses arrays (hostname pins included), so the same kernels run"""
    rng = np.random.default_rng([seed, 5])
    _, nodes, pools = gen_cluster(rng, 200, 1, 1)
    kinds = [{}, {POOL: "gpu"}, {POOL: "cpu", "zone": "1"}, {HOST: "node-3"}, {"zone": "2"}, {POOL: "nosuch"},
             {ITYPE: "type-mem"}, {HOST: "node-%d" % rng.integers(200), POOL: "spot"}]
    sels = [kinds[rng.integers(len(kinds))] for _ in range(150)]
    tols = [list(TOLERATION_SETS[rng.integers(len(TOLERATION_SETS))]) for _ in sels]
    by_sel = [SimpleNamespace(selectors=dict(s), tolerations=t, node_affinity=None) for s, t in zip(sels, tols)]
    by_aff = [SimpleNamespace(selectors={}, tolerations=t, node_affinity=kube.node_affinity_terms(
        aff(term([R(k, "In", v) for k, v in s.items()])) if s else None, "p")) for s, t in zip(sels, tols)]
    for use_taints in (False, True):
        a = snapshot.selector_classes(by_sel, nodes, pools, taints=use_taints, affinity=True)
        b = snapshot.selector_classes(by_aff, nodes, pools, taints=use_taints, affinity=True)
        for k in ("pod_class", "node_match", "pool_match"):
            assert getattr(a, k).tobytes() == getattr(b, k).tobytes(), k
        assert a.classes == b.classes
        assert snapshot.pending_match(by_sel, nodes, taints=use_taints, affinity=True).tolist() == \
            snapshot.pending_match(by_aff, nodes, taints=use_taints, affinity=True).tolist()


def test_pending_match_at_scale():
    """20 k nodes, hostname pins and NotIn terms: same answer as the per-pair evaluation"""
    rng = np.random.default_rng(9)
    pods, nodes, pools = gen_cluster(rng, 20000, 30, 120)
    assert snapshot.pending_match(pods, nodes, taints=True, affinity=True).tolist() == \
        restate_pending(pods, nodes, True, True)


# ---------------------------------------------------------------- the switch
def test_switch_reads_the_environment_and_needs_node_selectors(monkeypatch):
    monkeypatch.delenv("ACSFIT_NODE_SELECTORS", raising=False)
    monkeypatch.delenv("ACSFIT_NODE_TAINTS", raising=False)
    for value, want in ((None, False), ("", False), ("0", False), ("1", True), ("yes", True)):
        if value is None:
            monkeypatch.delenv("ACSFIT_NODE_AFFINITY", raising=False)
        else:
            monkeypatch.setenv("ACSFIT_NODE_AFFINITY", value)
        assert _cluster(node_selectors=True).node_affinity is want, value
        assert _cluster(node_selectors=False).node_affinity is False   # no effect without node selectors
        assert _cluster().node_affinity is False
    monkeypatch.setenv("ACSFIT_NODE_AFFINITY", "0")
    assert _cluster(node_selectors=True, node_affinity=True).node_affinity is True
    assert _cluster(node_selectors=True, node_affinity=False).node_affinity is False
    assert _cluster(node_selectors=False, node_affinity=False).node_affinity is False
    with pytest.raises(ValueError):
        _cluster(node_selectors=False, node_affinity=True)
    with pytest.raises(ValueError):
        _cluster(node_affinity=True)                                   # $ACSFIT_NODE_SELECTORS unset: off
    monkeypatch.setenv("ACSFIT_NODE_SELECTORS", "1")
    assert _cluster(node_affinity=True).node_affinity is True
    # independent of the other switches
    c = _cluster(node_affinity=True, node_taints=False, selector_node_states=False)
    assert (c.node_taints, c.selector_node_states) == (False, False)
    assert _cluster(node_affinity=False, node_taints=True).node_taints is True


class _Stop(Exception):
    pass


@pytest.mark.parametrize("on", [False, True])
def test_switch_reaches_engine_scaler_and_scaler(monkeypatch, on):
    from kubernetes_acs_engine_autoscaler_b200 import cluster, engine_scaler
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    assert Scaler("rg", [], 0, 1, 60, True, None, None).node_affinity is False
    seen = []

    class Rec(engine_scaler.EngineScaler):
        def __init__(self, **kw):
            engine_scaler.EngineScaler.__init__(self, **kw)
            seen.append(self.node_affinity)
            raise _Stop()
    monkeypatch.setattr(cluster, "EngineScaler", Rec)
    monkeypatch.delenv("ACSFIT_NODE_AFFINITY", raising=False)
    cl = _cluster(node_selectors=True, node_affinity=on)
    cl.list_nodes = lambda: [SimpleNamespace(obj=node_obj("k8s-cpu-1-0", {ITYPE: "Standard_D2_v2"}))]
    cl.create_kube_node = lambda n: SimpleNamespace(name=n.obj["metadata"]["name"], selectors=n.obj["metadata"]["labels"],
                                                    unschedulable=False)
    cl.arm_parameters, cl.arm_template = {"cpuVMSize": {"value": "Standard_D2_v2"}}, {}
    with pytest.raises(_Stop):
        cl.loop_logic()
    assert seen == [on]


def test_scaler_passes_the_switch_to_pending_match():
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    s = Scaler("rg", [], 0, 1, 60, True, None, None)
    s.selector_node_states = True
    nodes = [SimpleNamespace(selectors={POOL: "cpu"}, name="n0"), SimpleNamespace(selectors={POOL: "gpu"}, name="n1")]
    pods = [SimpleNamespace(selectors={}, node_affinity=kube.node_affinity_terms(aff(term([R(POOL, "In", "gpu")])), "p"))]
    assert s.no_pending_match(nodes, pods).tolist() == [False, False]
    s.node_affinity = True
    assert s.no_pending_match(nodes, pods).tolist() == [True, False]
    pods[0].node_affinity = kube.node_affinity_terms(aff(term(fields=[F("In", "elsewhere")])), "p")
    assert s.no_pending_match(nodes, pods).tolist() == [True, True]


# ---------------------------------------------------------------- warnings of get_pods_to_schedule
def test_warnings_and_their_precedence(tmp_path, monkeypatch, oracle_mod):
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", SelOracleEngine())
    j = []

    def node(pool, itype, taints=None):
        o = node_obj("k8s-%s-1-0" % pool, {POOL: pool, ITYPE: itype, "failure-domain.beta.kubernetes.io/region": "r",
                                           HOST: "k8s-%s-1-0" % pool}, taints)
        return KubeNode(gu.FakeKubeObject(o, j, "node"))
    # cpu: 2 cores, untainted; gpu: 6 cores, tainted sku=gpu:NoSchedule
    nodes = [node("cpu", "Standard_D2_v2"), node("gpu", "Standard_NC6", [T("sku", "gpu")])]
    pools = [AgentPool("cpu", "Standard_D2_v2", nodes[:1]), AgentPool("gpu", "Standard_NC6", nodes[1:])]
    gpu, tol = aff(term([R(POOL, "In", "gpu")])), [Tol("sku", "Exists")]
    U, A, S, X = UNTOLERATED, AFFINITY, NO_POOL, NO_FIT
    specs = [  # name, cpu, selector, affinity, tolerations, warning with (taints, affinity) on/on, off/on, on/off
        ("small", "1", None, None, None, (None, None, None)),
        ("aff-gpu", "1", None, gpu, None, (U, None, None)),                      # affinity holds, the taint fails
        ("aff-gpu-tol", "1", None, gpu, tol, (None, None, None)),
        ("aff-nowhere", "1", None, aff(term([R(POOL, "In", "nosuch")])), tol, (A, A, None)),
        ("aff-cpu-big", "5", None, aff(term([R(POOL, "In", "cpu")])), tol, (A, A, None)),
        ("sel-cpu-aff-gpu", "1", {POOL: "cpu"}, gpu, tol, (A, A, None)),          # the selector alone passes
        ("sel-nowhere-aff", "1", {POOL: "nosuch"}, gpu, tol, (S, S, S)),          # the selector fails first
        ("daemon", "1", None, aff(term(fields=[F("In", "k8s-cpu-1-0")])), tol, (A, A, None)),
        ("host-pin", "1", None, aff(term([R(HOST, "In", "k8s-gpu-1-0")])), tol, (A, A, None)),
        ("aff-big-untol", "5", None, aff(term([R(POOL, "NotIn", "cpu")])), None, (U, None, U)),
        ("huge-aff", "64", None, gpu, tol, (X, X, X)),                           # fits no pool at all
        ("big", "5", None, None, None, (U, None, U)),
    ]
    pods = [KubePod(gu.FakeKubeObject(pod_obj(name, a, sel, cpu, tols), j, "pod"))
            for name, cpu, sel, a, tols, _ in specs]
    log = logging.getLogger("autoscaler.cluster")
    for k, (taints, affinity) in enumerate(((True, True), (False, True), (True, False))):
        monkeypatch.setenv("ACSFIT_NODE_TAINTS", "0")
        monkeypatch.setenv("ACSFIT_NODE_AFFINITY", "0")
        cl = _cluster(node_selectors=True, node_taints=taints, node_affinity=affinity)
        handler = gu.ListHandler()
        log.addHandler(handler)
        try:
            got = cl.get_pods_to_schedule(pods, pools)
        finally:
            log.removeHandler(handler)
        assert [p.name for p in got] == [s[0] for s in specs if s[5][k] is None], k
        want = [s[5][k] % ((s[0], p.selectors) if s[5][k] == NO_POOL else s[0]) for s, p in zip(specs, pods)
                if s[5][k] is not None]
        assert [m for lvl, _, m in handler.records if lvl == "WARNING"] == want, k
