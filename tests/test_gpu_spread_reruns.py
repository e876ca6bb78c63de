"""`-m gpu`: the topology-spread node pass (acsfit_first_fit_nodes_ts) at the limits of its reruns, against the plain-C
oracle (tests/ts_oracle.c) exactly -- placements, used bits, node counts and masks, the rises and flips the reruns
fixed, and the bin pass over the pods left pending -- under both candidate scans and a multi-wave schedule:

* the 4096-rise cap: past its last fixed rise the pass keeps its levels, refusing pods the scheduler would place and
  accepting none it would refuse; a flip after the cap is still followed;
* events at one position: two keys rising together (lower key first), a flip and a rise, a rise at the first and at
  the last position of the list;
* 64 keys rising in turn over their own small domain sets;
* pod lists (pod_idx) that drop and shuffle rows, for the spread, pod-affinity and anti-affinity node passes, and the
  host layer's list that leaves out a pod with a non-finite request."""
import numpy as np
import pytest

import aa_cases as ac
import test_gpu_anti_affinity as aa
import test_gpu_pod_affinity as pa
from test_gpu_pod_affinity import SCHEDULES
from test_gpu_topology_spread import (INT32_MAX, MAX_SPREAD_RISES, U64, assert_equal, case, eng, host,  # noqa: F401
                                      oracle_of_case, run, tile_edge_case)

pytestmark = pytest.mark.gpu

FENCE = 1 << 20  # a start count outside a key's domain set that keeps its pods off the node


def check(eng, c, pod_idx=None, schedules=("default",), scans=(1, 0)):
    """the GPU against the oracle on case `c` over the pod list `pod_idx`; returns the oracle's results and the last
    GPU run"""
    o = oracle_of_case(c, pod_idx)
    try:
        for ranks in scans:
            eng.set_knob("ranks", ranks)
            for schedule in schedules:
                g = run(eng, c, o["pend"], o["present"], SCHEDULES[schedule], pod_idx=pod_idx)
                assert_equal(g, o)
    finally:
        eng.set_knob("ranks", 1)
    return o, g


def blank(P, N, D=2, cap=1000.0, keys=1):
    """P pods requesting 1.0 in D dims over N empty nodes of capacity `cap`, no masks, no key on any pod; a pool of
    at most 1000 nodes whose unit takes four pods"""
    return {"req": np.ones((P, D)), "cap_type": np.full((N, D), cap), "node_type": np.arange(N, dtype=np.int32),
            "used0": np.zeros((N, D)), "unit": np.full((1, D), 4.0), "pool_actual": np.zeros(1, np.int32),
            "pool_max": np.full(1, 1000, np.int32), "pool_ignored": np.zeros(1, np.uint8), "over_provision": 0,
            "pod_carries": np.zeros(P, U64), "pod_matches": np.zeros(P, U64), "node_carries0": np.zeros(N, U64),
            "node_matches0": np.zeros(N, U64), "pa_requires": np.zeros(P, U64), "pa_self": np.zeros(P, U64),
            "pa_matches": np.zeros(P, U64), "node_has0": np.zeros(N, U64),
            "ts_keys": keys, "ts_key": np.full(P, 0xFF, np.uint8), "ts_skew": np.zeros(P, np.int32),
            "ts_matches": np.zeros(P, U64), "ts_count0": np.zeros((keys, N), np.int32), "ts_domain": np.zeros(N, U64),
            "ts_floor": np.full(keys, INT32_MAX, np.int32)}


def spread_rule_violations(c, placed, pod_idx=None):
    """replays the placements `placed` (list positions) in plain Python with each key's minimum recomputed from the
    running counts at every pod, and returns the positions of the placed pods that rule refuses"""
    rows = np.arange(len(c["req"])) if pod_idx is None else np.asarray(pod_idx)
    count = c["ts_count0"].astype(np.int64)
    dom = [[n for n in range(len(c["ts_domain"])) if (int(c["ts_domain"][n]) >> k) & 1] for k in range(c["ts_keys"])]
    bad = []
    for i, n in enumerate(placed.tolist()):
        if n < 0:
            continue
        r = rows[i]
        k = int(c["ts_key"][r])
        if k != 0xFF:
            low = min([int(c["ts_floor"][k])] + [int(count[k, m]) for m in dom[k]])
            if count[k, n] > int(c["ts_skew"][r]) + low:
                bad.append(i)
        for b in range(c["ts_keys"]):
            if (int(c["ts_matches"][r]) >> b) & 1:
                count[b, n] += 1
    return bad


# ---------------------------------------------------------------- the 4096-rise cap
def cap_case():
    """8400 replicas of one group (maxSkew 1) over two roomy nodes: 4200 rises, 4096 of them followed"""
    return tile_edge_case(8400, 1e6)


def capped_keys_case():
    """three keys over overlapping domain sets of three roomy nodes, their replicas in turn, 4096 of their rises
    followed; then, past the cap, pods that need signature 0 before and after the self-affine pod that brings it"""
    P, N = 11000, 3
    c = blank(P + 6, N, cap=1e6, keys=3)
    c["ts_domain"] = np.asarray([0b101, 0b111, 0b110], U64)  # key 0: nodes 0, 1; key 1: 1, 2; key 2: all
    k = np.arange(P) % 3
    c["ts_key"][:P] = k
    c["ts_matches"][:P] = U64(1) << k.astype(U64)
    c["ts_skew"][:P] = np.where(k == 2, 1, 0)  # maxSkew 2 for key 2, 1 for the others; every replica selects itself
    sig = U64(1)
    c["pa_requires"][P:] = sig                 # pods P .. P+5: no key; P+2 is self-affine, the others need it
    c["pa_self"][P + 2] = c["pa_matches"][P + 2] = sig
    return c


def test_cap_worked_case(eng):
    c = cap_case()
    o, g = check(eng, c)
    assert g["rises"] == [(0, 2 * r + 1) for r in range(MAX_SPREAD_RISES)]
    placed = o["placed"]
    assert placed[:8192].tolist() == [0, 1] * 4096 and placed[8192:8194].tolist() == [0, 1]
    assert (placed[8194:] < 0).all() and o["count"].tolist() == [[4097, 4097]]
    # the 206 pods the capped pass refused: one replica per new node (unlimited, every pod lands on the two nodes)
    f = g["fulfill"]
    assert f["bins_opened"].tolist() == [206] and f["new_size"].tolist() == [206]
    assert f["bin_of"].tolist() == list(range(206))
    # what it placed, the scheduler's rule (the true minimums at each pod) admits too
    assert spread_rule_violations(c, g["placed"]) == []


def test_cap_with_keys_and_a_later_flip(eng):
    c = capped_keys_case()
    o, g = check(eng, c, scans=(1,))  # (4097 passes of 11006 pods: the worked case covers the float64 scan)
    assert len(g["rises"]) == MAX_SPREAD_RISES and {k for k, _ in g["rises"]} == {0, 1, 2}
    assert g["flips"] == [(0, 11002)] and g["flips"][0][1] > g["rises"][-1][1]
    placed = o["placed"]
    assert (placed[11000:11002] < 0).all() and (placed[11002:] >= 0).all()  # blocked before the flip, not after
    assert (placed[:11000] < 0).any() and spread_rule_violations(c, g["placed"]) == []


# ---------------------------------------------------------------- events at one position
def twin_keys_case(P=40):
    """two keys over the same two nodes, every pod selected by both and constrained by one of them in turn: both
    minimums rise at every second pod"""
    c = blank(P, 2, keys=2)
    c["ts_domain"][:] = 0b11
    c["ts_key"][:] = np.arange(P) % 2
    c["ts_matches"][:] = 0b11
    return c


def flip_and_rise_case():
    """pod 1 both raises key 0's minimum and brings signature 0, which the pods after it need"""
    P = 12
    c = blank(P, 3)
    c["ts_domain"][:2] = 1
    c["ts_count0"][0, 2] = FENCE
    c["ts_key"][:6] = 0
    c["ts_matches"][:6] = 1
    c["pa_requires"][1] = c["pa_self"][1] = c["pa_matches"][1] = 1
    c["pa_requires"][6:] = 1
    return c


def first_and_last_case(P=512):
    """pod 0 raises key 0 (one domain), the last pod of the list key 1 (two domains, one of them at 1 already)"""
    c = blank(P, 2, keys=2)
    c["ts_domain"][:] = [0b11, 0b10]
    c["ts_count0"][1, 0] = 1
    c["ts_key"][[0, P - 1]] = [0, 1]
    c["ts_matches"][[0, P - 1]] = [1, 2]
    return c


def test_two_keys_rise_at_one_position_lower_key_first(eng):
    _, g = check(eng, twin_keys_case())
    assert g["rises"] == [(k, p) for p in range(1, 40, 2) for k in (0, 1)]


def test_flip_and_rise_at_one_position(eng):
    o, g = check(eng, flip_and_rise_case())
    assert g["flips"] == [(0, 1)] and (0, 1) in g["rises"]
    assert o["placed"][:2].tolist() == [0, 1] and (o["placed"][6:] == 1).all()


def test_rises_at_the_first_and_last_position(eng):
    o, g = check(eng, first_and_last_case())
    assert g["rises"] == [(0, 0), (1, 511)] and o["placed"][-1] == 1


@pytest.mark.parametrize("name", ["twin_keys", "flip_and_rise", "first_and_last"])
def test_one_position_events_in_waves(eng, name):
    c = {"twin_keys": twin_keys_case, "flip_and_rise": flip_and_rise_case,
         "first_and_last": first_and_last_case}[name]()
    check(eng, c, schedules=("waves_prune", "waves_noprune"), scans=(1,))


# ---------------------------------------------------------------- 64 rising keys
def keys64_case(D, seed=0):
    """64 groups, each over a domain set of its own 2 or 3 nodes (the other nodes fenced off by their counts), with
    maxSkew 1 or 2; their replicas interleaved so that the rises alternate between the keys; a few pods without a key
    fill in"""
    rng = np.random.default_rng(seed)
    size = 2 + (np.arange(64) % 2)
    first = np.concatenate([[0], np.cumsum(size)])
    N = int(first[-1])
    reps = rng.integers(12, 17, size=64)
    order = [k for r in range(int(reps.max())) for k in range(64) if r < reps[k]]
    P = len(order)
    c = blank(P, N, D, cap=1000.0, keys=64)
    c["req"] = rng.integers(1, 4, size=(P, D)).astype(np.float64)
    k = np.asarray(order)
    c["ts_key"][:] = k
    c["ts_matches"][:] = U64(1) << k.astype(U64)
    c["ts_skew"][:] = (k % 3 == 0).astype(np.int32)  # maxSkew 2 for every third key
    c["ts_count0"][:] = FENCE
    for g in range(64):
        c["ts_domain"][first[g]:first[g + 1]] = U64(1) << U64(g)
        c["ts_count0"][g, first[g]:first[g + 1]] = 0
    free = rng.random(P) < 0.05
    c["ts_key"][free] = 0xFF
    c["ts_matches"][free] = 0
    return c


@pytest.mark.parametrize("D", [2, 16])
def test_64_keys_rise_in_turn(eng, D):
    o, g = check(eng, keys64_case(D))
    keys = [k for k, _ in g["rises"]]
    assert 63 in keys and len(set(keys)) == 64 and 300 <= len(keys) < MAX_SPREAD_RISES
    assert sum(a != b for a, b in zip(keys, keys[1:])) > len(keys) // 2  # the keys alternate


def test_64_keys_in_waves(eng):
    check(eng, keys64_case(2), schedules=("waves_prune",), scans=(1,))


# ---------------------------------------------------------------- pod lists
def pod_list(P, seed=0):
    """about 90 % of the rows 0 .. P-1, shuffled"""
    rng = np.random.default_rng(seed + 5)
    return rng.permutation(np.nonzero(rng.random(P) >= 0.1)[0]).astype(np.int32)


@pytest.mark.parametrize("base,ts_kind,pa_kind", [("with_sel", "rises", "mixed"), ("edges", "rises", "mixed"),
                                                  ("keys64", None, None)])
def test_ts_pod_list(eng, base, ts_kind, pa_kind):
    c = keys64_case(2) if base == "keys64" else case(base, ts_kind, pa_kind, 4)
    idx = pod_list(len(c["req"]))
    o, _ = check(eng, c, idx)
    assert o["rises"] and (pa_kind is None or o["flips"])


def test_pa_pod_list(eng):
    c = pa.case("with_sel", "sig2", 4)
    idx = pod_list(len(c["req"]))
    o = pa.oracle_of_case(c, idx)
    assert o["flips"]
    for ranks in (1, 0):
        eng.set_knob("ranks", ranks)
        try:
            pa.assert_equal(pa.run(eng, c, o["pend"], o["present"], {}, pod_idx=idx), o)
        finally:
            eng.set_knob("ranks", 1)


@pytest.mark.parametrize("kind", ["with_sel", "replicas"])
def test_aa_pod_list(eng, kind):
    c = ac.make_case(kind, 4)
    idx = pod_list(len(c["req"]))
    o = aa.oracle_of_case(c, idx)
    for ranks in (1, 0):
        eng.set_knob("ranks", ranks)
        try:
            g, _, _ = aa.run(eng, c, o["pend"], {}, pod_idx=idx)
            aa.assert_equal(g, o)
        finally:
            eng.set_knob("ranks", 1)


# ---------------------------------------------------------------- the host layer's pod list
INFINITE_CPU = "1" + "0" * 400  # 1e400 cores: parses to an infinite request


def rules_state(with_infinite):
    """pool `agentpool1` (Standard_D2_v2) of four nodes, two of them labelled disk=ssd, one running a `web` replica.
    Pending, in order: 15 `web` replicas spread with maxSkew 1 over kubernetes.io/hostname (the second one with an
    infinite cpu request when `with_infinite`), three self-affine `cache` pods that select disk=ssd nodes, and five
    `ha` pods that avoid each other (one too many for the nodes)"""
    names = ["k8s-agentpool1-16334397-%d" % i for i in range(4)]

    def node(i, name):
        labels = {"beta.kubernetes.io/instance-type": "Standard_D2_v2", "kubernetes.io/hostname": name,
                  "agentpool": "agentpool1", "failure-domain.beta.kubernetes.io/region": "southcentralus"}
        if i >= 2:
            labels["disk"] = "ssd"
        return {"metadata": {"name": name, "creationTimestamp": "2016-08-25T05:13:16Z", "labels": labels}, "spec": {}}

    def term(app):
        return {"topologyKey": "kubernetes.io/hostname", "labelSelector": {"matchLabels": {"app": app}}}

    def pod(n, app, cpu="100m", node_name=None, **spec):
        spec = dict(spec, containers=[{"name": "c", "resources": {"requests": {"cpu": cpu}}}])
        if node_name:
            spec["nodeName"] = node_name
        return {"metadata": {"name": n, "namespace": "default", "uid": "uid-" + n, "labels": {"app": app},
                             "creationTimestamp": "2026-09-20T07:00:00Z"}, "spec": spec,
                "status": {"phase": "Running" if node_name else "Pending"}}
    spread = [{"maxSkew": 1, "topologyKey": "kubernetes.io/hostname", "whenUnsatisfiable": "DoNotSchedule",
               "labelSelector": {"matchLabels": {"app": "web"}}}]
    pods = [pod("run-web", "web", node_name=names[0], topologySpreadConstraints=spread)]
    pods += [pod("web-%d" % i, "web", topologySpreadConstraints=spread) for i in range(15)]
    if with_infinite:
        pods.insert(3, pod("web-inf", "web", INFINITE_CPU, topologySpreadConstraints=spread))
    pods += [pod("cache-%d" % i, "cache", nodeSelector={"disk": "ssd"},
                 affinity={"podAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [term("cache")]}})
             for i in range(3)]
    pods += [pod("ha-%d" % i, "ha",
                 affinity={"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [term("ha")]}})
             for i in range(5)]
    return {"nodes": [node(i, n) for i, n in enumerate(names)], "pods": pods,
            "arm_parameters": {"agentpool1VMSize": {"value": "Standard_D2_v2"}}, "settings": {}}


def first_fit_with_every_rule(state):
    from kubernetes_acs_engine_autoscaler_b200 import snapshot
    from test_gpu_taints import _kube
    nodes, pods, _ = _kube(state)
    running = [p for p in pods if p.node_name]
    pending = [p for p in pods if not p.node_name]
    rules = dict(classes=snapshot.selector_classes(pending, nodes, [], taints=True, affinity=True),
                 anti_affinity=snapshot.anti_affinity(pending, nodes, running),
                 pod_affinity=snapshot.pod_affinity(pending, nodes, running),
                 topology_spread=snapshot.topology_spread(pending, nodes, running, []))
    assert not any(r.trivial for r in rules.values())
    placed = snapshot.first_fit_nodes(pending, nodes, **rules)
    return pending, placed, rules, [dict(n.used_capacity.raw) for n in nodes]


def test_host_pod_list_without_the_infinite_pod(host, eng):
    pending, with_inf, rules, used = first_fit_with_every_rule(rules_state(True))
    bad = [i for i, p in enumerate(pending) if p.name == "web-inf"]
    assert bad == [2] and with_inf[2] == -1
    _, without, rules0, used0 = first_fit_with_every_rule(rules_state(False))
    assert np.delete(with_inf, 2).tolist() == without.tolist() and used == used0
    ts, ts0 = rules["topology_spread"], rules0["topology_spread"]
    assert ts.keys == ts0.keys and ts.node_count.tolist() == ts0.node_count.tolist()
    np.testing.assert_array_equal(rules["pod_affinity"].node_has, rules0["pod_affinity"].node_has)
    np.testing.assert_array_equal(rules["anti_affinity"].node_carries, rules0["anti_affinity"].node_carries)
    np.testing.assert_array_equal(rules["anti_affinity"].node_matches, rules0["anti_affinity"].node_matches)
    # the rules were at work: the web replicas' minimum rose past the pod left out, and the fifth `ha` pod waits
    assert eng.last_spread_rises() and (without < 0).sum() == 1 and without[-1] == -1
