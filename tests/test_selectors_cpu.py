"""`-m "not gpu"`: the node-selector mode's host pieces -- the class builder, AgentPool.labels, the plain-C selector
oracle (tests/sel_oracle.c) against a pure-Python restatement of the upstream rules, and the tie of the selector
oracle to the pinned oracle when every pod is class 0 -- and the adversarial generator's targets."""
from types import SimpleNamespace

import numpy as np
import pytest

import sel_oracle
import selector_cases as sc
from kubernetes_acs_engine_autoscaler_b200 import snapshot
from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool
from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubeResource


def _node(labels):
    return SimpleNamespace(selectors=labels, unschedulable=False)


def _pool(name, nodes, itype="Standard_D2_v2"):
    return AgentPool(name, itype, nodes)


# ---------------------------------------------------------------- class builder
def test_classes_deduplicate_signatures_and_set_bit0():
    h, it = "kubernetes.io/hostname", "beta.kubernetes.io/instance-type"
    nodes = [_node({"agentpool": "a", h: "n0", it: "Standard_D2_v2"}), _node({"agentpool": "a", h: "n1", it: "Standard_D2_v2"}),
             _node({"agentpool": "b", h: "n2", it: "Standard_D2_v2"})]
    pools = [_pool("a", nodes[:2]), _pool("b", nodes[2:])]
    pods = [SimpleNamespace(selectors=s) for s in (
        {}, {"agentpool": "a"}, {"agentpool": "a", it: "Standard_D2_v2"},
        {h: "n2"}, {"agentpool": "b"}, {"agentpool": "b"}, {"agentpool": "zz"}, {"agentpool": "a", h: "n0"})]
    cls = snapshot.selector_classes(pods, nodes, pools)
    pc = cls.pod_class.tolist()
    assert pc[0] == 0
    assert pc[1] == pc[2] != 0                 # same nodes, same pools
    assert pc[4] == pc[5] != pc[3]             # {h: n2} matches node 2 but no pool; {agentpool: b} matches pool b
    assert len(set(pc)) == cls.classes == 6
    assert all(int(m) & 1 for m in cls.node_match) and all(int(m) & 1 for m in cls.pool_match)
    for i, pod in enumerate(pods):
        for n, node in enumerate(nodes):
            assert bool((int(cls.node_match[n]) >> pc[i]) & 1) == KubeNode.is_match(node, pod)
        for t, pool in enumerate(pools):
            want = all(pool.labels.get(k) == v for k, v in pod.selectors.items())
            assert bool((int(cls.pool_match[t]) >> pc[i]) & 1) == want
    # a selector that matches everything shares class 0
    every = snapshot.selector_classes([SimpleNamespace(selectors={"beta.kubernetes.io/instance-type": "Standard_D2_v2"})],
                                      [], pools)
    assert every.trivial and every.classes == 1


def test_classes_64_accepted_65_refused():
    nodes = [_node({"h": "n%d" % i}) for i in range(70)]
    pods = [SimpleNamespace(selectors={"h": "n%d" % i}) for i in range(63)]
    cls = snapshot.selector_classes(pods, nodes, [])
    assert cls.classes == 64 and cls.pod_class.max() == 63
    assert int(cls.node_match[62]) == 1 | (1 << 63)
    pods.append(SimpleNamespace(selectors={"h": "n63"}))
    with pytest.raises(ValueError):
        snapshot.selector_classes(pods, nodes, [])


# ---------------------------------------------------------------- AgentPool.labels
def test_pool_labels():
    a = _node({"agentpool": "old", "kubernetes.io/hostname": "x0", "openai/cordoned-by-autoscaler": "true",
               "zone": "1", "gpu": "yes", "beta.kubernetes.io/instance-type": "stale"})
    b = _node({"agentpool": "old", "kubernetes.io/hostname": "x1", "openai/cordoned-by-autoscaler": "true",
               "zone": "2", "gpu": "yes"})
    labels = _pool("p", [a, b], "Standard_NC6").labels
    assert labels == {"agentpool": "p", "beta.kubernetes.io/instance-type": "Standard_NC6", "gpu": "yes"}
    assert _pool("e", []).labels == {"agentpool": "e", "beta.kubernetes.io/instance-type": "Standard_D2_v2"}
    one = _pool("o", [_node({"kubernetes.io/hostname": "h", "zone": "3"})]).labels
    assert one == {"zone": "3", "agentpool": "o", "beta.kubernetes.io/instance-type": "Standard_D2_v2"}


# ---------------------------------------------------------------- the selector oracle vs a Python restatement
def _res(row):
    r = KubeResource()
    r.raw = {"k%d" % d: float(v) for d, v in enumerate(row)}
    return r


def _python_tick(c, used):
    """get_pods_to_schedule + get_pending_pods + fulfill_pending with the upstream selector rules, on KubeResource
    values and KubeNode.is_match.  Returns (feasible, placed, acc_pool, new_size, decisions, used)."""
    P = len(c["selectors"])
    pods = [SimpleNamespace(selectors=c["selectors"][i], resources=_res(c["req"][i])) for i in range(P)]
    units = [_res(u) for u in c["unit_all"]]
    pools = c["pools"]
    decisions = 0
    feasible = np.zeros(P, dtype=bool)
    for i, pod in enumerate(pods):
        for t, pool in enumerate(pools):
            decisions += 1
            if all(pool.labels.get(k) == v for k, v in pod.selectors.items()) and (units[t] - pod.resources).possible:
                feasible[i] = True
                break
    caps = [_res(c["cap_type"][k]) for k in c["node_type"]]
    used_r = [_res(u) for u in used]
    placed = np.where(feasible, -1, -2)
    for i in np.nonzero(feasible)[0]:
        for n, node in enumerate(c["nodes"]):
            decisions += 1
            if KubeNode.is_match(node, pods[i]) and (caps[n] - (used_r[n] + pods[i].resources)).possible:
                used_r[n] = used_r[n] + pods[i].resources
                placed[i] = n
                break
    pending = [i for i in range(P) if placed[i] == -1]
    acc = np.full(P, -1)
    new_size = np.asarray(c["pool_actual"], dtype=np.int64).copy()
    left = len(pending)
    for v, t in enumerate(c["order"]):
        if c["pool_ignored"][v] or not left or not pending:
            continue
        bins, bin_of = [], {}
        for i in pending:
            if acc[i] >= 0:
                continue
            decisions += 1
            if not (all(pools[t].labels.get(k) == val for k, val in pods[i].selectors.items())
                    and (units[t] - pods[i].resources).possible):
                continue
            for b, rem in enumerate(bins):
                decisions += 1
                if (rem - pods[i].resources).possible:
                    bins[b] = rem - pods[i].resources
                    bin_of[i] = b
                    break
            else:
                bins.append(units[t] - pods[i].resources)
                bin_of[i] = len(bins) - 1
        needed = len(bins) + c["over_provision"]
        room = int(c["pool_max"][v]) - int(c["pool_actual"][v])
        requested = needed - max(0, needed - room)
        new_size[v] = int(c["pool_actual"][v]) + requested
        for i, b in bin_of.items():
            if b < min(len(bins), requested):
                acc[i] = v
                left -= 1
    used_out = np.asarray([[u.raw["k%d" % d] for d in range(used.shape[1])] for u in used_r])
    return feasible, placed, acc, new_size, decisions, used_out


@pytest.mark.parametrize("kind", sc.KINDS)
def test_sel_oracle_matches_python_restatement(kind):
    c = sc.make_case(kind, 4, seed=3, n_nodes=40, n_pods=160)
    used = c["used0"].copy()
    got = sel_oracle.scale_up_sel(c, used)
    feasible, placed, acc, new_size, decisions, used_py = _python_tick(c, c["used0"])
    assert np.array_equal(got["feasible"].astype(bool), feasible)
    assert np.array_equal(got["placed"], placed)
    assert np.array_equal(got["acc_pool"], acc)
    assert np.array_equal(got["new_size"], new_size)
    assert got["decisions"] == decisions
    assert np.array_equal(used.view(np.uint64), used_py.view(np.uint64))


@pytest.mark.parametrize("D", sc.DIMS)
@pytest.mark.parametrize("kind", sc.KINDS)
def test_class0_sel_oracle_equals_pinned_oracle(kind, D, oracle_mod):
    c = sc.make_case(kind, D, seed=5)
    zero = np.zeros_like(c["pod_class"])
    ones_n, ones_t = np.ones(len(c["node_type"]), np.uint64), np.ones(4, np.uint64)
    m1, e1 = sel_oracle.feasible_mask_sel(c["req"], c["unit_all"], ones_t, zero)
    m0, e0 = oracle_mod.feasible_mask(c["req"], c["unit_all"])
    assert np.array_equal(m1, m0) and e1 == e0
    u1, u0 = c["used0"].copy(), c["used0"].copy()
    p1, d1 = sel_oracle.first_fit_nodes_sel(c["req"], c["cap_type"], c["node_type"], u1, ones_n, zero)
    p0, d0 = oracle_mod.first_fit_nodes(c["req"], c["cap_type"], c["node_type"], u0)
    assert np.array_equal(p1, p0) and d1 == d0 and np.array_equal(u1.view(np.uint64), u0.view(np.uint64))
    pend = np.nonzero(p0 < 0)[0]
    args = (c["req"][pend], len(pend), c["unit_ordered"], c["pool_actual"], c["pool_max"], c["pool_ignored"], 1)
    f1 = sel_oracle.fulfill_pending_sel(*args, ones_t, zero[pend])
    f0 = oracle_mod.fulfill_pending(*args)
    for k in f0:
        assert np.array_equal(np.asarray(f1[k]), np.asarray(f0[k])), k


# ---------------------------------------------------------------- the generator hits its targets
def _plain(c):
    zc = dict(c, pod_class=np.zeros_like(c["pod_class"]))
    used = c["used0"].copy()
    return sel_oracle.scale_up_sel(zc, used), used


@pytest.mark.parametrize("D", sc.DIMS)
@pytest.mark.parametrize("kind", sc.KINDS)
def test_cases_are_selector_sensitive(kind, D):
    c = sc.make_case(kind, D)
    used = c["used0"].copy()
    sel = sel_oracle.scale_up_sel(c, used)
    plain, used_p = _plain(c)
    same = all(np.array_equal(np.asarray(sel[k]), np.asarray(plain[k])) for k in ("feasible", "placed", "acc_pool", "new_size"))
    assert same == (kind not in sc.SENSITIVE)
    if kind == "classes_64":
        assert c["classes"] == 64
    if kind == "two_classes":
        assert c["classes"] == 2
    if kind == "no_selectors":
        assert c["classes"] == 1
    if kind in ("nothing",):
        assert (sel["placed"] == -2).sum() > (plain["placed"] == -2).sum()
    if kind in ("pool_only", "all_mismatched"):
        assert sel["new_size"][c["order"].index(3)] > c["pool_actual"][c["order"].index(3)]
    if kind == "first_mismatch":  # the first node with room does not match a pinned pod
        pinned = np.nonzero(c["pod_class"])[0]
        assert (plain["placed"][pinned] == 0).any() and not (sel["placed"][pinned] == 0).any()
