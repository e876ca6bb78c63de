"""Adversarial scale-up ticks for the node-selector mode (tests/test_gpu_selectors.py, tests/test_selectors_cpu.py).

Every case is a dense tick (the buffers of acsfit_scale_up_sel) built from labelled nodes, agent pools and pods
with nodeSelectors; the classes come from snapshot.selector_classes, the pool labels from AgentPool.labels.  Every
case except "no_selectors" is selector-sensitive: the plain path gives a different answer (SENSITIVE lists the
cases; the tests assert it).  Four pools, visited in cost order pool1, pool0, pool3, pool2 (`order`); pool3 has no
node at all.  Capacities are pool units; some node rows sit exactly at or one ulp below a fit.
"""
from types import SimpleNamespace

import numpy as np

from kubernetes_acs_engine_autoscaler_b200 import snapshot
from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool

POOLS = ("pool0", "pool1", "pool2", "pool3")
ORDER = (1, 0, 3, 2)  # visiting order (cheapest first) as indices into POOLS
KINDS = ("first_mismatch", "first_pool", "pool_only", "nothing", "all_mismatched", "last_pool", "two_classes",
         "classes_64", "ulp", "no_selectors")
SENSITIVE = tuple(k for k in KINDS if k != "no_selectors")
DIMS = (2, 4, 8, 16)


def _unit(D, t):
    u = np.zeros(D)
    u[0] = (4.0, 8.0, 16.0, 32.0)[t]             # cpu
    u[1] = (16.0, 32.0, 64.0, 128.0)[t] * 2 ** 30  # memory
    for d in range(2, D):
        u[d] = 110.0 + d
    return u


def make_case(kind, D, seed=0, n_nodes=300, n_pods=1500):
    rng = np.random.default_rng([seed, D, KINDS.index(kind)])
    T = len(POOLS)
    units = np.stack([_unit(D, t) for t in range(T)])
    # nodes: pool0 first (the first nodes in list order), then pool1, then pool2; pool3 is empty
    share = (n_nodes // 2, n_nodes // 4, n_nodes - n_nodes // 2 - n_nodes // 4)
    node_pool = np.concatenate([np.full(s, t, dtype=np.int32) for t, s in enumerate(share)])
    nodes = []
    for n, t in enumerate(node_pool):
        labels = {"agentpool": POOLS[t], "beta.kubernetes.io/instance-type": "type%d" % t,
                  "kubernetes.io/hostname": "k8s-%s-0-%d" % (POOLS[t], n), "zone": "z%d" % (n % 3)}
        if n % 7 == 0:
            labels["openai/cordoned-by-autoscaler"] = "true"
        nodes.append(SimpleNamespace(selectors=labels, unschedulable=False))
    pools = [AgentPool(POOLS[t], "type%d" % t, [nodes[n] for n in np.nonzero(node_pool == t)[0]]) for t in range(T)]
    cap_type = units[:3].copy()
    node_type = node_pool.copy()
    used = cap_type[node_type] * rng.uniform(0.0, 0.9, size=(n_nodes, 1))
    used[:, 2:] = 0.0
    # requests: small pods (fit many nodes) and a few large ones; the pods column stays 1
    req = np.zeros((n_pods, D))
    req[:, 0] = rng.choice([0.1, 0.25, 0.5, 1.0, 2.0, 6.0], size=n_pods, p=[.3, .25, .2, .15, .07, .03])
    req[:, 1] = rng.choice([0.5, 1.0, 2.0, 4.0, 12.0], size=n_pods) * 2 ** 30
    if D > 2:
        req[:, 2] = 1.0
    if kind == "ulp":
        # node rows exactly full for a 0.5-cpu pod, and others one ulp short of it
        k = np.arange(0, n_nodes, 5)
        used[k, 0] = cap_type[node_type[k], 0] - 0.5
        used[k[1::2], 0] = np.nextafter(used[k[1::2], 0], np.inf)
    selectors = [{} for _ in range(n_pods)]
    pick = rng.random(n_pods)
    if kind == "first_mismatch":  # pool0 nodes come first and have room; the pinned pods must skip them
        for i in np.nonzero(pick < 0.4)[0]:
            selectors[i] = {"agentpool": "pool2"}
    elif kind == "first_pool":  # pinned to pool1, the first pool visited: every pod stays eligible for it, so the
        # first bin pass may be chained behind the (selector) node pass; the pinned pods still skip pool0's nodes
        for i in np.nonzero(pick < 0.4)[0]:
            selectors[i] = {"agentpool": "pool1"}
    elif kind == "pool_only":  # matches no node, only the empty pool3
        for i in np.nonzero(pick < 0.3)[0]:
            selectors[i] = {"agentpool": "pool3"}
    elif kind == "nothing":  # matches nothing at all: infeasible
        for i in np.nonzero(pick < 0.3)[0]:
            selectors[i] = {"agentpool": "gpupool"}
    elif kind == "all_mismatched":  # every pod pinned where no node is
        selectors = [{"agentpool": "pool3"} for _ in range(n_pods)]
    elif kind == "last_pool":  # pool2 is visited last; its nodes are full
        used[node_pool == 2] = cap_type[2]
        for i in np.nonzero(pick < 0.3)[0]:
            selectors[i] = {"beta.kubernetes.io/instance-type": "type2"}
    elif kind == "two_classes":  # a few pods pinned to one host (class 1)
        host = nodes[n_nodes - 1].selectors["kubernetes.io/hostname"]
        for i in np.nonzero(pick < 0.05)[0]:
            selectors[i] = {"kubernetes.io/hostname": host}
    elif kind == "classes_64":  # 63 distinct hostname pins (+ class 0) = 64 classes
        hosts = [nodes[n].selectors["kubernetes.io/hostname"] for n in range(n_nodes - 63, n_nodes)]
        for j, i in enumerate(np.nonzero(pick < 0.3)[0]):
            selectors[i] = {"kubernetes.io/hostname": hosts[j % 63]}
    elif kind == "ulp":
        for i in np.nonzero(pick < 0.5)[0]:
            selectors[i] = {"zone": "z%d" % (i % 3)}
            req[i, 0] = 0.5
    pods = [SimpleNamespace(selectors=s) for s in selectors]
    cls = snapshot.selector_classes(pods, nodes, pools)
    order = list(ORDER)
    pool_match_ordered = cls.pool_match[order]
    return {
        "kind": kind, "D": D, "req": req, "cap_type": cap_type, "node_type": node_type, "used0": used,
        "unit_all": units, "unit_ordered": units[order], "order": order,
        "pool_actual": np.asarray([pools[t].actual_capacity for t in order], dtype=np.int32),
        "pool_max": np.full(T, 1000, dtype=np.int32), "pool_ignored": np.zeros(T, dtype=np.uint8),
        "over_provision": 1, "pod_class": cls.pod_class, "node_match": cls.node_match,
        "pool_match_all": cls.pool_match, "pool_match_ordered": pool_match_ordered, "classes": cls.classes,
        "selectors": selectors, "nodes": nodes, "pools": pools,
    }
