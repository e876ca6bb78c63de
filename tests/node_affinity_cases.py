"""Scale-up ticks whose match classes come from required node affinity (tests/test_gpu_node_affinity.py).

Every case is a dense tick (the buffers of acsfit_scale_up_sel) in the layout of tests/selector_cases.py -- four pools
visited in cost order pool1, pool0, pool3, pool2, pool3 without nodes, some node rows exactly at or one ulp short of a
fit -- but the pods carry required node affinity, and the classes come from
snapshot.selector_classes(..., taints=True, affinity=True).  Nodes carry a numeric label `gen` of any shape (integers
with a sign or leading zeros, non-integers, absent).  In "first_avoided" most pods may not use pool1, the first pool
visited; "daemonset" pods are pinned to one existing node by matchFields, so they match no pool; "with_taints" adds a
tainted pool; in "no_affinity" no pod has the field, so the classes equal those of selectors and taints alone.
"""
from types import SimpleNamespace

import numpy as np

import selector_cases as sc
from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot
from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool

KINDS = ("first_avoided", "pool_targeted", "numeric", "daemonset", "hostname_not_in", "with_taints", "ulp",
         "no_affinity")
DIMS = sc.DIMS
GEN = ("0", "1", "2", "3", "+4", "-1", "007", "x", "1_0", None)
GPU = {"key": "sku", "value": "gpu", "effect": "NoSchedule"}


def R(key, op, *values):
    return {"key": key, "operator": op, "values": list(values)} if values else {"key": key, "operator": op}


def required(*terms):
    return {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": list(terms)}}}


def make_case(kind, D, seed=0, n_nodes=300, n_pods=1500):
    rng = np.random.default_rng([seed, D, KINDS.index(kind), 13])
    T = len(sc.POOLS)
    units = np.stack([sc._unit(D, t) for t in range(T)])
    share = (n_nodes // 2, n_nodes // 4, n_nodes - n_nodes // 2 - n_nodes // 4)
    node_pool = np.concatenate([np.full(s, t, dtype=np.int32) for t, s in enumerate(share)])
    nodes = []
    for n, t in enumerate(node_pool):
        name = "k8s-%s-0-%d" % (sc.POOLS[t], n)
        labels = {"agentpool": sc.POOLS[t], "beta.kubernetes.io/instance-type": "type%d" % t,
                  "kubernetes.io/hostname": name, "zone": "z%d" % (n % 3)}
        gen = GEN[n % len(GEN)]
        if gen is not None:
            labels["gen"] = gen
        taints = [GPU] if kind == "with_taints" and t == 2 else []
        nodes.append(SimpleNamespace(selectors=labels, taints=taints, unschedulable=False, name=name))
    pools = [AgentPool(sc.POOLS[t], "type%d" % t, [nodes[n] for n in np.nonzero(node_pool == t)[0]]) for t in range(T)]
    cap_type = units[:3].copy()
    node_type = node_pool.copy()
    used = cap_type[node_type] * rng.uniform(0.0, 0.9, size=(n_nodes, 1))
    used[:, 2:] = 0.0
    req = np.zeros((n_pods, D))
    req[:, 0] = rng.choice([0.1, 0.25, 0.5, 1.0, 2.0, 6.0], size=n_pods, p=[.3, .25, .2, .15, .07, .03])
    req[:, 1] = rng.choice([0.5, 1.0, 2.0, 4.0, 12.0], size=n_pods) * 2 ** 30
    if D > 2:
        req[:, 2] = 1.0
    pick = rng.random(n_pods)
    selectors = [{} for _ in range(n_pods)]
    tolerations = [[] for _ in range(n_pods)]
    affinity = [None] * n_pods
    if kind == "first_avoided":  # pool1, visited first, is avoided by most pods: most are ineligible for its bins
        for i in np.nonzero(pick < 0.7)[0]:
            affinity[i] = required({"matchExpressions": [R("agentpool", "NotIn", "pool1")]})
        for i in np.nonzero((pick >= 0.7) & (pick < 0.8))[0]:
            selectors[i] = {"zone": "z%d" % (i % 3)}
    elif kind == "pool_targeted":  # pool2's nodes and bins (or pool3's bins) take only the pods that target them
        used[node_pool != 2] = cap_type[node_pool[node_pool != 2]]  # the other nodes are full
        for i in np.nonzero(pick < 0.4)[0]:
            affinity[i] = required({"matchExpressions": [R("agentpool", "In", "pool2", "pool3")]})
        for i in np.nonzero((pick >= 0.4) & (pick < 0.5))[0]:
            affinity[i] = required({"matchExpressions": [R("beta.kubernetes.io/instance-type", "In", "type3")]})
    elif kind == "numeric":  # Gt / Lt on `gen`, ORed with a pool term
        for i in np.nonzero(pick < 0.5)[0]:
            affinity[i] = required({"matchExpressions": [R("gen", "Gt", "1")]},
                                   {"matchExpressions": [R("agentpool", "In", "pool3")]}) if i % 2 else \
                required({"matchExpressions": [R("gen", "Lt", "+3"), R("zone", "NotIn", "z0")]})
    elif kind == "daemonset":  # pinned to an existing node by name: no pool can host them
        for i in np.nonzero(pick < 0.2)[0]:
            affinity[i] = required({"matchFields": [{"key": "metadata.name", "operator": "In",
                                                     "values": [nodes[(i * 7) % 40].name]}]})
    elif kind == "hostname_not_in":  # each avoids one of 40 nodes by hostname: one projection per such node
        for i in np.nonzero(pick < 0.5)[0]:
            affinity[i] = required({"matchExpressions": [R("kubernetes.io/hostname", "NotIn", nodes[i % 40].name),
                                                         R("agentpool", "Exists")]})
    elif kind == "with_taints":  # pool2 tainted: the pods that target it through affinity tolerate the taint or not
        for i in np.nonzero(pick < 0.4)[0]:
            affinity[i] = required({"matchExpressions": [R("agentpool", "In", "pool2")]})
            if i % 2:
                tolerations[i] = [{"key": "sku", "operator": "Exists"}]
        for i in np.nonzero((pick >= 0.4) & (pick < 0.5))[0]:
            selectors[i] = {"zone": "z%d" % (i % 3)}
    elif kind == "ulp":  # node rows exactly full for a 0.5-cpu pod, others one ulp short; pods avoid pool0
        k = np.arange(0, n_nodes, 5)
        used[k, 0] = cap_type[node_type[k], 0] - 0.5
        used[k[1::2], 0] = np.nextafter(used[k[1::2], 0], np.inf)
        for i in np.nonzero(pick < 0.5)[0]:
            req[i, 0] = 0.5
            if i % 2:
                affinity[i] = required({"matchExpressions": [R("agentpool", "NotIn", "pool0")]})
    elif kind == "no_affinity":  # selectors and taint-free pods only
        for i in np.nonzero(pick < 0.3)[0]:
            selectors[i] = {"agentpool": sc.POOLS[i % 3]}
    pods = [SimpleNamespace(selectors=s, tolerations=t, node_affinity=kube.node_affinity_terms(a, "pod %d" % i))
            for i, (s, t, a) in enumerate(zip(selectors, tolerations, affinity))]
    cls = snapshot.selector_classes(pods, nodes, pools, taints=True, affinity=True)
    order = list(sc.ORDER)
    return {
        "kind": kind, "D": D, "req": req, "cap_type": cap_type, "node_type": node_type, "used0": used,
        "unit_all": units, "unit_ordered": units[order], "order": order,
        "pool_actual": np.asarray([pools[t].actual_capacity for t in order], dtype=np.int32),
        "pool_max": np.full(T, 1000, dtype=np.int32), "pool_ignored": np.zeros(T, dtype=np.uint8),
        "over_provision": 1, "pod_class": cls.pod_class, "node_match": cls.node_match,
        "pool_match_all": cls.pool_match, "pool_match_ordered": cls.pool_match[order], "classes": cls.classes,
        "selectors": selectors, "nodes": nodes, "pools": pools, "pods": pods,
    }
