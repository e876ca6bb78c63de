"""Scale-up ticks whose match classes come from node taints and pod tolerations (tests/test_gpu_taints.py).

Every case is a dense tick (the buffers of acsfit_scale_up_sel) in the layout of tests/selector_cases.py -- four pools
visited in cost order pool1, pool0, pool3, pool2, pool3 without nodes, some node rows exactly at or one ulp short of a
fit -- but the nodes carry taints and the pods tolerations, and the classes come from
snapshot.selector_classes(..., taints=True) (pool taints from AgentPool.taints).  Lifecycle and PreferNoSchedule
taints are sprinkled over every case as noise.  Class 0 has no pod in "class0_empty" and "all_intolerant"; in
"noise_only" no taint blocks, so the classes equal those of the selectors alone.
"""
from types import SimpleNamespace

import numpy as np

import selector_cases as sc
from kubernetes_acs_engine_autoscaler_b200 import snapshot
from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool

KINDS = ("first_tainted", "tolerating_only", "class0_empty", "all_intolerant", "ulp", "noise_only")
DIMS = sc.DIMS
GPU = {"key": "sku", "value": "gpu", "effect": "NoSchedule"}
TEAM = {"key": "team", "value": "ml", "effect": "NoExecute"}
NOISE = ([{"key": "node.kubernetes.io/not-ready", "effect": "NoExecute"}],
         [{"key": "node.cloudprovider.kubernetes.io/uninitialized", "value": "true", "effect": "NoSchedule"}],
         [{"key": "soft", "value": "1", "effect": "PreferNoSchedule"}], [])
TOLERATE_GPU = ([{"key": "sku", "operator": "Equal", "value": "gpu"}], [{"key": "sku", "operator": "Exists"}],
                [{"operator": "Exists"}])
INTOLERANT = ([], [{"key": "sku", "operator": "Equal", "value": "cpu"}], [{"key": "soft", "operator": "Exists"}])


def make_case(kind, D, seed=0, n_nodes=300, n_pods=1500):
    rng = np.random.default_rng([seed, D, KINDS.index(kind), 7])
    T = len(sc.POOLS)
    units = np.stack([sc._unit(D, t) for t in range(T)])
    share = (n_nodes // 2, n_nodes // 4, n_nodes - n_nodes // 2 - n_nodes // 4)
    node_pool = np.concatenate([np.full(s, t, dtype=np.int32) for t, s in enumerate(share)])
    # the pool every node of which carries `pool_taints` (and which pool3, without nodes, never gets)
    pool_taints = {"first_tainted": {1: [GPU]}, "tolerating_only": {2: [GPU]}, "class0_empty": {0: [TEAM], 2: [GPU]},
                   "all_intolerant": {0: [GPU], 1: [GPU], 2: [GPU, TEAM]}, "ulp": {0: [TEAM]}, "noise_only": {}}[kind]
    nodes = []
    for n, t in enumerate(node_pool):
        labels = {"agentpool": sc.POOLS[t], "beta.kubernetes.io/instance-type": "type%d" % t,
                  "kubernetes.io/hostname": "k8s-%s-0-%d" % (sc.POOLS[t], n), "zone": "z%d" % (n % 3)}
        taints = list(pool_taints.get(int(t), [])) + list(NOISE[n % len(NOISE)])
        nodes.append(SimpleNamespace(selectors=labels, taints=taints, unschedulable=False))
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
    tolerations = [list(INTOLERANT[i % len(INTOLERANT)]) for i in range(n_pods)]
    if kind == "first_tainted":  # pool1, visited first, is tainted: most pods are ineligible for its bins
        for i in np.nonzero(pick < 0.1)[0]:
            tolerations[i] = list(TOLERATE_GPU[i % 3])
        for i in np.nonzero((pick >= 0.1) & (pick < 0.3))[0]:
            selectors[i] = {"zone": "z%d" % (i % 3)}
    elif kind == "tolerating_only":  # pool2's nodes and bins take only the pods that tolerate sku=gpu
        used[node_pool != 2] = cap_type[node_pool[node_pool != 2]]  # the other nodes are full
        for i in np.nonzero(pick < 0.4)[0]:
            tolerations[i] = list(TOLERATE_GPU[i % 3])
        for i in np.nonzero((pick >= 0.2) & (pick < 0.3))[0]:
            selectors[i] = {"agentpool": "pool2"}
    elif kind == "class0_empty":  # every pod is intolerant of some node: one of the two taints at least
        for i in range(n_pods):
            tolerations[i] = [[TOLERATE_GPU[0][0]], [{"key": "team", "operator": "Exists"}], []][i % 3]
        for i in np.nonzero(pick < 0.2)[0]:
            selectors[i] = {"agentpool": sc.POOLS[i % 3]}
    elif kind == "all_intolerant":  # every node is tainted, nobody tolerates: only pool3 (no node, no taint) is left
        pass
    elif kind == "ulp":  # node rows exactly full for a 0.5-cpu pod, others one ulp short; pool0 tainted
        k = np.arange(0, n_nodes, 5)
        used[k, 0] = cap_type[node_type[k], 0] - 0.5
        used[k[1::2], 0] = np.nextafter(used[k[1::2], 0], np.inf)
        for i in np.nonzero(pick < 0.5)[0]:
            req[i, 0] = 0.5
            if i % 2:
                tolerations[i] = [{"key": "team", "operator": "Equal", "value": "ml", "effect": "NoExecute"}]
            if i % 3 == 0:
                selectors[i] = {"zone": "z%d" % (i % 3)}
    elif kind == "noise_only":  # no blocking taint anywhere: selectors decide alone
        for i in np.nonzero(pick < 0.3)[0]:
            selectors[i] = {"agentpool": sc.POOLS[i % 3]}
    pods = [SimpleNamespace(selectors=s, tolerations=t) for s, t in zip(selectors, tolerations)]
    cls = snapshot.selector_classes(pods, nodes, pools, taints=True)
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
