#!/usr/bin/env python3
"""developer probe: cost of the node-affinity mode (Cluster(node_affinity=True)).

  builder   host time of snapshot.selector_classes(pods, nodes, pools, affinity=True) and
            snapshot.pending_match(pods, nodes, affinity=True) on KubeNode / KubePod objects: --nodes nodes in 8 pools,
            100 k pending pods whose required node affinities make 8 or 64 match signatures (pool targeting, NotIn,
            Gt on a numeric label, and with --hostname-not-in also `kubernetes.io/hostname NotIn [node]` terms, one
            projection per such node).  Against the same signatures written as nodeSelectors (pool pins; hostname pins
            for the hostname terms), selectors alone.  Best of --reps.  Host only: no GPU needed.
  tick      Cluster.loop_logic() in dry run at the c2 shape (100 k pending pods x 10 k nodes, D = 4) with 10 % of the
            nodes moved into a second pool `gpu` and 10 % of the pending pods targeting it through `agentpool In [gpu]`,
            against the same pods pinned with nodeSelector {agentpool: gpu}; alternated, best and median of --reps after
            one warm-up each, with the launch counts; prints the GPU and its power limit (read in the same run).
"""
import argparse
import copy
import datetime
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot  # noqa: E402
from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool  # noqa: E402
from perf_taints import Obj, cpu_model, gpu_info  # noqa: E402

HOST = "kubernetes.io/hostname"


def required(*exprs):
    return {"nodeAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": {"nodeSelectorTerms": [
        {"matchExpressions": [dict(zip(("key", "operator", "values"), e)) for e in exprs]}]}}}


def make_nodes(n_nodes):
    pools = ["pool%d" % t for t in range(8)]
    nodes = []
    for i in range(n_nodes):
        pool = pools[i % 8]
        name = "k8s-%s-1-%d" % (pool, i)
        nodes.append(kube.KubeNode(Obj({"metadata": {"name": name, "creationTimestamp": "2026-09-20T07:00:00Z",
                                                      "labels": {"agentpool": pool, HOST: name, "zone": "z%d" % (i % 3),
                                                                 "gen": str(i % 7)}}, "spec": {}})))
    agent_pools = [AgentPool(p, "Standard_D2_v2", [n for n in nodes if n.selectors["agentpool"] == p]) for p in pools]
    return nodes, agent_pools


def make_pods(nodes, signatures, hostname_not_in):
    """(pods with affinity, the same signatures as nodeSelector pods)"""
    kinds = [(required(("zone", "In", ["z2"])), {"zone": "z2"}),
             (required(("agentpool", "In", ["pool1"])), {"agentpool": "pool1"}),
             (required(("agentpool", "In", ["pool5"])), {"agentpool": "pool5"}),
             (required(("zone", "In", ["z1"])), {"zone": "z1"}),
             (required(("agentpool", "NotIn", ["pool0", "pool1", "pool2", "pool3", "pool4", "pool5", "pool7"])),
              {"agentpool": "pool6"}),
             (required(("agentpool", "In", ["pool2"]), ("zone", "In", ["z0"])), {"agentpool": "pool2", "zone": "z0"}),
             (required(("gen", "Gt", ["5"])), {"gen": "6"})]
    while len(kinds) < signatures - 1:  # class 0 (matches everything) has no pod: each kind is one more signature
        name = nodes[8 * len(kinds) + 1].name
        if hostname_not_in:
            kinds.append((required((HOST, "NotIn", [name]), ("agentpool", "In", ["pool1"])), {HOST: name}))
        else:
            kinds.append((required((HOST, "In", [name])), {HOST: name}))
    by_aff, by_sel = [], []
    for j in range(100000):
        a, sel = kinds[j % len(kinds)]
        for out, spec_extra in ((by_aff, {"affinity": copy.deepcopy(a)}),
                                (by_sel, {"nodeSelector": dict(sel)})):
            spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "100m"}}}], **spec_extra}
            out.append(kube.KubePod(Obj({"metadata": {"name": "p%d" % j, "namespace": "ns", "uid": "u%d" % j,
                                                      "creationTimestamp": "2026-09-21T07:00:00Z"},
                                         "spec": spec, "status": {"phase": "Pending"}})))
    return by_aff, by_sel


def best(fn, reps):
    times, res = [], None
    for _ in range(reps):
        t0 = time.perf_counter()
        res = fn()
        times.append(time.perf_counter() - t0)
    return min(times), res


def builder(n_nodes, signature_counts, reps):
    nodes, agent_pools = make_nodes(n_nodes)
    for signatures in signature_counts:
        for hostname_not_in in (False, True):
            by_aff, by_sel = make_pods(nodes, signatures, hostname_not_in)
            t_cls, cls = best(lambda: snapshot.selector_classes(by_aff, nodes, agent_pools, affinity=True), reps)
            t_pm, _ = best(lambda: snapshot.pending_match(by_aff, nodes, affinity=True), reps)
            s_cls, scls = best(lambda: snapshot.selector_classes(by_sel, nodes, agent_pools), reps)
            s_pm, _ = best(lambda: snapshot.pending_match(by_sel, nodes), reps)
            print("builder  N=%-8d %2d signatures%s (%d / %d classes): affinity selector_classes %.3f s, "
                  "pending_match %.3f s; selectors alone %.3f s, %.3f s  [best of %d, %s]" % (
                      n_nodes, signatures, " + hostname NotIn" if hostname_not_in else "", cls.classes, scls.classes,
                      t_cls, t_pm, s_cls, s_pm, reps, cpu_model()), flush=True)


def tick(reps):
    import logging
    import torch
    from kubernetes_acs_engine_autoscaler_b200 import agent_pool
    from kubernetes_acs_engine_autoscaler_b200 import synthetic as syn
    from kubernetes_acs_engine_autoscaler_b200.cluster import Cluster
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    print("GPU: %s" % gpu_info(), flush=True)
    eng = snapshot.set_engine(Engine(0))
    c = syn.make_cluster(100000, 10000, 4, 1, seed=0)
    base = syn.kube_objects(c)
    N = c["N"]
    renamed = {}
    for i, o in enumerate(base["nodes"]):  # the last 10 % of the nodes form pool `gpu`
        if i >= N - N // 10:
            old = o["metadata"]["name"]
            new = old.replace("-pool0-", "-gpu-")
            o["metadata"]["name"] = new
            o["metadata"]["labels"][HOST] = new
            renamed[old] = new
        o["metadata"]["labels"]["agentpool"] = o["metadata"]["name"].split("-")[1]
    for p in base["pods"]:
        nn = p["spec"].get("nodeName")
        if nn in renamed:
            p["spec"]["nodeName"] = renamed[nn]
    base["arm_parameters"]["gpuVMSize"] = dict(base["arm_parameters"]["pool0VMSize"])
    states = {}
    for name in ("affinity", "nodeSelector"):
        st = copy.deepcopy(base)
        pending = 0
        for p in st["pods"]:
            if p["status"]["phase"] == "Pending":
                if pending % 10 == 0:
                    if name == "affinity":
                        p["spec"]["affinity"] = required(("agentpool", "In", ["gpu"]))
                    else:
                        p["spec"]["nodeSelector"] = {"agentpool": "gpu"}
                pending += 1
        states[name] = st
    orig_init = agent_pool.AgentPool.__init__

    def pool_init(self, *a, **k):  # unbounded pools, as bench.py's python_surface
        orig_init(self, *a, **k)
        self.max_size = int(c["pool_max"][0])
    agent_pool.AgentPool.__init__ = pool_init
    logging.disable(logging.CRITICAL)
    clusters = {}
    for name, st in states.items():
        cl = Cluster(None, 1800, 1, "a", "b", "c", "d", "e", "f", 600, "rg", None, "",
                     over_provision=c["over_provision"], dry_run=True, node_selectors=True,
                     node_affinity=name == "affinity")
        nodes, pods = [Obj(o) for o in st["nodes"]], [Obj(o) for o in st["pods"]]
        cl.list_nodes, cl.list_pods = (lambda nodes=nodes: nodes), (lambda pods=pods: pods)
        cl.arm_template, cl.arm_parameters = {}, st["arm_parameters"]
        clusters[name] = cl
    times = {name: [] for name in clusters}
    launches = {}
    try:
        for rep in range(reps + 1):
            names = list(clusters) if rep % 2 == 0 else list(reversed(list(clusters)))
            for name in names:
                n0 = eng.launch_count
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                assert clusters[name].loop_logic()
                torch.cuda.synchronize()
                dt = time.perf_counter() - t0
                launches[name] = (eng.launch_count - n0, [r["pass"] for r in eng.last_launches()])
                if rep:
                    times[name].append(dt)
    finally:
        logging.disable(logging.NOTSET)
        agent_pool.AgentPool.__init__ = orig_init
    print("tick     c2 (P=%d pods, N=%d nodes, %d in pool `gpu`, 10%% of the pending pods target it), "
          "Cluster.loop_logic dry run, %d reps alternated after one warm-up:" % (c["P"], N, len(renamed), reps))
    for name in clusters:
        print("  %-13s best %.3f s  median %.3f s  launches %d %s" % (
            name, min(times[name]), statistics.median(times[name]), launches[name][0], launches[name][1]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("part", choices=("builder", "tick", "all"))
    ap.add_argument("--nodes", type=int, nargs="+", default=[100000, 1000000])
    ap.add_argument("--signatures", type=int, nargs="+", default=[8, 64])
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    print("date %s" % datetime.datetime.now(datetime.timezone.utc).isoformat(), flush=True)
    if args.part in ("tick", "all"):
        tick(args.reps)
    if args.part in ("builder", "all"):
        for n in args.nodes:
            builder(n, args.signatures, max(1, args.reps // 2))


if __name__ == "__main__":
    main()
