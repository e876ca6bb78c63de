#!/usr/bin/env python3
"""developer probe: cost of the node-taint mode (Cluster(node_taints=True)).

  builder   host time of snapshot.selector_classes(pods, nodes, pools, taints=True) and
            snapshot.pending_match(pods, nodes, taints=True) on KubeNode / KubePod objects: --nodes nodes in 8 pools,
            three of them tainted (plus lifecycle / PreferNoSchedule noise on some nodes), 100 k pending pods whose
            selectors and tolerations make 8 or 64 match signatures.  Best of --reps.  Host only: no GPU needed.
  tick      Cluster.loop_logic() in dry run at the c2 shape (100 k pending pods x 10 k nodes, D = 4) with 10 % of the
            nodes moved into a second pool tainted sku=gpu:NoSchedule and 10 % of the pods tolerating it: node
            selectors + taints against node selectors alone on the same tick, alternated, best and median of --reps
            after one warm-up each; prints the GPU and its power limit (read in the same run).
"""
import argparse
import copy
import datetime
import os
import platform
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot  # noqa: E402
from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool  # noqa: E402

GPU_TAINT = {"key": "sku", "value": "gpu", "effect": "NoSchedule"}
TOLERATE = [{"key": "sku", "operator": "Equal", "value": "gpu", "effect": "NoSchedule"}]


class Obj(object):
    __slots__ = ("obj",)

    def __init__(self, o):
        self.obj = o

    @property
    def name(self):
        return self.obj["metadata"]["name"]


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # the builder part runs where nvidia-smi is absent too
        return "unknown"


def cpu_model():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("model name"):
                    return line.split(":", 1)[1].strip()
    except OSError:
        pass
    return platform.processor() or "unknown"


def builder(n_nodes, signatures, reps):
    pools = ["pool%d" % t for t in range(8)]
    tainted = {"pool5": [GPU_TAINT], "pool6": [GPU_TAINT, {"key": "team", "value": "ml", "effect": "NoExecute"}],
               "pool7": [{"key": "spot", "effect": "NoSchedule"}]}
    noise = [[], [], [{"key": "soft", "value": "1", "effect": "PreferNoSchedule"}],
             [{"key": "node.kubernetes.io/not-ready", "effect": "NoExecute"}]]
    nodes = []
    for i in range(n_nodes):
        pool = pools[i % 8]
        name = "k8s-%s-1-%d" % (pool, i)
        taints = tainted.get(pool, []) + noise[i % 4]
        spec = {"taints": copy.deepcopy(taints)} if taints else {}
        nodes.append(kube.KubeNode(Obj({"metadata": {"name": name, "creationTimestamp": "2026-09-20T07:00:00Z",
                                                      "labels": {"agentpool": pool, "kubernetes.io/hostname": name,
                                                                 "zone": "z%d" % (i % 3)}}, "spec": spec})))
    agent_pools = [AgentPool(p, "Standard_D2_v2", [n for n in nodes if n.selectors["agentpool"] == p]) for p in pools]
    # 8 signatures: no selector / pool pins, with and without the gpu toleration; 64: plus hostname pins into pool1
    kinds = [({}, []), ({}, TOLERATE), ({"agentpool": "pool1"}, []), ({"agentpool": "pool5"}, TOLERATE),
             ({"zone": "z1"}, []), ({"agentpool": "pool6"}, [{"operator": "Exists"}]),
             ({"agentpool": "pool2", "zone": "z0"}, [])]
    while len(kinds) < signatures - 1:  # class 0 (matches everything) has no pod: each kind is one more signature
        kinds.append(({"kubernetes.io/hostname": nodes[8 * len(kinds) + 1].name}, []))
    pods = []
    for j in range(100000):
        sel, tol = kinds[j % len(kinds)]
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": "100m"}}}], "nodeSelector": dict(sel)}
        if tol:
            spec["tolerations"] = copy.deepcopy(tol)
        pods.append(kube.KubePod(Obj({"metadata": {"name": "p%d" % j, "namespace": "ns", "uid": "u%d" % j,
                                                   "creationTimestamp": "2026-09-21T07:00:00Z"},
                                      "spec": spec, "status": {"phase": "Pending"}})))
    out = {}
    for what, fn in (("selector_classes", lambda: snapshot.selector_classes(pods, nodes, agent_pools, taints=True)),
                     ("pending_match", lambda: snapshot.pending_match(pods, nodes, taints=True)),
                     ("selector_classes (selectors alone)", lambda: snapshot.selector_classes(pods, nodes, agent_pools))):
        times = []
        for _ in range(reps):
            t0 = time.perf_counter()
            res = fn()
            times.append(time.perf_counter() - t0)
        out[what] = min(times)
        if what == "selector_classes":
            classes = res.classes
    print("builder  N=%-8d %2d signatures (got %d classes): selector_classes %.3f s, pending_match %.3f s; "
          "selectors alone %.3f s  [best of %d, %s]" % (
              n_nodes, signatures, classes, out["selector_classes"], out["pending_match"],
              out["selector_classes (selectors alone)"], reps, cpu_model()), flush=True)


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
    st = syn.kube_objects(c)
    N = c["N"]
    moved = 0
    for i, o in enumerate(st["nodes"]):  # the last 10 % of the nodes form pool `gpu`, tainted
        if i >= N - N // 10:
            old = o["metadata"]["name"]
            new = old.replace("-pool0-", "-gpu-")
            o["metadata"]["name"] = new
            o["metadata"]["labels"]["kubernetes.io/hostname"] = new
            o["spec"]["taints"] = [dict(GPU_TAINT)]
            moved += 1
    renamed = {o["metadata"]["name"].replace("-gpu-", "-pool0-"): o["metadata"]["name"] for o in st["nodes"]
               if "-gpu-" in o["metadata"]["name"]}
    pending = 0
    for p in st["pods"]:
        nn = p["spec"].get("nodeName")
        if nn in renamed:
            p["spec"]["nodeName"] = renamed[nn]
        if p["status"]["phase"] == "Pending":
            if pending % 10 == 0:
                p["spec"]["tolerations"] = copy.deepcopy(TOLERATE)
            pending += 1
    st["arm_parameters"]["gpuVMSize"] = dict(st["arm_parameters"]["pool0VMSize"])
    nodes, pods = [Obj(o) for o in st["nodes"]], [Obj(o) for o in st["pods"]]
    orig_init = agent_pool.AgentPool.__init__

    def pool_init(self, *a, **k):  # unbounded pools, as bench.py's python_surface
        orig_init(self, *a, **k)
        self.max_size = int(c["pool_max"][0])
    agent_pool.AgentPool.__init__ = pool_init
    logging.disable(logging.CRITICAL)
    clusters = {}
    for name, taints in (("selectors+taints", True), ("selectors alone", False)):
        cl = Cluster(None, 1800, 1, "a", "b", "c", "d", "e", "f", 600, "rg", None, "",
                     over_provision=c["over_provision"], dry_run=True, node_selectors=True, node_taints=taints)
        cl.list_nodes, cl.list_pods = (lambda: nodes), (lambda: pods)
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
    print("tick     c2 (P=%d pending, N=%d nodes, %d in tainted pool `gpu`, 10%% of the pods tolerate it), "
          "Cluster.loop_logic dry run, %d reps alternated after one warm-up:" % (c["P"], N, moved, reps))
    for name in clusters:
        print("  %-18s best %.3f s  median %.3f s  launches %d" % (
            name, min(times[name]), statistics.median(times[name]), launches[name][0]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("part", choices=("builder", "tick", "all"))
    ap.add_argument("--nodes", type=int, nargs="+", default=[100000, 1000000])
    ap.add_argument("--signatures", type=int, nargs="+", default=[8, 64])
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    print("date %s" % datetime.datetime.now(datetime.timezone.utc).isoformat(), flush=True)
    if args.part in ("builder", "all"):
        for n in args.nodes:
            for s in args.signatures:
                builder(n, s, max(1, args.reps // 2))
    if args.part in ("tick", "all"):
        tick(args.reps)


if __name__ == "__main__":
    main()
