#!/usr/bin/env python3
"""developer probe: cost of required pod affinity in the node pass (get_pending_pods) at the c2 shape (100 000 pods x
10 000 nodes, D = 4).

Variants: first_fit_nodes_aa with every mask 0, and first_fit_nodes_pa with --share of the pods in self-affine groups
(one signature each) whose signatures are
  present   already on some node: no bootstrap signature, nothing watched, one pass
  flips1    absent, one group: the pass runs again once
  flips8    absent, eight groups: the pass runs again eight times
Median (min) of --reps CUDA-event timings after --warmup untimed rounds, variants interleaved in rotating order, `used`
and the node masks restored before each; prints the GPU and its power limit read in the same run, and the reruns each
variant made.
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # the probe must run where nvidia-smi is absent too
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=100000)
    ap.add_argument("--N", type=int, default=10000)
    ap.add_argument("--D", type=int, default=4)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--share", type=float, default=0.1)
    args = ap.parse_args()

    import torch
    from kubernetes_acs_engine_autoscaler_b200 import synthetic as syn
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    eng = Engine(0)
    c = syn.make_cluster(args.P, args.N, args.D, 1, seed=11)
    f64, i32, i64 = torch.float64, torch.int32, torch.int64
    req, cap, ntype = eng.dev(c["req"], f64), eng.dev(c["cap_type"], f64), eng.dev(c["node_type"], i32)
    used0 = eng.dev(syn.initial_used(c), f64)
    used = used0.clone()
    N, P = used0.shape[0], req.shape[0]
    rng = np.random.default_rng(3)
    zero_p, zero_n = eng.dev(np.zeros(P, np.int64), i64), eng.dev(np.zeros(N, np.int64), i64)
    nc, nx, has = zero_n.clone(), zero_n.clone(), zero_n.clone()

    def groups(k):
        who = rng.random(P) < args.share
        bits = np.where(who, np.uint64(1) << rng.integers(0, k, size=P).astype(np.uint64), np.uint64(0))
        d = eng.dev(bits.view(np.int64), i64)
        return d, d, d  # requires, self, matches: every member matches its own signature
    masks = {"present": groups(8), "flips1": groups(1), "flips8": groups(8)}
    has0 = {"present": np.zeros(N, np.uint64), "flips1": np.zeros(N, np.uint64), "flips8": np.zeros(N, np.uint64)}
    has0["present"][0] = np.uint64(0xFF)  # every signature of the group already on node 0
    has0 = {k: eng.dev(v.view(np.int64), i64) for k, v in has0.items()}

    def pa(name):
        return lambda: eng.first_fit_nodes_pa(req, None, cap, ntype, used, *masks[name], has, zero_p, zero_p, nc, nx)
    runs = {"aa/zero": lambda: eng.first_fit_nodes_aa(req, None, cap, ntype, used, zero_p, zero_p, nc, nx)}
    runs.update({"pa/" + k: pa(k) for k in masks})

    def once(name):
        used.copy_(used0)
        nc.zero_()
        nx.zero_()
        has.copy_(has0.get(name[3:], zero_n))
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = runs[name]()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), out

    print("GPU: %s; P=%d N=%d D=%d, share %.2f, median / min of %d, variants interleaved after %d warm-up rounds" % (
        gpu_info(), P, N, args.D, args.share, args.reps, args.warmup))
    names = list(runs)
    times = {name: [] for name in names}
    outs = {}
    for rep in range(args.warmup + args.reps):
        for k in range(len(names)):  # rotate the order every round: no variant always runs first
            name = names[(rep + k) % len(names)]
            t, out = once(name)
            if rep >= args.warmup:
                times[name].append(t)
            outs[name] = (int((out[0].cpu().numpy() >= 0).sum()), len(eng.last_affinity_reruns())
                          if name.startswith("pa/") else 0, eng.last_launches())
    print("node pass")
    for name in names:
        placed, reruns, rec = outs[name]
        print("  %-11s %8.3f ms  (min %.3f)  placed %d  reruns %d  launches: %s" % (
            name, float(np.median(times[name])), float(np.min(times[name])), placed, reruns,
            ["RW=%d prune=%d stages=%d" % (r["RW"], r["prune"], r["stages"]) for r in rec][:2]))


if __name__ == "__main__":
    main()
