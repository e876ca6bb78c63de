#!/usr/bin/env python3
"""developer probe: cost of the node-selector form of the node pass (get_pending_pods) at the c2 shape
(100 000 pods x 10 000 nodes, D = 4) with 4 pools, three ways:
  plain      acsfit_first_fit_nodes
  sel/c0     acsfit_first_fit_nodes_sel with every pod in class 0 (the SEL kernel, nothing pinned)
  sel/30%    acsfit_first_fit_nodes_sel with ~30 % of the pods pinned across 3 classes (one pool's nodes each)
Median of --reps CUDA-event timings of the call after --warmup untimed rounds, the three variants interleaved in
rotating order, `used` restored before each; prints the GPU and its power limit."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from kubernetes_acs_engine_autoscaler_b200 import synthetic as syn  # noqa: E402
from kubernetes_acs_engine_autoscaler_b200.engine import Engine  # noqa: E402


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
    ap.add_argument("--T", type=int, default=4)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--pinned", type=float, default=0.3)
    args = ap.parse_args()
    eng = Engine(0)
    c = syn.make_cluster(args.P, args.N, args.D, args.T, seed=11)
    f64, i32, u8, i64 = torch.float64, torch.int32, torch.uint8, torch.int64
    req, cap, ntype = eng.dev(c["req"], f64), eng.dev(c["cap_type"], f64), eng.dev(c["node_type"], i32)
    used0 = eng.dev(syn.initial_used(c), f64)
    used = used0.clone()
    N, P = used0.shape[0], req.shape[0]
    rng = np.random.default_rng(3)
    # classes 1..3 each match the nodes of one pool (node_pool), class 0 matches everything
    node_pool = np.asarray(c["node_pool"])
    node_match = np.ones(N, dtype=np.uint64)
    for k in (1, 2, 3):
        node_match[node_pool == (k - 1) % args.T] |= np.uint64(1 << k)
    cls0 = np.zeros(P, dtype=np.uint8)
    cls3 = np.where(rng.random(P) < args.pinned, rng.integers(1, 4, size=P), 0).astype(np.uint8)
    d_match = eng.dev(node_match.view(np.int64), i64)
    d_cls0, d_cls3 = eng.dev(cls0, u8), eng.dev(cls3, u8)

    def once(fn):
        used.copy_(used0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), out

    runs = {
        "plain": lambda: eng.first_fit_nodes(req, None, cap, ntype, used),
        "sel/c0": lambda: eng.first_fit_nodes_sel(req, None, cap, ntype, used, d_cls0, d_match, 4),
        "sel/%d%%" % round(100 * args.pinned):
            lambda: eng.first_fit_nodes_sel(req, None, cap, ntype, used, d_cls3, d_match, 4),
    }
    print("GPU: %s; P=%d N=%d D=%d T=%d, median / min of %d, variants interleaved after %d warm-up rounds" % (
        gpu_info(), P, N, args.D, args.T, args.reps, args.warmup))
    names = list(runs)
    times = {name: [] for name in names}
    outs = {}
    for rep in range(args.warmup + args.reps):
        for k in range(len(names)):  # rotate the order every round: no variant always runs first
            name = names[(rep + k) % len(names)]
            t, out = once(runs[name])
            if rep >= args.warmup:
                times[name].append(t)
            outs[name] = (out, eng.last_launches(), eng.last_sel_hits())
    for name in names:
        out, rec, hits = outs[name]
        placed = out[0].cpu().numpy()
        print("%-8s %8.3f ms  (min %.3f)  placed %d  scan hits %d  node pass: RW=%d prune=%d form=%d stages=%d" % (
            name, float(np.median(times[name])), float(np.min(times[name])), int((placed >= 0).sum()), hits,
            rec[0]["RW"], rec[0]["prune"], rec[0]["form"], rec[0]["stages"]))

if __name__ == "__main__":
    main()
