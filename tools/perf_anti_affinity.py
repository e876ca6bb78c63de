#!/usr/bin/env python3
"""developer probe: cost of required pod anti-affinity.

  kernels   the node pass (get_pending_pods) and the bin packing of its pending pods (fulfill_pending, one pool) at the
            c2 shape (100 000 pods x 10 000 nodes, D = 4), four ways: the plain kernel, SEL with every pod in class 0,
            AA with every mask 0, and AA with --share of the pods in --groups self-anti-affine deployments.  Median of
            --reps CUDA-event timings after --warmup untimed rounds, variants interleaved in rotating order, `used` and
            the node masks restored before each; prints the GPU and its power limit read in the same run.
  builder   host time of snapshot.anti_affinity for --pods pods to schedule and --running running pods (CPU only),
            with --groups deployments whose terms are kept and --lone-terms running pods that each carry a term of
            their own that selects only themselves (carried, never relevant: dropped before numbering).
"""
import argparse
import os
import subprocess
import sys
import time
from types import SimpleNamespace

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


def kernels(args):
    import torch
    from kubernetes_acs_engine_autoscaler_b200 import synthetic as syn
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    eng = Engine(0)
    c = syn.make_cluster(args.P, args.N, args.D, 1, seed=11)
    f64, i32, u8, i64 = torch.float64, torch.int32, torch.uint8, torch.int64
    req, cap, ntype = eng.dev(c["req"], f64), eng.dev(c["cap_type"], f64), eng.dev(c["node_type"], i32)
    used0 = eng.dev(syn.initial_used(c), f64)
    used = used0.clone()
    N, P = used0.shape[0], req.shape[0]
    rng = np.random.default_rng(3)
    who = rng.random(P) < args.share
    bits = np.where(who, np.uint64(1) << rng.integers(0, args.groups, size=P).astype(np.uint64), np.uint64(0))
    zero_p, zero_n = eng.dev(np.zeros(P, np.int64), i64), eng.dev(np.zeros(N, np.int64), i64)
    d_bits = eng.dev(bits.view(np.int64), i64)
    nc, nx = zero_n.clone(), zero_n.clone()
    cls0, match1 = eng.dev(np.zeros(P, np.uint8), u8), eng.dev(np.ones(N, np.int64), i64)
    unit = c["unit_ordered"][:1]
    pool = (np.array([0], np.int32), np.array([1 << 30], np.int32), np.array([0], np.uint8))

    def once(fn):
        used.copy_(used0)
        nc.zero_()
        nx.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), out

    nodes = {
        "plain": lambda: eng.first_fit_nodes(req, None, cap, ntype, used),
        "sel/c0": lambda: eng.first_fit_nodes_sel(req, None, cap, ntype, used, cls0, match1, 1),
        "aa/zero": lambda: eng.first_fit_nodes_aa(req, None, cap, ntype, used, zero_p, zero_p, nc, nx),
        "aa/%d%%" % round(100 * args.share): lambda: eng.first_fit_nodes_aa(req, None, cap, ntype, used, d_bits,
                                                                            d_bits, nc, nx),
    }
    print("GPU: %s; P=%d N=%d D=%d, median / min of %d, variants interleaved after %d warm-up rounds" % (
        gpu_info(), P, N, args.D, args.reps, args.warmup))
    # the bin pass packs the pods the plain node pass leaves pending (the same pods for every variant)
    _, (placed, _) = once(nodes["plain"])
    pend = np.nonzero(placed.cpu().numpy() < 0)[0]
    if len(pend) < 1000:  # too few to time a bin pass: pack a tenth of all pods instead
        pend = np.arange(0, P, 10)
    preq = eng.dev(c["req"][pend], f64)
    pz, pb = zero_p[:len(pend)].contiguous(), eng.dev(bits[pend].view(np.int64), i64)
    bins = {
        "plain": lambda: eng.fulfill_pending(preq, len(pend), unit, *pool, 0),
        "sel/c0": lambda: eng.fulfill_pending_sel(preq, len(pend), unit, *pool, 0, cls0[:len(pend)].contiguous(),
                                                  np.ones(1, np.uint64), 1),
        "aa/zero": lambda: eng.fulfill_pending_aa(preq, len(pend), unit, *pool, 0, pz, pz),
        "aa/%d%%" % round(100 * args.share): lambda: eng.fulfill_pending_aa(preq, len(pend), unit, *pool, 0, pb, pb),
    }
    for what, runs in (("node pass", nodes), ("bin pass (%d pods)" % len(pend), bins)):
        names = list(runs)
        times = {name: [] for name in names}
        outs = {}
        for rep in range(args.warmup + args.reps):
            for k in range(len(names)):  # rotate the order every round: no variant always runs first
                name = names[(rep + k) % len(names)]
                t, out = once(runs[name])
                if rep >= args.warmup:
                    times[name].append(t)
                outs[name] = (out, eng.last_launches())
        print(what)
        for name in names:
            out, rec = outs[name]
            got = out[0] if isinstance(out, tuple) else out["bins_opened"]
            summary = "placed %d" % int((got.cpu().numpy() >= 0).sum()) if isinstance(out, tuple) else \
                "bins %d" % int(got[0])
            print("  %-8s %8.3f ms  (min %.3f)  %s  launches: %s" % (
                name, float(np.median(times[name])), float(np.min(times[name])), summary,
                ["RW=%d prune=%d form=%d stages=%d" % (r["RW"], r["prune"], r["form"], r["stages"]) for r in rec][:2]))


def builder(args):
    from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot
    rng = np.random.default_rng(5)
    terms = [kube.anti_affinity_terms({"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
        {"topologyKey": "kubernetes.io/hostname", "labelSelector": {"matchLabels": {"app": "d%d" % g}}}]}}, "ns",
        "probe") for g in range(args.groups)]
    apps = rng.integers(0, 4 * args.groups, size=args.pods + args.running)
    aff = rng.random(args.pods + args.running) < args.share

    lone = [kube.anti_affinity_terms({"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
        {"topologyKey": "kubernetes.io/hostname", "labelSelector": {"matchLabels": {"solo": "s%d" % k}}}]}}, "ns",
        "probe") for k in range(args.lone_terms)]

    def pod(i, node=None):
        a, k = int(apps[i]), i - args.pods
        labels = {"app": "d%d" % a, "tier": "t%d" % (i % 3)}
        own = terms[a] if aff[i] and a < args.groups else ()
        if 0 <= k < args.lone_terms:
            labels["solo"] = "s%d" % k
            own = lone[k]
        return SimpleNamespace(namespace="ns", labels=labels, node_name=node, anti_affinity_terms=own)
    nodes = [SimpleNamespace(name="n%d" % n) for n in range(args.nodes)]
    sched = [pod(i) for i in range(args.pods)]
    running = [pod(args.pods + i, "n%d" % (i % args.nodes)) for i in range(args.running)]
    t0 = time.perf_counter()
    aa = snapshot.anti_affinity(sched, nodes, running)
    dt = time.perf_counter() - t0
    print("builder: %d pods to schedule, %d running pods on %d nodes, %d + %d lone terms carried, %d kept: %.2f s "
          "(one CPU core)" % (args.pods, args.running, args.nodes, args.groups, args.lone_terms, len(aa.terms), dt))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", choices=("kernels", "builder"))
    ap.add_argument("--P", type=int, default=100000)
    ap.add_argument("--N", type=int, default=10000)
    ap.add_argument("--D", type=int, default=4)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--share", type=float, default=0.1)
    ap.add_argument("--groups", type=int, default=32)
    ap.add_argument("--pods", type=int, default=100000)
    ap.add_argument("--running", type=int, default=1000000)
    ap.add_argument("--nodes", type=int, default=100000)
    ap.add_argument("--lone-terms", type=int, default=0)
    args = ap.parse_args()
    kernels(args) if args.what == "kernels" else builder(args)


if __name__ == "__main__":
    main()
