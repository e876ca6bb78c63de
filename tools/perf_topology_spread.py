#!/usr/bin/env python3
"""developer probe: cost of hostname topology spread in the node pass (get_pending_pods) and in the bin passes
(fulfill_pending) at the c2 shape (100 000 pods x 10 000 nodes, D = 4), against the pod-affinity form with every mask 0.

Variants (the `_ts` entry points; pod-affinity and anti-affinity masks absent):
  absent    one key that no pod has: the spread test is compiled in but never blocks
  flat      --share of the pods in 8 groups over every node, each minimum held at 0 by its floor: no rise
  rise1     --share of the pods in one group pinned to 8 nodes (count 1 on each; the nodes where most of the group lands
            without the rule), floor 2: one rise
  rises     the same group with no floor: the minimum rises as often as the pods fill those nodes (capped by --max-rises
            through the floor)
The bin passes take the pods the `pa` node pass left pending, with the variant's keys.  Median (min) of --reps
CUDA-event timings after --warmup untimed rounds, variants interleaved in rotating order, `used` and the counts restored
before each; prints the GPU, its power limit and maximum SM clock read in the same run, and the rises each variant
fixed.
"""
import argparse
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
INT32_MAX = 2 ** 31 - 1


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", "0"], capture_output=True, text=True, timeout=30).stdout.strip()
        return out or "unknown"
    except Exception:  # the probe must run where nvidia-smi is absent too
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--P", type=int, default=100000)
    ap.add_argument("--N", type=int, default=10000)
    ap.add_argument("--D", type=int, default=4)
    ap.add_argument("--reps", type=int, default=11)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--share", type=float, default=0.1)
    ap.add_argument("--max-rises", type=int, default=16)
    args = ap.parse_args()

    import torch
    from kubernetes_acs_engine_autoscaler_b200 import synthetic as syn
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    eng = Engine(0)
    c = syn.make_cluster(args.P, args.N, args.D, 1, seed=11)
    f64, i32, i64, u8 = torch.float64, torch.int32, torch.int64, torch.uint8
    req, cap, ntype = eng.dev(c["req"], f64), eng.dev(c["cap_type"], f64), eng.dev(c["node_type"], i32)
    used0_h = syn.initial_used(c)
    used0 = eng.dev(used0_h, f64)
    used = used0.clone()
    N, P = used0.shape[0], req.shape[0]
    rng = np.random.default_rng(3)
    zero_p, zero_n = eng.dev(np.zeros(P, np.int64), i64), eng.dev(np.zeros(N, np.int64), i64)
    has = zero_n.clone()
    # the plain node pass: where would each pod land without the rule?
    free, _ = eng.first_fit_nodes_pa(req, None, cap, ntype, used, zero_p, zero_p, zero_p, has)
    free = free.cpu().numpy()
    group = rng.random(P) < args.share  # the pinned group of rise1 / rises

    def pinned_nodes():
        landed = np.bincount(free[group & (free >= 0)], minlength=N)
        return np.argsort(-landed, kind="stable")[:8]
    pinned = pinned_nodes()

    def spread(kind):
        """(keys, pod_key, pod_skew, pod_matches, node_count, node_domain, floor) as host arrays"""
        key = np.full(P, 0xFF, np.uint8)
        skew = np.zeros(P, np.int32)
        match = np.zeros(P, np.uint64)
        if kind == "absent":
            return 1, key, skew, match, np.zeros((1, N), np.int32), np.full(N, 1, np.uint64), np.zeros(1, np.int32)
        who = rng.random(P) < args.share if kind == "flat" else group
        K = 8 if kind == "flat" else 1
        g = rng.integers(0, K, size=P)
        key[who] = g[who]
        match[who] = np.uint64(1) << g[who].astype(np.uint64)
        count = np.zeros((K, N), np.int32)
        domain = np.full(N, (1 << K) - 1, np.uint64)
        if kind == "flat":
            floor = np.zeros(K, np.int32)
        else:
            domain[:] = 0
            domain[pinned] = 1
            count[0, pinned] = 1
            floor = np.full(1, 2 if kind == "rise1" else 1 + args.max_rises, np.int32)
        return K, key, skew, match, count, domain, floor
    kinds = ["absent", "flat", "rise1", "rises"]
    host = {k: spread(k) for k in kinds}
    dev = {k: (h[0], eng.dev(h[1], u8), eng.dev(h[2], i32), eng.dev(h[3].view(np.int64), i64), eng.dev(h[4], i32),
               eng.dev(h[5].view(np.int64), i64), h[6]) for k, h in host.items()}
    counts = {k: d[4].clone() for k, d in dev.items()}

    def node_pass(name):
        if name == "pa":
            return eng.first_fit_nodes_pa(req, None, cap, ntype, used, zero_p, zero_p, zero_p, has)
        K, key, skew, match, _, dom, floor = dev[name]
        return eng.first_fit_nodes_ts(req, None, cap, ntype, used, K, key, skew, match, counts[name], dom, floor)

    def once(fn, name):
        used.copy_(used0)
        has.zero_()
        if name in counts:
            counts[name].copy_(dev[name][4])
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = fn(name)
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b), out

    def measure(fn, names):
        times = {name: [] for name in names}
        extra = {}
        for rep in range(args.warmup + args.reps):
            for k in range(len(names)):  # rotate the order every round: no variant always runs first
                name = names[(rep + k) % len(names)]
                t, out = once(fn, name)
                if rep >= args.warmup:
                    times[name].append(t)
                extra[name] = (out, len(eng.last_spread_rises()) if name != "pa" else 0)
        return times, extra

    print("GPU: %s; P=%d N=%d D=%d, share %.2f, median / min of %d, variants interleaved after %d warm-up rounds" % (
        gpu_info(), P, N, args.D, args.share, args.reps, args.warmup))
    names = ["pa"] + kinds
    times, extra = measure(node_pass, names)
    print("node pass")
    for name in names:
        out, rises = extra[name]
        print("  %-7s %9.3f ms  (min %.3f)  placed %d  rises %d" % (
            name, float(np.median(times[name])), float(np.min(times[name])), int((out[0].cpu().numpy() >= 0).sum()),
            rises))

    # the bins: the pods the plain node pass left pending, one pool
    used.copy_(used0)
    placed, _ = eng.first_fit_nodes_pa(req, None, cap, ntype, used, zero_p, zero_p, zero_p, has)
    pend = np.nonzero(placed.cpu().numpy() < 0)[0]
    preq = eng.dev(c["req"][pend], f64)
    unit = c["unit_ordered"][:1]
    pools = (np.zeros(1, np.int32), np.full(1, 1 << 30, np.int32), np.zeros(1, np.uint8))
    zq = eng.dev(np.zeros(len(pend), np.int64), i64)
    bins = {k: (h[0], eng.dev(h[1][pend], u8), eng.dev(h[2][pend], i32), eng.dev(h[3][pend].view(np.int64), i64))
            for k, h in host.items()}

    def bin_pass(name):
        if name == "pa":
            return eng.fulfill_pending_pa(preq, len(pend), unit, *pools, 0, zq, zq, zq)
        return eng.fulfill_pending_ts(preq, len(pend), unit, *pools, 0, *bins[name])
    names = ["pa", "absent", "flat", "rises"]
    times, extra = measure(bin_pass, names)
    print("bin passes (%d pending pods)" % len(pend))
    for name in names:
        out, _ = extra[name]
        print("  %-7s %9.3f ms  (min %.3f)  bins %d" % (name, float(np.median(times[name])), float(np.min(times[name])),
                                                      int(out["bins_opened"].sum())))


if __name__ == "__main__":
    main()
