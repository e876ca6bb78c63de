#!/usr/bin/env python3
"""developer probe: cost of node states with pod anti-affinity, pod affinity and hostname topology spread
(Cluster(anti_affinity_node_states=True), Cluster(pod_affinity_node_states=True),
Cluster(topology_spread_node_states=True)).

  kernel   for each form of --forms (`aa`: acsfit_pending_admit; `pa`: acsfit_pending_admit_pa without the anti-affinity
           masks; `aa+pa`: acsfit_pending_admit_pa with them; `ts`: acsfit_pending_admit_ts with the spread test alone;
           `aa+pa+ts`: acsfit_pending_admit_ts with all three tests) at --nodes nodes holding --rows running-pod rows,
           for each U of --sigs, on two tables: `typical` (signature u carries, is selected by and needs term /
           signature u % 64 and spreads over key u % 64 with maxSkew 1; half the running pods belong to one of 64 such
           deployments, counted on their node under their key, so most nodes are admitted by one of the first
           signatures) and `none` (no signature admits any node with pods: every thread walks the whole table; for
           `ts`, every node counts one pod of every key and the floor is 0).  Per
           call: median CUDA-event time of the entry point (table upload, row_ptr read-back, kernel) over --reps calls
           after --warmup; per kernel: the device time torch.profiler records for pending_admit_kernel in a separate run.
  host     snapshot.pending_admit for U pods to schedule against the same number of running pods and nodes (CPU
           only): term numbering, masks per running pod, the signature table.  Building the pod objects is not timed.
Prints the GPU and its power limit, read in the same run.
"""
import argparse
import os
import statistics
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


def table(N, R, U, kind, seed=5):
    """row_ptr, run_carries, run_matches, run_has, sig_class, sig_carries, sig_matches, sig_need"""
    rng = np.random.default_rng(seed)
    cuts = np.sort(rng.integers(0, R + 1, size=N - 1))
    row_ptr = np.concatenate([[0], cuts, [R]]).astype(np.int64)
    u = np.arange(U)
    if kind == "typical":
        dep = rng.integers(0, 64, size=R).astype(np.uint64)
        rc = np.where(rng.random(R) < 0.5, np.uint64(1) << dep, np.uint64(0))
        rm = rc.copy()
        rh = rc.copy()
        car = np.uint64(1) << (u % 64).astype(np.uint64)
        mat = car | (np.uint64(1) << (u // 64 % 64).astype(np.uint64))
        need = car.copy()
    else:
        rc = np.zeros(R, np.uint64)
        rm = np.ones(R, np.uint64)
        rh = np.zeros(R, np.uint64)
        car = np.ones(U, np.uint64)
        mat = (u.astype(np.uint64) + np.uint64(1)) << np.uint64(1)  # distinct signatures, all blocked by bit 0
        need = np.ones(U, np.uint64)  # and none held
    return row_ptr, rc, rm, rh, np.zeros(U, np.uint8), car, mat, need


def spread(N, R, U, kind, row_ptr, seed=5):
    """sig_key, sig_skew, node_count [64, N], node_domain, floor of the `ts` forms"""
    rng = np.random.default_rng([seed, 1])
    if kind == "typical":
        key = rng.integers(0, 64, size=R)
        grouped = rng.random(R) < 0.5
        node_of = np.repeat(np.arange(N), np.diff(row_ptr))
        count = np.zeros((64, N), np.int32)
        np.add.at(count, (key[grouped], node_of[grouped]), 1)
        floor = np.full(64, 2 ** 31 - 1, np.int32)
        skew = np.ones(U, np.int32)
    else:
        count = np.ones((64, N), np.int32)
        floor = np.zeros(64, np.int32)
        skew = np.zeros(U, np.int32)
    return (np.arange(U) % 64).astype(np.uint8), skew, count, np.full(N, ~np.uint64(0)), floor


def kernel(args):
    import torch
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    eng = Engine(0)
    i64 = torch.int64
    for form, kind in ((f, k) for f in args.forms for k in ("typical", "none")):
        for U in args.sigs:
            row_ptr, rc, rm, rh, cls, car, mat, need = table(args.nodes, args.rows, U, kind)
            d_rp, d_rc, d_rm = eng.dev(row_ptr, i64), eng.dev(rc.view(np.int64), i64), eng.dev(rm.view(np.int64), i64)
            d_rh = eng.dev(rh.view(np.int64), i64)
            flags = eng.dev(np.zeros(args.nodes, np.uint8), torch.uint8)
            if form.endswith("ts"):
                key, skew, count, domain, floor = spread(args.nodes, args.rows, U, kind, row_ptr)
                d_count, d_domain = eng.dev(count, torch.int32), eng.dev(domain.view(np.int64), i64)

            def call():
                if form == "aa":
                    eng.pending_admit(d_rp, d_rc, d_rm, None, cls, car, mat, flags)
                elif form == "pa":
                    eng.pending_admit_pa(d_rp, None, None, d_rh, None, cls, None, None, need, flags)
                elif form == "ts":
                    eng.pending_admit_ts(d_rp, None, None, None, None, cls, None, None, None, key, skew, 64, d_count,
                                         d_domain, floor, flags)
                elif form == "aa+pa+ts":
                    eng.pending_admit_ts(d_rp, d_rc, d_rm, d_rh, None, cls, car, mat, need, key, skew, 64, d_count,
                                         d_domain, floor, flags)
                else:
                    eng.pending_admit_pa(d_rp, d_rc, d_rm, d_rh, None, cls, car, mat, need, flags)
            for _ in range(args.warmup):
                call()
            times = []
            for _ in range(args.reps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                call()
                b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b))
            flagged = int(((flags.cpu().numpy() & 2) != 0).sum())
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    call()
                torch.cuda.synchronize()
            dev_us = [e.self_device_time_total / e.count for e in prof.key_averages() if "pending_admit_kernel" in e.key]
            print("kernel %-8s %-7s N=%d rows=%d U=%-5d call %.3f ms (median of %d)  kernel %s  flagged %d" % (
                form, kind, args.nodes, args.rows, U, statistics.median(times), args.reps,
                "%.3f ms" % (dev_us[0] / 1000.0) if dev_us else "n/a", flagged), flush=True)


def host(args):
    from kubernetes_acs_engine_autoscaler_b200 import kube, snapshot
    rng = np.random.default_rng(7)
    apps = ["app-%d" % d for d in range(64)]
    terms = [kube.anti_affinity_terms({"podAntiAffinity": {"requiredDuringSchedulingIgnoredDuringExecution": [
        {"topologyKey": "kubernetes.io/hostname", "labelSelector": {"matchLabels": {"app": a}}}]}}, "default", "probe")
        for a in apps]
    labels = [{"app": a} for a in apps]
    nodes = [SimpleNamespace(name="node-%d" % n) for n in range(args.nodes)]
    t0 = time.perf_counter()
    dep = rng.integers(0, 128, size=args.rows)  # deployments 64..127: pods without a term or a label the terms read
    owner = np.sort(rng.integers(0, args.nodes, size=args.rows))
    empty = {}
    running = [SimpleNamespace(namespace="default", labels=labels[d] if d < 64 else empty,
                               anti_affinity_terms=terms[d] if d < 64 else (), node_name=nodes[n].name)
               for d, n in zip(dep.tolist(), owner.tolist())]
    bounds = np.searchsorted(owner, np.arange(args.nodes + 1))
    lists = [running[bounds[n]:bounds[n + 1]] for n in range(args.nodes)]
    print("host: built %d running pods on %d nodes in %.1f s (not timed below)" % (
        len(running), args.nodes, time.perf_counter() - t0), flush=True)
    for U in args.sigs:
        pending = [SimpleNamespace(namespace="default", labels=labels[k % 64], name="p%d" % k,
                                   anti_affinity_terms=tuple(dict.fromkeys(terms[k % 64] + terms[k // 64 % 64])))
                   for k in range(U)]
        t0 = time.perf_counter()
        adm = snapshot.pending_admit(pending, running, nodes, lists)
        dt = time.perf_counter() - t0
        print("host U=%-5d snapshot.pending_admit %.2f s  (%d signatures)" % (U, dt, len(adm.sig_class)), flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("what", choices=("kernel", "host", "both"))
    ap.add_argument("--nodes", type=int, default=1_000_000)
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--sigs", type=int, nargs="+", default=[1, 64, 4096])
    ap.add_argument("--forms", nargs="+", choices=("aa", "pa", "aa+pa", "ts", "aa+pa+ts"),
                    default=["aa", "pa", "aa+pa", "ts", "aa+pa+ts"])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    print("gpu: %s" % gpu_info(), flush=True)
    if args.what in ("kernel", "both"):
        kernel(args)
    if args.what in ("host", "both"):
        host(args)


if __name__ == "__main__":
    main()
