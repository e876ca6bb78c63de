#!/usr/bin/env python3
"""TEST INFRASTRUCTURE -- records what the differential tests compare against into tests/golden/live_reference.json.xz,
from the UNMODIFIED reference, so that those tests run without it:

* "rows": the reference's own constructors (KubePod.resources, create_kube_node capacity, count_pod sums) on two small
  synthetic clusters (tests/test_reference_live_cpu.py);
* "oracle_tick": a mid-size D = 8 / T = 8 tick of the reference (tests/test_reference_live_cpu.py);
* "host_layer": the reference's Cluster path on the clusters of tests/test_host_layer_live_cpu.py: scale_pools
  argument or exception, used_capacity bits and key sets, node states, log counts;
* "templates": the reference's fixture templates (test/data) and what its template_processing functions return on
  them (tests/test_template_processing_cpu.py).

Each cluster is named by the arguments of synthetic.make_cluster that regenerate it, with a digest of the generated
arrays so that generator drift is caught.  xz keeps the near-identical templates small.

    python oracle/make_golden_live.py        (needs the reference tree, see oracle/ref_shim.py)
"""
import copy
import importlib
import json
import lzma
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (HERE, ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import ref_bench  # noqa: E402
import ref_shim  # noqa: E402
from make_golden_mid import digest, pack  # noqa: E402
from kubernetes_acs_engine_autoscaler_b200 import synthetic as syn  # noqa: E402

ROWS_CASES = [(4, 1), (8, 8)]            # make_cluster(400, 40, D, T, seed=77)
ORACLE_CASE = dict(P=700, N=90, D=8, T=8, seed=78)
HOST_CASES = [(1500, 200, 4, 2, 901, None), (900, 120, 4, 1, 902, None), (1200, 150, 4, 2, 903, 40),
              (1200, 160, 8, 8, 904, None)]  # P, N, D, T, seed, max_size
TEMPLATE_FILES = ["azuredeploy.original.json", "azuredeploy.expected_nic.json", "azuredeploy.expected_vm.json",
                  "azuredeploy.cluster.json"]


def values(res_raw, names):
    return np.array([float(res_raw.get(k, 0.0)) for k in names], dtype=np.float64)


def record_rows(tmp):
    out = []
    for D, T in ROWS_CASES:
        c = syn.make_cluster(400, 40, D, T, seed=77)
        tick = ref_bench.ReferenceTick(c, tmpdir=tmp)
        names = c["dim_names"]
        pending = [p for p in tick.pods if p.status == "Pending"]
        pend_rows = np.array([values(p.resources.raw, names) for p in pending])
        run_rows = np.array([values(p.resources.raw, names) for p in tick.running])
        caps = np.array([values(n.capacity.raw, names) for n in tick.nodes])
        tick.occupancy()
        used = np.array([values(n.used_capacity.raw, names) for n in tick.nodes])
        out.append({"D": D, "T": T, "digest": digest(c), "n_pending": len(pending), "n_running": len(tick.running),
                    "pending_keys": sorted(set().union(*(p.resources.raw for p in pending))),
                    "pending_bits": pack(pend_rows.view(np.uint64)), "running_bits": pack(run_rows.view(np.uint64)),
                    "capacity_bits": pack(caps.view(np.uint64)), "used_bits": pack(used.view(np.uint64))})
    return out


def record_oracle_tick(tmp):
    c = syn.make_cluster(ORACLE_CASE["P"], ORACLE_CASE["N"], ORACLE_CASE["D"], ORACLE_CASE["T"],
                         seed=ORACLE_CASE["seed"], over_provision=1)
    res = ref_bench.ReferenceTick(c, tmpdir=tmp).run()
    return dict(ORACLE_CASE, digest=digest(c), to_schedule=res["to_schedule"], pending=res["pending"],
                used_bits=pack(res["used"].view(np.uint64)), scale_calls=res["scale_calls"], exception=res["exception"])


def record_host_layer(tmp):
    out = []
    for P, N, D, T, seed, max_size in HOST_CASES:
        c = syn.make_cluster(P, N, D, T, seed=seed, over_provision=1)
        cap = int(max_size if max_size is not None else c["pool_max"][0])
        tick = ref_bench.ReferenceTick(c, tmpdir=tmp, max_size=cap)
        ref = tick.run(record=True)
        out.append({"P": P, "N": N, "D": D, "T": T, "seed": seed, "max_size": max_size, "digest": digest(c),
                    "exception": ref["exception"], "scale_calls": ref["scale_calls"],
                    "node_names": [n.name for n in tick.nodes], "used_bits": pack(ref["used"].view(np.uint64)),
                    "used_keys": [sorted(n.used_capacity.raw) for n in tick.nodes],
                    "n_to_schedule": len(ref["to_schedule"]), "n_pending": len(ref["pending"]),
                    "states": [str(s) for s in ref["states"]]})
    return out


def record_templates():
    from test_template_processing_cpu import Pool, fixture_pool_names, template_calls
    ref_shim.load_reference()
    sys.path.insert(0, ref_shim.REFERENCE_ROOT)
    try:
        ref_tp = importlib.import_module("autoscaler.template_processing")
    finally:
        sys.path.remove(ref_shim.REFERENCE_ROOT)
    files = {}
    for name in TEMPLATE_FILES:
        with open(os.path.join(ref_shim.REFERENCE_ROOT, "test", "data", name)) as f:
            files[name] = json.load(f)
    cluster = files["azuredeploy.cluster.json"]
    results = [fn(ref_tp, copy.deepcopy(cluster), Pool) for fn in template_calls(fixture_pool_names(cluster))]
    return {"files": files, "results": results}


def main():
    tmp = tempfile.mkdtemp(prefix="acsfit_golden_")
    out = {"source": "unmodified reference via oracle/ref_bench.py and oracle/ref_shim.py",
           "rows": record_rows(tmp), "oracle_tick": record_oracle_tick(tmp), "host_layer": record_host_layer(tmp),
           "templates": record_templates()}
    path = os.path.join(ROOT, "tests", "golden", "live_reference.json.xz")
    with lzma.open(path, "wb", preset=9 | lzma.PRESET_EXTREME) as f:
        f.write(json.dumps(out, sort_keys=True).encode())
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
