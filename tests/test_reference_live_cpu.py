"""`-m "not gpu"`: the reference's own constructors give the synthetic dense rows back bit for bit (SURVEY.md
section 7), and the C oracle equals the reference on a mid-size tick.  What the unmodified reference computed is
recorded in tests/golden/live_reference.json.xz (oracle/make_golden_live.py)."""
import numpy as np
import pytest

import golden_util as gu
import mid_golden
from kubernetes_acs_engine_autoscaler_b200 import synthetic as syn


def golden():
    return gu.load_json("live_reference.json.xz")


@pytest.mark.parametrize("D,T", [(4, 1), (8, 8)])
def test_synthetic_rows_equal_reference_constructors(D, T):
    rec = [r for r in golden()["rows"] if (r["D"], r["T"]) == (D, T)][0]
    c = mid_golden.cluster_of({"P": 400, "N": 40, "D": D, "T": T, "seed": 77, "digest": rec["digest"]})
    names = c["dim_names"]
    assert rec["n_pending"] == c["P"] and rec["n_running"] == c["req_run"].shape[0]
    assert set(rec["pending_keys"]) <= set(names)

    def bits(key, rows):
        return mid_golden._unpack(rec[key], np.uint64).reshape(rows, len(names))
    # KubePod.resources (kube.py:41-49) == the dense request rows, running and pending
    np.testing.assert_array_equal(bits("pending_bits", c["P"]), c["req"].view(np.uint64))
    np.testing.assert_array_equal(bits("running_bits", rec["n_running"]), c["req_run"][c["run_idx"]].view(np.uint64))
    # create_kube_node capacity (cluster.py:130-133) == cap_type row
    np.testing.assert_array_equal(bits("capacity_bits", c["N"]), c["cap_type"][c["node_type"]].view(np.uint64))
    # count_pod sums (cluster.py:165-168) == initial_used
    np.testing.assert_array_equal(bits("used_bits", c["N"]), syn.initial_used(c).view(np.uint64))


def test_oracle_equals_live_reference(oracle_mod):
    import ref_bench
    rec = golden()["oracle_tick"]
    c = mid_golden.cluster_of({k: rec[k] for k in ("P", "N", "D", "T", "seed", "digest")} | {"over_provision": 1})
    res = {"to_schedule": rec["to_schedule"], "pending": rec["pending"], "scale_calls": rec["scale_calls"],
           "exception": rec["exception"],
           "used": mid_golden._unpack(rec["used_bits"], np.uint64).reshape(c["N"], c["D"]).view(np.float64)}
    assert ref_bench.compare(c, res, ref_bench.dense_answer(oracle_mod, c)) == []
