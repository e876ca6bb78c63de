"""`-m "not gpu"`: tests/idle_cases.py hits what it aims at, and the K1 / K6 dispatch table of
csrc/acsfit_scan_plan.h (compiled with g++) gives every (D, layout, alignment, knob) row the intended form."""
import os
import subprocess

import numpy as np
import pytest

import idle_cases as ic

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DIMS = (2, 4, 8, 16, 1, 3, 5, 12, 15)
SMALL = tuple(n for n in ic.NAMES if n != "multigroup")


def oracle_states(oracle_mod, c, any_pending):
    return oracle_mod.node_states(c["row_ptr"], ic.identity_idx(c), c["req_run"], c["flags_run"], c["cap_type"],
                                  c["node_type"], c["node_flags"], c["node_age"], any_pending, c["thr"])


def busy_sum(c, n, d):
    k0, k1 = c["row_ptr"][n], c["row_ptr"][n + 1]
    take = (c["flags_run"][k0:k1] & ic.PODF_BUSY) != 0
    return ic.ordered_sum(c["req_run"][k0:k1, d][take])


@pytest.mark.parametrize("D", DIMS)
def test_left_exactly_zero_and_one_ulp_below(D):
    c = ic.case("boundary", D)
    for kind in ("left_zero", "left_ulp"):
        assert len(c["hits"][kind]) >= 2 * D, kind
        dims = set()
        for n, d in c["hits"][kind]:
            thr = ic.thresh(c["cap_type"][c["node_type"][n], d])
            left = thr - busy_sum(c, n, d)
            if kind == "left_zero":
                assert left == 0.0, (n, d, left)
            else:
                assert left < 0 and left == -(np.nextafter(thr, np.inf) - thr), (n, d, left)
            # every other dimension is under its threshold, so this one decides
            for e in range(D):
                if e != d:
                    assert ic.thresh(c["cap_type"][c["node_type"][n], e]) - busy_sum(c, n, e) >= 0
            # non-busy pods with requests far above the threshold sit between the busy ones
            k0 = c["row_ptr"][n]
            assert not (c["flags_run"][k0 + 1] & ic.PODF_BUSY) and c["req_run"][k0 + 1, d] > 1e11
            dims.add(d)
        assert dims == set(range(D)), kind  # a different dimension on different nodes


@pytest.mark.parametrize("D", DIMS)
def test_every_reachable_state_appears(oracle_mod, D):
    c = ic.case("boundary", D)
    seen = set()
    for any_pending in (False, True):
        seen |= set(np.unique(oracle_states(oracle_mod, c, any_pending)).tolist())
    assert seen == {1, 2, 4, 5, 6, 7, 8, 9}, sorted(seen)
    # ages on a threshold and one either side, and unschedulable nodes among the boundary nodes
    assert c["hits"]["age_on_threshold"] > 0
    diff = c["node_age"][:, None] - c["thr"][None, :]
    assert {-1, 0, 1} <= set(np.unique(diff).tolist())
    bn = np.array([n for n, _ in c["hits"]["left_zero"] + c["hits"]["left_ulp"]])
    assert 0 < c["node_flags"][bn].sum() < len(bn)


@pytest.mark.parametrize("D", DIMS)
def test_table_shapes(D):
    Ss = set()
    for name in ic.NAMES:
        c = ic.case(name, D)
        N, rp = c["N"], c["row_ptr"]
        Ss.add(c["S"])
        assert np.all(np.diff(rp) >= 0) and rp.shape == (N + 1,)
        assert c["req_run"].shape == (rp[-1], D) and c["flags_run"].shape == (rp[-1],)
        # the gathered layout holds the same rows per node, from a larger table
        idx = c["run_idx"][rp[0]:]
        assert c["req_tab"].shape[0] > rp[-1]
        np.testing.assert_array_equal(c["req_tab"][idx], c["req_run"][rp[0]:])
        np.testing.assert_array_equal(c["flags_tab"][idx], c["flags_run"][rp[0]:])
        assert len(np.unique(idx)) == len(idx)
    assert Ss == {1, 8, 64}
    assert ic.case("n1_all_entries", D)["N"] == 1 and ic.case("n1_all_entries", D)["hits"]["R"] > 3 * ic.LARGEST_CHUNK
    assert ic.case("row_ptr_offset", D)["row_ptr"][0] > 0
    e = ic.case("empty_table", D)
    assert e["N"] > 0 and e["hits"]["R"] == 0
    assert {ic.case(n, D)["N"] % 32 for n in ("n31", "n33", "ragged", "multigroup")} >= {31, 1}
    r = ic.case("ragged", D)
    assert r["hits"]["R"] % 16 != 0                       # the bulk form's plain-load tail of flag bytes
    assert np.any(np.diff(r["row_ptr"]) == 0)            # empty nodes
    g = ic.group_ends(r)                                  # and empty 32-node groups
    assert np.any(np.diff(g) == 0)


@pytest.mark.parametrize("D", (2, 4, 8, 16))
def test_slices_and_group_ends_against_chunks(D):
    sizes = ic.chunks_of(D)
    assert max(sizes) <= ic.LARGEST_CHUNK
    for name in ("n1_all_entries", "ragged", "multigroup"):
        c = ic.case(name, D)
        assert c["hits"]["max_slice"] >= 3 * max(sizes), name   # slices span >= 3 chunks of the largest kChunk
    # one chunk of the smallest kChunk holds the ends of >= 2 groups
    small = min(sizes)
    for name in ("ragged", "multigroup"):
        ends = ic.group_ends(ic.case(name, D))
        per_chunk = np.bincount(ends // small)
        assert per_chunk.max() >= 2, name


def test_multigroup_gives_every_warp_two_groups():
    c = ic.case("multigroup", 2)
    groups = (c["N"] + 31) // 32
    # the most warps any geometry can have resident on an H100 (132 SMs x 2048 threads)
    assert groups >= 2 * 132 * 2048 // 32
    assert c["N"] > 2 * 132 * 8 * 128                   # per-thread form: each thread takes >= 2 nodes


def test_scan_plan_table_on_host(tmp_path):
    """acsfit::plan_scan (csrc/acsfit_scan_plan.h): bulk geometries per bulk_cfg (out of range -> default), gather
    bytes per stream_bytes with the D = 8 and D = 16 clamps, and the per-thread form for every other D and for any
    table that is not 16-byte aligned."""
    exe = os.path.join(str(tmp_path), "test_scan_plan")
    subprocess.check_call(["g++", "-O2", "-Wall", "-x", "c++",
                           "-I", os.path.join(ROOT, "kubernetes_acs_engine_autoscaler_b200", "csrc"),
                           os.path.join(ROOT, "tests", "cpp", "test_scan_plan.cpp"), "-o", exe])
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout[-2000:]
    assert "failures=0" in out.stdout
