"""TEST INFRASTRUCTURE -- ctypes wrapper of tests/sel_oracle.c, the plain-C restatement of the scale-up path with
node selectors.  Compiled on first use into a temporary directory (never into the tree), with the flags of
oracle/Makefile."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="acsfit_sel_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        path = os.path.join(tmp, "libsel_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-ffp-contract=off",
                               "-fno-fast-math", "-fvisibility=hidden", "-Wall", "-Wextra", "-o", path,
                               os.path.join(_HERE, "sel_oracle.c")])
        _lib = ctypes.CDLL(path)
        for name in ("oracle_feasible_mask_sel", "oracle_first_fit_nodes_sel", "oracle_fulfill_pending_sel"):
            getattr(_lib, name).restype = ctypes.c_uint64
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def _u8(a):
    return np.ascontiguousarray(a, dtype=np.uint8)


def feasible_mask_sel(req, unit, pool_match, pod_class):
    req, unit, pool_match, pod_class = _f64(req), _f64(unit), _u64(pool_match), _u8(pod_class)
    P, D = req.shape
    mask = np.zeros(P, dtype=np.uint8)
    evals = lib().oracle_feasible_mask_sel(_p(req), ctypes.c_int64(P), ctypes.c_int(D), _p(unit),
                                           ctypes.c_int(unit.shape[0]), _p(pool_match), _p(pod_class), _p(mask))
    return mask, int(evals)


def first_fit_nodes_sel(req, cap_type, node_type, used, node_match, pod_class):
    """mutates `used` in place; returns (placed int32[P], can_fit calls)."""
    req, cap_type, node_match, pod_class = _f64(req), _f64(cap_type), _u64(node_match), _u8(pod_class)
    node_type = np.ascontiguousarray(node_type, dtype=np.int32)
    assert used.dtype == np.float64 and used.flags.c_contiguous
    P, D = req.shape
    placed = np.full(P, -1, dtype=np.int32)
    calls = lib().oracle_first_fit_nodes_sel(_p(req), ctypes.c_int64(P), ctypes.c_int(D), _p(cap_type),
                                             _p(node_type), _p(used), ctypes.c_int64(used.shape[0]), _p(node_match),
                                             _p(pod_class), _p(placed))
    return placed, int(calls)


def fulfill_pending_sel(req, num_listed, unit, pool_actual, pool_max, pool_ignored, over_provision, pool_match,
                        pod_class):
    req, unit, pool_match, pod_class = _f64(req), _f64(unit), _u64(pool_match), _u8(pod_class)
    Pp, D = req.shape
    T = unit.shape[0]
    pool_actual = np.ascontiguousarray(pool_actual, dtype=np.int32)
    pool_max = np.ascontiguousarray(pool_max, dtype=np.int32)
    pool_ignored = _u8(pool_ignored)
    new_size = np.zeros(T, dtype=np.int64)
    units_needed = np.zeros(T, dtype=np.int64)
    bins_opened = np.zeros(T, dtype=np.int64)
    acc_pool = np.full(Pp, -1, dtype=np.int32)
    bin_of = np.full(Pp, -1, dtype=np.int32)
    unacc = ctypes.c_int64(0)
    evals = lib().oracle_fulfill_pending_sel(
        _p(req), ctypes.c_int64(Pp), ctypes.c_int64(num_listed), ctypes.c_int(D), _p(unit), _p(pool_actual),
        _p(pool_max), _p(pool_ignored), ctypes.c_int(T), ctypes.c_int64(over_provision), _p(pool_match),
        _p(pod_class), _p(new_size), _p(units_needed), _p(bins_opened), _p(acc_pool), _p(bin_of),
        ctypes.byref(unacc))
    return {"new_size": new_size, "units_needed": units_needed, "bins_opened": bins_opened,
            "acc_pool": acc_pool, "bin_of": bin_of, "num_unaccounted": int(unacc.value), "evals": int(evals)}


def scale_up_sel(c, used):
    """the fused tick (acsfit_scale_up_sel) from the three functions above, for a case of tests/selector_cases.py;
    mutates `used`.  Returns the dict the engine's scale_up_sel_host returns, with numpy arrays."""
    req, P = c["req"], c["req"].shape[0]
    mask, ev0 = feasible_mask_sel(req, c["unit_all"], c["pool_match_all"], c["pod_class"])
    idx = np.nonzero(mask)[0]
    placed_f, ev1 = first_fit_nodes_sel(req[idx], c["cap_type"], c["node_type"], used, c["node_match"],
                                        c["pod_class"][idx])
    placed = np.where(mask.astype(bool), -1, -2).astype(np.int32)
    placed[idx] = placed_f
    pend = idx[placed_f < 0]
    T = c["unit_all"].shape[0]
    acc = np.full(P, -1, dtype=np.int32)
    if len(pend):
        f = fulfill_pending_sel(req[pend], len(pend), c["unit_ordered"], c["pool_actual"], c["pool_max"],
                                c["pool_ignored"], c["over_provision"], c["pool_match_ordered"], c["pod_class"][pend])
        acc[pend] = f["acc_pool"]
    else:
        f = {"new_size": np.asarray(c["pool_actual"], dtype=np.int64), "units_needed": np.full(T, -1, np.int64),
             "bins_opened": np.zeros(T, np.int64), "num_unaccounted": 0, "evals": 0}
    return {"feasible": mask, "placed": placed, "acc_pool": acc, "new_size": f["new_size"],
            "units_needed": f["units_needed"], "bins_opened": f["bins_opened"], "n_to_schedule": len(idx),
            "n_pending": len(pend), "num_unaccounted": f["num_unaccounted"], "decisions": ev0 + ev1 + f["evals"]}
