"""TEST INFRASTRUCTURE -- ctypes wrapper of tests/pa_oracle.c, the plain-C restatement of the node pass and the bin
pass with required pod affinity (and node selectors and anti-affinity).  Compiled on first use into a temporary
directory (never into the tree), with the flags of oracle/Makefile."""
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
        tmp = tempfile.mkdtemp(prefix="acsfit_pa_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        path = os.path.join(tmp, "libpa_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-ffp-contract=off",
                               "-fno-fast-math", "-fvisibility=hidden", "-Wall", "-Wextra", "-o", path,
                               os.path.join(_HERE, "pa_oracle.c")])
        _lib = ctypes.CDLL(path)
        for name in ("oracle_first_fit_nodes_pa", "oracle_fulfill_pending_pa"):
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


def _flips(buf, n):
    return [(int(buf[2 * k]), int(buf[2 * k + 1])) for k in range(n)]


def first_fit_nodes_pa(req, cap_type, node_type, used, pod_requires, pod_self, pod_aff_matches, node_has,
                       pod_carries=None, pod_matches=None, node_carries=None, node_matches=None, node_match=None,
                       pod_class=None):
    """mutates `used`, `node_has` (and the anti-affinity node masks when given; uint64, contiguous) in place; returns
    (placed int32[P], can_fit calls, flips [(signature, position)])"""
    req, cap_type = _f64(req), _f64(cap_type)
    P, D = req.shape
    N = used.shape[0]
    node_match = np.ones(N, np.uint64) if node_match is None else _u64(node_match)
    pod_class = np.zeros(P, np.uint8) if pod_class is None else _u8(pod_class)
    pod_carries = np.zeros(P, np.uint64) if pod_carries is None else _u64(pod_carries)
    pod_matches = np.zeros(P, np.uint64) if pod_matches is None else _u64(pod_matches)
    node_carries = np.zeros(N, np.uint64) if node_carries is None else node_carries
    node_matches = np.zeros(N, np.uint64) if node_matches is None else node_matches
    node_type = np.ascontiguousarray(node_type, dtype=np.int32)
    for a, dt in ((used, np.float64), (node_carries, np.uint64), (node_matches, np.uint64), (node_has, np.uint64)):
        assert a.dtype == dt and a.flags.c_contiguous
    placed = np.full(P, -1, dtype=np.int32)
    flips = np.zeros(2 * 64, dtype=np.int64)
    n_flips = ctypes.c_int64(0)
    calls = lib().oracle_first_fit_nodes_pa(
        _p(req), ctypes.c_int64(P), ctypes.c_int(D), _p(cap_type), _p(node_type), _p(used), ctypes.c_int64(N),
        _p(node_match), _p(pod_class), _p(pod_carries), _p(pod_matches), _p(node_carries), _p(node_matches),
        _p(_u64(pod_requires)), _p(_u64(pod_self)), _p(_u64(pod_aff_matches)), _p(node_has), _p(placed), _p(flips),
        ctypes.byref(n_flips))
    return placed, int(calls), _flips(flips, n_flips.value)


def fulfill_pending_pa(req, num_listed, unit, pool_actual, pool_max, pool_ignored, over_provision, pod_requires,
                       pod_self, pod_aff_matches, present=0, pod_carries=None, pod_matches=None, pool_match=None,
                       pod_class=None):
    req, unit = _f64(req), _f64(unit)
    Pp, D = req.shape
    T = unit.shape[0]
    pool_match = np.ones(T, np.uint64) if pool_match is None else _u64(pool_match)
    pod_class = np.zeros(Pp, np.uint8) if pod_class is None else _u8(pod_class)
    pod_carries = np.zeros(Pp, np.uint64) if pod_carries is None else _u64(pod_carries)
    pod_matches = np.zeros(Pp, np.uint64) if pod_matches is None else _u64(pod_matches)
    pool_actual = np.ascontiguousarray(pool_actual, dtype=np.int32)
    pool_max = np.ascontiguousarray(pool_max, dtype=np.int32)
    pool_ignored = _u8(pool_ignored)
    new_size = np.zeros(T, dtype=np.int64)
    units_needed = np.zeros(T, dtype=np.int64)
    bins_opened = np.zeros(T, dtype=np.int64)
    acc_pool = np.full(Pp, -1, dtype=np.int32)
    bin_of = np.full(Pp, -1, dtype=np.int32)
    unacc = ctypes.c_int64(0)
    flips = np.zeros(2 * 64 * max(T, 1), dtype=np.int64)
    n_flips = ctypes.c_int64(0)
    evals = lib().oracle_fulfill_pending_pa(
        _p(req), ctypes.c_int64(Pp), ctypes.c_int64(num_listed), ctypes.c_int(D), _p(unit), _p(pool_actual),
        _p(pool_max), _p(pool_ignored), ctypes.c_int(T), ctypes.c_int64(over_provision), _p(pool_match),
        _p(pod_class), _p(pod_carries), _p(pod_matches), _p(_u64(pod_requires)), _p(_u64(pod_self)),
        _p(_u64(pod_aff_matches)), ctypes.c_uint64(int(present)), _p(new_size), _p(units_needed), _p(bins_opened),
        _p(acc_pool), _p(bin_of), ctypes.byref(unacc), _p(flips), ctypes.byref(n_flips))
    return {"new_size": new_size, "units_needed": units_needed, "bins_opened": bins_opened,
            "acc_pool": acc_pool, "bin_of": bin_of, "num_unaccounted": int(unacc.value), "evals": int(evals),
            "flips": _flips(flips, n_flips.value)}
