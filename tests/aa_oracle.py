"""TEST INFRASTRUCTURE -- ctypes wrapper of tests/aa_oracle.c, the plain-C restatement of the node pass and the bin
pass with required pod anti-affinity.  Compiled on first use into a temporary directory (never into the tree), with
the flags of oracle/Makefile."""
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
        tmp = tempfile.mkdtemp(prefix="acsfit_aa_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        path = os.path.join(tmp, "libaa_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-ffp-contract=off",
                               "-fno-fast-math", "-fvisibility=hidden", "-Wall", "-Wextra", "-o", path,
                               os.path.join(_HERE, "aa_oracle.c")])
        _lib = ctypes.CDLL(path)
        for name in ("oracle_first_fit_nodes_aa", "oracle_fulfill_pending_aa"):
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


def first_fit_nodes_aa(req, cap_type, node_type, used, pod_carries, pod_matches, node_carries, node_matches,
                       node_match=None, pod_class=None):
    """mutates `used`, `node_carries` and `node_matches` (uint64, contiguous) in place; returns (placed int32[P],
    can_fit calls).  Without node_match / pod_class every pod is class 0 and every node matches."""
    req, cap_type = _f64(req), _f64(cap_type)
    P, D = req.shape
    N = used.shape[0]
    node_match = np.ones(N, np.uint64) if node_match is None else _u64(node_match)
    pod_class = np.zeros(P, np.uint8) if pod_class is None else _u8(pod_class)
    pod_carries, pod_matches = _u64(pod_carries), _u64(pod_matches)
    node_type = np.ascontiguousarray(node_type, dtype=np.int32)
    for a, dt in ((used, np.float64), (node_carries, np.uint64), (node_matches, np.uint64)):
        assert a.dtype == dt and a.flags.c_contiguous
    placed = np.full(P, -1, dtype=np.int32)
    calls = lib().oracle_first_fit_nodes_aa(_p(req), ctypes.c_int64(P), ctypes.c_int(D), _p(cap_type), _p(node_type),
                                            _p(used), ctypes.c_int64(N), _p(node_match), _p(pod_class),
                                            _p(pod_carries), _p(pod_matches), _p(node_carries), _p(node_matches),
                                            _p(placed))
    return placed, int(calls)


def fulfill_pending_aa(req, num_listed, unit, pool_actual, pool_max, pool_ignored, over_provision, pod_carries,
                       pod_matches, pool_match=None, pod_class=None):
    req, unit = _f64(req), _f64(unit)
    Pp, D = req.shape
    T = unit.shape[0]
    pool_match = np.ones(T, np.uint64) if pool_match is None else _u64(pool_match)
    pod_class = np.zeros(Pp, np.uint8) if pod_class is None else _u8(pod_class)
    pod_carries, pod_matches = _u64(pod_carries), _u64(pod_matches)
    pool_actual = np.ascontiguousarray(pool_actual, dtype=np.int32)
    pool_max = np.ascontiguousarray(pool_max, dtype=np.int32)
    pool_ignored = _u8(pool_ignored)
    new_size = np.zeros(T, dtype=np.int64)
    units_needed = np.zeros(T, dtype=np.int64)
    bins_opened = np.zeros(T, dtype=np.int64)
    acc_pool = np.full(Pp, -1, dtype=np.int32)
    bin_of = np.full(Pp, -1, dtype=np.int32)
    unacc = ctypes.c_int64(0)
    evals = lib().oracle_fulfill_pending_aa(
        _p(req), ctypes.c_int64(Pp), ctypes.c_int64(num_listed), ctypes.c_int(D), _p(unit), _p(pool_actual),
        _p(pool_max), _p(pool_ignored), ctypes.c_int(T), ctypes.c_int64(over_provision), _p(pool_match),
        _p(pod_class), _p(pod_carries), _p(pod_matches), _p(new_size), _p(units_needed), _p(bins_opened),
        _p(acc_pool), _p(bin_of), ctypes.byref(unacc))
    return {"new_size": new_size, "units_needed": units_needed, "bins_opened": bins_opened,
            "acc_pool": acc_pool, "bin_of": bin_of, "num_unaccounted": int(unacc.value), "evals": int(evals)}
