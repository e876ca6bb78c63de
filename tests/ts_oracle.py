"""TEST INFRASTRUCTURE -- ctypes wrapper of tests/ts_oracle.c, the plain-C restatement of the node pass and the bin
pass with hostname topology spread (and node selectors, anti-affinity and pod affinity).  Compiled on first use into a
temporary directory (never into the tree), with the flags of oracle/Makefile."""
import atexit
import ctypes
import os
import shutil
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_lib = None
NO_KEY = 0xFF


def lib():
    global _lib
    if _lib is None:
        tmp = tempfile.mkdtemp(prefix="acsfit_ts_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        path = os.path.join(tmp, "libts_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-ffp-contract=off",
                               "-fno-fast-math", "-fvisibility=hidden", "-Wall", "-Wextra", "-o", path,
                               os.path.join(_HERE, "ts_oracle.c")])
        _lib = ctypes.CDLL(path)
        for name in ("oracle_first_fit_nodes_ts", "oracle_fulfill_pending_ts"):
            getattr(_lib, name).restype = ctypes.c_uint64
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


def _pairs(buf, n):
    return [(int(buf[2 * k]), int(buf[2 * k + 1])) for k in range(n)]


def first_fit_nodes_ts(req, cap_type, node_type, used, keys, pod_key, pod_skew, ts_matches, node_count, node_domain,
                       floor, pod_requires=None, pod_self=None, pod_aff_matches=None, node_has=None, pod_carries=None,
                       pod_matches=None, node_carries=None, node_matches=None, node_match=None, pod_class=None,
                       follow=None):
    """mutates `used` and `node_count` (and the affinity node masks when given; contiguous, of their dtypes) in place;
    returns (placed int32[P], can_fit calls, flips [(signature, position)], rises [(key, position)]).  `follow`: the
    number of rises the pass follows (None: all); after the last one every key keeps its minimum."""
    req, cap_type = _c(req, np.float64), _c(cap_type, np.float64)
    P, D = req.shape
    N = used.shape[0]
    z = lambda n: np.zeros(n, np.uint64)  # noqa: E731
    node_match = np.ones(N, np.uint64) if node_match is None else _c(node_match, np.uint64)
    pod_class = np.zeros(P, np.uint8) if pod_class is None else _c(pod_class, np.uint8)
    pod_carries, pod_matches = (z(P) if a is None else _c(a, np.uint64) for a in (pod_carries, pod_matches))
    pod_requires, pod_self, pod_aff_matches = (z(P) if a is None else _c(a, np.uint64)
                                               for a in (pod_requires, pod_self, pod_aff_matches))
    node_carries = z(N) if node_carries is None else node_carries
    node_matches = z(N) if node_matches is None else node_matches
    node_has = z(N) if node_has is None else node_has
    for a, dt in ((used, np.float64), (node_carries, np.uint64), (node_matches, np.uint64), (node_has, np.uint64),
                  (node_count, np.int32)):
        assert a.dtype == dt and a.flags.c_contiguous
    assert node_count.shape == (keys, N)
    placed = np.full(P, -1, dtype=np.int32)
    flips = np.zeros(2 * 64, dtype=np.int64)
    n_flips = ctypes.c_int64(0)
    max_rises = keys * P + 16  # a pod that several keys select can raise several minimums
    rises = np.zeros(2 * max_rises, dtype=np.int64)
    n_rises = ctypes.c_int64(0)
    calls = lib().oracle_first_fit_nodes_ts(
        _p(req), ctypes.c_int64(P), ctypes.c_int(D), _p(cap_type), _p(_c(node_type, np.int32)), _p(used),
        ctypes.c_int64(N), _p(node_match), _p(pod_class), _p(pod_carries), _p(pod_matches), _p(node_carries),
        _p(node_matches), _p(pod_requires), _p(pod_self), _p(pod_aff_matches), _p(node_has), ctypes.c_int(keys),
        _p(_c(pod_key, np.uint8)), _p(_c(pod_skew, np.int32)), _p(_c(ts_matches, np.uint64)), _p(node_count),
        _p(_c(node_domain, np.uint64)), _p(_c(np.zeros(0) if floor is None else floor, np.int32)), _p(placed),
        _p(flips), ctypes.byref(n_flips), _p(rises), ctypes.byref(n_rises), ctypes.c_int64(max_rises),
        ctypes.c_int64(-1 if follow is None else follow))
    return placed, int(calls), _pairs(flips, n_flips.value), _pairs(rises, n_rises.value)


def fulfill_pending_ts(req, num_listed, unit, pool_actual, pool_max, pool_ignored, over_provision, keys, pod_key,
                       pod_skew, ts_matches, pod_requires=None, pod_self=None, pod_aff_matches=None, present=0,
                       pod_carries=None, pod_matches=None, pool_match=None, pod_class=None):
    req, unit = _c(req, np.float64), _c(unit, np.float64)
    Pp, D = req.shape
    T = unit.shape[0]
    z = lambda n: np.zeros(n, np.uint64)  # noqa: E731
    pool_match = np.ones(T, np.uint64) if pool_match is None else _c(pool_match, np.uint64)
    pod_class = np.zeros(Pp, np.uint8) if pod_class is None else _c(pod_class, np.uint8)
    pod_carries, pod_matches = (z(Pp) if a is None else _c(a, np.uint64) for a in (pod_carries, pod_matches))
    pod_requires, pod_self, pod_aff_matches = (z(Pp) if a is None else _c(a, np.uint64)
                                               for a in (pod_requires, pod_self, pod_aff_matches))
    new_size = np.zeros(T, dtype=np.int64)
    units_needed = np.zeros(T, dtype=np.int64)
    bins_opened = np.zeros(T, dtype=np.int64)
    acc_pool = np.full(Pp, -1, dtype=np.int32)
    bin_of = np.full(Pp, -1, dtype=np.int32)
    unacc = ctypes.c_int64(0)
    flips = np.zeros(2 * 64 * max(T, 1), dtype=np.int64)
    n_flips = ctypes.c_int64(0)
    evals = lib().oracle_fulfill_pending_ts(
        _p(req), ctypes.c_int64(Pp), ctypes.c_int64(num_listed), ctypes.c_int(D), _p(unit),
        _p(_c(pool_actual, np.int32)), _p(_c(pool_max, np.int32)), _p(_c(pool_ignored, np.uint8)), ctypes.c_int(T),
        ctypes.c_int64(over_provision), _p(pool_match), _p(pod_class), _p(pod_carries), _p(pod_matches),
        _p(pod_requires), _p(pod_self), _p(pod_aff_matches), ctypes.c_uint64(int(present)), ctypes.c_int(keys),
        _p(_c(pod_key, np.uint8)), _p(_c(pod_skew, np.int32)), _p(_c(ts_matches, np.uint64)), _p(new_size),
        _p(units_needed), _p(bins_opened), _p(acc_pool), _p(bin_of), ctypes.byref(unacc), _p(flips),
        ctypes.byref(n_flips))
    return {"new_size": new_size, "units_needed": units_needed, "bins_opened": bins_opened,
            "acc_pool": acc_pool, "bin_of": bin_of, "num_unaccounted": int(unacc.value), "evals": int(evals),
            "flips": _pairs(flips, n_flips.value)}
