"""TEST INFRASTRUCTURE -- ctypes wrapper of tests/ts_states_oracle.c, the plain-C statement of the pending-pod admission
rule of node states with hostname topology spread (and optionally anti-affinity and pod affinity).  Compiled on first
use into a temporary directory (never into the tree), with the flags of oracle/Makefile."""
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
        tmp = tempfile.mkdtemp(prefix="acsfit_ts_states_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        path = os.path.join(tmp, "libts_states_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-ffp-contract=off",
                               "-fno-fast-math", "-fvisibility=hidden", "-Wall", "-Wextra", "-o", path,
                               os.path.join(_HERE, "ts_states_oracle.c")])
        _lib = ctypes.CDLL(path)
        _lib.oracle_pending_admit_ts.restype = None
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def _u64(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.uint64)


def pending_admit_ts(row_ptr, run_carries, run_matches, run_has, node_match, pod_class, pod_carries, pod_matches,
                     pod_need, pod_key, pod_skew, node_count, node_domain, floor, node_flags):
    """returns a copy of node_flags (uint8[N]) with bit 1 set on the nodes no pod admits.  row_ptr int64[N+1] holds
    absolute row numbers into the run masks; run_carries / run_matches / pod_carries / pod_matches all None = no
    anti-affinity test; run_has / pod_need both None = no affinity test; node_match None = every node matches every
    class.  pod_key uint8[P] (0xFF none), pod_skew int32[P], node_count int32[keys, N], node_domain uint64[N], floor
    int32[keys]."""
    row_ptr = np.ascontiguousarray(row_ptr, dtype=np.int64)
    aa = run_carries is not None
    assert aa == (run_matches is not None) == (pod_carries is not None) == (pod_matches is not None)
    assert (run_has is None) == (pod_need is None)
    run_carries, run_matches, run_has = _u64(run_carries), _u64(run_matches), _u64(run_has)
    node_match = _u64(node_match)
    pod_class = np.ascontiguousarray(pod_class, dtype=np.uint8)
    pod_carries, pod_matches, pod_need = _u64(pod_carries), _u64(pod_matches), _u64(pod_need)
    pod_key = np.ascontiguousarray(pod_key, dtype=np.uint8)
    pod_skew = np.ascontiguousarray(pod_skew, dtype=np.int32)
    out = np.array(node_flags, dtype=np.uint8, copy=True)
    N, P = len(out), len(pod_class)
    floor = np.ascontiguousarray(floor, dtype=np.int32)
    keys = len(floor)
    node_count = np.ascontiguousarray(node_count, dtype=np.int32).reshape(keys, N)
    node_domain = _u64(node_domain)
    assert row_ptr.shape == (N + 1,) and pod_key.shape == pod_skew.shape == (P,) and node_domain.shape == (N,)
    assert ((pod_key == 0xFF) | (pod_key < keys)).all() and (pod_skew >= 0).all()
    assert pod_need is None or pod_need.shape == (P,)
    assert not aa or pod_carries.shape == pod_matches.shape == (P,)
    lib().oracle_pending_admit_ts(_p(row_ptr), _p(run_carries), _p(run_matches), _p(run_has), ctypes.c_int64(N),
                                  _p(node_match), _p(pod_class), _p(pod_carries), _p(pod_matches), _p(pod_need),
                                  _p(pod_key), _p(pod_skew), ctypes.c_int64(P), _p(node_count), _p(node_domain),
                                  _p(floor), _p(out))
    return out
