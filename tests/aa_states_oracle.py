"""TEST INFRASTRUCTURE -- ctypes wrapper of tests/aa_states_oracle.c, the plain-C statement of the pending-pod admission
rule of node states with pod anti-affinity.  Compiled on first use into a temporary directory (never into the tree),
with the flags of oracle/Makefile."""
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
        tmp = tempfile.mkdtemp(prefix="acsfit_aa_states_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        path = os.path.join(tmp, "libaa_states_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-shared", "-ffp-contract=off",
                               "-fno-fast-math", "-fvisibility=hidden", "-Wall", "-Wextra", "-o", path,
                               os.path.join(_HERE, "aa_states_oracle.c")])
        _lib = ctypes.CDLL(path)
        _lib.oracle_pending_admit.restype = None
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


def pending_admit(row_ptr, run_carries, run_matches, node_match, pod_class, pod_carries, pod_matches, node_flags):
    """returns a copy of node_flags (uint8[N]) with bit 1 set on the nodes no pod admits.  row_ptr int64[N+1] holds
    absolute row numbers into run_carries / run_matches; node_match None = every node matches every class."""
    row_ptr = np.ascontiguousarray(row_ptr, dtype=np.int64)
    run_carries = np.ascontiguousarray(run_carries, dtype=np.uint64)
    run_matches = np.ascontiguousarray(run_matches, dtype=np.uint64)
    node_match = None if node_match is None else np.ascontiguousarray(node_match, dtype=np.uint64)
    pod_class = np.ascontiguousarray(pod_class, dtype=np.uint8)
    pod_carries = np.ascontiguousarray(pod_carries, dtype=np.uint64)
    pod_matches = np.ascontiguousarray(pod_matches, dtype=np.uint64)
    out = np.array(node_flags, dtype=np.uint8, copy=True)
    N, P = len(out), len(pod_class)
    assert row_ptr.shape == (N + 1,) and pod_carries.shape == pod_matches.shape == (P,)
    assert N == 0 or (0 <= row_ptr[0] and row_ptr[N] <= len(run_carries) == len(run_matches))
    lib().oracle_pending_admit(_p(row_ptr), _p(run_carries), _p(run_matches), ctypes.c_int64(N), _p(node_match),
                               _p(pod_class), _p(pod_carries), _p(pod_matches), ctypes.c_int64(P), _p(out))
    return out
