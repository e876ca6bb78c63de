"""Dense ticks for the pod anti-affinity entry points (tests/test_gpu_anti_affinity.py): a node pass over every pod
and a bin pass over the pods it leaves pending, with term masks (bit k = term k) on the pods and on the nodes.

Kinds:
  replicas     self-anti-affine replicas (carries = matches = one bit) that outnumber the nodes
  symmetric    pending pods that carry no term, blocked by the terms of pods already on the nodes
  cross_ns     one group carries a term that selects a second group only (a term of another namespace)
  bits64       64 self-anti-affine deployments: every bit in use
  edges        blocked pods at the 256-pod tile edges and blocked nodes at the stage edges (128 / 256 nodes)
  all_blocked  every node already holds a pod every pending pod avoids
  with_sel     anti-affinity together with three selector classes
  zero         every mask 0: the results of the _sel and plain entry points
`overlay` puts replicas groups on any other dense tick (the rank-layout ticks of tests/variant_cases.py).
"""
import numpy as np

KINDS = ("replicas", "symmetric", "cross_ns", "bits64", "edges", "all_blocked", "with_sel", "zero")
DIMS = (2, 4, 8, 16)
U64 = np.uint64


def _bit(k):
    return U64(1) << U64(k)


def _base(D, P, N, rng):
    T = 3
    unit = np.zeros((T, D))
    unit[:, 0] = (4.0, 8.0, 16.0)
    unit[:, 1] = np.array((16.0, 32.0, 64.0)) * 2 ** 30
    for d in range(2, D):
        unit[:, d] = 110.0 + d
    cap_type = unit.copy()
    node_type = rng.integers(0, T, size=N).astype(np.int32)
    used = cap_type[node_type] * rng.uniform(0.0, 0.7, size=(N, 1))
    used[:, 2:] = 0.0
    req = np.zeros((P, D))
    req[:, 0] = rng.choice([0.1, 0.25, 0.5, 1.0, 2.0], size=P)
    req[:, 1] = rng.choice([0.5, 1.0, 2.0, 4.0], size=P) * 2 ** 30
    if D > 2:
        req[:, 2] = 1.0
    return {"req": req, "cap_type": cap_type, "node_type": node_type, "used0": np.ascontiguousarray(used),
            "unit": unit[::-1].copy(), "pool_actual": np.array([5, 2, 0], np.int32),
            "pool_max": np.array([400, 60, 1 << 20], np.int32), "pool_ignored": np.zeros(T, np.uint8),
            "over_provision": 1,
            "pod_carries": np.zeros(P, U64), "pod_matches": np.zeros(P, U64),
            "node_carries0": np.zeros(N, U64), "node_matches0": np.zeros(N, U64)}


def _replicas(c, groups, share, rng):
    """`share` of the pods, spread over `groups` self-anti-affine deployments (group g = bit g)"""
    P = c["req"].shape[0]
    who = np.nonzero(rng.random(P) < share)[0]
    g = rng.integers(0, groups, size=len(who)).astype(np.uint64)
    c["pod_carries"][who] |= U64(1) << g
    c["pod_matches"][who] |= U64(1) << g
    return c


def make_case(kind, D, seed=0):
    rng = np.random.default_rng([seed, D, KINDS.index(kind)])
    P, N = 1500, 300
    if kind == "edges":
        P, N = 4 * 256 + 17, 700
    c = _base(D, P, N, rng)
    if kind == "replicas":
        _replicas(c, 3, 1.0, rng)  # about 500 replicas per deployment on 300 nodes
    elif kind == "symmetric":
        c["pod_matches"][rng.random(P) < 0.6] |= _bit(5)  # selected by term 5, carry nothing
        c["node_carries0"][rng.random(N) < 0.5] |= _bit(5)  # a pod that carries term 5 already runs there
        c["node_matches0"][rng.random(N) < 0.3] |= _bit(9)
        c["pod_carries"][rng.random(P) < 0.1] |= _bit(9)
    elif kind == "cross_ns":
        a = rng.random(P) < 0.3
        b = ~a & (rng.random(P) < 0.5)
        c["pod_carries"][a] |= _bit(2)  # group a avoids group b (another namespace); b has no term
        c["pod_matches"][b] |= _bit(2)
        c["pod_matches"][a] |= _bit(7)  # a pod of a namespace nobody's term covers is selected by term 7 only
    elif kind == "bits64":
        _replicas(c, 64, 0.9, rng)
    elif kind == "edges":
        for j in (255, 256, 511, 512, 767, 768, 1023, 1024):
            c["pod_carries"][j] |= _bit(1)
            c["pod_matches"][j] |= _bit(1)
        for n in (0, 127, 128, 255, 256, 383, 384, 511, 512):
            c["node_matches0"][n] |= _bit(1)
        _replicas(c, 4, 0.3, rng)
    elif kind == "all_blocked":
        c["pod_carries"][:] = _bit(0)
        c["pod_matches"][:] = _bit(3)
        c["node_matches0"][:] = _bit(0) | _bit(40)
        c["pod_carries"][rng.random(P) < 0.2] |= _bit(3)  # some pending pods also avoid each other in the bins
    elif kind == "with_sel":
        _replicas(c, 5, 0.5, rng)
        c["classes"] = 3
        c["pod_class"] = rng.integers(0, 3, size=P).astype(np.uint8)
        c["node_match"] = (U64(1) | (rng.integers(0, 4, size=N).astype(np.uint64) << U64(1))).astype(U64)
        c["pool_match"] = np.array([1 | 2, 1 | 4, 1 | 2 | 4], U64)
    return c


def overlay(c, seed=0):
    """a copy of dense tick `c` (keys of tests/variant_cases.py plus used0) with the masks of this module: 10 % of the
    pods in 8 self-anti-affine deployments, and some nodes that already hold a replica of deployment 0"""
    rng = np.random.default_rng(seed)
    P, N = c["req"].shape[0], c["node_type"].shape[0]
    out = {"req": c["req"], "cap_type": c["cap_type"], "node_type": c["node_type"], "used0": c["used0"],
           "unit": c["unit_ordered"], "pool_actual": c["pool_actual"], "pool_max": c["pool_max"],
           "pool_ignored": c["pool_ignored"], "over_provision": c["over_provision"],
           "pod_carries": np.zeros(P, U64), "pod_matches": np.zeros(P, U64),
           "node_carries0": np.zeros(N, U64), "node_matches0": np.zeros(N, U64)}
    _replicas(out, 8, 0.1, rng)
    out["node_carries0"][rng.random(N) < 0.2] |= _bit(0)
    out["node_matches0"][rng.random(N) < 0.2] |= _bit(0)
    return out
