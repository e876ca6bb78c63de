"""Inputs for the K1 (occupancy) / K6 (node states) idle-scan kernels, pure numpy (tests/test_gpu_idle_variants.py).

Each case is a CSR running-pod table for one D, in two layouts with the same per-node rows in the same order:
  * contiguous: the pods of node n are rows row_ptr[n] .. row_ptr[n+1] of req_run / flags_run (run_idx = NULL,
    the bulk-copy form);
  * gathered: run_idx[k] points into a permuted table req_tab / flags_tab that is larger than the CSR (the index
    gather form).
So the oracle's answer is the same for both, and for every staging geometry.

What the cases aim at:
  * table shapes the streaming forms cut up: N in {1, 31, 33, ...} (not multiples of 32), runs of empty nodes, one
    node holding all R entries, slices far longer than the largest staging chunk (1024 entries), table lengths that
    are not multiples of 16 (the bulk form's plain-load tail of flag bytes), row_ptr[0] > 0, R = 0 with N > 0, and
    a table of ~560 k nodes on which every warp of every geometry owns two or more 32-node groups (the path that
    fetches a group ahead; the per-thread form's threads then also take several nodes each);
  * the decisions of get_node_state (reference scaler.py:61-114): busy sums built in the oracle's operation order
    (left-to-right float64 adds, then fl(cap * 0.3) - util, no FMA) that land exactly on fl(cap_d * 0.3) --
    left == 0, under-utilised -- or one ulp above it -- left == -ulp, busy -- each in a different dimension on
    different nodes; non-busy pods with huge requests between the busy ones (they must not count); node ages equal
    to an idle threshold and one either side; unschedulable nodes on every branch; S in {1, 8, 64}.  A node type
    with a negative capacity (finite: the ABI accepts it) is the only way a node without busy pods is not
    under-utilised, i.e. the only way to IDLE_SCHEDULABLE.
`case()` reports what it built in c["hits"]; tests/test_idle_cases_cpu.py checks that the targets are hit.
"""
import functools

import numpy as np

PODF_BUSY, PODF_UNDRAINABLE = 1, 2
NODEF_UNSCHEDULABLE = 1
LARGEST_CHUNK = 1024  # entries: D = 2 with the 32 KB-per-warp bulk geometry

# name -> (N, S, recipe); N is rounded by the recipe only where stated
CASES = {
    "n1_all_entries": (1, 1, "one"),
    "n31": (31, 64, "ragged"),
    "n33": (33, 8, "ragged"),
    "ragged": (2477, 8, "ragged"),
    "row_ptr_offset": (517, 1, "ragged"),
    "empty_table": (70, 64, "empty"),
    "boundary": (3001, 64, "boundary"),
    "multigroup": (560037, 8, "sparse"),
}
# cases small enough to run everywhere at no cost; the CPU self-check runs all of them
NAMES = tuple(CASES)

# capacity rows (resized to D); row 3 has a negative first dimension (IDLE_SCHEDULABLE without busy pods)
CAPS = ([4.0, 16.0 * 2 ** 30, 110.0, 8.0, 0.7],
        [2.5, 7096762368.0, 250.0, 0.7, 3.3],
        [0.1, 3.3, 1e-3, 96.0, 4.0],
        [-0.5, 1e10, 110.0, 8.0, 16.0])


def _caps(D):
    return np.stack([np.resize(np.array(r, dtype=np.float64), D) for r in CAPS])


def thresh(cap):
    """fl(cap * 0.3): UTIL_THRESHOLD * capacity as the reference (and every kernel) rounds it"""
    return float(np.float64(cap) * np.float64(0.3))


def ordered_sum(vals):
    s = 0.0
    for v in vals:
        s = s + float(v)
    return s


def _last_addend(prefix, target):
    """a >= 0 with fl(fl(prefix) + a) == target, or None"""
    p = ordered_sum(prefix)
    a = target - p
    for _ in range(8):
        if a < 0:
            return None
        s = p + a
        if s == target:
            return a
        a = np.nextafter(a, np.inf) if s < target else np.nextafter(a, -np.inf)
    return None


def _base_values(rng, R, D):
    v = np.zeros((R, D))
    v[:, 0] = rng.integers(1, 400, size=R) * 1e-3                        # millicores
    if D > 1:
        v[:, 1] = rng.integers(1, 64, size=R).astype(np.float64) * float(2 ** 20)  # bytes
    if D > 2:
        v[:, 2:] = rng.integers(0, 3, size=(R, D - 2)) * (rng.random((R, D - 2)) < 0.3)
    return v


def _counts(rng, N, recipe):
    if recipe == "one":
        return np.array([3 * LARGEST_CHUNK + 437], dtype=np.int64)
    if recipe == "empty":
        return np.zeros(N, dtype=np.int64)
    if recipe == "sparse":
        c = rng.poisson(1.2, size=N).astype(np.int64)
        c[rng.random(N) < 0.3] = 0
        c[rng.integers(0, N, size=6)] = 3 * LARGEST_CHUNK + rng.integers(1, 200, size=6)
        return c
    c = rng.poisson(6.0, size=N).astype(np.int64)
    c[rng.random(N) < 0.25] = 0
    # runs of empty nodes (whole 32-node groups and more)
    for s in rng.integers(0, N, size=max(1, N // 300)):
        c[s:s + int(rng.integers(1, 100))] = 0
    heavy = rng.integers(0, N, size=max(1, N // 400))
    c[heavy] = rng.integers(3 * LARGEST_CHUNK + 1, 4 * LARGEST_CHUNK, size=len(heavy))
    return c


@functools.lru_cache(maxsize=None)
def case(name, D):
    N, S, recipe = CASES[name]
    rng = np.random.default_rng([D, len(name), sum(map(ord, name))])
    caps = _caps(D)
    K = caps.shape[0]
    counts = _counts(rng, N, recipe)
    node_type = rng.integers(0, K, size=N).astype(np.int32)
    node_flags = (rng.random(N) < 0.15).astype(np.uint8)
    thr = np.sort(rng.integers(30, 86400, size=S)).astype(np.int64)
    node_age = rng.integers(0, 2 * 86400, size=N).astype(np.int64)

    # decision-boundary nodes: 5 pods each, busy / non-busy alternating
    nb = {"one": 0, "empty": 0, "boundary": N // 3}.get(recipe, max(2, min(N // 8, 400)))
    bnodes = np.sort(rng.choice(N, size=nb, replace=False)) if nb else np.zeros(0, np.int64)
    if recipe == "ragged" and N >= 200:
        bnodes = bnodes[(bnodes < 64) | (bnodes >= 64 + 70)]
        counts[64:64 + 70] = 0                                             # two whole 32-node groups without pods
    counts[bnodes] = 5
    start = 5 if name == "row_ptr_offset" else 0
    row_ptr = np.zeros(N + 1, dtype=np.int64)
    row_ptr[0] = start
    np.cumsum(counts, out=row_ptr[1:])
    row_ptr[1:] += start
    if recipe == "ragged" and (row_ptr[-1] - start) % 16 == 0 and N > 0:
        j = int(np.nonzero(~np.isin(np.arange(N), bnodes))[0][0])
        counts[j] += 3                                                     # table length not a multiple of 16
        np.cumsum(counts, out=row_ptr[1:])
        row_ptr[1:] += start
    Rc = int(row_ptr[-1])
    req_run = _base_values(rng, Rc, D)
    flags_run = rng.integers(0, 4, size=Rc).astype(np.uint8)

    hits = {"left_zero": [], "left_ulp": [], "age_on_threshold": 0}
    for i, n in enumerate(bnodes):
        k0 = int(row_ptr[n])
        t = int(node_type[n])
        kind = "left_zero" if i % 2 == 0 else "left_ulp"
        if t == 3:
            node_type[n] = t = i % 3                                       # the negative capacity is not a boundary
        d = (i // 2) % D
        target = thresh(caps[t, d])
        if kind == "left_ulp":
            target = float(np.nextafter(target, np.inf))
        while True:
            a1, a2 = rng.random(2) * target * 0.3
            a3 = _last_addend([a1, a2], target)
            if a3 is not None:
                break
        rows = np.zeros((5, D))
        # other dimensions: well under their threshold (zero where the capacity is not positive)
        for e in range(D):
            if e != d:
                rows[[0, 2, 4], e] = max(thresh(caps[t, e]), 0.0) * 0.1
        rows[0, d], rows[2, d], rows[4, d] = a1, a2, a3
        rows[1, :] = 1e12                                                  # non-busy pods with huge requests
        rows[3, :] = np.abs(caps[t]) * 5.0 + 1.0
        undrain = i % 4 < 2
        flags = np.array([PODF_BUSY, PODF_UNDRAINABLE if undrain else 0, PODF_BUSY | (PODF_UNDRAINABLE if i % 8 == 1 else 0),
                          0, PODF_BUSY], dtype=np.uint8)
        req_run[k0:k0 + 5] = rows
        flags_run[k0:k0 + 5] = flags
        node_flags[n] = 1 if i % 3 == 0 else 0                             # unschedulable on every branch
        hits[kind].append((int(n), d))
    # ages on, just under and just over a threshold
    if N > 0:
        m = max(1, N // 5)
        an = rng.choice(N, size=m, replace=False)
        s = rng.integers(0, S, size=m)
        node_age[an] = thr[s] + rng.integers(-1, 2, size=m)
        hits["age_on_threshold"] = int(np.sum(node_age[an] == thr[s]))
    if recipe == "boundary":
        # nodes of the negative-capacity type without busy pods, schedulable, past every threshold
        idle = np.nonzero(counts == 0)[0][:8]
        if len(idle) < 8:
            idle = np.nonzero(~np.isin(np.arange(N), bnodes))[0][:8]
            for n in idle:
                flags_run[row_ptr[n]:row_ptr[n + 1]] &= ~np.uint8(PODF_BUSY)
        node_type[idle] = 3
        node_flags[idle] = 0
        node_age[idle] = thr[-1] + 1 + np.arange(len(idle))

    used0 = rng.integers(0, 5, size=(N, D)).astype(np.float64) * 0.125
    if N:
        used0[rng.random((N, D)) < 0.05] = -0.0

    # the gathered layout: same rows per node, scattered over a larger table
    nnz = Rc - start
    Rtab = Rc + 17
    perm = rng.permutation(Rtab)[:nnz].astype(np.int32)
    run_idx = np.zeros(Rc, dtype=np.int32)
    run_idx[start:] = perm
    req_tab = _base_values(rng, Rtab, D) * 1e6 + 1.0                       # rows no node points to: never read
    flags_tab = np.full(Rtab, PODF_BUSY, dtype=np.uint8)
    req_tab[perm] = req_run[start:]
    flags_tab[perm] = flags_run[start:]

    hits["max_slice"] = int(counts.max()) if N else 0
    hits["N"], hits["R"], hits["S"] = N, nnz, S
    return {"N": N, "D": D, "S": S, "row_ptr": row_ptr, "req_run": req_run, "flags_run": flags_run,
            "run_idx": run_idx, "req_tab": req_tab, "flags_tab": flags_tab, "cap_type": caps,
            "node_type": node_type, "node_flags": node_flags, "node_age": node_age, "thr": thr, "used0": used0,
            "hits": hits}


def identity_idx(c):
    return np.arange(c["req_run"].shape[0], dtype=np.int32)


def group_ends(c):
    """entry index (from row_ptr[0]) where each 32-node group's slice ends"""
    N, rp = c["N"], c["row_ptr"]
    return rp[np.minimum(np.arange(1, (N + 31) // 32 + 1) * 32, N)] - rp[0]


# ---- the dispatch table of csrc/acsfit_scan_plan.h, restated: (form, bytes per warp, warps per CTA) ----------------
PER_THREAD, GATHER, BULK = 0, 1, 2
BULK_CFGS = {0: (8192, 8), 1: (16384, 12), 2: (16384, 8), 3: (32768, 6), 4: (8192, 16)}
PIPELINE_DIMS = (2, 4, 8, 16)


def bulk_geometry(D, cfg):
    return (16384, 8) if D > 8 else BULK_CFGS.get(cfg, BULK_CFGS[4])


def gather_bytes(D, stream_bytes):
    if D <= 4 and stream_bytes <= 2048:
        return 2048
    if D <= 8 and stream_bytes <= 4096:
        return 4096
    return 8192


def chunk(bytes_per_warp, D):
    return bytes_per_warp // 2 // (8 * D)


def chunks_of(D):
    """every staging chunk size (entries) a streaming form can use at D"""
    if D not in PIPELINE_DIMS:
        return []
    out = {chunk(bulk_geometry(D, cfg)[0], D) for cfg in BULK_CFGS}
    out |= {chunk(gather_bytes(D, sb), D) for sb in (2048, 4096, 8192)}
    return sorted(out)
