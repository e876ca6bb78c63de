"""TEST INFRASTRUCTURE: seeded ticks whose pending-pod request table forces a chosen packed-rank layout.

The first-fit kernels are instantiated per packed-rank word count RW (0 = float64 compare scan, 1, 2 or 4; a
3-word layout is padded to 4), and `build_ranks` (csrc/acsfit.cu) picks RW from the number of DISTINCT request
values per dimension.  `synthetic.make_cluster` only produces a few dozen distinct values at D = 4 or 8, so it
reaches RW = 1 only.  `layout_case(D, U, ...)` builds a tick with exactly U[d] distinct values in dimension d,
drawn from the value families the quantity parser produces (k * 1e-3 millicores, k * 2**20 MiB, integers, 0.0),
plus the smallest subnormal and -0.0 (which the rank tables fold into +0.0).  Capacities sit on table values or
one ulp either side, and half the nodes start empty, so many node thresholds are exactly a table value -- the
case a wrong `<=` in the rank search or a wrong field width gets wrong.
"""
import numpy as np

MILLI = 1e-3
MIB = float(2 ** 20)
TINY = 5e-324  # the smallest subnormal double
RANK_CAP = 8192  # kRankCap (csrc/acsfit_kernels.cuh): more distinct values in a dimension -> float64 scan
SMALL_TABLE = 8  # tables up to this size: uniform requests, capacities and units are multiples of the largest value


# name -> (D, U, words): `words` is the word count the field layout needs (None: more than 128 bits), before the
# 3 -> 4 padding; the U = 8193 cases exceed the rank table instead
LAYOUTS = {
    "d2_rw1": (2, (5, 40), 1),
    "d2_rw1_u8192": (2, (8192, 8192), 1),                  # 2 x 15 bits
    "d2_f64_u8193": (2, (8193, 9), 1),
    "d4_rw1_guard31": (4, (127, 127, 127, 127), 1),        # 4 x 8 bits: the last guard bit is bit 31
    "d4_rw2": (4, (127, 127, 128, 127), 2),                # 2^7 - 1 against 2^7
    "d4_f64_u8193": (4, (8193, 7, 6, 2), 1),
    "d8_rw1": (8, (7, 6, 2, 1, 5, 5, 5, 5), 1),
    "d8_rw2": (8, (127,) * 8, 2),
    "d8_rw3_padded": (8, (511,) * 8, 3),                   # 3 words, launched as RW = 4
    "d8_rw4_u8192": (8, (8192,) * 8, 4),                   # 8 x 15 bits = 120
    "d8_f64_u8193": (8, (8193, 7, 6, 2, 1, 5, 5, 5), 2),
    "d16_rw1": (16, (1,) * 16, 1),                         # 16 x 2 bits: exactly one word
    "d16_rw2": (16, (3,) * 16, 2),
    "d16_rw4": (16, (127,) * 16, 4),
    "d16_f64_width": (16, (128,) * 16, None),              # 16 x 9 bits = 144: does not fit 128
}
CASE_P, CASE_N, CASE_T = 12000, 3500, 3


def case(name, seed=1):
    D, U, _ = LAYOUTS[name]
    return layout_case(D, U, CASE_P, CASE_N, CASE_T, seed=seed)


def family_values(d, n):
    """n distinct positive request values of dimension d, formed like the parser forms them (float(k) * unit)"""
    k = np.arange(1, n + 1, dtype=np.float64)
    fam = d % 3
    if fam == 0:
        return k * MILLI   # "250m"
    if fam == 1:
        return k * MIB     # "64Mi"
    return k               # gpus, pods, extended resources


def value_table(d, u):
    """the u distinct values of dimension d, ascending (distinct as the rank tables count: -0.0 == +0.0)"""
    if u == 1:
        return np.array([0.0]) if d % 2 == 0 else family_values(d, 1)
    specials = [0.0] + ([TINY] if u >= 3 and d % 2 == 1 else [])
    return np.concatenate([specials, family_values(d, u - len(specials))])


def distinct_count(col):
    """distinct values of one request column as the library counts them (bit patterns, -0.0 folded into +0.0)"""
    col = np.asarray(col, dtype=np.float64)
    return len(np.unique(np.where(col == 0.0, 0.0, col).view(np.uint64)))


def expected_rw(U, layout):
    """RW of the first-fit instantiation the request table selects; `layout` is tests/test_rank_math_cpu.layout"""
    if max(U) > RANK_CAP:
        return 0
    lay = layout(U)
    if lay is None:
        return 0
    return 4 if lay[2] == 3 else lay[2]


def _on_table(rng, tab, size):
    """capacities: table values from the middle of the table or, for small tables, small multiples of the largest
    value; a quarter of them moved one ulp down and a quarter one ulp up"""
    u = len(tab)
    if u <= SMALL_TABLE:
        v = tab[-1] * rng.choice([1.0, 2.0], size=size)
    else:
        v = tab[rng.integers(int(0.2 * (u - 1)), int(0.6 * (u - 1)) + 1, size=size)]
    side = rng.permutation(np.arange(size) % 4)  # 0, 1: on the value, 2: one ulp below, 3: one ulp above
    v = np.where(side == 2, np.nextafter(v, -np.inf), np.where(side == 3, np.nextafter(v, np.inf), v))
    return np.maximum(v, 0.0)  # capacities stay >= 0 (one ulp below 0.0 is -TINY)


def layout_case(D, U, P, N, T, seed, K=8):
    """a make_cluster-shaped tick whose P pending pods have exactly U[d] distinct values in dimension d.

    Pools (visiting order == unit_ordered): pool 0 dominates every other pool, so every feasible pod is eligible
    for it (the first bin pass can be chained behind the node pass); its size limit clips it after 300 bins, so
    the later pools pack the rest.  With T >= 3 the last pool is ignored.  `unit_all` lists the pools in reverse.
    """
    U = [int(u) for u in U]
    assert len(U) == D and P >= max(U) and T >= 2
    rng = np.random.Generator(np.random.PCG64(seed))
    tables = [value_table(d, u) for d, u in enumerate(U)]

    req = np.empty((P, D), dtype=np.float64)
    for d, tab in enumerate(tables):
        u = len(tab)
        skew = 1 if u <= SMALL_TABLE else 3                                   # large tables: mostly small requests
        idx = np.minimum((u * rng.random(P) ** skew).astype(np.int64), u - 1)
        idx[rng.permutation(P)[:u]] = np.arange(u)                         # every table value at least once
        col = tab[idx]
        col[(col == 0.0) & (rng.random(P) < 0.5)] = -0.0
        req[:, d] = col

    cap_type = np.empty((K, D), dtype=np.float64)
    for d, tab in enumerate(tables):
        cap_type[:, d] = _on_table(rng, tab, K)
    node_type = rng.integers(0, K, size=N).astype(np.int32)
    # half the nodes start empty (threshold == capacity); the others run one pod of small table values
    busy = rng.random(N) < 0.5
    used = np.zeros((N, D), dtype=np.float64)
    for d, tab in enumerate(tables):
        used[busy, d] = tab[np.minimum((len(tab) * rng.random(int(busy.sum())) ** 2).astype(np.int64), len(tab) - 1)]
    row_ptr = np.zeros(N + 1, dtype=np.int64)
    np.cumsum(busy.astype(np.int64), out=row_ptr[1:])
    req_run = used[busy].copy()
    R = req_run.shape[0]

    unit = np.empty((T, D), dtype=np.float64)
    for d, tab in enumerate(tables):
        u = len(tab)
        if u <= SMALL_TABLE:
            unit[0, d] = tab[-1] * 4.0
            unit[1:, d] = tab[-1] * 2.0
        else:
            unit[0, d] = tab[int(0.7 * (u - 1))]
            unit[1:, d] = tab[rng.integers(int(0.3 * (u - 1)), int(0.7 * (u - 1)), size=T - 1)]
        unit[1:, d] = np.where(rng.random(T - 1) < 0.3, np.nextafter(unit[1:, d], np.inf), unit[1:, d])
        unit[1:, d] = np.minimum(unit[1:, d], unit[0, d])  # pool 0 dominates: every feasible pod is eligible for it
    node_pool = (node_type % T).astype(np.int32)
    pool_actual = np.bincount(node_pool, minlength=T).astype(np.int32)
    pool_max = np.full(T, P + N + 1000, dtype=np.int32)
    pool_max[0] = pool_actual[0] + 300
    pool_ignored = np.zeros(T, dtype=np.uint8)
    if T >= 3:
        pool_ignored[T - 1] = 1
    return {
        "P": P, "N": N, "D": D, "T": T, "seed": seed, "U": tuple(U), "tables": tables,
        "req": req, "cap_type": cap_type, "node_type": node_type, "node_pool": node_pool,
        "row_ptr": row_ptr, "run_idx": np.arange(R, dtype=np.int32), "req_run": req_run,
        "flags_run": np.ones(R, dtype=np.uint8), "node_flags": np.zeros(N, dtype=np.uint8),
        "node_age": rng.integers(0, 86400, size=N).astype(np.int64),
        "unit_all": unit[::-1].copy(), "unit_ordered": unit,
        "pool_actual": pool_actual, "pool_max": pool_max, "pool_ignored": pool_ignored, "over_provision": 1,
    }


def node_thresholds(cap, used):
    """exact scan threshold of every (node, dimension): the largest r >= 0 with cap - (used + r) >= 0 (-1 if none),
    found by bisection over the bit patterns of the non-negative doubles with the literal float64 predicate --
    the same definition as acsfit::node_threshold (csrc/acsfit_math.cuh)"""
    cap = np.asarray(cap, dtype=np.float64)
    used = np.asarray(used, dtype=np.float64)

    def fits(r):
        return (cap - (used + r)) >= 0.0

    inf_bits = np.uint64(0x7FF0000000000000)
    lo = np.zeros(cap.shape, dtype=np.uint64)
    hi = np.full(cap.shape, inf_bits, dtype=np.uint64)
    with np.errstate(invalid="ignore", over="ignore"):
        for _ in range(64):
            mid = lo + (hi - lo) // np.uint64(2)
            f = fits(mid.view(np.float64))
            lo = np.where(f, mid, lo)
            hi = np.where(f, hi, mid)
        thr = lo.view(np.float64).copy()
        thr[~fits(np.zeros_like(cap))] = -1.0
    return thr
