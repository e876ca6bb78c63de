"""TEST INFRASTRUCTURE: named cluster-mode cases (include/acsfit.h, "Cluster mode"; DESIGN §5).

In cluster mode rank r of `world` owns nodes [N*r // world, N*(r+1) // world) and the r-th run of bins of every bin
pass; the stage pipeline continues from rank to rank through peer memory.  Each case here is one tick plus the calls
every rank makes on it, chosen for a piece of that geometry: rank layouts (tests/variant_cases.py), node ranges that
are empty or not a multiple of the stage width, feasible-pod counts on tile edges, pods that stay inside rank 0 or
cross every rank, forced and automatic pod blocks, forced pruning, fulfill_pending on its own and bin packing that
needs several cluster passes (closed form).  Some ticks depend on the world size or the GPU's SM count; `build`
takes both.  tests/test_cluster_cases_cpu.py checks on the oracle that each case is what its name says;
tests/test_gpu_cluster.py runs them.
"""
import numpy as np

import bin_chain_cases as bcc
import variant_cases as vc
from kubernetes_acs_engine_autoscaler_b200 import synthetic as syn

TILE = 256          # kTile (csrc/acsfit_kernels.cuh): pods per tile
MIN_TN = 32         # the narrowest cluster-mode stage
H100_SMS = 132      # SM count the CPU checks size the SM-dependent ticks with
MAX_BLOCKS = 64     # kClusterBlocks (csrc/acsfit.cu)
FORCED_BLOCKS = (2, 3, 7, 64)
BLOCKS_TILES = 11   # tile count of the forced-blocks tick: none of 2, 3, 7 divides it, 64 is clamped to it
CLOSED_UNIT = (1.5, 7096762368.0, 110.0, 8.0)


def lo_of(N, world, r):
    """first node of rank r's range (cluster_lo in csrc/acsfit.cu)"""
    return N * r // world


def max_stage_nodes(D):
    return 256 if D <= 8 else 128


def block_plan(tiles, k):
    """pod blocks of a node pass cut into at most k blocks: (blocks, tiles per block)"""
    blocks = min(MAX_BLOCKS, max(1, min(tiles, k)))
    tpb = -(-tiles // blocks)
    return -(-tiles // tpb), tpb


def feasible_rows(req, unit_all):
    """capacity.is_possible of every row over all pools: some pool's unit minus the request is >= 0 everywhere"""
    return np.any(np.all(unit_all[None, :, :] - req[:, None, :] >= 0.0, axis=2), axis=1)


def _with_used(c):
    c = dict(c)
    c["used0"] = syn.initial_used(c)
    return c


def _mc(P, N, D, T, seed, **kw):
    return _with_used(syn.make_cluster(P, N, D, T, seed=seed, over_provision=1, **kw))


def _layout(name, N=900, seed=2):
    """a layout tick of tests/variant_cases.py at the size of this matrix; pool 0's size limit is lowered to 40
    units so that the later pools pack bins too"""
    D, U, _ = vc.LAYOUTS[name]
    c = _with_used(vc.layout_case(D, U, max(2000, max(U) + 1000), N, 3, seed=seed))
    c["pool_max"] = c["pool_max"].copy()
    c["pool_max"][0] = c["pool_actual"][0] + 40
    return c


def _force_feasible(c, F, seed):
    """exactly F feasible pods (at random positions); every other pod requests more than any unit in every dimension"""
    c = dict(c)
    rng = np.random.Generator(np.random.PCG64(seed))
    req = c["req"].copy()
    ok = feasible_rows(req, c["unit_all"])
    good = req[ok]
    assert len(good) > 0
    keep = np.zeros(c["P"], dtype=bool)
    keep[rng.permutation(c["P"])[:F]] = True
    req[keep] = good[rng.integers(0, len(good), size=F)]
    req[~keep] = 2.0 * c["unit_all"].max(axis=0) + 1.0
    c["req"] = req
    return c


def _subset(c, seed, frac=0.6):
    """a sorted pod_idx subset of the pod list"""
    rng = np.random.Generator(np.random.PCG64(seed))
    idx = np.nonzero(rng.random(c["req"].shape[0]) < frac)[0].astype(np.int32)
    c = dict(c)
    c["pod_idx"] = idx
    return c


def _rank0_only(world, seed):
    """the last node of rank 0's range holds every pod: each feasible pod is placed in rank 0's range"""
    c = _mc(800, 400, 4, 2, seed)
    big = np.full((1, 4), 1e15)
    c["cap_type"] = np.concatenate([c["cap_type"], big])
    nt = c["node_type"].copy()
    nt[lo_of(c["N"], world, 1) - 1] = c["cap_type"].shape[0] - 1
    c["node_type"] = nt
    return c


def _no_node_fits(seed):
    """every node is over capacity in dimension 0: every feasible pod crosses every rank and goes to bins"""
    c = _mc(800, 400, 4, 2, seed)
    used0 = c["used0"].copy()
    used0[:, 0] = c["cap_type"][c["node_type"], 0] + 1.0
    c["used0"] = used0
    return c


def auto_blocks_nodes(world, sms):
    """nodes for which every rank needs more widest (128-node, D = 16) stages than the GPU holds at once (one stage
    CTA per SM at D = 16), with a quarter of margin"""
    return world * (128 * sms + 32 * sms)


def _auto_blocks(world, sms):
    """the first three quarters of the nodes are over capacity in dimension 0, so every pod crosses the ranks that
    own them before it is placed"""
    c = _with_used(vc.layout_case(16, (3,) * 16, 1200, auto_blocks_nodes(world, sms), 2, seed=5))
    full = 3 * c["N"] // 4
    c["used0"][:full, 0] = c["cap_type"][c["node_type"][:full], 0] + 1.0
    return c


def _fulfill(D, seed):
    """fulfill_pending on its own: the feasible pods of a tick, listed with 41 duplicates, pool 0 clipped by its size
    limit, pool 1 ignored, over-provisioning 2"""
    if D <= 8:
        c = _mc(3000, 10, D, 4, seed)
    else:
        c = _with_used(vc.layout_case(16, (3,) * 16, 3000, 10, 4, seed=seed))
    rows = c["req"][feasible_rows(c["req"], c["unit_all"])]
    T = c["unit_ordered"].shape[0]
    pool_actual = c["pool_actual"].copy()
    pool_max = np.full(T, 1 << 20, np.int32)
    pool_max[0] = pool_actual[0] + 50
    ignored = np.zeros(T, np.uint8)
    ignored[1] = 1
    c = dict(c)
    c["fulfill"] = {"req": np.ascontiguousarray(rows), "num_listed": len(rows) + 41, "unit": c["unit_ordered"],
                    "pool_actual": pool_actual, "pool_max": pool_max, "pool_ignored": ignored, "over_provision": 2}
    return c


def closed_form_input(M, take, D):
    """every pod requests the unit in dimension 0 only, so it opens its own bin after failing every earlier one;
    pool 0's size limit keeps `take` of them and pool 1 packs the rest the same way"""
    unit = np.resize(np.array(CLOSED_UNIT), D)
    req = np.zeros((M, D))
    req[:, 0] = unit[0]
    return {"req": req, "num_listed": M, "unit": np.stack([unit, unit]), "pool_actual": np.array([3, 1], np.int32),
            "pool_max": np.array([3 + take, 1 << 30], np.int32), "pool_ignored": np.zeros(2, np.uint8),
            "over_provision": 0}


def closed_form_answer(M, take):
    j = np.arange(M)
    rest = M - take
    return {"bin_of": np.where(j < take, j, j - take).astype(np.int32),
            "acc_pool": np.where(j < take, 0, 1).astype(np.int32),
            "bins_opened": np.array([M, rest], np.int64), "units_needed": np.array([M, rest], np.int64),
            "new_size": np.array([3 + take, 1 + rest], np.int64), "num_unaccounted": 0,
            "evals": M + M * (M - 1) // 2 + rest + rest * (rest - 1) // 2}


CLOSED_SMALL = (600, 400)   # (M, take) of the first, single-pass closed-form call
RETIRE_STAGES = 40          # stages per rank of the retiring bin pass (retire_input)


def retire_input(world, tn, S=RETIRE_STAGES):
    """fulfill_pending input whose single cluster bin pass has S stages of tn bins on every rank (world * S * tn pods,
    one pool, D = 4).  Openers of 8 in a unit of 10 fill every bin of rank 0 and of rank 1's stage 0 (2 left: dead, the
    call's minimum is 3), so rank 1's stage 0 retires in the tile of its last opener and passes every later tile on,
    copying the alive words it gets from rank 0 into rank 1's bitmap; the rest (big pods of 9 and probes of 3,
    tests/bin_chain_cases.py) places on rank 1's later stages and on the next ranks"""
    M = world * S * tn
    n_open = S * tn + tn
    rest = M - n_open
    col = [bcc.DEAD] * n_open + bcc.tail(rest // 3, rest - rest // 3)
    req = bcc.rows(col, 4)
    return {"req": req, "num_listed": M, "unit": bcc.unit_row(4).reshape(1, -1), "pool_actual": np.zeros(1, np.int32),
            "pool_max": np.array([1 << 30], np.int32), "pool_ignored": np.zeros(1, np.uint8), "over_provision": 0}


def closed_full(world, resident, tn):
    """(M, take) of a closed-form call whose pool 0 needs two cluster passes of world * resident * tn bins"""
    first = world * resident * tn
    return first + 5000, first + 2000


# name -> (builder(world, sms), calls, knobs, in the reduced list of worlds 3 and 4)
# calls: "scale_up", "scale_up_host", "ff_all" (first_fit_nodes over every row, pod_idx None), "ff_subset" (the
# tick's sorted pod_idx), "fulfill" (the tick's fulfill input), "closed" (the multi-pass closed form), "retire" (a
# bin pass in which a stage of rank 1 retires, retire_input sized from a small first call's stage width)
CASES = {}


def _add(name, builder, calls, knobs=None, reduced=False):
    CASES[name] = (builder, tuple(calls), dict(knobs or {}), reduced)


_REDUCED_LAYOUTS = ("d2_rw1", "d4_rw2", "d8_rw3_padded", "d16_f64_width")
_HOST_LAYOUTS = ("d2_f64_u8193", "d8_rw4_u8192", "d16_rw1")
for _n in sorted(vc.LAYOUTS):
    _add("layout_" + _n, lambda w, s, n=_n: _subset(_layout(n), 3),
         ("scale_up", "ff_subset") + (("scale_up_host",) if _n in _HOST_LAYOUTS else ()),
         reduced=_n in _REDUCED_LAYOUTS)

# node splits
_add("nodes_0", lambda w, s: _mc(1500, 0, 4, 2, 11), ("scale_up", "ff_all", "scale_up_host"), reduced=True)
_add("nodes_1", lambda w, s: _subset(_mc(1500, 1, 4, 2, 12), 4), ("scale_up", "ff_subset"), reduced=True)
_add("nodes_world_minus_1", lambda w, s: _mc(1500, max(1, w - 1), 4, 2, 13), ("scale_up", "ff_all"), reduced=True)
_add("nodes_33", lambda w, s: _subset(_mc(1500, 33, 8, 3, 14), 5), ("scale_up", "ff_subset"), reduced=True)
_add("nodes_2tn_minus_1", lambda w, s: _mc(1500, 2 * MIN_TN - 1, 4, 2, 15), ("scale_up", "ff_all"), reduced=True)
_add("nodes_2tn_plus_1", lambda w, s: _mc(1500, 2 * MIN_TN + 1, 4, 2, 16), ("scale_up", "scale_up_host"), reduced=True)
_add("nodes_301", lambda w, s: _subset(_mc(2500, 301, 8, 3, 17), 6), ("scale_up", "ff_subset"), reduced=True)

# pod edges
for _f in (0, 1, 255, 256, 257):
    _add("feasible_%d" % _f, lambda w, s, f=_f: _force_feasible(_mc(600, 40, 8, 3, 20 + f), f, 21 + f),
         ("scale_up",) + (("scale_up_host",) if _f == 0 else ()), reduced=_f in (0, 1, 257))
_add("rank0_only", lambda w, s: _rank0_only(w, 30), ("scale_up", "ff_all"), reduced=True)
_add("no_node_fits", lambda w, s: _no_node_fits(31), ("scale_up", "ff_all"), reduced=True)

# pod blocks: forced (tile count BLOCKS_TILES) and automatic
for _k in FORCED_BLOCKS:
    _add("blocks_%d" % _k, lambda w, s: _force_feasible(_mc(2750, 1100, 8, 3, 40), 2700, 41),
         ("scale_up",) + (("ff_all",) if _k == 3 else ()), {"cluster_blocks": _k}, reduced=_k == 7)
_add("blocks_auto", _auto_blocks, ("scale_up",), reduced=True)

# forced pruning of the node pass
_add("prune_d8_rw2", lambda w, s: _layout("d8_rw2", seed=7), ("scale_up",), {"prune": 1}, reduced=True)
_add("prune_d16_rw2", lambda w, s: _layout("d16_rw2", seed=8), ("scale_up",), {"prune": 1})
_add("prune_nodes_301", lambda w, s: _mc(2500, 301, 4, 2, 18), ("scale_up",), {"prune": 1})

# fulfill_pending on its own, and bin packing across several cluster passes
_add("fulfill_d4", lambda w, s: _fulfill(4, 50), ("fulfill",), reduced=True)
_add("fulfill_d8", lambda w, s: _fulfill(8, 51), ("fulfill",))
_add("fulfill_d16", lambda w, s: _fulfill(16, 52), ("fulfill",))
_add("bins_closed_d16", lambda w, s: {"D": 16, "N": 0}, ("closed",), reduced=True)

# bin retirement: rank 1's stage 0 retires while later stages place (and once with retirement off)
_add("retire_rank1", lambda w, s: {"D": 4, "N": 0}, ("retire",), reduced=True)
_add("retire_rank1_off", lambda w, s: {"D": 4, "N": 0}, ("retire",), {"retire": 0}, reduced=True)


def oracle_call(oracle, c, call):
    """the oracle's answer to one call on tick c (every rank must return exactly this)"""
    if call in ("closed", "retire"):
        raise ValueError("the %s calls are sized on the GPU: answer them with their input" % call)
    if call == "fulfill":
        f = c["fulfill"]
        return oracle.fulfill_pending(f["req"], f["num_listed"], f["unit"], f["pool_actual"], f["pool_max"],
                                      f["pool_ignored"], f["over_provision"])
    used = c["used0"].copy()
    if call in ("ff_all", "ff_subset"):
        rows = c["req"] if call == "ff_all" else c["req"][c["pod_idx"]]
        placed, calls_ = oracle.first_fit_nodes(rows, c["cap_type"], c["node_type"], used)
        return {"placed": placed, "decisions": calls_, "used": used}
    # scale_up / scale_up_host: get_pods_to_schedule + get_pending_pods + fulfill_pending
    mask, ev0 = oracle.feasible_mask(c["req"], c["unit_all"])
    feas = np.nonzero(mask)[0]
    placed_f, ev1 = oracle.first_fit_nodes(c["req"][feas], c["cap_type"], c["node_type"], used)
    P = c["req"].shape[0]
    placed = np.where(mask.astype(bool), -1, -2).astype(np.int32)
    placed[feas] = placed_f
    pend = feas[placed_f < 0]
    T = c["unit_ordered"].shape[0]
    res = {"feasible": mask, "placed": placed, "acc_pool": np.full(P, -1, np.int32),
           "new_size": c["pool_actual"].astype(np.int64), "units_needed": np.full(T, -1, np.int64),
           "bins_opened": np.zeros(T, np.int64), "n_to_schedule": len(feas), "n_pending": len(pend),
           "num_unaccounted": 0, "decisions": ev0 + ev1, "used": used}
    if len(pend):
        f = oracle.fulfill_pending(c["req"][pend], len(pend), c["unit_ordered"], c["pool_actual"], c["pool_max"],
                                   c["pool_ignored"], c["over_provision"])
        res["acc_pool"][pend] = f["acc_pool"]
        for k in ("new_size", "units_needed", "bins_opened", "num_unaccounted"):
            res[k] = f[k]
        res["decisions"] += f["evals"]
    return res


def names(world):
    """the cases a world runs: all of them on 2 ranks, the reduced list on more"""
    return [n for n, (_, _, _, red) in CASES.items() if world == 2 or red]


def build(name, world, sms=H100_SMS):
    return CASES[name][0](world, sms)


def calls(name):
    return CASES[name][1]


def knobs(name):
    return CASES[name][2]
