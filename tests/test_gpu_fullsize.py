"""`-m gpu`: BASELINE.json's full sizes.
C2 (100k x 10k x 4, 1 pool) is small enough for the plain-C oracle (~2 s): exact comparison.
C3 (1M x 100k x 8, 8 pools) is checked through size-independent properties of sequential first fit
(prefix exactness against the oracle, state = ordered sum of the placed requests, idempotence on the
pending pods, split-run equivalence, decision count recomputed from the placement)."""
import numpy as np
import pytest
import torch

import bin_chain_cases as bcc
from kubernetes_acs_engine_autoscaler_b200 import synthetic as syn
from test_gpu_parity import bits, oracle_scale_up, to_np

pytestmark = pytest.mark.gpu


def test_c2_full_tick_matches_oracle(engine, oracle_mod):
    """the c2 tick, exactly against the oracle with bin retirement on and off.  Its bin pass opens about 30 k bins,
    almost all of them dead by the end: what retirement reports (dead warps, retired stages) must equal the model of
    tests/bin_chain_cases.py over the oracle's bins, and be nearly every warp of the pass"""
    c = syn.make_cluster(100000, 10000, 4, 1, seed=20260923)
    used0 = syn.initial_used(c)
    used_o = used0.copy()
    o = oracle_scale_up(oracle_mod, c, used_o)
    pend = np.nonzero(o["placed"] == -1)[0]
    f = oracle_mod.fulfill_pending(c["req"][pend], len(pend), c["unit_ordered"], c["pool_actual"], c["pool_max"],
                                   c["pool_ignored"], c["over_provision"])
    S = {0: bcc.remaining(c["req"][pend], f["bin_of"], c["unit_ordered"][0])}
    assert len(S[0]) == o["bins_opened"][0] > 25000
    try:
        for retire in (1, 0):
            engine.set_knob("retire", retire)
            used_h = used0.copy()
            h = engine.scale_up_host(c["req"], c["unit_all"], c["unit_ordered"], c["pool_actual"], c["pool_max"],
                                     c["pool_ignored"], c["over_provision"], c["cap_type"], c["node_type"], used_h)
            for k in ("feasible", "placed", "acc_pool", "new_size", "units_needed", "bins_opened"):
                np.testing.assert_array_equal(h[k], o[k], err_msg="%s (retire=%d)" % (k, retire))
            for k in ("n_to_schedule", "n_pending", "num_unaccounted", "decisions"):
                assert h[k] == o[k], (k, retire)
            np.testing.assert_array_equal(bits(used_h), bits(used_o))
            recs = engine.last_launches()
            got = engine.last_bin_retirement()
            want = bcc.retirement(recs, S, bcc.minreq(c["req"])) if retire else (0, 0)
            assert got == want, (retire, got, want, [r for r in recs if r["pass"] == 1])
            if retire and all(r["RW"] > 0 and r["form"] == 0 for r in recs if r["pass"] == 1):
                assert got[0] > 0.9 * len(S[0]) / 32, got  # nearly every warp over the opened bins is dead
    finally:
        engine.set_knob("retire", 1)
    assert o["decisions"] > 1.5e9  # the configuration the metric is quoted on


_C3_SHAPED = {}


def c3_shaped_oracle(oracle_mod):
    """the snapshot and the oracle's answer, computed once per process (the oracle needs about a minute) and shared by
    every engine mode"""
    if not _C3_SHAPED:
        c = syn.make_cluster(500000, 50000, 8, 8, seed=20260925)
        used0 = syn.initial_used(c)
        used_o = used0.copy()
        _C3_SHAPED.update(c=c, used0=used0, o=oracle_scale_up(oracle_mod, c, used_o), used_o=used_o)
    return _C3_SHAPED["c"], _C3_SHAPED["used0"], _C3_SHAPED["o"], _C3_SHAPED["used_o"]


def test_c3_shaped_tick_matches_oracle_exactly(engine, oracle_mod):
    """BASELINE config 3's SHAPE (8 dims, 8 pools, multi-wave node pass, several bin passes and pools) at half its
    size -- 500 k pods x 50 k nodes, about 30 G reference decisions -- compared EXACTLY with the plain-C oracle, in
    every engine mode."""
    c, used0, o, used_o = c3_shaped_oracle(oracle_mod)
    f64, i32 = torch.float64, torch.int32
    d_used = engine.dev(used0, f64)
    g = engine.scale_up(engine.dev(c["req"], f64), c["unit_all"], c["unit_ordered"], c["pool_actual"], c["pool_max"],
                        c["pool_ignored"], c["over_provision"], engine.dev(c["cap_type"], f64),
                        engine.dev(c["node_type"], i32), d_used)
    for k in ("feasible", "placed", "acc_pool"):
        np.testing.assert_array_equal(to_np(g[k]), o[k], err_msg=k)
    for k in ("new_size", "units_needed", "bins_opened"):
        np.testing.assert_array_equal(g[k], o[k], err_msg=k)
    for k in ("n_to_schedule", "n_pending", "num_unaccounted", "decisions"):
        assert g[k] == o[k], k
    np.testing.assert_array_equal(bits(to_np(d_used)), bits(used_o))
    assert o["decisions"] > 2e10 and (o["bins_opened"] > 0).sum() >= 3 and o["n_pending"] > 100000


def ordered_used(used0, req, placed):
    """used after counting the placed pods in pod order (numpy, host): the reference's count_pod."""
    used = used0.copy()
    idx = np.nonzero(placed >= 0)[0]
    node = placed[idx]
    order = np.argsort(node, kind="stable")  # keeps pod order inside every node
    idx, node = idx[order], node[order]
    starts = np.nonzero(np.r_[True, node[1:] != node[:-1]])[0]
    counts = np.diff(np.r_[starts, len(node)])
    for k in range(int(counts.max()) if len(counts) else 0):
        sel = counts > k
        used[node[starts[sel]]] = used[node[starts[sel]]] + req[idx[starts[sel] + k]]
    return used


def test_c3_first_fit_properties(engine, oracle_mod):
    P, N, D, T = 1000000, 100000, 8, 8
    c = syn.make_cluster(P, N, D, T, seed=20260924)
    used0 = syn.initial_used(c)
    f64, i32 = torch.float64, torch.int32
    d_req, d_cap, d_type = engine.dev(c["req"], f64), engine.dev(c["cap_type"], f64), engine.dev(c["node_type"], i32)
    d_used = engine.dev(used0, f64)
    placed, dec = engine.first_fit_nodes(d_req, None, d_cap, d_type, d_used)
    placed = to_np(placed)
    used = to_np(d_used)
    # (1) the credited decision count is a function of the placement
    assert int(to_np(dec)[0]) == int(np.where(placed >= 0, placed.astype(np.int64) + 1, N).sum())
    # (2) the node state is the ordered sum of exactly the placed requests, bit for bit, and never overflows
    np.testing.assert_array_equal(bits(ordered_used(used0, c["req"], placed)), bits(used))
    assert (c["cap_type"][c["node_type"]] - used >= 0).all()
    # (3) sequential first fit is prefix-exact: the first K pods are placed as the oracle places them
    K = 40000
    used_o = used0.copy()
    placed_o, _ = oracle_mod.first_fit_nodes(c["req"][:K], c["cap_type"], c["node_type"], used_o)
    np.testing.assert_array_equal(placed[:K], placed_o)
    # (4) idempotence: nodes only fill up, so the pending pods still fit nowhere in the final state
    pend = np.nonzero(placed < 0)[0].astype(np.int32)
    d_used2 = d_used.clone()
    again, _ = engine.first_fit_nodes(d_req, engine.dev(pend, i32), d_cap, d_type, d_used2)
    assert (to_np(again) == -1).all()
    np.testing.assert_array_equal(bits(to_np(d_used2)), bits(used))
    # (5) running the list in two pieces on the carried state equals one run
    d_used3 = engine.dev(used0, f64)
    cut = 456789
    a, _ = engine.first_fit_nodes(d_req, engine.dev(np.arange(cut, dtype=np.int32), i32), d_cap, d_type, d_used3)
    b, _ = engine.first_fit_nodes(d_req, engine.dev(np.arange(cut, P, dtype=np.int32), i32), d_cap, d_type, d_used3)
    np.testing.assert_array_equal(np.concatenate([to_np(a), to_np(b)]), placed)
    np.testing.assert_array_equal(bits(to_np(d_used3)), bits(used))


def test_c3_fulfill_properties(engine, oracle_mod):
    P, D, T = 600000, 8, 8
    c = syn.make_cluster(P, 64, D, T, seed=20260925)
    g = engine.fulfill_pending(engine.dev(c["req"], torch.float64), P, c["unit_ordered"], c["pool_actual"],
                               c["pool_max"], c["pool_ignored"], 1)
    acc, bin_of = to_np(g["acc_pool"]), to_np(g["bin_of"])
    unit = c["unit_ordered"]
    assert g["num_unaccounted"] == int((acc < 0).sum())
    for t in range(T):
        sel = acc == t
        if not sel.any():
            assert g["bins_opened"][t] == 0 or g["units_needed"][t] >= 0
            continue
        b = bin_of[sel]
        # bins are a dense prefix, every pod is eligible for its pool, and no bin is over-committed
        assert b.min() == 0 and len(np.unique(b)) == b.max() + 1 == g["bins_opened"][t]
        assert (unit[t] - c["req"][sel] >= 0).all()
        load = np.zeros((b.max() + 1, D))
        np.add.at(load, b, c["req"][sel])
        assert (load <= unit[t] * (1 + 1e-12)).all()
        assert g["new_size"][t] == c["pool_actual"][t] + g["units_needed"][t]
    # first-fit is prefix-exact here too: the oracle on the first K pods opens the same bins for them
    K = 30000
    o = oracle_mod.fulfill_pending(c["req"][:K], K, unit, c["pool_actual"], c["pool_max"], c["pool_ignored"], 1)
    first_pool = int(np.nonzero(g["units_needed"] >= 0)[0][0])
    sel = o["acc_pool"] == first_pool
    np.testing.assert_array_equal(bin_of[:K][sel], o["bin_of"][sel])


def test_c5_idle_scan_matches_oracle(engine, oracle_mod):
    """BASELINE config 5 at its full size: 1 M nodes, ~10 M running pods, 8 idle thresholds (the C oracle needs about a
    second per kernel for it), then the maintain decisions in both modes; plus the occupancy sums."""
    c = syn.make_idle_cluster(1000000, 8, 8, seed=31)
    thr = np.array([60, 300, 900, 1800, 3600, 7200, 21600, 86400], dtype=np.int64)
    st_o = oracle_mod.node_states(c["row_ptr"], c["run_idx"], c["req_run"], c["flags_run"], c["cap_type"],
                                  c["node_type"], c["node_flags"], c["node_age"], False, thr)
    i64, i32, f64, u8 = torch.int64, torch.int32, torch.float64, torch.uint8
    d_ptr, d_idx, d_req = engine.dev(c["row_ptr"], i64), engine.dev(c["run_idx"], i32), engine.dev(c["req_run"], f64)
    st = engine.node_states(d_ptr, d_idx, d_req, engine.dev(c["flags_run"], u8), engine.dev(c["cap_type"], f64),
                            engine.dev(c["node_type"], i32), engine.dev(c["node_flags"], u8),
                            engine.dev(c["node_age"], i64), False, thr)
    np.testing.assert_array_equal(to_np(st), st_o)
    assert len(np.unique(st_o)) >= 5
    # run_idx = NULL: the same table declared contiguous -> the bulk-copy streaming kernel (acsfit_stream.cuh)
    assert np.array_equal(c["run_idx"], np.arange(len(c["run_idx"])))
    st_b = engine.node_states(d_ptr, None, d_req, engine.dev(c["flags_run"], u8), engine.dev(c["cap_type"], f64),
                              engine.dev(c["node_type"], i32), engine.dev(c["node_flags"], u8),
                              engine.dev(c["node_age"], i64), False, thr)
    np.testing.assert_array_equal(to_np(st_b), st_o)
    budget = np.array([3, 0, 10 ** 6, -1, 5, 17, 0, 250], dtype=np.int64)
    scal = np.array([1, 1, 1, 1, 0, 1, 1, 1], dtype=np.uint8)
    for dry_run in (True, False):
        s_o, a_o = oracle_mod.maintain_actions(st_o[3], c["node_pool"], budget, scal, dry_run)
        s_g, a_g = engine.maintain_actions(engine.dev(st_o[3].copy(), u8), engine.dev(c["node_pool"], i32), budget,
                                           scal, dry_run)
        np.testing.assert_array_equal(to_np(s_g), s_o)
        np.testing.assert_array_equal(to_np(a_g), a_o)
    used_o = np.zeros((c["N"], 8))
    oracle_mod.occupancy(c["row_ptr"], c["run_idx"], c["req_run"], used_o)
    d_used = engine.dev(np.zeros((c["N"], 8)), f64)
    engine.occupancy(d_ptr, d_idx, d_req, d_used)
    np.testing.assert_array_equal(bits(to_np(d_used)), bits(used_o))
    d_used_b = engine.dev(np.zeros((c["N"], 8)), f64)
    engine.occupancy(d_ptr, None, d_req, d_used_b)
    np.testing.assert_array_equal(bits(to_np(d_used_b)), bits(used_o))
    # a shuffled pod list (run_idx is a gather, as in the real host layer) gives the same states
    perm = np.random.default_rng(1).permutation(c["req_run"].shape[0])
    inv = np.empty_like(perm)
    inv[perm] = np.arange(len(perm))
    st2 = engine.node_states(d_ptr, engine.dev(inv[c["run_idx"]].astype(np.int32), i32),
                             engine.dev(c["req_run"][perm], f64), engine.dev(c["flags_run"][perm], u8),
                             engine.dev(c["cap_type"], f64), engine.dev(c["node_type"], i32),
                             engine.dev(c["node_flags"], u8), engine.dev(c["node_age"], i64), False, thr)
    np.testing.assert_array_equal(to_np(st2), st_o)
