"""`-m "not gpu"`: the named cluster-mode cases (tests/cluster_cases.py) are what their names say, on the oracle:
node ranges, feasible-pod and tile counts, where the placements fall, pod-block arithmetic, and non-trivial
placements and bins where a case needs both.  The closed-form answers of the multi-pass bin case equal the oracle
at a reduced size."""
import numpy as np
import pytest

import cluster_cases as cc
import variant_cases as vc

WORLDS = (2, 3, 4)


def ranges(N, world):
    return [(cc.lo_of(N, world, r), cc.lo_of(N, world, r + 1)) for r in range(world)]


def scale_up(oracle_mod, name, world):
    c = cc.build(name, world)
    return c, cc.oracle_call(oracle_mod, c, "scale_up")


def test_case_lists():
    assert set(cc.names(3)) == set(cc.names(4)) < set(cc.names(2)) == set(cc.CASES)
    assert {"layout_" + n for n in vc.LAYOUTS} <= set(cc.CASES)
    for name in cc.CASES:
        for call in cc.calls(name):
            assert call in ("scale_up", "scale_up_host", "ff_all", "ff_subset", "fulfill", "closed", "retire"), (name, call)


@pytest.mark.parametrize("name", sorted(n for n in cc.CASES if n.startswith("layout_")))
def test_layout_case(oracle_mod, name):
    D, U, _ = vc.LAYOUTS[name[len("layout_"):]]
    c, o = scale_up(oracle_mod, name, 2)
    assert [vc.distinct_count(c["req"][:, d]) for d in range(D)] == list(U)
    idx = c["pod_idx"]
    assert np.all(np.diff(idx) > 0) and 0 < len(idx) < c["req"].shape[0]
    # placements, pending pods (they cross every rank), bins in at least two pools
    assert (o["placed"] >= 0).sum() >= 20
    assert o["n_pending"] > 50 and (o["bins_opened"] > 0).sum() >= 2


@pytest.mark.parametrize("world", WORLDS)
def test_node_splits(oracle_mod, world):
    Ns = {name: cc.build(name, world)["N"] for name in cc.names(world) if name.startswith("nodes_")}
    assert Ns["nodes_0"] == 0 and Ns["nodes_1"] == 1 and Ns["nodes_world_minus_1"] == world - 1
    assert Ns["nodes_33"] == 33 and Ns["nodes_301"] == 301
    assert (Ns["nodes_2tn_minus_1"], Ns["nodes_2tn_plus_1"]) == (2 * cc.MIN_TN - 1, 2 * cc.MIN_TN + 1)
    for n in (1, world - 1):
        assert ranges(n, world)[0] == (0, 0)  # rank 0 owns no node
    assert all(0 < hi - lo < cc.MIN_TN for lo, hi in ranges(33, world))  # every rank: part of one stage
    for n in (2 * cc.MIN_TN - 1, 2 * cc.MIN_TN + 1, 301):
        assert any((hi - lo) % cc.MIN_TN for lo, hi in ranges(n, world))
    if world == 3:
        assert sorted({hi - lo for lo, hi in ranges(301, 3)}) == [100, 101]
    # each tick places pods and leaves some pending; with no node every feasible pod is pending
    for name in Ns:
        c, o = scale_up(oracle_mod, name, world)
        assert o["n_pending"] > 0 and o["bins_opened"].sum() > 0, name
        assert ((o["placed"] >= 0).sum() > 0) == (c["N"] > 0), name
        if c["N"] >= world:
            assert len({int(np.searchsorted([lo for lo, _ in ranges(c["N"], world)], p, "right")) - 1
                        for p in o["placed"][o["placed"] >= 0]}) >= 2, name


@pytest.mark.parametrize("F", [0, 1, 255, 256, 257])
def test_feasible_counts(oracle_mod, F):
    c, o = scale_up(oracle_mod, "feasible_%d" % F, 2)
    mask, _ = oracle_mod.feasible_mask(c["req"], c["unit_all"])
    assert int(mask.sum()) == F == o["n_to_schedule"]
    assert np.array_equal(mask.astype(bool), cc.feasible_rows(c["req"], c["unit_all"]))
    assert -(-F // cc.TILE) == {0: 0, 1: 1, 255: 1, 256: 1, 257: 2}[F]
    if F >= 255:
        assert (o["placed"] >= 0).sum() > 0 and o["n_pending"] > 0 and o["bins_opened"].sum() > 0


@pytest.mark.parametrize("world", WORLDS)
def test_placements_stay_in_rank0(oracle_mod, world):
    c, o = scale_up(oracle_mod, "rank0_only", world)
    placed = o["placed"][o["placed"] >= 0]
    assert len(placed) == o["n_to_schedule"] > 100 and o["n_pending"] == 0
    assert placed.max() == cc.lo_of(c["N"], world, 1) - 1 and placed.min() < placed.max()
    ff = cc.oracle_call(oracle_mod, c, "ff_all")
    assert np.all((ff["placed"] >= 0) & (ff["placed"] < cc.lo_of(c["N"], world, 1)))


def test_no_pod_fits_any_node(oracle_mod):
    c, o = scale_up(oracle_mod, "no_node_fits", 2)
    assert not (o["placed"] >= 0).any()
    assert o["n_pending"] == o["n_to_schedule"] > 100 and (o["bins_opened"] > 0).sum() >= 1
    assert o["decisions"] >= o["n_to_schedule"] * c["N"]  # every feasible pod tried every node
    assert not (cc.oracle_call(oracle_mod, c, "ff_all")["placed"] >= 0).any()


def test_pod_blocks(oracle_mod):
    c, o = scale_up(oracle_mod, "blocks_2", 2)
    tiles = -(-o["n_to_schedule"] // cc.TILE)
    assert tiles == cc.BLOCKS_TILES
    for k in cc.FORCED_BLOCKS:
        assert tiles % k != 0 or k > tiles
        assert cc.knobs("blocks_%d" % k) == {"cluster_blocks": k}
    assert cc.block_plan(tiles, 64) == (tiles, 1)  # 64 is clamped to the tile count
    assert cc.block_plan(tiles, 7) == (6, 2)       # ceil(11 / 7) = 2 tiles per block: 6 blocks
    assert cc.block_plan(tiles, 2) == (2, 6) and cc.block_plan(tiles, 3) == (3, 4)
    assert (o["placed"] >= 0).sum() > 100 and o["n_pending"] > 100
    for world in WORLDS:
        c = cc.build("blocks_auto", world)
        n_max = max(hi - lo for lo, hi in ranges(c["N"], world))
        assert -(-n_max // 128) > cc.H100_SMS * 1.2  # widest D = 16 stages: more than the GPU holds at once
        assert c["D"] == 16 and c["req"].shape[0] > 2 * cc.TILE
    c, o = scale_up(oracle_mod, "blocks_auto", 2)
    assert cc.block_plan(-(-o["n_to_schedule"] // cc.TILE), 4 * 2)[0] > 1
    placed = o["placed"][o["placed"] >= 0]
    assert len(placed) > 100 and placed.min() >= 3 * c["N"] // 4  # every pod crossed rank 0


@pytest.mark.parametrize("name", ["fulfill_d4", "fulfill_d8", "fulfill_d16"])
def test_fulfill_case(oracle_mod, name):
    c = cc.build(name, 2)
    f = c["fulfill"]
    assert f["num_listed"] > f["req"].shape[0] > 1000  # duplicates in the listed count
    o = cc.oracle_call(oracle_mod, c, "fulfill")
    assert o["units_needed"][1] == -1 and o["new_size"][1] == f["pool_actual"][1]  # ignored pool
    assert o["bins_opened"][0] > f["pool_max"][0] - f["pool_actual"][0]            # clipped by max_size
    assert o["new_size"][0] == f["pool_max"][0]
    assert (o["acc_pool"] == 0).any() and (o["acc_pool"] >= 2).any()
    assert o["num_unaccounted"] > 0 or (o["acc_pool"] >= 0).all()


@pytest.mark.parametrize("D", [4, 16])
def test_closed_form_equals_oracle(oracle_mod, D):
    for M, take in (cc.CLOSED_SMALL, (900, 700)):
        f = cc.closed_form_input(M, take, D)
        o = oracle_mod.fulfill_pending(f["req"], f["num_listed"], f["unit"], f["pool_actual"], f["pool_max"],
                                       f["pool_ignored"], f["over_provision"])
        want = cc.closed_form_answer(M, take)
        for k in ("bin_of", "acc_pool", "bins_opened", "units_needed", "new_size"):
            np.testing.assert_array_equal(o[k], want[k], err_msg=k)
        assert o["num_unaccounted"] == want["num_unaccounted"] and o["evals"] == want["evals"]
    M, take = cc.closed_full(2, cc.H100_SMS, cc.MIN_TN)
    first = 2 * cc.H100_SMS * cc.MIN_TN
    assert first < take < M < 2 * first  # pool 0 is cut inside the second pass


@pytest.mark.parametrize("world", WORLDS)
def test_retire_case(oracle_mod, world):
    """rank 0's bins and rank 1's stage 0 are all dead, rank 1's stage 0 dies inside the pass (later tiles follow),
    and the pods after it are placed on rank 1's later stages and, with three ranks or more, on rank 2"""
    import bin_chain_cases as bcc
    tn, S = cc.MIN_TN, cc.RETIRE_STAGES
    f = cc.retire_input(world, tn)
    M = f["req"].shape[0]
    assert -(-(-(-M // tn)) // world) == S  # the cluster plan: S stages of tn bins per rank
    o = oracle_mod.fulfill_pending(f["req"], f["num_listed"], f["unit"], f["pool_actual"], f["pool_max"],
                                   f["pool_ignored"], f["over_provision"])
    assert (o["bin_of"] >= 0).all() and o["bins_opened"][0] <= M  # one pass
    Sb = bcc.remaining(f["req"], o["bin_of"], f["unit"][0])
    mr = bcc.minreq(f["req"])
    assert all(bcc.stage_dead_mask(Sb, mr, s * tn, tn) == 1 for s in range(S + 1))
    last_opener = S * tn + tn - 1
    assert last_opener // cc.TILE < (M - 1) // cc.TILE  # tiles come after the stage retired
    rank1 = o["bin_of"][last_opener + 1:]
    assert (rank1 < world * S * tn).all() and ((rank1 >= (S + 1) * tn) & (rank1 < 2 * S * tn)).sum() > 100
    if world >= 3:
        assert (rank1 >= 2 * S * tn).sum() > 100
    rec = [{"pass": 1, "RW": 1, "form": 0, "Tn": tn, "stages": S, "pool": 0, "bin_base": 0}]
    per_rank = [bcc.retirement(rec, {0: Sb}, mr, rank=r) for r in range(world)]
    assert per_rank[0] == (S, S) and per_rank[1][1] >= 1
