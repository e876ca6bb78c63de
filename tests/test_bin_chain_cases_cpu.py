"""`-m "not gpu"`: every named case of tests/bin_chain_cases.py builds the dead-warp pattern it is named after (checked
with the C oracle), and the retirement model gives the expected counts on hand-built bins."""
import numpy as np
import pytest

import bin_chain_cases as bcc

CASES = bcc.cases()


@pytest.mark.parametrize("name", sorted(CASES))
def test_case_builds_its_pattern(oracle_mod, name):
    c = CASES[name]
    o, S = bcc.oracle_pass(oracle_mod, c)
    mr = bcc.minreq(c["req"])
    Tn = c["Tn"]
    for s, want in c["expect"].items():
        got = bcc.stage_dead_mask(S, mr, s * Tn, Tn)
        assert got == want, "%s stage %d: dead warps %#x, want %#x" % (name, s, got, want)
    # the stages after the patterned ones exist and something reaches them through the patterned stages' chains
    assert len(S) > len(c["expect"]) * Tn, (len(S), len(c["expect"]) * Tn)
    # the model over one pass of the case's planned width counts exactly the masks
    nst = (len(S) + Tn - 1) // Tn
    rec = [{"pass": 1, "RW": 1, "form": 0, "Tn": Tn, "stages": nst, "pool": 0, "bin_base": 0}]
    warps, stages = bcc.retirement(rec, {0: S}, mr)
    masks = [bcc.stage_dead_mask(S, mr, s * Tn, Tn) for s in range(nst)]
    assert warps == sum(bin(m).count("1") for m in masks)
    assert stages == sum(m == (1 << ((Tn + 31) // 32)) - 1 for m in masks)
    if name.startswith("sweep"):  # right after its openers, stage s has live warps = s: every non-full pattern
        nw = (Tn + 31) // 32
        n_st = (1 << nw) - 1
        S0 = bcc.remaining(c["req"][:n_st * Tn], o["bin_of"][:n_st * Tn], c["unit"])
        live = [n_st & ~bcc.stage_dead_mask(S0, mr, s * Tn, Tn) for s in range(n_st)]
        assert live == list(range(n_st))
        assert sum(c["expect"][s] != n_st - s for s in range(n_st)) > 0  # ... and probes changed some of them


def test_min_from_an_unseen_row_retires_less(oracle_mod):
    """the infeasible row (2 in the pattern dimension) keeps every 8-opened bin (2 left) live: stage 0 has no dead
    warp, while without that row all its warps would be dead"""
    c = CASES["min_from_infeasible_row"]
    o, S = bcc.oracle_pass(oracle_mod, c)
    assert o["bin_of"][0] == -1 and bcc.minreq(c["req"])[0] == 2.0
    assert bcc.stage_dead_mask(S, bcc.minreq(c["req"]), 0, 256) == 0
    assert bcc.stage_dead_mask(S, bcc.minreq(c["req"][1:]), 0, 256) == 0xFF


def test_last_live_warp_dies_while_an_earlier_one_lives(oracle_mod):
    """after the probes of 4 (the second tile) warp 5 is dead and warps 0-1 are live; at the end warp 1 alone lives"""
    c = CASES["last_live_dies_first"]
    req = c["req"]
    o, S = bcc.oracle_pass(oracle_mod, c)
    mr = bcc.minreq(req)
    S2 = bcc.remaining(req[:512], o["bin_of"][:512], c["unit"])
    assert bcc.stage_dead_mask(S2, mr, 0, 256) == 0xFF & ~0x03
    assert bcc.stage_dead_mask(S, mr, 0, 256) == 0xFF & ~0x02


def test_widths_cover_the_narrow_plans():
    widths = sorted(c["Tn"] for n, c in CASES.items() if n.startswith("width_"))
    assert widths[0] < 32 and widths[-1] == 256


def test_model_on_hand_built_bins():
    mr = np.array([3.0, 1.0])
    S = np.tile([10.0, 110.0], (300, 1))
    S[:64, 0] = 2.0          # warps 0-1 of stage 0 dead
    S[64:96, 0] = 3.0        # warp 2 live: exactly the minimum
    S[96:128, 1] = 0.0       # warp 3 dead through the pods column
    S[128:256, 0] = 0.5      # warps 4-7 dead
    S[256:288, 0] = 2.5      # stage 1 (Tn 256): warp 0 dead, warp 1 partly opened (bins 288-299), rest unopened
    S[288:300, 0] = 1.0
    rec = {"pass": 1, "RW": 1, "form": 0, "Tn": 256, "stages": 2, "pool": 0, "bin_base": 0}
    assert bcc.retirement([rec], {0: S}, mr) == (7 + 1, 0)
    S[64:96, 0] = 2.999
    assert bcc.retirement([rec], {0: S}, mr) == (8 + 1, 1)
    # a second pass of the same pool starts at bin_base; node passes, RW = 0 and the streaming form count nothing
    rec2 = dict(rec, stages=1, bin_base=256)
    off = [dict(rec, RW=0), dict(rec, form=1), dict(rec, **{"pass": 0})]
    assert bcc.retirement([rec2] + off, {0: S}, mr) == (1, 0)
    # stages narrower than 32 bins: one warp, padding lanes count as dead
    S8 = np.tile([10.0, 110.0], (20, 1))
    S8[:16, 0] = 2.0
    r8 = dict(rec, Tn=8, stages=3)
    assert bcc.retirement([r8], {0: S8}, mr) == (2, 2)
    # a zero minimum retires nothing through its dimension
    assert bcc.retirement([r8], {0: S8}, np.array([0.0, 1.0])) == (0, 0)
    # several pools: each record reads its own pool's bins
    assert bcc.retirement([dict(r8, pool=1), dict(r8, pool=0)], {0: S8, 1: S8[:8]}, mr) == (3, 3)
