"""`-m "not gpu"`: the layout-forcing generator (tests/variant_cases.py) hits its targets -- exact distinct counts,
the intended rank layout, thresholds on and one ulp beside table values, and a non-trivial tick on the oracle."""
import numpy as np
import pytest

import variant_cases as vc
from test_rank_math_cpu import layout


@pytest.mark.parametrize("name", sorted(vc.LAYOUTS))
def test_layout_case_hits_its_targets(oracle_mod, name):
    D, U, words = vc.LAYOUTS[name]
    c = vc.case(name)
    req = c["req"]
    assert req.shape == (vc.CASE_P, D)
    # exactly U[d] distinct values per dimension, counted like the rank tables count them
    assert [vc.distinct_count(req[:, d]) for d in range(D)] == list(U)
    # the parser's families plus the specials: -0.0 next to +0.0, the smallest subnormal where the table has room
    assert np.all(req >= 0.0)
    assert np.signbit(req[req == 0.0]).any() and (~np.signbit(req[req == 0.0])).any()
    if max(U) >= 3:
        assert (req == vc.TINY).any()
    # the layout the rank-layout rule predicts has the intended word count
    lay = layout(U)
    assert (None if lay is None else lay[2]) == words
    want_rw = 0 if words is None or max(U) > vc.RANK_CAP else (4 if words == 3 else words)
    assert vc.expected_rw(U, layout) == want_rw

    # node thresholds exactly on a table value, and one ulp either side of one
    used0 = np.zeros((c["N"], D))
    used0[np.repeat(np.arange(c["N"]), np.diff(c["row_ptr"]))] = c["req_run"]
    thr = vc.node_thresholds(c["cap_type"][c["node_type"]], used0)
    on = below = above = 0
    for d, tab in enumerate(c["tables"]):
        on += np.isin(thr[:, d], tab).sum()
        below += np.isin(np.nextafter(thr[:, d], np.inf), tab).sum()
        above += np.isin(np.nextafter(thr[:, d], -np.inf), tab).sum()
    assert on >= c["N"] * D // 20, on
    assert below > 0 and above > 0

    # a non-trivial tick: pods placed and pending, some infeasible or not, bins opened in at least two pools
    used_o = used0.copy()
    mask, _ = oracle_mod.feasible_mask(req, c["unit_all"])
    feas = np.nonzero(mask)[0]
    placed, _ = oracle_mod.first_fit_nodes(req[feas], c["cap_type"], c["node_type"], used_o)
    pend = feas[placed < 0]
    assert (placed >= 0).sum() > 100 and len(pend) > 500
    f = oracle_mod.fulfill_pending(req[pend], len(pend), c["unit_ordered"], c["pool_actual"], c["pool_max"],
                                   c["pool_ignored"], c["over_provision"])
    assert (f["bins_opened"] > 0).sum() >= 2, f["bins_opened"]
    assert f["bins_opened"][0] > 300  # pool 0 is clipped by its size limit
