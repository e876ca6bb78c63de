"""`-m "not gpu"`: the plain-C oracle of the topology-spread node pass (tests/ts_oracle.c) following a limited number
of rises, as the GPU pass does past its 4096th: a pinned worked case, the capped oracle against the unlimited one on
the overlays of tests/test_gpu_topology_spread.py, and the cases of tests/test_gpu_spread_reruns.py."""
import numpy as np
import pytest

import ts_oracle
from test_gpu_spread_reruns import (capped_keys_case, cap_case, first_and_last_case, flip_and_rise_case, keys64_case,
                                    spread_rule_violations, twin_keys_case)
from test_gpu_topology_spread import MAX_SPREAD_RISES, case

INT32_MAX = 2 ** 31 - 1


def nodes_pass(c, follow=None):
    used, count, has = c["used0"].copy(), c["ts_count0"].copy(), c["node_has0"].copy()
    nc, nx = c["node_carries0"].copy(), c["node_matches0"].copy()
    placed, calls, flips, rises = ts_oracle.first_fit_nodes_ts(
        c["req"], c["cap_type"], c["node_type"], used, c["ts_keys"], c["ts_key"], c["ts_skew"], c["ts_matches"],
        count, c["ts_domain"], c["ts_floor"], c["pa_requires"], c["pa_self"], c["pa_matches"], has,
        c["pod_carries"], c["pod_matches"], nc, nx, c.get("node_match"), c.get("pod_class"), follow=follow)
    return {"placed": placed, "calls": calls, "flips": flips, "rises": rises, "used": used, "count": count,
            "has": has, "nc": nc, "nx": nx}


def same(a, b):
    assert a["placed"].tolist() == b["placed"].tolist() and a["calls"] == b["calls"]
    assert a["flips"] == b["flips"] and a["rises"] == b["rises"]
    for k in ("used", "count", "has", "nc", "nx"):
        np.testing.assert_array_equal(a[k], b[k], err_msg=k)


def test_worked_case():
    c = cap_case()
    assert len(c["req"]) == 8400 and c["cap_type"].tolist() == [[1e6, 1e6]] * 2
    assert c["ts_floor"].tolist() == [INT32_MAX]
    assert c["ts_skew"].tolist() == [0] * 8400 and c["ts_matches"].tolist() == [1] * 8400
    free = nodes_pass(c)
    assert free["rises"] == [(0, p) for p in range(1, 8400, 2)] and free["placed"].tolist() == [0, 1] * 4200
    capped = nodes_pass(c, follow=4096)
    assert capped["rises"] == [(0, p) for p in range(1, 8192, 2)]
    placed = capped["placed"]
    assert placed[:8194].tolist() == [0, 1] * 4097 and (placed[8194:] == -1).all() and (placed < 0).sum() == 206
    assert capped["count"].tolist() == [[4097, 4097]]
    # the refused replicas need new nodes, one each (with every rise followed, none)
    pend = np.nonzero(placed < 0)[0]
    f = ts_oracle.fulfill_pending_ts(c["req"][pend], len(pend), c["unit"], c["pool_actual"], c["pool_max"],
                                     c["pool_ignored"], 0, 1, c["ts_key"][pend], c["ts_skew"][pend],
                                     c["ts_matches"][pend])
    assert f["bins_opened"].tolist() == [206] and f["num_unaccounted"] == 0


OVERLAYS = [(base, ts_kind, pa_kind, D) for base, ts_kind, pa_kind in
            [("replicas", "rises", "none"), ("replicas", "pinned", "none"), ("replicas", "rise1", "none"),
             ("with_sel", "keys64", "none"), ("with_sel", "flat", "none"), ("with_sel", "rises", "sig2"),
             ("with_sel", "pinned", "mixed")] for D in (2, 16)]


@pytest.mark.parametrize("key", OVERLAYS, ids=["-".join(map(str, k)) for k in OVERLAYS])
def test_follow_limits_on_the_overlays(key):
    c = case(*key)
    free = nodes_pass(c)
    n = len(free["rises"])
    for follow in (n, n + 1, MAX_SPREAD_RISES):  # a limit never reached: the unlimited pass
        same(nodes_pass(c, follow), free)
    if n == 0:
        return
    # one rise short: the same pass up to the pod of the rise left out, the rises before it, and no placement the
    # scheduler's rule refuses
    short = nodes_pass(c, n - 1)
    p = free["rises"][-1][1]
    assert short["rises"] == free["rises"][:-1]
    assert short["placed"][:p + 1].tolist() == free["placed"][:p + 1].tolist()
    assert spread_rule_violations(c, short["placed"]) == []
    none = nodes_pass(c, 0)
    assert none["rises"] == [] and spread_rule_violations(c, none["placed"]) == []


def test_capped_keys_case():
    c = capped_keys_case()
    free, capped = nodes_pass(c), nodes_pass(c, MAX_SPREAD_RISES)
    assert len(free["rises"]) > MAX_SPREAD_RISES and len(capped["rises"]) == MAX_SPREAD_RISES
    assert capped["flips"] == free["flips"] == [(0, 11002)]
    assert capped["rises"][-1][1] < 11000 and (capped["placed"] < 0).sum() > (free["placed"] < 0).sum()
    assert spread_rule_violations(c, capped["placed"]) == []


def test_one_position_cases():
    r = nodes_pass(twin_keys_case())
    assert r["rises"] == [(k, p) for p in range(1, 40, 2) for k in (0, 1)]
    r = nodes_pass(flip_and_rise_case())
    assert r["flips"] == [(0, 1)] and r["rises"][0] == (0, 1) and r["placed"][6:].tolist() == [1] * 6
    r = nodes_pass(first_and_last_case())
    assert r["rises"] == [(0, 0), (1, 511)] and r["placed"][-1] == 1


@pytest.mark.parametrize("D", [2, 16])
def test_keys64_case(D):
    r = nodes_pass(keys64_case(D))
    keys = [k for k, _ in r["rises"]]
    assert 63 in keys and len(set(keys)) == 64 and 300 <= len(keys) < MAX_SPREAD_RISES
    assert sum(a != b for a, b in zip(keys, keys[1:])) > len(keys) // 2
