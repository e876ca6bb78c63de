"""`-m gpu`: every compiled form and staging geometry of the idle-scan kernels K1 (occupancy) and K6 (node states)
against the plain-C oracle, with proof from the launch record that it ran; then misaligned tables (the per-thread
fall-back), the first-fit entry points' alignment check, and the per-pool ranking of maintain_actions.

acsfit_scan_plan.h picks the form at run time: the bulk-copy form (contiguous table) in one of five geometries
(knob "bulk_cfg", D <= 8; one geometry at D = 16), the index-gather form (run_idx given) at 2048 / 4096 / 8192
staging bytes per warp (knob "stream_bytes"), or the per-thread form for every other D.  Each row of that table
runs every case of tests/idle_cases.py, compared exactly with the oracle -- `used` as uint64 bit patterns, states
byte for byte -- and Engine.last_scan_launch() must show the intended form, bytes, warps and chunk: a silent
fall-back to another geometry or form fails the case even when the answer is right."""
import functools

import numpy as np
import pytest
import torch

import idle_cases as ic
from kubernetes_acs_engine_autoscaler_b200._native import E_INVALID, AcsfitError

pytestmark = pytest.mark.gpu

DEFAULT_KNOBS = {"bulk_cfg": 4, "stream_bytes": 8192}

# (form, D, knobs, bytes per warp, warps per CTA)
ROWS = [(ic.BULK, D, {"bulk_cfg": cfg}) + ic.bulk_geometry(D, cfg) for D in (2, 4, 8) for cfg in sorted(ic.BULK_CFGS)]
ROWS += [(ic.BULK, 16, {}) + ic.bulk_geometry(16, 4)]
ROWS += [(ic.GATHER, D, {"stream_bytes": sb}, sb, 8) for D in (2, 4, 8, 16) for sb in (2048, 4096, 8192)
         if ic.gather_bytes(D, sb) == sb]
ROWS += [(ic.PER_THREAD, D, {}, 0, 4) for D in (1, 3, 5, 12, 15)]
ROW_IDS = ["%s_D%d_%s" % ({0: "thread", 1: "gather", 2: "bulk"}[r[0]], r[1], "%dx%d" % (r[3], r[4])) for r in ROWS]


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def to_np(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def eng():
    """one Engine for the module: the scan does not depend on the session fixture's scan modes"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from kubernetes_acs_engine_autoscaler_b200 import build as acs_build
    acs_build.build()
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    e = Engine(0)
    for k, v in DEFAULT_KNOBS.items():
        e.set_knob(k, v)
    yield e
    e.close()


@functools.lru_cache(maxsize=None)
def oracle_answers(name, D):
    """K1 and K6 (both any_pending values) of one case, plus maintain (first threshold); geometry-independent"""
    import oracle
    c = ic.case(name, D)
    idx = ic.identity_idx(c)
    used = c["used0"].copy()
    oracle.occupancy(c["row_ptr"], idx, c["req_run"], used)
    st = {ap: oracle.node_states(c["row_ptr"], idx, c["req_run"], c["flags_run"], c["cap_type"], c["node_type"],
                                 c["node_flags"], c["node_age"], ap, c["thr"]) for ap in (False, True)}
    pool = (c["node_type"] % 3).astype(np.int32)
    budget = np.array([3, 0, 1 << 40], dtype=np.int64)
    ms, ma = oracle.maintain_actions(st[False][0], pool, budget, np.ones(3, np.uint8), False)
    return used, st, (pool, budget, ms, ma)


_dev_cache = {}


def device_case(eng, name, D):
    """the case's tensors on the GPU, both layouts (kept for the module: the large case is ~100 MB at D = 16)"""
    key = (name, D)
    if key not in _dev_cache:
        if len(_dev_cache) > 24:
            _dev_cache.clear()
        c = ic.case(name, D)
        f64, i32, u8, i64 = torch.float64, torch.int32, torch.uint8, torch.int64
        _dev_cache[key] = {
            "row_ptr": eng.dev(c["row_ptr"], i64), "req_run": eng.dev(c["req_run"], f64),
            "flags_run": eng.dev(c["flags_run"], u8),
            # one spare entry past row_ptr[N]: run_idx is never NULL (= contiguous), not even for an empty CSR
            "run_idx": eng.dev(np.append(c["run_idx"], np.int32(0)), i32),
            "req_tab": eng.dev(c["req_tab"], f64), "flags_tab": eng.dev(c["flags_tab"], u8),
            "cap_type": eng.dev(c["cap_type"], f64), "node_type": eng.dev(c["node_type"], i32),
            "node_flags": eng.dev(c["node_flags"], u8), "node_age": eng.dev(c["node_age"], i64)}
    return _dev_cache[key]


def check_record(rec, kernel, form, D, nbytes, warps, S, N):
    assert rec["kernel"] == kernel and rec["form"] == form and rec["D"] == D, rec
    assert (rec["bytes"], rec["warps"]) == (nbytes, warps), rec
    assert rec["chunk"] == (ic.chunk(nbytes, D) if form != ic.PER_THREAD else 0), rec
    assert rec["S"] == S and rec["grid"] >= 1, rec
    if N >= 500000:  # the multigroup case reaches the multi-node paths of every form
        if form == ic.PER_THREAD:
            assert N > rec["grid"] * warps * 32, rec            # every thread takes >= 2 nodes
        else:
            groups = (N + 31) // 32
            assert -(-groups // (rec["grid"] * warps)) >= 2, rec  # every warp owns >= 2 groups


def run_layout(eng, c, dc, layout, form, D, nbytes, warps):
    """K1 and K6 (both any_pending values) through the device entry points in one layout"""
    used_o, st_o, _ = oracle_answers(c["name"], D)
    if layout == "contiguous":
        idx, req, flags = None, dc["req_run"], dc["flags_run"]
    else:
        idx, req, flags = dc["run_idx"], dc["req_tab"], dc["flags_tab"]
    d_used = eng.dev(c["used0"], torch.float64)
    eng.occupancy(dc["row_ptr"], idx, req, d_used)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(bits(to_np(d_used)), bits(used_o), err_msg="K1 used")
    check_record(eng.last_scan_launch(), 1, form, D, nbytes, warps, 0, c["N"])
    for ap in (False, True):
        st = eng.node_states(dc["row_ptr"], idx, req, flags, dc["cap_type"], dc["node_type"], dc["node_flags"],
                             dc["node_age"], ap, c["thr"])
        np.testing.assert_array_equal(to_np(st), st_o[ap], err_msg="K6 any_pending=%s" % ap)
        check_record(eng.last_scan_launch(), 2, form, D, nbytes, warps, c["S"], c["N"])


@pytest.mark.parametrize("name", ic.NAMES)
@pytest.mark.parametrize("row", range(len(ROWS)), ids=ROW_IDS)
def test_scan_variant_matches_oracle(eng, oracle_mod, row, name):
    form, D, knobs, nbytes, warps = ROWS[row]
    c = dict(ic.case(name, D), name=name)
    dc = device_case(eng, name, D)
    layouts = {ic.BULK: ["contiguous"], ic.GATHER: ["gathered"], ic.PER_THREAD: ["contiguous", "gathered"]}[form]
    try:
        for k, v in knobs.items():
            eng.set_knob(k, v)
        for layout in layouts:
            run_layout(eng, c, dc, layout, form, D, nbytes, warps)
        if form != ic.GATHER:
            # the host-buffer entry points take the contiguous path too
            used_o, st_o, (pool, budget, ms, ma) = oracle_answers(name, D)
            used_h = c["used0"].copy()
            eng.occupancy_host(c["row_ptr"], None, c["req_run"], used_h)
            np.testing.assert_array_equal(bits(used_h), bits(used_o), err_msg="occupancy_host")
            if c["N"]:
                check_record(eng.last_scan_launch(), 1, form, D, nbytes, warps, 0, c["N"])
            s_h, a_h = eng.maintain_host(c["row_ptr"], None, c["req_run"], c["flags_run"], c["cap_type"],
                                         c["node_type"], c["node_flags"], c["node_age"], pool, False, int(c["thr"][0]),
                                         budget, np.ones(3, np.uint8), False)
            np.testing.assert_array_equal(s_h, ms, err_msg="maintain_host state")
            np.testing.assert_array_equal(a_h, ma, err_msg="maintain_host action")
            if c["N"]:
                check_record(eng.last_scan_launch(), 2, form, D, nbytes, warps, 1, c["N"])
    finally:
        for k, v in DEFAULT_KNOBS.items():
            eng.set_knob(k, v)


def test_default_geometry_without_knobs(oracle_mod):
    """a fresh ctx (no knob set, no ACSFIT_BULK_CFG / ACSFIT_STREAM_BYTES) runs bulk copies at 8 KB x 16 warps and
    gathers at 8 KB per warp"""
    import os
    if os.environ.get("ACSFIT_BULK_CFG") or os.environ.get("ACSFIT_STREAM_BYTES"):
        pytest.skip("geometry set from the environment")
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    e = Engine(0)
    try:
        for D in (4, 8):
            c = dict(ic.case("ragged", D), name="ragged")
            dc = device_case(e, "ragged", D)
            run_layout(e, c, dc, "contiguous", ic.BULK, D, 8192, 16)
            run_layout(e, c, dc, "gathered", ic.GATHER, D, 8192, 8)
    finally:
        e.close()


def test_knobs_are_per_ctx(eng):
    """a second ctx's knobs do not change the first one's kernels"""
    from kubernetes_acs_engine_autoscaler_b200.engine import Engine
    c = dict(ic.case("n33", 4), name="n33")
    dc = device_case(eng, "n33", 4)
    other = Engine(0)
    try:
        eng.set_knob("bulk_cfg", 3)
        other.set_knob("bulk_cfg", 0)
        other.set_knob("stream_bytes", 2048)
        run_layout(eng, c, dc, "contiguous", ic.BULK, 4, 32768, 6)
        run_layout(eng, c, dc, "gathered", ic.GATHER, 4, 8192, 8)
    finally:
        other.close()
        for k, v in DEFAULT_KNOBS.items():
            eng.set_knob(k, v)


def _flags_view(eng, flags, off):
    base = torch.zeros(len(flags) + 32, dtype=torch.uint8, device=eng.device)
    v = base[off:off + len(flags)]
    v.copy_(torch.from_numpy(flags).to(eng.device))
    assert v.data_ptr() % 16 == off
    return v


def _req_view_8(eng, req):
    R, D = req.shape
    base = torch.zeros(R * D + 4, dtype=torch.float64, device=eng.device)
    v = base[1:1 + R * D].view(R, D)
    v.copy_(torch.from_numpy(np.ascontiguousarray(req)).to(eng.device))
    assert v.data_ptr() % 16 == 8
    return v


@pytest.mark.parametrize("what", ["flags+1", "flags+7", "flags+15", "req+8"])
@pytest.mark.parametrize("layout", ["contiguous", "gathered"])
@pytest.mark.parametrize("D", [2, 4, 8, 16])
def test_misaligned_views_fall_back_to_per_thread(eng, oracle_mod, D, layout, what):
    """contiguous views at an odd offset are legal device pointers: the streaming forms' 16-byte copies cannot read
    them, so the library runs the per-thread form (same result).  The gather form loads flag bytes one by one and
    keeps running with a misaligned flags_run."""
    name = "ragged"
    c = dict(ic.case(name, D), name=name)
    dc = dict(device_case(eng, name, D))
    used_o, st_o, _ = oracle_answers(name, D)
    gathered = layout == "gathered"
    req_key, flags_key = ("req_tab", "flags_tab") if gathered else ("req_run", "flags_run")
    if what.startswith("flags"):
        dc[flags_key] = _flags_view(eng, c[flags_key], int(what[6:]))
    else:
        dc[req_key] = _req_view_8(eng, c[req_key])
    aligned_form = ic.GATHER if gathered else ic.BULK
    aligned_geom = (8192, 8) if gathered else ic.bulk_geometry(D, 4)
    idx = dc["run_idx"] if gathered else None

    d_used = eng.dev(c["used0"], torch.float64)
    eng.occupancy(dc["row_ptr"], idx, dc[req_key], d_used)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(bits(to_np(d_used)), bits(used_o))
    rec = eng.last_scan_launch()
    if what == "req+8":
        check_record(rec, 1, ic.PER_THREAD, D, 0, 4, 0, c["N"])
    else:  # K1 reads no flags
        check_record(rec, 1, aligned_form, D, *aligned_geom, 0, c["N"])

    st = eng.node_states(dc["row_ptr"], idx, dc[req_key], dc[flags_key], dc["cap_type"], dc["node_type"],
                         dc["node_flags"], dc["node_age"], False, c["thr"])
    np.testing.assert_array_equal(to_np(st), st_o[False])
    rec = eng.last_scan_launch()
    if what == "req+8" or not gathered:
        check_record(rec, 2, ic.PER_THREAD, D, 0, 4, c["S"], c["N"])
    else:
        check_record(rec, 2, ic.GATHER, D, 8192, 8, c["S"], c["N"])


@pytest.mark.parametrize("D", [2, 16])
def test_pipeline_refuses_misaligned_req(eng, D):
    """the first-fit pipeline loads request rows as 16-byte vectors and has no scalar form: a request table at an
    8-byte offset is an argument error, raised before anything is launched"""
    P, N = 40, 7
    req = _req_view_8(eng, np.full((P, D), 0.25))
    cap = eng.dev(np.full((1, D), 4.0), torch.float64)
    ntype = eng.dev(np.zeros(N, np.int32), torch.int32)
    used = eng.dev(np.zeros((N, D)), torch.float64)
    unit = np.full((1, D), 4.0)
    one, big, zero = np.array([1], np.int32), np.array([100], np.int32), np.zeros(1, np.uint8)
    launches = eng.launch_count
    calls = [
        lambda: eng.first_fit_nodes(req, None, cap, ntype, used),
        lambda: eng.fulfill_pending(req, P, unit, one, big, zero, 0),
        lambda: eng.scale_up(req, unit, unit, one, big, zero, 0, cap, ntype, used),
    ]
    for call in calls:
        with pytest.raises(AcsfitError) as ei:
            call()
        assert ei.value.status == E_INVALID and "16-byte aligned" in str(ei.value)
        assert eng.last_launches() == []
    assert eng.launch_count == launches
    # the same table, aligned, is accepted
    placed, _ = eng.first_fit_nodes(eng.dev(to_np(req), torch.float64), None, cap, ntype, used)
    torch.cuda.synchronize()
    assert (to_np(placed) >= 0).all()


# ---- maintain_actions: the per-pool ranking of maintain_apply_kernel ----------------------------------------------
MAINT_BLOCK, MAINT_CHUNK = 256, 4096  # threads per CTA (one round), nodes per CTA (kMaintChunk)


def maintain_case(T, seed):
    rng = np.random.default_rng(seed)
    N = 3 * MAINT_CHUNK + 517
    states = np.array([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 255], dtype=np.uint8)
    state = rng.choice(states, size=N, p=[0.03] * 8 + [0.6, 0.1, 0.06]).astype(np.uint8)
    # drainable runs across the 256-thread round and the 4096-node block boundaries
    for b in (MAINT_BLOCK, 5 * MAINT_BLOCK, MAINT_CHUNK, 2 * MAINT_CHUNK + MAINT_BLOCK, 3 * MAINT_CHUNK):
        state[b - 40:b + 40] = 8
    node_pool = (np.arange(N) % T).astype(np.int32)            # pools interleaved node by node
    odd = rng.random(N) < 0.02
    node_pool[odd] = rng.choice(np.array([-1, T], np.int32), size=int(odd.sum()))
    scal = (rng.random(T) < 0.9).astype(np.uint8)
    scal[0] = 1
    # budget per pool: its drainable count, +-1, 0, negative, 2^40
    drainable = np.array([np.sum((node_pool == t) & (state == 8)) for t in range(T)], dtype=np.int64)
    pick = rng.integers(0, 7, size=T)
    budget = np.choose(pick, [drainable, drainable - 1, drainable + 1, np.zeros(T, np.int64),
                              np.full(T, -1, np.int64), np.full(T, -5, np.int64),
                              np.full(T, 1 << 40, np.int64)]).astype(np.int64)
    budget[0] = max(int(drainable[0]) - 1, 1)
    return state, node_pool, budget, scal


@pytest.mark.parametrize("dry_run", [False, True])
@pytest.mark.parametrize("T,seed", [(256, 1), (256, 2), (3, 3), (1, 4)])
def test_maintain_actions_edges(eng, oracle_mod, T, seed, dry_run):
    state, node_pool, budget, scal = maintain_case(T, seed)
    s_o, a_o = oracle_mod.maintain_actions(state, node_pool, budget, scal, dry_run)
    d_state = eng.dev(state, torch.uint8)
    s, a = eng.maintain_actions(d_state, eng.dev(node_pool, torch.int32), budget, scal, dry_run)
    torch.cuda.synchronize()
    np.testing.assert_array_equal(to_np(s), s_o)
    np.testing.assert_array_equal(to_np(a), a_o)
    if not dry_run:  # the budgets bite: some drainable nodes became spare agents, some were drained
        assert (s_o == 3).any() and (a_o == 1).any()
