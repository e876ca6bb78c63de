"""`-m gpu`: the cluster-mode matrix.  Every named case of tests/cluster_cases.py runs on every rank of one connected
session and each rank's result must equal the plain-C oracle exactly; the plan (`cluster_last_plan`) and the launch
records (`last_launches`) must show the geometry that ran: stages, stage width, pod blocks, RW, form, pruning and
the `bin_base` of every bin pass.

Harness: one process per rank and one spawn per (world, transport); all cases of a world run in that one session
under the three scan modes (packed ranks, float64, streaming), so sync sets are reused and barrier epochs must stay in
step across changing D, N, P and knobs.  Worlds 2, 3 and 4 run "loopback" (every rank on cuda:0, handles exchanged
over gloo; worlds 3 and 4 run the reduced case list); world 2 also runs over NCCL on two GPUs when there are two.
Workers write every call's outputs to a temporary directory and stop at their first exception; the main process
computes the oracle answers, joins the workers with a timeout and reaps any survivor.  Refusals (host-side and the
same on every rank) are checked on a second, small exchange region, each followed by a call that must still match
the oracle."""
import datetime
import functools
import json
import os
import socket
import sys
import time
import traceback

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import bin_chain_cases as bcc
import cluster_cases as cc
import variant_cases as vc
from test_rank_math_cpu import layout

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu

MODES = ("ranks", "f64", "stream")
SESSIONS = {"w2": (2, "gloo"), "w3": (3, "gloo"), "w4": (4, "gloo"), "w2_nccl": (2, "nccl")}
JOIN_TIMEOUT_S = 900
DEFAULT_KNOBS = {"cluster_blocks": 0, "prune": -1, "bin_pass_stages": 0, "retire": 1}
# the small exchange region the refusals are checked on
REF_PODS, REF_NODES, REF_DIMS = 600, 200, 8
REFUSALS = ("scale_up_sel", "first_fit_nodes_sel", "fulfill_pending_sel", "ff_pods_over", "ff_nodes_over",
            "ff_dims_over", "scale_up_pods_over", "scale_up_nodes_over", "scale_up_dims_over", "fulfill_pods_over")
SCALARS = ("n_to_schedule", "n_pending", "num_unaccounted", "decisions")


def exchange_sizes(world, sms):
    """max_pods / max_nodes of the main session's exchange region: the largest case of this world, with room"""
    M, _ = cc.closed_full(world, sms, cc.MIN_TN)
    return max(20000, 2 * M), cc.auto_blocks_nodes(world, sms) + 1024


def refusal_tick():
    return cc.build("feasible_257", 2)  # 600 pods (257 feasible), 40 nodes, D = 8


def refusal_inputs(label, c):
    """the arguments of one refused call: a valid tick pushed just past the small exchange region"""
    c = dict(c)
    if label.endswith("pods_over"):
        # ff: every row is a pod of the node pass; scale_up: the feasible rows; fulfill: the rows pool 0 admits
        rows = c["req"]
        if label == "scale_up_pods_over":
            rows = rows[cc.feasible_rows(rows, c["unit_all"])]
        elif label == "fulfill_pods_over":
            rows = rows[cc.feasible_rows(rows, c["unit_ordered"][:1])]
        c["req"] = np.tile(rows, (-(-(REF_PODS + 1) // rows.shape[0]), 1))
        c["P"] = c["req"].shape[0]
    elif label.endswith("nodes_over"):
        N = REF_NODES + 1
        c["node_type"] = np.resize(c["node_type"], N)
        c["used0"] = np.resize(c["used0"], (N, c["D"]))
    elif label.endswith("dims_over"):
        c = cc.build("layout_d16_rw2", 2)
        c["req"] = c["req"][:500]
        c["node_type"] = c["node_type"][:150]
        c["used0"] = c["used0"][:150]
    return c


# ------------------------------------------------------------------------------------------------- worker side
def _run_call(eng, c, call, knobs):
    f64, i32 = torch.float64, torch.int32
    out = {}
    if call in ("scale_up", "scale_up_host", "ff_all", "ff_subset"):
        args = (c["unit_all"], c["unit_ordered"], c["pool_actual"], c["pool_max"], c["pool_ignored"],
                c["over_provision"])
        if call == "scale_up_host":
            used = c["used0"].copy()
            g = eng.scale_up_host(c["req"], *args, c["cap_type"], c["node_type"], used)
        else:
            d_used = eng.dev(c["used0"], f64)
            d_req, d_cap, d_nt = eng.dev(c["req"], f64), eng.dev(c["cap_type"], f64), eng.dev(c["node_type"], i32)
            if call == "scale_up":
                g = eng.scale_up(d_req, *args, d_cap, d_nt, d_used)
            else:
                idx = None if call == "ff_all" else eng.dev(c["pod_idx"], i32)
                placed, dec = eng.first_fit_nodes(d_req, idx, d_cap, d_nt, d_used)
                g = {"placed": placed, "decisions": dec}
            torch.cuda.synchronize()
            used = d_used.cpu().numpy()
        for k, v in g.items():
            out[k] = v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
        out["used"] = np.ascontiguousarray(used).view(np.uint64)
    else:
        if call == "fulfill":
            f = c["fulfill"]
        else:  # closed / retire: a small single-pass call first, then one sized from its launch records
            f = cc.closed_form_input(*cc.CLOSED_SMALL, c["D"])
        g = eng.fulfill_pending(eng.dev(f["req"], f64), f["num_listed"], f["unit"], f["pool_actual"], f["pool_max"],
                                f["pool_ignored"], f["over_provision"])
        if call == "closed":
            torch.cuda.synchronize()
            small = [r for r in eng.last_launches() if r["pass"] == 1 and r["pool"] == 0][0]
            M, take = cc.closed_full(eng.cluster_world, small["resident"], small["Tn"])
            f = cc.closed_form_input(M, take, c["D"])
            eng.set_knob("bin_pass_stages", 2)  # a single-GPU knob: cluster mode plans its own passes
            g = eng.fulfill_pending(eng.dev(f["req"], f64), M, f["unit"], f["pool_actual"], f["pool_max"],
                                    f["pool_ignored"], f["over_provision"])
            out["closed"] = np.array([M, take, small["resident"], small["Tn"]])
        if call == "retire":
            torch.cuda.synchronize()
            small = [r for r in eng.last_launches() if r["pass"] == 1 and r["pool"] == 0][0]
            f = cc.retire_input(eng.cluster_world, small["Tn"])
            g = eng.fulfill_pending(eng.dev(f["req"], f64), f["num_listed"], f["unit"], f["pool_actual"],
                                    f["pool_max"], f["pool_ignored"], f["over_provision"])
            out["retire"] = np.array([small["Tn"]])
        torch.cuda.synchronize()
        for k, v in g.items():
            out[k] = v.cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)
    out["rec"] = np.array([[r[k] for k in _launch_fields()] for r in eng.last_launches()], np.int32).reshape(-1, 12)
    out["hook"] = np.array(eng.last_bin_retirement(), np.int64)
    p = eng.cluster_last_plan()
    out["plan"] = np.array([p["stage_nodes"], p["stages"], p["pod_blocks"], p["resident"]], np.int32)
    return out


def _launch_fields():
    from kubernetes_acs_engine_autoscaler_b200 import _native
    return _native.LAUNCH_FIELDS


def _refuse(eng, label, c):
    """issue one call that must be refused; returns the status it got (0 if it was not refused)"""
    from kubernetes_acs_engine_autoscaler_b200._native import AcsfitError
    f64, i32, u8 = torch.float64, torch.int32, torch.uint8
    c = refusal_inputs(label, c)
    P, N, T = c["req"].shape[0], c["node_type"].shape[0], c["unit_all"].shape[0]
    pod_class = eng.dev(np.zeros(P, np.uint8), u8)
    node_match = eng.dev(np.ones(N, np.int64), torch.int64)
    masks = np.ones(T, np.uint64)
    d = lambda: (eng.dev(c["req"], f64), eng.dev(c["cap_type"], f64), eng.dev(c["node_type"], i32),  # noqa: E731
                 eng.dev(c["used0"], f64))
    args = (c["unit_all"], c["unit_ordered"], c["pool_actual"], c["pool_max"], c["pool_ignored"], c["over_provision"])
    try:
        if label == "scale_up_sel":
            req, cap, nt, used = d()
            eng.scale_up_sel(req, *args, cap, nt, used, pod_class, node_match, masks, masks, 1)
        elif label == "first_fit_nodes_sel":
            req, cap, nt, used = d()
            eng.first_fit_nodes_sel(req, None, cap, nt, used, pod_class, node_match, 1)
        elif label == "fulfill_pending_sel":
            eng.fulfill_pending_sel(eng.dev(c["req"], f64), P, c["unit_ordered"], c["pool_actual"], c["pool_max"],
                                    c["pool_ignored"], 0, pod_class, masks, 1)
        elif label.startswith("ff_"):
            req, cap, nt, used = d()
            eng.first_fit_nodes(req, None, cap, nt, used)
        elif label.startswith("scale_up_"):
            req, cap, nt, used = d()
            eng.scale_up(req, *args, cap, nt, used)
        elif label == "fulfill_pods_over":
            eng.fulfill_pending(eng.dev(c["req"], f64), P, c["unit_ordered"], c["pool_actual"], c["pool_max"],
                                c["pool_ignored"], 0)
        torch.cuda.synchronize()
    except AcsfitError as e:
        return e.status
    return 0


def _worker(rank, world, port, out_dir, backend, devices, modes, names):
    os.environ.update({"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(devices[rank]),
                       "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)})
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    where = "connect"
    try:
        import torch.distributed as dist
        from kubernetes_acs_engine_autoscaler_b200.engine import Engine
        dev = devices[rank]
        torch.cuda.set_device(dev)
        # a rank that stopped early must not keep the others in a host-level collective for long
        timeout = datetime.timedelta(seconds=180)
        if backend == "nccl":
            dist.init_process_group("nccl", device_id=torch.device("cuda", dev), timeout=timeout)
        else:
            dist.init_process_group("gloo", timeout=timeout)
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        max_pods, max_nodes = exchange_sizes(world, sms)
        eng = Engine(dev)
        eng.cluster_connect(max_pods=max_pods, max_nodes=max_nodes, max_dims=16)
        small = Engine(dev)
        small.cluster_connect(max_pods=REF_PODS, max_nodes=REF_NODES, max_dims=REF_DIMS)

        # refusals, each followed by a valid call on the same exchange region
        tick = refusal_tick()
        status = {}
        for label in REFUSALS:
            where = "refusal " + label
            status[label] = _refuse(small, label, tick)
            np.savez(os.path.join(out_dir, "refusal__%s__r%d.npz" % (label, rank)),
                     **_run_call(small, tick, "scale_up", {}))
        with open(os.path.join(out_dir, "refusals_r%d.json" % rank), "w") as fh:
            json.dump(status, fh)
        where = "refusal scale_up_sel (main region)"
        status_main = _refuse(eng, "scale_up_sel", tick)
        with open(os.path.join(out_dir, "refusal_main_r%d.json" % rank), "w") as fh:
            json.dump({"scale_up_sel": status_main}, fh)

        ticks = {}
        for mode in modes:
            eng.set_knob("ranks", 0 if mode == "f64" else 1)
            eng.set_knob("stream", 1 if mode == "stream" else 0)
            for name in names:
                if name not in ticks:
                    ticks[name] = cc.build(name, world, sms)
                knobs = cc.knobs(name)
                for k, v in knobs.items():
                    eng.set_knob(k, v)
                for i, call in enumerate(cc.calls(name)):
                    where = "%s %s call %d (%s)" % (mode, name, i, call)
                    out = _run_call(eng, ticks[name], call, knobs)
                    np.savez(os.path.join(out_dir, "%s__%s__%d__r%d.npz" % (mode, name, i, rank)), **out)
                for k, v in DEFAULT_KNOBS.items():
                    eng.set_knob(k, v)
        dist.barrier()
        with open(os.path.join(out_dir, "done_r%d" % rank), "w") as fh:
            fh.write("ok")
        dist.destroy_process_group()
    except BaseException:
        with open(os.path.join(out_dir, "error_r%d.txt" % rank), "w") as fh:
            fh.write("rank %d stopped at %s:\n%s" % (rank, where, traceback.format_exc()))
        sys.stderr.flush()
        os._exit(1)  # issue no further call; the other ranks' barriers time out and they stop the same way


# ------------------------------------------------------------------------------------------------- main side
def _devices(sid):
    world, backend = SESSIONS[sid]
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    if backend == "nccl":
        if torch.cuda.device_count() < world:
            pytest.skip("needs %d GPUs" % world)
        return list(range(world))
    return [0] * world


def session_modes(sid):
    return MODES


def session_names(sid):
    return cc.names(SESSIONS[sid][0])


@functools.lru_cache(maxsize=None)
def session(sid, out_dir):
    """spawn the ranks of one session, wait for them (with a timeout) and return what they left"""
    world, backend = SESSIONS[sid]
    devices = _devices(sid)
    from kubernetes_acs_engine_autoscaler_b200 import build as acs_build
    acs_build.build()
    import oracle
    oracle.build()
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    t0 = time.time()
    procs = [ctx.Process(target=_worker, args=(r, world, port, out_dir, backend, devices, session_modes(sid),
                                               session_names(sid))) for r in range(world)]
    for p in procs:
        p.start()
    deadline = t0 + JOIN_TIMEOUT_S
    for p in procs:
        p.join(max(1.0, deadline - time.time()))
    survivors = [p.pid for p in procs if p.is_alive()]
    for p in procs:
        if p.is_alive():
            p.terminate()
            p.join(10)
        if p.is_alive():
            p.kill()
            p.join()
    errors = {}
    for r in range(world):
        path = os.path.join(out_dir, "error_r%d.txt" % r)
        if os.path.exists(path):
            with open(path) as fh:
                errors[r] = fh.read()
    return {"world": world, "exitcodes": [p.exitcode for p in procs], "survivors": survivors, "errors": errors,
            "seconds": time.time() - t0, "out_dir": out_dir}


@pytest.fixture(scope="module")
def out_root(tmp_path_factory):
    return str(tmp_path_factory.mktemp("cluster"))


def run_session(sid, out_root):
    d = os.path.join(out_root, sid)
    os.makedirs(d, exist_ok=True)
    return session(sid, d)


def load(s, stem, rank):
    path = os.path.join(s["out_dir"], "%s__r%d.npz" % (stem, rank))
    if not os.path.exists(path):
        pytest.fail("no output for %s on rank %d; the session stopped: %s" % (stem, rank, s["errors"] or s))
    with np.load(path) as z:
        return {k: z[k] for k in z.files}


@functools.lru_cache(maxsize=None)
def tick_and_oracle(name, world, sms, i):
    import oracle
    c = cc.build(name, world, sms)
    call = cc.calls(name)[i]
    return c, (None if call in ("closed", "retire") else cc.oracle_call(oracle, c, call))


@functools.lru_cache(maxsize=None)
def bins_and_min(name, world, sms, i, size):
    """(each pool's final bins, the call's smallest request per dimension) of one call, from the oracle; size: (M, take)
    of a closed-form call, (tn,) of a retire call.  A pool's bins come from the oracle packing the pods that reached
    it into that pool alone (tests/bin_chain_cases.py)."""
    import oracle
    c, o = tick_and_oracle(name, world, sms, i)
    call = cc.calls(name)[i]
    if call in ("ff_all", "ff_subset"):
        return {}, None
    if call in ("scale_up", "scale_up_host"):
        pend = np.nonzero(o["placed"] == -1)[0]
        rows, acc, all_rows = c["req"][pend], o["acc_pool"][pend], c["req"]
        unit, ignored = c["unit_ordered"], c["pool_ignored"]
    else:
        f = {"fulfill": lambda: c["fulfill"], "closed": lambda: cc.closed_form_input(*size, c["D"]),
             "retire": lambda: cc.retire_input(world, *size)}[call]()
        full = oracle.fulfill_pending(f["req"], f["num_listed"], f["unit"], f["pool_actual"], f["pool_max"],
                                      f["pool_ignored"], f["over_provision"])
        rows, acc, all_rows, unit, ignored = f["req"], full["acc_pool"], f["req"], f["unit"], f["pool_ignored"]

    def one(t, idx):
        return oracle.fulfill_pending(rows[idx], len(idx), unit[t:t + 1], np.zeros(1, np.int32),
                                      np.array([1 << 30], np.int32), np.zeros(1, np.uint8), 0)["bin_of"]
    return bcc.pool_bins(one, rows, acc, unit, ignored), bcc.minreq(all_rows)


def check_retirement(g, recs, name, world, sms, i, rank, knobs, size):
    """this rank's report of what bin retirement marked (dead warps, retired stages of its own stages) against the model
    over the oracle's bins; (0, 0) for calls without a bin pass and with retirement off"""
    S, mr = bins_and_min(name, world, sms, i, size)
    want = (0, 0) if mr is None or not knobs.get("retire", 1) else bcc.retirement(recs, S, mr, rank=rank)
    assert tuple(int(v) for v in g["hook"]) == want, ("hook (dead warps, retired stages)", tuple(g["hook"]), want)
    return want


def expected_rw(rows, mode):
    if mode == "f64":
        return 0
    return vc.expected_rw([vc.distinct_count(rows[:, d]) for d in range(rows.shape[1])], layout)


def records(g):
    from kubernetes_acs_engine_autoscaler_b200 import _native
    return [dict(zip(_native.LAUNCH_FIELDS, (int(v) for v in row))) for row in g["rec"]]


@functools.lru_cache(maxsize=None)
def retire_oracle(world, tn):
    import oracle
    f = cc.retire_input(world, tn)
    return oracle.fulfill_pending(f["req"], f["num_listed"], f["unit"], f["pool_actual"], f["pool_max"],
                                  f["pool_ignored"], f["over_provision"])


def check_result(g, o, call):
    if call in ("ff_all", "ff_subset"):
        np.testing.assert_array_equal(g["placed"], o["placed"], err_msg="placed")
        assert int(np.ravel(g["decisions"])[0]) == o["decisions"], "decisions"
    elif call == "fulfill":
        for k in ("acc_pool", "bin_of", "new_size", "units_needed", "bins_opened"):
            np.testing.assert_array_equal(g[k], o[k], err_msg=k)
        assert int(g["num_unaccounted"]) == o["num_unaccounted"] and int(g["evals"]) == o["evals"]
    else:
        for k in ("feasible", "placed", "acc_pool", "new_size", "units_needed", "bins_opened"):
            np.testing.assert_array_equal(g[k], o[k], err_msg=k)
        for k in SCALARS:
            assert int(g[k]) == o[k], k
    if "used" in o:
        np.testing.assert_array_equal(g["used"], o["used"].view(np.uint64), err_msg="used bits")


def check_plan(g, c, call, knobs, world, rank, mode, rw, node_pods, bins_opened):
    """the plan and the launch records of one call on one rank agree with the cluster geometry"""
    recs = records(g)
    tn, stages, blocks, resident = (int(v) for v in g["plan"])
    D = c["D"]
    prune_forced = knobs.get("prune", -1) == 1
    stream_ok = mode == "stream" and D <= 8 and rw > 0
    for r in recs:
        assert r["chained"] == 0 and r["D"] == D and r["RW"] == rw, r
    nodes = [r for r in recs if r["pass"] == 0]
    N = c["node_type"].shape[0] if call not in ("fulfill", "closed", "retire") else 0
    if call in ("fulfill", "closed", "retire") or node_pods == 0 or N == 0:
        assert not nodes, recs
    else:
        assert tn in (32, 64, 128, 256) and tn <= cc.max_stage_nodes(D), g["plan"]
        lo, hi = cc.lo_of(N, world, rank), cc.lo_of(N, world, rank + 1)
        assert stages == max(1, -(-(hi - lo) // tn)), (g["plan"], lo, hi)
        n_max = max(cc.lo_of(N, world, r + 1) - cc.lo_of(N, world, r) for r in range(world))
        tiles = -(-node_pods // cc.TILE)
        if knobs.get("cluster_blocks", 0):
            want = cc.block_plan(tiles, knobs["cluster_blocks"])[0]
        elif -(-n_max // tn) > resident:
            want = cc.block_plan(tiles, 4 * world)[0]
        else:
            want = 1
        assert blocks == want, (g["plan"], tiles, n_max)
        assert len(nodes) == blocks, recs
        for r in nodes:
            assert (r["stages"], r["Tn"]) == (stages, tn), (r, g["plan"])
            if prune_forced:
                assert (r["prune"], r["form"]) == (1, 0), r
            else:
                assert r["form"] == int(stream_ok), r
                assert r["prune"] == (0 if r["form"] else int(stages > resident)), (r, g["plan"])
    bins = [r for r in recs if r["pass"] == 1]
    for r in bins:
        assert r["prune"] == 0 and r["form"] == int(stream_ok) and r["Tn"] >= 32 and r["Tn"] % 32 == 0, r
    assert {r["pool"] for r in bins} == set(np.flatnonzero(bins_opened).tolist()), recs
    for t in {r["pool"] for r in bins}:
        passes = [r for r in bins if r["pool"] == t]
        assert passes[0]["bin_base"] == 0, passes
        for a, b in zip(passes, passes[1:]):
            assert b["bin_base"] == a["bin_base"] + world * a["stages"] * a["Tn"], (a, b)
    return recs, (tn, stages, blocks, resident)


def case_ids():
    out = []
    for sid in SESSIONS:
        for mode in session_modes(sid):
            for name in session_names(sid):
                out.append(pytest.param(sid, mode, name, id="%s-%s-%s" % (sid, mode, name)))
    return out


@pytest.mark.parametrize("sid,mode,name", case_ids())
def test_cluster_case(out_root, sid, mode, name):
    s = run_session(sid, out_root)
    world = s["world"]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    knobs = cc.knobs(name)
    for i, call in enumerate(cc.calls(name)):
        c, o = tick_and_oracle(name, world, sms, i)
        reports = []
        for rank in range(world):
            g = load(s, "%s__%s__%d" % (mode, name, i), rank)
            size = ()
            if call == "closed":
                M, take, resident, tn = (int(v) for v in g["closed"])
                o = cc.closed_form_answer(M, take)
                assert tn == cc.MIN_TN, g["closed"]
                rows = cc.closed_form_input(M, take, c["D"])["req"]
                size = (M, take)
            elif call == "retire":
                tn = int(g["retire"][0])
                assert tn == cc.MIN_TN, g["retire"]
                f = cc.retire_input(world, tn)
                o = retire_oracle(world, tn)
                rows = f["req"]
                size = (tn,)
            elif call == "fulfill":
                rows = c["fulfill"]["req"]
            else:
                rows = c["req"]
            try:
                check_result(g, o, "fulfill" if call in ("closed", "retire") else call)
                node_pods = {"ff_all": rows.shape[0], "ff_subset": len(c.get("pod_idx", ())),
                             "scale_up": o.get("n_to_schedule", 0), "scale_up_host": o.get("n_to_schedule", 0)}
                recs, plan = check_plan(g, c, call, knobs, world, rank, mode, expected_rw(rows, mode),
                                        node_pods.get(call, 0), o.get("bins_opened", ()))
                reports.append(check_retirement(g, recs, name, world, sms, i, rank, knobs, size))
                if call == "retire":  # one pass of RETIRE_STAGES stages per rank; rank 1's stage 0 retired in it
                    bins = [r for r in recs if r["pass"] == 1]
                    assert [(r["stages"], r["Tn"], r["bin_base"]) for r in bins] == [(cc.RETIRE_STAGES, tn, 0)], bins
                    if rank == 1 and knobs.get("retire", 1) and bins[0]["RW"] > 0 and bins[0]["form"] == 0:
                        assert reports[-1][1] >= 1, reports[-1]
                if name == "blocks_auto":
                    assert not knobs and plan[2] > 1 and plan[1] > plan[3], plan  # waves: blocks chosen by the library
                if call == "closed":
                    pool0 = [r for r in recs if r["pass"] == 1 and r["pool"] == 0]
                    assert len(pool0) == 2, pool0  # bin_pass_stages = 2 is ignored: two passes of world * resident
                    assert (pool0[0]["stages"], pool0[0]["Tn"], pool0[0]["resident"]) == (resident, tn, resident)
                    assert pool0[1]["bin_base"] == world * resident * tn
            except AssertionError as e:
                raise AssertionError("%s / %s call %d (%s), rank %d of %d: %s" % (mode, name, i, call, rank, world, e))
        if call == "retire" and knobs.get("retire", 1) and mode == "ranks":
            assert sum(r[1] for r in reports) > 0, reports  # the ranks together retired stages


@pytest.mark.parametrize("sid", list(SESSIONS))
def test_cluster_refusals(out_root, sid):
    from kubernetes_acs_engine_autoscaler_b200._native import E_INVALID
    s = run_session(sid, out_root)
    world = s["world"]
    c = refusal_tick()
    import oracle
    o = cc.oracle_call(oracle, c, "scale_up")
    for rank in range(world):
        path = os.path.join(s["out_dir"], "refusals_r%d.json" % rank)
        if not os.path.exists(path):
            pytest.fail("rank %d did not finish the refusals: %s" % (rank, s["errors"]))
        with open(path) as fh:
            status = json.load(fh)
        assert status == {label: E_INVALID for label in REFUSALS}, status
        with open(os.path.join(s["out_dir"], "refusal_main_r%d.json" % rank)) as fh:
            assert json.load(fh) == {"scale_up_sel": E_INVALID}
        for label in REFUSALS:  # the call after each refusal
            check_result(load(s, "refusal__" + label, rank), o, "scale_up")


@pytest.mark.parametrize("sid", list(SESSIONS))
def test_cluster_session_ends_clean(out_root, sid):
    s = run_session(sid, out_root)
    assert not s["survivors"], "ranks still running after %d s were terminated: %r" % (JOIN_TIMEOUT_S, s)
    assert not s["errors"], "\n".join(s["errors"].values())
    assert s["exitcodes"] == [0] * s["world"], s
    sys.stderr.write("cluster session %s: %.1f s\n" % (sid, s["seconds"]))
