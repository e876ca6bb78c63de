"""`-m gpu`: selector-aware node states -- ACSFIT_NODEF_NO_PENDING_MATCH in K6 and Cluster(selector_node_states=True).

* Every row of the scan's dispatch table (16 bulk geometries, 9 gather sizes, the per-thread form at D in
  {1, 3, 5, 12, 15}) on every case of tests/idle_cases.py, with any_pending in {0, 1} and seven patterns of the flag:
  K6 must equal np.where(flag, oracle(any_pending=0), oracle(any_pending)) exactly, through the device entry point
  and maintain_host, and the launch record must show the intended form.  The pinned oracle ignores the bit, so the
  expected answer needs no new C code (tests/test_selector_states_cpu.py ties this construction to the upstream
  get_node_state).
* The recorded reference ticks with both switches on and no selector: still the reference's tick, same launches, same
  node flags sent to the GPU.
* The recorded ticks with selectors: node states, the maintain journal, dry-run lines and deletions equal a
  plain-Python restatement of the upstream get_node_state and maintain; the scale-up is the same with the switch on
  and off.
* The tick that motivates the switch: a pod pinned to a pool at max_size no longer freezes scale-down elsewhere."""
import re

import numpy as np
import pytest
import torch

import golden_util as gu
import idle_cases as ic
from test_gpu_idle_variants import DEFAULT_KNOBS, ROW_IDS, ROWS, check_record, device_case, oracle_answers, to_np
from test_gpu_selectors_host import restate, with_selectors

pytestmark = pytest.mark.gpu

NO_MATCH = 2  # ACSFIT_NODEF_NO_PENDING_MATCH
ST_BUSY_UNSCHEDULABLE, ST_BUSY = 6, 7
PATTERNS = ("none", "all", "alternating", "seeded_half", "unschedulable_only", "busy_only", "group_ends")


@pytest.fixture(scope="module")
def eng():
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


def pattern(c, st_true, which):
    """bool[N]: the nodes that carry the flag"""
    N = c["N"]
    idx = np.arange(N)
    if which == "none":
        return np.zeros(N, bool)
    if which == "all":
        return np.ones(N, bool)
    if which == "alternating":
        return idx % 2 == 1
    if which == "seeded_half":
        return np.random.default_rng(N).random(N) < 0.5
    if which == "unschedulable_only":
        return (c["node_flags"] & ic.NODEF_UNSCHEDULABLE) != 0
    if which == "busy_only":
        return np.isin(st_true[0], (ST_BUSY, ST_BUSY_UNSCHEDULABLE))
    if which == "group_ends":
        return (idx % 32 == 0) | (idx % 32 == 31) | (idx == N - 1)
    raise ValueError(which)


def expected(st_o, flag, ap):
    return np.where(flag, st_o[False], st_o[True]) if ap else st_o[False]


@pytest.mark.parametrize("name", ic.NAMES)
@pytest.mark.parametrize("row", range(len(ROWS)), ids=ROW_IDS)
def test_no_pending_match_flag_in_every_scan_form(eng, oracle_mod, row, name):
    form, D, knobs, nbytes, warps = ROWS[row]
    c = ic.case(name, D)
    dc = device_case(eng, name, D)
    _, st_o, (pool, budget, _, _) = oracle_answers(name, D)
    layouts = {ic.BULK: ["contiguous"], ic.GATHER: ["gathered"], ic.PER_THREAD: ["contiguous", "gathered"]}[form]
    try:
        for k, v in knobs.items():
            eng.set_knob(k, v)
        for which in PATTERNS:
            flag = pattern(c, st_o[True], which)
            nflags = c["node_flags"] | np.where(flag, np.uint8(NO_MATCH), np.uint8(0))
            d_nflags = eng.dev(nflags, torch.uint8)
            for layout in layouts:
                if layout == "contiguous":
                    idx, req, flags = None, dc["req_run"], dc["flags_run"]
                else:
                    idx, req, flags = dc["run_idx"], dc["req_tab"], dc["flags_tab"]
                for ap in (False, True):
                    st = eng.node_states(dc["row_ptr"], idx, req, flags, dc["cap_type"], dc["node_type"], d_nflags,
                                         dc["node_age"], ap, c["thr"])
                    want = expected(st_o, flag, ap)
                    np.testing.assert_array_equal(to_np(st), want, err_msg="K6 %s %s any_pending=%s" % (which, layout, ap))
                    check_record(eng.last_scan_launch(), 2, form, D, nbytes, warps, c["S"], c["N"])
            if form != ic.GATHER:  # the host-buffer entry point forwards node_flags to the same kernels
                for ap in (False, True):
                    ms, ma = oracle_mod.maintain_actions(expected(st_o, flag, ap)[0], pool, budget, np.ones(3, np.uint8),
                                                         False)
                    s_h, a_h = eng.maintain_host(c["row_ptr"], None, c["req_run"], c["flags_run"], c["cap_type"],
                                                 c["node_type"], nflags, c["node_age"], pool, ap, int(c["thr"][0]),
                                                 budget, np.ones(3, np.uint8), False)
                    np.testing.assert_array_equal(s_h, ms, err_msg="maintain_host state %s %s" % (which, ap))
                    np.testing.assert_array_equal(a_h, ma, err_msg="maintain_host action %s %s" % (which, ap))
                    if c["N"]:
                        check_record(eng.last_scan_launch(), 2, form, D, nbytes, warps, 1, c["N"])
    finally:
        for k, v in DEFAULT_KNOBS.items():
            eng.set_knob(k, v)


def test_patterns_reach_the_pending_branch(oracle_mod):
    """the flag patterns are not vacuous: on the ragged case each one (but `none`) moves nodes off POD_PENDING"""
    c = ic.case("ragged", 4)
    _, st_o, _ = oracle_answers("ragged", 4)
    for which in PATTERNS:
        flag = pattern(c, st_o[True], which)
        moved = int((expected(st_o, flag, True) != st_o[True]).any(axis=0).sum())
        if which in ("none", "unschedulable_only", "busy_only"):  # these nodes never were POD_PENDING
            assert moved == 0, which
        else:
            assert moved > 0, which


# ---------------------------------------------------------------- through Cluster.loop_logic
TICKS = gu.load_json("ticks.json.gz")
DRY_MAINTAIN = re.compile(r"\[Dry run\] Would have (drained and cordoned|cordoned|uncordoned|scaled in) ")


@pytest.fixture()
def host(tmp_path, monkeypatch, engine):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", engine)
    return monkeypatch


def tick(state, engine, selectors, states_on):
    """one recorded tick through gu.run_tick with $ACSFIT_NODE_SELECTORS / $ACSFIT_SELECTOR_NODE_STATES set; adds the
    journal written from the start of maintain (None when maintain did not run), the node flags every K6 call was sent,
    and the launch count"""
    from kubernetes_acs_engine_autoscaler_b200 import engine_scaler
    marks, sent = [], []
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("ACSFIT_NODE_SELECTORS", selectors)
        mp.setenv("ACSFIT_SELECTOR_NODE_STATES", states_on)
        orig_maintain = engine_scaler.EngineScaler.maintain

        def maintain(self, pods_to_schedule, running):
            objs = [n.original for pool in self.agent_pools for n in pool.nodes]
            marks.append(len(objs[0]._journal) if objs else None)
            return orig_maintain(self, pods_to_schedule, running)
        mp.setattr(engine_scaler.EngineScaler, "maintain", maintain)
        orig_states = engine.node_states

        def node_states(*a):
            sent.append(to_np(a[6]).tolist())
            return orig_states(*a)
        mp.setattr(engine, "node_states", node_states)
        n0 = engine.launch_count
        got = gu.run_tick(state, mp)
        got["launches"] = engine.launch_count - n0
    got["node_flags_sent"] = sent
    got["maintain_journal"] = None if not marks else [] if marks[0] is None else got["journal"][marks[0]:]
    return got


@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_switches_on_without_selectors_is_the_reference_tick(host, engine, state):
    off = tick(state, engine, "0", "0")
    on = tick(state, engine, "1", "1")
    gu.assert_tick_matches(on, state["expected"])
    assert on["launches"] == off["launches"]
    assert on["node_flags_sent"] == off["node_flags_sent"]


def restate_maintain(state, to_schedule_names):
    """the upstream get_node_state (pending_list of matching pods) and maintain state machine in plain Python on fresh
    kube objects of the tick: (state calls, journal, node log lines, dry-run lines, deleted nodes)"""
    from kubernetes_acs_engine_autoscaler_b200 import capacity, utils
    from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod, KubePodStatus, KubeResource
    st = state["settings"]
    now = gu.parse_now(state)
    journal, calls, node_lines, dry_lines, deleted = [], [], [], [], []
    notifier = None
    if st.get("notifier") == "recording":
        class Rec(object):
            def notify_drained_node(self, node, pods):
                journal.append(["notify_drained_node", node.name, [p.name for p in pods]])
        notifier = Rec()
    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(utils, "now", lambda tz=None: now.astimezone(tz) if tz is not None else now.replace(tzinfo=None))
        nodes = []
        for o in state["nodes"]:
            n = KubeNode(gu.FakeKubeObject(o, journal, "node"))
            n.capacity = capacity.get_capacity_for_instance_type(n.instance_type)
            if utils.is_agent(n):
                nodes.append(n)
        pods = [KubePod(gu.FakeKubeObject(o, journal, "pod")) for o in state["pods"]]
        to_schedule = [p for p in pods if p.name in to_schedule_names]
        by_node = {}
        for p in pods:
            if p.status in (KubePodStatus.RUNNING, KubePodStatus.CONTAINER_CREATING) or \
                    (p.status == KubePodStatus.PENDING and p.node_name):
                by_node.setdefault(p.node_name, []).append(p)
        buckets = {}
        for param in state["arm_parameters"]:
            if param.endswith("VMSize") and param != "masterVMSize":
                buckets.setdefault(param[:-len("VMSize")], [])
        for n in nodes:
            buckets[utils.get_pool_name(n)].append(n)
        ignored = set(st["ignore_pools"].split(","))
        for name, members in buckets.items():
            if name in ignored:
                continue
            pool = AgentPool(name, "x", members)
            budget = pool.actual_capacity - len(pool.unschedulable_nodes) - st["spare_agents"]
            for node in pool.nodes:
                node_pods = by_node.get(node.name, [])
                busy_list = [p for p in node_pods if not p.is_mirrored() and "kube-proxy" not in p.name]
                age = (utils.now(node.creation_time.tzinfo) - node.creation_time).seconds
                undrainable_list = [p for p in node_pods if not (p.is_drainable() or "kube-proxy" in p.name)]
                utilization = sum((p.resources for p in busy_list), KubeResource())
                under = (0.3 * node.capacity - utilization).possible
                pending_list = [p for p in to_schedule if node.is_match(p)]
                if busy_list and not under:
                    state_ = "busy-unschedulable" if node.unschedulable else "busy"
                elif pending_list and not node.unschedulable:
                    state_ = "pod-pending"
                elif age <= st["idle_threshold"] and not node.unschedulable:
                    state_ = "grace-period"
                elif under and (busy_list or not node.unschedulable):
                    state_ = "under-utilized-undrainable" if undrainable_list else "under-utilized-drainable"
                else:
                    state_ = "idle-unschedulable" if node.unschedulable else "idle-schedulable"
                calls.append([node.name, state_])
                if state_ == "under-utilized-drainable" and budget == 0:
                    state_ = "spare-agent"
                node_lines.append("node: %-*s state: %s" % (75, node, state_))
                if state_ == "under-utilized-drainable":
                    if st["dry_run"]:
                        dry_lines.append("[Dry run] Would have drained and cordoned %s" % node)
                    else:
                        node.cordon()
                        node.drain(node_pods, notifier)
                        budget -= 1
                elif state_ == "idle-schedulable":
                    if st["dry_run"]:
                        dry_lines.append("[Dry run] Would have cordoned %s" % node)
                    else:
                        node.cordon()
                elif state_ == "busy-unschedulable":
                    if st["dry_run"]:
                        dry_lines.append("[Dry run] Would have uncordoned %s" % node)
                    else:
                        node.uncordon()
                elif state_ == "idle-unschedulable":
                    if st["dry_run"]:
                        dry_lines.append("[Dry run] Would have scaled in %s" % node)
                    else:
                        deleted.append(node.name)
    return calls, journal, node_lines, dry_lines, sorted(deleted)


def schedulable(state):
    """names of the pending, unassigned pods some pool matches and fits (the selector mode's feasibility)"""
    from kubernetes_acs_engine_autoscaler_b200 import capacity, utils
    from kubernetes_acs_engine_autoscaler_b200.agent_pool import AgentPool
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod, KubePodStatus
    j = []
    nodes = []
    for o in state["nodes"]:
        n = KubeNode(gu.FakeKubeObject(o, j, "node"))
        if utils.is_agent(n):
            nodes.append(n)
    buckets = {}
    for param, spec in state["arm_parameters"].items():
        if param.endswith("VMSize") and param != "masterVMSize":
            buckets.setdefault(param[:-len("VMSize")], (spec["value"], []))
    for n in nodes:
        buckets[utils.get_pool_name(n)][1].append(n)
    pools = [AgentPool(name, vm, members) for name, (vm, members) in buckets.items()]
    names = set()
    for o in state["pods"]:
        p = KubePod(gu.FakeKubeObject(o, j, "pod"))
        if p.status != KubePodStatus.PENDING or p.node_name:
            continue
        if any(all(pool.labels.get(k) == v for k, v in p.selectors.items())
               and (capacity.RESOURCE_SPEC[pool.instance_type] - p.resources).possible for pool in pools):
            names.add(p.name)
    return names


def assert_maintain_is_upstream(s, got, exc):
    """`exc`: the exception the scale-up raises (maintain is not reached), or None"""
    st = s["settings"]
    calls, journal, node_lines, dry_lines, deleted = restate_maintain(s, schedulable(s))
    if exc is not None or not st.get("maintainance", True) or not s["nodes"]:
        assert got["maintain_journal"] is None and got["state_calls"] == [], s["name"]
        return
    assert got["state_calls"] == calls, s["name"]
    assert got["maintain_journal"] == journal, s["name"]
    assert [m for _, _, m in got["log"] if m.startswith("node: ")] == node_lines, s["name"]
    assert [m for _, _, m in got["log"] if DRY_MAINTAIN.match(m)] == dry_lines, s["name"]
    assert got["deleted_nodes"] == deleted, s["name"]


SCALE_UP_KEYS = ("exception", "scale_pools_calls", "used")


@pytest.mark.parametrize("variant", (0, 1, 2))
def test_selector_ticks_match_upstream_maintain(host, engine, variant):
    differs = ran = 0
    for state in TICKS:
        s = with_selectors(state, variant)
        on = tick(s, engine, "1", "1")
        off = tick(s, engine, "1", "0")
        # the scale-up half is the same with the switch on and off
        for key in SCALE_UP_KEYS:
            assert on[key] == off[key], (s["name"], key)
        warn = lambda g: [m for lvl, _, m in g["log"] if lvl == "WARNING"]  # noqa: E731
        assert warn(on) == warn(off), s["name"]
        exc = restate(s)[0] if s["settings"].get("scale_up", True) else None
        assert (on["exception"] or [None])[0] == exc, s["name"]
        assert_maintain_is_upstream(s, on, exc)
        ran += on["maintain_journal"] is not None
        differs += on["state_calls"] != off["state_calls"]
    assert ran >= 5 and differs >= 1, (ran, differs)


# ---------------------------------------------------------------- the motivating tick
def pinned_pod_state(dry_run):
    """pool `agentpool1`: three old, idle, schedulable Standard_D2_v2 nodes.  Pool `gpupool` (Standard_NC6, max_size 1):
    one node with a small running pod.  One pending pod pinned to `gpupool` that does not fit its node: the pool is at
    max_size, so the pod waits."""
    def node(pool, i, itype):
        name = "k8s-%s-16334397-%d" % (pool, i)
        return {"metadata": {"name": name, "creationTimestamp": "2016-08-25T05:13:16Z",
                             "labels": {"beta.kubernetes.io/instance-type": itype, "agentpool": pool,
                                        "failure-domain.beta.kubernetes.io/region": "southcentralus",
                                        "kubernetes.io/hostname": name}}, "spec": {}}

    def pod(name, cpu, phase, node_name=None, selector=None):
        spec = {"containers": [{"name": "c", "resources": {"requests": {"cpu": cpu}}}]}
        if node_name:
            spec["nodeName"] = node_name
        if selector:
            spec["nodeSelector"] = selector
        status = {"phase": phase}
        if phase == "Running":
            status["startTime"] = "2026-09-20T07:00:00Z"
        return {"metadata": {"name": name, "namespace": "default", "uid": "uid-" + name,
                             "creationTimestamp": "2026-09-20T07:00:00Z"}, "spec": spec, "status": status}
    nodes = [node("agentpool1", i, "Standard_D2_v2") for i in range(3)] + [node("gpupool", 0, "Standard_NC6")]
    pods = [pod("small", "100m", "Running", nodes[3]["metadata"]["name"]),
            pod("trainer", "5950m", "Pending", selector={"agentpool": "gpupool"})]
    return {"name": "pinned_pod_%s" % ("dry" if dry_run else "live"), "now": "2026-09-21T12:00:00Z",
            "nodes": nodes, "pods": pods,
            "arm_parameters": {"masterVMSize": {"value": "Standard_D2_v2"}, "firstConsecutiveStaticIP": {"value": "10.0.0.1"},
                               "agentpool1VMSize": {"value": "Standard_D2_v2"}, "gpupoolVMSize": {"value": "Standard_NC6"}},
            "settings": {"idle_threshold": 1800, "spare_agents": 1, "over_provision": 0, "dry_run": dry_run,
                         "ignore_pools": "", "pool_max_size": {"gpupool": 1}}}


@pytest.mark.parametrize("dry_run", [True, False])
def test_pinned_pod_no_longer_freezes_scale_down(host, engine, dry_run):
    from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler
    host.setattr(Scaler, "REFERENCE_RAISE_ON_INSUFFICIENT", False)  # the saturated pool must not abort the tick
    s = pinned_pod_state(dry_run)
    cpu_nodes = [n["metadata"]["name"] for n in s["nodes"][:3]]
    off = tick(s, engine, "1", "0")
    on = tick(s, engine, "1", "1")
    assert off["exception"] is None and on["exception"] is None
    assert "Pods to schedule: 1" in [m for _, _, m in on["log"]]
    assert off["state_calls"] == [[n, "pod-pending"] for n in cpu_nodes] + [[s["nodes"][3]["metadata"]["name"], "pod-pending"]]
    assert off["maintain_journal"] == [] and not [m for _, _, m in off["log"] if DRY_MAINTAIN.match(m)]
    # on: the CPU nodes follow the idle rules; the pinned pod still holds its own pool's node
    assert on["state_calls"] == [[n, "under-utilized-drainable"] for n in cpu_nodes] + \
        [[s["nodes"][3]["metadata"]["name"], "pod-pending"]]
    if dry_run:  # no budget is spent in a dry run: every drainable node is reported
        assert [m for _, _, m in on["log"] if DRY_MAINTAIN.match(m)] == \
            ["[Dry run] Would have drained and cordoned %s" % n for n in cpu_nodes]
    else:        # budget 3 nodes - 1 spare: two are cordoned and drained, the third stays as a spare agent
        assert [e for e in on["maintain_journal"] if e[0] == "node.update"] == \
            [["node.update", n, True, "true"] for n in cpu_nodes[:2]]
        assert "node: %-*s state: spare-agent" % (75, cpu_nodes[2]) in [m for _, _, m in on["log"]]
    assert_maintain_is_upstream(s, on, None)
    for key in SCALE_UP_KEYS:
        assert on[key] == off[key], key
