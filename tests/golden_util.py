"""helpers shared by the golden-vector tests: fixture loading, fake kube objects and a harness that
drives the product's Cluster.loop_logic on a recorded cluster state the way oracle/make_golden.py
drove the reference."""
import copy
import datetime
import gzip
import json
import logging
import lzma
import os
from collections import OrderedDict

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load_json(name):
    path = os.path.join(GOLDEN, name)
    if name.endswith(".gz"):
        with gzip.open(path, "rt") as f:
            return json.load(f)
    if name.endswith(".xz"):
        with lzma.open(path, "rt") as f:
            return json.load(f)
    with open(path) as f:
        return json.load(f)


def write_capacity_file(tmp_path):
    """the reference's instance-type table as a CAPACITY_DATA file (values from the golden hex floats)."""
    rows = load_json("capacity_table.json")["rows"]
    table = OrderedDict((itype, OrderedDict((k, float.fromhex(v)) for k, v in spec.items())) for itype, spec in rows)
    path = os.path.join(str(tmp_path), "capacity.json")
    with open(path, "w") as f:
        json.dump(table, f)
    return path


class FakeKubeObject(object):
    """what the host layer needs from a pykube object: .obj, .name, reload/update/delete."""

    def __init__(self, obj, journal, kind):
        self.obj = copy.deepcopy(obj)
        self._journal = journal
        self._kind = kind

    @property
    def name(self):
        return self.obj["metadata"]["name"]

    def reload(self):
        self._journal.append([self._kind + ".reload", self.name])

    def update(self):
        self._journal.append([self._kind + ".update", self.name, bool(self.obj["spec"].get("unschedulable")),
                              self.obj["metadata"]["labels"].get("openai/cordoned-by-autoscaler")])

    def delete(self):
        self._journal.append([self._kind + ".delete", self.name])


class ListHandler(logging.Handler):
    def __init__(self):
        super().__init__(level=logging.DEBUG)
        self.records = []

    def emit(self, record):
        self.records.append([record.levelname, record.name, record.getMessage()])


def parse_now(state):
    return datetime.datetime.strptime(state["now"], "%Y-%m-%dT%H:%M:%SZ").replace(tzinfo=datetime.timezone.utc)


def run_tick(state, monkeypatch):
    """mirror of oracle/make_golden.py:run_tick for the product's classes. The engine must already be
    installed with snapshot.set_engine()."""
    from kubernetes_acs_engine_autoscaler_b200 import adapters, agent_pool, cluster, engine_scaler, scaler, utils
    st = state["settings"]
    journal = []
    now = parse_now(state)
    monkeypatch.setattr(utils, "now", lambda tz=None: now.astimezone(tz) if tz is not None else now.replace(tzinfo=None))

    max_sizes = st.get("pool_max_size", {})
    orig_init = agent_pool.AgentPool.__init__

    def pool_init(self, pool_name, instance_type, nodes):
        orig_init(self, pool_name, instance_type, nodes)
        if pool_name in max_sizes:
            self.max_size = max_sizes[pool_name]
    monkeypatch.setattr(agent_pool.AgentPool, "__init__", pool_init)

    scale_calls, state_calls, deleted = [], [], []
    orig_scale = engine_scaler.EngineScaler.scale_pools

    def scale_pools(self, new_pool_sizes):
        scale_calls.append(dict(new_pool_sizes))
        return orig_scale(self, new_pool_sizes)
    monkeypatch.setattr(engine_scaler.EngineScaler, "scale_pools", scale_pools)

    orig_maintain = engine_scaler.EngineScaler.maintain

    def maintain(self, pods_to_schedule, running):
        # exercise the single-node API too, in the reference's visiting order
        by_node = {}
        for p in running:
            by_node.setdefault(p.node_name, []).append(p)
        for pool in self.scalable_pools:
            for node in pool.nodes:
                state_calls.append([node.name, self.get_node_state(node, by_node.get(node.name, []), pods_to_schedule)])
        return orig_maintain(self, pods_to_schedule, running)
    monkeypatch.setattr(engine_scaler.EngineScaler, "maintain", maintain)

    adapters.register("delete_resources_for_node", lambda node, rg: deleted.append(node.name))

    class RecDeployments(object):
        def __init__(self):
            self.requested_pool_sizes = None

        def deploy(self, func, new_pool_sizes):
            journal.append(["deploy", dict(new_pool_sizes)])

    notifier = None
    if st.get("notifier") == "recording":
        class RecNotifier(object):
            def notify_scale(self, new, pods, cur):
                journal.append(["notify_scale", dict(new), [p.name for p in pods], dict(cur)])

            def notify_failed_to_scale(self, *a):
                journal.append(["notify_failed_to_scale"])

            def notify_drained_node(self, node, pods):
                journal.append(["notify_drained_node", node.name, [p.name for p in pods]])
        notifier = RecNotifier()

    handler = ListHandler()
    root = logging.getLogger("autoscaler")
    root.setLevel(logging.DEBUG)
    root.addHandler(handler)
    root.propagate = False

    node_objs = [FakeKubeObject(o, journal, "node") for o in state["nodes"]]
    pod_objs = [FakeKubeObject(o, journal, "pod") for o in state["pods"]]
    kube_nodes = []

    class TestCluster(cluster.Cluster):
        def list_nodes(self):
            return list(node_objs)

        def list_pods(self):
            return list(pod_objs)

        def create_kube_node(self, node):
            kn = cluster.Cluster.create_kube_node(self, node)
            kube_nodes.append(kn)
            return kn

    cl = TestCluster(
        kubeconfig=None, idle_threshold=st["idle_threshold"], spare_agents=st["spare_agents"],
        service_principal_app_id="x", service_principal_secret="x", service_principal_tenant_id="x",
        subscription_id="x", client_private_key="x", ca_private_key="x", instance_init_time=600,
        resource_group="rg", notifier=notifier, ignore_pools=st["ignore_pools"],
        scale_up=st.get("scale_up", True), maintainance=st.get("maintainance", True),
        over_provision=st["over_provision"], dry_run=st["dry_run"])
    cl.deployments = RecDeployments()
    cl.api = None
    cl.arm_template = {}
    cl.arm_parameters = copy.deepcopy(state["arm_parameters"])

    result = {}
    try:
        result["return"] = cl.loop_logic()
        result["exception"] = None
    except Exception as e:
        result["return"] = None
        result["exception"] = [type(e).__name__, str(e)]
    finally:
        root.removeHandler(handler)
    result["log"] = handler.records
    result["scale_pools_calls"] = scale_calls
    result["state_calls"] = state_calls
    result["journal"] = journal
    result["deleted_nodes"] = sorted(deleted)
    result["used"] = {kn.name: {k: float(v).hex() for k, v in kn.used_capacity.raw.items()}
                      for kn in kube_nodes if not utils.is_master(kn)}
    return result


def assert_tick_matches(got, exp):
    assert got["exception"] == exp["exception"]
    assert got["return"] == exp["return"]
    assert got["scale_pools_calls"] == exp["scale_pools_calls"]
    assert got["used"] == exp["used"]
    assert got["state_calls"] == exp["state_calls"]
    assert got["journal"] == exp["journal"]
    assert got["deleted_nodes"] == exp["deleted_nodes"]
    assert got["log"] == exp["log"]
