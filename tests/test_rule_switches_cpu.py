"""The ten opt-in scheduling-rule switches of Cluster, without a GPU: how each resolves from its keyword, its
environment variable and its prerequisite switch, and what reaches EngineScaler and Scaler.

* An explicit True or False wins over the environment; an explicit True without its prerequisite is a ValueError.
* None reads the environment variable ('' and '0' are off); an environment True without the prerequisite is off.
* Cluster hands every resolved switch to EngineScaler by name; Scaler starts with every switch False, and EngineScaler
  refuses a keyword that is no switch."""
import itertools
from types import SimpleNamespace

import pytest

from kubernetes_acs_engine_autoscaler_b200 import cluster, engine_scaler
from kubernetes_acs_engine_autoscaler_b200.scaler import Scaler

# (switch, environment variable, prerequisite switch)
SWITCHES = [
    ("node_selectors", "ACSFIT_NODE_SELECTORS", None),
    ("selector_node_states", "ACSFIT_SELECTOR_NODE_STATES", "node_selectors"),
    ("node_taints", "ACSFIT_NODE_TAINTS", "node_selectors"),
    ("node_affinity", "ACSFIT_NODE_AFFINITY", "node_selectors"),
    ("pod_anti_affinity", "ACSFIT_POD_ANTI_AFFINITY", None),
    ("anti_affinity_node_states", "ACSFIT_ANTI_AFFINITY_NODE_STATES", "pod_anti_affinity"),
    ("pod_affinity", "ACSFIT_POD_AFFINITY", None),
    ("pod_affinity_node_states", "ACSFIT_POD_AFFINITY_NODE_STATES", "pod_affinity"),
    ("topology_spread", "ACSFIT_TOPOLOGY_SPREAD", None),
    ("topology_spread_node_states", "ACSFIT_TOPOLOGY_SPREAD_NODE_STATES", "topology_spread"),
]
NAMES = [name for name, _, _ in SWITCHES]


@pytest.fixture(autouse=True)
def clean_env(monkeypatch):
    for _, env, _ in SWITCHES:
        monkeypatch.delenv(env, raising=False)


def _cluster(**kw):
    return cluster.Cluster(None, 1800, 1, "a", "b", "c", "d", "e", "f", 600, "rg", None, "", **kw)


def _resolved(c):
    return {name: getattr(c, name) for name in NAMES}


CASES = [(name, env, needs, value, env_value, pre)
         for name, env, needs in SWITCHES
         for value, env_value, pre in itertools.product((True, False, None), (None, "", "0", "1"),
                                                        (True, False) if needs else (None,))]


@pytest.mark.parametrize("name,env,needs,value,env_value,pre", CASES,
                         ids=["%s-%s-env%s-pre%s" % (c[0], c[3], c[4], c[5]) for c in CASES])
def test_switch_resolution(monkeypatch, name, env, needs, value, env_value, pre):
    if env_value is not None:
        monkeypatch.setenv(env, env_value)
    kw = {name: value}
    if needs:
        kw[needs] = pre
    if value is True and needs and not pre:
        with pytest.raises(ValueError) as err:
            _cluster(**kw)
        assert str(err.value) == "%s=True needs %s on" % (name, needs)
        return
    c = _cluster(**kw)
    on = value if value is not None else env_value not in (None, "", "0")
    want = dict.fromkeys(NAMES, False)
    if needs:
        want[needs] = pre
    want[name] = on and (pre if needs else True)
    got = _resolved(c)
    assert got == want
    assert all(type(v) is bool for v in got.values())


def test_environment_alone_resolves_in_table_order(monkeypatch):
    """a dependent switch sees its prerequisite as resolved from the environment too"""
    for _, env, _ in SWITCHES:
        monkeypatch.setenv(env, "1")
    assert _resolved(_cluster()) == dict.fromkeys(NAMES, True)
    monkeypatch.setenv("ACSFIT_POD_AFFINITY", "0")
    want = dict.fromkeys(NAMES, True)
    want["pod_affinity"] = want["pod_affinity_node_states"] = False
    assert _resolved(_cluster()) == want
    with pytest.raises(ValueError, match="^pod_affinity_node_states=True needs pod_affinity on$"):
        _cluster(pod_affinity_node_states=True)


class _Stop(Exception):
    pass


@pytest.mark.parametrize("on", [(), tuple(NAMES), ("node_selectors", "node_taints", "pod_affinity"),
                                ("topology_spread", "topology_spread_node_states", "pod_anti_affinity")],
                         ids=["none", "all", "some", "spread"])
def test_switches_reach_engine_scaler(monkeypatch, on):
    seen = []

    class Rec(engine_scaler.EngineScaler):
        def __init__(self, **kw):
            seen.append(kw)
            engine_scaler.EngineScaler.__init__(self, **kw)
            seen.append(self)
            raise _Stop()
    monkeypatch.setattr(cluster, "EngineScaler", Rec)
    cl = _cluster(**{name: name in on for name in NAMES})
    cl.list_nodes = lambda: [SimpleNamespace(name=name, unschedulable=False)
                             for name in ("k8s-cpu-1-0", "k8s-master-1-0")]
    cl.create_kube_node = lambda n: n
    cl.arm_parameters, cl.arm_template = {"cpuVMSize": {"value": "Standard_D2_v2"}}, {}
    with pytest.raises(_Stop):
        cl.loop_logic()
    kw, scaler = seen
    assert {name: kw[name] for name in NAMES} == {name: name in on for name in NAMES}
    assert set(kw) - set(NAMES) == {"resource_group", "nodes", "deployments", "arm_template", "arm_parameters",
                                    "dry_run", "ignore_pools", "over_provision", "spare_count", "idle_threshold",
                                    "notifier", "other_nodes"}
    assert [n.name for n in kw["other_nodes"]] == (["k8s-master-1-0"] if "topology_spread" in on else [])
    assert _resolved(scaler) == {name: name in on for name in NAMES}
    assert [n.name for n in scaler.other_nodes] == [n.name for n in kw["other_nodes"]]


def _engine_scaler(**kw):
    return engine_scaler.EngineScaler("rg", [], 0, 1, 1800, True, None, {}, {}, "", None, **kw)


def test_scaler_defaults_and_unknown_keyword():
    assert _resolved(Scaler("rg", [], 0, 1, 1800, True, None, None)) == dict.fromkeys(NAMES, False)
    s = _engine_scaler()
    assert _resolved(s) == dict.fromkeys(NAMES, False) and s.other_nodes == []
    for name in NAMES:
        s = _engine_scaler(**{name: True})
        assert _resolved(s) == {n: n == name for n in NAMES}
    assert _engine_scaler(other_nodes=("m",)).other_nodes == ["m"]
    with pytest.raises(TypeError, match="node_selector"):
        _engine_scaler(node_selector=True)
