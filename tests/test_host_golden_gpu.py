"""`-m gpu`: the reference's recorded ticks and known-answer tests through the product's public
classes with the REAL CUDA engine (C ABI -> sm_90a kernels): exceptions, scale_pools arguments,
used_capacity bit patterns, node states, adapter calls and the complete log text must match."""
import pytest

import golden_util as gu

pytestmark = pytest.mark.gpu

TICKS = gu.load_json("ticks.json.gz")


@pytest.fixture()
def host(tmp_path, monkeypatch, engine):
    from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
    capacity.load(gu.write_capacity_file(tmp_path), cpu_reserve=0.0)
    monkeypatch.setattr(snapshot, "_engine", engine)
    return monkeypatch


@pytest.mark.parametrize("state", TICKS, ids=[s["name"] for s in TICKS])
def test_tick_matches_reference_on_gpu(host, state):
    got = gu.run_tick(state, host)
    gu.assert_tick_matches(got, state["expected"])


def test_reference_known_answer_tests_on_gpu(host):
    import test_host_golden_cpu as cpu_tests
    cpu_tests.test_reference_known_answer_tests(host)


def test_single_item_api_on_gpu(host):
    """KubeNode.can_fit / capacity.is_possible / Scaler.get_node_state: the single-item forms."""
    from kubernetes_acs_engine_autoscaler_b200 import capacity
    from kubernetes_acs_engine_autoscaler_b200.kube import KubeNode, KubePod, KubeResource
    kat = gu.load_json("kat_reference_tests.json")["test_get_pending_pods"]
    n = KubeNode(gu.FakeKubeObject(kat["node"], [], "node"))
    n.capacity = capacity.get_capacity_for_instance_type(n.instance_type)
    p = KubePod(gu.FakeKubeObject(kat["pod"], [], "pod"))
    assert n.can_fit(p.resources)
    n.count_pod(p)
    assert not n.can_fit(p.resources)
    assert n.can_fit(KubeResource(cpu="500m"))
    assert not n.can_fit(KubeResource(**{"nvidia.com/gpu": 1}))

    class Pool(object):
        instance_type = "Standard_D2_v2"
    assert capacity.is_possible(p, [Pool()])
    Pool.instance_type = "Standard_M128s"  # the " pods" typo row: nothing ever fits (SURVEY 0.6)
    assert not capacity.is_possible(p, [Pool()])
