"""Agent pool = name + instance type + its nodes (mirror of reference autoscaler/agent_pool.py)."""
import logging

from . import kube
from .capacity import get_capacity_for_instance_type

logger = logging.getLogger('autoscaler.agent_pool')

# labels of one node that a new node of the same pool does not inherit
_NODE_ONLY_LABELS = ('kubernetes.io/hostname', 'openai/cordoned-by-autoscaler')


class AgentPool(object):
    def __init__(self, pool_name, instance_type, nodes):
        self.name = pool_name
        self.nodes = nodes
        self.unschedulable_nodes = [n for n in nodes if n.unschedulable]
        self.max_size = 100  # ACS limit (agent_pool.py:18); a plain attribute, callers may raise it
        self.instance_type = instance_type

    @property
    def actual_capacity(self):
        return len(self.nodes)

    @property
    def unit_capacity(self):
        return get_capacity_for_instance_type(self.instance_type)

    @property
    def labels(self):
        """the labels a new node of this pool will carry, for matching node selectors: every label all current nodes
        share with the same value, except the per-node hostname and the autoscaler's cordon mark, plus the pool name
        and instance type, which are always set (an empty pool has just those two)."""
        common = None
        for node in self.nodes:
            node_labels = node.selectors
            if common is None:
                common = dict(node_labels)
            else:
                common = {k: v for k, v in common.items() if k in node_labels and node_labels[k] == v}
        common = common or {}
        for key in _NODE_ONLY_LABELS:
            common.pop(key, None)
        common['agentpool'] = self.name
        common['beta.kubernetes.io/instance-type'] = self.instance_type
        return common

    @property
    def taints(self):
        """the blocking taints a new node of this pool will carry, for matching tolerations: every blocking,
        non-lifecycle taint (kube.blocking_taints) all current nodes carry with the same key, value and effect, as
        (key, value, effect) tuples in sorted order.  An empty pool has none."""
        common = None
        for node in self.nodes:
            mine = kube.blocking_taints(node.taints)
            common = mine if common is None else common & mine
        return sorted(common or ())

    def reclaim_unschedulable_nodes(self, new_desired_capacity):
        """uncordon just enough of our own cordoned nodes before asking for new VMs
        (agent_pool.py:30-44; the uncordon itself is the kube adapter)."""
        desired = min(self.max_size, new_desired_capacity)
        schedulable = self.actual_capacity - len(self.unschedulable_nodes)
        if schedulable >= desired:
            return
        for node in self.unschedulable_nodes:
            if node.uncordon():
                schedulable += 1
                if schedulable == desired:
                    break

    def has_node_with_index(self, index):
        return any(node.index == index for node in self.nodes)
