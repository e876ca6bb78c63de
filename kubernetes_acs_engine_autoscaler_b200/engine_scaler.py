"""acs-engine back end of the scaler (mirror of reference autoscaler/engine_scaler.py).

Pool discovery, the scale_pools hand-off (dry-run gate) and the maintain state machine keep the
reference's behaviour; node classification and the drain-budget ranks are computed for all nodes
at once on the GPU.  Deployments and VM deletion are the adapter boundary (adapters.py).
"""
import logging
import uuid
from threading import Lock, Thread

from . import adapters
from . import snapshot
from . import utils
from .agent_pool import AgentPool
from .scaler import RULE_SWITCHES, STATE_NAMES, ClusterNodeState, Scaler

logger = logging.getLogger('autoscaler.engine_scaler')

ACT_NONE, ACT_CORDON_DRAIN, ACT_CORDON, ACT_UNCORDON, ACT_SCALE_IN = range(5)
SWITCH_NAMES = frozenset(name for name, _, _ in RULE_SWITCHES)


class EngineScaler(Scaler):
    def __init__(self, resource_group, nodes, over_provision, spare_count, idle_threshold, dry_run,
                 deployments, arm_template, arm_parameters, ignore_pools, notifier, *, other_nodes=(), **switches):
        """`switches`: the rule switches of scaler.RULE_SWITCHES by name (False when not given)"""
        Scaler.__init__(self, resource_group, nodes, over_provision, spare_count, idle_threshold, dry_run,
                        deployments, notifier)
        for name, value in switches.items():
            if name not in SWITCH_NAMES:
                raise TypeError("EngineScaler() got an unexpected keyword argument '%s'" % name)
            setattr(self, name, value)
        self.other_nodes = list(other_nodes)
        self.arm_parameters = arm_parameters
        self.arm_template = arm_template
        for pool_name in ignore_pools.split(','):  # '' -> {'': True}, like the reference (:31-32)
            self.ignored_pool_names[pool_name] = True
        self.agent_pools, self.scalable_pools = self.get_agent_pools(nodes)

    def get_agent_pools(self, nodes):
        """one pool per `<name>VMSize` ARM parameter except the master's, in parameter order;
        nodes are bucketed by the pool part of their name (engine_scaler.py:35-56)."""
        buckets = {}
        for param, spec in self.arm_parameters.items():
            if param.endswith('VMSize') and param != 'masterVMSize':
                buckets.setdefault(param[:-len('VMSize')], (spec['value'], []))
        for node in nodes:
            buckets[utils.get_pool_name(node)][1].append(node)  # unknown pool -> KeyError, as upstream
        agent_pools, scalable_pools = [], []
        for name, (vm_size, members) in buckets.items():
            pool = AgentPool(name, vm_size, members)
            agent_pools.append(pool)
            if name not in self.ignored_pool_names:
                scalable_pools.append(pool)
        return agent_pools, scalable_pools

    def delete_node(self, pool, node, lock):
        sizes = {}
        with lock:
            for pool in self.agent_pools:  # (sic) the loop variable shadows the argument upstream too
                sizes[pool.name] = pool.actual_capacity
            sizes[pool.name] = pool.actual_capacity - 1
            self.deployments.requested_pool_sizes = sizes
        adapters.call("delete_resources_for_node", node, self.resource_group_name)

    def scale_pools(self, new_pool_sizes):
        """clamp to max_size, report or act (engine_scaler.py:68-88)."""
        has_changes = False
        for pool in self.scalable_pools:
            new_size = new_pool_sizes[pool.name]
            new_pool_sizes[pool.name] = min(pool.max_size, new_size)
            if new_pool_sizes[pool.name] == pool.actual_capacity:
                logger.info("Pool '{}' already at desired capacity ({})".format(pool.name, pool.actual_capacity))
                continue
            has_changes = True
            if not self.dry_run:
                if new_size > pool.actual_capacity:
                    pool.reclaim_unschedulable_nodes(new_size)
            else:
                logger.info("[Dry run] Would have scaled pool '{}' to {} agent(s) (currently at {})".format(
                    pool.name, new_size, pool.actual_capacity))
        if not self.dry_run and has_changes:
            self.deployments.deploy(lambda: self.deploy_pools(new_pool_sizes), new_pool_sizes)

    def deploy_pools(self, new_pool_sizes):
        """ARM incremental deployment of the new sizes -- adapter boundary (engine_scaler.py:90-118)."""
        from azure.mgmt.resource.resources.models import DeploymentProperties
        for pool in self.scalable_pools:
            if new_pool_sizes[pool.name] == 0:
                self.arm_parameters[pool.name + 'Count'] = {'value': 1}
                self.arm_parameters[pool.name + 'Offset'] = {'value': 1}
            else:
                self.arm_parameters[pool.name + 'Count'] = {'value': new_pool_sizes[pool.name]}
        template = adapters.call("prepare_template_for_scale_out", self.arm_template, self.agent_pools,
                                 new_pool_sizes)
        properties = DeploymentProperties(template=template, template_link=None,
                                          parameters=self.arm_parameters, mode='incremental')
        deployment_name = "autoscaler-deployment-{}".format(str(uuid.uuid4()).split('-')[0])
        logger.info('Deployment {} started...'.format(deployment_name))
        return adapters.call("create_deployment", self.resource_group_name, deployment_name, properties)

    def maintain(self, pods_to_schedule, running_or_pending_assigned_pods):
        """decide, per node of every scalable pool, whether to drain / cordon / uncordon / scale in
        (engine_scaler.py:120-192)."""
        logger.info("++++ Maintaining Nodes ++++++")
        pods_by_node = {}
        for p in running_or_pending_assigned_pods:
            pods_by_node.setdefault(p.node_name, []).append(p)

        # flatten: nodes of the scalable pools, pool by pool, in pool.nodes order
        nodes, node_pool, budget0 = [], [], []
        for t, pool in enumerate(self.scalable_pools):
            budget0.append(pool.actual_capacity - len(pool.unschedulable_nodes) - self.spare_count)
            nodes.extend(pool.nodes)
            node_pool.extend([t] * len(pool.nodes))
        delete_queue = []
        if nodes:
            lists = [pods_by_node.get(node.name, []) for node in nodes]
            state_dev = snapshot.node_states(nodes, lists, bool(pods_to_schedule), self.idle_threshold,
                                             **self.pending_flags(nodes, lists, pods_to_schedule,
                                                                  running_or_pending_assigned_pods,
                                                                  agent_pools=self.agent_pools))
            states, actions = snapshot.maintain_actions(state_dev, node_pool, budget0, [1] * len(budget0),
                                                        self.dry_run)
            info = logger.isEnabledFor(logging.INFO)  # (formatted eagerly, as upstream: skipped when nobody listens)
            states, actions = states.tolist(), actions.tolist()
            for i, node in enumerate(nodes):
                state = STATE_NAMES[states[i]]
                if info:
                    logger.info("node: %-*s state: %s" % (75, node, state))
                action = actions[i]
                if action == ACT_NONE:
                    if state not in (ClusterNodeState.POD_PENDING, ClusterNodeState.BUSY,
                                     ClusterNodeState.SPARE_AGENT, ClusterNodeState.GRACE_PERIOD,
                                     ClusterNodeState.UNDER_UTILIZED_UNDRAINABLE):
                        raise Exception("Unhandled state: {}".format(state))
                elif action == ACT_CORDON_DRAIN:
                    if not self.dry_run:
                        node.cordon()
                        node.drain(pods_by_node.get(node.name, []), self.notifier or None)
                    else:
                        logger.info('[Dry run] Would have drained and cordoned %s', node)
                elif action == ACT_CORDON:
                    if not self.dry_run:
                        node.cordon()
                    else:
                        logger.info('[Dry run] Would have cordoned %s', node)
                elif action == ACT_UNCORDON:
                    if not self.dry_run:
                        node.uncordon()
                    else:
                        logger.info('[Dry run] Would have uncordoned %s', node)
                elif action == ACT_SCALE_IN:
                    if not self.dry_run:
                        delete_queue.append({'node': node, 'pool': self.scalable_pools[node_pool[i]]})
                    else:
                        logger.info('[Dry run] Would have scaled in %s', node)

        threads, lock = [], Lock()
        for item in delete_queue:
            t = Thread(target=self.delete_node, args=(item['pool'], item['node'], lock,))
            threads.append(t)
            t.start()
        for t in threads:
            t.join()
