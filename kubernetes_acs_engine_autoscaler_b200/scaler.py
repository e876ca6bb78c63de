"""Scaling policy (mirror of reference autoscaler/scaler.py): fulfill_pending and get_node_state.

The packing / classification arithmetic runs in libacsfit.so (first-fit pipeline over bins,
idle scan); this class keeps the reference's surface, log lines and error behaviour.
"""
import logging
import os

import numpy as np

from . import capacity
from . import snapshot

logger = logging.getLogger('autoscaler.scaler')


class ClusterNodeState(object):
    INSTANCE_TERMINATED = 'instance-terminated'
    POD_PENDING = 'pod-pending'
    GRACE_PERIOD = 'grace-period'
    SPARE_AGENT = 'spare-agent'
    IDLE_SCHEDULABLE = 'idle-schedulable'
    IDLE_UNSCHEDULABLE = 'idle-unschedulable'
    BUSY_UNSCHEDULABLE = 'busy-unschedulable'
    BUSY = 'busy'
    UNDER_UTILIZED_DRAINABLE = 'under-utilized-drainable'
    UNDER_UTILIZED_UNDRAINABLE = 'under-utilized-undrainable'


# include/acsfit.h ACSFIT_ST_* code -> state string (listing order of scaler.py:19-29)
STATE_NAMES = [
    ClusterNodeState.INSTANCE_TERMINATED, ClusterNodeState.POD_PENDING, ClusterNodeState.GRACE_PERIOD,
    ClusterNodeState.SPARE_AGENT, ClusterNodeState.IDLE_SCHEDULABLE, ClusterNodeState.IDLE_UNSCHEDULABLE,
    ClusterNodeState.BUSY_UNSCHEDULABLE, ClusterNodeState.BUSY, ClusterNodeState.UNDER_UTILIZED_DRAINABLE,
    ClusterNodeState.UNDER_UTILIZED_UNDRAINABLE,
]
# per-pod log lines are only emitted up to this many pods (SURVEY.md section 5: O(P) strings)
LOG_DETAIL_LIMIT = 20000

# The opt-in scheduling rules, all off by default: (switch, environment variable read when Cluster gets None, the switch
# it needs on or None).  Cluster resolves them in this order and hands them to EngineScaler by name.
RULE_SWITCHES = (
    # honour spec.nodeSelector in scale-up; the reference ignores selectors, and its recorded ticks pin that
    ('node_selectors', 'ACSFIT_NODE_SELECTORS', None),
    # in maintain too: a pod pinned to one pool does not freeze scale-down in the others
    ('selector_node_states', 'ACSFIT_SELECTOR_NODE_STATES', 'node_selectors'),
    # a tainted (e.g. GPU) pool neither absorbs nor holds back the pods that do not tolerate its taints
    ('node_taints', 'ACSFIT_NODE_TAINTS', 'node_selectors'),
    # a pod pinned to a pool by required node affinity neither fits nor holds back other pools' nodes
    ('node_affinity', 'ACSFIT_NODE_AFFINITY', 'node_selectors'),
    # replicas that avoid each other (hostname anti-affinity) are not simulated onto one node or new node
    ('pod_anti_affinity', 'ACSFIT_POD_ANTI_AFFINITY', None),
    # in maintain too: a pending replica does not freeze the nodes that run its siblings
    ('anti_affinity_node_states', 'ACSFIT_ANTI_AFFINITY_NODE_STATES', 'pod_anti_affinity'),
    # a pod that must sit beside another (hostname affinity) lands neither on a node without one nor alone
    ('pod_affinity', 'ACSFIT_POD_AFFINITY', None),
    # in maintain too: a pod that needs a pod elsewhere does not freeze every idle node
    ('pod_affinity_node_states', 'ACSFIT_POD_AFFINITY_NODE_STATES', 'pod_affinity'),
    # replicas spread over hostnames (DoNotSchedule) are not simulated onto one roomy node
    ('topology_spread', 'ACSFIT_TOPOLOGY_SPREAD', None),
    # in maintain too: a replica that may not stack beside its siblings does not freeze their nodes
    ('topology_spread_node_states', 'ACSFIT_TOPOLOGY_SPREAD_NODE_STATES', 'topology_spread'),
)


class Scaler(object):
    # a node is under-utilised when its busy pods use <= 30 % of every capacity dimension
    UTIL_THRESHOLD = 0.3
    # What happens when some pending pods cannot be accounted for (a pool at max_size, duplicate uids).  The
    # reference evaluates an undefined name there (scaler.py:181) and therefore RAISES before scale_pools: one
    # saturated pool suppresses the scale-up of every other pool for the tick.  True (default) reproduces that, as
    # the recorded reference ticks require; False is the behaviour the reference evidently meant -- tell the
    # notifier, then still scale the pools that can grow.  ($ACSFIT_SCALE_WHEN_INSUFFICIENT=1 selects False.)
    REFERENCE_RAISE_ON_INSUFFICIENT = os.environ.get('ACSFIT_SCALE_WHEN_INSUFFICIENT', '0') in ('', '0')

    def __init__(self, resource_group, nodes, over_provision, spare_count, idle_threshold, dry_run,
                 deployments, notifier):
        self.resource_group_name = resource_group
        self.over_provision = over_provision
        self.spare_count = spare_count
        self.idle_threshold = idle_threshold
        self.dry_run = dry_run
        self.deployments = deployments
        self.notifier = notifier
        self.max_agent_pool_size = 100
        self.agent_pools = None
        self.scalable_pools = None
        self.ignored_pool_names = {}
        for name, _, _ in RULE_SWITCHES:  # Cluster(<name>=...)
            setattr(self, name, False)
        # the listed nodes that are not agents (the master): domains of the spread constraints
        self.other_nodes = []

    def get_agent_pools(self, nodes):
        raise NotImplementedError()

    def scale_pools(self, pool_sizes):
        raise NotImplementedError()

    def no_pending_match(self, nodes, pods_to_schedule):
        """bool[len(nodes)] for snapshot.node_states(no_match=...): the nodes no pod to schedule matches, or None
        when every node keeps the reference's "any pod to schedule" rule (the switch is off, or nothing is pending)."""
        if not self.selector_node_states or not pods_to_schedule:
            return None
        return ~snapshot.pending_match(pods_to_schedule, nodes, taints=self.node_taints, affinity=self.node_affinity)

    def pending_flags(self, nodes, pods_lists, pods_to_schedule, running_pods, agent_pools=None):
        """the keywords `no_match` and `admit` of snapshot.node_states.  With anti_affinity_node_states,
        pod_affinity_node_states or topology_spread_node_states on, something to schedule and some term or constraint
        that can exclude a pod to schedule, the GPU decides which nodes some pod to schedule is admitted to
        (snapshot.pending_admit: the enabled tests, node selectors included when selector_node_states is on);
        otherwise no_pending_match decides.  A self-affine group may bootstrap while no pod of `running_pods` on a node
        of `agent_pools` matches it (None: no pod of `pods_lists`).  The spread minimums count the nodes of
        `agent_pools` outside `nodes` and self.other_nodes as domains (None: `nodes` alone)."""
        admit = None
        if (self.anti_affinity_node_states or self.pod_affinity_node_states or self.topology_spread_node_states) and \
                pods_to_schedule:
            agent_nodes = None
            if self.pod_affinity_node_states and agent_pools is not None:
                agent_nodes = [n for pool in agent_pools for n in pool.nodes]
            other_nodes = ()
            if self.topology_spread_node_states and agent_pools is not None:
                listed = {n.name for n in nodes}
                other_nodes = [n for pool in agent_pools for n in pool.nodes if n.name not in listed] + \
                    list(self.other_nodes)
            admit = snapshot.pending_admit(pods_to_schedule, running_pods, nodes, pods_lists,
                                           selectors=self.selector_node_states, taints=self.node_taints,
                                           affinity=self.node_affinity, anti_affinity=self.anti_affinity_node_states,
                                           pod_affinity=self.pod_affinity_node_states, agent_nodes=agent_nodes,
                                           topology_spread=self.topology_spread_node_states, other_nodes=other_nodes)
        if admit is not None:
            return {"no_match": None, "admit": admit}
        return {"no_match": self.no_pending_match(nodes, pods_to_schedule), "admit": None}

    def get_node_state(self, node, node_pods, pods_to_schedule):
        """ClusterNodeState of one node (scaler.py:61-114): a one-node launch of the idle scan.
        EngineScaler.maintain classifies all nodes in a single launch instead.  The anti-affinity, pod-affinity and
        topology-spread rules see only `node` and `node_pods`: with pod_affinity_node_states on, a self-affine group may
        bootstrap here unless one of `node_pods` matches it, whereas maintain looks for a match on every agent node;
        with topology_spread_node_states on, a key's minimum is the node's own count (0 when the key has fewer domains
        than its minDomains), whereas maintain takes it over every listed node."""
        node_pods = list(node_pods)
        code = snapshot.node_states([node], [node_pods], bool(pods_to_schedule), self.idle_threshold,
                                    **self.pending_flags([node], [node_pods], pods_to_schedule, node_pods))
        return STATE_NAMES[int(code.cpu().numpy()[0])]

    def fulfill_pending(self, pods, affinity_present=()):
        """number of new VMs per pool needed for the pending pods (scaler.py:117-184).  `affinity_present`: with pod
        affinity on, the signatures the nodes already hold (Cluster.affinity_present); without it only the pods this
        call places count."""
        logger.info("====Scaling for %s pods ====", len(pods))
        # the reference keys its bookkeeping by pod (hash = uid): duplicates collapse onto their first
        # occurrence, but num_unaccounted starts at len(pods) (scaler.py:119-120)
        unique = list(dict((p, False) for p in pods).keys())
        ordered_pools = capacity.order_by_cost_asc(self.agent_pools)
        classes = None
        if self.node_selectors:
            classes = snapshot.selector_classes(unique, [], ordered_pools, taints=self.node_taints,
                                                affinity=self.node_affinity)
        anti_affinity = snapshot.anti_affinity(unique) if self.pod_anti_affinity else None
        pod_affinity = snapshot.pod_affinity(unique) if self.pod_affinity else None
        topology_spread = snapshot.topology_spread(unique) if self.topology_spread else None
        res = snapshot.fulfill(unique, len(pods), ordered_pools, self.ignored_pool_names, self.over_provision,
                               classes=classes, anti_affinity=anti_affinity, pod_affinity=pod_affinity,
                               affinity_present=affinity_present, topology_spread=topology_spread)

        new_pool_sizes, current_pool_sizes = {}, {}
        unaccounted = len(pods)
        acc = res["acc_pool"]
        for t, pool in enumerate(ordered_pools):
            current_pool_sizes[pool.name] = pool.actual_capacity
            new_pool_sizes[pool.name] = int(res["new_size"][t])
            needed = int(res["units_needed"][t])
            if needed < 0:  # pool skipped (ignored, or nothing left to place)  scaler.py:128-129
                continue
            requested = new_pool_sizes[pool.name] - pool.actual_capacity
            logger.debug("units_needed: %s", needed)
            logger.debug("units_requested: %s", requested)
            logger.debug('{} actual capacity: {} , units requested: {}'.format(
                pool.name, pool.actual_capacity, requested))
            logger.info("New capacity requested for pool {}: {} agents (current capacity: {} agents)".format(
                pool.name, new_pool_sizes[pool.name], pool.actual_capacity))
            unaccounted -= int(np.count_nonzero(acc == t))
            logger.debug("remaining pending: %s", unaccounted)
        assert unaccounted == res["num_unaccounted"]

        if unaccounted and pod_affinity is not None and logger.isEnabledFor(logging.WARNING):
            # a pod that no bin of any pool took although it passed the feasibility check: its affinity kept it out
            for p, t, b, r in zip(unique, acc.tolist(), res["bin_of"].tolist(), pod_affinity.pod_requires.tolist()):
                if t < 0 and b < 0 and r:
                    logger.warning("Pending pod %s cannot fit: no node or new node would hold a pod its required pod "
                                   "affinity selects. Scheduling skipped." % p.name)
        if unaccounted:
            logger.warning('Failed to scale sufficiently.')
            if self.REFERENCE_RAISE_ON_INSUFFICIENT:
                # the reference evaluates `self.notifier.notify_failed_to_scale(selectors_hash, pods)` here,
                # where `selectors_hash` is an undefined name (scaler.py:181): AttributeError when the
                # notifier lacks the method, NameError otherwise -- and scale_pools is never reached.
                self.notifier.notify_failed_to_scale
                raise NameError("name 'selectors_hash' is not defined")
            if self.notifier:
                left = [p for p, t in zip(unique, acc.tolist()) if t < 0]
                if not self.node_selectors:
                    self.notifier.notify_failed_to_scale({}, left)
                else:  # once per selector of the unaccounted pods, as the upstream code grouped them
                    groups = {}
                    for p in left:
                        groups.setdefault(tuple(sorted(p.selectors.items())), []).append(p)
                    for items, group in groups.items():
                        self.notifier.notify_failed_to_scale(dict(items), group)
        self.scale_pools(new_pool_sizes)
        if self.notifier:
            self.notifier.notify_scale(new_pool_sizes, pods, current_pool_sizes)
