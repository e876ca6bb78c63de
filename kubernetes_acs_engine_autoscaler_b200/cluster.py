"""One tick of the autoscaler (mirror of reference autoscaler/cluster.py).

`Cluster.loop` (alias `scale_loop`, the name the north-star uses) lists nodes and pods through
the kube adapter, then runs the whole decision path on the GPU:
    occupancy (K1) -> get_pods_to_schedule (K0) -> get_pending_pods (first-fit pipeline, nodes)
    -> Scaler.fulfill_pending (first-fit pipeline, bins) -> EngineScaler.maintain (idle scan)
and hands the results back through the same calls the reference makes (scale_pools, the
KubeNode mutators, the notifier).  `--dry-run` gates every side effect exactly as upstream.
"""
import base64
import logging
import os
import sys

from . import adapters
from . import capacity
from . import kube
from . import snapshot
from . import utils
from .deployments import Deployments
from .engine_scaler import EngineScaler
from .kube import KubeNode, KubePod, KubePodStatus
from .scaler import LOG_DETAIL_LIMIT

logger = logging.getLogger('autoscaler.cluster')

# inert stand-in for the certificate / key parameters an incremental agent-pool deployment never reads
PLACEHOLDER_KEY = base64.b64encode(b"-----BEGIN CERTIFICATE-----\r\nacsfit placeholder, not a key\r\n"
                                   b"-----END CERTIFICATE-----\r\n").decode("ascii")

_pykube_ready = False


def _pykube():
    """import pykube once and apply the two process-wide settings the reference applies at import
    (cluster.py:20-28): list pods of ALL namespaces (system pods count towards occupancy and may be
    pending), and let urllib3 accept IP addresses in the API server certificate."""
    global _pykube_ready
    import pykube
    if not _pykube_ready:
        pykube.Pod.objects.namespace = None
        try:
            import backports.ssl_match_hostname as _bsm
            pykube.http.requests.packages.urllib3.connection.match_hostname = _bsm.match_hostname
        except (ImportError, AttributeError):  # python >= 3.7 ssl matches IP SANs natively
            pass
        _pykube_ready = True
    return pykube


class Cluster(object):
    def __init__(self, kubeconfig, idle_threshold, spare_agents,
                 service_principal_app_id, service_principal_secret, service_principal_tenant_id,
                 subscription_id, client_private_key, ca_private_key,
                 instance_init_time, resource_group, notifier, ignore_pools,
                 acs_deployment='azuredeploy', scale_up=True, maintainance=True,
                 over_provision=5, dry_run=False, node_selectors=None, selector_node_states=None,
                 node_taints=None, pod_anti_affinity=None, node_affinity=None, anti_affinity_node_states=None,
                 pod_affinity=None, pod_affinity_node_states=None, topology_spread=None,
                 topology_spread_node_states=None):
        self.kubeconfig = kubeconfig
        # honour the pods' spec.nodeSelector in the scale-up decision (opt-in; None: $ACSFIT_NODE_SELECTORS, off
        # by default).  The reference ignores selectors, and the recorded reference ticks pin that behaviour.
        if node_selectors is None:
            node_selectors = os.environ.get('ACSFIT_NODE_SELECTORS', '0') not in ('', '0')
        self.node_selectors = bool(node_selectors)
        # with node selectors on, also in maintain: a node is pod-pending only when a pod to schedule matches it, so a
        # pod pinned to one pool does not freeze scale-down in the others (opt-in; None: $ACSFIT_SELECTOR_NODE_STATES)
        if selector_node_states is None:
            selector_node_states = os.environ.get('ACSFIT_SELECTOR_NODE_STATES', '0') not in ('', '0')
        elif selector_node_states and not self.node_selectors:
            raise ValueError("selector_node_states=True needs node_selectors on")
        self.selector_node_states = bool(selector_node_states) and self.node_selectors
        # with node selectors on, a pod matches a node or pool only when it also tolerates every blocking taint there,
        # so a tainted (e.g. GPU) pool neither absorbs nor holds back the pods it would refuse (opt-in; None:
        # $ACSFIT_NODE_TAINTS)
        if node_taints is None:
            node_taints = os.environ.get('ACSFIT_NODE_TAINTS', '0') not in ('', '0')
        elif node_taints and not self.node_selectors:
            raise ValueError("node_taints=True needs node_selectors on")
        self.node_taints = bool(node_taints) and self.node_selectors
        # with node selectors on, a pod matches a node or pool only when its required node affinity admits it too, so a
        # pod pinned to a pool by affinity neither "fits" other pools' nodes nor holds them back (opt-in; None:
        # $ACSFIT_NODE_AFFINITY)
        if node_affinity is None:
            node_affinity = os.environ.get('ACSFIT_NODE_AFFINITY', '0') not in ('', '0')
        elif node_affinity and not self.node_selectors:
            raise ValueError("node_affinity=True needs node_selectors on")
        self.node_affinity = bool(node_affinity) and self.node_selectors
        # honour required pod anti-affinity with topologyKey kubernetes.io/hostname in first fit and bin packing, so that
        # replicas which avoid each other are not simulated onto one node (opt-in; None: $ACSFIT_POD_ANTI_AFFINITY).
        # Independent of node_selectors; with both on, the node pass uses both.
        if pod_anti_affinity is None:
            pod_anti_affinity = os.environ.get('ACSFIT_POD_ANTI_AFFINITY', '0') not in ('', '0')
        self.pod_anti_affinity = bool(pod_anti_affinity)
        # with pod anti-affinity on, also in maintain: a node is pod-pending only when some pod to schedule could land on
        # it given the pods already there, so a pending replica does not freeze the nodes that run its siblings
        # (opt-in; None: $ACSFIT_ANTI_AFFINITY_NODE_STATES).  With selector_node_states on, both rules apply.
        if anti_affinity_node_states is None:
            anti_affinity_node_states = os.environ.get('ACSFIT_ANTI_AFFINITY_NODE_STATES', '0') not in ('', '0')
        elif anti_affinity_node_states and not self.pod_anti_affinity:
            raise ValueError("anti_affinity_node_states=True needs pod_anti_affinity on")
        self.anti_affinity_node_states = bool(anti_affinity_node_states) and self.pod_anti_affinity
        # honour required pod affinity with topologyKey kubernetes.io/hostname in first fit and bin packing, so that a pod
        # which must sit beside another is neither simulated onto a node without one nor packed into a new node alone
        # (opt-in; None: $ACSFIT_POD_AFFINITY).  Independent of node selectors and anti-affinity.
        if pod_affinity is None:
            pod_affinity = os.environ.get('ACSFIT_POD_AFFINITY', '0') not in ('', '0')
        self.pod_affinity = bool(pod_affinity)
        # with pod affinity on, also in maintain: a node is pod-pending only when some pod to schedule could land on it
        # given its required pod affinity, so a pod that needs a pod elsewhere does not freeze every idle node (opt-in;
        # None: $ACSFIT_POD_AFFINITY_NODE_STATES).  Combines with selector_node_states and anti_affinity_node_states.
        if pod_affinity_node_states is None:
            pod_affinity_node_states = os.environ.get('ACSFIT_POD_AFFINITY_NODE_STATES', '0') not in ('', '0')
        elif pod_affinity_node_states and not self.pod_affinity:
            raise ValueError("pod_affinity_node_states=True needs pod_affinity on")
        self.pod_affinity_node_states = bool(pod_affinity_node_states) and self.pod_affinity
        self.affinity_present = set()  # signatures the last node pass left on some node (scale() hands them on)
        # honour topologySpreadConstraints with topologyKey kubernetes.io/hostname and whenUnsatisfiable DoNotSchedule in
        # first fit and bin packing, so that replicas spread over nodes are not simulated onto one roomy node (opt-in;
        # None: $ACSFIT_TOPOLOGY_SPREAD).  Independent of the other switches.
        if topology_spread is None:
            topology_spread = os.environ.get('ACSFIT_TOPOLOGY_SPREAD', '0') not in ('', '0')
        self.topology_spread = bool(topology_spread)
        # with topology spread on, also in maintain: a node is pod-pending only when some pod to schedule could land on it
        # given its spread constraint, so a replica that may not stack beside its siblings does not freeze their nodes
        # (opt-in; None: $ACSFIT_TOPOLOGY_SPREAD_NODE_STATES).  Combines with the other node-states switches.
        if topology_spread_node_states is None:
            topology_spread_node_states = os.environ.get('ACSFIT_TOPOLOGY_SPREAD_NODE_STATES', '0') not in ('', '0')
        elif topology_spread_node_states and not self.topology_spread:
            raise ValueError("topology_spread_node_states=True needs topology_spread on")
        self.topology_spread_node_states = bool(topology_spread_node_states) and self.topology_spread
        self.other_nodes = []  # the listed nodes that are not agents (the master): domains of the spread constraints
        self.service_principal_app_id = service_principal_app_id
        self.service_principal_secret = service_principal_secret
        self.service_principal_tenant_id = service_principal_tenant_id
        self.subscription_id = subscription_id
        self.client_private_key = client_private_key
        self.ca_private_key = ca_private_key
        self._drained = {}
        self.resource_group = resource_group
        self.acs_deployment = acs_deployment
        self.agent_pools = {}
        self.pools_instance_type = {}
        self.instance_init_time = instance_init_time
        self.spare_agents = spare_agents
        self.idle_threshold = idle_threshold
        self.over_provision = over_provision
        self.scale_up = scale_up
        self.maintainance = maintainance
        self.notifier = notifier
        self.dry_run = dry_run
        self.deployments = Deployments()
        self.ignore_pools = ignore_pools

    # ---- adapter boundary: cloud + kube clients (reference cluster.py:65-109) -----------------------
    def login(self):
        pykube = _pykube()
        adapters.call("login", self.service_principal_app_id, self.service_principal_secret,
                      self.service_principal_tenant_id, self.subscription_id)
        self.arm_template = adapters.call("download_template", self.resource_group, self.acs_deployment)
        self.arm_parameters = adapters.call("download_parameters", self.resource_group, self.acs_deployment)
        self.fill_parameters_secure_strings()
        os.environ["PYKUBE_KUBERNETES_SERVICE_HOST"] = self.arm_parameters['firstConsecutiveStaticIP']['value']
        if self.kubeconfig:
            logger.debug('Using kubeconfig %s', self.kubeconfig)
            self.api = pykube.HTTPClient(pykube.KubeConfig.from_file(self.kubeconfig))
        else:
            logger.debug('Using kube service account')
            self.api = pykube.HTTPClient(pykube.KubeConfig.from_service_account())

    def fill_parameters_secure_strings(self):
        """downloaded parameters lack the SecureString ones; re-inject ours (cluster.py:91-109).  The
        certificate/key parameters only need to be syntactically present for an incremental
        deployment that does not touch the masters, so a placeholder is used for them."""
        params = self.arm_parameters
        params['clientPrivateKey'] = {'value': self.client_private_key}
        params['caPrivateKey'] = {'value': self.ca_private_key}
        params['servicePrincipalClientId'] = {'value': self.service_principal_app_id}
        params['servicePrincipalClientSecret'] = {'value': self.service_principal_secret}
        # never a real secret: a fixed, syntactically valid base64 blob (the reference sends an inert dummy
        # certificate in these slots, cluster.py:97-106); $ACSFIT_PLACEHOLDER_KEY overrides it
        placeholder = os.environ.get('ACSFIT_PLACEHOLDER_KEY', PLACEHOLDER_KEY)
        for key in ('kubeConfigPrivateKey', 'apiServerPrivateKey', 'etcdClientPrivateKey', 'etcdServerPrivateKey'):
            params[key] = {'value': placeholder}
        for i in range(5):
            key = "etcdPeerPrivateKey{}".format(i)
            if key in params:
                params[key] = {'value': placeholder}
        self.arm_template = adapters.call("delete_master_vm_extension", self.arm_template)

    def list_nodes(self):
        return _pykube().Node.objects(self.api)

    def list_pods(self):
        return _pykube().Pod.objects(self.api)  # all namespaces, see _pykube()

    # ---- the tick ---------------------------------------------------------------------------------------
    def loop(self, debug):
        """runs one loop of scaling to current needs; True when it went through."""
        logger.info("++++ Running Scaling Loop ++++++")
        if debug:
            logger.info('Debug mode is on')  # let errors crash the process
            return self.loop_logic()
        try:
            return self.loop_logic()
        except Exception as e:
            logger.error("Unexpected error: {}, {}".format(sys.exc_info()[0], e))
            return False

    scale_loop = loop  # the upstream (ec2 autoscaler) name of the same entry point

    def create_kube_node(self, node):
        kube_node = KubeNode(node)
        kube_node.capacity = capacity.get_capacity_for_instance_type(kube_node.instance_type)
        return kube_node

    def loop_logic(self):
        with utils.gc_paused():  # a tick builds 10^5 small objects at once: generational GC passes would double its time
            return self._loop_logic()

    def _loop_logic(self):
        pykube_nodes = self.list_nodes()
        if not pykube_nodes:
            logger.warning('Failed to list nodes. Please check kube configuration. Terminating scale loop.')
            return False
        listed = list(map(self.create_kube_node, pykube_nodes))
        all_nodes = [n for n in listed if utils.is_agent(n)]
        # with topology spread on, the scheduler counts the master among a constraint's domains
        self.other_nodes = [n for n in listed if not utils.is_agent(n)] if self.topology_spread else []

        scaler = EngineScaler(
            resource_group=self.resource_group, nodes=all_nodes, deployments=self.deployments,
            arm_template=self.arm_template, arm_parameters=self.arm_parameters, dry_run=self.dry_run,
            ignore_pools=self.ignore_pools, over_provision=self.over_provision, spare_count=self.spare_agents,
            idle_threshold=self.idle_threshold, notifier=self.notifier, node_selectors=self.node_selectors,
            selector_node_states=self.selector_node_states, node_taints=self.node_taints,
            pod_anti_affinity=self.pod_anti_affinity, node_affinity=self.node_affinity,
            anti_affinity_node_states=self.anti_affinity_node_states, pod_affinity=self.pod_affinity,
            pod_affinity_node_states=self.pod_affinity_node_states, topology_spread=self.topology_spread,
            topology_spread_node_states=self.topology_spread_node_states, other_nodes=self.other_nodes)

        pods = kube.make_pods(self.list_pods()) if KubePod is kube.KubePod else list(map(KubePod, self.list_pods()))
        running_or_pending_assigned_pods = [
            p for p in pods
            if p.status in (KubePodStatus.RUNNING, KubePodStatus.CONTAINER_CREATING)
            or (p.status == KubePodStatus.PENDING and p.node_name)]

        # occupancy: node.count_pod for every running pod on its node, in pod order (cluster.py:165-168)
        snapshot.count_running_pods(all_nodes, running_or_pending_assigned_pods)

        pods_to_schedule = self.get_pods_to_schedule(pods, scaler.agent_pools)
        logger.info("Pods to schedule: {}".format(len(pods_to_schedule)))

        if self.scale_up:
            logger.info("++++ Scaling Up Begins ++++++")
            self.scale(pods_to_schedule, all_nodes, scaler, running_pods=running_or_pending_assigned_pods)
            logger.info("++++ Scaling Up Ends ++++++")
        if self.maintainance:
            logger.info("++++ Maintenance Begins ++++++")
            self.maintain(pods_to_schedule, running_or_pending_assigned_pods, scaler)
            logger.info("++++ Maintenance Ends ++++++")
        return True

    def get_pending_pods(self, pods, nodes, running_pods=None):
        """sequential first fit of the pods over the nodes (cluster.py:184-204); placed pods are
        counted into node.used_capacity, the rest are returned in order.

        With topology spread on, `running_pods` also give each node's count and the non-agent nodes of the tick's listing
        (self.other_nodes) count as domains.  With pod anti-affinity on, `running_pods` are the pods already on the nodes (the tick's running or assigned
        pending pods, which scale() passes): their terms block pods, and pods' terms block them.  Without it, only the
        pods this call places count.  With pod affinity on they are also what a pod's affinity can find on a node, and
        the signatures the nodes hold afterwards are kept in self.affinity_present for the bin packing."""
        pods, nodes = list(pods), list(nodes)
        classes = None
        if self.node_selectors:
            classes = snapshot.selector_classes(pods, nodes, [], taints=self.node_taints, affinity=self.node_affinity)
        anti_affinity = None
        if self.pod_anti_affinity:
            anti_affinity = snapshot.anti_affinity(pods, nodes, running_pods or [])
        pod_affinity = None
        if self.pod_affinity:
            pod_affinity = snapshot.pod_affinity(pods, nodes, running_pods or [])
        topology_spread = None
        if self.topology_spread:
            topology_spread = snapshot.topology_spread(pods, nodes, running_pods or [], self.other_nodes)
        placed = snapshot.first_fit_nodes(pods, nodes, classes=classes, anti_affinity=anti_affinity,
                                          pod_affinity=pod_affinity, topology_spread=topology_spread)
        self.affinity_present = pod_affinity.present_signatures() if pod_affinity is not None else set()
        detail = len(pods) <= LOG_DETAIL_LIMIT
        pending_pods = []
        for i, pod in enumerate(pods):
            if placed[i] < 0:
                pending_pods.append(pod)
            elif detail:
                logger.info("{pod} fits on {node}".format(pod=pod, node=nodes[placed[i]]))
        if not detail:
            logger.info("%d pods fit on existing nodes", len(pods) - len(pending_pods))
        logger.info("Pending pods: {}".format(len(pending_pods)))
        if detail:
            for pod in pending_pods:
                logger.debug(pod.name)
        return pending_pods

    def scale(self, pods_to_schedule, nodes, scaler, running_pods=None):
        logger.info("Nodes: {}".format(len(nodes)))
        logger.info("To schedule: {}".format(len(pods_to_schedule)))
        pending_pods = self.get_pending_pods(pods_to_schedule, nodes, running_pods=running_pods)
        if len(pending_pods) > 0:
            if self.pod_affinity:
                scaler.fulfill_pending(pending_pods, affinity_present=self.affinity_present)
            else:
                scaler.fulfill_pending(pending_pods)

    def get_pods_to_schedule(self, pods, agent_pools):
        """pending, unassigned pods that fit an empty instance of at least one pool
        (cluster.py:217-240)."""
        pending_unassigned_pods = [p for p in pods if p.status == KubePodStatus.PENDING and (not p.node_name)]
        classes = None
        if self.node_selectors:
            classes = snapshot.selector_classes(pending_unassigned_pods, [], agent_pools, taints=self.node_taints,
                                                affinity=self.node_affinity)
        feasible = snapshot.feasible_pods(pending_unassigned_pods, agent_pools, classes=classes)
        unmatched = set()  # rejected only because no pool that would fit matches the node selector
        unaffine = set()  # some pool that would fit matches the selector, but none matches the required node affinity
        untolerated = set()  # some pool that would fit matches selector and affinity, but each has an untolerated taint
        if classes is not None and not classes.trivial:
            rejected = [p for p, ok, c in zip(pending_unassigned_pods, feasible, classes.pod_class) if not ok and c]
            if rejected:
                fits = snapshot.feasible_pods(rejected, agent_pools)
                unmatched = {id(p) for p, ok in zip(rejected, fits) if ok}
            if unmatched and (self.node_taints or self.node_affinity):
                fitting = [p for p in rejected if id(p) in unmatched]
                admitted = snapshot.feasible_pods(fitting, agent_pools,
                                                  classes=snapshot.selector_classes(fitting, [], agent_pools))
                selected = [p for p, a in zip(fitting, admitted) if a]
                if self.node_affinity and self.node_taints:
                    admitted = snapshot.feasible_pods(selected, agent_pools, classes=snapshot.selector_classes(
                        selected, [], agent_pools, affinity=True))
                    untolerated = {id(p) for p, a in zip(selected, admitted) if a}
                    unaffine = {id(p) for p in selected} - untolerated
                elif self.node_affinity:
                    unaffine = {id(p) for p in selected}
                else:
                    untolerated = {id(p) for p in selected}
        pods_to_schedule = []
        warn = logger.isEnabledFor(logging.WARNING)  # (the message is formatted eagerly, as upstream: skip it when nobody listens)
        for pod, ok in zip(pending_unassigned_pods, feasible):
            if ok:
                pods_to_schedule.append(pod)
            elif warn and id(pod) in untolerated:
                logger.warning("Pending pod %s cannot fit: every agent pool that would fit it and matches its node "
                               "selector has a taint it does not tolerate. Scheduling skipped." % pod.name)
            elif warn and id(pod) in unaffine:
                logger.warning("Pending pod %s cannot fit: no agent pool that would fit it matches its required node "
                               "affinity. Scheduling skipped." % pod.name)
            elif warn and id(pod) in unmatched:
                logger.warning("Pending pod %s cannot fit: no agent pool matches its node selector %s. "
                               "Scheduling skipped." % (pod.name, pod.selectors))
            elif warn:
                logger.warning("Pending pod %s cannot fit. "
                            "Please check that requested resource amount is "
                            "consistent with node size."
                            "Scheduling skipped." % (pod.name))
        return pods_to_schedule

    def maintain(self, pods_to_schedule, running_or_pending_assigned_pods, scaler):
        scaler.maintain(pods_to_schedule, running_or_pending_assigned_pods)
