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
from .scaler import LOG_DETAIL_LIMIT, RULE_SWITCHES

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
        switches = locals()  # the rule switches as given, by name
        self.kubeconfig = kubeconfig
        # each rule switch: None reads its environment variable, and it is on only while its prerequisite is on
        for name, env, needs in RULE_SWITCHES:
            value = switches[name]
            if value is None:
                value = os.environ.get(env, '0') not in ('', '0')
            elif value and needs and not getattr(self, needs):
                raise ValueError("%s=True needs %s on" % (name, needs))
            setattr(self, name, bool(value) and (needs is None or getattr(self, needs)))
        self.affinity_present = set()  # signatures the last node pass left on some node (scale() hands them on)
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
            idle_threshold=self.idle_threshold, notifier=self.notifier, other_nodes=self.other_nodes,
            **{name: getattr(self, name) for name, _, _ in RULE_SWITCHES})

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
