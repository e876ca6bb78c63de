"""Pod / node / resource-vector types of the tick (mirror of reference autoscaler/kube.py).

Same names, fields and error behaviour as the reference so that callers and tests read the
same.  The bulk arithmetic of a tick never goes through these Python objects: Cluster / Scaler
flatten them into dense float64 buffers (snapshot.py) and run the CUDA kernels.  The mutators
(cordon / uncordon / drain / delete) are the downward adapter boundary: they call straight
through to the wrapped pykube objects, exactly as the reference does (kube.py:124-167).
"""
import datetime
import json
import logging
import os
import re
from collections.abc import Mapping

from . import utils

logger = logging.getLogger('autoscaler.kube')

try:  # CPython twin of the two hottest host loops (csrc/hostfast.c); the Python code below is the definition
    if os.environ.get('ACSFIT_NO_HOSTFAST'):
        raise ImportError('disabled')
    from . import _hostfast
except ImportError:
    _hostfast = None

_CORDON_LABEL = 'openai/cordoned-by-autoscaler'

# taint effects that keep a pod which does not tolerate them off a node (PreferNoSchedule is only a preference)
BLOCKING_EFFECTS = ('NoSchedule', 'NoExecute')
# node-lifecycle taints (unschedulable, not-ready, unreachable, uninitialized) are not honoured: cordoning is modelled
# by spec.unschedulable, and a node booting from this autoscaler's own scale-up carries not-ready / uninitialized for
# a while -- honouring those would make the next tick scale up again for the same pods
LIFECYCLE_TAINT_PREFIXES = ('node.kubernetes.io/', 'node.alpha.kubernetes.io/', 'node.cloudprovider.kubernetes.io/')


def _field(entry, key):
    value = entry.get(key)
    return '' if value is None else value


def _entries(value, what, owner):
    """spec.taints / spec.tolerations as a list of mappings ([] when absent); ValueError naming the owner otherwise"""
    if value is None:
        return []
    if not isinstance(value, list) or not all(type(e) is dict or isinstance(e, Mapping) for e in value):
        raise ValueError("malformed %s of %s: expected a list of mappings, got %r" % (what, owner, value))
    return value


def blocking_taints(taints):
    """frozenset of (key, value, effect) of the taints that block scheduling: effect NoSchedule or NoExecute, and not
    a node-lifecycle taint (LIFECYCLE_TAINT_PREFIXES)"""
    out = set()
    for t in taints:
        key, effect = _field(t, 'key'), _field(t, 'effect')
        if effect in BLOCKING_EFFECTS and not key.startswith(LIFECYCLE_TAINT_PREFIXES):
            out.add((key, _field(t, 'value'), effect))
    return frozenset(out)


def tolerates(tolerations, taint):
    """some toleration tolerates the taint (Kubernetes' Toleration.ToleratesTaint): a non-empty effect must equal the
    taint's, a non-empty key must equal the taint's (an empty key matches every key); operator Exists matches any value,
    Equal or an empty operator needs equal values (a missing value reads as ''), any other operator tolerates nothing.
    tolerationSeconds is ignored.  `taint` is a mapping or a (key, value, effect) tuple."""
    if not isinstance(taint, Mapping):
        taint = dict(zip(('key', 'value', 'effect'), taint))
    key, value, effect = _field(taint, 'key'), _field(taint, 'value'), _field(taint, 'effect')
    for t in tolerations:
        if _field(t, 'effect') and _field(t, 'effect') != effect:
            continue
        if _field(t, 'key') and _field(t, 'key') != key:
            continue
        op = _field(t, 'operator')
        if op == 'Exists' or (op in ('', 'Equal') and _field(t, 'value') == value):
            return True
    return False


def tolerates_all(tolerations, taints):
    """the pod with these tolerations may be scheduled past every one of `taints` (blocking_taints tuples)"""
    return all(tolerates(tolerations, t) for t in taints)


# required pod anti-affinity: only terms with this topology key are honoured (one node = one topology domain)
HOSTNAME_TOPOLOGY_KEY = 'kubernetes.io/hostname'
SELECTOR_OPERATORS = ('In', 'NotIn', 'Exists', 'DoesNotExist')


def _str_list(value, what, owner):
    if not isinstance(value, list) or not all(isinstance(v, str) for v in value):
        raise ValueError("malformed %s of %s: expected a list of strings, got %r" % (what, owner, value))
    return value


def _mapping(value, what, owner):
    if not isinstance(value, Mapping):
        raise ValueError("malformed %s of %s: expected a mapping, got %r" % (what, owner, value))
    return value


def label_selector(selector, owner, what='labelSelector'):
    """the canonical, hashable form of a metav1.LabelSelector: (sorted matchLabels items, sorted (key, operator, sorted
    values) requirements).  Two selectors with equal forms select the same pods.  ValueError naming the owner when the
    selector is malformed (unknown operator, values with Exists / DoesNotExist, no values with In / NotIn)."""
    _mapping(selector, what, owner)
    labels = selector.get('matchLabels') or {}
    _mapping(labels, what + '.matchLabels', owner)
    if not all(isinstance(k, str) and isinstance(v, str) for k, v in labels.items()):
        raise ValueError("malformed %s.matchLabels of %s: %r" % (what, owner, labels))
    reqs = []
    for e in _entries(selector.get('matchExpressions'), what + '.matchExpressions', owner):
        key, op = e.get('key'), e.get('operator')
        values = e.get('values')
        values = [] if values is None else _str_list(values, what + '.matchExpressions.values', owner)
        if not isinstance(key, str) or op not in SELECTOR_OPERATORS or \
                (op in ('In', 'NotIn')) != bool(values):
            raise ValueError("malformed %s.matchExpressions entry of %s: %r" % (what, owner, e))
        reqs.append((key, op, tuple(sorted(set(values)))))
    return tuple(sorted(labels.items())), tuple(sorted(set(reqs)))


def selector_matches(selector, labels):
    """the canonical selector (label_selector) selects a pod with these labels (an empty selector selects every pod;
    NotIn and DoesNotExist hold when the key is absent)"""
    items, reqs = selector
    for key, value in items:
        if labels.get(key) != value:
            return False
    for key, op, values in reqs:
        have = labels.get(key)
        if op == 'In':
            ok = have is not None and have in values
        elif op == 'NotIn':
            ok = have is None or have not in values
        elif op == 'Exists':
            ok = have is not None
        else:
            ok = have is None
        if not ok:
            return False
    return True


def _required_pod_terms(affinity, field, namespace, owner):
    """the required terms of spec.affinity.<field> (podAffinity or podAntiAffinity) with topologyKey
    kubernetes.io/hostname and no namespaceSelector, as (namespaces, selector) pairs: frozenset of namespaces (empty
    `namespaces` = the carrying pod's own), canonical label_selector or None for an absent or null labelSelector.
    ValueError naming the owner when a field is malformed."""
    if affinity is None:
        return []
    _mapping(affinity, 'spec.affinity', owner)
    block = affinity.get(field)
    if block is None:
        return []
    _mapping(block, 'spec.affinity.' + field, owner)
    what = 'spec.affinity.%s.requiredDuringSchedulingIgnoredDuringExecution' % field
    terms = []
    for t in _entries(block.get('requiredDuringSchedulingIgnoredDuringExecution'), what, owner):
        topology = t.get('topologyKey')
        if not isinstance(topology, str):
            raise ValueError("malformed %s entry of %s: topologyKey %r" % (what, owner, topology))
        namespaces = t.get('namespaces')
        namespaces = [] if namespaces is None else _str_list(namespaces, what + '.namespaces', owner)
        selector = t.get('labelSelector')
        selector = None if selector is None else label_selector(selector, owner, what + '.labelSelector')
        if topology != HOSTNAME_TOPOLOGY_KEY or t.get('namespaceSelector') is not None:
            continue
        terms.append((frozenset(namespaces) if namespaces else frozenset((namespace,)), selector))
    return terms


def anti_affinity_terms(affinity, namespace, owner):
    """the required pod anti-affinity terms of spec.affinity that this project honours, as (namespaces, selector)
    pairs: frozenset of namespaces (empty `namespaces` = the carrying pod's own), canonical label_selector.  Only terms
    with topologyKey kubernetes.io/hostname count; a term with an absent or null labelSelector selects no pod and a
    term with a namespaceSelector is not honoured, so both are left out.  ValueError naming the owner when a field
    is malformed."""
    terms = _required_pod_terms(affinity, 'podAntiAffinity', namespace, owner)
    return tuple(dict.fromkeys(t for t in terms if t[1] is not None))


def affinity_terms(affinity, namespace, owner):
    """the required pod affinity terms of spec.affinity that this project honours, as anti_affinity_terms gives them,
    except that a term with an absent or null labelSelector is kept with selector None: it selects no pod, so the pod
    can land nowhere, as in Kubernetes (dropping it would make the pod look placeable).  Terms with another topology
    key or a namespaceSelector are left out; that never makes a pod harder to place than Kubernetes would."""
    return tuple(dict.fromkeys(_required_pod_terms(affinity, 'podAffinity', namespace, owner)))


def affinity_term_selects(term, namespace, labels):
    """the pod affinity term (namespaces, selector or None) selects a pod with this namespace and these labels"""
    namespaces, selector = term
    return selector is not None and namespace in namespaces and selector_matches(selector, labels)


# topology spread: the values Kubernetes validation accepts
WHEN_UNSATISFIABLE = ('DoNotSchedule', 'ScheduleAnyway')
NODE_INCLUSION_POLICIES = ('Honor', 'Ignore')


class SpreadConstraint(tuple):
    """the honoured topology spread constraint of a pod: (max_skew, selector, min_domains, honor_affinity,
    honor_taints).  `selector` is the canonical label_selector with the matchLabelKeys requirements added, or None
    (a null labelSelector selects no pod); min_domains defaults to 1; honor_affinity / honor_taints are the
    nodeAffinityPolicy (default Honor) and nodeTaintsPolicy (default Ignore) as booleans."""
    __slots__ = ()

    max_skew = property(lambda self: self[0])
    selector = property(lambda self: self[1])
    min_domains = property(lambda self: self[2])
    honor_affinity = property(lambda self: self[3])
    honor_taints = property(lambda self: self[4])


def _selector_keys(selector):
    """the label keys a raw labelSelector names (matchLabels and matchExpressions)"""
    keys = set((selector.get('matchLabels') or {}).keys())
    keys.update(e.get('key') for e in selector.get('matchExpressions') or ())
    return keys


def topology_spread_constraint(constraints, labels, owner):
    """the constraint of spec.topologySpreadConstraints that this project honours, as a SpreadConstraint, or None:
    the one with topologyKey kubernetes.io/hostname and whenUnsatisfiable DoNotSchedule (validation allows one).
    Every entry is validated as Kubernetes validates it, and ValueError names the owner when one is malformed:
    maxSkew an integer >= 1, whenUnsatisfiable one of WHEN_UNSATISFIABLE, a non-empty topologyKey, no duplicate
    (topologyKey, whenUnsatisfiable), minDomains >= 1 and only with DoNotSchedule, matchLabelKeys neither without a
    labelSelector nor naming a key the labelSelector names, each policy one of NODE_INCLUSION_POLICIES.  A key of
    matchLabelKeys adds `key In [the pod's value]` to the selector; a key the pod lacks (in `labels`) adds nothing."""
    what = 'spec.topologySpreadConstraints'
    honoured, seen = None, set()
    for c in _entries(constraints, what, owner):
        skew, when, topology = c.get('maxSkew'), c.get('whenUnsatisfiable'), c.get('topologyKey')
        if type(skew) is not int or skew < 1:
            raise ValueError("malformed %s entry of %s: maxSkew %r (an integer >= 1)" % (what, owner, skew))
        if when not in WHEN_UNSATISFIABLE:
            raise ValueError("malformed %s entry of %s: whenUnsatisfiable %r" % (what, owner, when))
        if not isinstance(topology, str) or not topology:
            raise ValueError("malformed %s entry of %s: topologyKey %r" % (what, owner, topology))
        if (topology, when) in seen:
            raise ValueError("malformed %s of %s: duplicate (topologyKey, whenUnsatisfiable) %r"
                             % (what, owner, (topology, when)))
        seen.add((topology, when))
        min_domains = c.get('minDomains')
        if min_domains is not None and (type(min_domains) is not int or min_domains < 1 or when != 'DoNotSchedule'):
            raise ValueError("malformed %s entry of %s: minDomains %r (an integer >= 1, with DoNotSchedule only)"
                             % (what, owner, min_domains))
        policies = []
        for field, default in (('nodeAffinityPolicy', 'Honor'), ('nodeTaintsPolicy', 'Ignore')):
            value = c.get(field)
            if value is not None and value not in NODE_INCLUSION_POLICIES:
                raise ValueError("malformed %s entry of %s: %s %r" % (what, owner, field, value))
            policies.append((default if value is None else value) == 'Honor')
        raw = c.get('labelSelector')
        selector = None if raw is None else label_selector(raw, owner, what + '.labelSelector')
        keys = _str_list(c.get('matchLabelKeys') or [], what + '.matchLabelKeys', owner)
        if keys and (raw is None or set(keys) & _selector_keys(raw)):
            raise ValueError("malformed %s entry of %s: matchLabelKeys %r without a labelSelector or naming one of "
                             "its keys" % (what, owner, keys))
        if topology != HOSTNAME_TOPOLOGY_KEY or when != 'DoNotSchedule':
            continue
        if selector is not None and keys:
            extra = [(k, 'In', (labels[k],)) for k in keys if k in labels]
            selector = (selector[0], tuple(sorted(set(selector[1] + tuple(extra)))))
        honoured = SpreadConstraint((skew, selector, 1 if min_domains is None else min_domains, *policies))
    return honoured


# required node affinity: the operators of a NodeSelectorRequirement, and the one field a matchFields entry may name
NODE_SELECTOR_OPERATORS = ('In', 'NotIn', 'Exists', 'DoesNotExist', 'Gt', 'Lt')
NODE_NAME_FIELD = 'metadata.name'
_INT64 = re.compile(r'[+-]?[0-9]+')


def parse_int64(text):
    """Go's strconv.ParseInt(text, 10, 64): an optional sign, then ASCII digits, within int64; None otherwise (no
    spaces or underscores, unlike int())"""
    if type(text) is not str or not _INT64.fullmatch(text):
        return None
    value = int(text)
    return value if -(1 << 63) <= value < (1 << 63) else None


def _node_requirements(entries, what, owner, fields):
    reqs = []
    for e in _entries(entries, what, owner):
        key, op = e.get('key'), e.get('operator')
        values = e.get('values')
        values = [] if values is None else _str_list(values, what + '.values', owner)
        if fields:
            ok = key == NODE_NAME_FIELD and op in ('In', 'NotIn') and len(values) == 1
        elif op in ('In', 'NotIn'):
            ok = bool(values)
        elif op in ('Gt', 'Lt'):
            ok = len(values) == 1 and parse_int64(values[0]) is not None
            values = [parse_int64(values[0])] if ok else values
        else:
            ok = op in ('Exists', 'DoesNotExist') and not values
        if not isinstance(key, str) or not ok:
            raise ValueError("malformed %s entry of %s: %r" % (what, owner, e))
        reqs.append((key, op, tuple(sorted(set(values)))))
    return tuple(sorted(set(reqs)))


def node_affinity_terms(affinity, owner):
    """the canonical, hashable form of spec.affinity.nodeAffinity.requiredDuringSchedulingIgnoredDuringExecution: None
    when there is no constraint (no affinity, no nodeAffinity, or a null required part; the preferred part is a scoring
    preference and is ignored), else a sorted tuple of the nodeSelectorTerms that can match, each (sorted matchExpressions
    requirements, sorted matchFields requirements) with a requirement (key, operator, sorted values); Gt / Lt values
    are parsed to int.  The terms are ORed and a term with neither list matches nothing, so it is dropped: () selects no
    node.  Equal forms select the same nodes.  ValueError naming the owner when a field is malformed, as Kubernetes'
    validation refuses it (empty or non-list nodeSelectorTerms, an unknown operator, a wrong number of values, a Gt /
    Lt value that is not an integer, a matchFields key other than metadata.name)."""
    if affinity is None:
        return None
    _mapping(affinity, 'spec.affinity', owner)
    node = affinity.get('nodeAffinity')
    if node is None:
        return None
    _mapping(node, 'spec.affinity.nodeAffinity', owner)
    required = node.get('requiredDuringSchedulingIgnoredDuringExecution')
    if required is None:
        return None
    what = 'spec.affinity.nodeAffinity.requiredDuringSchedulingIgnoredDuringExecution'
    _mapping(required, what, owner)
    what += '.nodeSelectorTerms'
    raw = required.get('nodeSelectorTerms')
    if not isinstance(raw, list) or not raw:
        raise ValueError("malformed %s of %s: expected a non-empty list, got %r" % (what, owner, raw))
    terms = set()
    for t in _entries(raw, what, owner):
        term = (_node_requirements(t.get('matchExpressions'), what + '.matchExpressions', owner, False),
                _node_requirements(t.get('matchFields'), what + '.matchFields', owner, True))
        if term != ((), ()):
            terms.add(term)
    return tuple(sorted(terms))


class _NewNode(object):
    """the name (and hostname label) of a node a pool has not created yet: always set, equal to no current node's"""

    def __repr__(self):
        return '<new node>'


NEW_NODE = _NewNode()


def requirement_holds(op, values, have):
    """one NodeSelectorRequirement against a label value or node name `have` (None when the label is absent)"""
    if op == 'In':
        return have is not None and have in values
    if op == 'NotIn':
        return have is None or have not in values
    if op == 'Exists':
        return have is not None
    if op == 'DoesNotExist':
        return have is None
    number = parse_int64(have)  # a missing or non-integer label (and a new node's name) makes Gt / Lt false
    return number is not None and (number > values[0] if op == 'Gt' else number < values[0])


def node_affinity_matches(terms, labels, name):
    """the canonical required node affinity (node_affinity_terms) admits a node with these labels and this name: no
    constraint (None), or some term all of whose requirements hold"""
    if terms is None:
        return True
    return any(all(requirement_holds(op, values, labels.get(key)) for key, op, values in exprs) and
               all(requirement_holds(op, values, name) for _, op, values in fields) for exprs, fields in terms)


def pool_affinity_matches(terms, labels):
    """node_affinity_matches for a new node of a pool with these labels (AgentPool.labels): its name and its
    kubernetes.io/hostname label are set, to a value no current node has (NEW_NODE), so Exists and NotIn hold there and
    In, DoesNotExist, Gt and Lt do not.  A pod pinned to existing nodes matches no pool."""
    return node_affinity_matches(terms, {**labels, HOSTNAME_TOPOLOGY_KEY: NEW_NODE}, NEW_NODE)


class KubePodStatus(object):
    RUNNING = 'Running'
    PENDING = 'Pending'
    CONTAINER_CREATING = 'ContainerCreating'
    SUCCEEDED = 'Succeeded'
    FAILED = 'Failed'


class KubeResource(object):
    """sparse resource vector: dict key -> float64, absent key == 0 (kube.py:197-249)."""

    def __init__(self, **kwargs):
        self.raw = {key: utils.parse_resource(value) for key, value in kwargs.items()}

    def _zip(self, other, op):
        merged = {}
        for key in set(self.raw) | set(other.raw):
            merged[key] = op(self.raw.get(key, 0), other.raw.get(key, 0))
        return KubeResource(**merged)

    def __add__(self, other):
        return self._zip(other, lambda a, b: a + b)

    def __sub__(self, other):
        return self._zip(other, lambda a, b: a - b)

    def __mul__(self, multiplier):
        return KubeResource(**{key: value * multiplier for key, value in self.raw.items()})

    __rmul__ = __mul__

    def get(self, key, default=None):
        return self.raw.get(key, default)

    @property
    def possible(self):
        return all(value >= 0 for value in self.raw.values())

    def __str__(self):
        return str(self.raw)


_RESOURCES_MEMO = {}
_CREATED_BY_MEMO = {}
_TIME_MEMO = {}
_AFFINITY_MEMO = {}
_MISSING = object()


def _remember_time(text):
    value = utils.parse_time(text)  # raises like the reference for a malformed timestamp (not cached)
    if type(text) is str:
        if len(_TIME_MEMO) > (1 << 16):
            _TIME_MEMO.clear()
        _TIME_MEMO[text] = value
    return value


def _pod_resources(containers):
    """KubePod.resources (kube.py:41-49): pods:1 + the per-key sum over the containers' requests, accumulated as
    0.0 + v1 + v2 ... in container order (the order fixes the float64 result).  A cluster's pods come from a few
    templates, so the result is memoised on the literal request texts; pods with the same requests then SHARE one
    KubeResource (they are values: nothing in this package mutates one in place), which also lets the snapshot
    flattening convert each distinct vector once (snapshot.Dims).  Failures are not cached: they raise again."""
    try:
        if len(containers) == 1:  # the common case, without building a generator
            r = containers[0].get('resources')
            q = r.get('requests') if r else None
            key = tuple(q.items()) if q else ()
        else:
            key = []
            for c in containers:
                r = c.get('resources')
                q = r.get('requests') if r else None
                key.append(tuple(q.items()) if q else ())
            key = (len(containers), tuple(key))
        hit = _RESOURCES_MEMO.get(key)
    except TypeError:  # unhashable quantity objects: the plain route
        key, hit = None, None
    if hit is not None:
        return hit
    totals = {}
    for container in containers:
        for name, quantity in container.get('resources', {}).get('requests', {}).items():
            totals[name] = totals.get(name, 0.0) + utils.parse_SI(quantity)
    res = KubeResource(pods=1, **totals)
    if key is not None:
        if len(_RESOURCES_MEMO) > (1 << 16):
            _RESOURCES_MEMO.clear()
        _RESOURCES_MEMO[key] = res
    return res


class KubePod(object):
    _DRAIN_GRACE_PERIOD = datetime.timedelta(seconds=60 * 60)

    def __init__(self, pod):
        self.original = pod
        obj = pod.obj
        meta, spec, status = obj['metadata'], obj['spec'], obj['status']
        self.name = meta['name']
        self.namespace = meta['namespace']
        self.node_name = spec.get('nodeName')
        self.status = status['phase']
        self.uid = meta['uid']
        self.selectors = spec.get('nodeSelector', {})
        self.labels = labels = meta.get('labels', {})
        self.annotations = meta.get('annotations', {})
        self.owner = labels.get('owner', None)
        # (timestamps: memoised per text, utils.parse_time; the memo is consulted directly on this hot path)
        text = meta['creationTimestamp']
        cached = _TIME_MEMO.get(text) if type(text) is str else None
        self.creation_time = cached if cached is not None else _remember_time(text)
        text = status.get('startTime', _MISSING)
        if text is _MISSING:
            self.start_time = None
        else:
            cached = _TIME_MEMO.get(text) if type(text) is str else None
            self.start_time = cached if cached is not None else _remember_time(text)
        self.resources = _pod_resources(spec['containers'])

    def _created_by(self):
        """the created-by annotation, decoded (kube.py:51-58 decode it on every call).  The decoded value is a pure
        function of the text and only ever read, so it is memoised per distinct text (the pods of one controller
        share theirs); a malformed annotation is not cached and raises on every call, as upstream."""
        text = self.annotations.get('kubernetes.io/created-by', '{}')
        try:
            return _CREATED_BY_MEMO[text]
        except (KeyError, TypeError):
            pass
        decoded = json.loads(text)
        if type(text) is str:
            if len(_CREATED_BY_MEMO) > (1 << 16):
                _CREATED_BY_MEMO.clear()
            _CREATED_BY_MEMO[text] = decoded
        return decoded

    @property
    def tolerations(self):
        """spec.tolerations ([] when absent); read on use, so pods built attribute by attribute (make_pods) have it too.
        ValueError when it is not a list of mappings."""
        return _entries(self.original.obj['spec'].get('tolerations'), 'spec.tolerations', 'pod %s' % self)

    @property
    def anti_affinity_terms(self):
        """the honoured required pod anti-affinity terms (kube.anti_affinity_terms); read on use, like tolerations."""
        return anti_affinity_terms(self.original.obj['spec'].get('affinity'), self.namespace, 'pod %s' % self)

    @property
    def affinity_terms(self):
        """the honoured required pod affinity terms (kube.affinity_terms); read on use, like tolerations."""
        return affinity_terms(self.original.obj['spec'].get('affinity'), self.namespace, 'pod %s' % self)

    @property
    def topology_spread(self):
        """the honoured hostname topology spread constraint (kube.topology_spread_constraint; None when there is none);
        read on use, like tolerations."""
        return topology_spread_constraint(self.original.obj['spec'].get('topologySpreadConstraints'), self.labels,
                                          'pod %s' % self)

    @property
    def node_affinity(self):
        """the required node affinity (kube.node_affinity_terms; None when there is none); read on use, like
        tolerations.  The pods of one controller carry the same affinity, so the parsed form is memoised on the text of
        the field (JSON values: equal texts are equal fields); a malformed field is not cached and raises on every read."""
        affinity = self.original.obj['spec'].get('affinity')
        if affinity is None:
            return None
        key = repr(affinity)
        terms = _AFFINITY_MEMO.get(key, _MISSING)
        if terms is _MISSING:
            terms = node_affinity_terms(affinity, 'pod %s' % self)
            if len(_AFFINITY_MEMO) > (1 << 16):
                _AFFINITY_MEMO.clear()
            _AFFINITY_MEMO[key] = terms
        return terms

    def is_mirrored(self):
        daemonset = self._created_by().get('reference', {}).get('kind') == 'DaemonSet'
        return daemonset or self.annotations.get('kubernetes.io/config.mirror')

    def is_replicated(self):
        return self._created_by()

    def is_critical(self):
        return utils.parse_bool_label(self.labels.get('openai/do-not-drain'))

    def is_in_drain_grace_period(self):
        """pods younger than an hour (or not started) are not drained (kube.py:63-68)."""
        if not self.start_time:
            return True
        return (utils.now(self.start_time.tzinfo) - self.start_time) < self._DRAIN_GRACE_PERIOD

    def is_drainable(self):
        return self.is_replicated() and not self.is_critical() and not self.is_in_drain_grace_period()

    def delete(self):
        logger.info('Deleting Pod %s/%s', self.namespace, self.name)
        return self.original.delete()

    def __hash__(self):
        return hash(self.uid)

    def __eq__(self, other):
        return self.uid == other.uid

    def __str__(self):
        return 'KubePod({namespace}, {name})'.format(namespace=self.namespace, name=self.name)

    __repr__ = __str__


_KUBEPOD_INIT = KubePod.__init__


def make_pods(raw_pods):
    """[KubePod(p) for p in raw_pods] (cluster.py:153 builds them with map).  With the C helper the plain pods (exact
    dicts, memoised timestamps and requests) are built in C attribute for attribute; everything else - and every
    pod when the helper is absent or KubePod.__init__ has been replaced - goes through the constructor."""
    if _hostfast is None or KubePod.__init__ is not _KUBEPOD_INIT:
        return list(map(KubePod, raw_pods))
    return _hostfast.make_pods(KubePod, raw_pods, _TIME_MEMO, _remember_time, _RESOURCES_MEMO, _pod_resources)


class KubeNode(object):
    def __init__(self, node):
        self.original = node
        self.pykube_node = node
        meta = node.obj['metadata']
        self.name = meta['name']
        self.index = int(self.name.split('-')[3])
        self.region, self.instance_type = self._get_instance_data()
        self.selectors = meta['labels']
        self.capacity = None  # set by Cluster.create_kube_node from the capacity table
        self.used_capacity = KubeResource()
        self.unschedulable = node.obj['spec'].get('unschedulable', False)
        self.creation_time = utils.parse_time(meta['creationTimestamp'])
        self.instance_index = utils.get_instance_index(node)

    @property
    def taints(self):
        """spec.taints as listed ([] when absent); read on use.  ValueError when it is not a list of mappings."""
        return _entries(self.original.obj['spec'].get('taints'), 'spec.taints', 'node %s' % self)

    def _get_instance_data(self):
        labels = self.original.obj['metadata']['labels']
        instance_type = labels.get('beta.kubernetes.io/instance-type')
        region = labels.get('failure-domain.beta.kubernetes.io/region')
        if instance_type and region:
            return (region, instance_type)
        return ('', None)

    # ---- adapter boundary: straight through to pykube (kube.py:124-167) -------------------------
    def drain(self, pods, notifier=None):
        for pod in pods:
            if pod.is_drainable():
                pod.delete()
        logger.info("drained %s", self)
        if notifier:
            notifier.notify_drained_node(self, pods)

    def _http_error(self):
        try:
            import pykube.exceptions
            return pykube.exceptions.HTTPError
        except ImportError:  # adapter not installed: nothing to catch
            return ()

    def uncordon(self):
        if not utils.parse_bool_label(self.selectors.get(_CORDON_LABEL)):
            logger.debug('uncordon %s ignored', self)
            return False
        try:
            self.original.reload()
            self.original.obj['spec']['unschedulable'] = False
            self.original.update()
            logger.info("uncordoned %s", self)
            return True
        except self._http_error() as ex:
            logger.info("uncordon failed %s %s", self, ex)
            return False

    def cordon(self):
        try:
            self.original.reload()
            self.original.obj['spec']['unschedulable'] = True
            self.original.obj['metadata']['labels'][_CORDON_LABEL] = 'true'
            self.original.update()
            logger.info("cordoned %s", self)
            return True
        except self._http_error() as ex:
            logger.info("cordon failed %s %s", self, ex)
            return False

    def delete(self):
        try:
            self.original.delete()
            logger.info("deleted %s", self)
            return True
        except self._http_error() as ex:
            logger.info("delete failed %s %s", self, ex)
            return False

    # ---- single-item forms of the hot-path arithmetic --------------------------------------------
    def count_pod(self, pod):
        assert isinstance(pod, KubePod)
        self.used_capacity += pod.resources

    def can_fit(self, resources):
        """capacity - (used + resources) possible (kube.py:173-176), evaluated on the GPU like the
        batched path (one pod x one node); Cluster.get_pending_pods never calls this per pair."""
        assert isinstance(resources, KubeResource)
        from . import snapshot
        return snapshot.single_can_fit(self, resources)

    def is_match(self, pod):
        return all(self.selectors.get(label) == value for label, value in pod.selectors.items())

    def __hash__(self):
        return hash(self.name)

    def __eq__(self, other):
        return self.name == other.name

    def __str__(self):
        return "{}".format(self.name)
