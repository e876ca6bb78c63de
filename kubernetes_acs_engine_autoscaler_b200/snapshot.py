"""Snapshot flattening: kube objects <-> dense float64 device buffers (host logic, no arithmetic).

One tick's cluster state is turned into contiguous arrays once, shipped to HBM, and the
decisions come back as index vectors that are mapped onto the original KubePod / KubeNode
objects, including `node.used_capacity`, so downstream Python sees the state the reference
would have produced (SURVEY.md section 3.2 "device boundary").

Layout: resource dims = sorted union of keys over every vector involved; a missing key is 0.0
(bit-exact with KubeResource's own missing-key rule, kube.py:204-206,:210-212); the column count
is padded with zero columns to 2/4/8/16 for the first-fit kernels.
"""
import itertools

import numpy as np
import torch

from . import kube
from .engine import Engine, padded_dims
from .kube import _hostfast

_engine = None


def get_engine():
    """the process-wide CUDA engine; raises when libacsfit.so or a GPU is missing (no fallback)."""
    global _engine
    if _engine is None:
        _engine = Engine()
    return _engine


def set_engine(engine):
    """install a specific engine (e.g. one bound to this rank's GPU)."""
    global _engine
    _engine = engine
    return engine


def _group(objects):
    """(group index per object, one representative per group): identity grouping in first-occurrence order."""
    objects = objects if isinstance(objects, list) else list(objects)
    inv = np.empty(len(objects), dtype=np.int64)
    if _hostfast is not None:
        return inv, _hostfast.group_ids(objects, inv)
    slot, uniq = {}, []
    for i, obj in enumerate(objects):
        j = slot.get(id(obj))
        if j is None:
            j = slot[id(obj)] = len(uniq)
            uniq.append(obj)
        inv[i] = j
    return inv, uniq


class Dims(object):
    """column order of one flattening.  Resource vectors are deduplicated by object identity first: pods of one
    template share their KubeResource (kube._pod_resources), so 10^5 pods flatten as a few dozen distinct rows
    plus one fancy-index, not as 10^5 Python dict walks."""

    def __init__(self, resources):
        keys = set()
        for res in _group(resources)[1]:
            keys.update(res.raw.keys())
        self.keys = sorted(keys)
        self.index = {k: i for i, k in enumerate(self.keys)}
        self.D = max(1, len(self.keys))
        self.Dp = padded_dims(self.D)

    def rows(self, resources, n=None, groups=False):
        """[len(resources), Dp] float64 rows; with groups=True also (group index per row, the distinct vectors)."""
        resources = list(resources)
        index = self.index
        inv, uniq = _group(resources)
        urows = np.zeros((len(uniq), self.Dp), dtype=np.float64)
        for j, res in enumerate(uniq):
            for key, value in res.raw.items():
                urows[j, index[key]] = value
        out = np.zeros((len(resources) if n is None else n, self.Dp), dtype=np.float64)
        if len(resources):
            out[:len(resources)] = urows[inv]
        return (out, inv, uniq) if groups else out


def _touched_keys(node_of, inv, uniq):
    """{node: union of the key sets of the vectors counted on it}: one set update per distinct (node, vector) pair
    instead of one per pod (the pods of a template share their vector)."""
    touched = {}
    if not len(node_of):
        return touched
    G = max(1, len(uniq))
    pairs = np.unique(np.asarray(node_of, dtype=np.int64) * G + np.asarray(inv, dtype=np.int64))
    keysets = [set(u.raw) for u in uniq]
    for pair in pairs.tolist():
        n, g = divmod(pair, G)
        have = touched.get(n)
        if have is None:
            touched[n] = set(keysets[g])
        else:
            have.update(keysets[g])
    return touched


def _check_finite(a, what):
    if not np.isfinite(a).all():
        raise ValueError("non-finite %s is outside the supported domain" % what)


def _nonfinite_rows(req):
    return ~np.isfinite(req).all(axis=1)


def _node_types(nodes, dims):
    """(cap_type[K, Dp], node_type[N]) -- one capacity row per distinct KubeResource object/type."""
    rows, index, node_type = [], {}, np.zeros(len(nodes), dtype=np.int32)
    for i, node in enumerate(nodes):
        key = id(node.capacity)
        if key not in index:
            index[key] = len(rows)
            rows.append(node.capacity)
        node_type[i] = index[key]
    cap = dims.rows(rows)
    _check_finite(cap, "node capacity")
    return cap, node_type


def _dev_masks(eng, *masks):
    """uint64 mask arrays -> int64 device tensors (the Engine takes masks as int64)"""
    return tuple(eng.dev(a.view(np.int64), torch.int64) for a in masks)


def _live(rule):
    """the rule when it can constrain a pod of the call, else None (the Engine forms without it give the same result)"""
    return rule if rule is not None and not rule.trivial else None


def _write_back_used(nodes, dims, used, touched_keys):
    """store used[n] into node.used_capacity with the key set the reference would hold: the
    node's previous keys plus the keys of every pod counted on it (KubeResource.__add__ unions)."""
    from .kube import KubeResource
    for n, keys in touched_keys.items():
        node = nodes[n]
        merged = set(node.used_capacity.raw) | keys
        res = KubeResource()
        res.raw = {k: float(used[n, dims.index[k]]) for k in merged}
        node.used_capacity = res


# ------------------------------------------------------------------------------------------------
# node selectors: match classes (include/acsfit.h, acsfit_selectors)
# ------------------------------------------------------------------------------------------------
MAX_SELECTOR_CLASSES = 64


class SelectorClasses(object):
    """pod_class uint8[P], node_match uint64[N], pool_match uint64[T] (in the order the pools were given) and the
    number of classes.  Bit c of a mask is set when the node / pool matches the selectors (and, with taints, the
    tolerations) of class c."""

    def __init__(self, pod_class, node_match, pool_match, classes):
        self.pod_class = pod_class
        self.node_match = node_match
        self.pool_match = pool_match
        self.classes = classes

    @property
    def trivial(self):
        """every pod is class 0 (no selector, or one that matches every node and pool)"""
        return not self.pod_class.any()

    def to_device(self, eng, nodes=True):
        """the Engine's selector arguments: (pod_class, node_match, classes) of a node pass, node_match on the device,
        or with nodes=False (pod_class, pool_match, classes) of a bin pass, pool_match on the host"""
        return (eng.dev(self.pod_class, torch.uint8), _dev_masks(eng, self.node_match)[0] if nodes else self.pool_match,
                self.classes)


def _selector_matches(labels, items):
    return all(labels.get(key) == value for key, value in items)  # KubeNode.is_match


def _toleration_items(tolerations):
    """a hashable key of a toleration list (two pods with equal keys tolerate the same taints)"""
    return tuple(tuple(sorted(t.items())) for t in tolerations)


class _Projection(object):
    """the nodes grouped by everything a match can see, so that a match is evaluated once per distinct projection,
    vectorised over the projections, instead of once per node.  Each label key in `keys` is read once per node and its
    values are numbered (a missing label reads as None, as labels.get does in is_match); with `names`, the node's name
    (for matchFields) is numbered as one more column; with `taints`, the node's blocking-taint set
    (kube.blocking_taints) is numbered as the last column.  `group[n]` is node n's projection."""

    def __init__(self, nodes, keys, taints, names=False):
        codes, self.code_of = [], []  # the number of every node's value per column; per label/name column: {value: number}
        labels = [n.selectors for n in nodes] if keys else []
        columns = [[l.get(key) for l in labels] for key in keys]
        if names:
            columns.append([n.name for n in nodes])
        for values in columns:
            code = {v: i for i, v in enumerate(dict.fromkeys(values))}
            self.code_of.append(code)
            codes.append(np.fromiter(map(code.__getitem__, values), dtype=np.int64, count=len(values)))
        self.taint_sets = []
        if taints:
            sets = [kube.blocking_taints(n.taints) for n in nodes]
            code = {s: i for i, s in enumerate(dict.fromkeys(sets))}
            self.taint_sets = list(code)
            codes.append(np.fromiter(map(code.__getitem__, sets), dtype=np.int64, count=len(sets)))
        group, bound = np.zeros(len(nodes), dtype=np.int64), 1  # mixed-radix projection number so far, and its range
        for c in codes:
            radix = int(c.max()) + 1 if len(c) else 1
            if bound * radix >= 1 << 62:  # renumber densely (below N) before the number could overflow
                _, group = np.unique(group, return_inverse=True)
                group, bound = group.reshape(-1), len(nodes)
            group, bound = group * radix + c, bound * radix
        _, first, group = np.unique(group, return_index=True, return_inverse=True)
        self.group = group.reshape(-1)
        self.proj = np.stack([c[first] for c in codes], axis=1) if codes else np.zeros((len(first), 0), np.int64)
        self.column = {key: k for k, key in enumerate(keys)}
        self.name_column = len(keys) if names else None
        self._ints = {}

    def _int_table(self, k):
        """(ok bool[codes], value int64[codes]): the values of column k parsed as kube.parse_int64, per value number"""
        table = self._ints.get(k)
        if table is None:
            parsed = [kube.parse_int64(v) for v in self.code_of[k]]
            table = self._ints[k] = (np.fromiter((p is not None for p in parsed), dtype=bool, count=len(parsed)),
                                     np.fromiter((0 if p is None else p for p in parsed), dtype=np.int64,
                                                 count=len(parsed)))
        return table

    def _requirement(self, k, op, values):
        """bool[projections]: the requirement (kube.requirement_holds) on column k"""
        col, code = self.proj[:, k], self.code_of[k]
        if op in ('Gt', 'Lt'):
            ok, number = self._int_table(k)
            return ok[col] & (number[col] > values[0] if op == 'Gt' else number[col] < values[0])
        if op in ('Exists', 'DoesNotExist'):
            op, values = ('NotIn' if op == 'Exists' else 'In'), (None,)
        hit = np.isin(col, [code[v] for v in values if v in code])
        return hit if op == 'In' else ~hit

    def affinity(self, terms):
        """bool[projections]: the canonical required node affinity (kube.node_affinity_terms) admits the nodes"""
        if terms is None:
            return np.ones(len(self.proj), dtype=bool)
        match = np.zeros(len(self.proj), dtype=bool)
        for exprs, fields in terms:
            term = np.ones(len(self.proj), dtype=bool)
            for key, op, values in exprs:
                term &= self._requirement(self.column[key], op, values)
            for _, op, values in fields:
                term &= self._requirement(self.name_column, op, values)
            match |= term
        return match

    def selector(self, items):
        """bool[projections]: the labels match the selector `items` (KubeNode.is_match)"""
        match = np.ones(len(self.proj), dtype=bool)
        for key, value in items:
            k = self.column[key]
            c = self.code_of[k].get(value)
            if c is None:  # no node carries this value (or, for None, lacks the key)
                match[:] = False
                break
            match &= self.proj[:, k] == c
        return match

    def tolerated(self, tolerations):
        """bool[projections]: a pod with these tolerations tolerates every blocking taint (needs taints=True)"""
        ok = np.fromiter((kube.tolerates_all(tolerations, s) for s in self.taint_sets), dtype=bool,
                         count=len(self.taint_sets))
        return ok[self.proj[:, -1]]


def _match_keys(pods, taints, affinity):
    """the distinct (selector items, toleration items, canonical node affinity) of the pods in first-occurrence order as
    (selector items, one toleration list, node affinity), and every pod's index into them.  Without taints a pod without
    a selector and without a required node affinity gets -1 (it matches everything)."""
    index, distinct = {}, []
    of_pod = np.full(len(pods), -1, dtype=np.int64)
    for i, pod in enumerate(pods):
        selectors = pod.selectors
        tolerations = pod.tolerations if taints else ()
        terms = pod.node_affinity if affinity else None
        if not selectors and not taints and terms is None:
            continue
        key = (tuple(sorted(selectors.items())) if selectors else (),
               _toleration_items(tolerations) if tolerations else (), terms)
        j = index.get(key)
        if j is None:
            j = index[key] = len(distinct)
            distinct.append((key[0], tolerations, terms))
        of_pod[i] = j
    return distinct, of_pod


def _projection(nodes, distinct, taints):
    """the _Projection of the nodes over every label key the selectors and node-affinity terms read, with the name
    column when some term has matchFields"""
    keys, names = set(), False
    for items, _, terms in distinct:
        keys.update(key for key, _ in items)
        for exprs, fields in terms or ():
            keys.update(key for key, _, _ in exprs)
            names = names or bool(fields)
    return _Projection(nodes, sorted(keys), taints, names)


def _node_match(proj, items, tolerations, terms, taints):
    """bool[projections]: selector, node affinity and (with taints) tolerations all admit the nodes"""
    match = proj.selector(items)
    if terms is not None:
        match &= proj.affinity(terms)
    if taints:
        match &= proj.tolerated(tolerations)
    return match


def selector_classes(pods, nodes, pools, taints=False, affinity=False):
    """map every distinct match signature (set of matching nodes, set of matching pools) of the pods' nodeSelectors
    to a class number.  Class 0 is "no selector": it matches everything, so a selector that matches every node and
    every pool shares it.  Pods whose selectors match the same nodes and pools share a class.  A pool matches with
    the labels a new node of it would carry (AgentPool.labels).  Raises ValueError above 64 classes.

    With `taints`, a pod matches a node or pool when its selector matches AND it tolerates every blocking taint there
    (kube.blocking_taints of KubeNode.taints, AgentPool.taints; KubePod.tolerations).  Class 0 keeps its meaning
    (matches every node and pool); it may then have no pod.  Without `taints`, taints and tolerations are never read.

    With `affinity`, the pod's required node affinity (KubePod.node_affinity) must admit the node too (a pool: a new
    node of it, kube.pool_affinity_matches); without it, the field is never read.  Each distinct (selector,
    tolerations, node affinity) is evaluated once per distinct node projection (_Projection)."""
    pods, nodes, pools = list(pods), list(nodes), list(pools)
    distinct, of_pod = _match_keys(pods, taints, affinity)
    if not distinct:
        return SelectorClasses(np.zeros(len(pods), dtype=np.uint8), np.ones(len(nodes), dtype=np.uint64),
                               np.ones(len(pools), dtype=np.uint64), 1)
    proj = _projection(nodes, distinct, taints)
    pool_labels = [p.labels for p in pools]
    pool_taints = [p.taints for p in pools] if taints else [()] * len(pools)
    everything = (b"\x01" * len(proj.proj), b"\x01" * len(pools))
    class_of_sig = {everything: 0}
    class_of_key = np.zeros(len(distinct) + 1, dtype=np.uint8)  # the last entry (index -1) is class 0
    for j, (items, tolerations, terms) in enumerate(distinct):
        nmatch = _node_match(proj, items, tolerations, terms, taints)
        sig = (nmatch.tobytes(), bytes(_selector_matches(l, items) and kube.tolerates_all(tolerations, t) and
                                       kube.pool_affinity_matches(terms, l)
                                       for l, t in zip(pool_labels, pool_taints)))
        c = class_of_sig.get(sig)
        if c is None:
            c = len(class_of_sig)
            if c >= MAX_SELECTOR_CLASSES:
                raise ValueError("more than %d distinct node-selector match signatures are not supported"
                                 % MAX_SELECTOR_CLASSES)
            class_of_sig[sig] = c
        class_of_key[j] = c
    node_match = np.ones(len(proj.proj), dtype=np.uint64)
    pool_match = np.ones(len(pools), dtype=np.uint64)
    for (nsig, psig), c in class_of_sig.items():
        if c:
            bit = np.uint64(1) << np.uint64(c)
            node_match[np.frombuffer(nsig, dtype=np.uint8).astype(bool)] |= bit
            pool_match[np.frombuffer(psig, dtype=np.uint8).astype(bool)] |= bit
    return SelectorClasses(class_of_key[of_pod], node_match[proj.group], pool_match, len(class_of_sig))


def pending_match(pods, nodes, taints=False, affinity=False):
    """bool[N]: some pod of `pods` matches node n (KubeNode.is_match).  All True when a pod has no selector.  With
    `taints` a pod matches a node when its selector matches AND it tolerates the node's blocking taints: a pod without
    a selector then matches only the nodes whose blocking taints it tolerates.  With `affinity` the pod's required node
    affinity (KubePod.node_affinity) must admit the node too.

    Maintain asks this of every node of the scalable pools (up to 10^6), so matches are not evaluated node by node:
    each distinct (selector, tolerations, node affinity) is evaluated once per distinct node projection (_Projection)."""
    nodes = list(nodes)
    if not taints and not affinity and any(not pod.selectors for pod in pods):
        return np.ones(len(nodes), dtype=bool)
    distinct, of_pod = _match_keys(pods, taints, affinity)
    if not taints and (of_pod < 0).any():  # a pod without selector and node affinity
        return np.ones(len(nodes), dtype=bool)
    if not distinct or not nodes:
        return np.zeros(len(nodes), dtype=bool)
    proj = _projection(nodes, distinct, taints)
    hit = np.zeros(len(proj.proj), dtype=bool)
    for items, tolerations, terms in distinct:
        hit |= _node_match(proj, items, tolerations, terms, taints)
    return hit[proj.group]


# ------------------------------------------------------------------------------------------------
# required pod anti-affinity: term masks (include/acsfit.h, acsfit_anti_affinity)
# ------------------------------------------------------------------------------------------------
MAX_AA_TERMS = 64


class AntiAffinity(object):
    """pod_carries / pod_matches uint64[P] (the terms each pod has / the terms that select it), node_carries /
    node_matches uint64[N] (the OR of both over the pods already on each node) and the number of terms.  Bit k = term k
    of `terms`, a list of (namespaces, canonical selector)."""

    def __init__(self, pod_carries, pod_matches, node_carries, node_matches, terms):
        self.pod_carries = pod_carries
        self.pod_matches = pod_matches
        self.node_carries = node_carries
        self.node_matches = node_matches
        self.terms = terms

    @property
    def trivial(self):
        """no term can block a pod of this call: the plain entry points give the same result"""
        return not self.terms

    def to_device(self, eng, nodes=True):
        """the Engine's anti-affinity arguments on the device: pod_carries, pod_matches and, with `nodes`,
        node_carries and node_matches"""
        masks = (self.pod_carries, self.pod_matches) + ((self.node_carries, self.node_matches) if nodes else ())
        return _dev_masks(eng, *masks)


def _pod_projection(pods, keys):
    """(group[len(pods)], proj[G, 1 + len(keys)], code_of): the pods grouped by (namespace, the values of the label keys
    the terms read), as _Projection groups nodes.  Column 0 numbers the namespace, column 1 + k the value of keys[k]
    (None when absent); code_of[c] maps a value of column c to its number."""
    columns = [[p.namespace for p in pods]]
    labels = [p.labels for p in pods] if keys else []
    for key in keys:
        columns.append([l.get(key) for l in labels])
    codes, code_of = [], []
    for values in columns:
        code = {v: i for i, v in enumerate(dict.fromkeys(values))}
        code_of.append(code)
        codes.append(np.fromiter(map(code.__getitem__, values), dtype=np.int64, count=len(values)))
    if not len(pods):
        return np.zeros(0, np.int64), np.zeros((0, len(columns)), np.int64), code_of
    stacked = np.stack(codes, axis=1)
    proj, group = np.unique(stacked, axis=0, return_inverse=True)
    return group.reshape(-1), proj, code_of


def _term_selects(term, proj, code_of, column):
    """bool[G]: the term (namespaces, canonical selector) selects the pods of each projection"""
    namespaces, (items, reqs) = term
    hit = np.isin(proj[:, 0], [code_of[0][ns] for ns in namespaces if ns in code_of[0]])

    def codes(key, values):
        return [code_of[column[key]][v] for v in values if v in code_of[column[key]]]
    for key, value in items:
        hit &= np.isin(proj[:, column[key]], codes(key, (value,)))
    for key, op, values in reqs:
        col = proj[:, column[key]]
        if op == 'In':
            hit &= np.isin(col, codes(key, values))
        elif op == 'NotIn':
            hit &= ~np.isin(col, codes(key, values))
        elif op == 'Exists':
            hit &= ~np.isin(col, codes(key, (None,)))
        else:
            hit &= np.isin(col, codes(key, (None,)))
    return hit


def anti_affinity(pods, nodes=(), running_pods=()):
    """term masks of the pods to place (`pods`) and of the nodes (the pods of `running_pods` on them count, matched by
    node name as the occupancy count matches them).  A term (KubePod.anti_affinity_terms) is kept only when it can
    block a pod to place: a pod to place carries it and it selects some other pod, or it selects a pod to place and some
    other pod carries it.  (A lone replica of a self-anti-affine deployment blocks nothing, so its term is dropped.)  The
    bin pass calls this with the pending pods alone: only they meet in new bins.  Kept terms are numbered in
    first-occurrence order; ValueError above 64.  Each term is evaluated once per distinct (namespace, label values it
    reads) projection of the pods, vectorised, not once per pod; nothing of size pods x terms is built."""
    pods, nodes = list(pods), list(nodes)
    row_ptr, run_idx = running_csr(nodes, running_pods) if nodes and running_pods else (None, np.zeros(0, np.int32))
    carries, matches, row_carries, row_matches, terms = _anti_affinity_masks(pods, list(running_pods), run_idx)
    node_carries = np.zeros(len(nodes), dtype=np.uint64)
    node_matches = np.zeros(len(nodes), dtype=np.uint64)
    if len(run_idx) and terms:
        # OR over the running pods of each node
        node_of = np.repeat(np.arange(len(nodes), dtype=np.int64), np.diff(row_ptr))
        np.bitwise_or.at(node_carries, node_of, row_carries)
        np.bitwise_or.at(node_matches, node_of, row_matches)
    return AntiAffinity(carries, matches, node_carries, node_matches, terms)


def anti_affinity_rows(pods, running_pods, pods_lists):
    """anti_affinity's masks without the OR per node: (pod_carries uint64[P], pod_matches uint64[P], row_carries uint64[R],
    row_matches uint64[R], terms), with one row per entry of the concatenated `pods_lists` (node_states' table).  Every
    pod of `pods_lists` is an object of `running_pods`, grouped per node as the occupancy count groups them; the terms,
    their numbering and their dropping are then those of anti_affinity(pods, nodes, running_pods).  Raises ValueError
    for a pod of `pods_lists` that is not in `running_pods`."""
    running = list(running_pods)
    return _anti_affinity_masks(list(pods), running, _row_index(running, pods_lists))


def _row_index(running, pods_lists):
    """int64[R]: the index in `running` of every pod of the concatenated `pods_lists` (matched by identity); ValueError
    for a pod that is not in `running`"""
    ids = np.fromiter(map(id, running), dtype=np.int64, count=len(running))
    order = np.argsort(ids, kind="stable")
    flat = np.fromiter(map(id, itertools.chain.from_iterable(pods_lists)), dtype=np.int64)
    pos = np.searchsorted(ids[order], flat)
    if len(flat) and ((pos >= len(ids)).any() or (ids[order[np.minimum(pos, len(ids) - 1)]] != flat).any()):
        raise ValueError("a pod of pods_lists is not one of running_pods")
    return order[pos] if len(flat) else np.zeros(0, np.int64)


def _anti_affinity_masks(pods, running, run_idx):
    """(pod_carries[P], pod_matches[P], row_carries, row_matches, kept terms): the masks of the pods to place and of
    running[run_idx[k]] for every k, for anti_affinity and anti_affinity_rows"""
    on_nodes = np.unique(run_idx)
    everyone = pods + [running[j] for j in on_nodes.tolist()]
    P = len(pods)
    term_id, terms = {}, []
    carried = []  # per pod of `everyone`: its term numbers (before dropping)
    for p in everyone:
        ids = []
        for t in p.anti_affinity_terms:
            k = term_id.get(t)
            if k is None:
                k = term_id[t] = len(terms)
                terms.append(t)
            ids.append(k)
        carried.append(ids)
    if not terms:
        return (np.zeros(P, np.uint64), np.zeros(P, np.uint64), np.zeros(len(run_idx), np.uint64),
                np.zeros(len(run_idx), np.uint64), [])
    T = len(terms)
    keys = sorted({key for _, (items, reqs) in terms for key, *_ in items + reqs})
    group, proj, code_of = _pod_projection(everyone, keys)
    column = {key: 1 + k for k, key in enumerate(keys)}
    G = len(proj)
    # (pod, term) pairs of the carried terms (anti_affinity_terms lists a term once per pod)
    lens = np.fromiter(map(len, carried), dtype=np.int64, count=len(everyone))
    pair_pod = np.repeat(np.arange(len(everyone), dtype=np.int64), lens)
    pair_term = np.fromiter(itertools.chain.from_iterable(carried), dtype=np.int64, count=int(lens.sum()))
    to_place = pair_pod < P
    n_carry = np.bincount(pair_term, minlength=T)               # pods that carry the term
    n_carry_p = np.bincount(pair_term[to_place], minlength=T)   # ... pods to place among them
    per_group = np.bincount(group, minlength=G)
    per_group_p = np.bincount(group[:P], minlength=G)
    order = np.argsort(pair_term[to_place], kind="stable")
    carrier_p, bounds = pair_pod[to_place][order], np.searchsorted(pair_term[to_place][order], np.arange(T + 1))
    n_sel, n_sel_p, n_both_p = (np.zeros(T, np.int64) for _ in range(3))  # selected pods, to place, to place + carrier
    for t in range(T):
        hit = _term_selects(terms[t], proj, code_of, column)
        n_sel[t], n_sel_p[t] = per_group[hit].sum(), per_group_p[hit].sum()
        n_both_p[t] = hit[group[carrier_p[bounds[t]:bounds[t + 1]]]].sum()
    # a pair of two different pods, one to place, where one carries the term and it selects the other: the only
    # carrier-and-selected pod of each count being the same pod is the one way to have counts but no such pair
    alone = n_both_p == 1
    relevant = ((n_carry_p >= 1) & (n_sel >= 1) & ~((n_sel == 1) & (n_carry_p == 1) & alone)) | \
        ((n_sel_p >= 1) & (n_carry >= 1) & ~((n_carry == 1) & (n_sel_p == 1) & alone))
    keep = np.nonzero(relevant)[0]
    if len(keep) > MAX_AA_TERMS:
        raise ValueError("more than %d distinct pod anti-affinity terms are not supported" % MAX_AA_TERMS)
    bit_of = np.full(T, -1, dtype=np.int64)
    bit_of[keep] = np.arange(len(keep))
    group_matches = np.zeros(G, dtype=np.uint64)
    for k, t in enumerate(keep.tolist()):
        group_matches[_term_selects(terms[t], proj, code_of, column)] |= np.uint64(1) << np.uint64(k)
    matches = group_matches[group]
    carries = np.zeros(len(everyone), dtype=np.uint64)
    kept = bit_of[pair_term] >= 0
    np.bitwise_or.at(carries, pair_pod[kept], np.uint64(1) << bit_of[pair_term[kept]].astype(np.uint64))
    at = P + np.searchsorted(on_nodes, run_idx)  # a running pod is in `everyone` at P + its rank in on_nodes
    return carries[:P], matches[:P], carries[at], matches[at], [terms[k] for k in keep.tolist()]


# ------------------------------------------------------------------------------------------------
# required pod affinity: signature masks (include/acsfit.h, acsfit_pod_affinity)
# ------------------------------------------------------------------------------------------------
MAX_PA_SIGNATURES = 64


class PodAffinity(object):
    """pod_requires uint64[P] (the bit of the pod's signature, 0 without one), pod_matches uint64[P] (the signatures the
    pod matches), pod_self = pod_requires & pod_matches, node_has uint64[N] (the OR of pod_matches over the pods already
    on each node), present (the OR of node_has) and the signatures: bit s = signatures[s], a frozenset of terms."""

    def __init__(self, pod_requires, pod_matches, node_has, signatures):
        self.pod_requires = pod_requires
        self.pod_matches = pod_matches
        self.pod_self = pod_requires & pod_matches
        self.node_has = node_has
        self.signatures = signatures

    @property
    def present(self):
        """the OR of node_has: the signatures some node holds"""
        return int(np.bitwise_or.reduce(self.node_has)) if len(self.node_has) else 0

    def present_signatures(self):
        """the signatures some node holds, as a set (the numbering of another call differs)"""
        present = self.present
        return {sig for k, sig in enumerate(self.signatures) if (present >> k) & 1}

    @property
    def trivial(self):
        """no pod of this call has a signature: the calls without pod affinity give the same result"""
        return not self.signatures

    def to_device(self, eng, nodes=True):
        """the Engine's pod-affinity arguments on the device: pod_requires, pod_self, pod_matches and, with `nodes`,
        node_has"""
        return _dev_masks(eng, self.pod_requires, self.pod_self, self.pod_matches, *((self.node_has,) if nodes else ()))


def pod_affinity(pods, nodes=(), running_pods=()):
    """signature masks of the pods to place (`pods`) and of the nodes (the pods of `running_pods` on them count, matched
    by node name as the occupancy count and anti_affinity match them).  A pod's signature is the set of its terms
    (KubePod.affinity_terms); a pod matches a signature when every term of it selects the pod.  Signatures are numbered
    in first-occurrence order over `pods`; ValueError above 64.  Each term is evaluated once per distinct (namespace,
    label values it reads) projection of the pods, as anti_affinity does."""
    pods, nodes, running = list(pods), list(nodes), list(running_pods)
    row_ptr, run_idx = running_csr(nodes, running) if nodes and running else (None, np.zeros(0, np.int32))
    requires, matches, run_matches, signatures = _pod_affinity_masks(pods, running, run_idx)
    node_has = np.zeros(len(nodes), dtype=np.uint64)
    if len(run_idx) and signatures:
        node_of = np.repeat(np.arange(len(nodes), dtype=np.int64), np.diff(row_ptr))
        np.bitwise_or.at(node_has, node_of, run_matches)
    return PodAffinity(requires, matches, node_has, signatures)


def pod_affinity_rows(pods, running_pods, pods_lists, nodes=None):
    """pod_affinity's masks for maintain's table: (pod_requires uint64[P], pod_self uint64[P], pod_matches uint64[P],
    row_has uint64[R], present, signatures).  row_has holds the signatures each entry of the concatenated `pods_lists`
    (node_states' table; objects of `running_pods`) matches, before the OR per node.  `present` (an int) is the OR of
    the signatures matched by the pods of `running_pods` on `nodes` (matched by node name, as pod_affinity matches
    them), or by the rows of the table when `nodes` is None: the pods whose presence ends a self-affine group's
    bootstrap.  The signatures and their numbering are those of pod_affinity(pods, nodes, running_pods).  Raises
    ValueError for a pod of `pods_lists` that is not in `running_pods`."""
    pods, running = list(pods), list(running_pods)
    rows = _row_index(running, pods_lists)
    if nodes is None:
        on_nodes = np.zeros(0, np.int64)
    else:
        names = {n.name for n in nodes}
        on_nodes = np.fromiter((j for j, p in enumerate(running) if p.node_name in names), dtype=np.int64)
    requires, matches, run_matches, signatures = _pod_affinity_masks(pods, running, np.concatenate([rows, on_nodes]))
    row_has = run_matches[:len(rows)]
    seen = row_has if nodes is None else run_matches[len(rows):]
    present = int(np.bitwise_or.reduce(seen)) if len(seen) else 0
    return requires, requires & matches, matches, row_has, present, signatures


def _pod_affinity_masks(pods, running, run_idx):
    """(pod_requires[P], pod_matches[P], run_matches, signatures): the signature masks of the pods to place and the
    signatures running[run_idx[k]] matches for every k, for pod_affinity and pod_affinity_rows.  Each term is
    evaluated once over the pods to place and the running pods run_idx names."""
    P = len(pods)
    sig_id, signatures, requires = {}, [], np.zeros(P, dtype=np.uint64)
    for i, p in enumerate(pods):
        terms = p.affinity_terms
        if not terms:
            continue
        sig = frozenset(terms)
        k = sig_id.get(sig)
        if k is None:
            if len(signatures) == MAX_PA_SIGNATURES:
                raise ValueError("more than %d distinct pod affinity signatures are not supported" % MAX_PA_SIGNATURES)
            k = sig_id[sig] = len(signatures)
            signatures.append(sig)
        requires[i] = np.uint64(1) << np.uint64(k)
    if not signatures:
        return requires, np.zeros(P, np.uint64), np.zeros(len(run_idx), np.uint64), signatures
    on_nodes = np.unique(run_idx)
    everyone = pods + [running[j] for j in on_nodes.tolist()]
    terms = list(dict.fromkeys(t for sig in signatures for t in sig))
    keys = sorted({key for _, sel in terms if sel is not None for key, *_ in sel[0] + sel[1]})
    group, proj, code_of = _pod_projection(everyone, keys)
    column = {key: 1 + k for k, key in enumerate(keys)}
    hit = {t: (_term_selects(t, proj, code_of, column) if t[1] is not None else np.zeros(len(proj), bool))
           for t in terms}
    group_matches = np.zeros(len(proj), dtype=np.uint64)
    for k, sig in enumerate(signatures):
        both = np.ones(len(proj), bool)
        for t in sig:
            both &= hit[t]
        group_matches[both] |= np.uint64(1) << np.uint64(k)
    matches = group_matches[group]
    at = P + np.searchsorted(on_nodes, run_idx)  # a running pod is in `everyone` at P + its rank in on_nodes
    return requires, matches[:P].copy(), matches[at], signatures


# ------------------------------------------------------------------------------------------------
# hostname topology spread: keys, counts and domains (include/acsfit.h, acsfit_topology_spread)
# ------------------------------------------------------------------------------------------------
MAX_TS_KEYS = 64
NO_SPREAD_KEY = 0xFF
INT32_MAX = 2 ** 31 - 1


class TopologySpread(object):
    """pod_key uint8[P] (the pod's key, NO_SPREAD_KEY without a constraint), pod_skew int32[P] (maxSkew - 1 when the
    pod's own selector selects it, else maxSkew), pod_matches uint64[P] (the keys whose selector selects the pod),
    node_count int32[keys, N] (the selected pods on each node), node_domain uint64[N] (the keys each node is a domain
    of), floor int32[keys] (the smallest count over the key's domains outside the node list, INT32_MAX without one, 0
    when the key has fewer domains in all than its minDomains) and the keys: (namespace, selector, domain set,
    minDomains) tuples, bit k = keys[k]."""

    def __init__(self, pod_key, pod_skew, pod_matches, node_count, node_domain, floor, keys):
        self.pod_key = pod_key
        self.pod_skew = pod_skew
        self.pod_matches = pod_matches
        self.node_count = node_count
        self.node_domain = node_domain
        self.floor = floor
        self.keys = keys

    @property
    def trivial(self):
        """no pod of this call has a constraint: the calls without topology spread give the same result"""
        return not self.keys

    def to_device(self, eng, nodes=True):
        """the Engine's topology-spread arguments: the key count, pod_key, pod_skew and pod_matches on the device and,
        with `nodes`, node_count and node_domain on the device and floor on the host"""
        pods = (len(self.keys), eng.dev(self.pod_key, torch.uint8), eng.dev(self.pod_skew, torch.int32),
                *_dev_masks(eng, self.pod_matches))
        if not nodes:
            return pods
        return pods + (eng.dev(self.node_count, torch.int32), *_dev_masks(eng, self.node_domain), self.floor)


def _spread_domains(pods, constraints, all_nodes):
    """(domain key per pod with a constraint, {domain key: bool[len(all_nodes)]}): the nodes counted for each pod's
    minimum.  nodeAffinityPolicy Honor: the pod's nodeSelector and required node affinity admit the node; nodeTaintsPolicy
    Honor: the pod tolerates its blocking taints.  Each distinct requirement is evaluated once per node projection."""
    spec_of, specs = {}, {}
    for i, c in constraints:
        pod = pods[i]
        items = tuple(sorted(pod.selectors.items())) if c.honor_affinity and pod.selectors else ()
        terms = pod.node_affinity if c.honor_affinity else None
        tolerations = pod.tolerations if c.honor_taints else None
        key = (items, terms, None if tolerations is None else _toleration_items(tolerations))
        spec_of[i] = key
        specs.setdefault(key, (items, tolerations, terms))
    if not specs:
        return spec_of, {}
    if not all_nodes:
        return spec_of, {key: np.zeros(0, dtype=bool) for key in specs}
    taints = any(t is not None for _, t, _ in specs.values())
    distinct = [(items, t, terms) for items, t, terms in specs.values()]
    proj = _projection(all_nodes, distinct, taints)
    domains = {}
    for key, (items, tolerations, terms) in specs.items():
        match = proj.selector(items)
        if terms is not None:
            match &= proj.affinity(terms)
        if tolerations is not None:
            match &= proj.tolerated(tolerations)
        domains[key] = match[proj.group]
    return spec_of, domains


def topology_spread(pods, nodes=(), running_pods=(), other_nodes=()):
    """the topology-spread arrays of the pods to place (`pods`) over the agent nodes `nodes`.  `other_nodes` are the
    nodes of the listing outside them (the master): they cannot take a pod here but they are domains, so their counts
    go into `floor`.  The pods of `running_pods` on a node count on it, matched by node name as the occupancy count
    matches them.  A key is a distinct (namespace, selector with the matchLabelKeys values, domain set, minDomains) of
    the pods' honoured constraints (KubePod.topology_spread), numbered in first-occurrence order; ValueError above 64.
    Each selector is evaluated once per distinct (namespace, label values it reads) projection of the pods, and each
    domain requirement once per node projection; nothing of size pods x nodes is built."""
    pods, nodes, other, running = list(pods), list(nodes), list(other_nodes), list(running_pods)
    P, N = len(pods), len(nodes)
    constraints = [(i, c) for i, c in ((i, p.topology_spread) for i, p in enumerate(pods)) if c is not None]
    pod_key = np.full(P, NO_SPREAD_KEY, dtype=np.uint8)
    pod_skew = np.zeros(P, dtype=np.int32)
    if not constraints:
        return TopologySpread(pod_key, pod_skew, np.zeros(P, np.uint64), np.zeros((0, N), np.int32),
                              np.zeros(N, np.uint64), np.zeros(0, np.int32), [])
    all_nodes = nodes + other
    spec_of, domains = _spread_domains(pods, constraints, all_nodes)
    dom_bytes = {spec: dom.tobytes() for spec, dom in domains.items()}  # once per distinct domain requirement
    key_id, keys, key_domain = {}, [], []
    for i, c in constraints:
        dom = domains[spec_of[i]]
        key = (pods[i].namespace, c.selector, dom_bytes[spec_of[i]], c.min_domains)
        k = key_id.get(key)
        if k is None:
            if len(keys) == MAX_TS_KEYS:
                raise ValueError("more than %d distinct topology spread keys are not supported" % MAX_TS_KEYS)
            k = key_id[key] = len(keys)
            keys.append(key)
            key_domain.append(dom)
        pod_key[i] = k
    K = len(keys)
    # the selected pods: the pods to place and the running pods on the listed nodes, grouped by projection
    row_ptr, run_idx = running_csr(all_nodes, running) if all_nodes and running else \
        (np.zeros(len(all_nodes) + 1, np.int64), np.zeros(0, np.int32))
    on_nodes = np.unique(run_idx)
    everyone = pods + [running[j] for j in on_nodes.tolist()]
    label_keys = sorted({key for _, sel, _, _ in keys if sel is not None for key, *_ in sel[0] + sel[1]})
    group, proj, code_of = _pod_projection(everyone, label_keys)
    column = {key: 1 + k for k, key in enumerate(label_keys)}
    node_of_row = np.repeat(np.arange(len(all_nodes), dtype=np.int64), np.diff(row_ptr))
    at = P + np.searchsorted(on_nodes, run_idx)  # a running pod is in `everyone` at P + its rank in on_nodes
    pod_matches = np.zeros(P, dtype=np.uint64)
    counts = np.zeros((K, len(all_nodes)), dtype=np.int64)
    for k, (ns, sel, _, _) in enumerate(keys):
        hit = _term_selects((frozenset((ns,)), sel), proj, code_of, column) if sel is not None else \
            np.zeros(len(proj), bool)
        pod_matches[hit[group[:P]]] |= np.uint64(1) << np.uint64(k)
        rows = hit[group[at]] if len(run_idx) else np.zeros(0, bool)
        counts[k] = np.bincount(node_of_row[rows], minlength=len(all_nodes))
    for i, c in constraints:
        k = int(pod_key[i])
        pod_skew[i] = c.max_skew - int((int(pod_matches[i]) >> k) & 1)
    node_domain = np.zeros(N, dtype=np.uint64)
    floor = np.full(K, INT32_MAX, dtype=np.int32)
    for k, dom in enumerate(key_domain):
        node_domain[dom[:N]] |= np.uint64(1) << np.uint64(k)
        outside = dom[N:]
        if int(dom.sum()) < keys[k][3]:
            floor[k] = 0
        elif outside.any():
            floor[k] = min(int(counts[k, N:][outside].min()), INT32_MAX)
    node_count = np.minimum(counts[:, :N], INT32_MAX).astype(np.int32)
    return TopologySpread(pod_key, pod_skew, pod_matches, node_count, node_domain, floor, keys)


_topology_spread = topology_spread  # (pending_admit's keyword of the same name hides it there)


# ------------------------------------------------------------------------------------------------
# K0: feasibility (capacity.is_possible over the pools)
# ------------------------------------------------------------------------------------------------
def feasible_pods(pods, agent_pools, classes=None):
    """bool[len(pods)]: (RESOURCE_SPEC[pool.instance_type] - pod.resources).possible for some pool.  With `classes`
    (selector_classes(pods, [], agent_pools)) the pool must also match the pod's nodeSelector."""
    from . import capacity
    pods = list(pods)
    if not pods:
        return np.zeros(0, dtype=bool)
    units = [capacity.RESOURCE_SPEC[pool.instance_type] for pool in agent_pools]
    if not units:
        return np.zeros(len(pods), dtype=bool)
    dims = Dims([p.resources for p in pods] + units)
    req = dims.rows(p.resources for p in pods)
    unit = dims.rows(units)
    _check_finite(unit, "unit capacity")
    bad = _nonfinite_rows(req)       # an infinite request fits nowhere (cap - inf < 0)
    req[bad] = 0.0
    eng = get_engine()
    if _live(classes) is not None:
        mask, _ = eng.feasible_mask_sel(eng.dev(req, torch.float64), eng.dev(unit, torch.float64),
                                        *classes.to_device(eng, nodes=False))
    else:
        mask, _ = eng.feasible_mask(eng.dev(req, torch.float64), eng.dev(unit, torch.float64))
    out = mask.cpu().numpy().astype(bool)
    out[bad] = False
    return out


# ------------------------------------------------------------------------------------------------
# K1: occupancy (node.count_pod over the running pods)
# ------------------------------------------------------------------------------------------------
def running_csr(nodes, running_pods):
    """CSR of running pods per node in pod-list order (cluster.py:165-168 / engine_scaler.py:129-131).
    Two nodes with the same name both get the pod, as the reference's name comparison does."""
    by_name = {}
    for j, pod in enumerate(running_pods):
        by_name.setdefault(pod.node_name, []).append(j)
    row_ptr = np.zeros(len(nodes) + 1, dtype=np.int64)
    idx = []
    for n, node in enumerate(nodes):
        lst = by_name.get(node.name, ())
        idx.extend(lst)
        row_ptr[n + 1] = len(idx)
    return row_ptr, np.asarray(idx, dtype=np.int32)


def count_running_pods(nodes, running_pods):
    """the occupancy loop of Cluster.loop_logic on the GPU; updates node.used_capacity."""
    nodes, running_pods = list(nodes), list(running_pods)
    if not nodes or not running_pods:
        return
    row_ptr, run_idx = running_csr(nodes, running_pods)
    if not len(run_idx):
        return
    dims = Dims([p.resources for p in running_pods] + [n.used_capacity for n in nodes])
    req_run, inv_run, uniq_run = dims.rows((running_pods[j].resources for j in run_idx), groups=True)  # rows in node order: a contiguous table
    if (req_run < 0).any() or np.isnan(req_run).any():
        raise ValueError("negative or NaN resource request")
    used = dims.rows(n.used_capacity for n in nodes)
    eng = get_engine()
    d_used = eng.dev(used, torch.float64)
    eng.occupancy(eng.dev(row_ptr, torch.int64), None, eng.dev(req_run, torch.float64), d_used)
    used = d_used.cpu().numpy()
    node_of_row = np.repeat(np.arange(len(nodes), dtype=np.int64), np.diff(row_ptr))
    _write_back_used(nodes, dims, used, _touched_keys(node_of_row, inv_run, uniq_run))


# ------------------------------------------------------------------------------------------------
# first fit over nodes (Cluster.get_pending_pods)
# ------------------------------------------------------------------------------------------------
def first_fit_nodes(pods, nodes, classes=None, anti_affinity=None, pod_affinity=None, topology_spread=None):
    """returns placed[len(pods)] (node index or -1) and mutates node.used_capacity like count_pod.  With `classes`
    (selector_classes(pods, nodes, [])) a pod only takes a node that matches its nodeSelector.  With `anti_affinity`
    (anti_affinity(pods, nodes, running_pods)) a pod only takes a node its required anti-affinity does not block; the
    node masks are updated in place.  With `pod_affinity` (pod_affinity(pods, nodes, running_pods)) a pod only takes a
    node its required pod affinity admits; node_has is updated in place.  With `topology_spread`
    (topology_spread(pods, nodes, running_pods, other_nodes)) a pod only takes a node where its key's skew stays within
    maxSkew; node_count is updated in place."""
    pods, nodes = list(pods), list(nodes)
    placed = np.full(len(pods), -1, dtype=np.int32)
    if not pods or not nodes:
        return placed
    dims = Dims([p.resources for p in pods] + [n.capacity for n in nodes] + [n.used_capacity for n in nodes])
    req, inv_req, uniq_req = dims.rows((p.resources for p in pods), groups=True)
    bad = _nonfinite_rows(req)  # infinite request: can_fit is False on every node
    ok_idx = np.nonzero(~bad)[0].astype(np.int32)
    cap, node_type = _node_types(nodes, dims)
    used = dims.rows(n.used_capacity for n in nodes)
    req[bad] = 0.0
    eng = get_engine()
    sel, aa, pa, ts = map(_live, (classes, anti_affinity, pod_affinity, topology_spread))
    d_sel, d_aa, d_pa, d_ts = (None if r is None else r.to_device(eng) for r in (sel, aa, pa, ts))
    d_used = eng.dev(used, torch.float64)
    head = (eng.dev(req, torch.float64), None if not bad.any() else eng.dev(ok_idx, torch.int32),
            eng.dev(cap, torch.float64), eng.dev(node_type, torch.int32), d_used)
    sel_kw = {} if sel is None else dict(zip(("pod_class", "node_match", "classes"), d_sel))
    if ts is not None:
        d_placed, _ = eng.first_fit_nodes_ts(*head, *d_ts, pa=d_pa, aa=d_aa, **sel_kw)
    elif pa is not None:
        d_placed, _ = eng.first_fit_nodes_pa(*head, *d_pa, *(d_aa or ()), **sel_kw)
    elif aa is not None:
        d_placed, _ = eng.first_fit_nodes_aa(*head, *d_aa, *(d_sel or ()))
    elif sel is not None:
        d_placed, _ = eng.first_fit_nodes_sel(*head, *d_sel)
    else:
        d_placed, _ = eng.first_fit_nodes(*head)
    updated = []  # (host array, device tensor) of the rules' node arrays the call updated in place
    if ts is not None:
        updated.append((ts.node_count, d_ts[4]))
    if pa is not None:
        updated.append((pa.node_has, d_pa[3]))
    if aa is not None:
        updated += [(aa.node_carries, d_aa[2]), (aa.node_matches, d_aa[3])]
    for host, d in updated:
        host[...] = d.cpu().numpy().view(host.dtype)
    res = d_placed.cpu().numpy()
    if bad.any():
        placed[ok_idx] = res
    else:
        placed = res
    used = d_used.cpu().numpy()
    took = np.nonzero(placed >= 0)[0]
    _write_back_used(nodes, dims, used, _touched_keys(placed[took], inv_req[took], uniq_req))
    return placed


def single_can_fit(node, resources):
    """KubeNode.can_fit for one vector: a 1 x 1 first fit on a scratch copy of the node row."""
    from .kube import KubeResource

    class _P(object):
        pass
    pod = _P()
    pod.resources = resources

    class _N(object):
        pass
    scratch = _N()
    scratch.capacity = node.capacity
    scratch.used_capacity = KubeResource()
    scratch.used_capacity.raw = dict(node.used_capacity.raw)
    return bool(first_fit_nodes([pod], [scratch])[0] >= 0)


# ------------------------------------------------------------------------------------------------
# fulfill_pending (bins)
# ------------------------------------------------------------------------------------------------
def fulfill(unique_pods, num_listed, ordered_pools, ignored_pool_names, over_provision, classes=None,
            anti_affinity=None, pod_affinity=None, affinity_present=(), topology_spread=None):
    """Scaler.fulfill_pending's packing + size arithmetic; pools already in visiting order.  With `classes`
    (selector_classes(unique_pods, [], ordered_pools)) a pool only takes the pods whose nodeSelector it matches.  With
    `anti_affinity` (anti_affinity(unique_pods)) a pod only takes a bin its required anti-affinity does not block.  With
    `pod_affinity` (pod_affinity(unique_pods)) a pod only takes a bin its required pod affinity admits;
    `affinity_present` holds the signatures the nodes already hold (PodAffinity.present_signatures of the node pass);
    without it only the pods this call places count.  With `topology_spread` (topology_spread(unique_pods)) a new node
    takes at most maxSkew pods its key's selector selects, counting the pod itself."""
    from . import capacity
    units = [capacity.RESOURCE_SPEC[pool.instance_type] for pool in ordered_pools]
    dims = Dims([p.resources for p in unique_pods] + units)
    req = dims.rows(p.resources for p in unique_pods)
    unit = dims.rows(units) if units else np.zeros((0, dims.Dp))
    _check_finite(unit, "unit capacity")
    _check_finite(req, "pending pod request")  # pending pods passed is_possible, so they are finite
    eng = get_engine()
    pools = (np.asarray([pool.actual_capacity for pool in ordered_pools], dtype=np.int32),
             np.asarray([min(pool.max_size, 2 ** 31 - 1) for pool in ordered_pools], dtype=np.int32),
             np.asarray([1 if pool.name in ignored_pool_names else 0 for pool in ordered_pools], dtype=np.uint8))
    sel, aa, pa, ts = map(_live, (classes, anti_affinity, pod_affinity, topology_spread))
    d_sel, d_aa, d_pa, d_ts = (None if r is None else r.to_device(eng, nodes=False) for r in (sel, aa, pa, ts))
    present = 0 if pa is None else sum(1 << k for k, sig in enumerate(pa.signatures) if sig in affinity_present)
    head = (eng.dev(req, torch.float64), num_listed, unit, *pools, over_provision)
    sel_kw = {} if sel is None else dict(zip(("pod_class", "pool_match", "classes"), d_sel))
    if ts is not None:
        res = eng.fulfill_pending_ts(*head, *d_ts, pa=d_pa, present=present, aa=d_aa, **sel_kw)
    elif pa is not None:
        res = eng.fulfill_pending_pa(*head, *d_pa, present, *(d_aa or (None, None)), *(d_sel or ()))
    elif aa is not None:
        res = eng.fulfill_pending_aa(*head, *d_aa, *(d_sel or ()))
    elif sel is not None:
        res = eng.fulfill_pending_sel(*head, *d_sel)
    else:
        res = eng.fulfill_pending(*head)
    res["acc_pool"] = res["acc_pool"].cpu().numpy()
    res["bin_of"] = res["bin_of"].cpu().numpy()
    return res


# ------------------------------------------------------------------------------------------------
# idle scan + maintain decisions
# ------------------------------------------------------------------------------------------------
POD_BUSY, POD_UNDRAINABLE = 1, 2
NODE_UNSCHEDULABLE, NODE_NO_PENDING_MATCH = 1, 2


def pod_flags(pod, now_by_tz=None):
    """host-computed booleans of get_node_state (scaler.py:76, :82-83).  `now_by_tz` (a dict) lets a batch read
    the clock once per time zone instead of once per pod (kube.py:68 reads it per call; within one maintain pass
    the readings differ by microseconds against a one-hour grace period)."""
    proxy = 'kube-proxy' in pod.name
    flags = 0
    if not pod.is_mirrored() and not proxy:
        flags |= POD_BUSY
    if proxy:
        return flags
    if now_by_tz is None:
        drainable = pod.is_drainable()
    else:  # is_drainable(), with the clock of the batch (same short-circuit order: replicated, critical, grace)
        drainable = pod.is_replicated() and not pod.is_critical()
        if drainable:
            start = pod.start_time
            if not start:
                drainable = False
            else:
                tz = start.tzinfo
                now = now_by_tz.get(id(tz))  # (tzinfo objects need not be hashable: keyed by identity)
                if now is None:
                    from . import utils
                    now = now_by_tz[id(tz)] = utils.now(tz)
                drainable = not ((now - start) < pod._DRAIN_GRACE_PERIOD)
    if not drainable:
        flags |= POD_UNDRAINABLE
    return flags


def node_age_seconds(node, now_by_tz=None):
    """(now - creation).seconds -- wraps at one day, like the reference (scaler.py:78).  `now_by_tz`: one clock
    reading per time zone and batch, as in pod_flags (now(tz) on a dateutil zone costs ~10 us: it converts from UTC)."""
    from . import utils
    tz = node.creation_time.tzinfo
    if now_by_tz is None:
        return (utils.now(tz) - node.creation_time).seconds
    now = now_by_tz.get(id(tz))
    if now is None:
        now = now_by_tz[id(tz)] = utils.now(tz)
    return (now - node.creation_time).seconds


class PendingAdmit(object):
    """what acsfit_pending_admit(_pa, _ts) reads beside node_states' table: row_carries / row_matches uint64[R] (one
    per row of the table; None without the anti-affinity test), row_has uint64[R] (None without the pod-affinity test),
    node_match uint64[N] class masks or None (every pod matches every node), and the U distinct signatures (class,
    carries, matches, need, key, skew) of the pods to schedule: sig_class uint8[U], sig_carries / sig_matches /
    sig_need uint64[U], sig_key uint8[U] and sig_skew int32[U] (None without the test they belong to).  With the
    spread test, node_count int32[keys, N], node_domain uint64[N] and floor int32[keys] are topology_spread's."""

    def __init__(self, row_carries, row_matches, node_match, sig_class, sig_carries, sig_matches, row_has=None,
                 sig_need=None, sig_key=None, sig_skew=None, node_count=None, node_domain=None, floor=None):
        self.row_carries = row_carries
        self.row_matches = row_matches
        self.node_match = node_match
        self.sig_class = sig_class
        self.sig_carries = sig_carries
        self.sig_matches = sig_matches
        self.row_has = row_has
        self.sig_need = sig_need
        self.sig_key = sig_key
        self.sig_skew = sig_skew
        self.node_count = node_count
        self.node_domain = node_domain
        self.floor = floor


def pending_admit(pods, running_pods, nodes, pods_lists, selectors=False, taints=False, affinity=False,
                  anti_affinity=True, pod_affinity=False, agent_nodes=None, topology_spread=False, other_nodes=()):
    """the PendingAdmit of node_states(admit=...): node n stays pod-pending only when some pod of `pods` (the pods to
    schedule) passes every enabled test against pods_lists[n] (the node's pods, objects of `running_pods`):
    * `anti_affinity`: no pod of the node blocks it and it blocks none of them (anti_affinity_rows' masks);
    * `pod_affinity`: it has no pod-affinity signature, or some pod of the node matches its signature, or it may
      bootstrap a self-affine group: it matches its own signature and no pod of `running_pods` on `agent_nodes` does
      (pod_affinity_rows' masks; `agent_nodes` None: the pods of the table).  The bootstrap is folded into the need:
      need = 0 when requires & present == 0 and self != 0, need = requires otherwise;
    * `topology_spread`: it has no honoured spread constraint, or the node's count of its key is at most its skew plus
      the key's minimum (topology_spread(pods, nodes, running_pods, other_nodes)'s keys, skews, counts, domains and
      floor; each pod is judged on its own, nothing is placed);
    * `selectors`: it matches the node as pending_match(pods, nodes, taints, affinity) decides (the classes are
      selector_classes(pods, nodes, [], taints, affinity)'s; ValueError above 64).
    None when no enabled test can exclude a pod to schedule (no anti-affinity term is kept, no need is nonzero and no
    pod has a spread key): pending_match alone decides.  Without a nonzero need and a key the table is the
    anti-affinity one (acsfit_pending_admit); without a key it is the one of acsfit_pending_admit_pa."""
    pods = list(pods)
    row_carries = row_matches = row_has = None
    columns = []
    if anti_affinity:
        pod_carries, pod_matches, rc, rm, terms = anti_affinity_rows(pods, running_pods, pods_lists)
        if terms:
            row_carries, row_matches = rc, rm
            columns += [pod_carries, pod_matches]
    if pod_affinity:
        requires, own, _, rh, present, _ = pod_affinity_rows(pods, running_pods, pods_lists, nodes=agent_nodes)
        need = np.where(((requires & np.uint64(present)) == 0) & (own != 0), np.uint64(0), requires)
        if need.any():
            row_has = rh
            columns.append(need)
    ts = None
    if topology_spread:
        ts = _topology_spread(pods, nodes, running_pods, other_nodes)
        if ts.trivial:
            ts = None
        else:
            columns += [ts.pod_key.astype(np.uint64), ts.pod_skew.astype(np.uint64)]
    if not columns:
        return None
    pod_class, node_match = np.zeros(len(pods), dtype=np.uint8), None
    if selectors:
        classes = selector_classes(pods, nodes, [], taints=taints, affinity=affinity)
        if not classes.trivial:
            pod_class, node_match = classes.pod_class, classes.node_match
    sig = np.unique(np.stack([pod_class.astype(np.uint64)] + columns, axis=1), axis=0)
    col = lambda k: np.ascontiguousarray(sig[:, k])  # noqa: E731
    aa, pa = row_carries is not None, row_has is not None
    adm = PendingAdmit(row_carries, row_matches, node_match, sig[:, 0].astype(np.uint8), col(1) if aa else None,
                       col(2) if aa else None, row_has, col(1 + 2 * aa) if pa else None)
    if ts is not None:
        k = 1 + 2 * aa + pa
        adm.sig_key, adm.sig_skew = col(k).astype(np.uint8), col(k + 1).astype(np.int32)
        adm.node_count, adm.node_domain, adm.floor = ts.node_count, ts.node_domain, ts.floor
    return adm


def node_states(nodes, pods_lists, any_pending, idle_threshold, no_match=None, admit=None):
    """state code per node (include/acsfit.h ACSFIT_ST_*); pods_lists[n] = the node's pods in order.  `no_match`
    (bool[N], optional): nodes no pod to schedule matches (~pending_match); they are classified as if there were no
    pod to schedule (ACSFIT_NODEF_NO_PENDING_MATCH).  `admit` (pending_admit(..., pods_lists=pods_lists), optional):
    the same flag for the nodes that no pod to schedule is admitted to, set on the GPU (acsfit_pending_admit,
    acsfit_pending_admit_pa when the table has row_has, acsfit_pending_admit_ts when it has sig_key)."""
    nodes = list(nodes)
    if not nodes:
        return np.zeros(0, dtype=np.uint8)
    flat, row_ptr = [], np.zeros(len(nodes) + 1, dtype=np.int64)
    for n, lst in enumerate(pods_lists):
        flat.extend(lst)
        row_ptr[n + 1] = len(flat)
    dims = Dims([p.resources for p in flat] + [n.capacity for n in nodes])
    req_run = dims.rows(p.resources for p in flat) if flat else np.zeros((0, dims.Dp))
    if (req_run < 0).any() or np.isnan(req_run).any():
        raise ValueError("negative or NaN resource request")
    clock = {}
    flags = np.asarray([pod_flags(p, clock) for p in flat], dtype=np.uint8)
    cap, node_type = _node_types(nodes, dims)
    node_flags = np.asarray([NODE_UNSCHEDULABLE if n.unschedulable else 0 for n in nodes], dtype=np.uint8)
    if no_match is not None:
        node_flags |= np.where(np.asarray(no_match, dtype=bool), np.uint8(NODE_NO_PENDING_MATCH), np.uint8(0))
    age = np.asarray([node_age_seconds(n, clock) for n in nodes], dtype=np.int64)
    eng = get_engine()
    d_row_ptr, d_node_flags = eng.dev(row_ptr, torch.int64), eng.dev(node_flags, torch.uint8)
    if admit is not None:
        rows = admit.row_carries if admit.row_carries is not None else admit.row_has
        if rows is not None and len(rows) != len(flat):
            raise ValueError("pending_admit masks of %d pods for a table of %d" % (len(rows), len(flat)))
        dev_masks = lambda a: None if a is None else _dev_masks(eng, a)[0]  # noqa: E731
        ts = admit.sig_key is not None
        pa = ts or admit.row_has is not None  # the _pa and _ts forms take the pod-affinity arrays, None or not
        rows = [dev_masks(admit.row_carries), dev_masks(admit.row_matches)] + \
            ([dev_masks(admit.row_has)] if pa else [])
        sigs = [admit.sig_class, admit.sig_carries, admit.sig_matches] + ([admit.sig_need] if pa else [])
        if ts:
            sigs += [admit.sig_key, admit.sig_skew, admit.node_count.shape[0], eng.dev(admit.node_count, torch.int32),
                     dev_masks(admit.node_domain), admit.floor]
        admit_fn = eng.pending_admit_ts if ts else eng.pending_admit_pa if pa else eng.pending_admit
        admit_fn(d_row_ptr, *rows, dev_masks(admit.node_match), *sigs, d_node_flags)
    st = eng.node_states(d_row_ptr,
                         None,  # contiguous table: the rows ARE in node order (bulk-copy streaming kernel)
                         eng.dev(req_run, torch.float64), eng.dev(flags, torch.uint8),
                         eng.dev(cap, torch.float64), eng.dev(node_type, torch.int32),
                         d_node_flags, eng.dev(age, torch.int64), any_pending,
                         np.asarray([idle_threshold], dtype=np.int64))
    return st[0].contiguous()


def maintain_actions(state_dev, node_pool, budget0, pool_scalable, dry_run):
    eng = get_engine()
    state, action = eng.maintain_actions(state_dev, eng.dev(np.asarray(node_pool, dtype=np.int32), torch.int32),
                                         np.asarray(budget0, dtype=np.int64),
                                         np.asarray(pool_scalable, dtype=np.uint8), dry_run)
    return state.cpu().numpy(), action.cpu().numpy()
