"""Which Engine method snapshot.first_fit_nodes, snapshot.fulfill and snapshot.node_states call, and with what, without
a GPU: a recording stand-in for the Engine takes every call.

For every combination of node selectors, anti-affinity, pod affinity and topology spread -- each absent, trivial (no
pod of the call is constrained) or live -- the call must go to the method of the highest live rule (spread, then pod
affinity, then anti-affinity, then selectors, then the plain form) with every argument, positional or keyword, of the
expected value, dtype and None-ness.  The stand-in writes distinctive values into the node arrays the kernels update
in place (used, node_count, node_has, node_carries, node_matches) and returns a placement; those writes must reach the
rule objects and node.used_capacity, and the placement must come back.  The expectations are stated here from the
Engine's documented argument lists, not from snapshot's code."""
import datetime
import itertools

import numpy as np
import pytest
import torch

from kubernetes_acs_engine_autoscaler_b200 import capacity, snapshot
from kubernetes_acs_engine_autoscaler_b200.engine import padded_dims
from kubernetes_acs_engine_autoscaler_b200.kube import KubeResource

U64 = np.uint64
INT32_MAX = 2 ** 31 - 1
P, N = 5, 4


def _snap(x):
    """a comparable copy of an argument: tensors and arrays by kind, dtype and values, tuples element-wise"""
    if isinstance(x, torch.Tensor):
        return ("tensor", x.dtype, x.tolist())
    if isinstance(x, np.ndarray):
        return ("array", str(x.dtype), x.tolist())
    if isinstance(x, tuple):
        return tuple(_snap(a) for a in x)
    assert x is None or type(x) in (int, bool), "unexpected argument %r" % (x,)
    return x


def t(a, dtype):
    """the expected device tensor of host values `a`"""
    return ("tensor", dtype, np.asarray(a).tolist())


def m(a):
    """the expected device tensor of a uint64 mask array (passed as int64)"""
    return t(np.asarray(a, dtype=U64).view(np.int64), torch.int64)


def h(a):
    """the expected host array (passed as is)"""
    return ("array", str(a.dtype), a.tolist())


def _fill(d, values):
    d.copy_(torch.as_tensor(np.asarray(values)).to(d.dtype).reshape(d.shape))


def written_mask(n, salt):
    """distinctive uint64 values with the high bit set, so that a lost uint64 view shows"""
    return (np.arange(n, dtype=U64) * U64(0x101) + U64(salt)) | (U64(1) << U64(63))


def written_count(shape):
    return (np.arange(int(np.prod(shape)), dtype=np.int32) + 700).reshape(shape)


def written_used(shape):
    return np.arange(int(np.prod(shape)), dtype=np.float64).reshape(shape) + 1000.5


def placement(rows):
    """the stand-in's placement of `rows` pods: -1, 0, .., N - 1, -1, .."""
    return (np.arange(rows, dtype=np.int32) % (N + 1)) - 1


class RecordingEngine(object):
    """records (method, args, kwargs) of every rule call with the argument values at entry, then writes the in-place
    outputs and returns a placement (first fit) or a result dict (bin packing)"""
    device = torch.device("cpu")

    def __init__(self):
        self.calls = []
        self.raw = []

    def dev(self, a, dtype):
        if isinstance(a, torch.Tensor):
            return a.to(dtype=dtype).contiguous().clone()
        return torch.from_numpy(np.ascontiguousarray(a)).to(dtype=dtype).contiguous().clone()

    def _record(self, name, args, kwargs):
        self.calls.append((name, [_snap(a) for a in args], {k: _snap(v) for k, v in kwargs.items()}))
        self.raw.append((name, args, kwargs))

    # -- first fit over nodes: used [N, Dp] and the node masks are updated in place
    def _first_fit(self, name, args, kwargs, node_arrays):
        self._record(name, args, kwargs)
        req, pod_idx, used = args[0], args[1], args[4]
        _fill(used, written_used(used.shape))
        for d, salt in node_arrays:
            if d is not None:
                _fill(d, written_count(d.shape) if d.dtype == torch.int32 else
                      written_mask(d.shape[0], salt).view(np.int64))
        rows = req.shape[0] if pod_idx is None else pod_idx.shape[0]
        return torch.from_numpy(placement(rows)), torch.zeros(1, dtype=torch.int64)

    def first_fit_nodes(self, *args, **kwargs):
        return self._first_fit("first_fit_nodes", args, kwargs, ())

    def first_fit_nodes_sel(self, *args, **kwargs):
        return self._first_fit("first_fit_nodes_sel", args, kwargs, ())

    def first_fit_nodes_aa(self, *args, **kwargs):
        return self._first_fit("first_fit_nodes_aa", args, kwargs, ((args[7], 11), (args[8], 12)))

    def first_fit_nodes_pa(self, *args, **kwargs):
        aa = args[11:13] if len(args) > 9 else (None, None)
        return self._first_fit("first_fit_nodes_pa", args, kwargs, ((args[8], 13), (aa[0], 11), (aa[1], 12)))

    def first_fit_nodes_ts(self, *args, **kwargs):
        pa, aa = kwargs.get("pa") or (None,) * 4, kwargs.get("aa") or (None,) * 4
        return self._first_fit("first_fit_nodes_ts", args, kwargs, ((args[9], 0), (pa[3], 13), (aa[2], 11),
                                                                    (aa[3], 12)))

    # -- bin packing
    def _fulfill(self, name, args, kwargs):
        self._record(name, args, kwargs)
        Pp = args[0].shape[0]
        return {"new_size": np.array([3, 1]), "units_needed": np.array([2, -1]), "bins_opened": np.array([2, 0]),
                "acc_pool": torch.from_numpy(placement(Pp) % 2), "bin_of": torch.from_numpy(placement(Pp)),
                "num_unaccounted": 1, "evals": 9}

    def fulfill_pending(self, *args, **kwargs):
        return self._fulfill("fulfill_pending", args, kwargs)

    def fulfill_pending_sel(self, *args, **kwargs):
        return self._fulfill("fulfill_pending_sel", args, kwargs)

    def fulfill_pending_aa(self, *args, **kwargs):
        return self._fulfill("fulfill_pending_aa", args, kwargs)

    def fulfill_pending_pa(self, *args, **kwargs):
        return self._fulfill("fulfill_pending_pa", args, kwargs)

    def fulfill_pending_ts(self, *args, **kwargs):
        return self._fulfill("fulfill_pending_ts", args, kwargs)

    # -- node states: the admit forms set flag 2 on nodes 1 and 3 of node_flags (their last argument)
    def _admit(self, name, args):
        self._record(name, args, {})
        args[-1][1::2] |= 2
        return args[-1]

    def pending_admit(self, *args):
        return self._admit("pending_admit", args)

    def pending_admit_pa(self, *args):
        return self._admit("pending_admit_pa", args)

    def pending_admit_ts(self, *args):
        return self._admit("pending_admit_ts", args)

    def node_states(self, *args):
        self._record("node_states", args, {})
        return torch.arange(len(args[6]), dtype=torch.uint8).reshape(1, -1) + 4


@pytest.fixture
def eng(monkeypatch):
    e = RecordingEngine()
    monkeypatch.setattr(snapshot, "_engine", e)
    return e


# ---------------------------------------------------------------------------------------------------- the inputs
class Obj(object):
    def __init__(self, **kw):
        self.__dict__.update(kw)


def res(**raw):
    r = KubeResource()
    r.raw = dict(raw)
    return r


KEYS = ["cpu", "memory", "pods"]  # the sorted union of every vector's keys below
DP = padded_dims(len(KEYS))


def row(r):
    return [r.raw.get(k, 0.0) for k in KEYS] + [0.0] * (DP - len(KEYS))


def make_pods(infinite=False):
    a, b = res(cpu=1.0), res(cpu=0.5, memory=2.0)
    pods = [Obj(resources=x) for x in (a, b, a, b, a)]
    if infinite:
        pods[2] = Obj(resources=res(cpu=float("inf")))
    return pods


def make_nodes():
    cap_a, cap_b = res(cpu=8.0, memory=16.0, pods=10.0), res(cpu=4.0, memory=8.0)
    return [Obj(name="n%d" % n, capacity=(cap_a, cap_b)[n % 2], used_capacity=res(pods=float(n)))
            for n in range(N)]


def rule(kind, which):
    """a fresh rule object of `kind` (sel, aa, pa, ts): None when absent, else trivial or live"""
    if which == "absent":
        return None
    live = which == "live"
    if kind == "sel":
        if not live:
            return snapshot.SelectorClasses(np.zeros(P, np.uint8), np.ones(N, U64), np.ones(2, U64), 1)
        return snapshot.SelectorClasses(np.array([0, 1, 2, 1, 0], np.uint8), np.array([1, 3, 5, 2 ** 63 + 7], U64),
                                        np.array([3, 2 ** 63 + 6], U64), 3)
    if kind == "aa":
        if not live:
            return snapshot.AntiAffinity(np.zeros(P, U64), np.zeros(P, U64), np.zeros(N, U64), np.zeros(N, U64), [])
        return snapshot.AntiAffinity(np.array([1, 2, 0, 4, 2 ** 63], U64), np.array([2, 0, 1, 8, 5], U64),
                                     np.array([1, 0, 2, 2 ** 64 - 1], U64), np.array([0, 4, 0, 1], U64), ["t0", "t1"])
    if kind == "pa":
        if not live:
            return snapshot.PodAffinity(np.zeros(P, U64), np.zeros(P, U64), np.zeros(N, U64), [])
        return snapshot.PodAffinity(np.array([1, 0, 2, 2, 1], U64), np.array([1, 2, 3, 0, 2 ** 63 + 1], U64),
                                    np.array([0, 2, 1, 2 ** 63], U64), [frozenset(["s0"]), frozenset(["s1"])])
    if not live:
        return snapshot.TopologySpread(np.full(P, snapshot.NO_SPREAD_KEY, np.uint8), np.zeros(P, np.int32),
                                       np.zeros(P, U64), np.zeros((0, N), np.int32), np.zeros(N, U64),
                                       np.zeros(0, np.int32), [])
    return snapshot.TopologySpread(np.array([0, 1, snapshot.NO_SPREAD_KEY, 0, 1], np.uint8),
                                   np.array([1, 0, 0, 2, 1], np.int32), np.array([1, 2, 0, 3, 2 ** 63 + 2], U64),
                                   np.array([[0, 1, 2, 3], [4, 0, 5, 1]], np.int32), np.array([3, 1, 2, 2 ** 63], U64),
                                   np.array([INT32_MAX, 0], np.int32), ["k0", "k1"])


STATES = ("absent", "trivial", "live")
COMBOS = list(itertools.product(STATES, repeat=4))  # (sel, aa, pa, ts)


def _live(r):
    return r if r is not None and not r.trivial else None


def _copies(r):
    return None if r is None else {k: v.copy() for k, v in vars(r).items() if isinstance(v, np.ndarray)}


# ---------------------------------------------------------------------------------------------------- first fit
def expected_first_fit(pods, nodes, sel, aa, pa, ts):
    bad = [i for i, p in enumerate(pods) if not np.isfinite(row(p.resources)).all()]
    req = np.array([[0.0] * DP if i in bad else row(p.resources) for i, p in enumerate(pods)])
    ok_idx = np.array([i for i in range(len(pods)) if i not in bad], np.int32)
    cap = np.array([row(nodes[0].capacity), row(nodes[1].capacity)])
    used = np.array([row(n.used_capacity) for n in nodes])
    head = [t(req, torch.float64), t(ok_idx, torch.int32) if bad else None, t(cap, torch.float64),
            t(np.arange(N) % 2, torch.int32), t(used, torch.float64)]
    S = None if sel is None else [t(sel.pod_class, torch.uint8), m(sel.node_match), sel.classes]
    A = None if aa is None else [m(aa.pod_carries), m(aa.pod_matches), m(aa.node_carries), m(aa.node_matches)]
    PA = None if pa is None else [m(pa.pod_requires), m(pa.pod_self), m(pa.pod_matches), m(pa.node_has)]
    sel_kw = {} if S is None else dict(pod_class=S[0], node_match=S[1], classes=S[2])
    if ts is not None:
        return ("first_fit_nodes_ts", head + [len(ts.keys), t(ts.pod_key, torch.uint8), t(ts.pod_skew, torch.int32),
                                              m(ts.pod_matches), t(ts.node_count, torch.int32), m(ts.node_domain),
                                              h(ts.floor)],
                dict(pa=None if PA is None else tuple(PA), aa=None if A is None else tuple(A), **sel_kw))
    if pa is not None:
        return "first_fit_nodes_pa", head + PA + (A or []), sel_kw
    if aa is not None:
        return "first_fit_nodes_aa", head + A + (S or []), {}
    if sel is not None:
        return "first_fit_nodes_sel", head + S, {}
    return "first_fit_nodes", head, {}


@pytest.mark.parametrize("infinite", [False, True], ids=["finite", "infinite"])
@pytest.mark.parametrize("combo", COMBOS, ids=["-".join(c) for c in COMBOS])
def test_first_fit_nodes_dispatch(eng, combo, infinite):
    pods, nodes = make_pods(infinite), make_nodes()
    rules = [rule(kind, which) for kind, which in zip(("sel", "aa", "pa", "ts"), combo)]
    before = [_copies(r) for r in rules]
    old_used = [n.used_capacity for n in nodes]
    sel, aa, pa, ts = map(_live, rules)
    want = expected_first_fit(pods, nodes, sel, aa, pa, ts)
    placed = snapshot.first_fit_nodes(pods, nodes, classes=rules[0], anti_affinity=rules[1], pod_affinity=rules[2],
                                      topology_spread=rules[3])
    assert len(eng.calls) == 1
    name, args, kwargs = eng.calls[0]
    assert (name, args, kwargs) == want

    # the placement, mapped back through the list of finite pods
    ok = [i for i in range(P) if not (infinite and i == 2)]
    want_placed = np.full(P, -1, np.int32)
    want_placed[ok] = placement(len(ok))
    assert placed.tolist() == want_placed.tolist()
    # used: written back, with the node's keys plus those of the pods placed on it, on the nodes that took a pod
    written = written_used((N, DP))
    for n, node in enumerate(nodes):
        took = [pods[i] for i in range(P) if placed[i] == n]
        if not took:
            assert node.used_capacity is old_used[n]
            continue
        keys = set(old_used[n].raw).union(*(p.resources.raw for p in took))
        assert node.used_capacity.raw == {k: written[n, KEYS.index(k)] for k in keys}
    # the node masks: the stand-in's values on the rules the call took, untouched elsewhere
    for r, kept in zip(rules, before):
        if r is None:
            continue
        after = _copies(r)
        if r is ts:
            kept["node_count"] = written_count(r.node_count.shape)
        if r is pa:
            kept["node_has"] = written_mask(N, 13)
        if r is aa:
            kept["node_carries"], kept["node_matches"] = written_mask(N, 11), written_mask(N, 12)
        assert after.keys() == kept.keys()
        for k in kept:
            assert after[k].dtype == kept[k].dtype and after[k].tolist() == kept[k].tolist(), k


# ---------------------------------------------------------------------------------------------------- bin packing
def make_pools(monkeypatch):
    monkeypatch.setitem(capacity.RESOURCE_SPEC, "dispatch-a", res(cpu=6.0, memory=12.0))
    monkeypatch.setitem(capacity.RESOURCE_SPEC, "dispatch-b", res(cpu=3.0, pods=4.0))
    return [Obj(name="pool-a", instance_type="dispatch-a", actual_capacity=2, max_size=2 ** 40),
            Obj(name="pool-b", instance_type="dispatch-b", actual_capacity=0, max_size=7)]


def expected_fulfill(pods, pools, sel, aa, pa, ts, present):
    unit = np.array([row(capacity.RESOURCE_SPEC[p.instance_type]) for p in pools])
    head = [t([row(p.resources) for p in pods], torch.float64), P + 2, h(unit),
            h(np.array([2, 0], np.int32)), h(np.array([INT32_MAX, 7], np.int32)), h(np.array([0, 1], np.uint8)), 5]
    S = None if sel is None else [t(sel.pod_class, torch.uint8), h(sel.pool_match), sel.classes]
    A = None if aa is None else [m(aa.pod_carries), m(aa.pod_matches)]
    PA = None if pa is None else [m(pa.pod_requires), m(pa.pod_self), m(pa.pod_matches)]
    if ts is not None:
        sel_kw = {} if S is None else dict(pod_class=S[0], pool_match=S[1], classes=S[2])
        return ("fulfill_pending_ts", head + [len(ts.keys), t(ts.pod_key, torch.uint8), t(ts.pod_skew, torch.int32),
                                              m(ts.pod_matches)],
                dict(pa=None if PA is None else tuple(PA), present=0 if pa is None else present,
                     aa=None if A is None else tuple(A), **sel_kw))
    if pa is not None:
        return "fulfill_pending_pa", head + PA + [present] + (A or [None, None]) + (S or []), {}
    if aa is not None:
        return "fulfill_pending_aa", head + A + (S or []), {}
    if sel is not None:
        return "fulfill_pending_sel", head + S, {}
    return "fulfill_pending", head, {}


@pytest.mark.parametrize("combo", COMBOS, ids=["-".join(c) for c in COMBOS])
def test_fulfill_dispatch(eng, monkeypatch, combo):
    pods, pools = make_pods(), make_pools(monkeypatch)
    rules = [rule(kind, which) for kind, which in zip(("sel", "aa", "pa", "ts"), combo)]
    before = [_copies(r) for r in rules]
    sel, aa, pa, ts = map(_live, rules)
    # the nodes hold s1 (bit 1) and a signature this call does not have
    want = expected_fulfill(pods, pools, sel, aa, pa, ts, present=2)
    out = snapshot.fulfill(pods, P + 2, pools, {"pool-b"}, 5, classes=rules[0], anti_affinity=rules[1],
                           pod_affinity=rules[2], affinity_present={frozenset(["s1"]), frozenset(["other"])},
                           topology_spread=rules[3])
    assert len(eng.calls) == 1
    assert eng.calls[0] == want
    assert isinstance(out["acc_pool"], np.ndarray) and out["acc_pool"].tolist() == (placement(P) % 2).tolist()
    assert isinstance(out["bin_of"], np.ndarray) and out["bin_of"].tolist() == placement(P).tolist()
    assert out["new_size"].tolist() == [3, 1] and out["units_needed"].tolist() == [2, -1]
    assert (out["num_unaccounted"], out["evals"]) == (1, 9)
    for r, kept in zip(rules, before):  # the bin pass updates no rule array
        if r is not None:
            assert {k: (v.dtype, v.tolist()) for k, v in _copies(r).items()} == \
                {k: (v.dtype, v.tolist()) for k, v in kept.items()}


# ---------------------------------------------------------------------------------------------------- node states
class StatePod(Obj):
    """a kube-proxy pod: pod_flags reads its name and is_mirrored() only"""

    def is_mirrored(self):
        return False


def admit_table(form, aa, node_match):
    """a PendingAdmit of the acsfit_pending_admit (form "aa"), _pa or _ts table, over R = 3 rows and U = 2 signatures"""
    rc, rm = (np.array([1, 2 ** 63, 4], U64), np.array([2, 0, 2 ** 64 - 1], U64)) if aa else (None, None)
    adm = snapshot.PendingAdmit(rc, rm, np.array([1, 3, 2 ** 63 + 1, 0], U64) if node_match else None,
                                np.array([0, 2], np.uint8), np.array([1, 2 ** 63], U64) if aa else None,
                                np.array([4, 1], U64) if aa else None)
    if form in ("pa", "ts_pa"):
        adm.row_has, adm.sig_need = np.array([0, 2 ** 63 + 3, 1], U64), np.array([1, 0], U64)
    if form.startswith("ts"):
        adm.sig_key, adm.sig_skew = np.array([snapshot.NO_SPREAD_KEY, 1], np.uint8), np.array([0, 2], np.int32)
        adm.node_count = np.array([[0, 1, 2, 3], [3, 2, 1, 0]], np.int32)
        adm.node_domain, adm.floor = np.array([3, 0, 1, 2 ** 63], U64), np.array([INT32_MAX, 1], np.int32)
    return adm


def opt(a, f):
    return None if a is None else f(a)


ADMITS = [("aa", True, False), ("aa", True, True), ("pa", True, True), ("pa", False, False), ("ts", True, True),
          ("ts", False, False), ("ts_pa", True, False), ("ts_pa", False, True)]


@pytest.mark.parametrize("form,aa,node_match", ADMITS)
def test_node_states_admit_dispatch(eng, form, aa, node_match):
    when = datetime.datetime(2026, 1, 1, tzinfo=datetime.timezone.utc)
    nodes = [Obj(name="n%d" % n, capacity=res(cpu=4.0), unschedulable=n == 2, creation_time=when) for n in range(N)]
    lists = [[StatePod(name="kube-proxy-%d-%d" % (n, k), resources=res(cpu=0.5)) for k in range(c)]
             for n, c in enumerate((2, 0, 1, 0))]
    adm = admit_table(form, aa, node_match)
    st = snapshot.node_states(nodes, lists, True, 1800, admit=adm)
    assert [c[0] for c in eng.calls][1:] == ["node_states"]
    name, args, kwargs = eng.calls[0]
    flags0 = t(np.array([0, 0, 1, 0], np.uint8), torch.uint8)
    head = [t([0, 2, 2, 3, 3], torch.int64), opt(adm.row_carries, m), opt(adm.row_matches, m)]
    tail = [h(adm.sig_class), opt(adm.sig_carries, h), opt(adm.sig_matches, h)]
    if form == "aa":
        want = "pending_admit", head + [opt(adm.node_match, m)] + tail + [flags0]
    elif form == "pa":
        want = "pending_admit_pa", head + [m(adm.row_has), opt(adm.node_match, m)] + tail + [h(adm.sig_need), flags0]
    else:
        want = ("pending_admit_ts", head + [opt(adm.row_has, m), opt(adm.node_match, m)] + tail +
                [opt(adm.sig_need, h), h(adm.sig_key), h(adm.sig_skew), 2, t(adm.node_count, torch.int32),
                 m(adm.node_domain), h(adm.floor), flags0])
    assert (name, args, kwargs) == want + ({},)
    # node_states classifies with the flags the admission wrote, in the same buffer
    assert eng.raw[1][1][6] is eng.raw[0][1][-1]
    assert eng.calls[1][1][6] == t(np.array([0, 2, 1, 2], np.uint8), torch.uint8)
    assert st.tolist() == [4, 5, 6, 7]
