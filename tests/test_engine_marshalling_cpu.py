"""Engine argument passing, without a GPU: a recording stand-in replaces libacsfit.so, and every public entry point
is checked for the acsfit_* function it calls, every scalar it passes, and what each pointer -- plain or a field of a
rule struct -- points at: a named input array (or the array converted from it), or a fresh output.

Pointers are resolved while the call is in flight, so an array the engine converted and then let go before the C
call returned (a use-after-free in the real library) fails here: every array made by engine._np is tracked by a weak
reference, and a pointer to one that is already gone is an error."""
import ctypes
import weakref

import numpy as np
import pytest
import torch

from kubernetes_acs_engine_autoscaler_b200 import _native
from kubernetes_acs_engine_autoscaler_b200 import engine as engine_mod
from kubernetes_acs_engine_autoscaler_b200.engine import Engine

CTX, STREAM = 0xC7C0, 0x5700
U64 = 0xFFFFFFFFFFFFFFFF
P, D, N, T, K = 3, 2, 4, 2, 2


def S(cls, *fields):
    """expected struct: field values in declaration order (labels for pointers, ints for counts)"""
    return (cls, dict(zip([f for f, _ in cls._fields_], fields)))


def _addr(a):
    if isinstance(a, ctypes.c_void_p):
        return a.value
    if type(a).__name__ == "CArgObject":  # ctypes.byref(x) passed as is
        return ctypes.addressof(a._obj)
    raise TypeError("unexpected argument %r" % (a,))


class FakeLib(object):
    """records each acsfit_* call as a list of tokens: ints / bytes / None as passed, pointers as labels"""

    def __init__(self):
        self.calls = []
        self.known = {CTX: "ctx", STREAM: "stream"}  # address -> label of the test's own arrays
        self.ids = {}  # id -> label, to name what engine._np converts
        self.tracked = []  # (weakref, address, label) of every array engine._np returned
        self.structs = {}  # position -> struct class, for the next call
        self.effect = None  # callable(args) run inside the call (writes the library's outputs)

    def name(self, label, a):
        self.known[a.data_ptr() if isinstance(a, torch.Tensor) else a.ctypes.data] = label
        self.ids[id(a)] = label
        return a

    def track(self, src, out):
        self.tracked.append((weakref.ref(out), out.ctypes.data, self.ids.get(id(src), "?")))

    def label(self, addr):
        if addr is None:
            return None
        if addr in self.known:
            return self.known[addr]
        hits = [(ref(), lab) for ref, a, lab in self.tracked if a == addr]
        live = [lab for obj, lab in hits if obj is not None]
        if live:  # the first conversion names it (a later _np of the converted array is a no-op)
            return live[0]
        assert not hits, "pointer to %s, which was freed before the call returned" % hits[0][1]
        return ("out", addr)

    def token(self, i, a):
        if a is None or isinstance(a, (int, bytes)):
            return a
        addr = _addr(a)
        cls = self.structs.get(i)
        if cls is None:
            return self.label(addr)
        s = cls.from_address(addr)
        return (cls, {f: self.label(getattr(s, f)) if t is ctypes.c_void_p else getattr(s, f)
                      for f, t in cls._fields_})

    def __getattr__(self, name):
        if not name.startswith("acsfit_"):
            raise AttributeError(name)

        def call(*args):
            self.calls.append((name, [self.token(i, a) for i, a in enumerate(args)]))
            if self.effect is not None:
                self.effect(args)
            return 0
        return call


@pytest.fixture
def eng(monkeypatch):
    lib = FakeLib()
    np_ = engine_mod._np

    def tracking_np(a, dtype):
        out = np_(a, dtype)
        lib.track(a, out)
        return out
    monkeypatch.setattr(engine_mod, "_np", tracking_np)
    e = object.__new__(Engine)
    e._lib = lib
    e._ctx = ctypes.c_void_p(CTX)
    e.device = torch.device("cpu")
    e._stream = lambda: ctypes.c_void_p(STREAM)
    yield e
    e._ctx = ctypes.c_void_p()  # nothing to destroy


def calls_of(e, outputs=None):
    """the recorded calls with outputs named: `outputs` label -> returned array; any other pointer is "fresh"
    (a buffer the engine made for the call), and fresh buffers are distinct within a call"""
    outputs = outputs or {}
    by_addr = {(v.data_ptr() if isinstance(v, torch.Tensor) else v.ctypes.data): k for k, v in outputs.items()}
    res = []
    for name, toks in e._lib.calls:
        fresh = []

        def fix(t):
            if isinstance(t, tuple) and t[0] == "out":
                if t[1] in by_addr:
                    return by_addr[t[1]]
                fresh.append(t[1])
                return "fresh"
            if isinstance(t, tuple):
                return (t[0], {k: fix(v) for k, v in t[1].items()})
            return t
        toks = [fix(t) for t in toks]
        assert len(set(fresh)) == len(fresh), "%s: two outputs share a buffer" % name
        res.append((name, toks))
    e._lib.calls = []
    return res


def expect_call(e, expected, outputs=None):
    got = calls_of(e, outputs)
    assert [n for n, _ in got] == [n for n, _ in expected]
    for (name, toks), (_, want) in zip(got, expected):
        assert len(toks) == len(want), name
        for i, (g, w) in enumerate(zip(toks, want)):
            assert g == w, "%s argument %d: %r, expected %r" % (name, i, g, w)


def struct_positions(e, want):
    e._lib.structs = {i: w[0] for i, w in enumerate(want) if isinstance(w, tuple)}


def write(addr_arg, ctype, values):
    """an effect writing `values` to the buffer a call argument points at"""
    def eff(args):
        a = args[addr_arg]
        if a is None:
            return
        arr = (ctype * len(values)).from_address(_addr(a))
        arr[:] = values
    return eff


# ---------------------------------------------------------------------------------------------------- inputs
def dev_f64(lib, label, *shape):
    return lib.name(label, torch.arange(int(np.prod(shape)), dtype=torch.float64).reshape(shape).contiguous())


def dev(lib, label, n, dtype):
    return lib.name(label, torch.zeros(n, dtype=dtype))


def pools(lib):
    """host pool arrays, given as lists so the engine converts them"""
    return (lib.name("unit", np.arange(T * D, dtype=np.float64)), [3, 4], [5, 6], [0, 1])


def pool_inputs(lib, args):
    """name the arrays engine._np makes from the pool lists (by the id of each list)"""
    for label, a in zip(("pool_actual", "pool_max", "pool_ignored"), args[1:]):
        lib.ids[id(a)] = label


FULFILL_KEYS = {"new_size", "units_needed", "bins_opened", "acc_pool", "bin_of", "num_unaccounted", "evals"}
SCALE_UP_KEYS = {"feasible", "placed", "acc_pool", "new_size", "units_needed", "bins_opened", "n_to_schedule",
                 "n_pending", "num_unaccounted", "decisions"}
FULFILL_OUT = ["new_size", "units_needed", "bins_opened", "acc_pool", "bin_of", "fresh", "fresh"]
SCALE_UP_OUT = ["feasible", "placed", "new_size", "units_needed", "bins_opened", "acc_pool", "fresh"]


def fulfill_outputs(res):
    return {k: res[k] for k in ("new_size", "units_needed", "bins_opened", "acc_pool", "bin_of")}


def scale_up_outputs(res):
    return {k: res[k] for k in ("feasible", "placed", "new_size", "units_needed", "bins_opened", "acc_pool")}


def run_fulfill(e, method, want, *extra, **kw):
    """a fulfill_pending* call: unacc / evals written by the library come back as num_unaccounted / evals"""
    lib = e._lib
    req = dev_f64(lib, "req", P, D)
    pl = pools(lib)
    pool_inputs(lib, pl)
    struct_positions(e, want)
    n = len(want)
    effects = [write(n - 3, ctypes.c_int64, [7]), write(n - 2, ctypes.c_uint64, [9])]
    lib.effect = lambda args: [f(args) for f in effects]
    res = getattr(e, method)(req, 5, *pl, 2, *extra, **kw)
    assert set(res) == FULFILL_KEYS
    assert res["num_unaccounted"] == 7 and res["evals"] == 9
    assert res["new_size"].shape == (T,) and res["acc_pool"].shape == (P,)
    expect_call(e, [("acsfit_" + method, want)], fulfill_outputs(res))


def fulfill_head():
    return ["ctx", "req", P, 5, D, "unit", "pool_actual", "pool_max", "pool_ignored", T, 2]


def first_fit_head():
    return ["ctx", "req", P, "pod_idx", 2, D, "cap_type", "node_type", "used", N]


def first_fit_inputs(lib):
    return (dev_f64(lib, "req", P, D), dev(lib, "pod_idx", 2, torch.int32), dev_f64(lib, "cap_type", K, D),
            dev(lib, "node_type", N, torch.int32), dev_f64(lib, "used", N, D))


def run_first_fit(e, method, want, *extra, **kw):
    lib = e._lib
    ins = first_fit_inputs(lib)
    struct_positions(e, want)
    placed, decisions = getattr(e, method)(*ins, *extra, **kw)
    assert placed.shape == (2,) and placed.dtype == torch.int32 and decisions.shape == (1,)
    expect_call(e, [("acsfit_" + method, want)], {"placed": placed, "decisions": decisions})


# ---------------------------------------------------------------------------------------------------- plain forms
def test_feasible_mask(eng):
    lib = eng._lib
    req, unit = dev_f64(lib, "req", P, D), dev_f64(lib, "unit", T, D)
    mask, evals = eng.feasible_mask(req, unit)
    expect_call(eng, [("acsfit_feasible_mask", ["ctx", "req", P, D, "unit", T, "mask", "evals", "stream"])],
                {"mask": mask, "evals": evals})


def test_occupancy(eng):
    lib = eng._lib
    args = (dev(lib, "row_ptr", N + 1, torch.int64), dev(lib, "run_idx", 3, torch.int32),
            dev_f64(lib, "req_run", 3, D), dev_f64(lib, "used", N, D))
    assert eng.occupancy(*args) is args[3]
    expect_call(eng, [("acsfit_occupancy", ["ctx", "row_ptr", "run_idx", "req_run", N, D, "used", "stream"])])


def test_first_fit_nodes(eng):
    run_first_fit(eng, "first_fit_nodes", first_fit_head() + ["placed", "decisions", "stream"])


def test_fulfill_pending(eng):
    run_fulfill(eng, "fulfill_pending", fulfill_head() + FULFILL_OUT + ["stream"])


def test_node_states(eng):
    lib = eng._lib
    args = (dev(lib, "row_ptr", N + 1, torch.int64), dev(lib, "run_idx", 3, torch.int32),
            dev_f64(lib, "req_run", 3, D), dev(lib, "flags_run", 3, torch.uint8), dev_f64(lib, "cap_type", K, D),
            dev(lib, "node_type", N, torch.int32), dev(lib, "node_flags", N, torch.uint8),
            dev(lib, "node_age", N, torch.int64))
    thr = [600, 1800]
    lib.ids[id(thr)] = "idle_thresholds"
    out = eng.node_states(*args, True, thr)
    assert out.shape == (2, N) and out.dtype == torch.uint8
    expect_call(eng, [("acsfit_node_states", ["ctx", "row_ptr", "run_idx", "req_run", "flags_run", "cap_type",
                                              "node_type", "node_flags", "node_age", N, D, 1, "idle_thresholds", 2,
                                              "out", "stream"])], {"out": out})


def admit_inputs(lib):
    return (dev(lib, "row_ptr", N + 1, torch.int64), dev(lib, "run_carries", 3, torch.int64),
            dev(lib, "run_matches", 3, torch.int64))


def named(lib, label, values):
    """a host list the engine converts: the array made from it carries `label`"""
    lib.ids[id(values)] = label
    return values


def test_pending_admit(eng):
    lib = eng._lib
    row_ptr, rc, rm = admit_inputs(lib)
    node_match, node_flags = dev(lib, "node_match", N, torch.int64), dev(lib, "node_flags", N, torch.uint8)
    got = eng.pending_admit(row_ptr, rc, rm, node_match, named(lib, "sig_class", [0, 1]),
                            named(lib, "sig_carries", [1, 2]), named(lib, "sig_matches", [3, 4]), node_flags)
    assert got is node_flags
    expect_call(eng, [("acsfit_pending_admit", ["ctx", "row_ptr", "run_carries", "run_matches", N, "node_match",
                                                "sig_class", "sig_carries", "sig_matches", 2, "node_flags",
                                                "stream"])])


@pytest.mark.parametrize("with_aa", [True, False])
def test_pending_admit_pa(eng, with_aa):
    lib = eng._lib
    row_ptr, rc, rm = admit_inputs(lib)
    run_has, node_flags = dev(lib, "run_has", 3, torch.int64), dev(lib, "node_flags", N, torch.uint8)
    sc, sm = (named(lib, "sig_carries", [1, 2]), named(lib, "sig_matches", [3, 4])) if with_aa else (None, None)
    if not with_aa:
        rc = rm = None
    got = eng.pending_admit_pa(row_ptr, rc, rm, run_has, None, named(lib, "sig_class", [0, 1]), sc, sm,
                               named(lib, "sig_need", [0, 8]), node_flags)
    assert got is node_flags
    aa = ["run_carries", "run_matches"] if with_aa else [None, None]
    saa = ["sig_carries", "sig_matches"] if with_aa else [None, None]
    expect_call(eng, [("acsfit_pending_admit_pa", ["ctx", "row_ptr"] + aa + ["run_has", N, None, "sig_class"] + saa +
                       ["sig_need", 2, "node_flags", "stream"])])


@pytest.mark.parametrize("with_rules", [True, False])
def test_pending_admit_ts(eng, with_rules):
    lib = eng._lib
    row_ptr, rc, rm = admit_inputs(lib)
    run_has = dev(lib, "run_has", 3, torch.int64)
    node_count, node_domain = dev(lib, "node_count", 2 * N, torch.int32), dev(lib, "node_domain", N, torch.int64)
    floor = lib.name("floor", np.array([0, 1], dtype=np.int32))
    node_flags = dev(lib, "node_flags", N, torch.uint8)
    if with_rules:
        sc, sm = named(lib, "sig_carries", [1, 2]), named(lib, "sig_matches", [3, 4])
        need = named(lib, "sig_need", [0, 8])
    else:
        rc = rm = run_has = sc = sm = need = None
    want = ["ctx", "row_ptr", "run_carries", "run_matches", "run_has", N, None, "sig_class", "sig_carries",
            "sig_matches", "sig_need", "sig_key", "sig_skew", 2,
            S(_native.TopologySpread, None, None, None, "node_count", "node_domain", "floor", 2), "node_flags",
            "stream"]
    if not with_rules:
        want = [None if w in ("run_carries", "run_matches", "run_has", "sig_carries", "sig_matches", "sig_need")
                else w for w in want]
    struct_positions(eng, want)
    got = eng.pending_admit_ts(row_ptr, rc, rm, run_has, None, named(lib, "sig_class", [0, 1]), sc, sm, need,
                               named(lib, "sig_key", [0, 0xFF]), named(lib, "sig_skew", [1, 0]), 2, node_count,
                               node_domain, floor, node_flags)
    assert got is node_flags
    expect_call(eng, [("acsfit_pending_admit_ts", want)])


def test_maintain_actions(eng):
    lib = eng._lib
    state, node_pool = dev(lib, "state", N, torch.uint8), dev(lib, "node_pool", N, torch.int32)
    s, action = eng.maintain_actions(state, node_pool, named(lib, "budget0", [1, 0]),
                                     named(lib, "pool_scalable", [1, 1]), True)
    assert s is state and action.shape == (N,)
    expect_call(eng, [("acsfit_maintain_actions", ["ctx", "state", "node_pool", N, "budget0", "pool_scalable", T, 1,
                                                   "action", "stream"])], {"action": action})


def scale_up_inputs(lib, host):
    if host:
        def f64(label, *shape):
            return lib.name(label, np.arange(int(np.prod(shape)), dtype=np.float64).reshape(shape))
        node_type = lib.name("node_type", np.zeros(N, dtype=np.int32))
    else:
        def f64(label, *shape):
            return dev_f64(lib, label, *shape)
        node_type = dev(lib, "node_type", N, torch.int32)
    req = f64("req", P, D)
    unit_all, unit_ordered = [lib.name(k, np.arange(T * D, dtype=np.float64)) for k in ("unit_all", "unit_ordered")]
    pl = [3, 4], [5, 6], [0, 1]
    for label, a in zip(("pool_actual", "pool_max", "pool_ignored"), pl):
        lib.ids[id(a)] = label
    return (req, unit_all, unit_ordered) + pl + (2, f64("cap_type", K, D), node_type, f64("used", N, D))


def run_scale_up(e, method, want, *extra, host=False, **kw):
    """a scale_up* call: the counters written by the library come back as the four counts"""
    lib = e._lib
    struct_positions(e, want)
    lib.effect = write(len(want) - (1 if host else 2), ctypes.c_uint64, [11, 12, 13, 14])
    res = getattr(e, method)(*scale_up_inputs(lib, host), *extra, **kw)
    assert set(res) == SCALE_UP_KEYS
    assert (res["n_to_schedule"], res["n_pending"], res["num_unaccounted"], res["decisions"]) == (11, 12, 13, 14)
    expect_call(e, [("acsfit_" + method, want)], scale_up_outputs(res))
    return res


SCALE_UP_HEAD = ["ctx", "req", P, D, "unit_all", "unit_ordered", "pool_actual", "pool_max", "pool_ignored", T, 2,
                 "cap_type"]


def test_scale_up(eng):
    run_scale_up(eng, "scale_up", SCALE_UP_HEAD + ["node_type", "used", N] + SCALE_UP_OUT + ["stream"])


@pytest.mark.parametrize("given_out", [False, True])
def test_scale_up_host(eng, given_out):
    lib = eng._lib
    want = SCALE_UP_HEAD + [K, "node_type", "used", N] + SCALE_UP_OUT
    out = None
    if given_out:
        out = {"feasible": lib.name("out_feasible", np.empty(P, np.uint8)),
               "placed": lib.name("out_placed", np.empty(P, np.int32)),
               "acc_pool": lib.name("out_acc_pool", np.empty(P, np.int32))}
        want = [{"feasible": "out_feasible", "placed": "out_placed", "acc_pool": "out_acc_pool"}.get(w, w)
                for w in want]
    res = run_scale_up(eng, "scale_up_host", want, host=True, out=out)
    if given_out:
        assert all(res[k] is out[k] for k in out)


def test_occupancy_host(eng):
    lib = eng._lib
    row_ptr = lib.name("row_ptr", np.array([0, 1, 2, 3, 3], dtype=np.int64))
    run_idx = lib.name("run_idx", np.array([0, 1, 2], dtype=np.int32))
    req_run = lib.name("req_run", np.arange(3 * D, dtype=np.float64))
    used = lib.name("used", np.zeros((N, D)))
    assert eng.occupancy_host(row_ptr, run_idx, req_run, used) is used
    assert eng.occupancy_host(row_ptr, None, req_run, used) is used
    expect_call(eng, [("acsfit_occupancy_host", ["ctx", "row_ptr", "run_idx", "req_run", 3, N, D, "used"]),
                      ("acsfit_occupancy_host", ["ctx", "row_ptr", None, "req_run", 3, N, D, "used"])])


def test_maintain_host(eng):
    lib = eng._lib
    args = [named(lib, k, v) for k, v in (("row_ptr", [0, 1, 2, 3, 3]), ("run_idx", [0, 1, 2]),
                                        ("req_run", [[1.0, 2.0]] * 3), ("flags_run", [0, 0, 1]),
                                        ("cap_type", [[4.0, 4.0]] * K), ("node_type", [0, 1, 0, 1]),
                                        ("node_flags", [0] * N), ("node_age", [10] * N), ("node_pool", [0, 1, 0, 1]))]
    budget0, scalable = named(lib, "budget0", [1, 1]), named(lib, "pool_scalable", [1, 0])
    state, action = eng.maintain_host(*args, False, 1800, budget0, scalable, True)
    assert state.shape == action.shape == (N,)
    expect_call(eng, [("acsfit_maintain_host", ["ctx", "row_ptr", "run_idx", "req_run", "flags_run", 3, "cap_type", K,
                                                "node_type", "node_flags", "node_age", "node_pool", N, D, 0, 1800,
                                                "budget0", "pool_scalable", T, 1, "state", "action"])],
                {"state": state, "action": action})


# ---------------------------------------------------------------------------------------------------- rule forms
def sel_inputs(lib, nodes=True):
    pod_class = dev(lib, "pod_class", P, torch.uint8)
    return pod_class, (dev(lib, "node_match", N, torch.int64) if nodes else None)


def pool_mask(lib, label):
    return named(lib, label, [1, 3])


def test_feasible_mask_sel(eng):
    lib = eng._lib
    req, unit = dev_f64(lib, "req", P, D), dev_f64(lib, "unit", T, D)
    pod_class, _ = sel_inputs(lib, nodes=False)
    want = ["ctx", "req", P, D, "unit", T, S(_native.Selectors, "pod_class", None, "pool_match", None, 3), "mask",
            "evals", "stream"]
    struct_positions(eng, want)
    mask, evals = eng.feasible_mask_sel(req, unit, pod_class, pool_mask(lib, "pool_match"), 3)
    expect_call(eng, [("acsfit_feasible_mask_sel", want)], {"mask": mask, "evals": evals})


def test_first_fit_nodes_sel(eng):
    pod_class, node_match = sel_inputs(eng._lib)
    run_first_fit(eng, "first_fit_nodes_sel", first_fit_head() + [
        S(_native.Selectors, "pod_class", "node_match", None, None, 3), "placed", "decisions", "stream"],
        pod_class, node_match, 3)


def test_fulfill_pending_sel(eng):
    pod_class, _ = sel_inputs(eng._lib, nodes=False)
    run_fulfill(eng, "fulfill_pending_sel", fulfill_head() + [
        S(_native.Selectors, "pod_class", None, None, "pool_match", 3)] + FULFILL_OUT + ["stream"],
        pod_class, pool_mask(eng._lib, "pool_match"), 3)


def test_scale_up_sel(eng):
    lib = eng._lib
    pod_class, node_match = sel_inputs(lib)
    run_scale_up(eng, "scale_up_sel", SCALE_UP_HEAD + ["node_type", "used", N] + [
        S(_native.Selectors, "pod_class", "node_match", "pool_match_all", "pool_match_ordered", 3)] + SCALE_UP_OUT +
        ["stream"], pod_class, node_match, pool_mask(lib, "pool_match_all"), pool_mask(lib, "pool_match_ordered"), 3)


def test_scale_up_sel_host(eng):
    lib = eng._lib
    run_scale_up(eng, "scale_up_sel_host", SCALE_UP_HEAD + [K, "node_type", "used", N] + [
        S(_native.Selectors, "pod_class", "node_match", "pool_match_all", "pool_match_ordered", 3)] + SCALE_UP_OUT,
        named(lib, "pod_class", [0, 1, 2]), named(lib, "node_match", [1, 3, 5, 7]), pool_mask(lib, "pool_match_all"),
        pool_mask(lib, "pool_match_ordered"), 3, host=True)


def aa_inputs(lib, nodes=True):
    names = ("pod_carries", "pod_matches_aa") + (("node_carries", "node_matches") if nodes else ())
    return [dev(lib, k, P if k.startswith("pod") else N, torch.int64) for k in names]


def pa_inputs(lib, nodes=True):
    names = ("pod_requires", "pod_self", "pod_matches_pa") + (("node_has",) if nodes else ())
    return [dev(lib, k, P if k.startswith("pod") else N, torch.int64) for k in names]


def ts_inputs(lib):
    return (dev(lib, "pod_key", P, torch.uint8), dev(lib, "pod_skew", P, torch.int32),
            dev(lib, "pod_matches_ts", P, torch.int64))


SEL_NODES = S(_native.Selectors, "pod_class", "node_match", None, None, 3)
SEL_POOLS = S(_native.Selectors, "pod_class", None, None, "pool_match", 3)
AA_NODES = S(_native.AntiAffinity, "pod_carries", "pod_matches_aa", "node_carries", "node_matches")
AA_PODS = S(_native.AntiAffinity, "pod_carries", "pod_matches_aa", None, None)
PA_NODES = S(_native.PodAffinity, "pod_requires", "pod_self", "pod_matches_pa", "node_has")
PA_PODS = S(_native.PodAffinity, "pod_requires", "pod_self", "pod_matches_pa", None)


@pytest.mark.parametrize("with_sel", [False, True])
def test_first_fit_nodes_aa(eng, with_sel):
    lib = eng._lib
    kw = {}
    if with_sel:
        kw["pod_class"], kw["node_match"] = sel_inputs(lib)
        kw["classes"] = 3
    run_first_fit(eng, "first_fit_nodes_aa", first_fit_head() + [SEL_NODES if with_sel else None, AA_NODES, "placed",
                                                                 "decisions", "stream"], *aa_inputs(lib), **kw)


@pytest.mark.parametrize("with_sel", [False, True])
def test_fulfill_pending_aa(eng, with_sel):
    lib = eng._lib
    kw = {}
    if with_sel:
        kw["pod_class"], _ = sel_inputs(lib, nodes=False)
        kw["pool_match"], kw["classes"] = pool_mask(lib, "pool_match"), 3
    run_fulfill(eng, "fulfill_pending_aa", fulfill_head() + [SEL_POOLS if with_sel else None, AA_PODS] + FULFILL_OUT +
                ["stream"], *aa_inputs(lib, nodes=False), **kw)


@pytest.mark.parametrize("with_rules", [False, True])
def test_first_fit_nodes_pa(eng, with_rules):
    lib = eng._lib
    kw = {}
    if with_rules:
        pc, pm, nc, nm = aa_inputs(lib)
        kw.update(pod_carries=pc, pod_matches_aa=pm, node_carries=nc, node_matches=nm, classes=3)
        kw["pod_class"], kw["node_match"] = sel_inputs(lib)
    run_first_fit(eng, "first_fit_nodes_pa", first_fit_head() + [
        SEL_NODES if with_rules else None, AA_NODES if with_rules else None, PA_NODES, "placed", "decisions",
        "stream"], *pa_inputs(lib), **kw)


@pytest.mark.parametrize("with_rules", [False, True])
def test_fulfill_pending_pa(eng, with_rules):
    lib = eng._lib
    kw = {}
    if with_rules:
        kw["pod_carries"], kw["pod_matches_aa"] = aa_inputs(lib, nodes=False)
        kw["pod_class"], _ = sel_inputs(lib, nodes=False)
        kw["pool_match"], kw["classes"] = pool_mask(lib, "pool_match"), 3
    run_fulfill(eng, "fulfill_pending_pa", fulfill_head() + [
        SEL_POOLS if with_rules else None, AA_PODS if with_rules else None, PA_PODS, U64 if with_rules else 0] +
        FULFILL_OUT + ["stream"], *pa_inputs(lib, nodes=False), present=-1 if with_rules else 0, **kw)


@pytest.mark.parametrize("with_rules", [False, True])
def test_first_fit_nodes_ts(eng, with_rules):
    lib = eng._lib
    node_count, node_domain = dev(lib, "node_count", 2 * N, torch.int32), dev(lib, "node_domain", N, torch.int64)
    floor = lib.name("floor", np.array([0, 1], dtype=np.int32))
    kw = {}
    if with_rules:
        kw["pa"], kw["aa"] = tuple(pa_inputs(lib)), tuple(aa_inputs(lib))
        kw["pod_class"], kw["node_match"] = sel_inputs(lib)
        kw["classes"] = 3
    ts = S(_native.TopologySpread, "pod_key", "pod_skew", "pod_matches_ts", "node_count", "node_domain", "floor", 2)
    rules = [SEL_NODES, AA_NODES, PA_NODES] if with_rules else [None] * 3
    run_first_fit(eng, "first_fit_nodes_ts", first_fit_head() + rules + [ts, "placed", "decisions", "stream"], 2,
                  *ts_inputs(lib), node_count, node_domain, floor, **kw)


@pytest.mark.parametrize("with_rules", [False, True])
def test_fulfill_pending_ts(eng, with_rules):
    lib = eng._lib
    kw = {}
    if with_rules:
        kw["pa"], kw["aa"] = tuple(pa_inputs(lib, nodes=False)), tuple(aa_inputs(lib, nodes=False))
        kw["pod_class"], _ = sel_inputs(lib, nodes=False)
        kw["pool_match"], kw["classes"], kw["present"] = pool_mask(lib, "pool_match"), 3, (1 << 64) + 5
    # the empty floor the engine passes when fulfill has no nodes: a fresh array, not one of the inputs
    ts = S(_native.TopologySpread, "pod_key", "pod_skew", "pod_matches_ts", None, None, "fresh", 2)
    rules = [SEL_POOLS, AA_PODS, PA_PODS, 5] if with_rules else [None, None, None, 0]
    run_fulfill(eng, "fulfill_pending_ts", fulfill_head() + rules + [ts] + FULFILL_OUT + ["stream"], 2,
                *ts_inputs(lib), **kw)


# ---------------------------------------------------------------------------------------------------- readers and knobs
@pytest.mark.parametrize("method", ["last_affinity_reruns", "last_spread_rises"])
def test_pair_readers(eng, method):
    def eff(args):
        ctypes.c_int64.from_address(_addr(args[1])).value = 2
        if args[2] is not None:
            (ctypes.c_int64 * 4).from_address(_addr(args[2]))[:] = [5, 6, 7, 8]
    eng._lib.effect = eff
    assert getattr(eng, method)() == [(5, 6), (7, 8)]
    name = "acsfit_" + method
    expect_call(eng, [(name, ["ctx", "fresh", None]), (name, ["ctx", "fresh", "fresh"])])


def test_counters_and_records(eng):
    lib = eng._lib
    lib.effect = lambda args: [setattr(ctypes.c_int.from_address(_addr(a)), "value", 10 + i)
                               for i, a in enumerate(args[1:])]
    assert eng.cluster_last_plan() == {"stage_nodes": 10, "stages": 11, "pod_blocks": 12, "resident": 13}
    lib.effect = write(1, ctypes.c_uint64, [42])
    assert eng.last_sel_hits() == 42
    lib.effect = write(1, ctypes.c_uint64, [3, 4])
    assert eng.last_bin_retirement() == (3, 4)
    lib.effect = None
    assert eng.last_scan_launch() == dict.fromkeys(_native.SCAN_FIELDS, 0)
    stats = eng.pipeline_stats()
    assert set(stats) == {"ms", "decisions", "stages", "tiles"}
    lib.effect = write(3, ctypes.c_int, [1])
    assert len(eng.last_launches()) == 1
    lib.effect = None
    eng.debug_profile(False)
    eng.debug_trace(3, tiles=16)
    expect_call(eng, [("acsfit_cluster_last_plan", ["ctx", "fresh", "fresh", "fresh", "fresh"]),
                      ("acsfit_last_sel_hits", ["ctx", "fresh"]),
                      ("acsfit_last_bin_retirement", ["ctx", "fresh"]),
                      ("acsfit_last_scan_launch", ["ctx", "fresh"]),
                      ("acsfit_last_pipeline_stats", ["ctx", "fresh", "fresh", "fresh", "fresh"]),
                      ("acsfit_last_launches", ["ctx", None, 0, "fresh"]),
                      ("acsfit_last_launches", ["ctx", "fresh", 1, "fresh"]),
                      ("acsfit_debug_profile", ["ctx", 0, "fresh", 4096, "fresh"]),
                      ("acsfit_debug_trace", ["ctx", 3, "fresh", 16])])


def test_knobs(eng):
    eng.set_timing(True)
    eng.set_knob("ranks", 0)
    eng.configure(2, 500)
    eng.cluster_barrier()
    assert eng.launch_count == 0
    expect_call(eng, [("acsfit_ctx_set_timing", ["ctx", 1]), ("acsfit_ctx_set_knob", ["ctx", b"ranks", 0]),
                      ("acsfit_ctx_configure", ["ctx", 2, 500]), ("acsfit_cluster_barrier", ["ctx", "stream"]),
                      ("acsfit_launch_count", ["ctx"])])
