"""Device engine: thin Python face of libacsfit.so on dense float64 snapshots.

PyTorch is only the buffer container here (device memory, streams); every computation is a
hand-written sm_90a kernel behind the C ABI of include/acsfit.h.  There is no CPU
implementation: constructing an Engine without a CUDA device raises.
"""
import ctypes

import numpy as np
import torch

from . import _native
from ._native import AcsfitError

PIPELINE_DIMS = (2, 4, 8, 16)


def padded_dims(D):
    """columns the first-fit kernels are instantiated for; zero columns are neutral because an
    absent resource key is 0.0 on both sides of every test (kube.py:204-206, :210-212)."""
    for d in PIPELINE_DIMS:
        if D <= d:
            return d
    raise ValueError("more than %d resource dimensions are not supported" % PIPELINE_DIMS[-1])


def _ptr(t):
    if t is None:
        return None
    if isinstance(t, torch.Tensor):
        assert t.is_contiguous()
        return ctypes.c_void_p(t.data_ptr())
    assert isinstance(t, np.ndarray) and t.flags.c_contiguous
    return ctypes.c_void_p(t.ctypes.data)


def _np(a, dtype):
    return np.ascontiguousarray(a, dtype=dtype)


def _ref(s):
    """pointer to a ctypes object (a rule struct, or a value the library writes back), NULL for None"""
    return None if s is None else ctypes.cast(ctypes.byref(s), ctypes.c_void_p)


def _pools(D, units, pool_actual, pool_max, pool_ignored):
    """host pool arguments as the C ABI takes them: each unit table as float64 [T, D], then the per-pool arrays"""
    return tuple(_np(u, np.float64).reshape(-1, D) for u in units) + (
        _np(pool_actual, np.int32), _np(pool_max, np.int32), _np(pool_ignored, np.uint8))


def _fulfill_result(out):
    """the result dict of a fulfill_pending* call from the outputs of Engine._fulfill_out"""
    return dict(out, num_unaccounted=int(out["num_unaccounted"].value), evals=int(out["evals"].value))


def _host_pod_outputs(P):
    return {"feasible": np.empty(P, dtype=np.uint8), "placed": np.empty(P, dtype=np.int32),
            "acc_pool": np.empty(P, dtype=np.int32)}


def _scale_up_out(out, T):
    """(result dict, its pointer arguments in ABI order, counters) of a scale_up* call around `out`, the per-pod
    arrays feasible / placed / acc_pool"""
    res = dict(out)
    for k in ("new_size", "units_needed", "bins_opened"):
        res[k] = np.zeros(T, dtype=np.int64)
    counters = np.zeros(4, dtype=np.uint64)
    args = [_ptr(res[k]) for k in ("feasible", "placed", "new_size", "units_needed", "bins_opened", "acc_pool")]
    return res, args + [_ptr(counters)], counters


def _scale_up_result(res, counters):
    res.update({"n_to_schedule": int(counters[0]), "n_pending": int(counters[1]),
                "num_unaccounted": int(counters[2]), "decisions": int(counters[3])})
    return res


class Engine(object):
    """one acsfit context on one GPU (one per process / per rank)."""

    def __init__(self, device=None, min_stages=0, watchdog_ms=0):
        self._lib = _native.load()
        if not torch.cuda.is_available():
            raise RuntimeError("acsfit needs a CUDA device (sm_90a); there is no CPU fallback")
        if device is None:
            device = torch.cuda.current_device()
        self.device = torch.device("cuda", int(device))
        self._ctx = ctypes.c_void_p()
        st = self._lib.acsfit_ctx_create(int(device), ctypes.byref(self._ctx))
        if st != 0:
            raise AcsfitError(st, "acsfit_ctx_create failed on device %s" % device)
        if min_stages or watchdog_ms:
            self._check(self._lib.acsfit_ctx_configure(self._ctx, int(min_stages), int(watchdog_ms)))

    def close(self):
        if self._ctx:
            self._lib.acsfit_ctx_destroy(self._ctx)
            self._ctx = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ------------------------------------------------------------------ helpers
    def _check(self, status):
        if status != 0:
            raise AcsfitError(status, self._lib.acsfit_last_error(self._ctx).decode())

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def dev(self, a, dtype):
        """host array -> contiguous device tensor (H2D through pinned memory when large)."""
        if isinstance(a, torch.Tensor):
            return a.to(device=self.device, dtype=dtype).contiguous()
        t = torch.from_numpy(np.ascontiguousarray(a))
        return t.to(device=self.device, dtype=dtype, non_blocking=False).contiguous()

    def empty(self, shape, dtype):
        return torch.empty(shape, dtype=dtype, device=self.device)

    def _first_fit_out(self, req, pod_idx, used):
        """(rows, D, P, N, placed, decisions) of a first_fit_nodes* call"""
        rows, D = req.shape
        P = rows if pod_idx is None else pod_idx.shape[0]
        return rows, D, P, used.shape[0], self.empty((P,), torch.int32), \
            torch.zeros(1, dtype=torch.int64, device=self.device)

    def _fulfill_out(self, Pp, T):
        """(outputs, their pointer arguments in ABI order) of a fulfill_pending* call; see _fulfill_result"""
        out = {"new_size": np.zeros(T, dtype=np.int64), "units_needed": np.zeros(T, dtype=np.int64),
               "bins_opened": np.zeros(T, dtype=np.int64), "acc_pool": self.empty((Pp,), torch.int32),
               "bin_of": self.empty((Pp,), torch.int32), "num_unaccounted": ctypes.c_int64(0),
               "evals": ctypes.c_uint64(0)}
        args = [_ptr(out[k]) for k in ("new_size", "units_needed", "bins_opened", "acc_pool", "bin_of")]
        return out, args + [_ref(out["num_unaccounted"]), _ref(out["evals"])]

    def _pod_outputs(self, P):
        return {"feasible": self.empty((P,), torch.uint8), "placed": self.empty((P,), torch.int32),
                "acc_pool": self.empty((P,), torch.int32)}

    def _pairs(self, fn):
        """the (a, b) pairs a two-call test hook reports: the count first, then the pairs"""
        n = ctypes.c_int64(0)
        self._check(fn(self._ctx, _ref(n), None))
        out = np.zeros(2 * n.value, dtype=np.int64)
        self._check(fn(self._ctx, _ref(n), _ptr(out)))
        return [(int(out[2 * k]), int(out[2 * k + 1])) for k in range(n.value)]

    def set_timing(self, enabled):
        self._check(self._lib.acsfit_ctx_set_timing(self._ctx, 1 if enabled else 0))

    def set_knob(self, name, value):
        """developer knobs of include/acsfit.h ("ranks", "stream", "retire", "prune", "overlap", "min_stages", "cluster_blocks",
        "bulk_cfg", "stream_bytes", and the test hooks "inject_chain_timeout", "bin_pass_stages")."""
        self._check(self._lib.acsfit_ctx_set_knob(self._ctx, name.encode(), int(value)))

    def configure(self, min_stages=0, watchdog_ms=0):
        self._check(self._lib.acsfit_ctx_configure(self._ctx, int(min_stages), int(watchdog_ms)))

    # ------------------------------------------------------------------ cluster mode (one cluster, all GPUs of a box)
    def cluster_connect(self, max_pods, max_nodes, max_dims=16):
        """join the ranks of the default torch.distributed group into ONE cluster (include/acsfit.h, "Cluster
        mode"): every rank exports its exchange region (CUDA IPC), the handles are all-gathered here and opened
        by the library.  Afterwards first_fit_nodes / fulfill_pending / scale_up / scale_up_host must be called by
        all ranks with identical (replicated) inputs; each returns the complete result."""
        import torch.distributed as dist
        rank, world = dist.get_rank(), dist.get_world_size()
        handle = (ctypes.c_ubyte * 64)()
        self._check(self._lib.acsfit_cluster_init(self._ctx, rank, world, int(max_pods), int(max_nodes),
                                                  int(max_dims), ctypes.cast(handle, ctypes.c_void_p)))
        where = self.device if dist.get_backend() == "nccl" else torch.device("cpu")
        mine = torch.tensor(list(bytes(handle)), dtype=torch.uint8, device=where)
        gathered = [torch.empty_like(mine) for _ in range(world)]
        dist.all_gather(gathered, mine)
        blob = b"".join(bytes(t.cpu().numpy().tobytes()) for t in gathered)
        buf = ctypes.create_string_buffer(blob, len(blob))
        self._check(self._lib.acsfit_cluster_connect(self._ctx, ctypes.cast(buf, ctypes.c_void_p)))
        dist.barrier()  # every rank has zeroed and mapped every region before the first in-stream barrier
        self.cluster_world = world
        return world

    def cluster_barrier(self):
        self._check(self._lib.acsfit_cluster_barrier(self._ctx, self._stream()))

    def cluster_last_plan(self):
        v = [ctypes.c_int() for _ in range(4)]
        self._check(self._lib.acsfit_cluster_last_plan(self._ctx, *[_ref(x) for x in v]))
        return {"stage_nodes": v[0].value, "stages": v[1].value, "pod_blocks": v[2].value, "resident": v[3].value}

    @property
    def launch_count(self):
        return int(self._lib.acsfit_launch_count(self._ctx))

    def pipeline_stats(self):
        ms = ctypes.c_double()
        dec = ctypes.c_uint64()
        stages = ctypes.c_int()
        tiles = ctypes.c_int()
        self._check(self._lib.acsfit_last_pipeline_stats(self._ctx, ctypes.byref(ms), ctypes.byref(dec),
                                                         ctypes.byref(stages), ctypes.byref(tiles)))
        return {"ms": ms.value, "decisions": dec.value, "stages": stages.value, "tiles": tiles.value}

    def last_launches(self):
        """test hook: the first-fit pipeline kernels the last call launched, one dict per launch in launch order
        (keys: _native.LAUNCH_FIELDS; "pass" 0 = nodes / 1 = bins, "RW" 0 = float64 scan, "form" 1 = streaming)."""
        nf = len(_native.LAUNCH_FIELDS)
        n = ctypes.c_int(0)
        self._check(self._lib.acsfit_last_launches(self._ctx, None, 0, _ref(n)))
        out = np.zeros((max(n.value, 1), nf), dtype=np.int32)
        self._check(self._lib.acsfit_last_launches(self._ctx, _ptr(out), n.value, _ref(n)))
        return [dict(zip(_native.LAUNCH_FIELDS, (int(v) for v in row))) for row in out[:n.value]]

    def last_scan_launch(self):
        """test hook: the K1 / K6 kernel the last call launched, as a dict (keys: _native.SCAN_FIELDS; "kernel"
        0 = none / 1 = occupancy / 2 = node states, "form" 0 = per thread / 1 = index gather / 2 = bulk copy)."""
        out = np.zeros(len(_native.SCAN_FIELDS), dtype=np.int32)
        self._check(self._lib.acsfit_last_scan_launch(self._ctx, _ptr(out)))
        return dict(zip(_native.SCAN_FIELDS, (int(v) for v in out)))

    def last_sel_hits(self):
        """test hook: pods the candidate scan of the last call's selector node passes handed to the resolver (summed over
        tiles and stages; a pod counts in a stage only when some node there fits it AND matches its selector class)."""
        out = ctypes.c_uint64(0)
        self._check(self._lib.acsfit_last_sel_hits(self._ctx, _ref(out)))
        return int(out.value)

    def last_bin_retirement(self):
        """test hook: (dead warps, retired stages) that bin retirement marked in the last call's bin passes (barrier form
        with rank tables; summed over stages and passes; in cluster mode this rank's stages)."""
        out = np.zeros(2, dtype=np.uint64)
        self._check(self._lib.acsfit_last_bin_retirement(self._ctx, _ptr(out)))
        return int(out[0]), int(out[1])

    def last_affinity_reruns(self):
        """test hook: the (signature, position) flips the last pod-affinity call fixed, one per pass it ran again."""
        return self._pairs(self._lib.acsfit_last_affinity_reruns)

    def debug_profile(self, enabled=True):
        """developer probe: per-stage clock64 totals [stages, 8] of the last pipeline launch
        (wait, load, scan, resolve, publish, refresh, hits, tiles)."""
        out = np.zeros((4096, 8), dtype=np.uint64)
        n = ctypes.c_int(0)
        self._check(self._lib.acsfit_debug_profile(self._ctx, 1 if enabled else 0, _ptr(out), 4096, _ref(n)))
        return out[:n.value]

    def debug_trace(self, stage, tiles=8192):
        """developer probe: select the stage to trace / fetch its per-tile trace [tiles, 8]."""
        out = np.zeros((tiles, 8), dtype=np.uint64)
        self._check(self._lib.acsfit_debug_trace(self._ctx, int(stage), _ptr(out), tiles))
        return out

    # ------------------------------------------------------------------ device entry points
    def feasible_mask(self, req, unit):
        """capacity.is_possible over all pools (capacity.py:24-32). req [P,D], unit [T,D] device."""
        P, D = req.shape
        T = unit.shape[0]
        mask = self.empty((P,), torch.uint8)
        evals = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._check(self._lib.acsfit_feasible_mask(self._ctx, _ptr(req), P, D, _ptr(unit), T, _ptr(mask),
                                                   _ptr(evals), self._stream()))
        return mask, evals

    def occupancy(self, row_ptr, run_idx, req_run, used):
        """cluster.py:165-168: ordered used += req per node; `used` [N,D] device, in place."""
        N, D = used.shape
        self._check(self._lib.acsfit_occupancy(self._ctx, _ptr(row_ptr), _ptr(run_idx), _ptr(req_run), N, D,
                                               _ptr(used), self._stream()))
        return used

    def first_fit_nodes(self, req, pod_idx, cap_type, node_type, used):
        """Cluster.get_pending_pods (cluster.py:184-204). Returns (placed int32[P] device,
        decisions int64[1] device); `used` is updated in place."""
        rows, D, P, N, placed, decisions = self._first_fit_out(req, pod_idx, used)
        self._check(self._lib.acsfit_first_fit_nodes(self._ctx, _ptr(req), rows, _ptr(pod_idx), P, D, _ptr(cap_type),
                                                     _ptr(node_type), _ptr(used), N, _ptr(placed), _ptr(decisions),
                                                     self._stream()))
        return placed, decisions

    def fulfill_pending(self, req, num_listed, unit, pool_actual, pool_max, pool_ignored, over_provision):
        """Scaler.fulfill_pending up to scaler.py:177. req [Pp,D] device; pool arrays host (visiting order)."""
        Pp, D = req.shape
        unit, pool_actual, pool_max, pool_ignored = _pools(D, [unit], pool_actual, pool_max, pool_ignored)
        T = unit.shape[0]
        out, outs = self._fulfill_out(Pp, T)
        self._check(self._lib.acsfit_fulfill_pending(
            self._ctx, _ptr(req), Pp, int(num_listed), D, _ptr(unit), _ptr(pool_actual), _ptr(pool_max),
            _ptr(pool_ignored), T, int(over_provision), *outs, self._stream()))
        return _fulfill_result(out)

    def node_states(self, row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags, node_age,
                    any_pending, idle_thresholds):
        """Scaler.get_node_state for all nodes x S thresholds (scaler.py:61-114). returns uint8 [S,N] device."""
        N = node_type.shape[0]
        D = cap_type.shape[1]
        thr = _np(idle_thresholds, np.int64)
        S = thr.shape[0]
        out = self.empty((S, N), torch.uint8)
        self._check(self._lib.acsfit_node_states(self._ctx, _ptr(row_ptr), _ptr(run_idx), _ptr(req_run),
                                                 _ptr(flags_run), _ptr(cap_type), _ptr(node_type), _ptr(node_flags),
                                                 _ptr(node_age), N, D, 1 if any_pending else 0, _ptr(thr), S,
                                                 _ptr(out), self._stream()))
        return out

    def pending_admit(self, row_ptr, run_carries, run_matches, node_match, sig_class, sig_carries, sig_matches,
                      node_flags):
        """set ACSFIT_NODEF_NO_PENDING_MATCH on the nodes no signature (class, carries, matches) admits (include/acsfit.h,
        acsfit_pending_admit).  row_ptr int64 [N+1], run_carries / run_matches uint64 [rows] (stored as int64),
        node_match uint64 [N] or None, node_flags uint8 [N]: device, node_flags updated in place.  The signature
        arrays are host arrays of one length U."""
        N = node_flags.shape[0]
        sig_class = _np(sig_class, np.uint8)
        sig_carries, sig_matches = _np(sig_carries, np.uint64), _np(sig_matches, np.uint64)
        U = sig_class.shape[0]
        assert sig_carries.shape == sig_matches.shape == (U,)
        self._check(self._lib.acsfit_pending_admit(self._ctx, _ptr(row_ptr), _ptr(run_carries), _ptr(run_matches), N,
                                                   _ptr(node_match), _ptr(sig_class), _ptr(sig_carries),
                                                   _ptr(sig_matches), U, _ptr(node_flags), self._stream()))
        return node_flags

    def pending_admit_pa(self, row_ptr, run_carries, run_matches, run_has, node_match, sig_class, sig_carries,
                         sig_matches, sig_need, node_flags):
        """pending_admit with the pod-affinity test (include/acsfit.h, acsfit_pending_admit_pa): a signature (class,
        carries, matches, need) admits a node only when need is 0 or the node's pods match some signature of need too.
        run_has uint64 [rows] (stored as int64) on the device; sig_need a host array of length U.  run_carries,
        run_matches, sig_carries and sig_matches are all None (no anti-affinity test) or all given."""
        N = node_flags.shape[0]
        sig_class, sig_need = _np(sig_class, np.uint8), _np(sig_need, np.uint64)
        U = sig_class.shape[0]
        assert sig_need.shape == (U,)
        if sig_carries is not None or sig_matches is not None:
            sig_carries, sig_matches = _np(sig_carries, np.uint64), _np(sig_matches, np.uint64)
            assert sig_carries.shape == sig_matches.shape == (U,)
        self._check(self._lib.acsfit_pending_admit_pa(self._ctx, _ptr(row_ptr), _ptr(run_carries), _ptr(run_matches),
                                                      _ptr(run_has), N, _ptr(node_match), _ptr(sig_class),
                                                      _ptr(sig_carries), _ptr(sig_matches), _ptr(sig_need), U,
                                                      _ptr(node_flags), self._stream()))
        return node_flags

    def pending_admit_ts(self, row_ptr, run_carries, run_matches, run_has, node_match, sig_class, sig_carries,
                         sig_matches, sig_need, sig_key, sig_skew, keys, node_count, node_domain, floor, node_flags):
        """pending_admit_pa with the topology-spread test (include/acsfit.h, acsfit_pending_admit_ts): a signature with
        a key (sig_key != 0xFF) admits a node only when the node's count of that key is at most sig_skew plus the key's
        minimum.  sig_key uint8 and sig_skew int32 host arrays of length U; node_count int32 [keys, N] and node_domain
        uint64 [N] (stored as int64) on the device, floor int32 [keys] host.  The anti-affinity quadruple and the
        pod-affinity pair (run_has, sig_need) are each all None (that test does not run) or all given."""
        N = node_flags.shape[0]
        sig_class, sig_key, sig_skew = _np(sig_class, np.uint8), _np(sig_key, np.uint8), _np(sig_skew, np.int32)
        U = sig_class.shape[0]
        assert sig_key.shape == sig_skew.shape == (U,)
        if sig_carries is not None or sig_matches is not None:
            sig_carries, sig_matches = _np(sig_carries, np.uint64), _np(sig_matches, np.uint64)
            assert sig_carries.shape == sig_matches.shape == (U,)
        if sig_need is not None:
            sig_need = _np(sig_need, np.uint64)
            assert sig_need.shape == (U,)
        ts, keep_t = self._spread(keys, None, None, None, node_count, node_domain, floor)
        self._check(self._lib.acsfit_pending_admit_ts(self._ctx, _ptr(row_ptr), _ptr(run_carries), _ptr(run_matches),
                                                      _ptr(run_has), N, _ptr(node_match), _ptr(sig_class),
                                                      _ptr(sig_carries), _ptr(sig_matches), _ptr(sig_need),
                                                      _ptr(sig_key), _ptr(sig_skew), U, _ref(ts), _ptr(node_flags),
                                                      self._stream()))
        return node_flags

    def maintain_actions(self, state, node_pool, budget0, pool_scalable, dry_run):
        """engine_scaler.py:133-182 decisions. `state` uint8[N] device is rewritten; returns action uint8[N]."""
        N = state.shape[0]
        budget0 = _np(budget0, np.int64)
        pool_scalable = _np(pool_scalable, np.uint8)
        T = budget0.shape[0]
        action = self.empty((N,), torch.uint8)
        self._check(self._lib.acsfit_maintain_actions(self._ctx, _ptr(state), _ptr(node_pool), N, _ptr(budget0),
                                                      _ptr(pool_scalable), T, 1 if dry_run else 0, _ptr(action),
                                                      self._stream()))
        return state, action

    def scale_up(self, req, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, over_provision,
                 cap_type, node_type, used):
        """fused get_pods_to_schedule + get_pending_pods + fulfill_pending on device buffers."""
        P, D = req.shape
        N = used.shape[0]
        unit_all, unit_ordered, pool_actual, pool_max, pool_ignored = _pools(D, [unit_all, unit_ordered], pool_actual,
                                                                             pool_max, pool_ignored)
        T = unit_all.shape[0]
        res, outs, counters = _scale_up_out(self._pod_outputs(P), T)
        self._check(self._lib.acsfit_scale_up(
            self._ctx, _ptr(req), P, D, _ptr(unit_all), _ptr(unit_ordered), _ptr(pool_actual), _ptr(pool_max),
            _ptr(pool_ignored), T, int(over_provision), _ptr(cap_type), _ptr(node_type), _ptr(used), N, *outs,
            self._stream()))
        return _scale_up_result(res, counters)

    # ------------------------------------------------------------------ node selectors (include/acsfit.h)
    @staticmethod
    def _selectors(classes, pod_class=None, node_match=None, pool_match_all=None, pool_match_ordered=None):
        """(struct acsfit_selectors, the arrays it points to -- keep them alive over the call).  Pool masks are host
        arrays; pod_class / node_match are whatever the entry point expects (device tensors, or host arrays for
        scale_up_sel_host)."""
        keep = [None if a is None else (a if isinstance(a, torch.Tensor) else _np(a, a.dtype))
                for a in (pod_class, node_match)]
        keep += [None if a is None else _np(a, np.uint64) for a in (pool_match_all, pool_match_ordered)]
        sel = _native.Selectors(*[None if a is None else _ptr(a).value for a in keep], int(classes))
        return sel, keep

    @staticmethod
    def _selectors_if(classes, pod_class, **masks):
        """_selectors when pod_class is given (the rule forms take selectors as an option), else (None, None)"""
        return (None, None) if pod_class is None else Engine._selectors(classes, pod_class, **masks)

    def feasible_mask_sel(self, req, unit, pod_class, pool_match, classes):
        """feasible_mask with node selectors: pod_class uint8 [P] device, pool_match uint64 [T] host
        (agent_pools order)."""
        P, D = req.shape
        T = unit.shape[0]
        mask = self.empty((P,), torch.uint8)
        evals = torch.zeros(1, dtype=torch.int64, device=self.device)
        sel, keep = self._selectors(classes, pod_class=pod_class, pool_match_all=pool_match)
        self._check(self._lib.acsfit_feasible_mask_sel(self._ctx, _ptr(req), P, D, _ptr(unit), T, _ref(sel),
                                                       _ptr(mask), _ptr(evals), self._stream()))
        return mask, evals

    def first_fit_nodes_sel(self, req, pod_idx, cap_type, node_type, used, pod_class, node_match, classes):
        """first_fit_nodes with node selectors: pod_class uint8 [req rows] device, node_match uint64 [N] device."""
        rows, D, P, N, placed, decisions = self._first_fit_out(req, pod_idx, used)
        sel, keep = self._selectors(classes, pod_class=pod_class, node_match=node_match)
        self._check(self._lib.acsfit_first_fit_nodes_sel(
            self._ctx, _ptr(req), rows, _ptr(pod_idx), P, D, _ptr(cap_type), _ptr(node_type), _ptr(used), N,
            _ref(sel), _ptr(placed), _ptr(decisions), self._stream()))
        return placed, decisions

    def fulfill_pending_sel(self, req, num_listed, unit, pool_actual, pool_max, pool_ignored, over_provision,
                            pod_class, pool_match, classes):
        """fulfill_pending with node selectors: pod_class uint8 [Pp] device, pool_match uint64 [T] host (visiting
        order, like every other pool array here)."""
        Pp, D = req.shape
        unit, pool_actual, pool_max, pool_ignored = _pools(D, [unit], pool_actual, pool_max, pool_ignored)
        T = unit.shape[0]
        out, outs = self._fulfill_out(Pp, T)
        sel, keep = self._selectors(classes, pod_class=pod_class, pool_match_ordered=pool_match)
        self._check(self._lib.acsfit_fulfill_pending_sel(
            self._ctx, _ptr(req), Pp, int(num_listed), D, _ptr(unit), _ptr(pool_actual), _ptr(pool_max),
            _ptr(pool_ignored), T, int(over_provision), _ref(sel), *outs, self._stream()))
        return _fulfill_result(out)

    def scale_up_sel(self, req, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, over_provision,
                     cap_type, node_type, used, pod_class, node_match, pool_match_all, pool_match_ordered, classes):
        """scale_up with node selectors: pod_class uint8 [P] / node_match uint64 [N] device, the pool masks host."""
        P, D = req.shape
        N = used.shape[0]
        unit_all, unit_ordered, pool_actual, pool_max, pool_ignored = _pools(D, [unit_all, unit_ordered], pool_actual,
                                                                             pool_max, pool_ignored)
        T = unit_all.shape[0]
        res, outs, counters = _scale_up_out(self._pod_outputs(P), T)
        sel, keep = self._selectors(classes, pod_class, node_match, pool_match_all, pool_match_ordered)
        self._check(self._lib.acsfit_scale_up_sel(
            self._ctx, _ptr(req), P, D, _ptr(unit_all), _ptr(unit_ordered), _ptr(pool_actual), _ptr(pool_max),
            _ptr(pool_ignored), T, int(over_provision), _ptr(cap_type), _ptr(node_type), _ptr(used), N, _ref(sel),
            *outs, self._stream()))
        return _scale_up_result(res, counters)

    def scale_up_sel_host(self, req, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, over_provision,
                          cap_type, node_type, used, pod_class, node_match, pool_match_all, pool_match_ordered,
                          classes):
        """scale_up_host with node selectors: every buffer, pod_class and node_match included, is a HOST array."""
        req = _np(req, np.float64)
        P, D = req.shape
        cap_type = _np(cap_type, np.float64).reshape(-1, D)
        K = cap_type.shape[0]
        node_type = _np(node_type, np.int32)
        assert isinstance(used, np.ndarray) and used.dtype == np.float64 and used.flags.c_contiguous
        N = used.shape[0]
        unit_all, unit_ordered, pool_actual, pool_max, pool_ignored = _pools(D, [unit_all, unit_ordered], pool_actual,
                                                                             pool_max, pool_ignored)
        T = unit_all.shape[0]
        res, outs, counters = _scale_up_out(_host_pod_outputs(P), T)
        sel, keep = self._selectors(classes, _np(pod_class, np.uint8), _np(node_match, np.uint64), pool_match_all,
                                    pool_match_ordered)
        self._check(self._lib.acsfit_scale_up_sel_host(
            self._ctx, _ptr(req), P, D, _ptr(unit_all), _ptr(unit_ordered), _ptr(pool_actual), _ptr(pool_max),
            _ptr(pool_ignored), T, int(over_provision), _ptr(cap_type), K, _ptr(node_type), _ptr(used), N, _ref(sel),
            *outs))
        return _scale_up_result(res, counters)

    # ------------------------------------------------------------------ pod anti-affinity (include/acsfit.h)
    @staticmethod
    def _anti_affinity(pod_carries, pod_matches, node_carries=None, node_matches=None):
        """(struct acsfit_anti_affinity, the tensors it points to -- keep them alive over the call); device tensors."""
        keep = [pod_carries, pod_matches, node_carries, node_matches]
        aa = _native.AntiAffinity(*[None if a is None else _ptr(a).value for a in keep])
        return aa, keep

    @staticmethod
    def _anti_affinity_if(pod_carries, *masks):
        """_anti_affinity when pod_carries is given (the later rule forms take it as an option), else (None, None)"""
        return (None, None) if pod_carries is None else Engine._anti_affinity(pod_carries, *masks)

    def first_fit_nodes_aa(self, req, pod_idx, cap_type, node_type, used, pod_carries, pod_matches, node_carries,
                           node_matches, pod_class=None, node_match=None, classes=1):
        """first_fit_nodes with required pod anti-affinity: pod_carries / pod_matches uint64 [req rows] device (stored
        as int64), node_carries / node_matches uint64 [N] device, updated in place like `used`.  pod_class /
        node_match (both or neither): node selectors as in first_fit_nodes_sel."""
        rows, D, P, N, placed, decisions = self._first_fit_out(req, pod_idx, used)
        sel, keep_s = self._selectors_if(classes, pod_class, node_match=node_match)
        aa, keep_a = self._anti_affinity(pod_carries, pod_matches, node_carries, node_matches)
        self._check(self._lib.acsfit_first_fit_nodes_aa(
            self._ctx, _ptr(req), rows, _ptr(pod_idx), P, D, _ptr(cap_type), _ptr(node_type), _ptr(used), N,
            _ref(sel), _ref(aa), _ptr(placed), _ptr(decisions), self._stream()))
        return placed, decisions

    def fulfill_pending_aa(self, req, num_listed, unit, pool_actual, pool_max, pool_ignored, over_provision,
                           pod_carries, pod_matches, pod_class=None, pool_match=None, classes=1):
        """fulfill_pending with required pod anti-affinity in the bins: pod_carries / pod_matches uint64 [Pp] device
        (stored as int64).  pod_class / pool_match (both or neither): node selectors as in fulfill_pending_sel."""
        Pp, D = req.shape
        unit, pool_actual, pool_max, pool_ignored = _pools(D, [unit], pool_actual, pool_max, pool_ignored)
        T = unit.shape[0]
        out, outs = self._fulfill_out(Pp, T)
        sel, keep_s = self._selectors_if(classes, pod_class, pool_match_ordered=pool_match)
        aa, keep_a = self._anti_affinity(pod_carries, pod_matches)
        self._check(self._lib.acsfit_fulfill_pending_aa(
            self._ctx, _ptr(req), Pp, int(num_listed), D, _ptr(unit), _ptr(pool_actual), _ptr(pool_max),
            _ptr(pool_ignored), T, int(over_provision), _ref(sel), _ref(aa), *outs, self._stream()))
        return _fulfill_result(out)

    # ------------------------------------------------------------------ topology spread (include/acsfit.h)
    def last_spread_rises(self):
        """test hook: the (key, position) rises the last topology-spread call fixed, one per pass it ran again."""
        return self._pairs(self._lib.acsfit_last_spread_rises)

    @staticmethod
    def _spread(keys, pod_key, pod_skew, pod_matches, node_count=None, node_domain=None, floor=None):
        floor = np.ascontiguousarray(np.zeros(0, np.int32) if floor is None else floor, dtype=np.int32)
        keep = [pod_key, pod_skew, pod_matches, node_count, node_domain, floor]
        ts = _native.TopologySpread(*[None if a is None else _ptr(a).value for a in keep[:5]], _ptr(floor).value,
                                    int(keys))
        return ts, keep

    def first_fit_nodes_ts(self, req, pod_idx, cap_type, node_type, used, keys, pod_key, pod_skew, pod_matches,
                           node_count, node_domain, floor, pa=None, aa=None, pod_class=None, node_match=None, classes=1):
        """first_fit_nodes with hostname topology spread: pod_key uint8 [req rows], pod_skew int32 [req rows],
        pod_matches uint64 [req rows] (stored as int64), node_count int32 [keys, N] and node_domain uint64 [N] device,
        floor int32 [keys] host; node_count is updated in place like `used`.  `pa` (pod_requires, pod_self,
        pod_matches, node_has) and `aa` (pod_carries, pod_matches, node_carries, node_matches) device tuples or None;
        pod_class / node_match (both or neither) as in first_fit_nodes_aa."""
        rows, D, P, N, placed, decisions = self._first_fit_out(req, pod_idx, used)
        sel, keep_s = self._selectors_if(classes, pod_class, node_match=node_match)
        a, keep_a = self._anti_affinity_if(*(aa or (None,)))
        p = None if pa is None else _native.PodAffinity(*[_ptr(t).value for t in pa])
        ts, keep_t = self._spread(keys, pod_key, pod_skew, pod_matches, node_count, node_domain, floor)
        self._check(self._lib.acsfit_first_fit_nodes_ts(
            self._ctx, _ptr(req), rows, _ptr(pod_idx), P, D, _ptr(cap_type), _ptr(node_type), _ptr(used), N,
            _ref(sel), _ref(a), _ref(p), _ref(ts), _ptr(placed), _ptr(decisions), self._stream()))
        return placed, decisions

    def fulfill_pending_ts(self, req, num_listed, unit, pool_actual, pool_max, pool_ignored, over_provision, keys,
                           pod_key, pod_skew, pod_matches, pa=None, present=0, aa=None, pod_class=None,
                           pool_match=None, classes=1):
        """fulfill_pending with hostname topology spread in the bins: pod_key / pod_skew / pod_matches [Pp] device as
        in first_fit_nodes_ts.  `pa` (pod_requires, pod_self, pod_matches) and `aa` (pod_carries, pod_matches) device
        tuples or None; `present` and pod_class / pool_match as in fulfill_pending_pa."""
        Pp, D = req.shape
        unit, pool_actual, pool_max, pool_ignored = _pools(D, [unit], pool_actual, pool_max, pool_ignored)
        T = unit.shape[0]
        out, outs = self._fulfill_out(Pp, T)
        sel, keep_s = self._selectors_if(classes, pod_class, pool_match_ordered=pool_match)
        a, keep_a = self._anti_affinity_if(*(aa or (None,)))
        p = None if pa is None else _native.PodAffinity(*[_ptr(t).value for t in pa], None)
        ts, keep_t = self._spread(keys, pod_key, pod_skew, pod_matches)
        self._check(self._lib.acsfit_fulfill_pending_ts(
            self._ctx, _ptr(req), Pp, int(num_listed), D, _ptr(unit), _ptr(pool_actual), _ptr(pool_max),
            _ptr(pool_ignored), T, int(over_provision), _ref(sel), _ref(a), _ref(p), int(present) & 0xFFFFFFFFFFFFFFFF,
            _ref(ts), *outs, self._stream()))
        return _fulfill_result(out)

    # ------------------------------------------------------------------ pod affinity (include/acsfit.h)
    def first_fit_nodes_pa(self, req, pod_idx, cap_type, node_type, used, pod_requires, pod_self, pod_matches, node_has,
                           pod_carries=None, pod_matches_aa=None, node_carries=None, node_matches=None, pod_class=None,
                           node_match=None, classes=1):
        """first_fit_nodes with required pod affinity: pod_requires / pod_self / pod_matches uint64 [req rows] device
        (stored as int64), node_has uint64 [N] device, updated in place like `used`.  The anti-affinity masks (all four
        or none) and pod_class / node_match (both or neither) as in first_fit_nodes_aa."""
        rows, D, P, N, placed, decisions = self._first_fit_out(req, pod_idx, used)
        sel, keep_s = self._selectors_if(classes, pod_class, node_match=node_match)
        aa, keep_a = self._anti_affinity_if(pod_carries, pod_matches_aa, node_carries, node_matches)
        keep_p = [pod_requires, pod_self, pod_matches, node_has]
        pa = _native.PodAffinity(*[None if a is None else _ptr(a).value for a in keep_p])
        self._check(self._lib.acsfit_first_fit_nodes_pa(
            self._ctx, _ptr(req), rows, _ptr(pod_idx), P, D, _ptr(cap_type), _ptr(node_type), _ptr(used), N,
            _ref(sel), _ref(aa), _ref(pa), _ptr(placed), _ptr(decisions), self._stream()))
        return placed, decisions

    def fulfill_pending_pa(self, req, num_listed, unit, pool_actual, pool_max, pool_ignored, over_provision,
                           pod_requires, pod_self, pod_matches, present=0, pod_carries=None, pod_matches_aa=None,
                           pod_class=None, pool_match=None, classes=1):
        """fulfill_pending with required pod affinity in the bins: pod_requires / pod_self / pod_matches uint64 [Pp]
        device (stored as int64); `present` the signatures the nodes already hold (0: only pods this call places
        count).  The anti-affinity masks (both or neither) and pod_class / pool_match as in fulfill_pending_aa."""
        Pp, D = req.shape
        unit, pool_actual, pool_max, pool_ignored = _pools(D, [unit], pool_actual, pool_max, pool_ignored)
        T = unit.shape[0]
        out, outs = self._fulfill_out(Pp, T)
        sel, keep_s = self._selectors_if(classes, pod_class, pool_match_ordered=pool_match)
        aa, keep_a = self._anti_affinity_if(pod_carries, pod_matches_aa)
        keep_p = [pod_requires, pod_self, pod_matches]
        pa = _native.PodAffinity(*[None if a is None else _ptr(a).value for a in keep_p], None)
        self._check(self._lib.acsfit_fulfill_pending_pa(
            self._ctx, _ptr(req), Pp, int(num_listed), D, _ptr(unit), _ptr(pool_actual), _ptr(pool_max),
            _ptr(pool_ignored), T, int(over_provision), _ref(sel), _ref(aa), _ref(pa),
            int(present) & 0xFFFFFFFFFFFFFFFF, *outs, self._stream()))
        return _fulfill_result(out)

    # ------------------------------------------------------------------ host-buffer entry points
    def scale_up_host(self, req, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, over_provision,
                      cap_type, node_type, used, out=None):
        """the plugin call: all buffers are HOST numpy arrays (pinned for speed); `used` is updated in place."""
        req = _np(req, np.float64)
        P, D = req.shape
        cap_type = _np(cap_type, np.float64).reshape(-1, D)
        K = cap_type.shape[0]
        node_type = _np(node_type, np.int32)
        assert isinstance(used, np.ndarray) and used.dtype == np.float64 and used.flags.c_contiguous
        N = used.shape[0]
        unit_all, unit_ordered, pool_actual, pool_max, pool_ignored = _pools(D, [unit_all, unit_ordered], pool_actual,
                                                                             pool_max, pool_ignored)
        T = unit_all.shape[0]
        res, outs, counters = _scale_up_out(_host_pod_outputs(P) if out is None else out, T)
        self._check(self._lib.acsfit_scale_up_host(
            self._ctx, _ptr(req), P, D, _ptr(unit_all), _ptr(unit_ordered), _ptr(pool_actual), _ptr(pool_max),
            _ptr(pool_ignored), T, int(over_provision), _ptr(cap_type), K, _ptr(node_type), _ptr(used), N, *outs))
        return _scale_up_result(res, counters)

    def occupancy_host(self, row_ptr, run_idx, req_run, used):
        """cluster.py:165-168 with HOST arrays; `used` [N, D] float64 is updated in place."""
        assert isinstance(used, np.ndarray) and used.dtype == np.float64 and used.flags.c_contiguous
        N, D = used.shape
        req_run = _np(req_run, np.float64).reshape(-1, D)
        self._check(self._lib.acsfit_occupancy_host(self._ctx, _ptr(_np(row_ptr, np.int64)),
                                                    _ptr(None if run_idx is None else _np(run_idx, np.int32)),
                                                    _ptr(req_run), req_run.shape[0], N, D, _ptr(used)))
        return used

    def maintain_host(self, row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags, node_age,
                      node_pool, any_pending, idle_threshold, budget0, pool_scalable, dry_run):
        cap_type = _np(cap_type, np.float64)
        K, D = cap_type.shape
        req_run = _np(req_run, np.float64).reshape(-1, D)
        R = req_run.shape[0]
        row_ptr = _np(row_ptr, np.int64)
        run_idx = None if run_idx is None else _np(run_idx, np.int32)  # None: contiguous table
        flags_run = _np(flags_run, np.uint8)
        node_type = _np(node_type, np.int32)
        node_flags = _np(node_flags, np.uint8)
        node_age = _np(node_age, np.int64)
        node_pool = _np(node_pool, np.int32)
        budget0 = _np(budget0, np.int64)
        pool_scalable = _np(pool_scalable, np.uint8)
        N = node_type.shape[0]
        T = budget0.shape[0]
        state = np.empty(N, dtype=np.uint8)
        action = np.empty(N, dtype=np.uint8)
        self._check(self._lib.acsfit_maintain_host(
            self._ctx, _ptr(row_ptr), _ptr(run_idx), _ptr(req_run), _ptr(flags_run), R, _ptr(cap_type), K,
            _ptr(node_type), _ptr(node_flags), _ptr(node_age), _ptr(node_pool), N, D, 1 if any_pending else 0,
            int(idle_threshold), _ptr(budget0), _ptr(pool_scalable), T, 1 if dry_run else 0, _ptr(state),
            _ptr(action)))
        return state, action
