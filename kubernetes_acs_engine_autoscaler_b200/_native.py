"""ctypes binding of libacsfit.so (include/acsfit.h).  No CPU fallback: if the shared object is
missing or cannot be loaded this module raises, and every product entry point with it."""
import ctypes
import os

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG_DIR, "libacsfit.so")

OK, E_INVALID, E_CUDA, E_DOMAIN, E_TIMEOUT, E_NOMEM, E_PEER = 0, -1, -2, -3, -4, -5, -6
_STATUS_NAMES = {E_INVALID: "ACSFIT_E_INVALID", E_CUDA: "ACSFIT_E_CUDA", E_DOMAIN: "ACSFIT_E_DOMAIN",
                 E_TIMEOUT: "ACSFIT_E_TIMEOUT", E_NOMEM: "ACSFIT_E_NOMEM", E_PEER: "ACSFIT_E_PEER"}

c_i64, c_int, c_vp, c_u64 = ctypes.c_int64, ctypes.c_int, ctypes.c_void_p, ctypes.c_uint64

# every symbol include/acsfit.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "acsfit_abi_version": (c_int, []),
    "acsfit_last_error": (ctypes.c_char_p, [c_vp]),
    "acsfit_ctx_create": (c_int, [c_int, ctypes.POINTER(c_vp)]),
    "acsfit_ctx_destroy": (c_int, [c_vp]),
    "acsfit_ctx_configure": (c_int, [c_vp, c_int, c_int]),
    "acsfit_ctx_set_timing": (c_int, [c_vp, c_int]),
    "acsfit_ctx_set_knob": (c_int, [c_vp, ctypes.c_char_p, c_int]),
    "acsfit_feasible_mask": (c_int, [c_vp, c_vp, c_i64, c_int, c_vp, c_int, c_vp, c_vp, c_vp]),
    "acsfit_occupancy": (c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_vp, c_vp]),
    "acsfit_first_fit_nodes": (c_int, [c_vp, c_vp, c_i64, c_vp, c_i64, c_int, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp]),
    "acsfit_fulfill_pending": (c_int, [c_vp, c_vp, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_int, c_i64,
                                       c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "acsfit_node_states": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_int, c_int,
                                   c_vp, c_int, c_vp, c_vp]),
    "acsfit_pending_admit": (c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_int, c_vp, c_vp]),
    "acsfit_pending_admit_pa": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_int,
                                        c_vp, c_vp]),
    "acsfit_maintain_actions": (c_int, [c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_int, c_int, c_vp, c_vp]),
    "acsfit_scale_up": (c_int, [c_vp, c_vp, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_i64,
                                c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "acsfit_scale_up_host": (c_int, [c_vp, c_vp, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_i64,
                                     c_vp, c_int, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "acsfit_occupancy_host": (c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_int, c_vp]),
    "acsfit_maintain_host": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_int, c_vp, c_vp, c_vp, c_vp,
                                     c_i64, c_int, c_int, c_i64, c_vp, c_vp, c_int, c_int, c_vp, c_vp]),
    "acsfit_cluster_init": (c_int, [c_vp, c_int, c_int, c_i64, c_i64, c_int, c_vp]),
    "acsfit_cluster_connect": (c_int, [c_vp, c_vp]),
    "acsfit_cluster_barrier": (c_int, [c_vp, c_vp]),
    "acsfit_cluster_last_plan": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp]),
    "acsfit_launch_count": (c_u64, [c_vp]),
    "acsfit_debug_profile": (c_int, [c_vp, c_int, c_vp, c_int, c_vp]),
    "acsfit_debug_trace": (c_int, [c_vp, c_int, c_vp, c_int]),
    "acsfit_last_pipeline_stats": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp]),
    "acsfit_last_launches": (c_int, [c_vp, c_vp, c_int, c_vp]),
    "acsfit_last_scan_launch": (c_int, [c_vp, c_vp]),
    "acsfit_last_sel_hits": (c_int, [c_vp, c_vp]),
    "acsfit_last_bin_retirement": (c_int, [c_vp, c_vp]),
    # node selectors: the arguments of the plain form plus a `const acsfit_selectors *` (Selectors below)
    "acsfit_feasible_mask_sel": (c_int, [c_vp, c_vp, c_i64, c_int, c_vp, c_int, c_vp, c_vp, c_vp, c_vp]),
    "acsfit_first_fit_nodes_sel": (c_int, [c_vp, c_vp, c_i64, c_vp, c_i64, c_int, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp,
                                           c_vp, c_vp]),
    "acsfit_fulfill_pending_sel": (c_int, [c_vp, c_vp, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_int, c_i64,
                                           c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "acsfit_scale_up_sel": (c_int, [c_vp, c_vp, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_i64,
                                    c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "acsfit_scale_up_sel_host": (c_int, [c_vp, c_vp, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_int, c_i64,
                                         c_vp, c_int, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                         c_vp]),
    # pod anti-affinity: the arguments of the _sel form (sel may be NULL) plus a `const acsfit_anti_affinity *`
    "acsfit_first_fit_nodes_aa": (c_int, [c_vp, c_vp, c_i64, c_vp, c_i64, c_int, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp,
                                          c_vp, c_vp, c_vp]),
    "acsfit_fulfill_pending_aa": (c_int, [c_vp, c_vp, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_int, c_i64,
                                          c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    # pod affinity: the arguments of the _aa form (sel and aa may be NULL) plus a `const acsfit_pod_affinity *`
    # (and, fulfill, the uint64 `present`)
    "acsfit_first_fit_nodes_pa": (c_int, [c_vp, c_vp, c_i64, c_vp, c_i64, c_int, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp,
                                          c_vp, c_vp, c_vp, c_vp]),
    "acsfit_fulfill_pending_pa": (c_int, [c_vp, c_vp, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_int, c_i64,
                                          c_vp, c_vp, c_vp, ctypes.c_uint64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                          c_vp]),
    "acsfit_last_affinity_reruns": (c_int, [c_vp, c_vp, c_vp]),
    # topology spread: the arguments of the _pa form (sel, aa and pa may be NULL) plus a
    # `const acsfit_topology_spread *` (fulfill: after `present`)
    "acsfit_first_fit_nodes_ts": (c_int, [c_vp, c_vp, c_i64, c_vp, c_i64, c_int, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp,
                                          c_vp, c_vp, c_vp, c_vp, c_vp]),
    "acsfit_fulfill_pending_ts": (c_int, [c_vp, c_vp, c_i64, c_i64, c_int, c_vp, c_vp, c_vp, c_vp, c_int, c_i64,
                                          c_vp, c_vp, c_vp, ctypes.c_uint64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                          c_vp, c_vp]),
    "acsfit_last_spread_rises": (c_int, [c_vp, c_vp, c_vp]),
    "acsfit_pending_admit_ts": (c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                        c_vp, c_int, c_vp, c_vp, c_vp]),
}


class Selectors(ctypes.Structure):
    """struct acsfit_selectors (include/acsfit.h)"""
    _fields_ = [("pod_class", c_vp), ("node_match", c_vp), ("pool_match_all", c_vp),
                ("pool_match_ordered", c_vp), ("classes", c_int)]


class AntiAffinity(ctypes.Structure):
    """struct acsfit_anti_affinity (include/acsfit.h)"""
    _fields_ = [("pod_carries", c_vp), ("pod_matches", c_vp), ("node_carries", c_vp), ("node_matches", c_vp)]


class PodAffinity(ctypes.Structure):
    """struct acsfit_pod_affinity (include/acsfit.h)"""
    _fields_ = [("pod_requires", c_vp), ("pod_self", c_vp), ("pod_matches", c_vp), ("node_has", c_vp)]


class TopologySpread(ctypes.Structure):
    """struct acsfit_topology_spread (include/acsfit.h)"""
    _fields_ = [("pod_key", c_vp), ("pod_skew", c_vp), ("pod_matches", c_vp), ("node_count", c_vp),
                ("node_domain", c_vp), ("floor", c_vp), ("keys", ctypes.c_int32)]


# one record of acsfit_last_launches (ACSFIT_LAUNCH_FIELDS ints), field names in order
LAUNCH_FIELDS = ("pass", "chained", "D", "RW", "prune", "form", "Tn", "stages", "resident", "pool", "bin_base",
                 "publish_every")
# the record of acsfit_last_scan_launch (ACSFIT_SCAN_FIELDS ints), field names in order
SCAN_FIELDS = ("kernel", "form", "D", "bytes", "warps", "chunk", "grid", "S")


class AcsfitError(RuntimeError):
    def __init__(self, status, message):
        super().__init__("%s: %s" % (_STATUS_NAMES.get(status, "status %d" % status), message))
        self.status = status


_lib = None


def load():
    """load libacsfit.so (raises if it has not been built: there is no CPU fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "%s is missing: build it with `python -m kubernetes_acs_engine_autoscaler_b200.build` "
                "(nvcc, sm_90a). The pod-fit path has no CPU fallback." % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the ABI is incomplete
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
    return _lib
