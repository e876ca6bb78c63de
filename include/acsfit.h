/*
 * acsfit.h -- C ABI of libacsfit.so, the H100 (sm_90a) decision engine behind the
 * acs-engine autoscaler's per-tick hot path.
 *
 * The reference (wbuchwalter/Kubernetes-acs-engine-autoscaler) is pure Python and has no
 * FFI: the boundary it offers is a set of Python methods.  Each entry point below replaces
 * the arithmetic of one of those methods on a dense float64 snapshot ("absent resource key
 * == 0.0", SURVEY.md section 0.4); the Python classes of the same names in
 * kubernetes_acs_engine_autoscaler_b200/ translate between kube objects and these buffers
 * (INTEGRATION.md shows the ctypes binding a reference maintainer would add).
 *
 * Conventions
 *  - plain C: pointers and sizes only, no torch / CUDA types in the signatures.
 *    `acsfit_stream_t` is a `cudaStream_t` passed as `void*` (NULL = default stream).
 *  - every function returns an `acsfit_status` (0 = ok, < 0 = error); nothing throws
 *    across the boundary.  `acsfit_last_error(ctx)` gives the message.
 *  - pointers marked [dev] are device pointers owned by the caller (e.g.
 *    torch.Tensor.data_ptr()); the library never frees or retains them past the call.
 *    Pointers marked [host] are host pointers.  Small per-pool results come back through
 *    [host] pointers, so those calls synchronise the stream before returning.
 *  - matrices are row-major float64 with exactly D columns; D <= ACSFIT_MAX_DIMS.
 *  - one ctx per host thread (thread-compatible, not thread-safe); the ctx owns a reusable
 *    scratch arena so a steady-state tick performs no cudaMalloc.
 *  - input domain: requests are >= 0 and not NaN (reference: utils.py:33 regex admits no
 *    sign); capacity / unit rows are finite.  Violations return ACSFIT_E_DOMAIN.
 */
#ifndef ACSFIT_H
#define ACSFIT_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ACSFIT_ABI_VERSION 2
#define ACSFIT_MAX_DIMS 16
#define ACSFIT_MAX_POOLS 256

#if defined(__GNUC__)
#define ACSFIT_API __attribute__((visibility("default")))
#else
#define ACSFIT_API
#endif

typedef int acsfit_status;
enum {
    ACSFIT_OK = 0,
    ACSFIT_E_INVALID = -1,  /* bad argument (NULL pointer, negative size, D too large ...) */
    ACSFIT_E_CUDA = -2,     /* a CUDA runtime call or kernel failed */
    ACSFIT_E_DOMAIN = -3,   /* input outside the reference's domain (negative / NaN request) */
    ACSFIT_E_TIMEOUT = -4,  /* device-side watchdog fired (inter-stage pipeline stalled) */
    ACSFIT_E_NOMEM = -5,
    ACSFIT_E_PEER = -6      /* cluster mode: a peer rank failed / did not arrive (in-stream barrier timed out) */
};

/* ClusterNodeState codes, in the order reference autoscaler/scaler.py:19-29 lists them */
enum {
    ACSFIT_ST_INSTANCE_TERMINATED = 0,
    ACSFIT_ST_POD_PENDING = 1,
    ACSFIT_ST_GRACE_PERIOD = 2,
    ACSFIT_ST_SPARE_AGENT = 3,
    ACSFIT_ST_IDLE_SCHEDULABLE = 4,
    ACSFIT_ST_IDLE_UNSCHEDULABLE = 5,
    ACSFIT_ST_BUSY_UNSCHEDULABLE = 6,
    ACSFIT_ST_BUSY = 7,
    ACSFIT_ST_UNDER_UTILIZED_DRAINABLE = 8,
    ACSFIT_ST_UNDER_UTILIZED_UNDRAINABLE = 9,
    ACSFIT_ST_NOT_EVALUATED = 255 /* node of an ignored pool: the reference never asks */
};
/* maintain() actions (reference autoscaler/engine_scaler.py:149-182) */
enum {
    ACSFIT_ACT_NONE = 0,
    ACSFIT_ACT_CORDON_DRAIN = 1, /* UNDER_UTILIZED_DRAINABLE :153-161 */
    ACSFIT_ACT_CORDON = 2,       /* IDLE_SCHEDULABLE         :162-166 */
    ACSFIT_ACT_UNCORDON = 3,     /* BUSY_UNSCHEDULABLE       :167-172 */
    ACSFIT_ACT_SCALE_IN = 4      /* IDLE_UNSCHEDULABLE       :173-177 */
};
/* per running-pod flag bits, computed by the host from annotations / labels / name */
#define ACSFIT_PODF_BUSY 1u        /* not is_mirrored() and 'kube-proxy' not in name  scaler.py:76    */
#define ACSFIT_PODF_UNDRAINABLE 2u /* not (is_drainable() or 'kube-proxy' in name)    scaler.py:82-83 */
/* per node flag bits */
#define ACSFIT_NODEF_UNSCHEDULABLE 1u /* spec.unschedulable  kube.py:105 */
#define ACSFIT_NODEF_NO_PENDING_MATCH 2u /* no pod to schedule matches the node's labels (opt-in, see node_states) */

typedef struct acsfit_ctx acsfit_ctx;
typedef void *acsfit_stream_t;

ACSFIT_API int acsfit_abi_version(void);
ACSFIT_API const char *acsfit_last_error(const acsfit_ctx *ctx);

/* `device` is the CUDA device ordinal.  Fails (ACSFIT_E_CUDA) when no sm_90 device is there:
 * there is no CPU fallback. */
ACSFIT_API acsfit_status acsfit_ctx_create(int device, acsfit_ctx **out_ctx);
ACSFIT_API acsfit_status acsfit_ctx_destroy(acsfit_ctx *ctx);
/* pipeline tuning knobs (0 = library default): stages the node/bin axis is cut into at least,
 * and the watchdog in milliseconds.
 * Developer knobs read from the environment at acsfit_ctx_create (none changes a result, only the schedule):
 *   ACSFIT_OVERLAP=0        do not chain the first bin pass behind the node pass on a second stream
 *   ACSFIT_PRUNE=0|1        never / always use the scan-list-pruning instantiation of the node pass
 *                           (default: only when the pass has more stages than the GPU holds at once)
 *   ACSFIT_MIN_STAGES=n     same as acsfit_ctx_configure(min_stages) (default: one stage per SM)
 *   ACSFIT_SMEM_FLOOR_KB=n  request at least n KB of shared memory per stage CTA (limits CTAs per SM)
 *   ACSFIT_STREAM_BYTES=n   initial value of knob "stream_bytes" (below)
 *   ACSFIT_BULK_CFG=n       initial value of knob "bulk_cfg" (below)
 *   ACSFIT_RANKS=0          never use the packed-rank scan (float64 compares instead; same results) */
ACSFIT_API acsfit_status acsfit_ctx_configure(acsfit_ctx *ctx, int min_stages, int watchdog_ms);
/* the same developer knobs by name, after ctx creation: "ranks" (0: float64 compare scan, 1: packed-rank scan when
 * the tick's request table allows it -- the default), "stream" (1: the barrier-free streaming form of the pipeline
 * kernel, csrc/acsfit_stream_ff.cuh, where it applies; env ACSFIT_STREAM), "retire" (0: bin passes keep testing
 * bins that can take no pod of the pass any more; default 1), "prune", "overlap", "min_stages", "inject_chain_timeout" (test hook), "cluster_blocks" (cluster
 * mode: cut the pod list of the node pass into this many blocks; 0 = automatic), and for the K1 / K6 idle scan
 * (csrc/acsfit_scan_plan.h): "bulk_cfg" (geometry of the bulk-copy form, contiguous tables, D <= 8:
 * 0 = 8 KB x 8 warps, 1 = 16 KB x 12, 2 = 16 KB x 8, 3 = 32 KB x 6, anything else = 8 KB x 16, the default 4;
 * D = 16 always uses 16 KB x 8) and "stream_bytes" (staging bytes per warp of the gather form, tables with
 * run_idx: the smallest of 2048 (D <= 4) / 4096 (D <= 8) / 8192 that is >= the value; default 8192).
 * Both are per ctx.  None changes a result.
 * Test hooks: "inject_chain_timeout" = n treats the next n chained node+bin launches as timed out (exercises the
 * unchained redo); "bin_pass_stages" = n cuts every single-GPU bin pass, the chained first pass included, to at most
 * n stages (0 = the library's limit of 1024), so that small inputs pack their bins in several passes. */
ACSFIT_API acsfit_status acsfit_ctx_set_knob(acsfit_ctx *ctx, const char *name, int value);
/* when enabled, the first-fit / bin-pack pipeline launches are bracketed with CUDA events on the
 * launching stream (read back with acsfit_last_pipeline_stats) */
ACSFIT_API acsfit_status acsfit_ctx_set_timing(acsfit_ctx *ctx, int enabled);

/*
 * K0 feasible_mask -- capacity.is_possible over all agent pools, as used by
 * Cluster.get_pods_to_schedule (reference autoscaler/capacity.py:24-32, cluster.py:217-240).
 *   req   [dev] P x D   pending-unassigned pods, list order
 *   unit  [dev] T x D   RESOURCE_SPEC[pool.instance_type] per agent pool (ignored pools included)
 *   out_mask  [dev] P bytes: 1 when (unit[t] - req).possible for some t
 *   out_evals [dev] one uint64 (may be NULL): number of `.possible` evaluations the reference
 *             performs (it stops at the first pool that fits)
 */
ACSFIT_API acsfit_status acsfit_feasible_mask(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                   const double *unit, int T, uint8_t *out_mask,
                                   uint64_t *out_evals, acsfit_stream_t stream);

/*
 * K1 occupancy -- the node.count_pod loop of Cluster.loop_logic (reference cluster.py:165-168,
 * kube.py:169-171): used[n] = used[n] + req_run[j] for the node's running/assigned pods in
 * POD-LIST order (left-to-right float64 sum, no tree reduction).
 *   row_ptr [dev] N+1 int64, run_idx [dev] row_ptr[N] int32 indices into req_run (ascending
 *   inside each node), req_run [dev] R x D, used_inout [dev] N x D (zero = KubeResource()).
 *   run_idx may be NULL (here, in acsfit_node_states and in the *_host forms): the table is then CONTIGUOUS, the
 *   pods of node n are rows row_ptr[n] .. row_ptr[n+1] of req_run / flags_run.  That is the layout the host
 *   layer produces, and it lets K1 / K6 stream the table with bulk copies (csrc/acsfit_stream.cuh).
 *   Alignment (here and in acsfit_node_states): the streaming forms for D in {2,4,8,16} read req_run -- and, for
 *   a contiguous table in K6, flags_run -- with 16-byte copies, so they run only when those pointers are 16-byte
 *   aligned.  Any other table (a view at an odd offset, e.g. flags[1:]) runs the per-thread form with scalar
 *   loads: the same result, only slower.  acsfit_last_scan_launch reports which form ran.
 */
ACSFIT_API acsfit_status acsfit_occupancy(acsfit_ctx *ctx, const int64_t *row_ptr, const int32_t *run_idx,
                               const double *req_run, int64_t N, int D, double *used_inout,
                               acsfit_stream_t stream);

/*
 * K2+K3 first_fit_nodes -- Cluster.get_pending_pods (reference cluster.py:184-204) with
 * KubeNode.can_fit (kube.py:173-176): sequential first-fit of pods (list order) over nodes
 * (list order); a hit mutates used[node] += req.  Exact and order-preserving.
 *   req        [dev] req_rows x D     (D must be 2, 4, 8 or 16: zero columns are neutral, because
 *                                      an absent resource key is 0.0 on both sides of the test;
 *                                      16-byte aligned, else ACSFIT_E_INVALID -- the same holds for req
 *                                      of acsfit_fulfill_pending and acsfit_scale_up)
 *   pod_idx    [dev] P int32 row numbers into req, the pods to schedule in order; NULL = rows 0..P-1
 *   cap_type   [dev] K x D, node_type [dev] N int32 (row of cap_type per node)
 *   used_inout [dev] N x D
 *   out_placed [dev] P int32: node index, or -1 = pending
 *   out_decisions [dev] one uint64 (may be NULL): number of KubeNode.can_fit calls the
 *                 reference makes = sum(placed >= 0 ? placed + 1 : N)
 */
ACSFIT_API acsfit_status acsfit_first_fit_nodes(acsfit_ctx *ctx, const double *req, int64_t req_rows,
                                     const int32_t *pod_idx, int64_t P, int D, const double *cap_type,
                                     const int32_t *node_type, double *used_inout, int64_t N,
                                     int32_t *out_placed, uint64_t *out_decisions,
                                     acsfit_stream_t stream);

/*
 * K4+K5 fulfill_pending -- Scaler.fulfill_pending (reference scaler.py:117-177): per pool in
 * cost order, first-fit of the still-unaccounted eligible pods into new-instance bins, the
 * pool-size clamp arithmetic and the accounting of the first min(len(bins), units_requested)
 * bins.  The raise / scale_pools hand-off (:179-184) stays in the host layer.
 *   req [dev] Pp x D      UNIQUE pending pods in dict order (duplicate uids collapsed, :119);
 *                         D must be 2, 4, 8 or 16 (zero columns are neutral)
 *   num_listed            len(pods) including duplicates (:120)
 *   unit [host] T x D     pool unit capacities, pools ALREADY in visiting order (capacity.py:34-36)
 *   pool_actual/pool_max [host] T int32, pool_ignored [host] T bytes
 *   out_new_size/out_units_needed/out_bins_opened [host] T int64 (units_needed = -1: pool skipped)
 *   out_acc_pool [dev] Pp int32 visiting index of the pool that accounted the pod, -1 = none
 *   out_bin_of   [dev] Pp int32 bin index inside the last pool that packed the pod, -1 = none
 *   out_unaccounted [host] one int64 (num_unaccounted at :179)
 *   out_evals [host] one uint64 (may be NULL): `.possible` evaluations (pool gate :134 + bins :139)
 */
ACSFIT_API acsfit_status acsfit_fulfill_pending(acsfit_ctx *ctx, const double *req, int64_t Pp,
                                     int64_t num_listed, int D, const double *unit,
                                     const int32_t *pool_actual, const int32_t *pool_max,
                                     const uint8_t *pool_ignored, int T, int64_t over_provision,
                                     int64_t *out_new_size, int64_t *out_units_needed,
                                     int64_t *out_bins_opened, int32_t *out_acc_pool,
                                     int32_t *out_bin_of, int64_t *out_unaccounted,
                                     uint64_t *out_evals, acsfit_stream_t stream);

/*
 * K6 node_states -- Scaler.get_node_state (reference scaler.py:61-114) for every node and S
 * idle thresholds at once.  The node's pods are run_idx[row_ptr[n]..row_ptr[n+1]) in
 * pods_by_node order (engine_scaler.py:129-131).
 *   flags_run [dev] R bytes (ACSFIT_PODF_*), node_flags [dev] N bytes (ACSFIT_NODEF_*),
 *   node_age [dev] N int64 seconds ((now - creation).seconds, scaler.py:78),
 *   any_pending = len(pods_to_schedule) > 0, idle_threshold [host] S int64,
 *   out_state [dev] S x N bytes.
 * A node with ACSFIT_NODEF_NO_PENDING_MATCH is classified as if any_pending were 0: the caller sets
 * it when no pod to schedule matches the node's nodeSelector labels, so POD_PENDING means "some
 * pending pod could land here" (upstream ec2-autoscaler get_node_state).  A caller that never sets
 * the bit gets the reference's "any pod to schedule" rule.  acsfit_maintain_host reads the same bits.
 */
ACSFIT_API acsfit_status acsfit_node_states(acsfit_ctx *ctx, const int64_t *row_ptr, const int32_t *run_idx,
                                 const double *req_run, const uint8_t *flags_run,
                                 const double *cap_type, const int32_t *node_type,
                                 const uint8_t *node_flags, const int64_t *node_age, int64_t N,
                                 int D, int any_pending, const int64_t *idle_threshold, int S,
                                 uint8_t *out_state, acsfit_stream_t stream);

/*
 * Pending-pod admission with required pod anti-affinity (opt-in): sets ACSFIT_NODEF_NO_PENDING_MATCH on every node
 * that no pod to schedule could land on, for acsfit_node_states.  NC(n) / NX(n) are the OR of the carries / matches
 * masks (acsfit_anti_affinity's term numbering) over the pods already on node n.  A signature (class c, carries,
 * matches) admits node n when bit c of node_match[n] is set and (carries & NX(n)) | (matches & NC(n)) == 0, the
 * scheduler's block test in both directions.  The host passes the DISTINCT signatures of the pods to schedule, so a
 * node admits some pod to schedule exactly when some signature admits it.  A node no signature admits gains the flag
 * bit; every other bit of node_flags_inout is left as it is.  A node with no pods is blocked by nothing.
 *   row_ptr     [dev] N+1 int64: the pods of node n are rows row_ptr[n] .. row_ptr[n+1] of the run masks (absolute
 *               row numbers: row_ptr[0] may be > 0); this is the contiguous node-order table of acsfit_node_states
 *   run_carries, run_matches [dev] one mask per row (may be NULL when row_ptr[N] == row_ptr[0])
 *   node_match  [dev] N class masks as in acsfit_selectors, or NULL: every node matches every class
 *   sig_class   [host] U bytes, each < ACSFIT_MAX_CLASSES; sig_carries, sig_matches [host] U masks each
 *   node_flags_inout [dev] N bytes (ACSFIT_NODEF_*)
 * U may be 0 (every node gains the flag) and has no upper bound: the kernel stages the table through shared memory
 * in tiles.  row_ptr and the [dev] masks must be 8-byte aligned.  ACSFIT_E_INVALID: N < 0, U < 0, a class >= 64, a
 * NULL array that is read, a misaligned array, or row_ptr[N] < row_ptr[0].  The call synchronises the stream (the
 * table is a host buffer).  acsfit_last_scan_launch reports the launch as kernel 3.
 */
ACSFIT_API acsfit_status acsfit_pending_admit(acsfit_ctx *ctx, const int64_t *row_ptr, const uint64_t *run_carries,
                                              const uint64_t *run_matches, int64_t N, const uint64_t *node_match,
                                              const uint8_t *sig_class, const uint64_t *sig_carries,
                                              const uint64_t *sig_matches, int U, uint8_t *node_flags_inout,
                                              acsfit_stream_t stream);

/*
 * Pending-pod admission with required pod affinity (opt-in), with or without anti-affinity: acsfit_pending_admit
 * plus the affinity test.  HAS(n) is the OR of run_has (the pod-affinity signatures each pod matches, acsfit's
 * pod-affinity numbering) over the pods already on node n.  A signature (class c, carries, matches, need) admits node n
 * when acsfit_pending_admit's test passes (only the class test when the anti-affinity arrays are NULL) and need == 0 or
 * (need & HAS(n)) != 0.  need is the pod's signature bit, or 0 for a pod without pod-affinity terms and for the first
 * pod of a self-affine group (the host folds that exception in: no pod in the cluster matches the signature yet and
 * the pod matches it itself).
 *   run_carries, run_matches, sig_carries, sig_matches: all four NULL (the affinity test alone; the anti-affinity
 *               masks are never read) or given as in acsfit_pending_admit (the run pair may be NULL when there are no
 *               rows, the signature pair when U == 0)
 *   run_has     [dev] one mask per row (may be NULL when row_ptr[N] == row_ptr[0])
 *   sig_need    [host] U masks
 * The other arguments are those of acsfit_pending_admit.  ACSFIT_E_INVALID: its refusals (with the anti-affinity
 * test: a NULL run_carries or run_matches when there are rows, a NULL sig_carries or sig_matches when U > 0), a NULL
 * run_has when there are rows, a NULL sig_need when U > 0, or a misaligned run_has; the flags are then left untouched.  acsfit_last_scan_launch reports the launch as kernel 4.
 */
ACSFIT_API acsfit_status acsfit_pending_admit_pa(acsfit_ctx *ctx, const int64_t *row_ptr, const uint64_t *run_carries,
                                                 const uint64_t *run_matches, const uint64_t *run_has, int64_t N,
                                                 const uint64_t *node_match, const uint8_t *sig_class,
                                                 const uint64_t *sig_carries, const uint64_t *sig_matches,
                                                 const uint64_t *sig_need, int U, uint8_t *node_flags_inout,
                                                 acsfit_stream_t stream);

/*
 * K6b maintain_actions -- the decision part of EngineScaler.maintain (reference
 * engine_scaler.py:133-182): SPARE_AGENT substitution against the per-pool drain budget
 * (budget0 = actual - len(unschedulable) - spare, :136; it only decrements when not dry_run,
 * :154-159) and the state -> action table.
 *   io_state [dev] N bytes (rewritten; nodes of non-scalable pools become ACSFIT_ST_NOT_EVALUATED)
 *   node_pool [dev] N int32, budget0 [host] T int64, pool_scalable [host] T bytes,
 *   out_action [dev] N bytes (ACSFIT_ACT_*).
 */
ACSFIT_API acsfit_status acsfit_maintain_actions(acsfit_ctx *ctx, uint8_t *io_state, const int32_t *node_pool,
                                      int64_t N, const int64_t *budget0,
                                      const uint8_t *pool_scalable, int T, int dry_run,
                                      uint8_t *out_action, acsfit_stream_t stream);

/*
 * Fused scale-up tick on DEVICE buffers: get_pods_to_schedule + get_pending_pods +
 * fulfill_pending (reference cluster.py:169-175, :206-215).  Precondition: pod uids are unique
 * (otherwise the host layer applies the dict collapse of scaler.py:119 between the individual
 * entry points).  D must be 2, 4, 8 or 16.
 *   in : req [dev] P x D (pending-unassigned pods, list order)
 *        unit_all [host] T x D in agent_pools order (feasibility, capacity.py:24-32)
 *        unit_ordered / pool_actual / pool_max / pool_ignored [host] in VISITING order
 *        cap_type [dev] K x D, node_type [dev] N, used_inout [dev] N x D
 *   out: out_feasible [dev] P bytes
 *        out_placed   [dev] P int32: node index, -1 = pending, -2 = infeasible (skipped)
 *        out_new_size / out_units_needed / out_bins_opened [host] T int64
 *        out_acc_pool [dev] P int32: visiting index of the pool that accounted the pod, else -1
 *        out_counters [host] 4 x uint64 = {pods to schedule, pending, num_unaccounted, decisions}
 *        where decisions = every `.possible` / can_fit evaluation the reference would perform.
 */
ACSFIT_API acsfit_status acsfit_scale_up(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                              const double *unit_all, const double *unit_ordered,
                              const int32_t *pool_actual, const int32_t *pool_max,
                              const uint8_t *pool_ignored, int T, int64_t over_provision,
                              const double *cap_type, const int32_t *node_type, double *used_inout,
                              int64_t N, uint8_t *out_feasible, int32_t *out_placed,
                              int64_t *out_new_size, int64_t *out_units_needed,
                              int64_t *out_bins_opened, int32_t *out_acc_pool,
                              uint64_t *out_counters, acsfit_stream_t stream);

/*
 * Host-buffer entry points (the "plugin" calls): the same computations with HOST pointers
 * everywhere; the library copies H2D (fastest from pinned memory), runs the kernels on the
 * default stream and copies the results back before returning.
 * acsfit_scale_up_host = acsfit_scale_up with host buffers (cap_type has K rows).
 */
ACSFIT_API acsfit_status acsfit_scale_up_host(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                   const double *unit_all, const double *unit_ordered,
                                   const int32_t *pool_actual, const int32_t *pool_max,
                                   const uint8_t *pool_ignored, int T, int64_t over_provision,
                                   const double *cap_type, int K, const int32_t *node_type,
                                   double *used_inout, int64_t N, uint8_t *out_feasible,
                                   int32_t *out_placed, int64_t *out_new_size,
                                   int64_t *out_units_needed, int64_t *out_bins_opened,
                                   int32_t *out_acc_pool, uint64_t *out_counters);

/*
 * Node selectors (opt-in): the scale-up decision honours the pods' spec.nodeSelector, with the rules of the upstream
 * ec2 autoscaler the reference descends from:
 *   feasibility   a pod is schedulable when some agent pool (ignored pools included) matches its selector AND
 *                 (unit - req).possible
 *   first fit     the first node in list order with node.is_match(pod) and node.can_fit(pod.resources) takes it
 *   bin packing   the pool gate of fulfill_pending is "pool matches AND (unit - req).possible"; bins, clamp
 *                 arithmetic and accounting are unchanged (every new node of a pool carries the pool's labels)
 *   counters      unchanged formulas: one evaluation per (pod, node) pair or (pod, pool) visited, one per gate
 *                 and bin test (the match is evaluated first and short-circuits; it is not an extra evaluation)
 * The host maps every distinct match signature (set of matching nodes, set of matching pools) to a class number
 * < classes <= ACSFIT_MAX_CLASSES.  Class 0 = no selector: its bit must be set in every mask (checked: pool masks on
 * the host, node masks on the device, ACSFIT_E_INVALID otherwise).  A pod may take a node / pool exactly when bit
 * pod_class of that mask is set.
 *   pod_class          [dev] one byte per row of req (indexed like req rows), each < classes (else ACSFIT_E_INVALID)
 *   node_match         [dev] N masks
 *   pool_match_all     [host] T masks in agent_pools order (feasibility)
 *   pool_match_ordered [host] T masks in VISITING order (pool gate of fulfill_pending)
 * In acsfit_scale_up_sel_host pod_class and node_match are host pointers too.  An entry point reads only the
 * fields it needs.  Scope: the node pass with selectors runs the barrier form of the pipeline kernel only (it
 * ignores the "stream" knob: acsfit_last_launches shows form 0), and cluster mode (world > 1) refuses the
 * *_sel entry points with ACSFIT_E_INVALID.
 */
#define ACSFIT_MAX_CLASSES 64
typedef struct acsfit_selectors {
    const uint8_t *pod_class;
    const uint64_t *node_match;
    const uint64_t *pool_match_all;
    const uint64_t *pool_match_ordered;
    int classes;
} acsfit_selectors;

/* the selector forms of the entry points above: the same arguments plus `sel`, the same outputs */
ACSFIT_API acsfit_status acsfit_feasible_mask_sel(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                                  const double *unit, int T, const acsfit_selectors *sel,
                                                  uint8_t *out_mask, uint64_t *out_evals, acsfit_stream_t stream);
ACSFIT_API acsfit_status acsfit_first_fit_nodes_sel(acsfit_ctx *ctx, const double *req, int64_t req_rows,
                                                    const int32_t *pod_idx, int64_t P, int D, const double *cap_type,
                                                    const int32_t *node_type, double *used_inout, int64_t N,
                                                    const acsfit_selectors *sel, int32_t *out_placed,
                                                    uint64_t *out_decisions, acsfit_stream_t stream);
ACSFIT_API acsfit_status acsfit_fulfill_pending_sel(acsfit_ctx *ctx, const double *req, int64_t Pp,
                                                    int64_t num_listed, int D, const double *unit,
                                                    const int32_t *pool_actual, const int32_t *pool_max,
                                                    const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                    const acsfit_selectors *sel, int64_t *out_new_size,
                                                    int64_t *out_units_needed, int64_t *out_bins_opened,
                                                    int32_t *out_acc_pool, int32_t *out_bin_of,
                                                    int64_t *out_unaccounted, uint64_t *out_evals,
                                                    acsfit_stream_t stream);
/* including the chained node + first-bin-pass launch (when every pod to schedule is eligible for the first pool
 * visited, match included) and its watchdog redo */
ACSFIT_API acsfit_status acsfit_scale_up_sel(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                             const double *unit_all, const double *unit_ordered,
                                             const int32_t *pool_actual, const int32_t *pool_max,
                                             const uint8_t *pool_ignored, int T, int64_t over_provision,
                                             const double *cap_type, const int32_t *node_type, double *used_inout,
                                             int64_t N, const acsfit_selectors *sel, uint8_t *out_feasible,
                                             int32_t *out_placed, int64_t *out_new_size, int64_t *out_units_needed,
                                             int64_t *out_bins_opened, int32_t *out_acc_pool,
                                             uint64_t *out_counters, acsfit_stream_t stream);
ACSFIT_API acsfit_status acsfit_scale_up_sel_host(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                                  const double *unit_all, const double *unit_ordered,
                                                  const int32_t *pool_actual, const int32_t *pool_max,
                                                  const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                  const double *cap_type, int K, const int32_t *node_type,
                                                  double *used_inout, int64_t N, const acsfit_selectors *sel,
                                                  uint8_t *out_feasible, int32_t *out_placed,
                                                  int64_t *out_new_size, int64_t *out_units_needed,
                                                  int64_t *out_bins_opened, int32_t *out_acc_pool,
                                                  uint64_t *out_counters);

/*
 * Required pod anti-affinity (opt-in): spec.affinity.podAntiAffinity.requiredDuringSchedulingIgnoredDuringExecution
 * terms with topologyKey kubernetes.io/hostname.  The host numbers the distinct terms (at most ACSFIT_MAX_AA_TERMS);
 * bit k of a mask is term k.  Per pod: pod_carries = the terms it has, pod_matches = the terms that select it.  Per
 * node (bin): the OR of both over the pods on it, which the pass updates as it places pods.  A pod is blocked on a node
 * when (pod_carries & node_matches) | (pod_matches & node_carries) != 0, the scheduler's check in both directions.
 *   first fit     the first node in list order that is not blocked, matches (with `sel`) and can_fit takes the pod;
 *                 both masks of that node then gain the pod's bits
 *   bin packing   the same over the bins; a new bin starts with both masks 0.  The pool gate, the clamp arithmetic
 *                 and the accounting are unchanged
 *   counters      unchanged formulas (the block test is evaluated first and short-circuits)
 *   pod_carries, pod_matches   [dev] one mask per row of req (indexed like req rows)
 *   node_carries, node_matches [dev] N masks each, read and written (node pass only; the bin pass ignores them)
 * acsfit_first_fit_nodes_aa takes the arguments of acsfit_first_fit_nodes_sel with `sel` allowed to be NULL (every
 * pod in class 0, every node matching); acsfit_fulfill_pending_aa those of acsfit_fulfill_pending_sel with `sel`
 * allowed to be NULL (plain pool gate).  Cost: the node pass always runs the selector form of the pipeline kernel,
 * with trivial classes when `sel` is NULL, plus the block test: at 100 000 pods x 10 000 nodes, D = 4, it took 4.7 ms
 * against 2.9 ms for acsfit_first_fit_nodes (H100 80GB HBM3, 700 W limit); the bin passes 9.3 ms against 7.5 ms.  Both run the barrier form of the pipeline kernel, unchained (they ignore the
 * "stream" knob), and refuse with ACSFIT_E_INVALID: a NULL mask array that is read, the `sel` checks of the *_sel
 * forms, and cluster mode (world > 1).
 */
#define ACSFIT_MAX_AA_TERMS 64
typedef struct acsfit_anti_affinity {
    const uint64_t *pod_carries, *pod_matches;  /* [dev] one per row of req */
    uint64_t *node_carries, *node_matches;      /* [dev] N each, in/out (node pass only) */
} acsfit_anti_affinity;

ACSFIT_API acsfit_status acsfit_first_fit_nodes_aa(acsfit_ctx *ctx, const double *req, int64_t req_rows,
                                                   const int32_t *pod_idx, int64_t P, int D, const double *cap_type,
                                                   const int32_t *node_type, double *used_inout, int64_t N,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   int32_t *out_placed, uint64_t *out_decisions,
                                                   acsfit_stream_t stream);
ACSFIT_API acsfit_status acsfit_fulfill_pending_aa(acsfit_ctx *ctx, const double *req, int64_t Pp,
                                                   int64_t num_listed, int D, const double *unit,
                                                   const int32_t *pool_actual, const int32_t *pool_max,
                                                   const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   int64_t *out_new_size, int64_t *out_units_needed,
                                                   int64_t *out_bins_opened, int32_t *out_acc_pool,
                                                   int32_t *out_bin_of, int64_t *out_unaccounted,
                                                   uint64_t *out_evals, acsfit_stream_t stream);

/*
 * Required pod affinity (opt-in): spec.affinity.podAffinity.requiredDuringSchedulingIgnoredDuringExecution terms with
 * topologyKey kubernetes.io/hostname.  A pod's signature is the set of its honoured terms; the host numbers the
 * distinct signatures of the pods to place (at most ACSFIT_MAX_PA_SIGNATURES), bit s = signature s.  A pod matches a
 * signature when every term of it selects the pod.  Per pod: pod_requires = its signature's bit (0: no constraint),
 * pod_matches = the signatures it matches, pod_self = pod_requires & pod_matches.  Per node: node_has = the OR of
 * pod_matches over the pods on it, which the pass updates as it places pods; a new bin starts with 0.
 *   rule          a pod with pod_requires != 0 may take a node (bin) only when (pod_requires & node_has) != 0, or
 *                 (bootstrap) when no pod anywhere matches its signature at its turn and it matches it itself.
 *                 "Anywhere": every node of the node pass, the signatures `present` names (fulfill: what the node pass
 *                 left, typically the OR of node_has), and every bin opened so far in this call, pool after pool.
 *                 The rule is one-way (placed pods' terms never constrain the incoming pod) and ANDs with resources,
 *                 `sel` and `aa`
 *   bin packing   a pod the rule keeps out of every bin, a new one included, opens no bin and is credited no bin
 *                 test; the passes over fresh bins stop once a pass places no pod, and such pods stay unaccounted
 *                 for the pool (they go on to the next pool)
 *   counters      otherwise unchanged formulas (the affinity test is evaluated first and short-circuits)
 *   exactness     the bootstrap exception depends on global order, so a pass runs with a flip position per
 *                 signature absent at its start (+inf at first); a pod at position pos treats signature s as absent
 *                 iff pos <= flip[s].  After a pass the earliest placement of a pod matching a still unfixed such
 *                 signature fixes flip[s] there, and the pass (node pass: from its saved state; bins: the pool's whole
 *                 packing) is run again.  Pods up to that position decide as before, so the result is the sequential
 *                 scheduler's after at most 1 + (absent self-affine signatures that get placed) passes, and after one
 *                 pass when no signature is absent (acsfit_last_affinity_reruns)
 *   pod_requires, pod_self, pod_matches   [dev] one per row of req
 *   node_has      [dev] N masks, read and written (node pass only; fulfill ignores it)
 * acsfit_first_fit_nodes_pa / acsfit_fulfill_pending_pa take the arguments of the *_aa forms with `sel` and `aa` both
 * allowed to be NULL, plus `pa` and (fulfill) `present`.  They run the anti-affinity form of the pipeline kernel with
 * the affinity test added (zero anti-affinity masks when `aa` is NULL), barrier form only and unchained, and refuse
 * with ACSFIT_E_INVALID: a NULL `pa` or mask array that is read, the checks of `sel` and `aa`, and cluster mode.
 */
#define ACSFIT_MAX_PA_SIGNATURES 64
typedef struct acsfit_pod_affinity {
    const uint64_t *pod_requires, *pod_self, *pod_matches;  /* [dev] one per row of req */
    uint64_t *node_has;                                     /* [dev] N, in/out (node pass only) */
} acsfit_pod_affinity;

ACSFIT_API acsfit_status acsfit_first_fit_nodes_pa(acsfit_ctx *ctx, const double *req, int64_t req_rows,
                                                   const int32_t *pod_idx, int64_t P, int D, const double *cap_type,
                                                   const int32_t *node_type, double *used_inout, int64_t N,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   const acsfit_pod_affinity *pa, int32_t *out_placed,
                                                   uint64_t *out_decisions, acsfit_stream_t stream);
ACSFIT_API acsfit_status acsfit_fulfill_pending_pa(acsfit_ctx *ctx, const double *req, int64_t Pp,
                                                   int64_t num_listed, int D, const double *unit,
                                                   const int32_t *pool_actual, const int32_t *pool_max,
                                                   const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   const acsfit_pod_affinity *pa, uint64_t present,
                                                   int64_t *out_new_size, int64_t *out_units_needed,
                                                   int64_t *out_bins_opened, int32_t *out_acc_pool,
                                                   int32_t *out_bin_of, int64_t *out_unaccounted,
                                                   uint64_t *out_evals, acsfit_stream_t stream);
/* test hook: passes the last *_pa call ran again (each fixes one flip) and those flips in order: out_flips[2k] =
 * signature, out_flips[2k + 1] = position (fulfill: pending position; 2 * *out_reruns entries; may be NULL) */
ACSFIT_API acsfit_status acsfit_last_affinity_reruns(const acsfit_ctx *ctx, int64_t *out_reruns, int64_t *out_flips);

/*
 * Hostname topology spread (opt-in): spec.topologySpreadConstraints with topologyKey kubernetes.io/hostname and
 * whenUnsatisfiable DoNotSchedule (at most one per pod).  The host numbers the distinct keys (namespace, selector with
 * the matchLabelKeys values, domain set) of the pods to place, at most ACSFIT_MAX_TS_KEYS, bit k = key k.
 *   cnt(k, n)     the pods on node n that key k's selector selects; the pass adds 1 for every key of pod_matches
 *                 when it places a pod.  A new bin starts at 0
 *   min(k)        the smallest cnt(k, n) over k's domains: the nodes with bit k in node_domain, and the domains
 *                 outside the node list (non-agent nodes) whose smallest count the host folds into floor[k]
 *                 (INT32_MAX: none; 0 when k has fewer domains than its minDomains)
 *   rule          a pod with pod_key = k (0xFF: none) may take node n only when cnt(k, n) <= pod_skew + min(k),
 *                 pod_skew = maxSkew - (1 if k's selector selects the pod itself else 0) >= 0.  In the bins min(k) is
 *                 taken as 0 (a scale-up's new nodes join empty), so a new node takes at most maxSkew self-selecting
 *                 pods of a key, which may ask for more nodes than the scheduler needs, never fewer.  ANDs with
 *                 resources, `sel`, `aa` and `pa`; counters otherwise unchanged
 *   exactness     min(k) rises as the node pass places pods.  The pass runs with a level per key and position, which
 *                 rises at the fixed rise positions; it watches each key's next rise (every domain of the list at
 *                 level + 1, unless floor[k] is below that), and the earliest rise or pod-affinity flip it observes is
 *                 fixed and the pass run again from its saved state: exact after 1 + rises + flips passes, and after
 *                 one pass when no key can rise (acsfit_last_spread_rises).  After 4096 fixed rises in one call
 *                 no further rise is watched: the rest of the pass keeps the last fixed levels, which are at most the
 *                 true minimums (the pass then refuses pods the scheduler would place, and is no longer exact)
 *   pod_key, pod_skew, pod_matches   [dev] one per row of req
 *   node_count    [dev] keys x N (key-major), read and written (node pass only; fulfill ignores it)
 *   node_domain   [dev] N (node pass only)
 *   floor         [host] keys (node pass only)
 * acsfit_pending_admit_ts reads node_count (read only), node_domain, floor and keys, and none of the pod_* fields.
 * acsfit_first_fit_nodes_ts / acsfit_fulfill_pending_ts take the arguments of the *_pa forms with `sel`, `aa` and `pa`
 * all allowed to be NULL, plus `ts`.  They run the pod-affinity form of the pipeline kernel with the spread test
 * added, and refuse with ACSFIT_E_INVALID: a NULL `ts` or array that is read, keys outside [0, 64], a pod_key >= keys
 * other than 0xFF, a pod_matches bit at or above keys, a negative pod_skew, node count or floor, the checks of `sel`, `aa` and `pa`, and cluster mode.
 */
#define ACSFIT_MAX_TS_KEYS 64
typedef struct acsfit_topology_spread {
    const uint8_t *pod_key;        /* [dev] one per row of req: the pod's key, 0xFF none */
    const int32_t *pod_skew;       /* [dev] one per row of req: maxSkew - self */
    const uint64_t *pod_matches;   /* [dev] one per row of req: the keys whose selector selects the pod */
    int32_t *node_count;           /* [dev] keys x N, in/out (node pass only) */
    const uint64_t *node_domain;   /* [dev] N: the keys each node is a domain of (node pass only) */
    const int32_t *floor;          /* [host] keys (node pass only) */
    int32_t keys;
} acsfit_topology_spread;

ACSFIT_API acsfit_status acsfit_first_fit_nodes_ts(acsfit_ctx *ctx, const double *req, int64_t req_rows,
                                                   const int32_t *pod_idx, int64_t P, int D, const double *cap_type,
                                                   const int32_t *node_type, double *used_inout, int64_t N,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   const acsfit_pod_affinity *pa, const acsfit_topology_spread *ts,
                                                   int32_t *out_placed, uint64_t *out_decisions, acsfit_stream_t stream);
ACSFIT_API acsfit_status acsfit_fulfill_pending_ts(acsfit_ctx *ctx, const double *req, int64_t Pp,
                                                   int64_t num_listed, int D, const double *unit,
                                                   const int32_t *pool_actual, const int32_t *pool_max,
                                                   const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   const acsfit_pod_affinity *pa, uint64_t present,
                                                   const acsfit_topology_spread *ts, int64_t *out_new_size,
                                                   int64_t *out_units_needed, int64_t *out_bins_opened,
                                                   int32_t *out_acc_pool, int32_t *out_bin_of,
                                                   int64_t *out_unaccounted, uint64_t *out_evals,
                                                   acsfit_stream_t stream);
/*
 * Pending-pod admission with hostname topology spread (opt-in), with or without anti-affinity and pod affinity:
 * acsfit_pending_admit_pa's tests plus the spread test.  A signature (class, carries, matches, need, key, skew) admits
 * node n when the enabled tests of acsfit_pending_admit_pa pass and key == 0xFF or node_count[key * N + n] <= skew +
 * min(key), the rule of acsfit_topology_spread with nothing placed (each pending pod is judged on its own, so no
 * minimum rises).  key and skew are the pod's pod_key and pod_skew.
 *   run_carries, run_matches, sig_carries, sig_matches: all four NULL (no anti-affinity test) or given as in
 *               acsfit_pending_admit
 *   run_has, sig_need: both NULL (no affinity test) or given as in acsfit_pending_admit_pa
 *   sig_key     [host] U bytes: the signature's key, 0xFF none; sig_skew [host] U int32 >= 0
 *   ts          node_count (read only here), node_domain, floor and keys of acsfit_topology_spread over these N nodes;
 *               pod_key, pod_skew and pod_matches are not read (the signatures carry key and skew).  node_count
 *               must be 4-byte and node_domain 8-byte aligned
 * The limit skew + min(key) is computed in 64 bits and clamped to INT32_MAX, so a key without any domain (min
 * INT32_MAX) admits every node.  The other arguments are those of acsfit_pending_admit.  ACSFIT_E_INVALID: the
 * refusals of acsfit_pending_admit_pa for the tests that run, a NULL ts, keys outside [0, 64], a NULL node_count or
 * node_domain when N > 0 and keys > 0, a NULL floor when keys > 0, a NULL sig_key or sig_skew when U > 0, a sig_key
 * >= keys other than 0xFF, a negative sig_skew, floor or node count, a misaligned node_count or node_domain; the flags
 * are then left untouched.  acsfit_last_scan_launch reports the launch as kernel 5.
 */
ACSFIT_API acsfit_status acsfit_pending_admit_ts(acsfit_ctx *ctx, const int64_t *row_ptr, const uint64_t *run_carries,
                                                 const uint64_t *run_matches, const uint64_t *run_has, int64_t N,
                                                 const uint64_t *node_match, const uint8_t *sig_class,
                                                 const uint64_t *sig_carries, const uint64_t *sig_matches,
                                                 const uint64_t *sig_need, const uint8_t *sig_key,
                                                 const int32_t *sig_skew, int U, const acsfit_topology_spread *ts,
                                                 uint8_t *node_flags_inout, acsfit_stream_t stream);
/* test hook: the rises the last *_ts call fixed, in order: out_pairs[2k] = key, out_pairs[2k + 1] = position (the
 * node pass's list entry after which the key's minimum rose; 2 * *out_rises entries; may be NULL) */
ACSFIT_API acsfit_status acsfit_last_spread_rises(const acsfit_ctx *ctx, int64_t *out_rises, int64_t *out_pairs);

/* acsfit_occupancy_host = acsfit_occupancy with host buffers (reference cluster.py:165-168): R rows of req_run,
 * used_inout N x D is read, updated and written back. */
ACSFIT_API acsfit_status acsfit_occupancy_host(acsfit_ctx *ctx, const int64_t *row_ptr, const int32_t *run_idx,
                                    const double *req_run, int64_t R, int64_t N, int D, double *used_inout);

/* acsfit_maintain_host = node_states (one threshold) + maintain_actions with host buffers
 * (reference engine_scaler.py:120-182, scaler.py:61-114). out_state/out_action N bytes. */
ACSFIT_API acsfit_status acsfit_maintain_host(acsfit_ctx *ctx, const int64_t *row_ptr, const int32_t *run_idx,
                                   const double *req_run, const uint8_t *flags_run, int64_t R,
                                   const double *cap_type, int K, const int32_t *node_type,
                                   const uint8_t *node_flags, const int64_t *node_age,
                                   const int32_t *node_pool, int64_t N, int D, int any_pending,
                                   int64_t idle_threshold, const int64_t *budget0,
                                   const uint8_t *pool_scalable, int T, int dry_run,
                                   uint8_t *out_state, uint8_t *out_action);

/*
 * Cluster mode: ONE cluster (one pod list, one node list) on the `world` GPUs of one box, one process and one
 * ctx per GPU.  The two sequential first-fit loops (reference cluster.py:184-204 and scaler.py:131-147) are
 * parallel over the NODE (bin) axis, so rank r owns the r-th contiguous range of nodes (of every bin pass) and
 * the pipeline of stages simply continues on the next GPU: stage 0 of rank r polls the progress counter of the
 * last stage of rank r-1 and reads that rank's "still unplaced" bitmap, both through NVLink peer memory
 * (CUDA IPC), tile by tile, inside the kernel.  Pods visit nodes in list order and every node sees the pods in
 * list order, so placements, `used` bit patterns, pool sizes and the credited decisions are exactly those of
 * the single-GPU call.  The only other exchanges are in-stream peer-memory barriers and element-wise merges of
 * the placement vectors (each pod is placed by exactly one rank).
 *
 * Protocol: every rank calls acsfit_cluster_init, the 64-byte handles are all-gathered by the host layer
 * (torch.distributed) and passed to acsfit_cluster_connect.  From then on acsfit_first_fit_nodes,
 * acsfit_fulfill_pending, acsfit_scale_up and acsfit_scale_up_host must be called by ALL ranks with IDENTICAL
 * arguments (replicated inputs); every rank returns the complete, identical result.
 *   max_pods / max_nodes / max_dims size the exchange region this rank exports (cudaMalloc'ed by the library).
 */
#define ACSFIT_IPC_HANDLE_BYTES 64
#define ACSFIT_MAX_RANKS 8
ACSFIT_API acsfit_status acsfit_cluster_init(acsfit_ctx *ctx, int rank, int world, int64_t max_pods,
                                             int64_t max_nodes, int max_dims, void *out_handle);
/* all_handles [host]: world x ACSFIT_IPC_HANDLE_BYTES, rank-major (this rank's own entry included) */
ACSFIT_API acsfit_status acsfit_cluster_connect(acsfit_ctx *ctx, const void *all_handles);
/* in-stream barrier over the ranks (peer-memory flags); the first call must follow a host-level barrier */
ACSFIT_API acsfit_status acsfit_cluster_barrier(acsfit_ctx *ctx, acsfit_stream_t stream);
/* geometry of the last cluster-mode node pass: stage width, stages of this rank, pod blocks, resident stage CTAs */
ACSFIT_API acsfit_status acsfit_cluster_last_plan(const acsfit_ctx *ctx, int *out_tn, int *out_stages,
                                                  int *out_blocks, int *out_resident);

/* number of kernels this ctx has launched so far (bench.py reports it as gpu_launches) */
ACSFIT_API uint64_t acsfit_launch_count(const acsfit_ctx *ctx);
/* CUDA-event time (ms) of the last first-fit / bin-pack pipeline kernel sequence and the
 * decisions it evaluated, measured on the launching stream (bench.py roofline leg) */
ACSFIT_API acsfit_status acsfit_last_pipeline_stats(const acsfit_ctx *ctx, double *out_ms,
                                         uint64_t *out_decisions, int *out_stages, int *out_tiles);

/* test hook (read-only): the first-fit pipeline kernels the last API call on this ctx launched, in launch order,
 * one record of ACSFIT_LAUNCH_FIELDS ints each, as launched (not as planned):
 *   {pass (0 nodes, 1 bins), chained (1: node pass and first bin pass launched together on two streams), D,
 *    RW (packed-rank words per row; 0 = float64 compare scan), prune (0/1), form (0 barrier, 1 streaming),
 *    Tn (nodes / bins per stage), stages, resident (stage CTAs of this instantiation the GPU holds at once),
 *    pool (visiting index; -1 for node passes), bin_base (first bin of the pass, clamped to INT32_MAX; -1 for
 *    node passes), publish_every (barrier form: tiles between progress publications of an idle stage; 0 for the
 *    streaming form)}
 * At most max_records records are written to out; *out_n receives the number of records there are. */
#define ACSFIT_LAUNCH_FIELDS 12
ACSFIT_API acsfit_status acsfit_last_launches(const acsfit_ctx *ctx, int *out, int max_records, int *out_n);

/* test hook (read-only): the K1 (occupancy) / K6 (node states) kernel the last API call on this ctx launched, as
 * launched, one record of ACSFIT_SCAN_FIELDS ints written to out:
 *   {kernel (0 none, 1 occupancy, 2 node states), form (0 per thread, 1 index gather, 2 bulk copy), D,
 *    staging bytes per warp (0 per thread), warps per CTA, table entries per staging chunk (0 per thread),
 *    grid (CTAs), S (idle thresholds; 0 for occupancy)}
 * acsfit_pending_admit reports {3, 0, 0, shared-memory bytes per CTA, warps per CTA, signatures per tile, grid, U};
 * acsfit_pending_admit_pa {4, 1 with the anti-affinity test (0 without), 0, shared-memory bytes per CTA, warps per CTA,
 * signatures per tile, grid, U}; acsfit_pending_admit_ts {5, 1 with the anti-affinity test | 2 with the affinity test,
 * 0, shared-memory bytes per CTA, warps per CTA, signatures per tile, grid, U}. */
#define ACSFIT_SCAN_FIELDS 8
ACSFIT_API acsfit_status acsfit_last_scan_launch(const acsfit_ctx *ctx, int *out);

/* test hook (read-only): the pods the candidate scan of the last call's selector node passes handed to the resolver,
 * summed over tiles and stages (a pod counts once per stage in which some node fits it AND matches its class); 0 after a
 * call without a selector node pass */
ACSFIT_API acsfit_status acsfit_last_sel_hits(const acsfit_ctx *ctx, uint64_t *out);

/* test hook (read-only): what bin retirement marked in the last API call's bin passes (barrier form with rank tables,
 * the chained first pass of scale_up included; in cluster mode this rank's stages only):
 *   out[0] = resolver warps whose 32 bins were all dead when their stage exited, summed over stages and passes,
 *   out[1] = stages whose warps were all dead at exit.
 * A warp is dead when every bin of it holds a pod and is below the call's smallest request in some dimension.  Both are
 * 0 after a call without such a pass, with knob "retire" = 0, or for passes that hit the watchdog. */
ACSFIT_API acsfit_status acsfit_last_bin_retirement(const acsfit_ctx *ctx, uint64_t out[2]);

/* developer probes (tools/perf_probe.py): per-stage clock64 phase totals [stages][8] of the last
 * pipeline launch (wait, load, scan, resolve, publish, refresh, hits, tiles) and a per-tile trace
 * [tiles][8] of one chosen stage.  Enabling them adds a clock read per phase on thread 0. */
ACSFIT_API acsfit_status acsfit_debug_profile(acsfit_ctx *ctx, int enabled, unsigned long long *out,
                                              int max_stages, int *out_stages);
ACSFIT_API acsfit_status acsfit_debug_trace(acsfit_ctx *ctx, int stage, unsigned long long *out,
                                            int max_tiles);

#ifdef __cplusplus
}
#endif
#endif /* ACSFIT_H */
