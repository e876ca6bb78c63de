// acsfit_kernels.cuh -- sm_90a kernels of the pod-fit path (no tensor cores: this is
// compare / reduce work on float64, see DESIGN.md).
//
// The centrepiece is firstfit_pipeline_kernel: an EXACT, order-preserving parallelisation of
// the reference's two sequential first-fit loops
//     Cluster.get_pending_pods   autoscaler/cluster.py:184-204   (nodes, state = used)
//     Scaler.fulfill_pending     autoscaler/scaler.py:131-147    (bins,  state = remaining)
// as a systolic pipeline over the node (bin) axis:
//
//   * the node list is cut into consecutive STAGES of Tn nodes; one CTA owns one stage and
//     keeps that stage's per-node thresholds (acsfit_math.cuh) in shared memory / registers;
//   * the ordered pod list flows through the stages in TILES of 256 pods.  Stage s may
//     process tile i once stage s-1 has published it (a release/acquire counter in global
//     memory) - stage s works on tile i while stage s-1 already works on tile i+1;
//   * inside a tile, every (alive pod, node) pair of the stage is evaluated in parallel under
//     the tile-start state (pure DSETP work, pod rows broadcast from shared memory).  Because
//     a node only ever fills up (requests are >= 0, rounding is monotone) a pod that fits no
//     node of the stage under the tile-start state fits none later either: it is forwarded
//     untouched.  The few pods that do hit are resolved strictly in pod order by a chain of
//     warps (warp w = nodes 32w..32w+31 of the stage, state in registers, the literal reference
//     expression, one vote per entry), which is exactly the reference's loop restricted to this
//     stage's nodes;
//   * a pod that is placed has its alive bit cleared; pods still alive after the last stage
//     are the pending pods (nodes) / flow into the next pass of fresh bins (bins).
//
// Stage numbers are taken from an atomic ticket at CTA start, so stage s only ever waits for
// a CTA that is already running or finished: no co-residency assumption, no deadlock, and
// more stages than resident CTAs simply run as successive waves.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "acsfit_math.cuh"

namespace acsfit {

constexpr int kTile = 256;         // pods per tile == threads per CTA
constexpr int kThreads = 256;
// K: node rows a scanning thread keeps in registers.  float64 scan (NW == 0): K * D = 16 doubles whatever the
// dimension count.  Packed-rank scan (NW = 32-bit words per row, see RankLayout): K * NW = 8 words.
__host__ __device__ constexpr int nodes_per_thread(int D, int NW = 0)
{
    return NW == 0 ? (D <= 4 ? 4 : D <= 8 ? 2 : 1) : NW == 1 ? 8 : NW == 2 ? 4 : 2;
}
constexpr unsigned kNoCand = 0xFFFFFFFFu;
constexpr unsigned kQueueEnd = 0xFFFFFFFFu;
#ifndef ACSFIT_PROFILE
#define ACSFIT_PROFILE 0
#endif
constexpr bool kProfileBuild = ACSFIT_PROFILE != 0;
constexpr int kPublishEvery = 4;  // multi-wave passes: tiles between two progress publications of a stage that is not placing
constexpr int kPublishGrace = 8;  // ... once it has not placed anything for this many tiles
constexpr int kMinBatch = 4;  // entries a consumer warp waits for before it starts a batch
constexpr int kMaxDims = 16;
constexpr int kRing = 8;      // tiles whose alive words a stage fetches in one go once its upstream is that far ahead

// Packed-rank form of the scan predicate (SURVEY.md section 7, "rank compression").  Per resource dimension d the
// distinct request values of this tick's pod table are sorted; a pod's request is replaced by r' = 1 + its rank,
// a node's (bin's) scan threshold by t' = #{distinct values <= thr}.  Because every request value is IN the
// table,  req_d <= thr_d  <=>  r'_d <= t'_d  exactly.  All D fields of a row are packed into NW 32-bit words,
// each field followed by one guard bit; then
//        fits in every dimension  <=>  (((T | G) - R) & G) == G          (G = the guard bits)
// one integer subtract and one three-input logic op per word instead of D float64 compares per pair.  No field
// borrows from its neighbour: a field of (T | G) - R is 2^bits + t' - r' >= 1.  The resolver keeps evaluating
// the literal float64 reference expression; only the candidate scan uses ranks.
constexpr int kRankCap = 8192;     // distinct values per dimension the table can hold (else: float64 scan)
constexpr int kRankSlots = 32768;  // hash slots per dimension while the table is built
struct RankLayout {
    int nw;                        // words per row: 0 (not available), 1, 2 or 4
    uint32_t guard[4];             // G
    uint8_t word[16];              // word that holds dimension d
    uint8_t shift[16];             // bit position of its field
    int32_t count[16];             // U_d = number of distinct values
    const double *sorted;          // [D][kRankCap] ascending distinct values (device)
    const uint32_t *packed;        // [req rows][nw] packed pod ranks (device)
};

// t' = number of table values <= thr   (thr = -1: none fits -> 0; thr = +inf -> U)
__device__ __forceinline__ uint32_t rank_upper(const double *__restrict__ sorted_d, int U, double thr)
{
    int lo = 0, hi = U;  // invariant: sorted[< lo] <= thr, sorted[>= hi] > thr
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(sorted_d + mid) <= thr) lo = mid + 1; else hi = mid;
    }
    return (uint32_t)lo;
}

// the same search over a table a bin stage staged in shared memory (see kRankStaged)
__device__ __forceinline__ uint32_t rank_upper_shared(const double *sorted_d, int U, double thr)
{
    int lo = 0, hi = U;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (sorted_d[mid] <= thr) lo = mid + 1; else hi = mid;
    }
    return (uint32_t)lo;
}

// bin stages (RW > 0) copy the sorted values of every dimension with at most this many distinct values into shared
// memory at stage start: the threshold refresh after each placing tile then searches shared memory, not L2
constexpr int kRankStaged = 256;

struct PipelineParams {
    // pod side
    const double *req;      // rows of D doubles
    const int32_t *pod_idx; // list entry -> pod number, or nullptr (identity)
    const int32_t *row_map; // pod number -> row of req, or nullptr (identity)
    int64_t M;              // list length
    uint32_t *alive;        // ceil(M/32) words, bit = still unplaced (in/out)
    int32_t *placed;        // M entries, written with the GLOBAL node / bin index on placement
    // node side (nodes mode)
    const double *cap_type; // K x D
    const int32_t *node_type;
    double *used;           // N x D (in/out)
    // bin side (bins mode)
    const double *unit;     // D doubles (device)
    int64_t bin_base;       // global index of the first bin of this pass
    // geometry
    int64_t node_lo;        // first node (local numbering of stage 0 starts here)
    int64_t node_hi;        // one past the last node (nodes mode) / bin_base + stages*Tn (bins)
    int Tn;                 // nodes per stage (NS * K)
    int NS;                 // node slots = Tn / K (power of two, <= kThreads)
    int num_tiles;
    // synchronisation
    int *ticket;            // 1 int, zeroed
    int *progress;          // num_stages ints, zeroed: tiles published by the stage
    int *status;            // 1 int, zeroed: != 0 -> abort (watchdog)
    int *drained;           // 1 int, zeroed: set by the first stage that forwards no pod at all
    const int *upstream;    // optional: progress counter of ANOTHER pipeline's last stage that feeds stage 0
                            // of this one (bins pipeline chained behind the nodes pipeline; or the previous
                            // rank's pipeline in cluster mode, then a peer-memory pointer), or nullptr
    const uint32_t *alive_in; // optional: stage 0 reads the tile's alive words HERE (the upstream pipeline's
                            // bitmap in a peer GPU's memory) and always writes them to `alive`
    int sys_scope;          // cluster mode: upstream poll and the last stage's publish use system scope
    int publish_every;      // progress of a stage that is not placing is published every this many tiles (>= 1)
    int tile_lo;            // first tile of this launch in the pod list (pod blocks); tiles are numbered
                            // locally in the progress counters, globally in alive / placed / pod_idx
    RankLayout rk;          // packed-rank scan tables (rk.nw == NW of the instantiation)
    unsigned long long *evals; // bins mode: credited bin tests (atomicAdd)
    unsigned long long watchdog_ns;
    unsigned long long *prof;  // optional [stages][8] clock64 phase totals (developer probe), or nullptr
    unsigned long long *trace; // optional [num_tiles][8] per-tile trace of stage `trace_stage`
    int trace_stage;
    // node selectors (SEL instantiations of a node pass only; appended so that no other field moves):
    // a pod may take a node only when bit pod_class[row] of node_match[node] is set (class 0 = no selector,
    // its bit is set in every mask)
    const uint8_t *pod_class;               // [req rows] selector class of each request row
    const unsigned long long *node_match;   // [N] classes each node matches
    unsigned long long *sel_hits;           // optional: += the scan's hit entries of every tile of every stage
    // required pod anti-affinity (AA instantiations only; appended): bit k = term k.  A pod may take a node (bin) only
    // when (pod_carries & node_matches) | (pod_matches & node_carries) == 0; the taker ORs the pod's masks into the
    // node's.  Node passes read and write node_carries / node_matches; bins start at 0 and are not written back.
    const unsigned long long *pod_carries;  // [req rows] terms the pod has
    const unsigned long long *pod_matches;  // [req rows] terms that select the pod
    unsigned long long *node_carries;       // [N] in/out (node pass)
    unsigned long long *node_matches;       // [N] in/out (node pass)
    // bin passes with the packed-rank scan (RW > 0; appended): != 0 retires bins that can take no pod of the pass any
    // more, i.e. S[d] < the smallest request value of dimension d (rk.sorted[d * kRankCap]) in some d
    int retire;
    // bin passes with the packed-rank scan (appended; test hook acsfit_last_bin_retirement): [0] += warps whose bins
    // were all dead when their stage exited, [1] += stages whose warps were all dead.  nullptr: not counted
    unsigned long long *retire_count;
    // required pod affinity (PA instantiations, built on the AA form; appended).  A pod may take a node (bin) only when
    // its need is 0 or shares a bit with the node's node_has (the signatures the node's pods match); the taker ORs the
    // pod's pod_aff_matches into node_has.  pod_need is the pod's signature bit with the bootstrap exception already
    // applied (0 while the pod may land anywhere), indexed by position: list entry (node pass) or pending pod (bins).
    // Node passes read and write node_has; bins start at 0 and are not written back.
    const unsigned long long *pod_need;         // [positions]
    const unsigned long long *pod_aff_matches;  // [req rows] signatures the pod matches
    unsigned long long *node_has;               // [N] in/out (node pass)
    unsigned long long *first_placed;           // [64]: atomicMin of the position of each placed pod that matches a watched signature
    unsigned long long watch;                   // signatures whose first placement is recorded (0: none, nothing recorded)
    // hostname topology spread (TS instantiations, built on the PA form; appended).  A pod with a key (ts_key != 0xFF)
    // may take a node (bin) only when the node's count of that key is <= the pod's limit ts_lim (maxSkew - self +
    // the key's minimum at the pod's position, indexed like pod_need); the taker adds 1 to the node's count of every
    // key of its ts_matches.  Node passes read and write ts_count (key-major, row stride ts_stride); bins start at 0
    // and are not written back.  Node passes also report, per key k with ts_target[k] != INT_MAX, every take that
    // brings a domain of k (ts_domain) to exactly ts_target[k]: ts_reached[k] += 1, ts_rise_pos[k] = max position.
    const uint8_t *ts_key;                      // [req rows] the pod's key, 0xFF none
    const int32_t *ts_lim;                      // [positions]
    const unsigned long long *ts_matches;       // [req rows] keys whose selector selects the pod
    int32_t *ts_count;                          // [ts_keys][ts_stride] in/out (node pass)
    const unsigned long long *ts_domain;        // [N] keys each node is a domain of (node pass)
    const int *ts_target;                       // [64] (node pass)
    int *ts_reached;                            // [64] (node pass)
    unsigned long long *ts_rise_pos;            // [64] (node pass)
    int64_t ts_stride;
    int ts_keys;
};

__device__ __forceinline__ int ld_acquire(const int *p)
{
    int v;
    asm volatile("ld.acquire.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(int *p, int v)
{
    asm volatile("st.release.gpu.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// system scope: the counter / flag is polled by a kernel running on ANOTHER GPU (NVLink peer memory)
__device__ __forceinline__ int ld_acquire_sys(const int *p)
{
    int v;
    asm volatile("ld.acquire.sys.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(int *p, int v)
{
    asm volatile("st.release.sys.global.s32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_relaxed_sys_u32(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ unsigned long long global_timer_ns()
{
    unsigned long long t;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
    return t;
}

// shared-memory byte store predicated on `loses` == 0 (one predicated STS: no divergent branch inside the placement loop)
__device__ __forceinline__ void note_take(unsigned smem_addr, unsigned v, unsigned loses)
{
    asm volatile("{ .reg .pred p; setp.eq.u32 p, %2, 0; @p st.shared.u8 [%0], %1; }" ::"r"(smem_addr), "r"(v), "r"(loses) : "memory");
}

// m <- m | v when `loses` == 0 (AA: the taker's node masks gain the entry's bits, predicated like state_take)
__device__ __forceinline__ void mask_take(unsigned long long &m, unsigned long long v, unsigned loses)
{
    asm("{ .reg .pred p; setp.eq.u32 p, %2, 0; @p or.b64 %0, %0, %1; }" : "+l"(m) : "l"(v), "r"(loses));
}

// S <- S -/+ r when `loses` == 0, as ONE predicated instruction in place (the compiler's own if-conversion computes
// into a temporary and adds a predicated move per register half - one more dependent step on the placement chain).
template <bool BINS>
__device__ __forceinline__ void state_take(double &S, double r, unsigned loses)
{
    if (BINS)
        asm("{ .reg .pred p; setp.eq.u32 p, %2, 0; @p sub.rn.f64 %0, %0, %1; }" : "+d"(S) : "d"(r), "r"(loses));
    else
        asm("{ .reg .pred p; setp.eq.u32 p, %2, 0; @p add.rn.f64 %0, %0, %1; }" : "+d"(S) : "d"(r), "r"(loses));
}

template <int D>
__device__ __forceinline__ void load_row(double (&r)[D], const double *src)
{
    static_assert(D % 2 == 0, "rows are padded to an even number of dims");
#pragma unroll
    for (int d = 0; d < D; d += 2) {
        double2 v = *reinterpret_cast<const double2 *>(src + d);
        r[d] = v.x;
        r[d + 1] = v.y;
    }
}

// dynamic shared memory layout (doubles first for alignment).
// nodes mode keeps three [D][Tn] arrays: scan thresholds, used (the mutable state) and capacity;
// bins mode keeps one: the remaining capacity IS the threshold (finite values, Lemma B).
template <int D, bool BINS, int NT, bool PRUNE = false, int RW = 0, bool SEL = false, bool AA = false, bool PA = false,
          bool TS = false>
struct PipelineSmem {
    static constexpr int NW = NT / 32;  // warps per stage CTA == resolver warps
    // TS: the counts are sized by the call's key count, not by 64
    static __host__ __device__ size_t bytes(int Tn, int ts_keys = 0)
    {
        return sizeof(double) * ((size_t)kTile * D + (size_t)(BINS ? 1 : 3) * D * Tn + (size_t)NW * 36 * D /*batch rows*/ + (PRUNE ? (size_t)(NW + 1) * D : 0) /*warp bounds + stage bound*/)
               + sizeof(unsigned) * (kTile /*cand*/ + kTile / 32 /*hit*/ + kTile / 32 /*alive*/ + NW /*opened*/ +
                                     NW /*dirty*/ + 8 /*scan counts*/ + 8 /*alive counts*/ + 8 /*misc*/ + kRing * 8 /*alive words of the next tiles*/ + (kTile + 1) /*hitlist*/ +
                                     (NW - 1) * (kTile + 1) /*warp queues*/ + 1 /*pad*/)
               + sizeof(unsigned short) * kTile /*slot_of*/ + (size_t)NW * 32 /*accepted node per dense entry*/
               + sizeof(unsigned) * ((size_t)RW * Tn /*packed node words*/ + (size_t)RW * kTile /*packed pod words*/ + 4 /*alignment*/)
               + (SEL ? sizeof(unsigned long long) * (size_t)Tn /*node masks*/ + kTile /*pod classes*/ + (size_t)NW * 36 /*batch classes*/ : 0)
               + (AA ? sizeof(unsigned long long) * 2 * ((size_t)Tn /*node carries / matches*/ + kTile /*pod masks*/ + (size_t)NW * 36 /*batch masks*/) : 0)
               + (PA ? sizeof(unsigned long long) * ((size_t)Tn /*node has*/ + 2 * ((size_t)kTile /*pod need / matches*/ + (size_t)NW * 36 /*batch*/)) : 0)
               + (BINS && RW > 0 ? sizeof(double) * (size_t)D * (1 /*smallest request*/ + kRankStaged /*staged rank tables*/) : 0)
               + (TS ? sizeof(unsigned long long) * (2 * ((size_t)kTile /*pod key+limit / matches*/ + (size_t)NW * 36 /*batch*/) + (size_t)Tn /*node domains*/)
                           + sizeof(int) * (64 /*targets*/ + (size_t)ts_keys * Tn /*counts*/) : 0);
    }
};

// threads per stage CTA (the kernel is generic in it; 16-warp stages of 512 bins were measured and do not
// beat 8 warps: the placement chain, not stage straddling, bounds bin packing)
__host__ __device__ constexpr int stage_threads(int /*D*/, bool /*bins*/) { return 256; }
// one node per lane of the resolver warps; 128 for D = 16 keeps shared memory small
__host__ __device__ constexpr int max_stage_nodes(int D, bool bins) { return D <= 8 ? stage_threads(D, bins) : 128; }

// An upper bound of the warp-wide maximum of v (v >= 0, or negative for "no node"): the largest high word with
// the low word saturated -- one integer REDUX per dimension instead of a five-step shuffle ladder on doubles.
__device__ __forceinline__ double warp_upper_bound(double v)
{
    const int hi = __reduce_max_sync(0xFFFFFFFFu, __double2hiint(v));
    return hi >= 0x7FF00000 ? __longlong_as_double(0x7FF0000000000000ll) : __hiloint2double(hi, (int)0xFFFFFFFFu);
}

// spin on a shared-memory queue word until the producer warp has written it (0 = not yet)
__device__ __forceinline__ unsigned wait_entry(const volatile unsigned *slot, int *status)
{
    unsigned e = *slot;
    for (unsigned spins = 0; e == 0; e = *slot)
        if (++spins > (1u << 27)) {  // never expected: refuse to hang the GPU
            atomicExch(status, 2);
            return kQueueEnd;
        }
    return e;
}

// D <= 4: two stage CTAs per SM are part of the design (the node and the bin launch of a tick run chained, both resident),
// so the register budget is pinned to 128 instead of being left to the allocator's mood; D >= 8 runs one CTA per SM.
//
// SEL (node passes only): node selectors.  A pod may take a node only when bit pod_class of the node's match mask is
// set.  The predicate is static per (pod, node) pair, so it is ANDed into both candidate scans and into the resolver's
// vote, and everything else keeps its meaning: a node's threshold only shrinks, so a stale threshold is still a
// superset filter of "fits AND matches"; the per-warp and per-stage bounds stay resource-only (see the PRUNE test in
// the tile loader).  Bin passes need no SEL form: every bin of a pool carries the pool's labels, so the host gates the
// pods by match before a bin pass and the "untouched bin takes every eligible pod" shortcut stays exact.
//
// AA (node passes with SEL, and bin passes): required pod anti-affinity.  Whether pod p may take node n depends on the
// pods that reached n earlier in the pass, so it is not a static class: each node (bin) keeps two u64 term masks that
// the taker ORs the entry's masks into, and the resolver ANDs "not blocked" into its vote.  A node's masks only gain
// bits, so a pod blocked under older state is blocked now too: the resource-only (plus class) scan, the stale
// thresholds, the bounds, pruning and the untouched-bin shortcut (a new bin has both masks 0 and blocks nobody) all
// stay exact.  AA runs the barrier form only.
//
// PA (on top of the AA form): required pod affinity.  A pod whose need is non-zero may take a node (bin) only when the
// node's has mask shares a bit with it; the taker ORs the pod's signature matches into the node's mask.  A node's mask
// only gains bits, so the test is NOT monotone the way the block test is: it is left out of the scan and the bounds,
// which stay resource (plus class) only and hence a superset filter, and is evaluated in the resolver alone, whose
// chain sees every node's state exactly as the sequential loop does.  The need itself is fixed for the pass (the host
// applies the bootstrap exception through flip positions, see acsfit.cu).
//
// TS (on top of the PA form): hostname topology spread.  A pod with a key may take a node (bin) only while the node's
// count of that key stays within the pod's limit; the taker adds 1 to its node's count of every key the pod matches.
// Counts only grow, but in a node pass the limit (which carries the key's minimum over its domains) is fixed per
// position by the host and rises where the minimum does, so the test is not monotone: like PA it lives in the
// resolver alone, and the scan, bounds, pruning and retirement stay resource (plus class) only.  A new bin starts
// with count 0 and admits any pod (limit >= 0), so the untouched-bin shortcut stays exact.  Node passes report the
// takes that bring a watched key's domain to its target count (the next rise of its minimum, see acsfit.cu).
template <int D, bool BINS, int NT, bool PRUNE, int RW, bool SEL = false, bool AA = false, bool PA = false, bool TS = false>
__global__ void __launch_bounds__(NT, D <= 4 ? 2 : 1)
firstfit_pipeline_kernel(const PipelineParams p)
{
    static_assert(!(SEL && BINS), "selectors apply to node passes only");
    static_assert(!AA || BINS || SEL, "the anti-affinity node pass builds on the selector form");
    static_assert(!PA || AA, "the pod-affinity form builds on the anti-affinity form");
    static_assert(!TS || PA, "the topology-spread form builds on the pod-affinity form");
    constexpr int K = nodes_per_thread(D, RW);  // RW: 32-bit words of a packed-rank row, 0 = float64 scan
    constexpr int NW = NT / 32;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int Tn = p.Tn;
    double *rows = reinterpret_cast<double *>(smem_raw);        // [kTile][D]   compacted pod rows of the tile
    double *state_s = rows + (size_t)kTile * D;                 // [D][Tn]      used (nodes) / remaining (bins)
    double *thr_s = BINS ? state_s : state_s + (size_t)D * Tn;  // [D][Tn]      scan thresholds
    double *cap_s = BINS ? state_s : thr_s + (size_t)D * Tn;    // [D][Tn]      capacity (nodes only)
    double *brows = state_s + (size_t)(BINS ? 1 : 3) * D * Tn;  // [NW warps][36][D] rows of a resolver batch (+4 padding rows)
    double *wmax = brows + (size_t)NW * 36 * D;                 // [NW][D] per-warp upper bound of what still fits a node
    double *smax = wmax + (size_t)NW * D;                       // [D] the same bound over the whole stage
    unsigned *cand = reinterpret_cast<unsigned *>(PRUNE ? smax + D : wmax);  // [kTile]
    unsigned *hitmask = cand + kTile;                           // [kTile/32]
    unsigned *alive_w = hitmask + kTile / 32;                   // [kTile/32]   alive words of the tile
    unsigned *opened = alive_w + kTile / 32;                    // [NW] bins: bin already holds a pod (bit per node)
    unsigned *dirty = opened + NW;                              // [NW] nodes: threshold is stale (bit per node)
    unsigned *wcount = dirty + NW;                              // [8] pods to scan per tile word
    unsigned *acount = wcount + 8;                              // [8] alive pods per tile word
    unsigned *misc = acount + 8;                                // [8]: 0 stage, 1 abort, 2 drained, 3 any dirty, 4 placed, 5 first candidate, 6 dead warps (bins)
    unsigned *nextw = misc + 8;                                 // [kRing][8] alive words of the next tiles (ring, slot = tile % kRing)
    unsigned *hitlist = nextw + kRing * 8;                      // [kTile+1] ordered hit entries (q+1), then kQueueEnd
    unsigned *queue = hitlist + (kTile + 1);                    // [NW-1][kTile+1] forward queue of warp w -> w+1
    unsigned short *slot_of = reinterpret_cast<unsigned short *>(queue + (NW - 1) * (kTile + 1) + 1);  // [kTile]
    unsigned char *found_s = reinterpret_cast<unsigned char *>(slot_of + kTile);  // [NW][32] node that took dense entry k
    // packed-rank rows (RW > 0): scan thresholds of the stage's nodes and the compacted pods of the tile
    unsigned *tw_s = reinterpret_cast<unsigned *>((reinterpret_cast<uintptr_t>(found_s + NW * 32) + 15) & ~(uintptr_t)15);  // [Tn][RW]
    unsigned *rw_s = tw_s + (size_t)RW * Tn;                                                                              // [kTile][RW]
    // SEL: match masks of the stage's nodes, classes of the tile's compacted pods and of each resolver batch
    // (rw_s + RW * kTile is 16-byte aligned: tw_s is, and RW * (Tn + kTile) words are a multiple of 4)
    unsigned long long *nm_s = reinterpret_cast<unsigned long long *>(rw_s + (size_t)RW * kTile);  // [Tn]
    unsigned char *cls_s = reinterpret_cast<unsigned char *>(nm_s + Tn);                           // [kTile]
    unsigned char *bcls_s = cls_s + kTile;                                                         // [NW][36]
    // AA: carries / matches of the stage's nodes, of the tile's compacted pods and of each resolver batch (8-byte
    // aligned: the SEL arrays above take a multiple of 8 bytes)
    unsigned long long *nc_s = SEL ? reinterpret_cast<unsigned long long *>(bcls_s + NW * 36) : nm_s;  // [Tn]
    unsigned long long *nx_s = nc_s + Tn;                                                               // [Tn]
    unsigned long long *pc_s = nx_s + Tn;                                                               // [kTile]
    unsigned long long *px_s = pc_s + kTile;                                                            // [kTile]
    unsigned long long *bc_s = px_s + kTile;                                                            // [NW][36]
    unsigned long long *bx_s = bc_s + NW * 36;                                                          // [NW][36]
    // PA: has masks of the stage's nodes, need / matches of the tile's compacted pods and of each resolver batch
    unsigned long long *nh_s = AA ? bx_s + NW * 36 : nm_s;  // [Tn]
    unsigned long long *pn_s = nh_s + Tn;                   // [kTile]
    unsigned long long *pm_s = pn_s + kTile;                // [kTile]
    unsigned long long *bn_s = pm_s + kTile;                // [NW][36]
    unsigned long long *bm_s = bn_s + NW * 36;              // [NW][36]
    // bins with the packed-rank scan: the smallest request of each dimension and the staged rank tables
    double *minreq_s = reinterpret_cast<double *>(PA ? bm_s + NW * 36 : AA ? bx_s + NW * 36 : nm_s);  // [D]
    double *rt_s = minreq_s + D;                                                 // [D][kRankStaged]
    // TS: key + limit (+ slot, in the batch) and key matches of the tile's compacted pods and of each resolver batch,
    // domain masks, targets and counts ([key][Tn]) of the stage's nodes
    unsigned long long *tk_s = reinterpret_cast<unsigned long long *>(minreq_s + (BINS && RW > 0 ? D * (1 + kRankStaged) : 0));  // [kTile]
    unsigned long long *tm_s = tk_s + kTile;       // [kTile]
    unsigned long long *bk_s = tm_s + kTile;       // [NW][36]
    unsigned long long *bt_s = bk_s + NW * 36;     // [NW][36]
    unsigned long long *nd_s = bt_s + NW * 36;     // [Tn]
    int *tgt_s = reinterpret_cast<int *>(nd_s + Tn);  // [64]
    int *cnt_s = tgt_s + 64;                          // [ts_keys][Tn]

    const int tid = threadIdx.x;
    const int lane = tid & 31;
    const int warp = tid >> 5;

    if (tid == 0) {
        misc[0] = (unsigned)atomicAdd(p.ticket, 1);
        misc[1] = 0;
        misc[2] = 0;
        misc[3] = 0;
        misc[4] = 0;
        if (BINS) misc[6] = 0;
    }
    __syncthreads();
    const int stage = (int)misc[0];
    const bool remote_in = stage == 0 && p.alive_in != nullptr;            // this stage is fed by another GPU
    const bool sys_out = p.sys_scope && stage == (int)gridDim.x - 1;       // ... and this one feeds another GPU
    auto publish = [&](int tiles_done) {
        if (sys_out) {
            __threadfence_system();
            st_release_sys(p.progress + stage, tiles_done);
        } else {
            st_release(p.progress + stage, tiles_done);
        }
    };
    const int64_t stage_lo = p.node_lo + (int64_t)stage * Tn;   // global index of local node 0
    const int n_valid = (int)max((int64_t)0, min((int64_t)Tn, p.node_hi - stage_lo));
    const int n_warps = (n_valid + 31) >> 5;                     // resolver warps that own a real node

    // ---- stage start: state + thresholds of this stage's nodes into shared memory ----------
    for (int i = tid; i < Tn * D; i += NT) {
        const int n = i / D, d = i - n * D;
        if (BINS) {
            // untouched bin: remaining == unit (scaler.py:145-146); padding bins never fit
            state_s[(size_t)d * Tn + n] = n < n_valid ? p.unit[d] : -1.0;
        } else {
            double u = 0.0, c = -1.0, t = -1.0;  // padding nodes never fit
            if (n < n_valid) {
                const int64_t gn = stage_lo + n;
                u = p.used[(size_t)gn * D + d];
                c = p.cap_type[(size_t)p.node_type[gn] * D + d];
                t = node_threshold(c, u);
            }
            state_s[(size_t)d * Tn + n] = u;
            cap_s[(size_t)d * Tn + n] = c;
            thr_s[(size_t)d * Tn + n] = t;
        }
    }
    if (tid < NW) {
        opened[tid] = 0;
        dirty[tid] = 0;
    }
    for (int i = tid; i < NW * (kTile + 1) + 1; i += NT) hitlist[i] = 0;  // hit list + the NW-1 queues
    if constexpr (RW > 0)
        for (int i = tid; i < Tn * RW; i += NT) tw_s[i] = 0;
    if constexpr (SEL)  // padding nodes match nothing (they never fit either)
        for (int n = tid; n < Tn; n += NT) nm_s[n] = n < n_valid ? __ldg(p.node_match + stage_lo + n) : 0ull;
    if constexpr (AA)  // bins (and padding nodes) start empty
        for (int n = tid; n < Tn; n += NT) {
            nc_s[n] = !BINS && n < n_valid ? p.node_carries[stage_lo + n] : 0ull;
            nx_s[n] = !BINS && n < n_valid ? p.node_matches[stage_lo + n] : 0ull;
        }
    if constexpr (PA)
        for (int n = tid; n < Tn; n += NT) nh_s[n] = !BINS && n < n_valid ? p.node_has[stage_lo + n] : 0ull;
    if constexpr (TS) {  // bins (and padding nodes) start with count 0 and are nobody's domain
        for (int n = tid; n < Tn; n += NT) nd_s[n] = !BINS && n < n_valid ? p.ts_domain[stage_lo + n] : 0ull;
        for (int i = tid; i < p.ts_keys * Tn; i += NT) {
            const int k = i / Tn, n = i - k * Tn;
            cnt_s[i] = !BINS && n < n_valid ? p.ts_count[(size_t)k * p.ts_stride + stage_lo + n] : 0;
        }
        if (tid < 64) tgt_s[tid] = !BINS && tid < p.ts_keys ? p.ts_target[tid] : INT_MAX;
    }
    // Bin retirement (RW > 0).  The rank tables are built over every request row of the call, a superset of the pass's
    // pods, so sorted[d][0] is a lower bound of every request of the pass in dimension d.  A bin with S[d] < that
    // bound in some d can take no pod of the pass now, and S only shrinks: it is dead for good.  Without rank tables
    // (RW == 0, the float64 scan) there is no such bound at hand and nothing retires; retire == 0 turns it off too
    // (the bound becomes -inf).  A zero bound (a padded dimension) simply retires nothing through that dimension.
    if constexpr (BINS && RW > 0) {
        if (tid < D) minreq_s[tid] = p.retire ? __ldg(p.rk.sorted + (size_t)tid * kRankCap) : -__longlong_as_double(0x7FF0000000000000ll);
        for (int i = tid; i < D * kRankStaged; i += NT) {
            const int d = i / kRankStaged, k = i - d * kRankStaged;
            if (p.rk.count[d] <= kRankStaged && k < p.rk.count[d]) rt_s[i] = __ldg(p.rk.sorted + (size_t)d * kRankCap + k);
        }
    }
    __syncthreads();
    // (n, d) -> field t' of the node's packed threshold row; callers zero the row first
    auto pack_field = [&](int i) {
        const int d = i / Tn, n = i - d * Tn;
        const double thr = BINS ? state_s[i] : thr_s[i];
        uint32_t t;
        if (BINS && p.rk.count[d] <= kRankStaged) t = rank_upper_shared(rt_s + (size_t)d * kRankStaged, p.rk.count[d], thr);
        else t = rank_upper(p.rk.sorted + (size_t)d * kRankCap, p.rk.count[d], thr);
        atomicOr(&tw_s[n * RW + p.rk.word[d]], t << p.rk.shift[d]);
    };
    if constexpr (RW > 0) {
        for (int i = tid; i < Tn * D; i += NT) pack_field(i);
        // made visible by the barrier inside / after refresh_bounds or by (S1) of the first tile
    }

    // Per-warp, per-dimension upper bound of the request that can still fit SOME node of the warp (nodes: the
    // scan thresholds, bins: the remaining amounts).  Kept in shared memory, refreshed after every tile that
    // placed a pod.  Two users: the resolver (skips a whole batch against a full warp) and the tile loader
    // below, which leaves pods that exceed the bound of EVERY warp in some dimension out of the scan: they can
    // fit no node of this stage now, hence - state only shrinks - none later in the tile either.  Pruning
    // earns time, never credit: the credited decisions are derived from the placements, not from the tests run.
    auto refresh_bounds = [&]() {
        // bin stages, and node passes that fit the GPU in one wave: the placement chain is the critical path, not
        // the scan, and the extra barrier per placing tile costs more than the pruning saves (measured)
        if (!PRUNE) return;
        if (warp < n_warps) {
            const int n = (warp << 5) + lane;
#pragma unroll
            for (int d = 0; d < D; ++d) {
                const double b = warp_upper_bound(n < Tn ? (BINS ? state_s[(size_t)d * Tn + n] : thr_s[(size_t)d * Tn + n]) : -1.0);
                if (lane == 0) wmax[warp * D + d] = b;
            }
        }
        __syncthreads();
        if (tid < D) {
            double m = wmax[tid];
            for (int w = 1; w < n_warps; ++w) m = fmax(m, wmax[w * D + tid]);
            smax[tid] = m;
        }
    };
    refresh_bounds();  // visible after the first (S1)

    const int NS = p.NS;
    const int slot = tid & (NS - 1);
    const int group = tid / NS;
    const int PG = NT / NS;
    unsigned long long my_evals = 0;
    long long forwarded = 0;  // (warp 0) pods this stage passed on to the next one
    int since_placed = 1 << 20;  // (thread 0) tiles since this stage last placed a pod
    // developer probe (tools/perf_probe.py): compiled in only with -DACSFIT_PROFILE=1 (python -m ...build --profile); the
    // accumulators and clock reads cost registers the placement loop wants
    const bool PROF_ON = kProfileBuild && p.prof != nullptr;
    unsigned long long prof_acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // (thread 0) wait/load/scan/resolve/publish/refresh/hits/tiles
    unsigned long long trace_prev[6] = {0, 0, 0, 0, 0, 0};
    long long tp = 0;
#define ACSFIT_PROF(i)                                   \
    if (PROF_ON && tid == 0) {                            \
        const long long now__ = clock64();               \
        prof_acc[i] += (unsigned long long)(now__ - tp); \
        tp = now__;                                      \
    }
    const unsigned long long t_start = global_timer_ns();

    // the pod list is static, so the row of this thread's entry in the NEXT tile can be fetched from L2
    // while the current tile is scanned; only the alive word has to wait for the upstream stage.
    double pre[D];
    unsigned prew[RW > 0 ? RW : 1];
    unsigned pre_cls = 0;  // SEL: the entry's selector class
    unsigned long long pre_c = 0ull, pre_x = 0ull;  // AA: the entry's carries / matches
    unsigned long long pre_n = 0ull, pre_m = 0ull;  // PA: the entry's need / signature matches
    unsigned long long pre_k = 0ull, pre_t = 0ull;  // TS: the entry's key << 32 | limit, and key matches
    auto prefetch_row = [&](int tile) {
        const int64_t j = (int64_t)(p.tile_lo + tile) * kTile + tid;
        if (tid < kTile && tile < p.num_tiles && j < p.M) {
            int64_t row = p.pod_idx ? (int64_t)__ldg(p.pod_idx + j) : j;
            if (p.row_map) row = (int64_t)__ldg(p.row_map + row);
            const double *src = p.req + (size_t)row * D;
#pragma unroll
            for (int d = 0; d < D; d += 2) {
                const double2 v = __ldg(reinterpret_cast<const double2 *>(src + d));
                pre[d] = v.x;
                pre[d + 1] = v.y;
            }
            if constexpr (RW > 0) {
#pragma unroll
                for (int w = 0; w < RW; ++w) prew[w] = __ldg(p.rk.packed + (size_t)row * RW + w);
            }
            if constexpr (SEL) pre_cls = __ldg(p.pod_class + row);
            if constexpr (AA) {
                pre_c = __ldg(p.pod_carries + row);
                pre_x = __ldg(p.pod_matches + row);
            }
            if constexpr (PA) {
                pre_n = __ldg(p.pod_need + (BINS ? (int64_t)__ldg(p.pod_idx + j) : j));
                pre_m = __ldg(p.pod_aff_matches + row);
            }
            if constexpr (TS) {
                const int lim = __ldg(p.ts_lim + (BINS ? (int64_t)__ldg(p.pod_idx + j) : j));
                pre_k = ((unsigned long long)__ldg(p.ts_key + row) << 32) | (unsigned)lim;
                pre_t = __ldg(p.ts_matches + row);
            }
        }
    };
    prefetch_row(0);
    int known = 0, ring_hi = 0;  // (warp 1) tiles the upstream is known to have published / whose alive words are in the ring

    for (int tile = 0; tile < p.num_tiles; ++tile) {
        if (PROF_ON && tid == 0) tp = clock64();
        // ---- wait until the previous stage has published this tile (warp 1 polls, so that warp 0
        //      can still be publishing the previous tile) ---------------------------------------
        //      The same warp then fetches the tile's alive words, so that their L2 (or NVLink) latency is
        //      paid while the other warps are still finishing the previous tile, not after the barrier.
        //      The upstream counter is re-read only when this stage has caught up with what it last saw, and the
        //      alive words of every tile known to be published (up to kRing ahead) are fetched in one go: a stage
        //      that lags its upstream -- always the case across NVLink, where one poll costs microseconds -- pays
        //      the hand-off latency once per kRing tiles instead of once per tile.
        if (warp == 1) {
            if (known <= tile) {  // (known / ring_hi are warp-uniform registers of warp 1)
                int seen = known;
                if (lane == 0) {
                    if (!(stage > 0 || p.upstream)) {
                        seen = p.num_tiles;  // the head of the pipeline: every tile is there from the start
                    } else if (stage > 0 && *(volatile int *)p.drained) {
                        misc[2] = 1;  // an earlier stage finished with nothing left alive: every remaining tile is empty
                    } else {
                        const int *flag = stage > 0 ? p.progress + (stage - 1) : p.upstream;
                        unsigned spins = 0;
                        while ((seen = (p.sys_scope && stage == 0 ? ld_acquire_sys(flag) : ld_acquire(flag))) <= tile) {
                            if ((++spins & 63u) == 0) {
                                if (*(volatile int *)p.status != 0 || global_timer_ns() - t_start > p.watchdog_ns) {
                                    atomicExch(p.status, 1);
                                    misc[1] = 1;
                                    break;
                                }
                            }
                            __nanosleep(20);
                        }
                    }
                }
                known = __shfl_sync(0xFFFFFFFFu, seen, 0);  // also orders the loads below after lane 0's acquire
            }
            if (tile >= ring_hi && known > tile) {  // refill: tiles [tile, min(known, tile + kRing))
                const int hi_t = min(known, tile + kRing);
                for (int i = lane; i < (hi_t - tile) * (kTile / 32); i += 32) {
                    const int t = tile + i / (kTile / 32);
                    const int64_t wj = (int64_t)(p.tile_lo + t) * (kTile / 32) + (i % (kTile / 32));
                    unsigned w = 0u;
                    if (wj * 32 < p.M) w = remote_in ? ld_relaxed_sys_u32(p.alive_in + wj) : __ldcg(p.alive + wj);
                    nextw[(t % kRing) * (kTile / 32) + (i % (kTile / 32))] = w;
                }
                ring_hi = hi_t;
            }
        }
        __syncthreads();  // (S1) previous tile fully retired (publish included), poll result and alive words visible
        if (misc[1]) return;  // watchdog: give up (host reports ACSFIT_E_TIMEOUT)
        if (misc[2]) break;   // drained: nothing left to do (state write-back below)
        ACSFIT_PROF(0)

        // ---- load the tile: compact the alive pods' rows into shared memory ----------------
        const int64_t j = (int64_t)(p.tile_lo + tile) * kTile + tid;
        const unsigned word = nextw[(tile % kRing) * (kTile / 32) + warp];
        const bool is_alive = (word >> lane) & 1u;
        // bins: once every warp of the stage is dead (every bin holds a pod and is too full for the smallest request in
        // some dimension) the stage can take no pod of any later tile: it forwards every tile untouched
        const bool retired = BINS && RW > 0 && p.retire && misc[6] == (1u << n_warps) - 1u;
        bool pass = is_alive && !retired;
        // SEL: the bounds stay resource-only.  A pod they prune exceeds, in some dimension, every threshold of the
        // stage, so it fits no node here whatever the node matches: leaving it out is exact.  A pod that passes
        // only because a node it does not match has room is scanned in vain, which costs time, never a result.
        if (PRUNE && is_alive) {  // can the pod fit any node of the stage at all?  (per-dimension bound over the warps)
#pragma unroll
            for (int d = 0; d < D; ++d) pass = pass & (pre[d] <= smax[d]);
        }
        const unsigned pword = PRUNE ? __ballot_sync(0xFFFFFFFFu, pass) : retired ? 0u : word;
        if (lane == 0 && warp < kTile / 32) {
            wcount[warp] = __popc(pword);
            if (PRUNE || retired) acount[warp] = __popc(word);
            alive_w[warp] = word;
        }
        if (tid < kTile / 32) hitmask[tid] = 0;
        if (tid < NW) dirty[tid] = 0;
        if (tid == 0) {
            misc[4] = 0;
            misc[5] = 0xFFFFFFFFu;
        }
        __syncthreads();
        unsigned base = 0, total = 0, alive_total = 0;  // total: pods to scan (compacted rows)
#pragma unroll
        for (int w = 0; w < kTile / 32; ++w) {
            const unsigned c = wcount[w];
            base += (w < warp) ? c : 0u;
            total += c;
            if (PRUNE || retired) alive_total += acount[w];
        }
        if (!PRUNE && !retired) alive_total = total;
        if (total == 0) {  // nothing alive, or nothing that could fit here: forward the tile untouched
            if (PRUNE || retired) forwarded += (long long)alive_total;
            if (remote_in && warp == 0) {  // the words came from the upstream GPU: this GPU's bitmap must hold them too
                const int64_t wj = (int64_t)(p.tile_lo + tile) * (kTile / 32) + lane;
                if (lane < kTile / 32 && wj * 32 < p.M) __stcg(p.alive + wj, alive_w[lane]);
                __syncwarp();
                if (lane == 0) __threadfence();
            }
            if (tid == 0) publish(tile + 1);
            prefetch_row(tile + 1);
            continue;  // uniform: every thread sees the same total; (S1) protects the shared words
        }
        if (pass) {
            const unsigned pos = base + __popc(pword & ((1u << lane) - 1u));
            double *dst = rows + (size_t)pos * D;
#pragma unroll
            for (int d = 0; d < D; d += 2) *reinterpret_cast<double2 *>(dst + d) = make_double2(pre[d], pre[d + 1]);
            slot_of[pos] = (unsigned short)tid;
            cand[pos] = kNoCand;
            if constexpr (RW > 0) {
#pragma unroll
                for (int w = 0; w < RW; ++w) rw_s[pos * RW + w] = prew[w];
            }
            if constexpr (SEL) cls_s[pos] = (unsigned char)pre_cls;
            if constexpr (AA) {
                pc_s[pos] = pre_c;
                px_s[pos] = pre_x;
            }
            if constexpr (PA) {
                pn_s[pos] = pre_n;
                pm_s[pos] = pre_m;
            }
            if constexpr (TS) {
                tk_s[pos] = pre_k;
                tm_s[pos] = pre_t;
            }
        }
        prefetch_row(tile + 1);
        __syncthreads();
        ACSFIT_PROF(1)

        // ---- scan: every (alive pod, stage node) pair under the tile-start thresholds -------
        // bins: while the stage still owns an untouched bin every eligible pod fits it (scaler.py:134 is the
        // same test), so every alive pod is a hit and the resolver starts it at the stage's first bin.
        bool all_hit = false;
        if (BINS) {
            int n_open = 0;
#pragma unroll
            for (int w = 0; w < NW; ++w) n_open += __popc(opened[w]);
            all_hit = n_open < n_valid;
        }
        if (all_hit) {
            if (tid < total) cand[tid] = 0;
        } else if constexpr (RW > 0) {
            // packed-rank scan: fits in every dimension <=> (((T | G) - R) & G) == G, word by word (RankLayout)
            unsigned g[RW], tg[K][RW];
#pragma unroll
            for (int w = 0; w < RW; ++w) g[w] = p.rk.guard[w];
#pragma unroll
            for (int k = 0; k < K; ++k)
#pragma unroll
                for (int w = 0; w < RW; ++w) tg[k][w] = tw_s[(slot + k * NS) * RW + w] | g[w];
            unsigned long long nm[SEL ? K : 1];  // SEL: match masks of this thread's nodes
            if constexpr (SEL) {
#pragma unroll
                for (int k = 0; k < K; ++k) nm[k] = nm_s[slot + k * NS];
            }
            constexpr int PPI = 4;  // pods per thread and iteration
            for (unsigned qb = 0; qb < total; qb += PPI * PG) {
                unsigned q[PPI], best[PPI], r[PPI][RW], c[PPI];
                bool live[PPI];
#pragma unroll
                for (int i = 0; i < PPI; ++i) {
                    q[i] = qb + (unsigned)(i * PG + group);
                    live[i] = q[i] < total;
                    const unsigned *src = rw_s + (size_t)(live[i] ? q[i] : total - 1) * RW;
#pragma unroll
                    for (int w = 0; w < RW; ++w) r[i][w] = src[w];
                    if constexpr (SEL) c[i] = cls_s[live[i] ? q[i] : total - 1];
                    best[i] = kNoCand;
                }
#pragma unroll
                for (int k = K - 1; k >= 0; --k) {
#pragma unroll
                    for (int i = 0; i < PPI; ++i) {
                        unsigned miss = 0;
#pragma unroll
                        for (int w = 0; w < RW; ++w) miss |= ((tg[k][w] - r[i][w]) & g[w]) ^ g[w];
                        if constexpr (SEL) {
                            if (miss == 0 && live[i] && ((nm[k] >> c[i]) & 1ull)) best[i] = (unsigned)(slot + k * NS);
                        } else {
                            if (miss == 0 && live[i]) best[i] = (unsigned)(slot + k * NS);
                        }
                    }
                }
                unsigned any_best = best[0];
#pragma unroll
                for (int i = 1; i < PPI; ++i) any_best &= best[i];
                if (__any_sync(0xFFFFFFFFu, any_best != kNoCand)) {
                    const int seg = NS < 32 ? NS : 32;
                    for (int o = seg >> 1; o > 0; o >>= 1) {
#pragma unroll
                        for (int i = 0; i < PPI; ++i) best[i] = min(best[i], __shfl_xor_sync(0xFFFFFFFFu, best[i], o));
                    }
                    if ((lane & (seg - 1)) == 0) {
#pragma unroll
                        for (int i = 0; i < PPI; ++i) {
                            if (best[i] != kNoCand) {
                                if (NS <= 32) cand[q[i]] = best[i];
                                else atomicMin(&cand[q[i]], best[i]);
                            }
                        }
                    }
                }
            }
        } else {
            double t[K][D];
#pragma unroll
            for (int k = 0; k < K; ++k)
#pragma unroll
                for (int d = 0; d < D; ++d) t[k][d] = thr_s[(size_t)d * Tn + slot + k * NS];
            unsigned long long nm[SEL ? K : 1];  // SEL: match masks of this thread's nodes
            if constexpr (SEL) {
#pragma unroll
                for (int k = 0; k < K; ++k) nm[k] = nm_s[slot + k * NS];
            }
            // several pods per iteration: their compares are independent, which keeps the fp64 pipe fed with
            // only eight warps per stage, and the vote / loop overhead is paid once per group of pods;
            // trip count is warp-uniform (votes inside)
            constexpr int PPI = (D == 8) ? 4 : 2;  // pods per thread and iteration
            for (unsigned qb = 0; qb < total; qb += PPI * PG) {
                unsigned q[PPI], c[PPI];
                bool live[PPI];
                double r[PPI][D];
                unsigned best[PPI];
#pragma unroll
                for (int i = 0; i < PPI; ++i) {
                    q[i] = qb + (unsigned)(i * PG + group);
                    live[i] = q[i] < total;
                    load_row<D>(r[i], rows + (size_t)(live[i] ? q[i] : total - 1) * D);
                    if constexpr (SEL) c[i] = cls_s[live[i] ? q[i] : total - 1];
                    best[i] = kNoCand;
                }
#pragma unroll
                for (int k = K - 1; k >= 0; --k) {
#pragma unroll
                    for (int i = 0; i < PPI; ++i) {
                        bool ok = live[i];
#pragma unroll
                        for (int d = 0; d < D; ++d) ok = ok & (r[i][d] <= t[k][d]);
                        if constexpr (SEL) ok = ok & (((nm[k] >> c[i]) & 1ull) != 0ull);
                        if (ok) best[i] = (unsigned)(slot + k * NS);
                    }
                }
                // hits are rare: one vote, and only then a segmented min over the lanes that share a pod
                // (NS consecutive lanes; when NS > 32 several warps share the pod and an atomic min merges them)
                unsigned any_best = best[0];
#pragma unroll
                for (int i = 1; i < PPI; ++i) any_best &= best[i];
                if (__any_sync(0xFFFFFFFFu, any_best != kNoCand)) {
                    const int seg = NS < 32 ? NS : 32;
                    for (int o = seg >> 1; o > 0; o >>= 1) {
#pragma unroll
                        for (int i = 0; i < PPI; ++i) best[i] = min(best[i], __shfl_xor_sync(0xFFFFFFFFu, best[i], o));
                    }
                    // with NS <= 32 exactly one segment handles a given pod: a plain store; wider stages
                    // spread a pod over NS / 32 warps, whose minima an atomic merges
                    if ((lane & (seg - 1)) == 0) {
#pragma unroll
                        for (int i = 0; i < PPI; ++i) {
                            if (best[i] != kNoCand) {
                                if (NS <= 32) cand[q[i]] = best[i];
                                else atomicMin(&cand[q[i]], best[i]);
                            }
                        }
                    }
                }
            }
        }
        __syncthreads();
        {   // hit mask of the tile from the candidates (no shared atomics in the scan)
            const bool hit = tid < (int)total && cand[tid] != kNoCand;
            const unsigned hw = __ballot_sync(0xFFFFFFFFu, hit);
            if (lane == 0 && warp < kTile / 32) hitmask[warp] = hw;
            // the first candidate of the whole tile: no pod has one in a warp before it, so those warps (nodes that were
            // full at tile start) need not pass the hit list along - the resolver chain starts at that warp
            if (hw) {
                const unsigned cmin = __reduce_min_sync(0xFFFFFFFFu, hit ? cand[tid] : 0xFFFFFFFFu);
                if (lane == 0) atomicMin(&misc[5], cmin);
            }
        }
        __syncthreads();
        ACSFIT_PROF(2)

        // ---- resolve hits strictly in pod order: an intra-CTA systolic chain of warps -----------
        // warp w owns nodes [32w, 32w+32) of the stage with their state in registers (lane <-> node)
        // and evaluates the LITERAL reference predicate, so no threshold sits on this critical path.
        // The ordered hit list enters warp 0; a warp either places the pod on its first fitting node
        // or forwards it, in order, to warp w+1 through a shared-memory queue of self-validating words.
        unsigned nh;
        {
            unsigned hb = 0, ht = 0;
#pragma unroll
            for (int w = 0; w < kTile / 32; ++w) {
                const unsigned c = __popc(hitmask[w]);
                hb += (w < warp) ? c : 0u;
                ht += c;
            }
            nh = ht;
            if (nh > 0) {
                // queue entries: 0 = not written yet, q + 1 = compacted pod position q, kQueueEnd = end
                const unsigned hw = warp < kTile / 32 ? hitmask[warp] : 0u;  // CTAs may have more warps than tile words
                if ((hw >> lane) & 1u) hitlist[hb + __popc(hw & ((1u << lane) - 1u))] = (unsigned)tid + 1u;
                if (tid == 0) hitlist[ht] = kQueueEnd;
            }
        }
        // SEL: count the pods the scan handed to the resolver (pods with a candidate node that fits AND matches);
        // the count is exposed so that a scan whose match filter stopped working is caught by a test, although the
        // resolver's own match test keeps every placement right
        if constexpr (SEL) {
            if (tid == 0 && nh && p.sel_hits) atomicAdd(p.sel_hits, (unsigned long long)nh);
        }
        bool became_dead = false;  // bins: this warp's bins all died in this tile
        if (nh > 0) {
            __syncthreads();
            unsigned out = 0;
            const int first_w = min((int)(misc[5] >> 5), n_warps - 1);
            // bins: the chain runs over the live warps at or after first_w only.  A warp reads the queue of the previous
            // live warp (none: the hit list) and the last live warp forwards nothing.  A dead warp could take no entry
            // anyway.  The dead bits change only after the barrier at the end of the resolver.
            const unsigned chain = BINS ? ((1u << n_warps) - 1u) & ~misc[6] & ~((1u << first_w) - 1u) : 0u;
            const unsigned chain_below = chain & ((1u << warp) - 1u);  // bins: live warps of the chain before this one
            const bool chain_last = (chain & ~((2u << warp) - 1u)) == 0u;
            if (BINS ? ((chain >> warp) & 1u) != 0u : warp < n_warps && warp >= first_w) {
                const int my_lo = warp << 5;
                const int n = my_lo + lane;
                const bool last = BINS ? chain_last : warp == n_warps - 1;
                double S[D], C[D];
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    S[d] = n < Tn ? state_s[(size_t)d * Tn + n] : (BINS ? -1.0 : 0.0);
                    C[d] = (!BINS && n < Tn) ? cap_s[(size_t)d * Tn + n] : -1.0;
                }
                // per-dimension maximum a pod may request and still fit SOME node of this warp: an upper bound.
                // bins: the largest remaining amount; nodes: the largest tile-start threshold (exact at tile start,
                // and thresholds only shrink while the tile is resolved).
                double Mx[D];
#pragma unroll
                for (int d = 0; d < D; ++d)
                    Mx[d] = BINS ? warp_upper_bound(S[d])
                                 : PRUNE ? wmax[warp * D + d] : warp_upper_bound(n < Tn ? thr_s[(size_t)d * Tn + n] : -1.0);
                // bins: bit per lane = the bin already holds a pod (persists over tiles); nodes: threshold is stale
                unsigned touched_or_open = BINS ? opened[warp] : 0u;
                unsigned touched_tile = 0u;  // nodes / bins of this warp that took a pod in this tile
                unsigned long long my_nm = 0ull;  // SEL: the classes this lane's node matches
                if constexpr (SEL) my_nm = n < Tn ? nm_s[n] : 0ull;
                unsigned long long my_nc = 0ull, my_nx = 0ull;  // AA: this lane's node's carries / matches
                if constexpr (AA) {
                    my_nc = n < Tn ? nc_s[n] : 0ull;
                    my_nx = n < Tn ? nx_s[n] : 0ull;
                }
                unsigned long long my_nh = 0ull;  // PA: this lane's node's has mask
                if constexpr (PA) my_nh = n < Tn ? nh_s[n] : 0ull;
                unsigned long long my_nd = 0ull;  // TS: the keys this lane's node is a domain of (node pass)
                if constexpr (TS) my_nd = n < Tn ? nd_s[n] : 0ull;
                // TS: this lane's column of the counts.  A lane past the stage's nodes (stages narrower than a warp)
                // fits no entry and so never takes: it reads column 0, which keeps every access inside the array.
                const int my_cn = n < Tn ? n : 0;

                unsigned my_takes = 0;  // pods this lane's node / bin took in this tile
                const volatile unsigned *in_q = BINS ? (chain_below ? queue + (size_t)(31 - __clz(chain_below)) * (kTile + 1) : hitlist)
                                                     : warp == first_w ? hitlist : queue + (size_t)(warp - 1) * (kTile + 1);
                volatile unsigned *out_q = queue + (size_t)warp * (kTile + 1);
                unsigned head = 0;
                int n_placed = 0;
                bool done = false;
                const bool tracing = PROF_ON && p.trace && stage == p.trace_stage;
                long long tw = 0, tb = 0, t_loop = 0, t_mark = tracing ? clock64() : 0;
                unsigned n_batches = 0, n_iter = 0;
                // this lane's bit, and all bits up to it (read once from the special registers: the compiler would
                // otherwise rematerialise shift/add sequences for them inside the loop, on the placement chain)
                unsigned me, le;
                asm volatile("mov.u32 %0, %%lanemask_eq;" : "=r"(me));
                asm volatile("mov.u32 %0, %%lanemask_le;" : "=r"(le));
                while (!done) {
                    // a batch of up to 32 entries: lane i takes entry head+i with its candidate and slot;
                    // only the node state S carries a dependency from one entry to the next.
                    const unsigned idx = head + lane <= (unsigned)kTile ? head + lane : (unsigned)kTile;
                    unsigned e, present, endmask;
                    int nb;
                    for (unsigned spins = 0;; ++spins) {
                        e = in_q[idx];
                        if (head + lane > (unsigned)kTile) e = 0;
                        present = __ballot_sync(0xFFFFFFFFu, e != 0);
                        nb = __ffs(~present) ? __ffs(~present) - 1 : 32;  // written entries form a prefix
                        // a consumer warp takes entries in batches of >= kMinBatch (or up to the end marker):
                        // one-entry batches would pay the batch set-up for every pod the producer forwards
                        endmask = __ballot_sync(0xFFFFFFFFu, lane < nb && e == kQueueEnd);
                        if (endmask || nb >= kMinBatch) break;
                        __nanosleep(64);  // do not hammer the shared-memory pipe the producer warp needs
                        
                        if (spins > (1u << 26)) {  // never expected: refuse to hang the GPU
                            atomicExch(p.status, 2);
                            e = lane == 0 ? kQueueEnd : 0u;
                            present = 1u;
                            endmask = 1u;
                            nb = 1;
                            break;
                        }
                    }
                    if (tracing) { const long long now = clock64(); tw += now - t_mark; t_mark = now; ++n_batches; }
                    const int n_ent = endmask ? __ffs(endmask) - 1 : nb;
                    const bool mine = lane < n_ent;  // words after the end marker are stale: never touch them
                    const unsigned q_l = mine ? e - 1 : 0;
                    const unsigned c_l = mine ? cand[q_l] : kNoCand;
                    const unsigned s_l = mine ? slot_of[q_l] : 0;
                    int placed_here = -1;  // lane i: LOCAL node (of this warp) that took entry i of the batch
                    // Which entries of the batch can this warp take at all?  Lane i checks its own entry against
                    // the per-dimension maximum over the warp's 32 nodes (an upper bound that only gets looser
                    // as nodes fill up, so a "no" is final) - 32 entries in one step.  Only the entries that
                    // pass are staged, densely, for the sequential loop; the others are forwarded in bulk.
                    // (In the scan every pair is compared; this bound only spares the resolver, which sees <= 2 %
                    // of the pairs, from re-testing pods against a warp whose nodes are all too full.)
                    double *brow = brows + (size_t)warp * 36 * D;
                    volatile unsigned char *fnd = found_s + warp * 32;
                    double own[D];
                    load_row<D>(own, rows + (size_t)q_l * D);
                    // nodes before cand[q] did not fit at tile start, hence not now either
                    bool poss = mine && (int)c_l < my_lo + 32;
#pragma unroll
                    for (int d = 0; d < D; ++d) poss = poss & (own[d] <= Mx[d]);

                    const unsigned possmask = __ballot_sync(0xFFFFFFFFu, poss);
                    const int n_poss = __popc(possmask);
                    if (possmask == 0u) {  // nothing this warp could take (it is full): pass the batch along and go on
                        if (!last) {
                            if (mine) out_q[out + lane] = e;  // the batch's entries are a prefix of the lanes
                            out += (unsigned)n_ent;
                        }
                        head += (unsigned)n_ent;
                        done = endmask != 0;
                        if (tracing) { const long long now = clock64(); tb += now - t_mark; t_mark = now; }
                        continue;
                    }
                    const int my_rank = __popc(possmask & ((1u << lane) - 1u));
                    unsigned char *bcls = bcls_s + warp * 36;  // SEL: class of each dense entry (+4 padding entries)
                    unsigned long long *bc = bc_s + warp * 36, *bx = bx_s + warp * 36;  // AA: masks of each dense entry
                    unsigned long long *bn = bn_s + warp * 36, *bm = bm_s + warp * 36;  // PA: need / matches of each dense entry
                    unsigned long long *bk = bk_s + warp * 36, *bt = bt_s + warp * 36;  // TS: key + limit + slot / matches
                    if (poss) {
#pragma unroll
                        for (int d = 0; d < D; d += 2)
                            *reinterpret_cast<double2 *>(brow + (size_t)my_rank * D + d) = make_double2(own[d], own[d + 1]);
                        if constexpr (SEL) bcls[my_rank] = cls_s[q_l];
                        if constexpr (AA) {
                            bc[my_rank] = pc_s[q_l];
                            bx[my_rank] = px_s[q_l];
                        }
                        if constexpr (PA) {
                            bn[my_rank] = pn_s[q_l];
                            bm[my_rank] = pm_s[q_l];
                        }
                        if constexpr (TS) {
                            bk[my_rank] = tk_s[q_l] | ((unsigned long long)s_l << 40);
                            bt[my_rank] = tm_s[q_l];
                        }
                    }
                    fnd[lane] = 0xFF;  // "nobody took dense entry `lane`" until a taker says otherwise
                    const unsigned fnd_sa = (unsigned)__cvta_generic_to_shared(const_cast<unsigned char *>(fnd));
                    if (lane < 4) {
                        double *pad = brow + (size_t)(n_poss + lane) * D;
                        pad[0] = __longlong_as_double(0x7FF0000000000000ll);
#pragma unroll
                        for (int d = 1; d < D; ++d) pad[d] = 0.0;
                        if constexpr (SEL) bcls[n_poss + lane] = 0;
                        if constexpr (AA) {
                            bc[n_poss + lane] = 0ull;
                            bx[n_poss + lane] = 0ull;
                        }
                        if constexpr (PA) {
                            bn[n_poss + lane] = 0ull;
                            bm[n_poss + lane] = 0ull;
                        }
                        if constexpr (TS) {
                            bk[n_poss + lane] = 0xFFull << 32;  // no key
                            bt[n_poss + lane] = 0ull;
                        }
                    }
                    __syncwarp();
                    double r[D];
                    load_row<D>(r, brow);
                    // SEL: does this lane's node match entry k?  It does not depend on S, so it is computed one entry
                    // ahead, beside the row load, and is ready before the add-compare-vote chain needs it.
                    bool mt = true;
                    if constexpr (SEL) mt = ((my_nm >> bcls[0]) & 1ull) != 0ull;
                    // AA: the entry's masks, loaded one entry ahead; the block test itself needs the node masks the
                    // previous vote left, so it is evaluated beside the resource test
                    unsigned long long ec = 0ull, ex = 0ull;
                    if constexpr (AA) {
                        ec = bc[0];
                        ex = bx[0];
                    }
                    unsigned long long en = 0ull, em = 0ull;  // PA: the entry's need / matches, loaded one entry ahead
                    if constexpr (PA) {
                        en = bn[0];
                        em = bm[0];
                    }
                    // TS: the entry's key + limit + slot and key matches, loaded one entry ahead; the count itself is
                    // read after the previous entry's take (this lane alone writes its node's counts)
                    unsigned long long ek = 0ull, et = 0ull;
                    if constexpr (TS) {
                        ek = bk[0];
                        et = bt[0];
                    }
                    const long long t_l0 = tracing ? clock64() : 0;
                    if (tracing) n_iter += (unsigned)n_poss;
                    // The placement chain.  Entry k's test needs the state left by entry k-1, which is only known once the
                    // vote of entry k-1 has named its taker: the vote-to-vote path below is compare -> ballot -> mask test
                    // -> select of the new state.  (A variant that prepared both outcomes of the next test beside the vote
                    // was measured against this loop and dropped: it doubles the float64 work for no gain.)
                    // nodes: the reference's  cap - (used + req) >= 0  (kube.py:175).  For finite float64 values the rounded
                    // difference has the sign of the exact one and is zero only for equal operands (gradual underflow), so
                    // fl(cap - t) >= 0  <=>  t <= cap  with t = fl(used + req): one add and one compare on the chain instead
                    // of two adds and a compare; t is also the state the node takes on when it accepts the entry.
                    auto fits = [&](const double (&st)[D], const double (&row)[D]) {
                        bool ok = true, ok2 = true;  // two independent and-chains over the dimensions
#pragma unroll
                        for (int d = 0; d < D / 2; ++d) {
                            if (BINS) ok = ok & (row[d] <= st[d]);   // == (st - row >= 0) for finite values (scaler.py:139)
                            else ok = ok & (__dadd_rn(st[d], row[d]) <= C[d]);
                        }
#pragma unroll
                        for (int d = D / 2; d < D; ++d) {
                            if (BINS) ok2 = ok2 & (row[d] <= st[d]);
                            else ok2 = ok2 & (__dadd_rn(st[d], row[d]) <= C[d]);
                        }
                        return ok & ok2;
                    };
                    for (int k0 = 0; k0 < n_poss; k0 += 4)
#pragma unroll
                    for (int k = k0; k < k0 + 4; ++k) {  // slots past n_poss hold never-fitting rows
                        double r_next[D];
                        load_row<D>(r_next, brow + (size_t)(k + 1) * D);
                        bool mt_next = true;
                        if constexpr (SEL) mt_next = ((my_nm >> bcls[k + 1]) & 1ull) != 0ull;
                        unsigned long long ec_next = 0ull, ex_next = 0ull;
                        if constexpr (AA) {
                            ec_next = bc[k + 1];
                            ex_next = bx[k + 1];
                        }
                        unsigned long long en_next = 0ull, em_next = 0ull;
                        if constexpr (PA) {
                            en_next = bn[k + 1];
                            em_next = bm[k + 1];
                        }
                        unsigned long long ek_next = 0ull, et_next = 0ull;
                        if constexpr (TS) {
                            ek_next = bk[k + 1];
                            et_next = bt[k + 1];
                        }
                        bool ok = fits(S, r);
                        if constexpr (SEL) ok = ok & mt;
                        if constexpr (AA) ok = ok & (((ec & my_nx) | (ex & my_nc)) == 0ull);
                        if constexpr (PA) ok = ok & (en == 0ull || (en & my_nh) != 0ull);
                        if constexpr (TS) {
                            const unsigned key = (unsigned)(ek >> 32) & 0xFFu;
                            ok = ok & (key == 0xFFu || cnt_s[key * Tn + my_cn] <= (int)(unsigned)ek);
                        }
                        // the vote-to-vote path: ballot -> "no fitting lane before me" -> predicated update of S -> next
                        // test.  No branch on it (at the frontier nearly every entry is taken) and no mask arithmetic
                        // beyond one and + compare.
                        const unsigned m = __ballot_sync(0xFFFFFFFFu, ok);
                        const unsigned loses = (m & le) ^ me;  // 0 <=> this is the first fitting node of the warp
#pragma unroll
                        for (int d = 0; d < D; ++d) state_take<BINS>(S[d], r[d], loses);  // scaler.py:140 / kube.py:171
                        if constexpr (AA) {
                            mask_take(my_nc, ec, loses);
                            mask_take(my_nx, ex, loses);
                        }
                        if constexpr (PA) mask_take(my_nh, em, loses);
                        if constexpr (TS) {
                            if (!loses && et) {  // the taker counts the pod on its node under every key it matches
                                const int64_t jj = (int64_t)(p.tile_lo + tile) * kTile + (int64_t)((ek >> 40) & 0xFFu);
                                for (unsigned long long w = et; w; w &= w - 1) {
                                    const int b = __ffsll((long long)w) - 1;
                                    const int c = cnt_s[b * Tn + my_cn] + 1;
                                    cnt_s[b * Tn + my_cn] = c;
                                    if (!BINS && c == tgt_s[b] && ((my_nd >> b) & 1ull)) {  // a domain reached the target
                                        atomicAdd(p.ts_reached + b, 1);
                                        atomicMax(p.ts_rise_pos + b, (unsigned long long)jj);
                                    }
                                }
                            }
                        }
                        note_take(fnd_sa + (unsigned)k, (unsigned)lane, loses);  // off the chain: who took entry k
                        my_takes += loses ? 0u : 1u;
#pragma unroll
                        for (int d = 0; d < D; ++d) r[d] = r_next[d];
                        if constexpr (SEL) mt = mt_next;
                        if constexpr (AA) {
                            ec = ec_next;
                            ex = ex_next;
                        }
                        if constexpr (PA) {
                            en = en_next;
                            em = em_next;
                        }
                        if constexpr (TS) {
                            ek = ek_next;
                            et = et_next;
                        }
                    }
                    __syncwarp();
                    {
                        const int found = poss ? (int)fnd[my_rank] : 0xFF;
                        if (found != 0xFF) placed_here = found;
                    }
                    const unsigned gotmask = __ballot_sync(0xFFFFFFFFu, placed_here >= 0);
                    n_placed += __popc(gotmask);
                    if (BINS && gotmask) {  // tighten the bound: the remaining amounts just shrank
#pragma unroll
                        for (int d = 0; d < D; ++d) Mx[d] = warp_upper_bound(S[d]);
                    }
                    if (!last) {
                        // forward what this warp did not take, in order, with one coalesced store
                        const unsigned fwd = __ballot_sync(0xFFFFFFFFu, mine && placed_here < 0);
                        if (mine && placed_here < 0) out_q[out + __popc(fwd & ((1u << lane) - 1u))] = e;
                        out += __popc(fwd);
                    }
                    if (tracing) t_loop += clock64() - t_l0;
                    if (placed_here >= 0) {  // bookkeeping off the critical path, one lane per placed entry
                        p.placed[(int64_t)(p.tile_lo + tile) * kTile + s_l] = (int32_t)(stage_lo + my_lo + placed_here);
                        atomicAnd(&alive_w[s_l >> 5], ~(1u << (s_l & 31)));
                        if constexpr (PA) {  // the first placement of a watched signature (rare; never with watch == 0)
                            unsigned long long w = pm_s[q_l] & p.watch;
                            if (w) {
                                const int64_t jj = (int64_t)(p.tile_lo + tile) * kTile + s_l;
                                const unsigned long long pos = (unsigned long long)(BINS ? (int64_t)p.pod_idx[jj] : jj);
                                for (; w; w &= w - 1) atomicMin(p.first_placed + (__ffsll((long long)w) - 1), pos);
                            }
                        }
                    }
                    head += (unsigned)n_ent;
                    done = endmask != 0;
                    if (tracing) { const long long now = clock64(); tb += now - t_mark; t_mark = now; }
                }
                if (!last && lane == 0) out_q[out] = kQueueEnd;
                if (lane == 0 && n_placed) atomicAdd(&misc[4], (unsigned)n_placed);
                if (tracing && lane == 0 && tile < 4096 && warp < 8)
                    p.trace[(size_t)(4096 + tile) * 8 + warp] = ((unsigned long long)(tb >> 5) & 0x7FFF) |
                        (((unsigned long long)(t_loop >> 5) & 0x7FFF) << 15) | ((unsigned long long)(head & 0x1FF) << 30) |
                        ((unsigned long long)(n_batches & 0x3F) << 39) | ((unsigned long long)(n_iter & 0x3FF) << 45) |
                        ((unsigned long long)(n_placed & 0x1FF) << 55);
                if (n_placed) {
                    // once per tile (not per batch): which lanes took a pod, and - bins - the credited tests: every bin
                    // before the chosen one plus the chosen one unless this pod opened it (= the first pod ever placed
                    // in that bin); the stage / warp base is added per placed pod
                    touched_tile = __ballot_sync(0xFFFFFFFFu, my_takes != 0u);
                    if (BINS) {
                        const unsigned ev_local = __reduce_add_sync(0xFFFFFFFFu, my_takes * (unsigned)(lane + 1)) -
                                                  (unsigned)__popc(touched_tile & ~touched_or_open);
                        touched_or_open |= touched_tile;
                        my_evals += (unsigned long long)ev_local + (unsigned long long)n_placed * (unsigned long long)(stage_lo + my_lo);
                    }
                    if constexpr (BINS && RW > 0) {  // a bin dies only by taking a pod: the warp's bins are checked here
                        bool short_d = false;
#pragma unroll
                        for (int d = 0; d < D; ++d) short_d = short_d | (S[d] < minreq_s[d]);
                        became_dead = __all_sync(0xFFFFFFFFu, n >= n_valid || (((touched_or_open >> lane) & 1u) && short_d));
                    }
                    if (n < Tn) {
#pragma unroll
                        for (int d = 0; d < D; ++d) state_s[(size_t)d * Tn + n] = S[d];
                        if constexpr (AA) {
                            nc_s[n] = my_nc;
                            nx_s[n] = my_nx;
                        }
                        if constexpr (PA) nh_s[n] = my_nh;
                    }
                    if (lane == 0) {
                        if (BINS) opened[warp] = touched_or_open;
                        dirty[warp] = touched_tile;
                    }
                }
            }
            __syncthreads();
            // wipe the queue entries this warp wrote so that the next tile starts from "not written"
            if (BINS ? ((chain >> warp) & 1u) && !chain_last : warp < n_warps - 1) {
                unsigned *out_q = queue + (size_t)warp * (kTile + 1);
                for (unsigned i = lane; i <= out; i += 32) out_q[i] = 0;
            }
            if (BINS && became_dead && lane == 0) atomicOr(&misc[6], 1u << warp);  // read from the next tile's (S1) on
        }
        ACSFIT_PROF(3)
        if (PROF_ON && tid == 0) { prof_acc[6] += nh; prof_acc[7] += 1; }
        const unsigned n_placed_tile = nh ? misc[4] : 0u;

        // ---- publish the surviving pods of the tile FIRST (warp 0): the next stage can start on the tile while this one
        // refreshes its own thresholds (the refresh only concerns this stage's later tiles) ----
        if (warp == 0) {
            forwarded += (long long)alive_total - (long long)n_placed_tile;
            if (lane == 0) {
                // ONE lane writes the tile's alive words and then the progress counter with a release store: the words
                // precede the release in program order, so no separate fence is needed (a fence costs about as much as
                // the release itself).  A tile in which this stage placed nothing wrote nothing: the release alone
                // carries the upstream stages' writes forward (release / acquire are cumulative).
                if (n_placed_tile || remote_in) {
#pragma unroll
                    for (int w = 0; w < kTile / 32; ++w) {
                        const int64_t wj = (int64_t)(p.tile_lo + tile) * (kTile / 32) + w;
                        if (wj * 32 < p.M) __stcg(p.alive + wj, alive_w[w]);
                    }
                }
                // A tile this stage placed nothing in changes nothing downstream needs at once.  In a pass of several
                // waves of stage CTAs (throughput-bound: every wave streams the whole pod list) its progress is published
                // with the next placing tile, every p.publish_every-th tile or the last one, whichever comes first - a
                // release store costs > 1000 cycles, as much as the rest of such a tile (c4 node pass 2.97 -> 2.63 s).
                // The frontier, which places, and the stages it has just left publish every tile; so does every stage of
                // a single-wave pass (latency-bound: publish_every = 1; batching cost the c2 tick 2 %).
                since_placed = n_placed_tile ? 0 : since_placed + 1;
                if (since_placed < kPublishGrace || remote_in || sys_out || ((tile + 1) % p.publish_every) == 0 ||
                    tile + 1 == p.num_tiles)
                    publish(tile + 1);
            }
        }
        ACSFIT_PROF(4)
        // ---- nodes: refresh the scan thresholds of the nodes that took a pod (all threads) ----
        if ((!BINS || RW > 0) && n_placed_tile) {
            if constexpr (RW > 0) {  // the packed rows of the nodes that took a pod are rebuilt field by field
                for (int i = tid; i < Tn * RW; i += NT) {
                    const int n = i / RW;
                    if ((dirty[n >> 5] >> (n & 31)) & 1u) tw_s[i] = 0;
                }
                __syncthreads();
            }
            for (int i = tid; i < Tn * D; i += NT) {
                const int d = i / Tn, n = i - d * Tn;
                if ((dirty[n >> 5] >> (n & 31)) & 1u) {
                    if (!BINS) thr_s[i] = node_threshold(cap_s[i], state_s[i]);
                    if constexpr (RW > 0) pack_field(i);
                }
            }
        }
        // node state changed: new bounds for the next tile (visible after its (S1))
        if (PRUNE && n_placed_tile) {
            __syncthreads();  // thresholds just rewritten by all threads
            refresh_bounds();
        }
        ACSFIT_PROF(5)
        if (PROF_ON && p.trace && tid == 0 && stage == p.trace_stage) {
            for (int i = 0; i < 6; ++i) {
                p.trace[(size_t)tile * 8 + i] = prof_acc[i] - trace_prev[i];
                trace_prev[i] = prof_acc[i];
            }
            p.trace[(size_t)tile * 8 + 6] = nh;
            p.trace[(size_t)tile * 8 + 7] = total;
        }
    }
#undef ACSFIT_PROF
    // ---- stage end: write the mutated node state back -------------------------------------
    __syncthreads();
    if (!BINS) {
        for (int i = tid; i < Tn * D; i += NT) {
            const int n = i / D, d = i - n * D;
            if (n < n_valid) p.used[(size_t)(stage_lo + n) * D + d] = state_s[(size_t)d * Tn + n];
        }
        if constexpr (AA)
            for (int n = tid; n < n_valid; n += NT) {
                p.node_carries[stage_lo + n] = nc_s[n];
                p.node_matches[stage_lo + n] = nx_s[n];
            }
        if constexpr (PA)
            for (int n = tid; n < n_valid; n += NT) p.node_has[stage_lo + n] = nh_s[n];
        if constexpr (TS)
            for (int i = tid; i < p.ts_keys * Tn; i += NT) {
                const int k = i / Tn, n = i - k * Tn;
                if (n < n_valid) p.ts_count[(size_t)k * p.ts_stride + stage_lo + n] = cnt_s[i];
            }
    }
    if (BINS && lane == 0 && my_evals) atomicAdd(p.evals, my_evals);  // every warp credits its own placements
    if (tid == 0) {
        if (misc[2]) publish(p.num_tiles);
        if (forwarded == 0) atomicExch(p.drained, 1);
        if (PROF_ON) {
            for (int i = 0; i < 8; ++i) p.prof[(size_t)stage * 8 + i] = prof_acc[i];
        }
    }
    // misc[6] is final: its last atomicOr precedes the barrier above.  The stage's warp count is recomputed from the
    // parameters and misc[0] so that no register stays live across the tile loop for it.
    if constexpr (BINS && RW > 0) {
        if (tid == 0 && p.retire_count && misc[6]) {
            const unsigned dead = misc[6];
            const int64_t lo = p.node_lo + (int64_t)misc[0] * p.Tn;
            const int nw = (int)((max((int64_t)0, min((int64_t)p.Tn, p.node_hi - lo)) + 31) >> 5);
            atomicAdd(p.retire_count, (unsigned long long)__popc(dead));
            if (dead == (1u << nw) - 1u) atomicAdd(p.retire_count + 1, 1ull);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// small kernels
// ---------------------------------------------------------------------------------------------

// K0: capacity.is_possible over the pools (capacity.py:24-32): literal (unit - req) >= 0
__global__ void feasible_mask_kernel(const double *__restrict__ req, int64_t P, int D,
                                     const double *__restrict__ unit, int T,
                                     uint8_t *__restrict__ out_mask, unsigned long long *out_evals)
{
    extern __shared__ double unit_s[];
    for (int i = threadIdx.x; i < T * D; i += blockDim.x) unit_s[i] = unit[i];
    __syncthreads();
    unsigned long long evals = 0;
    for (int64_t pidx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; pidx < P;
         pidx += (int64_t)gridDim.x * blockDim.x) {
        const double *r = req + (size_t)pidx * D;
        uint8_t ok = 0;
        for (int t = 0; t < T && !ok; ++t) {
            ++evals;
            bool all = true;
            for (int d = 0; d < D; ++d) all = all && fits_bin(unit_s[t * D + d], r[d]);
            ok = all ? 1 : 0;
        }
        out_mask[pidx] = ok;
    }
    if (out_evals) {
        for (int o = 16; o > 0; o >>= 1) evals += __shfl_down_sync(0xFFFFFFFFu, evals, o);
        if ((threadIdx.x & 31) == 0 && evals) atomicAdd(out_evals, evals);
    }
}

// pool gate of fulfill_pending (scaler.py:134) over the still-unaccounted pods
__global__ void eligible_kernel(const double *__restrict__ req, const int32_t *__restrict__ row_map,
                                int64_t P, int D, const double *__restrict__ unit /*D, device*/,
                                const int32_t *__restrict__ acc_pool, uint8_t *__restrict__ out_flag)
{
    for (int64_t pidx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; pidx < P;
         pidx += (int64_t)gridDim.x * blockDim.x) {
        uint8_t f = 0;
        if (acc_pool[pidx] < 0) {
            const double *r = req + (size_t)(row_map ? row_map[pidx] : pidx) * D;
            bool all = true;
            for (int d = 0; d < D; ++d) all = all && fits_bin(unit[d], r[d]);
            f = all ? 1 : 0;
        }
        out_flag[pidx] = f;
    }
}

// K0 with node selectors: a pool counts only when it matches the pod's selector class as well; one evaluation per
// pool visited (the match test is evaluated first and short-circuits, it is not a second evaluation)
__global__ void feasible_mask_sel_kernel(const double *__restrict__ req, int64_t P, int D,
                                         const double *__restrict__ unit, const unsigned long long *__restrict__ pool_match,
                                         int T, const uint8_t *__restrict__ pod_class,
                                         uint8_t *__restrict__ out_mask, unsigned long long *out_evals)
{
    extern __shared__ double unit_s[];
    unsigned long long *match_s = reinterpret_cast<unsigned long long *>(unit_s + T * D);
    for (int i = threadIdx.x; i < T * D; i += blockDim.x) unit_s[i] = unit[i];
    for (int i = threadIdx.x; i < T; i += blockDim.x) match_s[i] = pool_match[i];
    __syncthreads();
    unsigned long long evals = 0;
    for (int64_t pidx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; pidx < P;
         pidx += (int64_t)gridDim.x * blockDim.x) {
        const double *r = req + (size_t)pidx * D;
        const unsigned c = pod_class[pidx];
        uint8_t ok = 0;
        for (int t = 0; t < T && !ok; ++t) {
            ++evals;
            bool all = ((match_s[t] >> c) & 1ull) != 0ull;
            for (int d = 0; d < D; ++d) all = all && fits_bin(unit_s[t * D + d], r[d]);
            ok = all ? 1 : 0;
        }
        out_mask[pidx] = ok;
    }
    if (out_evals) {
        for (int o = 16; o > 0; o >>= 1) evals += __shfl_down_sync(0xFFFFFFFFu, evals, o);
        if ((threadIdx.x & 31) == 0 && evals) atomicAdd(out_evals, evals);
    }
}

// pool gate of fulfill_pending with node selectors: the pool matches the pod's class and (unit - req).possible
__global__ void eligible_sel_kernel(const double *__restrict__ req, const int32_t *__restrict__ row_map,
                                    int64_t P, int D, const double *__restrict__ unit /*D, device*/,
                                    unsigned long long pool_match, const uint8_t *__restrict__ pod_class,
                                    const int32_t *__restrict__ acc_pool, uint8_t *__restrict__ out_flag)
{
    for (int64_t pidx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; pidx < P;
         pidx += (int64_t)gridDim.x * blockDim.x) {
        uint8_t f = 0;
        if (acc_pool[pidx] < 0) {
            const int64_t row = row_map ? row_map[pidx] : pidx;
            const double *r = req + (size_t)row * D;
            bool all = ((pool_match >> pod_class[row]) & 1ull) != 0ull;
            for (int d = 0; d < D; ++d) all = all && fits_bin(unit[d], r[d]);
            f = all ? 1 : 0;
        }
        out_flag[pidx] = f;
    }
}

// K1: ordered occupancy sum per node (cluster.py:165-168), one thread per node
__global__ void occupancy_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ run_idx,
                                 const double *__restrict__ req_run, int64_t N, int D,
                                 double *__restrict__ used)
{
    for (int64_t n = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; n < N;
         n += (int64_t)gridDim.x * blockDim.x) {
        double acc[kMaxDims];
        for (int d = 0; d < D; ++d) acc[d] = used[(size_t)n * D + d];
        for (int64_t k = row_ptr[n]; k < row_ptr[n + 1]; ++k) {
            const double *r = req_run + (size_t)(run_idx ? (int64_t)run_idx[k] : k) * D;
            for (int d = 0; d < D; ++d) acc[d] = __dadd_rn(acc[d], r[d]);
        }
        for (int d = 0; d < D; ++d) used[(size_t)n * D + d] = acc[d];
    }
}

}  // namespace acsfit
