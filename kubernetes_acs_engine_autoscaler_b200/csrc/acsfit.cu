// acsfit.cu -- C ABI (include/acsfit.h) over the sm_90a kernels in acsfit_kernels.cuh.
// Host orchestration only: argument checks, scratch arena, launches, the per-pool loop of
// fulfill_pending.  There is no CPU implementation of any computation in this file: without a
// CUDA device acsfit_ctx_create fails and nothing else can be called.
#include "../../include/acsfit.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <array>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <tuple>
#include <vector>

#include "acsfit_admit.cuh"
#include "acsfit_kernels.cuh"
#include "acsfit_rank.cuh"
#include "acsfit_stream.cuh"
#include "acsfit_stream_ff.cuh"

using namespace acsfit;

// ---------------------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------------------
struct acsfit_ctx {
    int device = 0;
    int num_sms = 0;
    int min_stages = 0;       // 0 = number of SMs
    int watchdog_ms = 20000;
    std::map<std::tuple<int, int, int, int, int>, int> resident_cache;  // (D, bins, prune, rank words, Tn) -> stage CTAs the GPU holds
    int prune = -1;           // -1: automatic (node passes that run in waves), 0 / 1: forced (ACSFIT_PRUNE)
    int use_stream = 0;       // barrier-free streaming form of the pipeline kernel (acsfit_stream_ff.cuh; ACSFIT_STREAM / knob "stream")
    int use_ranks = 1;        // packed-rank scan when the tick's distinct request values allow it (ACSFIT_RANKS=0: never)
    RankLayout rk;            // rank tables of the current API call (rk.nw == 0: float64 scan)
    int retire = 1;           // bin passes with rank tables retire bins that can take no pod of the pass (knob "retire")
    // cluster mode (one cluster on `world` GPUs; see include/acsfit.h)
    int rank = 0, world = 1;
    unsigned char *xbase = nullptr;                     // this rank's exchange region (cudaMalloc, IPC-exported)
    unsigned char *peer[ACSFIT_MAX_RANKS] = {nullptr};  // every rank's region as mapped here (peer[rank] == xbase)
    size_t x_sync = 0, x_alive = 0, x_placed = 0, x_used = 0, x_bytes = 0;  // offsets inside a region
    int64_t x_max_pods = 0, x_max_nodes = 0;
    int x_max_dims = 0;
    int epoch = 0;                                      // in-stream barrier count (same on every rank)
    int force_blocks = 0;                               // developer knob "cluster_blocks"
    int inject_chain_timeout = 0;                       // test knob: treat the next n chained launches as timed out
    int bin_pass_stages = 0;                            // test knob: at most this many stages per bin pass (0: kMaxStagesPerPass)
    int chain_fallbacks = 0;                            // chained nodes+bins launches that hit the watchdog and were redone unchained
    uint64_t last_sel_hits = 0;                         // hit entries of the selector node passes of the last call (acsfit_last_sel_hits)
    unsigned long long *retire_dev = nullptr;           // [2] dead warps / retired stages of the last call's bin passes
    bool retire_counted = false;                        // retire_dev was zeroed by a bin pass of the last call (acsfit_last_bin_retirement)
    std::vector<int64_t> pa_flips;                      // (signature, position) fixed by the last *_pa call, one per rerun
    std::vector<int64_t> ts_rises;                      // (key, position) fixed by the last *_ts call, one per rerun
    // launch records of the current API call (acsfit_last_launches); rec_* are set by the caller of a pipeline launch
    std::vector<std::array<int, ACSFIT_LAUNCH_FIELDS>> launch_log;
    int rec_chained = 0, rec_pool = -1;
    ScanLaunch scan_rec = {};  // the K1 / K6 kernel of the current API call (acsfit_last_scan_launch); kernel 0 = none
    int bulk_cfg = 4;          // geometry of the K1 / K6 bulk-copy form (knob "bulk_cfg", env ACSFIT_BULK_CFG)
    int stream_bytes = 8192;   // staging bytes per warp of the K1 / K6 gather form (knob "stream_bytes", env ACSFIT_STREAM_BYTES)
    int cl_tn = 0, cl_stages = 0, cl_blocks = 0, cl_resident = 0;  // geometry of the last cluster node pass
    int smem_floor_kb = 0;    // >0: request at least this much dynamic smem per stage CTA (limits CTAs per SM)
    char err[512] = {0};
    // grow-only device arena, bump-allocated per API call
    unsigned char *arena = nullptr;
    size_t arena_cap = 0, arena_off = 0;
    // device copies of the host-entry buffers (grow-only)
    unsigned char *hbuf = nullptr;
    size_t hbuf_cap = 0, hbuf_off = 0;
    uint64_t launches = 0;
    // pipeline statistics of the last first-fit / bin-pack call
    bool timing = false;
    bool overlap = true;          // chain the first pool's bin pipeline behind the node pipeline (two streams)
    cudaStream_t side = nullptr;  // second stream for that
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    unsigned long long *prof_dev = nullptr;  // developer probe buffer [kProfStages][8] + trace [kProfTiles][8]
    int trace_stage = -1;
    std::vector<unsigned long long> prof_host;
    int prof_stages = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    double last_ms = 0.0;
    uint64_t last_decisions = 0;
    int last_stages = 0, last_tiles = 0;
};

static acsfit_status fail(acsfit_ctx *ctx, acsfit_status code, const char *fmt, ...)
{
    if (ctx) {
        va_list ap;
        va_start(ap, fmt);
        vsnprintf(ctx->err, sizeof ctx->err, fmt, ap);
        va_end(ap);
    }
    return code;
}

#define CUDA_TRY(expr)                                                                           \
    do {                                                                                         \
        cudaError_t e__ = (expr);                                                                \
        if (e__ != cudaSuccess)                                                                  \
            return fail(ctx, ACSFIT_E_CUDA, "%s failed: %s (%s:%d)", #expr,                      \
                        cudaGetErrorString(e__), __FILE__, __LINE__);                            \
    } while (0)

#define TRY(expr)                                \
    do {                                         \
        acsfit_status s__ = (expr);              \
        if (s__ != ACSFIT_OK) return s__;        \
    } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static acsfit_status arena_reserve(acsfit_ctx *ctx, size_t bytes, cudaStream_t st)
{
    if (bytes <= ctx->arena_cap) return ACSFIT_OK;
    CUDA_TRY(cudaStreamSynchronize(st));
    if (ctx->arena) CUDA_TRY(cudaFree(ctx->arena));
    ctx->arena = nullptr;
    ctx->arena_cap = 0;
    size_t cap = align_up(bytes + bytes / 4, 1 << 20);
    CUDA_TRY(cudaMalloc(&ctx->arena, cap));
    ctx->arena_cap = cap;
    return ACSFIT_OK;
}

template <typename T>
static T *arena_take(acsfit_ctx *ctx, size_t count)
{
    size_t off = align_up(ctx->arena_off, 256);
    size_t bytes = sizeof(T) * std::max<size_t>(count, 1);
    if (off + bytes > ctx->arena_cap) return nullptr;  // callers reserve an upper bound first
    ctx->arena_off = off + bytes;
    return reinterpret_cast<T *>(ctx->arena + off);
}

#define TAKE(var, T, count)                                                                 \
    T *var = arena_take<T>(ctx, (count));                                                   \
    if (!var) return fail(ctx, ACSFIT_E_NOMEM, "scratch arena too small for %s", #var)

static inline int grid_for(const acsfit_ctx *ctx, int64_t n, int block)
{
    int64_t g = (n + block - 1) / block;
    int64_t cap = (int64_t)ctx->num_sms * 8;
    return (int)std::max<int64_t>(1, std::min(g, cap));
}

// ---------------------------------------------------------------------------------------------
// utility kernels (ordered compaction, reductions, scatter)
// ---------------------------------------------------------------------------------------------
namespace {

constexpr int kCompactBlock = 256;
constexpr int kCompactItems = 8;  // per thread, consecutive
constexpr int kCompactChunk = kCompactBlock * kCompactItems;

struct FlagPred {
    const uint8_t *flag;
    __device__ bool operator()(int64_t i) const { return flag[i] != 0; }
};
struct BitPred {
    const uint32_t *bits;
    __device__ bool operator()(int64_t i) const { return (bits[i >> 5] >> (i & 31)) & 1u; }
};

template <typename Pred>
__global__ void compact_count_kernel(Pred pred, int64_t n, int *block_counts)
{
    __shared__ int wsum[kCompactBlock / 32];
    const int64_t base = (int64_t)blockIdx.x * kCompactChunk + (int64_t)threadIdx.x * kCompactItems;
    int c = 0;
    for (int i = 0; i < kCompactItems; ++i) c += (base + i < n && pred(base + i)) ? 1 : 0;
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xFFFFFFFFu, c, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
    __syncthreads();
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < kCompactBlock / 32; ++w) t += wsum[w];
        block_counts[blockIdx.x] = t;
    }
}

// exclusive scan of block_counts (single block), total -> *out_total
__global__ void compact_scan_kernel(int *block_counts, int nblocks, int64_t *out_total)
{
    __shared__ long long carry;
    __shared__ int wsum[32];
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += blockDim.x) {
        const int i = base + threadIdx.x;
        const int v = i < nblocks ? block_counts[i] : 0;
        int x = v;
        for (int o = 1; o < 32; o <<= 1) {
            int y = __shfl_up_sync(0xFFFFFFFFu, x, o);
            if ((threadIdx.x & 31) >= o) x += y;
        }
        if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            int w = threadIdx.x < (blockDim.x >> 5) ? wsum[threadIdx.x] : 0;
            for (int o = 1; o < 32; o <<= 1) {
                int y = __shfl_up_sync(0xFFFFFFFFu, w, o);
                if (threadIdx.x >= o) w += y;
            }
            wsum[threadIdx.x] = w;
        }
        __syncthreads();
        const long long warp_off = (threadIdx.x >> 5) ? wsum[(threadIdx.x >> 5) - 1] : 0;
        const long long incl = carry + warp_off + x;
        if (i < nblocks) block_counts[i] = (int)(incl - v);  // exclusive (fits: total <= 2^31)
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) carry = incl;
        __syncthreads();
    }
    if (threadIdx.x == 0) *out_total = carry;
}

// scatter: out[offset + rank] = map ? map[i] : i   for every i with pred(i), order preserved
template <typename Pred>
__global__ void compact_scatter_kernel(Pred pred, int64_t n, const int *block_offsets,
                                       const int32_t *map, int32_t *out)
{
    __shared__ int wsum[kCompactBlock / 32];
    const int64_t base = (int64_t)blockIdx.x * kCompactChunk + (int64_t)threadIdx.x * kCompactItems;
    bool f[kCompactItems];
    int c = 0;
    for (int i = 0; i < kCompactItems; ++i) {
        f[i] = base + i < n && pred(base + i);
        c += f[i] ? 1 : 0;
    }
    int x = c;
    for (int o = 1; o < 32; o <<= 1) {
        int y = __shfl_up_sync(0xFFFFFFFFu, x, o);
        if ((threadIdx.x & 31) >= o) x += y;
    }
    if ((threadIdx.x & 31) == 31) wsum[threadIdx.x >> 5] = x;
    __syncthreads();
    int warp_off = 0;
    for (int w = 0; w < (int)(threadIdx.x >> 5); ++w) warp_off += wsum[w];
    int pos = block_offsets[blockIdx.x] + warp_off + x - c;
    for (int i = 0; i < kCompactItems; ++i)
        if (f[i]) out[pos++] = map ? map[base + i] : (int32_t)(base + i);
}

__global__ void fill_i32_kernel(int32_t *p, int64_t n, int32_t v)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        p[i] = v;
}

// alive bits: all ones for entries < n
__global__ void fill_alive_kernel(uint32_t *w, int64_t n)
{
    const int64_t nw = (n + 31) / 32;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nw; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t rem = n - i * 32;
        w[i] = rem >= 32 ? 0xFFFFFFFFu : ((1u << rem) - 1u);
    }
}

// credited can_fit calls from a placement vector: sum(placed >= 0 ? placed + 1 : N)
__global__ void decisions_kernel(const int32_t *placed, int64_t P, int64_t N, unsigned long long *out)
{
    unsigned long long c = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t v = placed[i];
        c += v >= 0 ? (unsigned long long)v + 1ull : (unsigned long long)N;
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xFFFFFFFFu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}

// after a bins pass: cur_bin[pod] = placed[j] for the placed list entries; also max bin
__global__ void scatter_bins_kernel(const int32_t *list, const int32_t *placed, int64_t M,
                                    int32_t *cur_bin, int32_t *bin_of, int *max_bin)
{
    int m = -1;
    for (int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; j < M; j += (int64_t)gridDim.x * blockDim.x) {
        const int32_t b = placed[j];
        if (b >= 0) {
            const int32_t pod = list[j];
            cur_bin[pod] = b;
            bin_of[pod] = b;
            m = max(m, b);
        }
    }
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_down_sync(0xFFFFFFFFu, m, o));
    if ((threadIdx.x & 31) == 0 && m >= 0) atomicMax(max_bin, m);
}

// bins already assigned by a chained first pass: copy into bin_of and track the highest bin
__global__ void record_bins_kernel(const int32_t *cur_bin, int64_t P, int32_t *bin_of, int *max_bin)
{
    int m = -1;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t b = cur_bin[i];
        if (b >= 0) {
            bin_of[i] = b;
            m = max(m, b);
        }
    }
    for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_down_sync(0xFFFFFFFFu, m, o));
    if ((threadIdx.x & 31) == 0 && m >= 0) atomicMax(max_bin, m);
}
struct NegPredI32 {
    const int32_t *v;
    __device__ bool operator()(int64_t i) const { return v[i] < 0; }
};
// out[i] = src[idx[i]]
__global__ void gather_i32_kernel(const int32_t *src, const int32_t *idx, int64_t n, int32_t *out)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = src[idx[i]];
}
// count pods that are feasible for some pool but not eligible for one given pool
__global__ void count_ineligible_kernel(const uint8_t *feasible, const double *req, int64_t P, int D,
                                        const double *unit, unsigned long long *out)
{
    unsigned long long c = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x)
        if (feasible[i]) {
            bool all = true;
            for (int d = 0; d < D; ++d) all = all && fits_bin(unit[d], req[(size_t)i * D + d]);
            c += all ? 0 : 1;
        }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xFFFFFFFFu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
// the same with node selectors: a feasible pod is ineligible when the pool does not match its class either
__global__ void count_ineligible_sel_kernel(const uint8_t *feasible, const double *req, int64_t P, int D,
                                            const double *unit, unsigned long long pool_match, const uint8_t *pod_class,
                                            unsigned long long *out)
{
    unsigned long long c = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x)
        if (feasible[i]) {
            bool all = ((pool_match >> pod_class[i]) & 1ull) != 0ull;
            for (int d = 0; d < D; ++d) all = all && fits_bin(unit[d], req[(size_t)i * D + d]);
            c += all ? 0 : 1;
        }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xFFFFFFFFu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, c);
}
// selector classes must be < classes (<= 64): the kernels shift a 64-bit mask by the class; flag[0] |= 1 otherwise
// class 0 (no selector) matches every node: bit 0 of every node mask must be set; flag[0] |= 2 otherwise
__global__ void node_mask_check_kernel(const unsigned long long *node_match, int64_t n, int *flag)
{
    int bad = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        bad |= !(node_match[i] & 1ull);
    if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 2);
}
__global__ void class_check_kernel(const uint8_t *pod_class, int64_t n, int classes, int *flag)
{
    int bad = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        bad |= pod_class[i] >= classes;
    if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 1);
}

// scaler.py:172-175: pods of the first `take` bins become accounted
__global__ void account_kernel(const int32_t *cur_bin, int64_t P, int32_t take, int32_t pool,
                               int32_t *acc_pool, unsigned long long *count)
{
    unsigned long long c = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x) {
        const int32_t b = cur_bin[i];
        if (b >= 0 && b < take) {
            acc_pool[i] = pool;
            ++c;
        }
    }
    for (int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xFFFFFFFFu, c, o);
    if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, c);
}

// pod affinity: out[0] |= the OR of v[idx ? idx[i] : i] over i < n with gate == nullptr or gate[i] >= 0
__global__ void or_rows_kernel(const unsigned long long *v, const int32_t *idx, int64_t n, const int32_t *gate,
                               unsigned long long *out)
{
    unsigned long long m = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        if (!gate || gate[i] >= 0) m |= v[idx ? idx[i] : i];
    for (int o = 16; o > 0; o >>= 1) m |= __shfl_down_sync(0xFFFFFFFFu, m, o);
    if ((threadIdx.x & 31) == 0 && m) atomicOr(out, m);
}
// flip position of each signature: a pod at position pos treats signature s as absent iff pos <= f[s]
// (-1: present from the start, INT64_MAX: not placed yet)
struct PaFlips {
    long long f[64];
};
// pod affinity: the need of the pod at each position i < n (row idx ? idx[i] : i): its signature bit, or 0 while the
// bootstrap exception lets it land anywhere (it matches its own signature, and the signature is absent at its turn)
__global__ void pa_need_kernel(const unsigned long long *requires_, const unsigned long long *self, const int32_t *idx,
                               int64_t n, const PaFlips fl, unsigned long long *need)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = idx ? idx[i] : i;
        const unsigned long long r = requires_[row], sf = self[row];
        need[i] = sf && i <= fl.f[__ffsll((long long)sf) - 1] ? 0ull : r;
    }
}
// pod affinity: every pod_requires has at most one bit and pod_self is a subset of it; flag[0] |= 4 otherwise
__global__ void pa_check_kernel(const unsigned long long *requires_, const unsigned long long *self, int64_t n, int *flag)
{
    int bad = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const unsigned long long r = requires_[i];
        bad |= (r & (r - 1)) != 0 || (self[i] & ~r) != 0;
    }
    if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31) == 0) atomicOr(flag, 4);
}

// topology spread: the rises of the keys' minimums fixed so far, as the positions of each key's rises in ascending
// order (key k: pos[off[k]] .. pos[off[k + 1] - 1]): a pod at position p of key k sees the level base[k] + #{fixed
// rises of k at positions < p}
struct TsLevels {
    int base[64];
    int off[65];
    const long long *pos;  // [off[64]] (device)
};
// topology spread: the limit of the pod at each position i < n (row idx ? idx[i] : i), maxSkew - self + its key's
// level there, saturated at INT_MAX (a count never exceeds the pods placed, so a saturated limit never blocks)
__global__ void ts_lim_kernel(const uint8_t *key, const int32_t *skew, const int32_t *idx, int64_t n, const TsLevels lv,
                              int32_t *lim)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t row = idx ? idx[i] : i;
        const unsigned k = key[row];
        long long l = skew[row];
        if (k < 64u) {
            int lo = lv.off[k], hi = lv.off[k + 1];  // binary search: the rises of k before position i
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (lv.pos[mid] < i) lo = mid + 1;
                else hi = mid;
            }
            l += lv.base[k] + (lo - lv.off[k]);
        }
        lim[i] = (int32_t)min(l, (long long)INT_MAX);
    }
}
// topology spread, over the N nodes: target == nullptr: out_min[k] = min of the counts of k's domains, out_ndom[k] =
// their number; otherwise out_reached[k] = k's domains whose count is >= target[k]
__global__ void ts_domains_kernel(const int32_t *count, const unsigned long long *domain, int64_t N, int keys,
                                  const int *target, int *out_min, int *out_ndom, int *out_reached)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < N * keys; i += (int64_t)gridDim.x * blockDim.x) {
        const int k = (int)(i / N);
        const int64_t n = i - (int64_t)k * N;
        if (!((domain[n] >> k) & 1ull)) continue;
        const int c = count[i];
        if (target) {
            if (c >= target[k]) atomicAdd(out_reached + k, 1);
        } else {
            atomicMin(out_min + k, c);
            atomicAdd(out_ndom + k, 1);
        }
    }
}
// topology spread: flag[0] |= 8 for a pod_key >= keys (other than 0xFF), a negative pod_skew or a pod_matches bit at or
// above keys, |= 16 for a negative node count
__global__ void ts_check_kernel(const uint8_t *key, const int32_t *skew, const unsigned long long *matches, int64_t rows,
                                int keys, const int32_t *count, int64_t counts, int *flag)
{
    const unsigned long long outside = keys >= 64 ? 0ull : ~((1ull << keys) - 1ull);
    int bad = 0;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < rows || i < counts;
         i += (int64_t)gridDim.x * blockDim.x) {
        if (i < rows) bad |= ((key[i] != 0xFF && key[i] >= keys) || skew[i] < 0 || (matches[i] & outside) != 0) ? 8 : 0;
        if (i < counts) bad |= count[i] < 0 ? 16 : 0;
    }
    for (int o = 16; o > 0; o >>= 1) bad |= __shfl_down_sync(0xFFFFFFFFu, bad, o);
    if ((threadIdx.x & 31) == 0 && bad) atomicOr(flag, bad);
}

// domain check: requests must be >= 0 and not NaN; flag[0] |= 1 otherwise
__global__ void domain_kernel(const double *v, int64_t n, int *flag)
{
    bool bad = false;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        bad = bad || !(v[i] >= 0.0);
    if (bad) atomicOr(flag, 1);
}

// K6: Scaler.get_node_state (scaler.py:61-114), one thread per node, S thresholds at once
__global__ void node_states_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ run_idx,
                                   const double *__restrict__ req_run, const uint8_t *__restrict__ flags_run,
                                   const double *__restrict__ cap_type, const int32_t *__restrict__ node_type,
                                   const uint8_t *__restrict__ node_flags, const int64_t *__restrict__ node_age,
                                   int64_t N, int D, int any_pending,
                                   const int64_t *__restrict__ idle_threshold, int S,
                                   uint8_t *__restrict__ out_state)
{
    for (int64_t n = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; n < N; n += (int64_t)gridDim.x * blockDim.x) {
        double util[kMaxDims];
        for (int d = 0; d < D; ++d) util[d] = 0.0;
        bool busy = false, undrainable = false;
        const int64_t k1 = row_ptr[n + 1];
        for (int64_t k = row_ptr[n]; k < k1; ++k) {
            const int64_t j = run_idx ? (int64_t)run_idx[k] : k;
            const uint8_t f = flags_run[j];
            undrainable = undrainable || (f & ACSFIT_PODF_UNDRAINABLE);
            if (f & ACSFIT_PODF_BUSY) {
                busy = true;
                const double *r = req_run + (size_t)j * D;
                for (int d = 0; d < D; ++d) util[d] = __dadd_rn(util[d], r[d]);  // ordered sum
            }
        }
        const double *cap = cap_type + (size_t)node_type[n] * D;
        bool under = true;
        for (int d = 0; d < D; ++d) {
            // (UTIL_THRESHOLD * capacity - utilization).possible: multiply THEN subtract, no FMA
            const double left = __dsub_rn(__dmul_rn(cap[d], 0.3), util[d]);
            under = under && (left >= 0.0);
        }
        const uint8_t nf = node_flags[n];
        const bool unsched = nf & ACSFIT_NODEF_UNSCHEDULABLE;
        const bool pending = any_pending && !(nf & ACSFIT_NODEF_NO_PENDING_MATCH);
        const int64_t age = node_age[n];
        for (int s = 0; s < S; ++s) {
            uint8_t st;
            if (busy && !under) st = unsched ? ACSFIT_ST_BUSY_UNSCHEDULABLE : ACSFIT_ST_BUSY;
            else if (pending && !unsched) st = ACSFIT_ST_POD_PENDING;
            else if (age <= idle_threshold[s] && !unsched) st = ACSFIT_ST_GRACE_PERIOD;
            else if (under && (busy || !unsched))
                st = undrainable ? ACSFIT_ST_UNDER_UTILIZED_UNDRAINABLE : ACSFIT_ST_UNDER_UTILIZED_DRAINABLE;
            else st = unsched ? ACSFIT_ST_IDLE_UNSCHEDULABLE : ACSFIT_ST_IDLE_SCHEDULABLE;
            out_state[(size_t)s * N + n] = st;
        }
    }
}

// K1 / K6, warp-cooperative form (D in {2,4,8,16}): a warp owns 32 consecutive nodes; the CSR slice of
// those nodes is streamed through shared memory in chunks with one row per lane per load (full 16-byte
// vector loads, consecutive lanes -> consecutive CSR entries), then every lane consumes its own node's
// entries in order.  The ordered left-to-right float64 sum of the reference is preserved; only the memory
// access pattern changes (coalesced streaming instead of one scattered row per thread).
// kStreamWarps warps per CTA (acsfit_scan_plan.h, where the staging bytes per warp are chosen).
static int g_trace = 0;           // ACSFIT_TRACE=1: per-pass timings on stderr (with acsfit_ctx_set_timing)

template <int D, bool STATES, int kStreamBytesPerWarp>
__global__ void __launch_bounds__(kStreamWarps * 32)
node_stream_kernel(const int64_t *__restrict__ row_ptr, const int32_t *__restrict__ run_idx,
                   const double *__restrict__ req_run, const uint8_t *__restrict__ flags_run,
                   const double *__restrict__ cap_type, const int32_t *__restrict__ node_type,
                   const uint8_t *__restrict__ node_flags, const int64_t *__restrict__ node_age, int64_t N,
                   int any_pending, const int64_t *__restrict__ idle_threshold, int S,
                   uint8_t *__restrict__ out_state, double *__restrict__ used_inout)
{
    // A warp owns a CONTIGUOUS range of node groups (32 nodes each), hence one contiguous CSR range, which it
    // streams through two staging buffers without ever draining the pipe: chunk c+1 is in flight (cp.async, no
    // register staging) while chunk c is consumed, across group boundaries.
    constexpr int kChunk = kStreamBytesPerWarp / 2 / (8 * D);  // CSR entries per chunk
    constexpr int kIter = kChunk / 32;                         // entries per lane per chunk
    static_assert(kIter >= 1, "chunk smaller than a warp");
    extern __shared__ __align__(16) unsigned char stream_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *rows_s = reinterpret_cast<double *>(stream_smem) + (size_t)warp * 2 * kChunk * D;
    uint8_t *flags_s = stream_smem + (size_t)kStreamWarps * kStreamBytesPerWarp + (size_t)warp * 2 * kChunk;
    const int64_t groups = (N + 31) / 32;
    const int64_t n_warps = (int64_t)gridDim.x * kStreamWarps;
    const int64_t per = (groups + n_warps - 1) / n_warps;
    const int64_t g0 = ((int64_t)blockIdx.x * kStreamWarps + warp) * per;
    const int64_t g1 = min(groups, g0 + per);
    if (g0 >= g1) return;
    const int64_t K0 = row_ptr[g0 * 32], K1 = row_ptr[min(g1 * 32, N)];

    uint8_t fpend[kIter];  // flags of the chunk in flight
    // the CSR indices of a chunk are fetched one chunk before its rows are requested, so that no gather ever
    // waits for the index it depends on: round c issues rows(c+1) with indices loaded in round c-1
    constexpr int kPieces = D / 2;
    int32_t jp[kIter * kPieces];  // row of the 16-byte piece this lane copies (consecutive lanes, consecutive pieces)
    int32_t je[kIter];            // row of the entry whose flag byte this lane fetches
    auto load_idx = [&](int64_t kc) {
        const int len = (int)min((int64_t)kChunk, K1 - kc);
#pragma unroll
        for (int i = 0; i < kIter * kPieces; ++i) {
            const int e = (lane + 32 * i) / kPieces;
            jp[i] = e < len ? __ldg(run_idx + kc + e) : -1;
        }
        if (STATES) {
#pragma unroll
            for (int i = 0; i < kIter; ++i) {
                const int e = lane + 32 * i;
                je[i] = e < len ? __ldg(run_idx + kc + e) : -1;
            }
        }
    };
    auto issue = [&](int buf) {  // rows (cp.async, no register staging) and flag bytes of the chunk jp/je describe
#pragma unroll
        for (int i = 0; i < kIter * kPieces; ++i) {
            if (jp[i] >= 0) {
                const int piece = lane + 32 * i;
                const double *src = req_run + (size_t)jp[i] * D + 2 * (piece % kPieces);
                const unsigned dst = (unsigned)__cvta_generic_to_shared(rows_s + (size_t)buf * kChunk * D) + 16u * (unsigned)piece;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        if (STATES) {  // flag bytes travel through registers; they are parked in shared memory one chunk later
#pragma unroll
            for (int i = 0; i < kIter; ++i) fpend[i] = je[i] >= 0 ? __ldg(flags_run + je[i]) : (uint8_t)0;
        }
    };
    auto park_flags = [&](int buf) {
        if (STATES) {
#pragma unroll
            for (int i = 0; i < kIter; ++i) flags_s[buf * kChunk + lane + 32 * i] = fpend[i];
        }
    };

    // per-group state of this lane's node; the next group's row pointers (and used row) are fetched a group ahead
    int64_t g = g0;
    int64_t lo, hi, lo_n = 0, hi_n = 0;
    double acc[D], acc_n[D];
    bool busy = false, undrainable = false;
    auto fetch_group = [&](int64_t gg, int64_t &l, int64_t &h, double (&a0)[D]) {
        const int64_t nn = gg * 32 + lane;
        l = row_ptr[min(nn, N)];
        h = row_ptr[min(nn + 1, N)];  // lanes past N get an empty range
#pragma unroll
        for (int d = 0; d < D; ++d) a0[d] = (!STATES && nn < N) ? used_inout[(size_t)nn * D + d] : 0.0;
    };
    fetch_group(g0, lo, hi, acc);
    if (g0 + 1 < g1) fetch_group(g0 + 1, lo_n, hi_n, acc_n);
    int64_t group_end = __shfl_sync(0xFFFFFFFFu, hi, 31);

    auto finalize = [&]() {
        const int64_t n = g * 32 + lane;
        if (n >= N) return;
        if (!STATES) {
#pragma unroll
            for (int d = 0; d < D; ++d) used_inout[(size_t)n * D + d] = acc[d];
            return;
        }
        const double *cap = cap_type + (size_t)node_type[n] * D;
        bool under = true;
#pragma unroll
        for (int d = 0; d < D; ++d) {
            // (UTIL_THRESHOLD * capacity - utilization).possible: multiply THEN subtract, no FMA
            const double left = __dsub_rn(__dmul_rn(cap[d], 0.3), acc[d]);
            under = under && (left >= 0.0);
        }
        const uint8_t nf = node_flags[n];
        const bool unsched = nf & ACSFIT_NODEF_UNSCHEDULABLE;
        const bool pending = any_pending && !(nf & ACSFIT_NODEF_NO_PENDING_MATCH);
        const int64_t age = node_age[n];
        for (int s = 0; s < S; ++s) {
            uint8_t st;
            if (busy && !under) st = unsched ? ACSFIT_ST_BUSY_UNSCHEDULABLE : ACSFIT_ST_BUSY;
            else if (pending && !unsched) st = ACSFIT_ST_POD_PENDING;
            else if (age <= idle_threshold[s] && !unsched) st = ACSFIT_ST_GRACE_PERIOD;
            else if (under && (busy || !unsched))
                st = undrainable ? ACSFIT_ST_UNDER_UTILIZED_UNDRAINABLE : ACSFIT_ST_UNDER_UTILIZED_DRAINABLE;
            else st = unsched ? ACSFIT_ST_IDLE_UNSCHEDULABLE : ACSFIT_ST_IDLE_SCHEDULABLE;
            out_state[(size_t)s * N + n] = st;
        }
    };

    int buf = 0;
    if (K0 < K1) {
        load_idx(K0);
        issue(0);
        if (K0 + kChunk < K1) load_idx(K0 + kChunk);
    }
    for (int64_t kc = K0;; kc += kChunk, buf ^= 1) {
        const bool has_chunk = kc < K1;
        const int64_t chunk_end = has_chunk ? min(kc + kChunk, K1) : K1;
        if (has_chunk) {
            park_flags(buf);  // requested a whole chunk ago
            if (kc + kChunk < K1) {
                issue(buf ^ 1);                                          // chunk c+1: its indices are in registers
                if (kc + 2 * kChunk < K1) load_idx(kc + 2 * kChunk);    // chunk c+2: indices only
                asm volatile("cp.async.wait_group 1;" ::: "memory");
            } else {
                asm volatile("cp.async.wait_group 0;" ::: "memory");
            }
            __syncwarp();
        }
        const double *rows_b = rows_s + (size_t)buf * kChunk * D;
        const uint8_t *flags_b = flags_s + buf * kChunk;
        // every group with entries in this chunk; a group is closed as soon as its last entry has been seen
        while (g < g1) {
            if (has_chunk) {
                const int64_t a = max(lo, kc), b = min(hi, chunk_end);
                for (int64_t k = a; k < b; ++k) {
                    const int e = (int)(k - kc);
                    bool take = true;
                    if (STATES) {
                        const uint8_t f = flags_b[e];
                        undrainable = undrainable || (f & ACSFIT_PODF_UNDRAINABLE);
                        take = f & ACSFIT_PODF_BUSY;
                        busy = busy || take;
                    }
                    if (take) {
                        const double2 *r = reinterpret_cast<const double2 *>(rows_b + (size_t)e * D);
#pragma unroll
                        for (int d = 0; d < D / 2; ++d) {
                            const double2 v = r[d];
                            acc[2 * d] = __dadd_rn(acc[2 * d], v.x);      // ordered sum, pod-list order
                            acc[2 * d + 1] = __dadd_rn(acc[2 * d + 1], v.y);
                        }
                    }
                }
            }
            if (group_end > chunk_end) break;  // the group continues in the next chunk
            finalize();
            ++g;
            lo = lo_n;
            hi = hi_n;
#pragma unroll
            for (int d = 0; d < D; ++d) acc[d] = acc_n[d];
            busy = false;
            undrainable = false;
            group_end = __shfl_sync(0xFFFFFFFFu, hi, 31);
            if (g + 1 < g1) fetch_group(g + 1, lo_n, hi_n, acc_n);
        }
        if (g >= g1) break;
        __syncwarp();  // everyone is done with this buffer before it is refilled (two chunks from now)
    }
}

template <int D, bool STATES, int kStreamBytesPerWarp>
static cudaError_t launch_node_stream_b(int grid, cudaStream_t st, const int64_t *row_ptr, const int32_t *run_idx,
                                      const double *req_run, const uint8_t *flags_run, const double *cap_type,
                                      const int32_t *node_type, const uint8_t *node_flags, const int64_t *node_age,
                                      int64_t N, int any_pending, const int64_t *thr, int S, uint8_t *out_state,
                                      double *used, ScanLaunch *rec)
{
    constexpr int kChunk = kStreamBytesPerWarp / 2 / (8 * D);
    const size_t smem = (size_t)kStreamWarps * kStreamBytesPerWarp + (size_t)kStreamWarps * 2 * kChunk;
    auto kern = node_stream_kernel<D, STATES, kStreamBytesPerWarp>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    // persistent grid: exactly the CTAs that are resident at once (the caller passes SMs * 8 as an upper bound)
    int per_sm = 0, dev = 0, sms = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kStreamWarps * 32, smem) == cudaSuccess && per_sm > 0 &&
        cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess)
        grid = std::min(grid, per_sm * sms);
    kern<<<grid, kStreamWarps * 32, smem, st>>>(row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags,
                                                node_age, N, any_pending, thr, S, out_state, used);
    *rec = {STATES ? 2 : 1, kScanGather, D, kStreamBytesPerWarp, kStreamWarps, kChunk, grid, S};
    return cudaGetLastError();
}

// the bulk-copy or gather instantiation plan_scan chose (p.form is kScanBulk or kScanGather)
template <int D, bool STATES>
static cudaError_t launch_node_stream(const ScanPlan &p, int grid, cudaStream_t st, const int64_t *row_ptr,
                                      const int32_t *run_idx, const double *req_run, const uint8_t *flags_run,
                                      const double *cap_type, const int32_t *node_type, const uint8_t *node_flags,
                                      const int64_t *node_age, int64_t N, int any_pending, const int64_t *thr, int S,
                                      uint8_t *out_state, double *used, ScanLaunch *rec)
{
    if (p.form == kScanBulk) {  // contiguous table: TMA bulk copies (acsfit_stream.cuh); geometry = <bytes per warp, warps>
#define ACSFIT_BULK_ARGS grid, st, row_ptr, req_run, flags_run, cap_type, node_type, node_flags, node_age, N, any_pending, thr, S, out_state, used, rec
        if constexpr (D <= 8) {
            if (p.bytes_per_warp == 8192 && p.warps == 8) return launch_node_stream_bulk<D, STATES, 8192, 8>(ACSFIT_BULK_ARGS);
            if (p.bytes_per_warp == 16384 && p.warps == 12) return launch_node_stream_bulk<D, STATES, 16384, 12>(ACSFIT_BULK_ARGS);
            if (p.bytes_per_warp == 16384 && p.warps == 8) return launch_node_stream_bulk<D, STATES, 16384, 8>(ACSFIT_BULK_ARGS);
            if (p.bytes_per_warp == 32768 && p.warps == 6) return launch_node_stream_bulk<D, STATES, 32768, 6>(ACSFIT_BULK_ARGS);
            return launch_node_stream_bulk<D, STATES, 8192, 16>(ACSFIT_BULK_ARGS);  // measured best on H100 (DESIGN.md section 6)
        } else {
            return launch_node_stream_bulk<D, STATES, 16384, 8>(ACSFIT_BULK_ARGS);
        }
#undef ACSFIT_BULK_ARGS
    }
#define ACSFIT_STREAM_ARGS grid, st, row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags, node_age, N, any_pending, thr, S, out_state, used, rec
    if constexpr (D <= 4) { if (p.bytes_per_warp == 2048) return launch_node_stream_b<D, STATES, 2048>(ACSFIT_STREAM_ARGS); }
    if constexpr (D <= 8) { if (p.bytes_per_warp == 4096) return launch_node_stream_b<D, STATES, 4096>(ACSFIT_STREAM_ARGS); }
    return launch_node_stream_b<D, STATES, 8192>(ACSFIT_STREAM_ARGS);
#undef ACSFIT_STREAM_ARGS
}

// maintain actions ------------------------------------------------------------------------
constexpr int kMaintBlock = 256;
constexpr int kMaintRounds = 16;                       // nodes per block = 256 * 16
constexpr int kMaintChunk = kMaintBlock * kMaintRounds;

// phase 1 (only when the budget decrements, i.e. not dry_run): per-chunk, per-pool count of
// UNDER_UTILIZED_DRAINABLE nodes of scalable pools
__global__ void maintain_count_kernel(const uint8_t *state, const int32_t *node_pool, int64_t N,
                                      const uint8_t *pool_scalable, int T, int *counts /*[chunks][T]*/)
{
    extern __shared__ int hist[];
    for (int t = threadIdx.x; t < T; t += blockDim.x) hist[t] = 0;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * kMaintChunk;
    for (int r = 0; r < kMaintRounds; ++r) {
        const int64_t n = base + (int64_t)r * kMaintBlock + threadIdx.x;
        if (n < N) {
            const int t = node_pool[n];
            if (t >= 0 && t < T && pool_scalable[t] && state[n] == ACSFIT_ST_UNDER_UTILIZED_DRAINABLE)
                atomicAdd(&hist[t], 1);
        }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < T; t += blockDim.x) counts[(size_t)blockIdx.x * T + t] = hist[t];
}

// phase 2: exclusive scan over chunks for every pool (one thread per pool)
__global__ void maintain_scan_kernel(int *counts, int chunks, int T)
{
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= T) return;
    long long run = 0;
    for (int c = 0; c < chunks; ++c) {
        const int v = counts[(size_t)c * T + t];
        counts[(size_t)c * T + t] = (int)run;
        run += v;
    }
}

// phase 3: SPARE_AGENT substitution + action table, in node order inside each pool
__global__ void maintain_apply_kernel(uint8_t *state, const int32_t *node_pool, int64_t N,
                                      const long long *budget0, const uint8_t *pool_scalable, int T,
                                      int dry_run, const int *chunk_rank /*[chunks][T] or null*/,
                                      uint8_t *action)
{
    extern __shared__ int running[];  // per pool: UUD nodes seen so far in this chunk
    for (int t = threadIdx.x; t < T; t += blockDim.x)
        running[t] = chunk_rank ? chunk_rank[(size_t)blockIdx.x * T + t] : 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int64_t base = (int64_t)blockIdx.x * kMaintChunk;
    for (int r = 0; r < kMaintRounds; ++r) {
        const int64_t n = base + (int64_t)r * kMaintBlock + threadIdx.x;
        const bool in = n < N;
        int t = in ? node_pool[n] : -1;
        const bool scal = in && t >= 0 && t < T && pool_scalable[t];
        uint8_t st = in ? state[n] : 0;
        const bool uud = scal && st == ACSFIT_ST_UNDER_UTILIZED_DRAINABLE;
        int rank = 0;
        if (!dry_run) {
            // rank of this node among the UUD nodes of its pool, in node order: warps take turns
            for (int w = 0; w < kMaintBlock / 32; ++w) {
                if (warp == w) {
                    const unsigned um = __ballot_sync(0xFFFFFFFFu, uud);
                    if (uud) {
                        const unsigned same = __match_any_sync(um, t);
                        const int seen = running[t];
                        __syncwarp(um);  // everyone has read the counter before a leader bumps it
                        rank = seen + __popc(same & ((1u << lane) - 1u));
                        if ((int)(__ffs(same) - 1) == lane) running[t] = seen + __popc(same);
                    }
                }
                __syncthreads();
            }
        }
        if (!in) continue;
        uint8_t act = ACSFIT_ACT_NONE;
        if (!scal) {
            st = ACSFIT_ST_NOT_EVALUATED;
        } else {
            if (uud) {
                const long long b0 = budget0[t];
                // engine_scaler.py:142-144: spare when the budget is exactly 0 at this node's turn.
                // dry run: the budget never moves.  otherwise it drops by one per drained node and
                // stays at 0 once it got there (a negative start never reaches 0).
                const bool spare = dry_run ? (b0 == 0) : (b0 >= 0 && (long long)rank >= b0);
                if (spare) st = ACSFIT_ST_SPARE_AGENT;
            }
            switch (st) {
            case ACSFIT_ST_UNDER_UTILIZED_DRAINABLE: act = ACSFIT_ACT_CORDON_DRAIN; break;
            case ACSFIT_ST_IDLE_SCHEDULABLE: act = ACSFIT_ACT_CORDON; break;
            case ACSFIT_ST_BUSY_UNSCHEDULABLE: act = ACSFIT_ACT_UNCORDON; break;
            case ACSFIT_ST_IDLE_UNSCHEDULABLE: act = ACSFIT_ACT_SCALE_IN; break;
            default: break;
            }
        }
        state[n] = st;
        action[n] = act;
    }
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// ABI: context
// ---------------------------------------------------------------------------------------------
extern "C" int acsfit_abi_version(void) { return ACSFIT_ABI_VERSION; }

extern "C" const char *acsfit_last_error(const acsfit_ctx *ctx) { return ctx ? ctx->err : "null ctx"; }

extern "C" acsfit_status acsfit_ctx_create(int device, acsfit_ctx **out_ctx)
{
    if (!out_ctx) return ACSFIT_E_INVALID;
    *out_ctx = nullptr;
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count)
        return ACSFIT_E_CUDA;  // no GPU: there is no CPU fallback
    acsfit_ctx *ctx = new (std::nothrow) acsfit_ctx();
    if (!ctx) return ACSFIT_E_NOMEM;
    ctx->device = device;
    cudaDeviceProp prop;
    if (cudaSetDevice(device) != cudaSuccess || cudaGetDeviceProperties(&prop, device) != cudaSuccess ||
        prop.major != 9 || prop.minor != 0) {
        delete ctx;
        return ACSFIT_E_CUDA;  // built for sm_90a only
    }
    ctx->num_sms = prop.multiProcessorCount;
    if (cudaEventCreate(&ctx->ev0) != cudaSuccess || cudaEventCreate(&ctx->ev1) != cudaSuccess) {
        delete ctx;
        return ACSFIT_E_CUDA;
    }
    if (const char *env = getenv("ACSFIT_SMEM_FLOOR_KB")) ctx->smem_floor_kb = atoi(env);
    if (const char *env = getenv("ACSFIT_OVERLAP")) ctx->overlap = atoi(env) != 0;
    if (const char *env = getenv("ACSFIT_PRUNE")) ctx->prune = atoi(env);
    if (const char *env = getenv("ACSFIT_RANKS")) ctx->use_ranks = atoi(env) != 0;
    if (const char *env = getenv("ACSFIT_STREAM")) ctx->use_stream = atoi(env) != 0;
    memset(&ctx->rk, 0, sizeof ctx->rk);
    if (const char *env = getenv("ACSFIT_MIN_STAGES")) ctx->min_stages = std::max(0, atoi(env));
    if (const char *env = getenv("ACSFIT_STREAM_BYTES")) ctx->stream_bytes = atoi(env);
    if (const char *env = getenv("ACSFIT_BULK_CFG")) ctx->bulk_cfg = atoi(env);
    if (const char *env = getenv("ACSFIT_TRACE")) g_trace = atoi(env);
    if (cudaStreamCreateWithFlags(&ctx->side, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_join, cudaEventDisableTiming) != cudaSuccess ||
        cudaMalloc(&ctx->retire_dev, 2 * sizeof(unsigned long long)) != cudaSuccess) {
        delete ctx;
        return ACSFIT_E_CUDA;
    }
    *out_ctx = ctx;
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_ctx_destroy(acsfit_ctx *ctx)
{
    if (!ctx) return ACSFIT_E_INVALID;
    cudaSetDevice(ctx->device);
    if (ctx->arena) cudaFree(ctx->arena);
    if (ctx->hbuf) cudaFree(ctx->hbuf);
    for (int r = 0; r < ACSFIT_MAX_RANKS; ++r)  // cluster mode: unmap the peers' exchange regions, free our own
        if (ctx->peer[r] && ctx->peer[r] != ctx->xbase) cudaIpcCloseMemHandle(ctx->peer[r]);
    if (ctx->xbase) cudaFree(ctx->xbase);
    if (ctx->prof_dev) cudaFree(ctx->prof_dev);
    if (ctx->retire_dev) cudaFree(ctx->retire_dev);
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_join) cudaEventDestroy(ctx->ev_join);
    if (ctx->side) cudaStreamDestroy(ctx->side);
    delete ctx;
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_ctx_configure(acsfit_ctx *ctx, int min_stages, int watchdog_ms)
{
    if (!ctx || min_stages < 0 || watchdog_ms < 0) return ACSFIT_E_INVALID;
    ctx->min_stages = min_stages;
    if (watchdog_ms) ctx->watchdog_ms = watchdog_ms;
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_ctx_set_knob(acsfit_ctx *ctx, const char *name, int value)
{
    if (!ctx || !name) return ACSFIT_E_INVALID;
    if (!strcmp(name, "ranks")) ctx->use_ranks = value != 0;
    else if (!strcmp(name, "stream")) ctx->use_stream = value != 0;
    else if (!strcmp(name, "retire")) ctx->retire = value != 0;
    else if (!strcmp(name, "prune")) ctx->prune = value;
    else if (!strcmp(name, "overlap")) ctx->overlap = value != 0;
    else if (!strcmp(name, "min_stages")) ctx->min_stages = std::max(0, value);
    else if (!strcmp(name, "cluster_blocks")) ctx->force_blocks = std::max(0, value);
    else if (!strcmp(name, "inject_chain_timeout")) ctx->inject_chain_timeout = std::max(0, value);
    else if (!strcmp(name, "bin_pass_stages")) ctx->bin_pass_stages = std::max(0, value);
    else if (!strcmp(name, "bulk_cfg")) ctx->bulk_cfg = value;
    else if (!strcmp(name, "stream_bytes")) ctx->stream_bytes = value;
    else return fail(ctx, ACSFIT_E_INVALID, "unknown knob %s", name);
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_ctx_set_timing(acsfit_ctx *ctx, int enabled)
{
    if (!ctx) return ACSFIT_E_INVALID;
    ctx->timing = enabled != 0;
    return ACSFIT_OK;
}

// developer probe (not part of the stable ABI surface the host layer uses): per-stage clock64 phase
// totals of the LAST pipeline launch. rows = stages, 8 columns.
constexpr int kProfStages = 4096;
constexpr int kProfTiles = 8192;
extern "C" ACSFIT_API acsfit_status acsfit_debug_trace(acsfit_ctx *ctx, int stage, unsigned long long *out, int max_tiles)
{
    if (!ctx) return ACSFIT_E_INVALID;
    ctx->trace_stage = stage;
    if (out && ctx->prof_dev) {
        const int n = std::min(max_tiles, kProfTiles);
        CUDA_TRY(cudaMemcpy(out, ctx->prof_dev + (size_t)kProfStages * 8, sizeof(unsigned long long) * n * 8,
                            cudaMemcpyDeviceToHost));
    }
    return ACSFIT_OK;
}
extern "C" ACSFIT_API acsfit_status acsfit_debug_profile(acsfit_ctx *ctx, int enabled, unsigned long long *out,
                                                         int max_stages, int *out_stages)
{
    if (!ctx) return ACSFIT_E_INVALID;
    if (enabled && !kProfileBuild)
        return fail(ctx, ACSFIT_E_INVALID, "the stage profile is compiled out: rebuild with `python -m kubernetes_acs_engine_autoscaler_b200.build --profile`");
    if (enabled && !ctx->prof_dev) {
        CUDA_TRY(cudaMalloc(&ctx->prof_dev, sizeof(unsigned long long) * (kProfStages + kProfTiles) * 8));
    }
    if (!enabled && ctx->prof_dev) {
        cudaFree(ctx->prof_dev);
        ctx->prof_dev = nullptr;
    }
    if (out && ctx->prof_dev && ctx->prof_stages > 0) {
        const int n = std::min(std::min(ctx->prof_stages, max_stages), kProfStages);
        CUDA_TRY(cudaMemcpy(out, ctx->prof_dev, sizeof(unsigned long long) * n * 8, cudaMemcpyDeviceToHost));
        if (out_stages) *out_stages = n;
    } else if (out_stages) {
        *out_stages = 0;
    }
    return ACSFIT_OK;
}

extern "C" uint64_t acsfit_launch_count(const acsfit_ctx *ctx) { return ctx ? ctx->launches : 0; }

extern "C" acsfit_status acsfit_last_pipeline_stats(const acsfit_ctx *ctx, double *out_ms,
                                                    uint64_t *out_decisions, int *out_stages, int *out_tiles)
{
    if (!ctx) return ACSFIT_E_INVALID;
    if (out_ms) *out_ms = ctx->last_ms;
    if (out_decisions) *out_decisions = ctx->last_decisions;
    if (out_stages) *out_stages = ctx->last_stages;
    if (out_tiles) *out_tiles = ctx->last_tiles;
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_last_launches(const acsfit_ctx *ctx, int *out, int max_records, int *out_n)
{
    if (!ctx || !out_n || max_records < 0 || (max_records > 0 && !out)) return ACSFIT_E_INVALID;
    const int n = (int)std::min<size_t>(ctx->launch_log.size(), (size_t)max_records);
    for (int i = 0; i < n; ++i) memcpy(out + (size_t)i * ACSFIT_LAUNCH_FIELDS, ctx->launch_log[i].data(), sizeof(int) * ACSFIT_LAUNCH_FIELDS);
    *out_n = (int)ctx->launch_log.size();
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_last_sel_hits(const acsfit_ctx *ctx, uint64_t *out)
{
    if (!ctx || !out) return ACSFIT_E_INVALID;
    *out = ctx->last_sel_hits;
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_last_bin_retirement(const acsfit_ctx *ctx, uint64_t out[2])
{
    if (!ctx || !out) return ACSFIT_E_INVALID;
    out[0] = out[1] = 0;
    if (!ctx->retire_counted) return ACSFIT_OK;
    // every bin pass of the call has finished: the entry points synchronise before they return
    if (cudaSetDevice(ctx->device) != cudaSuccess ||
        cudaMemcpy(out, ctx->retire_dev, 2 * sizeof(uint64_t), cudaMemcpyDeviceToHost) != cudaSuccess)
        return ACSFIT_E_CUDA;
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_last_affinity_reruns(const acsfit_ctx *ctx, int64_t *out_reruns, int64_t *out_flips)
{
    if (!ctx || !out_reruns) return ACSFIT_E_INVALID;
    *out_reruns = (int64_t)ctx->pa_flips.size() / 2;
    if (out_flips) std::copy(ctx->pa_flips.begin(), ctx->pa_flips.end(), out_flips);
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_last_spread_rises(const acsfit_ctx *ctx, int64_t *out_rises, int64_t *out_pairs)
{
    if (!ctx || !out_rises) return ACSFIT_E_INVALID;
    *out_rises = (int64_t)ctx->ts_rises.size() / 2;
    if (out_pairs) std::copy(ctx->ts_rises.begin(), ctx->ts_rises.end(), out_pairs);
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_last_scan_launch(const acsfit_ctx *ctx, int *out)
{
    static_assert(sizeof(ScanLaunch) == sizeof(int) * ACSFIT_SCAN_FIELDS, "one int per record field");
    if (!ctx || !out) return ACSFIT_E_INVALID;
    memcpy(out, &ctx->scan_rec, sizeof(ScanLaunch));
    return ACSFIT_OK;
}

// ---------------------------------------------------------------------------------------------
// helpers shared by the entry points
// ---------------------------------------------------------------------------------------------
static bool pipeline_dims_ok(int D) { return D == 2 || D == 4 || D == 8 || D == 16; }

// the first-fit pipeline reads request rows as 16-byte double2 vectors (load_row / prefetch_row); there is no
// scalar fall-back, so a table that is not 16-byte aligned is refused before anything is launched
static acsfit_status check_req_aligned(acsfit_ctx *ctx, const double *req, const char *what)
{
    if (!aligned16(req)) return fail(ctx, ACSFIT_E_INVALID, "%s: req must be 16-byte aligned", what);
    return ACSFIT_OK;
}

// the argument checks every first_fit_nodes* entry point makes before anything else
static acsfit_status check_first_fit_args(acsfit_ctx *ctx, const char *what, const double *req, int64_t req_rows,
                                          const void *pod_idx, int64_t P, int D, const void *cap_type,
                                          const void *node_type, const void *used, int64_t N, const void *placed)
{
    if (P < 0 || N < 0 || req_rows < 0 || P > INT32_MAX || N > INT32_MAX || (!pod_idx && P > req_rows) ||
        (P > 0 && (!req || !placed)) || (N > 0 && (!cap_type || !node_type || !used)))
        return fail(ctx, ACSFIT_E_INVALID, "%s: bad arguments", what);
    if (!pipeline_dims_ok(D))
        return fail(ctx, ACSFIT_E_INVALID, "%s: D=%d, need 2/4/8/16 (zero columns are neutral)", what, D);
    return check_req_aligned(ctx, req, what);
}

// the argument checks every fulfill_pending* entry point makes before anything else
static acsfit_status check_fulfill_args(acsfit_ctx *ctx, const char *what, const double *req, int64_t Pp,
                                        int64_t num_listed, int D, const void *unit, const void *pool_actual,
                                        const void *pool_max, const void *pool_ignored, int T, const void *new_size,
                                        const void *units_needed, const void *bins_opened, const void *acc_pool,
                                        const void *bin_of, const void *unaccounted)
{
    if (Pp < 0 || Pp > INT32_MAX || num_listed < Pp || T < 0 || T > ACSFIT_MAX_POOLS ||
        (Pp > 0 && (!req || !acc_pool || !bin_of)) ||
        (T > 0 && (!unit || !pool_actual || !pool_max || !pool_ignored || !new_size || !units_needed || !bins_opened)) ||
        !unaccounted)
        return fail(ctx, ACSFIT_E_INVALID, "%s: bad arguments", what);
    if (!pipeline_dims_ok(D))
        return fail(ctx, ACSFIT_E_INVALID, "%s: D=%d, need 2/4/8/16 (zero columns are neutral)", what, D);
    return check_req_aligned(ctx, req, what);
}

// the end of every device-side check: copy its flag word to the host and wait for it
static acsfit_status flag_to_host(acsfit_ctx *ctx, const int *flag_dev, cudaStream_t st, int *flag)
{
    CUDA_TRY(cudaMemcpyAsync(flag, flag_dev, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return ACSFIT_OK;
}

static acsfit_status enter(acsfit_ctx *ctx, int D)
{
    if (!ctx) return ACSFIT_E_INVALID;
    if (D < 1 || D > ACSFIT_MAX_DIMS) return fail(ctx, ACSFIT_E_INVALID, "D=%d outside [1,%d]", D, ACSFIT_MAX_DIMS);
    cudaError_t e = cudaSetDevice(ctx->device);
    if (e != cudaSuccess) return fail(ctx, ACSFIT_E_CUDA, "cudaSetDevice: %s", cudaGetErrorString(e));
    ctx->arena_off = 0;
    ctx->rk.nw = 0;  // rank tables live in the arena of one API call
    ctx->launch_log.clear();
    ctx->scan_rec = ScanLaunch{};
    ctx->rec_chained = 0;
    ctx->rec_pool = -1;
    ctx->retire_counted = false;  // (reset_stats clears it too: the redo of a timed-out chained launch)
    return ACSFIT_OK;
}

static acsfit_status check_domain(acsfit_ctx *ctx, const double *v, int64_t n, int *flag_dev, cudaStream_t st,
                                  const char *what)
{
    if (n <= 0) return ACSFIT_OK;
    CUDA_TRY(cudaMemsetAsync(flag_dev, 0, sizeof(int), st));
    domain_kernel<<<grid_for(ctx, n, 256), 256, 0, st>>>(v, n, flag_dev);
    ++ctx->launches;
    int flag = 0;
    TRY(flag_to_host(ctx, flag_dev, st, &flag));
    if (flag) return fail(ctx, ACSFIT_E_DOMAIN, "%s contains a negative or NaN quantity", what);
    return ACSFIT_OK;
}

// ordered compaction: out_list = [map ? map[i] : i  for i in range(n) if pred(i)]; count to host
template <typename Pred>
static acsfit_status compact(acsfit_ctx *ctx, Pred pred, int64_t n, const int32_t *map, int32_t *out_list,
                             int *block_counts, int64_t *total_dev, int64_t *total_host, cudaStream_t st)
{
    *total_host = 0;
    if (n <= 0) return ACSFIT_OK;
    const int nblocks = (int)((n + kCompactChunk - 1) / kCompactChunk);
    compact_count_kernel<<<nblocks, kCompactBlock, 0, st>>>(pred, n, block_counts);
    compact_scan_kernel<<<1, 1024, 0, st>>>(block_counts, nblocks, total_dev);
    compact_scatter_kernel<<<nblocks, kCompactBlock, 0, st>>>(pred, n, block_counts, map, out_list);
    ctx->launches += 3;
    CUDA_TRY(cudaMemcpyAsync(total_host, total_dev, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    return ACSFIT_OK;
}

// ---------------------------------------------------------------------------------------------
// rank tables of the packed-rank scan (acsfit_rank.cuh).  On success ctx->rk describes the layout; when a
// dimension has too many distinct values, or the fields need more than 128 bits, ctx->rk.nw stays 0 and the
// pipelines run their float64 compare scan.  Scratch comes from the arena of the current API call.
// ---------------------------------------------------------------------------------------------
static size_t rank_scratch(int64_t rows, int D)
{
    return (size_t)D * kRankSlots * (sizeof(unsigned long long) + sizeof(unsigned short)) +
           (size_t)D * kRankCap * sizeof(double) + sizeof(uint32_t) * 4 * (size_t)std::max<int64_t>(rows, 1) + 16 * 256;
}

static acsfit_status build_ranks(acsfit_ctx *ctx, const double *req, int64_t rows, int D, cudaStream_t st)
{
    ctx->rk.nw = 0;
    if (!ctx->use_ranks || rows <= 0) return ACSFIT_OK;
    TAKE(keys, unsigned long long, (size_t)D * kRankSlots);
    TAKE(ranks, unsigned short, (size_t)D * kRankSlots);
    TAKE(sorted, double, (size_t)D * kRankCap);
    TAKE(counts, int, 16);
    TAKE(packed, uint32_t, 4 * (size_t)rows);
    CUDA_TRY(cudaMemsetAsync(keys, 0xFF, sizeof(unsigned long long) * (size_t)D * kRankSlots, st));
    CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(int) * 16, st));
    rank_insert_kernel<<<grid_for(ctx, rows * D, 256), 256, 0, st>>>(req, rows, D, keys, counts);
    // function attributes are per device: set at every call, like every other launch here, so that a ctx on a
    // second device of the process gets the 64 KB too
    CUDA_TRY(cudaFuncSetAttribute(rank_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)(sizeof(unsigned long long) * kRankCap)));
    rank_sort_kernel<<<D, 1024, sizeof(unsigned long long) * kRankCap, st>>>(keys, counts, sorted, ranks);
    ctx->launches += 2;
    int U[16];
    CUDA_TRY(cudaMemcpyAsync(U, counts, sizeof(int) * 16, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    // field layout: dimension d needs bitlen(U_d) bits for t' in [0, U_d] plus one guard bit; fields are placed
    // in dimension order and never straddle a 32-bit word
    RankLayout rk;
    memset(&rk, 0, sizeof rk);
    RankFields f;
    memset(&f, 0, sizeof f);
    int word = 0, used = 0;
    for (int d = 0; d < D; ++d) {
        if (U[d] > kRankCap || U[d] < 1) return ACSFIT_OK;  // too many distinct values: float64 scan
        int bits = 0;
        while ((1 << bits) <= U[d]) ++bits;
        if (used + bits + 1 > 32) {
            ++word;
            used = 0;
        }
        if (word >= 4) return ACSFIT_OK;  // does not fit 128 bits: float64 scan
        rk.word[d] = f.word[d] = (uint8_t)word;
        rk.shift[d] = f.shift[d] = (uint8_t)used;
        rk.guard[word] |= 1u << (used + bits);
        rk.count[d] = U[d];
        used += bits + 1;
    }
    const int nw = word + 1 == 3 ? 4 : word + 1;
    rank_pack_kernel<<<grid_for(ctx, rows, 256), 256, 0, st>>>(req, rows, D, keys, ranks, f, nw, packed);
    ++ctx->launches;
    CUDA_TRY(cudaGetLastError());
    rk.nw = nw;
    rk.sorted = sorted;
    rk.packed = packed;
    ctx->rk = rk;
    return ACSFIT_OK;
}

struct StagePlan {
    int Tn, NS, stages;
};

// cut `n_nodes` nodes into stages: the widest stage (<= 1024 nodes) that still gives at
// least `min_stages` stages, so that every SM has a stage to run.
static StagePlan plan_stages(const acsfit_ctx *ctx, int64_t n_nodes, int max_stages, int D, bool bins)
{
    const int want = ctx->min_stages > 0 ? ctx->min_stages : ctx->num_sms;  // one stage per SM measured best
    const int K = nodes_per_thread(D, ctx->rk.nw);
    int NS = max_stage_nodes(D, bins) / K;
    const int ns_min = (ctx->use_stream && ctx->rk.nw > 0 && D <= 8) ? std::max(1, 32 / K) : 1;  // streaming form: stages of >= 32 nodes
    while (NS > ns_min && (n_nodes + (int64_t)NS * K - 1) / ((int64_t)NS * K) < want) NS >>= 1;
    StagePlan p;
    p.NS = NS;
    p.Tn = NS * K;
    int64_t stages = (n_nodes + p.Tn - 1) / p.Tn;
    if (stages < 1) stages = 1;
    if (max_stages > 0 && stages > max_stages) stages = max_stages;
    p.stages = (int)stages;
    return p;
}

static bool stream_form_ok(const acsfit_ctx *ctx, int D, int nw, int Tn)
{
    return ctx->use_stream && nw > 0 && D <= 8 && Tn >= 32 && Tn % 32 == 0;
}

// one acsfit_last_launches record, written by the two functions that launch a pipeline kernel, from the
// instantiation they launch and the parameters it receives
static void record_launch(acsfit_ctx *ctx, bool bins, int D, int rw, bool prune, bool streaming,
                          const PipelineParams &q, int stages, int resident)
{
    ctx->launch_log.push_back({bins ? 1 : 0, ctx->rec_chained, D, rw, prune ? 1 : 0, streaming ? 1 : 0, q.Tn, stages,
                               resident, bins ? ctx->rec_pool : -1,
                               bins ? (int)std::min<int64_t>(q.bin_base, INT32_MAX) : -1, streaming ? 0 : q.publish_every});
}

template <int D, bool BINS, int RW>
static acsfit_status launch_stream(acsfit_ctx *ctx, const PipelineParams &pp, int stages, cudaStream_t st, int *resident)
{
    const size_t smem = StreamSmem<D, BINS, RW>::bytes(pp.Tn);
    auto kern = firstfit_stream_kernel<D, BINS, RW>;
    if (resident) {
        const auto key = std::make_tuple(D, (int)BINS, 2 /*streaming form*/, RW, pp.Tn);
        auto it = ctx->resident_cache.find(key);
        if (it == ctx->resident_cache.end()) {
            int per_sm = 0;
            CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, 256, smem));
            it = ctx->resident_cache.emplace(key, per_sm * ctx->num_sms).first;
        }
        *resident = it->second;
        return ACSFIT_OK;
    }
    int held = 0;
    TRY((launch_stream<D, BINS, RW>(ctx, pp, stages, st, &held)));
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<stages, 256, smem, st>>>(pp);
    ++ctx->launches;
    CUDA_TRY(cudaGetLastError());
    record_launch(ctx, BINS, D, RW, false, true, pp, stages, held);
    return ACSFIT_OK;
}

constexpr int kOneCtaSmemKb = 116;  // more than half of the 227 KB an SM offers: a second CTA cannot be resident
// SEL: the node-selector form of a node pass, AA: the anti-affinity form of a node or bin pass (barrier form only:
// both ignore the "stream" knob)
template <int D, bool BINS, bool PRUNE, int RW, bool SEL = false, bool AA = false, bool PA = false, bool TS = false>
static acsfit_status launch_pipeline_w(acsfit_ctx *ctx, const PipelineParams &pp, int stages, cudaStream_t st, int *resident)
{
    if constexpr (RW > 0 && D <= 8 && !PRUNE && !SEL && !AA) {
        if (stream_form_ok(ctx, D, RW, pp.Tn)) return launch_stream<D, BINS, RW>(ctx, pp, stages, st, resident);
    }
    constexpr int NT = stage_threads(D, BINS);
    size_t smem = PipelineSmem<D, BINS, NT, PRUNE, RW, SEL, AA, PA, TS>::bytes(pp.Tn, TS ? pp.ts_keys : 0);
    // D >= 8: ONE stage CTA per SM.  Whether two fit is an accident of the register allocation (the bins kernel has
    // been compiled to 128 and to 237 registers by neighbouring source revisions); at c3 a second CTA on the
    // frontier's SM costs the placement chain more than the extra resident stages give back.
    if (D >= 8) smem = std::max(smem, (size_t)kOneCtaSmemKb * 1024);
    if (ctx->smem_floor_kb > 0) smem = std::max(smem, (size_t)ctx->smem_floor_kb * 1024);  // occupancy knob
    auto kern = firstfit_pipeline_kernel<D, BINS, NT, PRUNE, RW, SEL, AA, PA, TS>;
    if (resident) {  // only asked: how many stages does the GPU hold at once?  (cached: the query costs ~10 us)
        const auto key = std::make_tuple(D, (int)BINS, (int)PRUNE | (SEL ? 4 : 0) | (AA ? 8 : 0) | (PA ? 16 : 0) | (TS ? 32 + (pp.ts_keys << 6) : 0), RW, pp.Tn);
        auto it = ctx->resident_cache.find(key);
        if (it == ctx->resident_cache.end()) {
            int per_sm = 0;
            CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, NT, smem));
            it = ctx->resident_cache.emplace(key, per_sm * ctx->num_sms).first;
        }
        *resident = it->second;
        return ACSFIT_OK;
    }
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    PipelineParams q = pp;
    // more stages than the GPU holds at once: several waves, each streaming the whole pod list (see the kernel's publish)
    int held = 0;
    TRY((launch_pipeline_w<D, BINS, PRUNE, RW, SEL, AA, PA, TS>(ctx, pp, stages, st, &held)));
    q.publish_every = (held > 0 && stages > held) ? kPublishEvery : 1;
    q.retire = BINS && ctx->retire;
    if (BINS && RW > 0) {  // the first counted bin pass of a call zeroes the counters (in stream order before the later ones)
        if (!ctx->retire_counted) CUDA_TRY(cudaMemsetAsync(ctx->retire_dev, 0, 2 * sizeof(unsigned long long), st));
        ctx->retire_counted = true;
        q.retire_count = ctx->retire_dev;
    }
    q.prof = (ctx->prof_dev && stages <= kProfStages) ? ctx->prof_dev : nullptr;
    if (q.prof) {
        CUDA_TRY(cudaMemsetAsync(ctx->prof_dev, 0, sizeof(unsigned long long) * (kProfStages + kProfTiles) * 8, st));
        ctx->prof_stages = stages;
        q.trace = (ctx->trace_stage >= 0 && pp.num_tiles <= kProfTiles) ? ctx->prof_dev + (size_t)kProfStages * 8 : nullptr;
        q.trace_stage = ctx->trace_stage;
    }
    kern<<<stages, NT, smem, st>>>(q);
    ++ctx->launches;
    CUDA_TRY(cudaGetLastError());
    record_launch(ctx, BINS, D, RW, PRUNE, false, q, stages, held);
    return ACSFIT_OK;
}

// the instantiation is chosen by the rank layout of the call: 0 (float64 scan), 1, 2 or 4 packed words per row
template <int D, bool BINS, bool PRUNE, bool SEL = false, bool AA = false, bool PA = false, bool TS = false>
static acsfit_status launch_pipeline_v(acsfit_ctx *ctx, const PipelineParams &pp, int stages, cudaStream_t st, int *resident)
{
    switch (pp.rk.nw) {
    case 0: return launch_pipeline_w<D, BINS, PRUNE, 0, SEL, AA, PA, TS>(ctx, pp, stages, st, resident);
    case 1: return launch_pipeline_w<D, BINS, PRUNE, 1, SEL, AA, PA, TS>(ctx, pp, stages, st, resident);
    case 2: return launch_pipeline_w<D, BINS, PRUNE, 2, SEL, AA, PA, TS>(ctx, pp, stages, st, resident);
    case 4: return launch_pipeline_w<D, BINS, PRUNE, 4, SEL, AA, PA, TS>(ctx, pp, stages, st, resident);
    default: return fail(ctx, ACSFIT_E_INVALID, "rank layout with %d words", pp.rk.nw);
    }
}

// node pass with node selectors (pp.node_match != nullptr), AA: and anti-affinity masks, PA: and pod-affinity masks:
// the same pruning rule as below, barrier form only
template <int D, bool AA = false, bool PA = false, bool TS = false>
static acsfit_status launch_pipeline_sel(acsfit_ctx *ctx, const PipelineParams &pp, int stages, cudaStream_t st)
{
    int prune = ctx->prune;
    if (prune < 0) {
        int resident = 0;
        TRY((launch_pipeline_v<D, false, false, true, AA, PA, TS>(ctx, pp, stages, st, &resident)));
        prune = stages > resident;
    }
    if (prune) return launch_pipeline_v<D, false, true, true, AA, PA, TS>(ctx, pp, stages, st, nullptr);
    return launch_pipeline_v<D, false, false, true, AA, PA, TS>(ctx, pp, stages, st, nullptr);
}

template <int D, bool BINS>
static acsfit_status launch_pipeline_t(acsfit_ctx *ctx, const PipelineParams &pp, int stages, cudaStream_t st)
{
    if constexpr (BINS) {
        if (pp.ts_key) return launch_pipeline_v<D, true, false, false, true, true, true>(ctx, pp, stages, st, nullptr);
        if (pp.pod_need) return launch_pipeline_v<D, true, false, false, true, true>(ctx, pp, stages, st, nullptr);
        if (pp.pod_carries) return launch_pipeline_v<D, true, false, false, true>(ctx, pp, stages, st, nullptr);
    } else {
        if (pp.ts_key) return launch_pipeline_sel<D, true, true, true>(ctx, pp, stages, st);  // the entry point set node_match
        if (pp.pod_need) return launch_pipeline_sel<D, true, true>(ctx, pp, stages, st);  // the entry point set node_match
        if (pp.pod_carries) return launch_pipeline_sel<D, true>(ctx, pp, stages, st);  // the entry point set node_match
        if (pp.node_match) return launch_pipeline_sel<D>(ctx, pp, stages, st);
        // Stage bounds + scan-list pruning (the PRUNE instantiation) pay when the pass is throughput-bound, i.e.
        // when there are more stages than the GPU holds at once (waves); a pass that fits is bound by its
        // placement chain and runs the plain instantiation.  ACSFIT_PRUNE=0/1 forces either.
        int prune = ctx->prune;
        if (prune != 1 && stream_form_ok(ctx, D, pp.rk.nw, pp.Tn)) prune = 0;  // the streaming form has no pruning variant
        if (prune < 0) {
            int resident = 0;
            TRY((launch_pipeline_v<D, BINS, false>(ctx, pp, stages, st, &resident)));
            prune = stages > resident;
        }
        if (prune) return launch_pipeline_v<D, false, true>(ctx, pp, stages, st, nullptr);
    }
    return launch_pipeline_v<D, BINS, false>(ctx, pp, stages, st, nullptr);
}

template <bool BINS>
static acsfit_status launch_pipeline(acsfit_ctx *ctx, int D, const PipelineParams &pp, int stages, cudaStream_t st)
{
    switch (D) {
    case 2: return launch_pipeline_t<2, BINS>(ctx, pp, stages, st);
    case 4: return launch_pipeline_t<4, BINS>(ctx, pp, stages, st);
    case 8: return launch_pipeline_t<8, BINS>(ctx, pp, stages, st);
    case 16: return launch_pipeline_t<16, BINS>(ctx, pp, stages, st);
    default: return fail(ctx, ACSFIT_E_INVALID, "D=%d: the first-fit entry points need D in {2,4,8,16}", D);
    }
}

static acsfit_status check_pipeline_status(acsfit_ctx *ctx, const int *status_dev, cudaStream_t st)
{
    int status = 0;
    CUDA_TRY(cudaMemcpyAsync(&status, status_dev, sizeof(int), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    if (status) return fail(ctx, ACSFIT_E_TIMEOUT, "first-fit pipeline watchdog fired after %d ms", ctx->watchdog_ms);
    return ACSFIT_OK;
}


// ---------------------------------------------------------------------------------------------
// cluster mode: one cluster on the GPUs of one box (include/acsfit.h).  Exchange region of a rank:
//   [0, 1024)   header: arrive[ACSFIT_MAX_RANKS] ints (barrier flags, slot r written by rank r), status int at
//               +64, 16 uint64 scalars at +128
//   x_sync      kClusterBlocks sync sets of kClusterSyncInts ints (ticket, status, drained, ..., progress[stages])
//   x_alive     "still unplaced" bitmap of the running pass (read by the next rank's stage 0)
//   x_placed    this rank's placements of the running pass (merged element-wise by every rank)
//   x_used      this rank's node rows after the node pass (gathered by every rank)
// ---------------------------------------------------------------------------------------------
constexpr int kClusterBlocks = 64;
constexpr int kClusterSyncInts = 8 + 4096;
constexpr size_t kClusterHdr = 1024;

namespace {
struct PeerInts { int *p[ACSFIT_MAX_RANKS]; };
struct PeerI32 { const int32_t *p[ACSFIT_MAX_RANKS]; };
struct PeerF64 { const double *p[ACSFIT_MAX_RANKS]; };
struct PeerU64 { const unsigned long long *p[ACSFIT_MAX_RANKS]; };
struct RangeTable { int64_t lo[ACSFIT_MAX_RANKS + 1]; };

// every rank tells every rank "I am at barrier `epoch`", then waits until all have said so.  The flags are
// written and polled with system scope (they live in peer memory); kernels that ran before this one on the
// stream have completed, so their global writes are visible to whoever passes the barrier.
__global__ void cluster_barrier_kernel(PeerInts arrive, int rank, int world, int epoch, int *status,
                                       unsigned long long timeout_ns)
{
    const int r = threadIdx.x;
    if (r >= world) return;
    __threadfence_system();
    st_release_sys(arrive.p[r] + rank, epoch);
    const unsigned long long t0 = global_timer_ns();
    unsigned spins = 0;
    while (ld_acquire_sys(arrive.p[rank] + r) < epoch) {
        if ((++spins & 255u) == 0 && global_timer_ns() - t0 > timeout_ns) {
            atomicExch(status, 3);
            break;
        }
        __nanosleep(100);
    }
}

// element-wise maximum over the ranks' vectors (each pod is placed by at most one rank, the others hold -1)
__global__ void merge_max_i32_kernel(PeerI32 src, int world, int64_t n, int32_t *out)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        int32_t m = __ldcg(src.p[0] + i);
        for (int r = 1; r < world; ++r) m = max(m, __ldcg(src.p[r] + i));
        out[i] = m;
    }
}

// used[n] of every node from the rank that owns it (rows are stored at their GLOBAL position in x_used)
__global__ void gather_rows_kernel(PeerF64 src, RangeTable rt, int world, int rank, int64_t N, int D, double *used)
{
    const int64_t total = N * D;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t n = i / D;
        int r = 0;
        while (r + 1 < world && n >= rt.lo[r + 1]) ++r;
        if (r != rank) used[i] = __ldcg(src.p[r] + i);
    }
}

// out[k] = sum over ranks of scalars_r[k] (k < 8), out[8 + k] = max over ranks of scalars_r[k]; out[16] = max status
__global__ void cluster_scalars_kernel(PeerU64 scal, PeerInts status, int world, unsigned long long *out)
{
    const int k = threadIdx.x;
    if (k < 8) {
        unsigned long long sum = 0, mx = 0;
        for (int r = 0; r < world; ++r) {
            const unsigned long long v = __ldcg(scal.p[r] + k);
            sum += v;
            mx = v > mx ? v : mx;
        }
        out[k] = sum;
        out[8 + k] = mx;
    }
    if (k == 8) {
        int m = 0;
        for (int r = 0; r < world; ++r) m = max(m, __ldcg(status.p[r]));
        out[16] = (unsigned long long)m;
    }
}
}  // namespace

static int *x_arrive(const acsfit_ctx *ctx, int r) { return reinterpret_cast<int *>(ctx->peer[r]); }
static int *x_status(const acsfit_ctx *ctx, int r) { return reinterpret_cast<int *>(ctx->peer[r] + 64); }
static unsigned long long *x_scalars(const acsfit_ctx *ctx, int r) { return reinterpret_cast<unsigned long long *>(ctx->peer[r] + 128); }
static int *x_syncset(const acsfit_ctx *ctx, int r, int b) { return reinterpret_cast<int *>(ctx->peer[r] + ctx->x_sync) + (size_t)b * kClusterSyncInts; }
static uint32_t *x_alive_of(const acsfit_ctx *ctx, int r) { return reinterpret_cast<uint32_t *>(ctx->peer[r] + ctx->x_alive); }
static int32_t *x_placed_of(const acsfit_ctx *ctx, int r) { return reinterpret_cast<int32_t *>(ctx->peer[r] + ctx->x_placed); }
static double *x_used_of(const acsfit_ctx *ctx, int r) { return reinterpret_cast<double *>(ctx->peer[r] + ctx->x_used); }

static acsfit_status cluster_barrier(acsfit_ctx *ctx, cudaStream_t st)
{
    PeerInts a;
    for (int r = 0; r < ACSFIT_MAX_RANKS; ++r) a.p[r] = r < ctx->world ? x_arrive(ctx, r) : nullptr;
    ++ctx->epoch;
    cluster_barrier_kernel<<<1, 32, 0, st>>>(a, ctx->rank, ctx->world, ctx->epoch, x_status(ctx, ctx->rank),
                                             (unsigned long long)ctx->watchdog_ms * 1000000ull);
    ++ctx->launches;
    CUDA_TRY(cudaGetLastError());
    return ACSFIT_OK;
}

// out[i] = max over the ranks of their x_placed[i]; bracketed by the two barriers that make the vectors final
// before they are read and keep them untouched until every rank has read them
static acsfit_status cluster_merge_placed(acsfit_ctx *ctx, int64_t n, int32_t *out, cudaStream_t st)
{
    TRY(cluster_barrier(ctx, st));
    PeerI32 src;
    for (int r = 0; r < ACSFIT_MAX_RANKS; ++r) src.p[r] = r < ctx->world ? x_placed_of(ctx, r) : nullptr;
    if (n > 0) {
        merge_max_i32_kernel<<<grid_for(ctx, n, 256), 256, 0, st>>>(src, ctx->world, n, out);
        ++ctx->launches;
    }
    TRY(cluster_barrier(ctx, st));
    CUDA_TRY(cudaGetLastError());
    return ACSFIT_OK;
}

// sums one device-side uint64 over the ranks (e.g. the credited bin tests each rank counted) and returns the
// highest pipeline status any rank recorded; synchronises the stream
static acsfit_status cluster_sum_u64(acsfit_ctx *ctx, const unsigned long long *value_dev, unsigned long long *scratch17_dev,
                                     unsigned long long *out_sum, cudaStream_t st)
{
    if (value_dev)
        CUDA_TRY(cudaMemcpyAsync(x_scalars(ctx, ctx->rank), value_dev, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
    else
        CUDA_TRY(cudaMemsetAsync(x_scalars(ctx, ctx->rank), 0, sizeof(unsigned long long), st));
    TRY(cluster_barrier(ctx, st));
    PeerU64 sc;
    PeerInts stw;
    for (int r = 0; r < ACSFIT_MAX_RANKS; ++r) {
        sc.p[r] = r < ctx->world ? x_scalars(ctx, r) : nullptr;
        stw.p[r] = r < ctx->world ? x_status(ctx, r) : nullptr;
    }
    cluster_scalars_kernel<<<1, 32, 0, st>>>(sc, stw, ctx->world, scratch17_dev);
    ++ctx->launches;
    TRY(cluster_barrier(ctx, st));
    unsigned long long h[17];
    CUDA_TRY(cudaMemcpyAsync(h, scratch17_dev, sizeof h, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    if (out_sum) *out_sum = h[0];
    if (h[16] == 3) return fail(ctx, ACSFIT_E_PEER, "cluster barrier timed out: a peer rank did not arrive");
    if (h[16] != 0) return fail(ctx, ACSFIT_E_TIMEOUT, "first-fit pipeline watchdog fired on some rank");
    return ACSFIT_OK;
}

// first node of rank r's range
static int64_t cluster_lo(int64_t N, int world, int r) { return N * r / world; }

extern "C" acsfit_status acsfit_cluster_init(acsfit_ctx *ctx, int rank, int world, int64_t max_pods, int64_t max_nodes,
                                             int max_dims, void *out_handle)
{
    if (!ctx || !out_handle || world < 1 || world > ACSFIT_MAX_RANKS || rank < 0 || rank >= world || max_pods < 0 ||
        max_nodes < 0 || max_dims < 1 || max_dims > ACSFIT_MAX_DIMS)
        return fail(ctx, ACSFIT_E_INVALID, "cluster_init: bad arguments");
    CUDA_TRY(cudaSetDevice(ctx->device));
    if (ctx->xbase) return fail(ctx, ACSFIT_E_INVALID, "cluster_init: already initialised");
    ctx->x_sync = kClusterHdr;
    ctx->x_alive = align_up(ctx->x_sync + sizeof(int) * (size_t)kClusterBlocks * kClusterSyncInts, 256);
    ctx->x_placed = align_up(ctx->x_alive + sizeof(uint32_t) * (size_t)((max_pods + 31) / 32 + 8), 256);
    ctx->x_used = align_up(ctx->x_placed + sizeof(int32_t) * (size_t)(max_pods + 8), 256);
    ctx->x_bytes = align_up(ctx->x_used + sizeof(double) * (size_t)(max_nodes + 1) * max_dims, 1 << 20);
    CUDA_TRY(cudaMalloc(&ctx->xbase, ctx->x_bytes));
    CUDA_TRY(cudaMemset(ctx->xbase, 0, ctx->x_bytes));
    CUDA_TRY(cudaDeviceSynchronize());
    cudaIpcMemHandle_t h;
    static_assert(sizeof(cudaIpcMemHandle_t) == ACSFIT_IPC_HANDLE_BYTES, "IPC handle size");
    CUDA_TRY(cudaIpcGetMemHandle(&h, ctx->xbase));
    memcpy(out_handle, &h, sizeof h);
    ctx->rank = rank;
    ctx->world = 1;  // becomes `world` in cluster_connect
    ctx->x_max_pods = max_pods;
    ctx->x_max_nodes = max_nodes;
    ctx->x_max_dims = max_dims;
    ctx->epoch = 0;
    ctx->peer[rank] = ctx->xbase;
    ctx->cl_tn = -world;  // remembered until connect
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_cluster_connect(acsfit_ctx *ctx, const void *all_handles)
{
    if (!ctx || !all_handles || !ctx->xbase || ctx->cl_tn >= 0) return fail(ctx, ACSFIT_E_INVALID, "cluster_connect: call cluster_init first");
    CUDA_TRY(cudaSetDevice(ctx->device));
    const int world = -ctx->cl_tn;
    const unsigned char *hs = static_cast<const unsigned char *>(all_handles);
    for (int r = 0; r < world; ++r) {
        if (r == ctx->rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, hs + (size_t)r * ACSFIT_IPC_HANDLE_BYTES, sizeof h);
        void *ptr = nullptr;
        CUDA_TRY(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
        ctx->peer[r] = static_cast<unsigned char *>(ptr);
    }
    ctx->world = world;
    ctx->cl_tn = 0;
    if (ctx->watchdog_ms < 60000) ctx->watchdog_ms = 60000;  // a rank legitimately waits for all the ranks before it
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_cluster_barrier(acsfit_ctx *ctx, acsfit_stream_t stream)
{
    if (!ctx || ctx->world < 2) return fail(ctx, ACSFIT_E_INVALID, "cluster_barrier: not in cluster mode");
    CUDA_TRY(cudaSetDevice(ctx->device));
    TRY(cluster_barrier(ctx, (cudaStream_t)stream));
    CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
    int status = 0;
    CUDA_TRY(cudaMemcpy(&status, x_status(ctx, ctx->rank), sizeof status, cudaMemcpyDeviceToHost));
    if (status) return fail(ctx, ACSFIT_E_PEER, "cluster barrier timed out");
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_cluster_last_plan(const acsfit_ctx *ctx, int *out_tn, int *out_stages, int *out_blocks,
                                                  int *out_resident)
{
    if (!ctx) return ACSFIT_E_INVALID;
    if (out_tn) *out_tn = ctx->cl_tn;
    if (out_stages) *out_stages = ctx->cl_stages;
    if (out_blocks) *out_blocks = ctx->cl_blocks;
    if (out_resident) *out_resident = ctx->cl_resident;
    return ACSFIT_OK;
}

// stage CTAs of one pipeline instantiation the GPU holds at once (D, mode and rank layout of the current call)
static int resident_stages(acsfit_ctx *ctx, int D, bool bins, int Tn)
{
    PipelineParams q;
    memset(&q, 0, sizeof q);
    q.Tn = Tn;
    q.rk = ctx->rk;
    int resident = 0;
    acsfit_status s = ACSFIT_E_INVALID;
    switch (D) {
    case 2: s = bins ? launch_pipeline_v<2, true, false>(ctx, q, 0, nullptr, &resident) : launch_pipeline_v<2, false, false>(ctx, q, 0, nullptr, &resident); break;
    case 4: s = bins ? launch_pipeline_v<4, true, false>(ctx, q, 0, nullptr, &resident) : launch_pipeline_v<4, false, false>(ctx, q, 0, nullptr, &resident); break;
    case 8: s = bins ? launch_pipeline_v<8, true, false>(ctx, q, 0, nullptr, &resident) : launch_pipeline_v<8, false, false>(ctx, q, 0, nullptr, &resident); break;
    case 16: s = bins ? launch_pipeline_v<16, true, false>(ctx, q, 0, nullptr, &resident) : launch_pipeline_v<16, false, false>(ctx, q, 0, nullptr, &resident); break;
    default: break;
    }
    return s == ACSFIT_OK ? resident : 0;
}

// Cluster.get_pending_pods for one cluster on all ranks (include/acsfit.h, "Cluster mode").  Inputs are
// replicated; rank r fits the pods that reach it onto nodes [lo_r, lo_{r+1}).  When a rank's stages fit the GPU
// at once the whole pod list is one launch per rank and the ranks overlap tile by tile; otherwise (waves) the
// list is cut into pod blocks, one launch per block and rank, and the ranks overlap block by block.
// On return placed_out[F] and used[N, D] are complete and identical on every rank.
static acsfit_status cluster_first_fit(acsfit_ctx *ctx, const double *req, const int32_t *list_f, int64_t F, int D,
                                       const double *cap_type, const int32_t *node_type, double *used, int64_t N,
                                       int32_t *placed_out, unsigned long long *decisions_dev, cudaStream_t st)
{
    const int W = ctx->world, rank = ctx->rank;
    if (decisions_dev) CUDA_TRY(cudaMemsetAsync(decisions_dev, 0, sizeof(unsigned long long), st));
    if (F == 0) return ACSFIT_OK;
    if (F > ctx->x_max_pods || N > ctx->x_max_nodes || D > ctx->x_max_dims)
        return fail(ctx, ACSFIT_E_INVALID, "cluster mode: %lld pods / %lld nodes / %d dims exceed the exchange region "
                    "(cluster_init: %lld / %lld / %d)", (long long)F, (long long)N, D, (long long)ctx->x_max_pods,
                    (long long)ctx->x_max_nodes, ctx->x_max_dims);
    fill_i32_kernel<<<grid_for(ctx, F, 256), 256, 0, st>>>(placed_out, F, -1);
    ++ctx->launches;
    if (N == 0) {
        CUDA_TRY(cudaGetLastError());
        return ACSFIT_OK;
    }
    // geometry, identical on every rank: the narrowest stage (>= 32 nodes) whose stage count still fits the GPU
    // at once for the largest node range; the full width and pod blocks when even that runs in waves
    int64_t n_max = 0;
    for (int r = 0; r < W; ++r) n_max = std::max(n_max, cluster_lo(N, W, r + 1) - cluster_lo(N, W, r));
    const int K = nodes_per_thread(D, ctx->rk.nw);
    const int tn_max = max_stage_nodes(D, false);
    int Tn = tn_max, resident = resident_stages(ctx, D, false, tn_max);
    for (int t = std::max(32, K); t <= tn_max; t <<= 1) {
        const int res = resident_stages(ctx, D, false, t);
        if (res > 0 && (n_max + t - 1) / t <= res) {
            Tn = t;
            resident = res;
            break;
        }
    }
    if (resident <= 0) return fail(ctx, ACSFIT_E_CUDA, "cluster mode: occupancy query failed");
    const int64_t stages_max = (n_max + Tn - 1) / Tn;
    if (stages_max + 8 > kClusterSyncInts) return fail(ctx, ACSFIT_E_INVALID, "cluster mode: %lld stages per rank", (long long)stages_max);
    const int tiles = (int)((F + kTile - 1) / kTile);
    int blocks = 1, tpb = tiles;
    if (stages_max > resident || ctx->force_blocks > 0) {
        blocks = std::min(kClusterBlocks, std::max(1, std::min(tiles, ctx->force_blocks > 0 ? ctx->force_blocks : 4 * W)));
        tpb = (tiles + blocks - 1) / blocks;
        blocks = (tiles + tpb - 1) / tpb;
    }
    const int64_t lo = cluster_lo(N, W, rank), hi = cluster_lo(N, W, rank + 1);
    const int my_stages = (int)std::max<int64_t>(1, (hi - lo + Tn - 1) / Tn);
    int up_stages = 0;
    if (rank > 0) up_stages = (int)std::max<int64_t>(1, (lo - cluster_lo(N, W, rank - 1) + Tn - 1) / Tn);
    ctx->cl_tn = Tn;
    ctx->cl_stages = my_stages;
    ctx->cl_blocks = blocks;
    ctx->cl_resident = resident;

    uint32_t *alive = x_alive_of(ctx, rank);
    int32_t *placed_x = x_placed_of(ctx, rank);
    CUDA_TRY(cudaMemsetAsync(x_status(ctx, rank), 0, sizeof(int), st));  // (peers read it only between barriers)
    CUDA_TRY(cudaMemsetAsync(x_syncset(ctx, rank, 0), 0, sizeof(int) * (size_t)blocks * kClusterSyncInts, st));
    fill_i32_kernel<<<grid_for(ctx, F, 256), 256, 0, st>>>(placed_x, F, -1);
    if (rank == 0) fill_alive_kernel<<<grid_for(ctx, (F + 31) / 32, 256), 256, 0, st>>>(alive, F);
    ctx->launches += 2;
    TRY(cluster_barrier(ctx, st));  // every rank's counters are zero before anybody polls them

    if (ctx->timing) CUDA_TRY(cudaEventRecord(ctx->ev0, st));
    for (int b = 0; b < blocks; ++b) {
        PipelineParams pp;
        memset(&pp, 0, sizeof pp);
        int *sync = x_syncset(ctx, rank, b);
        pp.req = req;
        pp.pod_idx = list_f;
        pp.M = F;
        pp.alive = alive;
        pp.placed = placed_x;
        pp.cap_type = cap_type;
        pp.node_type = node_type;
        pp.used = used;
        pp.node_lo = lo;
        pp.node_hi = hi;
        pp.Tn = Tn;
        pp.NS = Tn / K;
        pp.tile_lo = b * tpb;
        pp.num_tiles = std::min(tpb, tiles - b * tpb);
        pp.ticket = sync;
        pp.status = x_status(ctx, rank);  // one abort word per rank
        pp.drained = sync + 2;
        pp.progress = sync + 8;
        pp.sys_scope = 1;
        if (rank > 0) {
            pp.upstream = x_syncset(ctx, rank - 1, b) + 8 + (up_stages - 1);
            pp.alive_in = x_alive_of(ctx, rank - 1);
        }
        pp.watchdog_ns = (unsigned long long)ctx->watchdog_ms * 1000000ull;
        pp.rk = ctx->rk;
        TRY(launch_pipeline<false>(ctx, D, pp, my_stages, st));
    }
    if (ctx->timing) CUDA_TRY(cudaEventRecord(ctx->ev1, st));
    // this rank's node rows, at their global position, for the other ranks to fetch
    if (hi > lo)
        CUDA_TRY(cudaMemcpyAsync(x_used_of(ctx, rank) + (size_t)lo * D, used + (size_t)lo * D,
                                 sizeof(double) * (size_t)(hi - lo) * D, cudaMemcpyDeviceToDevice, st));
    TRY(cluster_barrier(ctx, st));
    {
        PeerI32 src;
        PeerF64 us;
        RangeTable rt;
        for (int r = 0; r < ACSFIT_MAX_RANKS; ++r) {
            src.p[r] = r < W ? x_placed_of(ctx, r) : nullptr;
            us.p[r] = r < W ? x_used_of(ctx, r) : nullptr;
        }
        for (int r = 0; r <= ACSFIT_MAX_RANKS; ++r) rt.lo[r] = cluster_lo(N, W, std::min(r, W));
        merge_max_i32_kernel<<<grid_for(ctx, F, 256), 256, 0, st>>>(src, W, F, placed_out);
        gather_rows_kernel<<<grid_for(ctx, N * D, 256), 256, 0, st>>>(us, rt, W, rank, N, D, used);
        ctx->launches += 2;
    }
    TRY(cluster_barrier(ctx, st));
    if (decisions_dev) {
        decisions_kernel<<<grid_for(ctx, F, 256), 256, 0, st>>>(placed_out, F, N, decisions_dev);
        ++ctx->launches;
    }
    TAKE(sc17, unsigned long long, 17);
    TRY(cluster_sum_u64(ctx, nullptr, sc17, nullptr, st));  // status of all ranks (synchronises)
    ctx->last_stages += my_stages * blocks;
    ctx->last_tiles += tiles;
    if (ctx->timing) {
        float ms = 0.f;
        CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
        ctx->last_ms += ms;
        if (g_trace) fprintf(stderr, "[acsfit r%d] cluster nodes pass: %lld pods, %d stages x %d nodes, %d block(s): %.3f ms\n",
                             ctx->rank, (long long)F, my_stages, Tn, blocks, ms);
        if (decisions_dev) {
            unsigned long long d = 0;
            CUDA_TRY(cudaMemcpy(&d, decisions_dev, sizeof d, cudaMemcpyDeviceToHost));
            ctx->last_decisions += d;
        }
    }
    return ACSFIT_OK;
}

static void reset_stats(acsfit_ctx *ctx)
{
    ctx->last_ms = 0.0;
    ctx->last_decisions = 0;
    ctx->last_stages = ctx->last_tiles = 0;
    ctx->last_sel_hits = 0;
    ctx->retire_counted = false;
    ctx->pa_flips.clear();
    ctx->ts_rises.clear();
}

// ---------------------------------------------------------------------------------------------
// first fit over nodes (implementation; scratch must already be reserved)
// ---------------------------------------------------------------------------------------------
static size_t first_fit_scratch(const acsfit_ctx *ctx, int64_t P, int64_t N)
{
    // stages: whatever plan_stages picks for any D / rank layout stays below this bound
    const size_t stages = (size_t)std::max<int64_t>(4 * std::max(ctx->min_stages, ctx->num_sms), N / 16 + 2);
    return 8192 + sizeof(uint32_t) * (size_t)((P + 31) / 32) + sizeof(int) * (stages + 8);
}

// pod_class / node_match (device, both or neither): node selectors (the SEL form of the node pass; single GPU only)
// pod affinity, before a pass: the needs of positions [0, n) under the flips and, when a signature is watched, the
// first-placement slots reset to "not placed" (all ones)
static acsfit_status pa_prepare(acsfit_ctx *ctx, const acsfit_pod_affinity *pa, const int32_t *idx, int64_t n,
                                const PaFlips &fl, uint64_t watch, unsigned long long *need,
                                unsigned long long *first_placed, cudaStream_t st)
{
    if (n > 0) {
        pa_need_kernel<<<grid_for(ctx, n, 256), 256, 0, st>>>(reinterpret_cast<const unsigned long long *>(pa->pod_requires),
                                                             reinterpret_cast<const unsigned long long *>(pa->pod_self),
                                                             idx, n, fl, need);
        ++ctx->launches;
        CUDA_TRY(cudaGetLastError());
    }
    if (watch) CUDA_TRY(cudaMemsetAsync(first_placed, 0xFF, sizeof(unsigned long long) * 64, st));
    return ACSFIT_OK;
}

// pod affinity, after a pass that watched the still unfixed signatures of `watch`: fixes the flip of the one placed
// earliest (the lowest signature on a tie) and sets `again`; leaves `again` false when none was placed
static acsfit_status pa_next_flip(acsfit_ctx *ctx, const unsigned long long *first_placed, uint64_t watch,
                                  uint64_t &fixed, PaFlips &fl, bool &again, cudaStream_t st)
{
    again = false;
    const uint64_t open = watch & ~fixed;
    if (!open) return ACSFIT_OK;
    unsigned long long fp[64];
    CUDA_TRY(cudaMemcpyAsync(fp, first_placed, sizeof fp, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    int best = -1;
    for (int s = 0; s < 64; ++s)
        if (((open >> s) & 1u) && fp[s] != ~0ull && (best < 0 || fp[s] < fp[best])) best = s;
    if (best < 0) return ACSFIT_OK;
    fl.f[best] = (long long)fp[best];
    fixed |= 1ull << best;
    ctx->pa_flips.push_back(best);
    ctx->pa_flips.push_back((int64_t)fp[best]);
    again = true;
    return ACSFIT_OK;
}

// OR of v[idx ? idx[i] : i] over i < n (gate: only where gate[i] >= 0), to the host
static acsfit_status or_rows(acsfit_ctx *ctx, const uint64_t *v, const int32_t *idx, int64_t n, const int32_t *gate,
                             unsigned long long *scratch, uint64_t *out, cudaStream_t st)
{
    *out = 0;
    if (n <= 0) return ACSFIT_OK;
    CUDA_TRY(cudaMemsetAsync(scratch, 0, sizeof(unsigned long long), st));
    or_rows_kernel<<<grid_for(ctx, n, 256), 256, 0, st>>>(reinterpret_cast<const unsigned long long *>(v), idx, n, gate,
                                                         scratch);
    ++ctx->launches;
    CUDA_TRY(cudaMemcpyAsync(out, scratch, sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    return ACSFIT_OK;
}

// topology spread: one pass's levels, targets and device scratch (include/acsfit.h, acsfit_topology_spread)
constexpr int kMaxSpreadRises = 4096;  // rises one node pass may fix (each costs a rerun of the pass)
struct TsPass {
    const acsfit_topology_spread *ts = nullptr;
    int32_t *lim = nullptr;                     // [positions]
    int *target = nullptr, *reached = nullptr;  // [64] each
    unsigned long long *rise_pos = nullptr;     // [64]
    int *dmin = nullptr, *dndom = nullptr;      // [64] each
    long long *rises_dev = nullptr;             // [kMaxSpreadRises]: the fixed rises' positions, per key ascending
    int base[64], ndom[64], tgt[64], nfixed[64];
    std::vector<long long> rises;               // fixed (key, position) pairs
    bool watching = false;                      // some key's next rise is watched in the current pass
};

static size_t ts_scratch(int64_t positions)
{
    return sizeof(int32_t) * (size_t)positions + sizeof(int) * 64 * 4 + sizeof(unsigned long long) * 64 +
           sizeof(long long) * kMaxSpreadRises + 2048;
}

static acsfit_status ts_alloc(acsfit_ctx *ctx, const acsfit_topology_spread *ts, int64_t positions, TsPass &tp)
{
    tp.ts = ts;
    tp.lim = arena_take<int32_t>(ctx, (size_t)std::max<int64_t>(1, positions));
    tp.target = arena_take<int>(ctx, 64);
    tp.reached = arena_take<int>(ctx, 64);
    tp.dmin = arena_take<int>(ctx, 64);
    tp.dndom = arena_take<int>(ctx, 64);
    tp.rise_pos = arena_take<unsigned long long>(ctx, 64);
    tp.rises_dev = arena_take<long long>(ctx, kMaxSpreadRises);
    if (!tp.lim || !tp.target || !tp.reached || !tp.dmin || !tp.dndom || !tp.rise_pos || !tp.rises_dev)
        return fail(ctx, ACSFIT_E_NOMEM, "scratch arena too small for topology spread");
    for (int k = 0; k < 64; ++k) {
        tp.base[k] = 0;
        tp.ndom[k] = 0;
        tp.tgt[k] = INT_MAX;
        tp.nfixed[k] = 0;
    }
    return ACSFIT_OK;
}

// node pass: each key's minimum at the start, min(floor, the smallest count of its domains in the list), and its
// number of domains in the list
static acsfit_status ts_begin_nodes(acsfit_ctx *ctx, TsPass &tp, int64_t N, cudaStream_t st)
{
    const acsfit_topology_spread *ts = tp.ts;
    int init[128];
    for (int k = 0; k < 64; ++k) {
        init[k] = INT_MAX;
        init[64 + k] = 0;
    }
    CUDA_TRY(cudaMemcpyAsync(tp.dmin, init, sizeof(int) * 64, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemcpyAsync(tp.dndom, init + 64, sizeof(int) * 64, cudaMemcpyHostToDevice, st));
    if (N > 0 && ts->keys > 0) {
        ts_domains_kernel<<<grid_for(ctx, N * ts->keys, 256), 256, 0, st>>>(
            ts->node_count, reinterpret_cast<const unsigned long long *>(ts->node_domain), N, ts->keys, nullptr,
            tp.dmin, tp.dndom, nullptr);
        ++ctx->launches;
    }
    int dmin[64];
    CUDA_TRY(cudaMemcpyAsync(dmin, tp.dmin, sizeof dmin, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(tp.ndom, tp.dndom, sizeof tp.ndom, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    CUDA_TRY(cudaGetLastError());
    for (int k = 0; k < ts->keys; ++k) tp.base[k] = std::min(ts->floor[k], dmin[k]);
    return ACSFIT_OK;
}

// before a pass: the limits of positions [0, n) under the fixed rises and (node pass) the watch of each key's next
// rise: its target is its current top level + 1, unless the key has no domain in the list or its floor (the fixed
// domains outside it) is below the target -- then its minimum can never reach it.  Once kMaxSpreadRises rises are
// fixed nothing is watched any more: the pass keeps the levels it has, which are at most the true minimums, so beyond
// the last fixed rise it refuses some pods the scheduler would place and accepts none it would refuse on that count
static acsfit_status ts_prepare(acsfit_ctx *ctx, TsPass &tp, const int32_t *idx, int64_t n, int64_t N, bool nodes,
                                cudaStream_t st)
{
    const acsfit_topology_spread *ts = tp.ts;
    tp.watching = false;
    for (int k = 0; k < 64; ++k) {
        tp.tgt[k] = INT_MAX;
        if (!nodes || k >= ts->keys) continue;
        const long long t = (long long)tp.base[k] + tp.nfixed[k] + 1;
        if (tp.ndom[k] > 0 && t < INT_MAX && (long long)ts->floor[k] >= t &&
            (int)tp.rises.size() / 2 < kMaxSpreadRises) {
            tp.tgt[k] = (int)t;
            tp.watching = true;
        }
    }
    if (nodes) {
        CUDA_TRY(cudaMemcpyAsync(tp.target, tp.tgt, sizeof tp.tgt, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemsetAsync(tp.reached, 0, sizeof(int) * 64, st));
        CUDA_TRY(cudaMemsetAsync(tp.rise_pos, 0, sizeof(unsigned long long) * 64, st));
        if (tp.watching && N > 0) {  // domains already at the target count as reached
            ts_domains_kernel<<<grid_for(ctx, N * ts->keys, 256), 256, 0, st>>>(
                ts->node_count, reinterpret_cast<const unsigned long long *>(ts->node_domain), N, ts->keys, tp.target,
                nullptr, nullptr, tp.reached);
            ++ctx->launches;
        }
    }
    TsLevels lv;
    const int n_rises = (int)tp.rises.size() / 2;
    std::vector<long long> pos(n_rises);
    for (int k = 0; k < 64; ++k) {
        lv.base[k] = tp.base[k];
        lv.off[k] = 0;
    }
    lv.off[64] = 0;
    for (int r = 0; r < n_rises; ++r) ++lv.off[tp.rises[2 * r] + 1];
    for (int k = 0; k < 64; ++k) lv.off[k + 1] += lv.off[k];
    int fill[64];
    std::copy(lv.off, lv.off + 64, fill);
    for (int r = 0; r < n_rises; ++r) pos[fill[tp.rises[2 * r]]++] = tp.rises[2 * r + 1];
    for (int k = 0; k < 64; ++k) std::sort(pos.begin() + lv.off[k], pos.begin() + lv.off[k + 1]);  // (fixed in order)
    lv.pos = tp.rises_dev;
    if (n_rises > 0)
        CUDA_TRY(cudaMemcpyAsync(tp.rises_dev, pos.data(), sizeof(long long) * n_rises, cudaMemcpyHostToDevice, st));
    if (n > 0) {
        ts_lim_kernel<<<grid_for(ctx, n, 256), 256, 0, st>>>(ts->pod_key, ts->pod_skew, idx, n, lv, tp.lim);
        ++ctx->launches;
    }
    CUDA_TRY(cudaGetLastError());
    if (n_rises > 0) CUDA_TRY(cudaStreamSynchronize(st));  // the host copy of the rises must outlive the transfer
    return ACSFIT_OK;
}

// after a node pass with topology spread: the earliest event among the placed watched pod-affinity signatures and
// the keys whose every domain reached its target (the lower event on a tie, a flip before a rise, then the lowest
// signature / key) is fixed and `again` set; `again` stays false when there is none
static acsfit_status ts_next_event(acsfit_ctx *ctx, const unsigned long long *first_placed, uint64_t watch,
                                   uint64_t &fixed, PaFlips &fl, TsPass &tp, bool &again, cudaStream_t st)
{
    again = false;
    const uint64_t open = watch & ~fixed;
    unsigned long long fp[64], rp[64];
    int reached[64];
    if (open) CUDA_TRY(cudaMemcpyAsync(fp, first_placed, sizeof fp, cudaMemcpyDeviceToHost, st));
    if (tp.watching) {
        CUDA_TRY(cudaMemcpyAsync(rp, tp.rise_pos, sizeof rp, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaMemcpyAsync(reached, tp.reached, sizeof reached, cudaMemcpyDeviceToHost, st));
    }
    CUDA_TRY(cudaStreamSynchronize(st));
    int best_s = -1, best_k = -1;
    for (int s = 0; open && s < 64; ++s)
        if (((open >> s) & 1u) && fp[s] != ~0ull && (best_s < 0 || fp[s] < fp[best_s])) best_s = s;
    for (int k = 0; tp.watching && k < 64; ++k)
        if (tp.tgt[k] != INT_MAX && reached[k] >= tp.ndom[k] && (best_k < 0 || rp[k] < rp[best_k])) best_k = k;
    if (best_s >= 0 && (best_k < 0 || fp[best_s] <= rp[best_k])) {
        fl.f[best_s] = (long long)fp[best_s];
        fixed |= 1ull << best_s;
        ctx->pa_flips.push_back(best_s);
        ctx->pa_flips.push_back((int64_t)fp[best_s]);
        again = true;
    } else if (best_k >= 0) {  // (ts_prepare watches nothing once kMaxSpreadRises are fixed)
        tp.rises.push_back(best_k);
        tp.rises.push_back((long long)rp[best_k]);
        ++tp.nfixed[best_k];
        ctx->ts_rises.push_back(best_k);
        ctx->ts_rises.push_back((int64_t)rp[best_k]);
        again = true;
    }
    return ACSFIT_OK;
}

// aa (needs pod_class / node_match): anti-affinity masks (the SEL + AA form; single GPU only)
// pa (needs aa): pod-affinity masks (the SEL + AA + PA form), run again from the saved node state per fixed flip
// ts (needs pa): topology spread (the SEL + AA + PA + TS form), run again per fixed flip or rise
static acsfit_status first_fit_impl(acsfit_ctx *ctx, const double *req, const int32_t *pod_idx, int64_t P, int D,
                                    const double *cap_type, const int32_t *node_type, double *used, int64_t N,
                                    int32_t *out_placed, unsigned long long *out_decisions, cudaStream_t st,
                                    const uint8_t *pod_class = nullptr, const unsigned long long *node_match = nullptr,
                                    const acsfit_anti_affinity *aa = nullptr, const acsfit_pod_affinity *pa = nullptr,
                                    const acsfit_topology_spread *ts = nullptr)
{
    if (ctx->world > 1)
        return cluster_first_fit(ctx, req, pod_idx, P, D, cap_type, node_type, used, N, out_placed, out_decisions, st);
    if (out_decisions) CUDA_TRY(cudaMemsetAsync(out_decisions, 0, sizeof(unsigned long long), st));
    if (P == 0) return ACSFIT_OK;
    fill_i32_kernel<<<grid_for(ctx, P, 256), 256, 0, st>>>(out_placed, P, -1);
    ++ctx->launches;
    if (N == 0) {  // every pod is pending and the reference makes no can_fit call
        CUDA_TRY(cudaGetLastError());
        return ACSFIT_OK;
    }
    const StagePlan plan = plan_stages(ctx, N, 0, D, false);
    const int64_t alive_words = (P + 31) / 32;
    TAKE(alive, uint32_t, alive_words);
    TAKE(sync_words, int, plan.stages + 8);
    int *ticket = sync_words, *status = sync_words + 1, *drained = sync_words + 2, *progress = sync_words + 8;
    CUDA_TRY(cudaMemsetAsync(sync_words, 0, sizeof(int) * (plan.stages + 8), st));
    fill_alive_kernel<<<grid_for(ctx, alive_words, 256), 256, 0, st>>>(alive, P);
    ++ctx->launches;

    PipelineParams pp;
    memset(&pp, 0, sizeof pp);
    pp.req = req;
    pp.pod_idx = pod_idx;
    pp.M = P;
    pp.alive = alive;
    pp.placed = out_placed;
    pp.cap_type = cap_type;
    pp.node_type = node_type;
    pp.used = used;
    pp.node_lo = 0;
    pp.node_hi = N;
    pp.Tn = plan.Tn;
    pp.NS = plan.NS;
    pp.num_tiles = (int)((P + kTile - 1) / kTile);
    pp.ticket = ticket;
    pp.progress = progress;
    pp.status = status;
    pp.drained = drained;
    pp.watchdog_ns = (unsigned long long)ctx->watchdog_ms * 1000000ull;
    pp.rk = ctx->rk;
    pp.pod_class = pod_class;
    pp.node_match = node_match;
    if (aa) {
        pp.pod_carries = reinterpret_cast<const unsigned long long *>(aa->pod_carries);
        pp.pod_matches = reinterpret_cast<const unsigned long long *>(aa->pod_matches);
        pp.node_carries = reinterpret_cast<unsigned long long *>(aa->node_carries);
        pp.node_matches = reinterpret_cast<unsigned long long *>(aa->node_matches);
    }
    unsigned long long *hits = nullptr;
    if (node_match) {
        hits = arena_take<unsigned long long>(ctx, 1);
        if (!hits) return fail(ctx, ACSFIT_E_NOMEM, "scratch arena too small for hits");
        CUDA_TRY(cudaMemsetAsync(hits, 0, sizeof(unsigned long long), st));
        pp.sel_hits = hits;
    }
    // pod affinity: the signatures no node holds at the start that some pod of the list matches itself are watched;
    // the pass runs again, from the saved node state, for every one that gets placed (include/acsfit.h)
    // topology spread: the keys' minimums at the start, the watched next rises and the limits of the first pass
    TsPass tp;
    int32_t *counts0 = nullptr;
    if (ts) {
        TRY(ts_alloc(ctx, ts, P, tp));
        TRY(ts_begin_nodes(ctx, tp, N, st));
        TRY(ts_prepare(ctx, tp, pod_idx, P, N, true, st));
        pp.ts_key = ts->pod_key;
        pp.ts_lim = tp.lim;
        pp.ts_matches = reinterpret_cast<const unsigned long long *>(ts->pod_matches);
        pp.ts_count = ts->node_count;
        pp.ts_domain = reinterpret_cast<const unsigned long long *>(ts->node_domain);
        pp.ts_target = tp.target;
        pp.ts_reached = tp.reached;
        pp.ts_rise_pos = tp.rise_pos;
        pp.ts_stride = N;
        pp.ts_keys = ts->keys;
    }
    PaFlips fl;
    uint64_t watch = 0, fixed = 0;
    bool rerun = false;  // a later pass may be needed: the node state is saved
    double *used0 = nullptr;
    unsigned long long *masks0 = nullptr, *need = nullptr;
    if (pa) {
        need = arena_take<unsigned long long>(ctx, P);
        pp.pod_need = need;
        pp.first_placed = arena_take<unsigned long long>(ctx, 64);
        unsigned long long *red = arena_take<unsigned long long>(ctx, 1);
        if (!need || !pp.first_placed || !red) return fail(ctx, ACSFIT_E_NOMEM, "scratch arena too small for pod affinity");
        pp.pod_aff_matches = reinterpret_cast<const unsigned long long *>(pa->pod_matches);
        pp.node_has = reinterpret_cast<unsigned long long *>(pa->node_has);
        uint64_t present = 0, selfs = 0;
        TRY(or_rows(ctx, pa->node_has, nullptr, N, nullptr, red, &present, st));
        TRY(or_rows(ctx, pa->pod_self, pod_idx, P, nullptr, red, &selfs, st));
        for (int s = 0; s < 64; ++s) fl.f[s] = ((present >> s) & 1u) ? -1 : INT64_MAX;
        watch = selfs & ~present;
        rerun = watch || (ts && tp.watching);
        if (ts && rerun && ts->keys > 0) {  // the counts change in a pass: a rerun starts from the saved ones
            counts0 = arena_take<int32_t>(ctx, (size_t)N * ts->keys);
            if (!counts0) return fail(ctx, ACSFIT_E_NOMEM, "scratch arena too small for topology spread");
            CUDA_TRY(cudaMemcpyAsync(counts0, ts->node_count, sizeof(int32_t) * N * ts->keys, cudaMemcpyDeviceToDevice, st));
        }
        if (rerun) {
            used0 = arena_take<double>(ctx, (size_t)N * D);
            masks0 = arena_take<unsigned long long>(ctx, (size_t)N * 3);
            if (!used0 || !masks0) return fail(ctx, ACSFIT_E_NOMEM, "scratch arena too small for pod affinity");
            CUDA_TRY(cudaMemcpyAsync(used0, used, sizeof(double) * N * D, cudaMemcpyDeviceToDevice, st));
            CUDA_TRY(cudaMemcpyAsync(masks0, pp.node_has, sizeof(uint64_t) * N, cudaMemcpyDeviceToDevice, st));
            CUDA_TRY(cudaMemcpyAsync(masks0 + N, pp.node_carries, sizeof(uint64_t) * N, cudaMemcpyDeviceToDevice, st));
            CUDA_TRY(cudaMemcpyAsync(masks0 + 2 * N, pp.node_matches, sizeof(uint64_t) * N, cudaMemcpyDeviceToDevice, st));
        }
        pp.watch = watch;
        TRY(pa_prepare(ctx, pa, pod_idx, P, fl, watch, need, pp.first_placed, st));
    }

    if (ctx->timing) CUDA_TRY(cudaEventRecord(ctx->ev0, st));
    TRY(launch_pipeline<false>(ctx, D, pp, plan.stages, st));
    for (bool again = pa && rerun;;) {
        if (again) {
            TRY(check_pipeline_status(ctx, status, st));
            if (ts) TRY(ts_next_event(ctx, pp.first_placed, watch, fixed, fl, tp, again, st));
            else TRY(pa_next_flip(ctx, pp.first_placed, watch, fixed, fl, again, st));
        }
        if (!again) break;
        // run the pass again from its start: node state, sync words, alive bits and placements
        CUDA_TRY(cudaMemcpyAsync(used, used0, sizeof(double) * N * D, cudaMemcpyDeviceToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(pp.node_has, masks0, sizeof(uint64_t) * N, cudaMemcpyDeviceToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(pp.node_carries, masks0 + N, sizeof(uint64_t) * N, cudaMemcpyDeviceToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(pp.node_matches, masks0 + 2 * N, sizeof(uint64_t) * N, cudaMemcpyDeviceToDevice, st));
        CUDA_TRY(cudaMemsetAsync(sync_words, 0, sizeof(int) * (plan.stages + 8), st));
        fill_alive_kernel<<<grid_for(ctx, alive_words, 256), 256, 0, st>>>(alive, P);
        fill_i32_kernel<<<grid_for(ctx, P, 256), 256, 0, st>>>(out_placed, P, -1);
        ctx->launches += 2;
        pp.watch = watch & ~fixed;
        TRY(pa_prepare(ctx, pa, pod_idx, P, fl, pp.watch, need, pp.first_placed, st));
        if (ts) {
            if (counts0)
                CUDA_TRY(cudaMemcpyAsync(ts->node_count, counts0, sizeof(int32_t) * N * ts->keys, cudaMemcpyDeviceToDevice, st));
            TRY(ts_prepare(ctx, tp, pod_idx, P, N, true, st));
        }
        TRY(launch_pipeline<false>(ctx, D, pp, plan.stages, st));
    }
    if (ctx->timing) CUDA_TRY(cudaEventRecord(ctx->ev1, st));
    if (out_decisions) {
        decisions_kernel<<<grid_for(ctx, P, 256), 256, 0, st>>>(out_placed, P, N, out_decisions);
        ++ctx->launches;
    }
    TRY(check_pipeline_status(ctx, status, st));
    if (hits) {
        unsigned long long h = 0;
        CUDA_TRY(cudaMemcpy(&h, hits, sizeof h, cudaMemcpyDeviceToHost));
        ctx->last_sel_hits += h;
    }
    ctx->last_stages += plan.stages;
    ctx->last_tiles += pp.num_tiles;
    if (ctx->timing) {
        float ms = 0.f;
        CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
        ctx->last_ms += ms;
        if (g_trace) fprintf(stderr, "[acsfit] nodes pass: %lld pods, %d stages x %d nodes: %.3f ms\n", (long long)P, plan.stages, plan.Tn, ms);
        if (out_decisions) {
            unsigned long long d = 0;
            CUDA_TRY(cudaMemcpy(&d, out_decisions, sizeof d, cudaMemcpyDeviceToHost));
            ctx->last_decisions += d;
        }
    }
    return ACSFIT_OK;
}

// ---------------------------------------------------------------------------------------------
// fulfill_pending (implementation; scratch must already be reserved)
// ---------------------------------------------------------------------------------------------
constexpr int kMaxStagesPerPass = 1024;

// stages of one single-GPU bin pass at most (test knob "bin_pass_stages" lowers it; cluster mode plans its own)
static int bin_pass_cap(const acsfit_ctx *ctx)
{
    return ctx->bin_pass_stages > 0 ? std::min(ctx->bin_pass_stages, kMaxStagesPerPass) : kMaxStagesPerPass;
}

static size_t fulfill_scratch(int64_t Pp, int T, int D)
{
    const size_t nblocks = (size_t)((Pp + kCompactChunk - 1) / kCompactChunk) + 1;
    return 32768 + (size_t)Pp + sizeof(int32_t) * (size_t)Pp * 4 + sizeof(uint32_t) * (size_t)((Pp + 31) / 32) +
           sizeof(int) * (kMaxStagesPerPass + 8) + sizeof(int) * nblocks + sizeof(double) * (size_t)T * D + 256 * 16;
}

// req row of pending pod p is req[(row_map ? row_map[p] : p) * D]
// a first bin-packing pass that already ran (chained behind the node pipeline): for pool `pool` every pending
// pod was eligible, cur_bin[p] holds its bin (or -1) over bins [0, bins_covered), `evals` its credited tests
struct FirstPassDone {
    int pool;
    const int32_t *cur_bin;
    int64_t bins_covered;
    uint64_t evals;
};

static acsfit_status fulfill_impl(acsfit_ctx *ctx, const double *req, const int32_t *row_map, int64_t Pp,
                                  int64_t num_listed, int D, const double *unit_host, const int32_t *pool_actual,
                                  const int32_t *pool_max, const uint8_t *pool_ignored, int T, int64_t over_provision,
                                  int64_t *out_new_size, int64_t *out_units_needed, int64_t *out_bins_opened,
                                  int32_t *out_acc_pool, int32_t *out_bin_of, int64_t *out_unaccounted,
                                  uint64_t *out_evals, cudaStream_t st, const FirstPassDone *pre = nullptr,
                                  const uint8_t *pod_class = nullptr, const uint64_t *pool_match_host = nullptr,
                                  const acsfit_anti_affinity *aa = nullptr, const acsfit_pod_affinity *pa = nullptr,
                                  uint64_t present = 0, const acsfit_topology_spread *ts = nullptr)
{
    // ts (needs pa): topology spread; every bin pass runs the AA + PA + TS form.  A new bin starts with count 0 and
    // the minimum is taken as 0 there, so the limits are maxSkew - self throughout: no rises, no reruns.
    // aa: anti-affinity masks of the pods (indexed like req rows); every bin pass runs the AA form, unchained
    // pa (needs aa): pod-affinity masks; every bin pass runs the AA + PA form.  `present`: the signatures already held
    // (by the nodes); it gains those of the pods placed in each pool's bins.  A pool's packing runs again for every
    // flip it fixes, and bin_of is written from the final run.
    // pod_class [dev] (indexed like req rows) + pool_match_host [host] T (visiting order): node selectors.  They only
    // change the pool gate: every bin of a pool carries the pool's labels, so the bin passes are the plain ones.
    for (int i = 0; i < T * D; ++i)
        if (!std::isfinite(unit_host[i])) return fail(ctx, ACSFIT_E_DOMAIN, "fulfill_pending: non-finite unit capacity");
    const int64_t alive_words = (Pp + 31) / 32;
    const int nblocks = (int)((Pp + kCompactChunk - 1) / kCompactChunk) + 1;
    TAKE(elig, uint8_t, Pp);
    TAKE(list_a, int32_t, Pp);
    TAKE(list_b, int32_t, Pp);
    TAKE(placed, int32_t, Pp);
    TAKE(cur_bin, int32_t, Pp);
    TAKE(alive, uint32_t, alive_words);
    TAKE(sync_words, int, kMaxStagesPerPass + 8);
    TAKE(block_counts, int, nblocks);
    TAKE(unit_dev, double, (size_t)T * D);
    TAKE(total_dev, int64_t, 1);
    TAKE(evals_dev, unsigned long long, 1);
    TAKE(count_dev, unsigned long long, 1);
    TAKE(max_bin_dev, int, 1);
    PaFlips fl;
    uint64_t selfs = 0;
    unsigned long long *need = nullptr, *first_placed = nullptr, *evals_save = nullptr;
    if (pa) {
        TAKE(need_, unsigned long long, Pp);
        TAKE(fp_, unsigned long long, 64);
        TAKE(red_, unsigned long long, 2);
        need = need_;
        first_placed = fp_;
        evals_save = red_ + 1;
        TRY(or_rows(ctx, pa->pod_self, row_map, Pp, nullptr, red_, &selfs, st));
    }
    TsPass tp;
    if (ts) {
        TRY(ts_alloc(ctx, ts, Pp, tp));
        TRY(ts_prepare(ctx, tp, row_map, Pp, 0, false, st));
    }

    if (T > 0) CUDA_TRY(cudaMemcpyAsync(unit_dev, unit_host, sizeof(double) * T * D, cudaMemcpyHostToDevice, st));
    CUDA_TRY(cudaMemsetAsync(evals_dev, 0, sizeof(unsigned long long), st));
    if (Pp > 0) {
        fill_i32_kernel<<<grid_for(ctx, Pp, 256), 256, 0, st>>>(out_acc_pool, Pp, -1);
        fill_i32_kernel<<<grid_for(ctx, Pp, 256), 256, 0, st>>>(out_bin_of, Pp, -1);
        ctx->launches += 2;
    }

    uint64_t evals = 0;
    int64_t num_unaccounted = num_listed;  // scaler.py:120 (duplicates counted)
    int64_t unique_unaccounted = Pp;
    float total_ms = 0.f;

    for (int t = 0; t < T; ++t) {
        out_new_size[t] = pool_actual[t];  // scaler.py:125-126
        out_units_needed[t] = -1;
        out_bins_opened[t] = 0;
        if (pool_ignored[t] || !num_unaccounted) continue;  // scaler.py:128-129

        int64_t nb = 0, E = 0;
        const bool first_done = pre && pre->pool == t && Pp > 0;
        if (first_done) {
            // the gate held for every pending pod and the first pass over bins [0, bins_covered) is done
            E = Pp;
            evals += (uint64_t)unique_unaccounted + pre->evals;
        } else if (Pp > 0) {
            // pool gate (scaler.py:134) over the not-yet-accounted pods -> ordered list of eligible pods
            if (pod_class)
                eligible_sel_kernel<<<grid_for(ctx, Pp, 256), 256, 0, st>>>(req, row_map, Pp, D, unit_dev + (size_t)t * D,
                                                                           (unsigned long long)pool_match_host[t], pod_class,
                                                                           out_acc_pool, elig);
            else
                eligible_kernel<<<grid_for(ctx, Pp, 256), 256, 0, st>>>(req, row_map, Pp, D, unit_dev + (size_t)t * D,
                                                                       out_acc_pool, elig);
            ++ctx->launches;
            evals += (uint64_t)unique_unaccounted;
            TRY(compact(ctx, FlagPred{elig}, Pp, nullptr, list_a, block_counts, total_dev, &E, st));
        }
        if (E > 0) {
            CUDA_TRY(cudaMemsetAsync(max_bin_dev, 0xFF, sizeof(int), st));  // -1
            int32_t *list = list_a, *next = list_b;
            int64_t M = E, bin_base = 0;
            uint64_t watch = 0, fixed = 0;
            if (pa) {  // the signatures absent so far that some pod matches itself are watched
                for (int s = 0; s < 64; ++s) fl.f[s] = ((present >> s) & 1u) ? -1 : INT64_MAX;
                watch = selfs & ~present;
                TRY(pa_prepare(ctx, pa, row_map, Pp, fl, watch, need, first_placed, st));
                if (watch) CUDA_TRY(cudaMemcpyAsync(evals_save, evals_dev, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
            }
            if (first_done) {
                CUDA_TRY(cudaMemcpyAsync(cur_bin, pre->cur_bin, sizeof(int32_t) * Pp, cudaMemcpyDeviceToDevice, st));
                record_bins_kernel<<<grid_for(ctx, Pp, 256), 256, 0, st>>>(cur_bin, Pp, out_bin_of, max_bin_dev);
                ++ctx->launches;
                TRY(compact(ctx, NegPredI32{cur_bin}, Pp, nullptr, list_a, block_counts, total_dev, &M, st));
                bin_base = pre->bins_covered;
            } else {
                fill_i32_kernel<<<grid_for(ctx, Pp, 256), 256, 0, st>>>(cur_bin, Pp, -1);
                ++ctx->launches;
            }
            while (M > 0) {
                const bool cl = ctx->world > 1;
                StagePlan plan = plan_stages(ctx, M, bin_pass_cap(ctx), D, true);  // at most one bin per pod
                int64_t pass_bins = (int64_t)plan.stages * plan.Tn;
                int *sy = sync_words;
                uint32_t *al = alive;
                int32_t *pl = placed;
                if (cl) {
                    // cluster mode: the pass's bins are split over the ranks, rank r takes the r-th run of S stages and
                    // its stage 0 is fed by rank r-1's last stage; all S stages of a rank are resident at once
                    const int K = nodes_per_thread(D, ctx->rk.nw);
                    int NS = max_stage_nodes(D, true) / K;
                    while (NS * K > 32 && (M + (int64_t)NS * K - 1) / ((int64_t)NS * K) < (int64_t)ctx->world * ctx->num_sms) NS >>= 1;
                    plan.NS = NS;
                    plan.Tn = NS * K;
                    const int resident = resident_stages(ctx, D, true, plan.Tn);
                    if (resident <= 0) return fail(ctx, ACSFIT_E_CUDA, "cluster mode: occupancy query failed");
                    const int64_t total = std::min<int64_t>((M + plan.Tn - 1) / plan.Tn, (int64_t)ctx->world * resident);
                    plan.stages = (int)std::max<int64_t>(1, (total + ctx->world - 1) / ctx->world);
                    if (plan.stages + 8 > kClusterSyncInts) plan.stages = kClusterSyncInts - 8;
                    pass_bins = (int64_t)ctx->world * plan.stages * plan.Tn;
                    sy = x_syncset(ctx, ctx->rank, 0);
                    al = x_alive_of(ctx, ctx->rank);
                    pl = x_placed_of(ctx, ctx->rank);
                    if (M > ctx->x_max_pods) return fail(ctx, ACSFIT_E_INVALID, "cluster mode: %lld pods exceed the exchange region", (long long)M);
                    CUDA_TRY(cudaMemsetAsync(x_status(ctx, ctx->rank), 0, sizeof(int), st));
                }
                CUDA_TRY(cudaMemsetAsync(sy, 0, sizeof(int) * (plan.stages + 8), st));
                if (!cl || ctx->rank == 0) fill_alive_kernel<<<grid_for(ctx, (M + 31) / 32, 256), 256, 0, st>>>(al, M);
                fill_i32_kernel<<<grid_for(ctx, M, 256), 256, 0, st>>>(pl, M, -1);
                ctx->launches += 2;
                if (cl) TRY(cluster_barrier(ctx, st));  // every rank's counters are zero before anybody polls them
                PipelineParams pp;
                memset(&pp, 0, sizeof pp);
                pp.req = req;
                pp.pod_idx = list;
                pp.row_map = row_map;
                pp.M = M;
                pp.alive = al;
                pp.placed = pl;
                pp.unit = unit_dev + (size_t)t * D;
                pp.bin_base = bin_base;
                pp.node_lo = bin_base + (cl ? (int64_t)ctx->rank * plan.stages * plan.Tn : 0);
                pp.node_hi = pp.node_lo + (int64_t)plan.stages * plan.Tn;
                pp.Tn = plan.Tn;
                pp.NS = plan.NS;
                pp.num_tiles = (int)((M + kTile - 1) / kTile);
                pp.ticket = sy;
                pp.progress = sy + 8;
                pp.status = cl ? x_status(ctx, ctx->rank) : sy + 1;
                pp.drained = sy + 2;
                pp.evals = evals_dev;
                if (cl) {
                    pp.sys_scope = 1;
                    if (ctx->rank > 0) {
                        pp.upstream = x_syncset(ctx, ctx->rank - 1, 0) + 8 + (plan.stages - 1);
                        pp.alive_in = x_alive_of(ctx, ctx->rank - 1);
                    }
                }
                pp.watchdog_ns = (unsigned long long)ctx->watchdog_ms * 1000000ull;
                pp.rk = ctx->rk;
                if (aa) {
                    pp.pod_carries = reinterpret_cast<const unsigned long long *>(aa->pod_carries);
                    pp.pod_matches = reinterpret_cast<const unsigned long long *>(aa->pod_matches);
                }
                if (pa) {
                    pp.pod_need = need;
                    pp.pod_aff_matches = reinterpret_cast<const unsigned long long *>(pa->pod_matches);
                    pp.first_placed = first_placed;
                    pp.watch = watch & ~fixed;
                }
                if (ts) {
                    pp.ts_key = ts->pod_key;
                    pp.ts_lim = tp.lim;
                    pp.ts_matches = reinterpret_cast<const unsigned long long *>(ts->pod_matches);
                    pp.ts_keys = ts->keys;
                }
                if (ctx->timing) CUDA_TRY(cudaEventRecord(ctx->ev0, st));
                ctx->rec_pool = t;
                TRY(launch_pipeline<true>(ctx, D, pp, plan.stages, st));
                if (ctx->timing) CUDA_TRY(cudaEventRecord(ctx->ev1, st));
                if (cl) TRY(cluster_merge_placed(ctx, M, placed, st));  // every rank: the pass's complete placements
                scatter_bins_kernel<<<grid_for(ctx, M, 256), 256, 0, st>>>(list, placed, M, cur_bin,
                                                                          pa ? cur_bin : out_bin_of, max_bin_dev);
                ++ctx->launches;
                TRY(check_pipeline_status(ctx, pp.status, st));
                if (ctx->timing) {
                    float ms = 0.f;
                    CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
                    total_ms += ms;
                    if (g_trace) fprintf(stderr, "[acsfit r%d] bins pass: pool %d, %lld pods, %d stages x %d bins, base %lld: %.3f ms\n",
                                         ctx->rank, t, (long long)M, plan.stages, plan.Tn, (long long)bin_base, ms);
                }
                ctx->last_stages += plan.stages;
                ctx->last_tiles += pp.num_tiles;
                // pods that fitted none of this pass's bins go on to a pass of fresh bins
                int64_t left = 0;
                if (cl) TRY(compact(ctx, NegPredI32{placed}, M, list, next, block_counts, total_dev, &left, st));
                else TRY(compact(ctx, BitPred{alive}, M, list, next, block_counts, total_dev, &left, st));
                bin_base += pass_bins;
                std::swap(list, next);
                // pod affinity: a pod may fit no bin, a fresh one included; once a pass places nothing the rest stays
                // unaccounted for this pool.  When the packing is over and it placed a watched signature, it runs
                // again from scratch with that signature's flip fixed.
                if (pa && left == M) left = 0;
                M = left;
                if (pa && M == 0) {
                    bool again = false;
                    TRY(pa_next_flip(ctx, first_placed, watch, fixed, fl, again, st));
                    if (again) {
                        CUDA_TRY(cudaMemcpyAsync(evals_dev, evals_save, sizeof(unsigned long long), cudaMemcpyDeviceToDevice, st));
                        CUDA_TRY(cudaMemsetAsync(max_bin_dev, 0xFF, sizeof(int), st));
                        fill_i32_kernel<<<grid_for(ctx, Pp, 256), 256, 0, st>>>(cur_bin, Pp, -1);
                        ++ctx->launches;
                        list = list_a;
                        next = list_b;
                        TRY(compact(ctx, FlagPred{elig}, Pp, nullptr, list, block_counts, total_dev, &M, st));
                        bin_base = 0;
                        TRY(pa_prepare(ctx, pa, row_map, Pp, fl, watch & ~fixed, need, first_placed, st));
                    }
                }
            }
            if (pa) {  // bin_of from the final run; the signatures of the pods it placed are present from now on
                record_bins_kernel<<<grid_for(ctx, Pp, 256), 256, 0, st>>>(cur_bin, Pp, out_bin_of, max_bin_dev);
                ++ctx->launches;
                uint64_t placed_sigs = 0;
                TRY(or_rows(ctx, pa->pod_matches, row_map, Pp, cur_bin, first_placed, &placed_sigs, st));
                present |= placed_sigs;
            }
            int max_bin = -1;
            CUDA_TRY(cudaMemcpyAsync(&max_bin, max_bin_dev, sizeof(int), cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            nb = (int64_t)max_bin + 1;  // opened bins form a prefix
        }
        // scaler.py:152-167
        const int64_t needed = nb + over_provision;
        const int64_t room = (int64_t)pool_max[t] - (int64_t)pool_actual[t];
        const int64_t unavailable = std::max<int64_t>(0, needed - room);
        const int64_t requested = needed - unavailable;
        out_units_needed[t] = needed;
        out_bins_opened[t] = nb;
        out_new_size[t] = (int64_t)pool_actual[t] + requested;
        const int64_t take = std::min(nb, requested);  // range(min(len(bins), units_requested))
        if (take > 0 && E > 0) {
            CUDA_TRY(cudaMemsetAsync(count_dev, 0, sizeof(unsigned long long), st));
            account_kernel<<<grid_for(ctx, Pp, 256), 256, 0, st>>>(
                cur_bin, Pp, (int32_t)std::min<int64_t>(take, INT32_MAX), t, out_acc_pool, count_dev);
            ++ctx->launches;
            unsigned long long cnt = 0;
            CUDA_TRY(cudaMemcpyAsync(&cnt, count_dev, sizeof cnt, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            num_unaccounted -= (int64_t)cnt;
            unique_unaccounted -= (int64_t)cnt;
        }
    }
    unsigned long long bin_evals = 0;
    if (ctx->world > 1) {  // every rank credited the tests of its own bins: sum them (also checks every rank's status)
        TAKE(sc17, unsigned long long, 17);
        TRY(cluster_sum_u64(ctx, evals_dev, sc17, &bin_evals, st));
    } else {
        CUDA_TRY(cudaMemcpyAsync(&bin_evals, evals_dev, sizeof bin_evals, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
    }
    CUDA_TRY(cudaGetLastError());
    evals += bin_evals;
    *out_unaccounted = num_unaccounted;
    if (out_evals) *out_evals = evals;
    ctx->last_ms += total_ms;
    ctx->last_decisions += evals;
    return ACSFIT_OK;
}

// upper bound of the streaming forms' grid (they shrink it to the CTAs the GPU holds at once)
static int stream_grid(const acsfit_ctx *ctx, int64_t N)
{
    return (int)std::max<int64_t>(1, std::min<int64_t>(((N + 31) / 32 + kStreamWarps - 1) / kStreamWarps,
                                                       (int64_t)ctx->num_sms * 16));
}

// K6 dispatch: the form plan_scan picks (acsfit_scan_plan.h) -- a streaming form for padded column counts and
// 16-byte aligned tables, the simple per-thread form otherwise
static acsfit_status run_node_states(acsfit_ctx *ctx, const int64_t *row_ptr, const int32_t *run_idx,
                                     const double *req_run, const uint8_t *flags_run, const double *cap_type,
                                     const int32_t *node_type, const uint8_t *node_flags, const int64_t *node_age,
                                     int64_t N, int D, int any_pending, const int64_t *thr_dev, int S,
                                     uint8_t *out_state, cudaStream_t st)
{
    const ScanPlan p = plan_scan(D, true, run_idx, req_run, flags_run, ctx->bulk_cfg, ctx->stream_bytes);
    ScanLaunch *rec = &ctx->scan_rec;
    if (p.form != kScanPerThread) {
        const int grid = stream_grid(ctx, N);
        cudaError_t e;
        switch (D) {
        case 2: e = launch_node_stream<2, true>(p, grid, st, row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags, node_age, N, any_pending, thr_dev, S, out_state, nullptr, rec); break;
        case 4: e = launch_node_stream<4, true>(p, grid, st, row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags, node_age, N, any_pending, thr_dev, S, out_state, nullptr, rec); break;
        case 8: e = launch_node_stream<8, true>(p, grid, st, row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags, node_age, N, any_pending, thr_dev, S, out_state, nullptr, rec); break;
        default: e = launch_node_stream<16, true>(p, grid, st, row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags, node_age, N, any_pending, thr_dev, S, out_state, nullptr, rec); break;
        }
        ++ctx->launches;
        if (e != cudaSuccess) return fail(ctx, ACSFIT_E_CUDA, "node_states: %s", cudaGetErrorString(e));
        return ACSFIT_OK;
    }
    const int grid = grid_for(ctx, N, kPerThreadBlock);
    node_states_kernel<<<grid, kPerThreadBlock, 0, st>>>(row_ptr, run_idx, req_run, flags_run, cap_type, node_type,
                                                         node_flags, node_age, N, D, any_pending, thr_dev, S, out_state);
    *rec = {2, kScanPerThread, D, 0, kPerThreadBlock / 32, 0, grid, S};
    ++ctx->launches;
    CUDA_TRY(cudaGetLastError());
    return ACSFIT_OK;
}

// ---------------------------------------------------------------------------------------------
// ABI: device-pointer entry points
// ---------------------------------------------------------------------------------------------
extern "C" acsfit_status acsfit_feasible_mask(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                              const double *unit, int T, uint8_t *out_mask,
                                              uint64_t *out_evals, acsfit_stream_t stream)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    if (P < 0 || T < 0 || T > ACSFIT_MAX_POOLS || (P > 0 && (!req || !out_mask)) || (T > 0 && !unit))
        return fail(ctx, ACSFIT_E_INVALID, "feasible_mask: bad arguments");
    if (out_evals) CUDA_TRY(cudaMemsetAsync(out_evals, 0, sizeof(uint64_t), st));
    if (P == 0) return ACSFIT_OK;
    feasible_mask_kernel<<<grid_for(ctx, P, 256), 256, sizeof(double) * std::max(1, T * D), st>>>(
        req, P, D, unit, T, out_mask, reinterpret_cast<unsigned long long *>(out_evals));
    ++ctx->launches;
    CUDA_TRY(cudaGetLastError());
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_occupancy(acsfit_ctx *ctx, const int64_t *row_ptr, const int32_t *run_idx,
                                          const double *req_run, int64_t N, int D, double *used_inout,
                                          acsfit_stream_t stream)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    if (N < 0 || (N > 0 && (!row_ptr || !used_inout)))
        return fail(ctx, ACSFIT_E_INVALID, "occupancy: bad arguments");
    if (N == 0) return ACSFIT_OK;
    const ScanPlan p = plan_scan(D, false, run_idx, req_run, nullptr, ctx->bulk_cfg, ctx->stream_bytes);
    ScanLaunch *rec = &ctx->scan_rec;
    if (p.form != kScanPerThread) {
        const int grid = stream_grid(ctx, N);
        cudaError_t e;
        switch (D) {
        case 2: e = launch_node_stream<2, false>(p, grid, st, row_ptr, run_idx, req_run, nullptr, nullptr, nullptr, nullptr, nullptr, N, 0, nullptr, 0, nullptr, used_inout, rec); break;
        case 4: e = launch_node_stream<4, false>(p, grid, st, row_ptr, run_idx, req_run, nullptr, nullptr, nullptr, nullptr, nullptr, N, 0, nullptr, 0, nullptr, used_inout, rec); break;
        case 8: e = launch_node_stream<8, false>(p, grid, st, row_ptr, run_idx, req_run, nullptr, nullptr, nullptr, nullptr, nullptr, N, 0, nullptr, 0, nullptr, used_inout, rec); break;
        default: e = launch_node_stream<16, false>(p, grid, st, row_ptr, run_idx, req_run, nullptr, nullptr, nullptr, nullptr, nullptr, N, 0, nullptr, 0, nullptr, used_inout, rec); break;
        }
        ++ctx->launches;
        if (e != cudaSuccess) return fail(ctx, ACSFIT_E_CUDA, "occupancy: %s", cudaGetErrorString(e));
        return ACSFIT_OK;
    }
    const int grid = grid_for(ctx, N, kPerThreadBlock);
    occupancy_kernel<<<grid, kPerThreadBlock, 0, st>>>(row_ptr, run_idx, req_run, N, D, used_inout);
    *rec = {1, kScanPerThread, D, 0, kPerThreadBlock / 32, 0, grid, 0};
    ++ctx->launches;
    CUDA_TRY(cudaGetLastError());
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_first_fit_nodes(acsfit_ctx *ctx, const double *req, int64_t req_rows,
                                                const int32_t *pod_idx, int64_t P, int D,
                                                const double *cap_type, const int32_t *node_type,
                                                double *used_inout, int64_t N, int32_t *out_placed,
                                                uint64_t *out_decisions, acsfit_stream_t stream)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(check_first_fit_args(ctx, "first_fit_nodes", req, req_rows, pod_idx, P, D, cap_type, node_type, used_inout, N,
                             out_placed));
    reset_stats(ctx);
    TRY(arena_reserve(ctx, first_fit_scratch(ctx, P, N) + rank_scratch(req_rows, D) + 1024, st));
    ctx->arena_off = 0;
    TAKE(flag, int, 1);
    TRY(check_domain(ctx, req, req_rows * D, flag, st, "req"));
    if (P > 0 && N > 0) TRY(build_ranks(ctx, req, req_rows, D, st));
    return first_fit_impl(ctx, req, pod_idx, P, D, cap_type, node_type, used_inout, N, out_placed,
                          reinterpret_cast<unsigned long long *>(out_decisions), st);
}

extern "C" acsfit_status acsfit_fulfill_pending(acsfit_ctx *ctx, const double *req, int64_t Pp,
                                                int64_t num_listed, int D, const double *unit,
                                                const int32_t *pool_actual, const int32_t *pool_max,
                                                const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                int64_t *out_new_size, int64_t *out_units_needed,
                                                int64_t *out_bins_opened, int32_t *out_acc_pool,
                                                int32_t *out_bin_of, int64_t *out_unaccounted,
                                                uint64_t *out_evals, acsfit_stream_t stream)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(check_fulfill_args(ctx, "fulfill_pending", req, Pp, num_listed, D, unit, pool_actual, pool_max, pool_ignored,
                           T, out_new_size, out_units_needed, out_bins_opened, out_acc_pool, out_bin_of,
                           out_unaccounted));
    reset_stats(ctx);
    TRY(arena_reserve(ctx, fulfill_scratch(Pp, T, D) + rank_scratch(Pp, D) + 1024, st));
    ctx->arena_off = 0;
    TAKE(flag, int, 1);
    TRY(check_domain(ctx, req, Pp * D, flag, st, "req"));
    TRY(build_ranks(ctx, req, Pp, D, st));
    return fulfill_impl(ctx, req, nullptr, Pp, num_listed, D, unit, pool_actual, pool_max, pool_ignored, T,
                        over_provision, out_new_size, out_units_needed, out_bins_opened, out_acc_pool, out_bin_of,
                        out_unaccounted, out_evals, st);
}

extern "C" acsfit_status acsfit_node_states(acsfit_ctx *ctx, const int64_t *row_ptr, const int32_t *run_idx,
                                            const double *req_run, const uint8_t *flags_run,
                                            const double *cap_type, const int32_t *node_type,
                                            const uint8_t *node_flags, const int64_t *node_age, int64_t N,
                                            int D, int any_pending, const int64_t *idle_threshold, int S,
                                            uint8_t *out_state, acsfit_stream_t stream)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    if (N < 0 || S < 1 || S > 64 || !idle_threshold ||
        (N > 0 && (!row_ptr || !cap_type || !node_type || !node_flags || !node_age || !out_state)))
        return fail(ctx, ACSFIT_E_INVALID, "node_states: bad arguments");
    if (N == 0) return ACSFIT_OK;
    TRY(arena_reserve(ctx, 8192, st));
    ctx->arena_off = 0;
    TAKE(thr_dev, int64_t, S);
    CUDA_TRY(cudaMemcpyAsync(thr_dev, idle_threshold, sizeof(int64_t) * S, cudaMemcpyHostToDevice, st));
    TRY(run_node_states(ctx, row_ptr, run_idx, req_run, flags_run, cap_type, node_type, node_flags, node_age, N, D,
                        any_pending, thr_dev, S, out_state, st));
    CUDA_TRY(cudaStreamSynchronize(st));  // idle_threshold is a host buffer
    return ACSFIT_OK;
}

static bool aligned8(const void *p) { return ((uintptr_t)p & 7u) == 0; }

// acsfit_pending_admit, acsfit_pending_admit_pa and acsfit_pending_admit_ts: one validation, arena and launch.
// `entry` is the entry point's launch record kernel (3, 4 or 5).  The anti-affinity test runs when any of the four
// anti-affinity arrays is given (always, for acsfit_pending_admit); the run pair must then be given when there are rows
// and the signature pair when U > 0.  The affinity test runs for acsfit_pending_admit_pa, and for
// acsfit_pending_admit_ts when run_has or sig_need is given.  The spread test runs for acsfit_pending_admit_ts: each
// key's minimum over the listed domains comes from ts_domains_kernel, the host folds floor in and stages each
// signature's limit, min(INT32_MAX, skew + min).
static acsfit_status pending_admit_impl(acsfit_ctx *ctx, int entry, const int64_t *row_ptr,
                                        const uint64_t *run_carries, const uint64_t *run_matches,
                                        const uint64_t *run_has, int64_t N, const uint64_t *node_match,
                                        const uint8_t *sig_class, const uint64_t *sig_carries,
                                        const uint64_t *sig_matches, const uint64_t *sig_need, const uint8_t *sig_key,
                                        const int32_t *sig_skew, int U, const acsfit_topology_spread *ts,
                                        uint8_t *node_flags_inout, cudaStream_t st)
{
    const char *what = entry == 3 ? "pending_admit" : entry == 4 ? "pending_admit_pa" : "pending_admit_ts";
    const bool aa = entry == 3 || run_carries || run_matches || sig_carries || sig_matches;
    const bool pa = entry == 4 || (entry == 5 && (run_has || sig_need));
    const bool tsf = entry == 5;
    if (N < 0 || U < 0 || (N > 0 && (!row_ptr || !node_flags_inout)) ||
        (N > 0 && U > 0 && (!sig_class || (aa && (!sig_carries || !sig_matches)) || (pa && !sig_need))))
        return fail(ctx, ACSFIT_E_INVALID, "%s: bad arguments", what);
    const int keys = tsf && ts ? ts->keys : 0;
    if (tsf) {
        if (!ts) return fail(ctx, ACSFIT_E_INVALID, "%s: topology-spread arrays missing", what);
        if (keys < 0 || keys > ACSFIT_MAX_TS_KEYS)
            return fail(ctx, ACSFIT_E_INVALID, "%s: %d spread keys, at most %d", what, keys, ACSFIT_MAX_TS_KEYS);
        if ((N > 0 && keys > 0 && (!ts->node_count || !ts->node_domain)) || (keys > 0 && !ts->floor) ||
            (U > 0 && (!sig_key || !sig_skew)))
            return fail(ctx, ACSFIT_E_INVALID, "%s: topology-spread field missing", what);
        for (int k = 0; k < keys; ++k)
            if (ts->floor[k] < 0)
                return fail(ctx, ACSFIT_E_INVALID, "%s: floor[%d] = %d is negative", what, k, ts->floor[k]);
        for (int u = 0; u < U; ++u)
            if ((sig_key[u] != kAdmitNoKey && sig_key[u] >= keys) || sig_skew[u] < 0)
                return fail(ctx, ACSFIT_E_INVALID, "%s: signature %d has key %d and skew %d (%d keys)", what, u,
                            sig_key[u], sig_skew[u], keys);
        if (((uintptr_t)ts->node_count & 3u) != 0 || ((uintptr_t)ts->node_domain & 7u) != 0)
            return fail(ctx, ACSFIT_E_INVALID, "%s: node_count must be 4-byte and node_domain 8-byte aligned", what);
    }
    if (N == 0) return ACSFIT_OK;
    if ((N + kAdmitBlock - 1) / kAdmitBlock > INT32_MAX)
        return fail(ctx, ACSFIT_E_INVALID, "%s: N=%lld nodes is too many", what, (long long)N);
    if (!aligned8(row_ptr) || !aligned8(run_carries) || !aligned8(run_matches) || !aligned8(run_has) ||
        !aligned8(node_match))
        return fail(ctx, ACSFIT_E_INVALID, "%s: row_ptr and the mask arrays must be 8-byte aligned", what);
    for (int u = 0; u < U; ++u)
        if (sig_class[u] >= ACSFIT_MAX_CLASSES)
            return fail(ctx, ACSFIT_E_INVALID, "%s: signature %d has class %d, need < %d", what, u, sig_class[u],
                        ACSFIT_MAX_CLASSES);
    int64_t ends[2] = {0, 0};  // row_ptr[0], row_ptr[N]: the rows the kernel reads
    CUDA_TRY(cudaMemcpyAsync(&ends[0], row_ptr, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaMemcpyAsync(&ends[1], row_ptr + N, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    if (ends[0] < 0 || ends[1] < ends[0])
        return fail(ctx, ACSFIT_E_INVALID, "%s: row_ptr[0]=%lld, row_ptr[N]=%lld", what, (long long)ends[0],
                    (long long)ends[1]);
    if (ends[1] > ends[0] && ((aa && (!run_carries || !run_matches)) || (pa && !run_has)))
        return fail(ctx, ACSFIT_E_INVALID, "%s: %lld rows but a NULL run mask array", what,
                    (long long)(ends[1] - ends[0]));
    const size_t Uq = (size_t)std::max(U, 1);
    TRY(arena_reserve(ctx, Uq * ((aa ? 2 : 0) * sizeof(uint64_t) + (pa ? sizeof(uint64_t) : 0) + 1) + 1024 +
                               (tsf ? Uq * (1 + sizeof(int32_t)) + sizeof(int) * (2 * 64 + 1) + 1024 : 0), st));
    ctx->arena_off = 0;
    unsigned long long *d_carries = nullptr, *d_matches = nullptr, *d_need = nullptr;
    if (aa) {
        TAKE(carries, unsigned long long, Uq);
        TAKE(matches, unsigned long long, Uq);
        d_carries = carries;
        d_matches = matches;
    }
    if (pa) {
        TAKE(need, unsigned long long, Uq);
        d_need = need;
    }
    TAKE(d_class, uint8_t, Uq);
    uint8_t *d_key = nullptr;
    int32_t *d_limit = nullptr;
    if (tsf) {
        TAKE(key, uint8_t, Uq);
        TAKE(limit, int32_t, Uq);
        d_key = key;
        d_limit = limit;
    }
    if (tsf && keys > 0) {  // refuse negative counts, then each key's minimum over the listed domains
        TAKE(scratch, int, 2 * 64 + 1);
        int init[2 * 64 + 1];
        for (int k = 0; k < 64; ++k) {
            init[k] = INT_MAX;
            init[64 + k] = 0;
        }
        init[128] = 0;
        CUDA_TRY(cudaMemcpyAsync(scratch, init, sizeof init, cudaMemcpyHostToDevice, st));
        ts_check_kernel<<<grid_for(ctx, N * keys, 256), 256, 0, st>>>(nullptr, nullptr, nullptr, 0, keys,
                                                                      ts->node_count, N * keys, scratch + 128);
        ts_domains_kernel<<<grid_for(ctx, N * keys, 256), 256, 0, st>>>(
            ts->node_count, reinterpret_cast<const unsigned long long *>(ts->node_domain), N, keys, nullptr, scratch,
            scratch + 64, nullptr);
        ctx->launches += 2;
        int got[2 * 64 + 1];
        CUDA_TRY(cudaMemcpyAsync(got, scratch, sizeof got, cudaMemcpyDeviceToHost, st));
        CUDA_TRY(cudaStreamSynchronize(st));
        CUDA_TRY(cudaGetLastError());
        if (got[128] & 16) return fail(ctx, ACSFIT_E_INVALID, "%s: a node count is negative", what);
        std::vector<int32_t> limit(U);
        for (int u = 0; u < U; ++u) {
            const int k = sig_key[u];
            const long long m = k == kAdmitNoKey ? 0 : std::min(ts->floor[k], got[k]);
            limit[u] = (int32_t)std::min<long long>(INT32_MAX, (long long)sig_skew[u] + m);
        }
        if (U > 0) CUDA_TRY(cudaMemcpyAsync(d_limit, limit.data(), sizeof(int32_t) * U, cudaMemcpyHostToDevice, st));
    } else if (tsf && U > 0) {  // no key: every signature is 0xFF and its limit is never read
        CUDA_TRY(cudaMemsetAsync(d_limit, 0, sizeof(int32_t) * U, st));
    }
    if (U > 0) {
        if (aa) {
            CUDA_TRY(cudaMemcpyAsync(d_carries, sig_carries, sizeof(uint64_t) * U, cudaMemcpyHostToDevice, st));
            CUDA_TRY(cudaMemcpyAsync(d_matches, sig_matches, sizeof(uint64_t) * U, cudaMemcpyHostToDevice, st));
        }
        if (pa) CUDA_TRY(cudaMemcpyAsync(d_need, sig_need, sizeof(uint64_t) * U, cudaMemcpyHostToDevice, st));
        if (tsf) CUDA_TRY(cudaMemcpyAsync(d_key, sig_key, U, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(d_class, sig_class, U, cudaMemcpyHostToDevice, st));
    }
    const int grid = (int)((N + kAdmitBlock - 1) / kAdmitBlock);
    auto kernel = !tsf ? (!pa ? pending_admit_kernel<true, false, false>
                              : aa ? pending_admit_kernel<true, true, false> : pending_admit_kernel<false, true, false>)
                       : aa ? (pa ? pending_admit_kernel<true, true, true> : pending_admit_kernel<true, false, true>)
                            : (pa ? pending_admit_kernel<false, true, true> : pending_admit_kernel<false, false, true>);
    kernel<<<grid, kAdmitBlock, 0, st>>>(
        row_ptr, reinterpret_cast<const unsigned long long *>(run_carries),
        reinterpret_cast<const unsigned long long *>(run_matches), N,
        reinterpret_cast<const unsigned long long *>(node_match), d_class, d_carries, d_matches, U, node_flags_inout,
        reinterpret_cast<const unsigned long long *>(run_has), d_need, d_key, d_limit, keys > 0 ? ts->node_count : nullptr);
    if (tsf)
        ctx->scan_rec = {5, (aa ? 1 : 0) | (pa ? 2 : 0), 0, admit_smem_ts(aa, pa), kAdmitBlock / 32, kAdmitBlock, grid,
                         U};
    else if (pa)
        ctx->scan_rec = {4, aa ? 1 : 0, 0, aa ? kAdmitSmemAaPa : kAdmitSmemPa, kAdmitBlock / 32, kAdmitBlock, grid, U};
    else
        ctx->scan_rec = {3, kScanPerThread, 0, kAdmitSmem, kAdmitBlock / 32, kAdmitBlock, grid, U};
    ++ctx->launches;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(st));  // the signature table is a host buffer
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_pending_admit(acsfit_ctx *ctx, const int64_t *row_ptr, const uint64_t *run_carries,
                                              const uint64_t *run_matches, int64_t N, const uint64_t *node_match,
                                              const uint8_t *sig_class, const uint64_t *sig_carries,
                                              const uint64_t *sig_matches, int U, uint8_t *node_flags_inout,
                                              acsfit_stream_t stream)
{
    TRY(enter(ctx, 1));
    return pending_admit_impl(ctx, 3, row_ptr, run_carries, run_matches, nullptr, N, node_match, sig_class,
                              sig_carries, sig_matches, nullptr, nullptr, nullptr, U, nullptr, node_flags_inout,
                              (cudaStream_t)stream);
}

extern "C" acsfit_status acsfit_pending_admit_pa(acsfit_ctx *ctx, const int64_t *row_ptr, const uint64_t *run_carries,
                                                 const uint64_t *run_matches, const uint64_t *run_has, int64_t N,
                                                 const uint64_t *node_match, const uint8_t *sig_class,
                                                 const uint64_t *sig_carries, const uint64_t *sig_matches,
                                                 const uint64_t *sig_need, int U, uint8_t *node_flags_inout,
                                                 acsfit_stream_t stream)
{
    TRY(enter(ctx, 1));
    return pending_admit_impl(ctx, 4, row_ptr, run_carries, run_matches, run_has, N, node_match, sig_class,
                              sig_carries, sig_matches, sig_need, nullptr, nullptr, U, nullptr, node_flags_inout,
                              (cudaStream_t)stream);
}

extern "C" acsfit_status acsfit_pending_admit_ts(acsfit_ctx *ctx, const int64_t *row_ptr, const uint64_t *run_carries,
                                                 const uint64_t *run_matches, const uint64_t *run_has, int64_t N,
                                                 const uint64_t *node_match, const uint8_t *sig_class,
                                                 const uint64_t *sig_carries, const uint64_t *sig_matches,
                                                 const uint64_t *sig_need, const uint8_t *sig_key,
                                                 const int32_t *sig_skew, int U, const acsfit_topology_spread *ts,
                                                 uint8_t *node_flags_inout, acsfit_stream_t stream)
{
    TRY(enter(ctx, 1));
    return pending_admit_impl(ctx, 5, row_ptr, run_carries, run_matches, run_has, N, node_match, sig_class,
                              sig_carries, sig_matches, sig_need, sig_key, sig_skew, U, ts, node_flags_inout,
                              (cudaStream_t)stream);
}

static acsfit_status maintain_actions_impl(acsfit_ctx *ctx, uint8_t *io_state, const int32_t *node_pool, int64_t N,
                                           const int64_t *budget0, const uint8_t *pool_scalable, int T, int dry_run,
                                           uint8_t *out_action, cudaStream_t st)
{
    const int chunks = (int)((N + kMaintChunk - 1) / kMaintChunk);
    const int Tq = std::max(T, 1);
    TAKE(budget_dev, long long, Tq);
    TAKE(scal_dev, uint8_t, Tq);
    TAKE(counts, int, (size_t)chunks * Tq);
    if (T > 0) {
        CUDA_TRY(cudaMemcpyAsync(budget_dev, budget0, sizeof(long long) * T, cudaMemcpyHostToDevice, st));
        CUDA_TRY(cudaMemcpyAsync(scal_dev, pool_scalable, T, cudaMemcpyHostToDevice, st));
    }
    const int *rank_base = nullptr;
    if (!dry_run && T > 0) {
        maintain_count_kernel<<<chunks, kMaintBlock, sizeof(int) * Tq, st>>>(io_state, node_pool, N, scal_dev, T, counts);
        maintain_scan_kernel<<<(T + 63) / 64, 64, 0, st>>>(counts, chunks, T);
        ctx->launches += 2;
        rank_base = counts;
    }
    maintain_apply_kernel<<<chunks, kMaintBlock, sizeof(int) * Tq, st>>>(io_state, node_pool, N, budget_dev, scal_dev,
                                                                        T, dry_run, rank_base, out_action);
    ++ctx->launches;
    CUDA_TRY(cudaGetLastError());
    CUDA_TRY(cudaStreamSynchronize(st));  // budget0 / pool_scalable are host buffers
    return ACSFIT_OK;
}

static size_t maintain_scratch(int64_t N, int T)
{
    const size_t chunks = (size_t)((N + kMaintChunk - 1) / kMaintChunk) + 1;
    const size_t Tq = (size_t)std::max(T, 1);
    return 8192 + sizeof(int) * chunks * Tq + sizeof(long long) * Tq + Tq;
}

extern "C" acsfit_status acsfit_maintain_actions(acsfit_ctx *ctx, uint8_t *io_state, const int32_t *node_pool,
                                                 int64_t N, const int64_t *budget0, const uint8_t *pool_scalable,
                                                 int T, int dry_run, uint8_t *out_action, acsfit_stream_t stream)
{
    TRY(enter(ctx, 1));
    cudaStream_t st = (cudaStream_t)stream;
    if (N < 0 || T < 0 || T > ACSFIT_MAX_POOLS || (T > 0 && (!budget0 || !pool_scalable)) ||
        (N > 0 && (!io_state || !node_pool || !out_action)))
        return fail(ctx, ACSFIT_E_INVALID, "maintain_actions: bad arguments");
    if (N == 0) return ACSFIT_OK;
    TRY(arena_reserve(ctx, maintain_scratch(N, T), st));
    ctx->arena_off = 0;
    return maintain_actions_impl(ctx, io_state, node_pool, N, budget0, pool_scalable, T, dry_run, out_action, st);
}

// resident stage CTAs the device can hold for the nodes pipeline (all of them must be running before a
// chained bins pipeline may spin on their progress counters)
template <int D, bool BINS, bool SEL = false>
static int stage_capacity_t(acsfit_ctx *ctx, int Tn)
{
    PipelineParams q;
    memset(&q, 0, sizeof q);
    q.Tn = Tn;
    q.rk = ctx->rk;
    int resident = 0;  // a chained pass fits the GPU, hence runs unpruned
    if (launch_pipeline_v<D, BINS, false, SEL>(ctx, q, 0, nullptr, &resident) != ACSFIT_OK) return 0;
    return resident;
}
template <int D>
static int chained_capacity_t(acsfit_ctx *ctx, int Tn_nodes, int Tn_bins, bool sel)
{
    const int nodes = sel ? stage_capacity_t<D, false, true>(ctx, Tn_nodes) : stage_capacity_t<D, false>(ctx, Tn_nodes);
    return std::min(nodes, stage_capacity_t<D, true>(ctx, Tn_bins));
}
// stage CTAs of BOTH pipelines that can be resident together (conservatively: the smaller of the two
// per-kernel occupancies, slots taken as interchangeable); sel: the node pass is the node-selector form
static int chained_capacity(acsfit_ctx *ctx, int D, int Tn_nodes, int Tn_bins, bool sel)
{
    switch (D) {
    case 2: return chained_capacity_t<2>(ctx, Tn_nodes, Tn_bins, sel);
    case 4: return chained_capacity_t<4>(ctx, Tn_nodes, Tn_bins, sel);
    case 8: return chained_capacity_t<8>(ctx, Tn_nodes, Tn_bins, sel);
    case 16: return chained_capacity_t<16>(ctx, Tn_nodes, Tn_bins, sel);
    default: return 0;
    }
}

// get_pending_pods with the FIRST pool's bin packing chained behind it: the bins pipeline runs on a second
// stream and its stage 0 consumes every tile as soon as the last node stage has published it, so the two
// sequential placement chains overlap instead of adding up.  Only valid when every pod of the list is
// eligible for that pool (the caller checks) and all node stages are resident at once (checked here).
// bins_f[j] = bin of list entry j over bins [0, *bins_covered), or -1.
static acsfit_status first_fit_chained(acsfit_ctx *ctx, const double *req, const int32_t *list_f, int64_t F, int D,
                                       const double *cap_type, const int32_t *node_type, double *used, int64_t N,
                                       int32_t *placed_f, unsigned long long *decisions_dev,
                                       int pool, const double *unit_row_dev, int32_t *bins_f, int64_t *bins_covered,
                                       uint64_t *bin_evals, bool *did, cudaStream_t st,
                                       const uint8_t *pod_class = nullptr, const unsigned long long *node_match = nullptr)
{
    *did = false;
    const StagePlan pn = plan_stages(ctx, N, 0, D, false);
    StagePlan pb = plan_stages(ctx, F, bin_pass_cap(ctx), D, true);
    // every stage CTA of both pipelines must be resident at the same time: the bins stages spin on the node
    // stages' counters, and the two grids are dispatched in no particular order
    const int room = chained_capacity(ctx, D, pn.Tn, pb.Tn, node_match != nullptr) - pn.stages - 4;  // a little headroom
    if (room < 8) return ACSFIT_OK;  // node stages (nearly) fill the device: no chaining
    pb.stages = std::min(pb.stages, room);
    const int64_t alive_words = (F + 31) / 32;
    TAKE(alive, uint32_t, alive_words);
    TAKE(sync_n, int, pn.stages + 8);
    TAKE(sync_b, int, pb.stages + 8);
    TAKE(evals_dev, unsigned long long, 1);
    CUDA_TRY(cudaMemsetAsync(decisions_dev, 0, sizeof(unsigned long long), st));
    CUDA_TRY(cudaMemsetAsync(evals_dev, 0, sizeof(unsigned long long), st));
    CUDA_TRY(cudaMemsetAsync(sync_n, 0, sizeof(int) * (pn.stages + 8), st));
    CUDA_TRY(cudaMemsetAsync(sync_b, 0, sizeof(int) * (pb.stages + 8), st));
    fill_i32_kernel<<<grid_for(ctx, F, 256), 256, 0, st>>>(placed_f, F, -1);
    fill_i32_kernel<<<grid_for(ctx, F, 256), 256, 0, st>>>(bins_f, F, -1);
    fill_alive_kernel<<<grid_for(ctx, alive_words, 256), 256, 0, st>>>(alive, F);
    ctx->launches += 3;

    PipelineParams a;
    memset(&a, 0, sizeof a);
    a.req = req;
    a.pod_idx = list_f;
    a.M = F;
    a.alive = alive;
    a.placed = placed_f;
    a.cap_type = cap_type;
    a.node_type = node_type;
    a.used = used;
    a.node_lo = 0;
    a.node_hi = N;
    a.Tn = pn.Tn;
    a.NS = pn.NS;
    a.num_tiles = (int)((F + kTile - 1) / kTile);
    a.ticket = sync_n;
    a.status = sync_n + 1;
    a.drained = sync_n + 2;
    a.progress = sync_n + 8;
    a.watchdog_ns = (unsigned long long)ctx->watchdog_ms * 1000000ull;
    a.rk = ctx->rk;

    PipelineParams b = a;
    a.pod_class = pod_class;  // (the node pass only: the caller checked that every pod matches the pool)
    a.node_match = node_match;
    unsigned long long *hits = nullptr;
    if (node_match) {
        TAKE(hits_dev, unsigned long long, 1);
        CUDA_TRY(cudaMemsetAsync(hits_dev, 0, sizeof(unsigned long long), st));
        a.sel_hits = hits = hits_dev;
    }
    b.placed = bins_f;
    b.cap_type = nullptr;
    b.node_type = nullptr;
    b.used = nullptr;
    b.unit = unit_row_dev;
    b.bin_base = 0;
    b.node_lo = 0;
    b.node_hi = (int64_t)pb.stages * pb.Tn;
    b.Tn = pb.Tn;
    b.NS = pb.NS;
    b.ticket = sync_b;
    b.status = sync_n + 1;  // one abort word for both pipelines
    b.drained = sync_b + 2;
    b.progress = sync_b + 8;
    b.upstream = a.progress + (pn.stages - 1);
    b.evals = evals_dev;

    if (ctx->timing) CUDA_TRY(cudaEventRecord(ctx->ev0, st));
    CUDA_TRY(cudaEventRecord(ctx->ev_fork, st));
    ctx->rec_chained = 1;
    ctx->rec_pool = pool;
    TRY(launch_pipeline<false>(ctx, D, a, pn.stages, st));        // nodes first: its CTAs are dispatched first
    CUDA_TRY(cudaStreamWaitEvent(ctx->side, ctx->ev_fork, 0));
    TRY(launch_pipeline<true>(ctx, D, b, pb.stages, ctx->side));
    ctx->rec_chained = 0;
    CUDA_TRY(cudaEventRecord(ctx->ev_join, ctx->side));
    CUDA_TRY(cudaStreamWaitEvent(st, ctx->ev_join, 0));
    if (ctx->timing) CUDA_TRY(cudaEventRecord(ctx->ev1, st));
    decisions_kernel<<<grid_for(ctx, F, 256), 256, 0, st>>>(placed_f, F, N, decisions_dev);
    ++ctx->launches;
    unsigned long long ev = 0;
    CUDA_TRY(cudaMemcpyAsync(&ev, evals_dev, sizeof ev, cudaMemcpyDeviceToHost, st));
    TRY(check_pipeline_status(ctx, a.status, st));
    if (hits) {
        unsigned long long h = 0;
        CUDA_TRY(cudaMemcpy(&h, hits, sizeof h, cudaMemcpyDeviceToHost));
        ctx->last_sel_hits += h;
    }
    ctx->last_stages += pn.stages + pb.stages;
    ctx->last_tiles += 2 * a.num_tiles;
    if (ctx->timing) {
        float ms = 0.f;
        CUDA_TRY(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
        ctx->last_ms += ms;
        unsigned long long d = 0;
        CUDA_TRY(cudaMemcpy(&d, decisions_dev, sizeof d, cudaMemcpyDeviceToHost));
        ctx->last_decisions += d;
    }
    *bins_covered = (int64_t)pb.stages * pb.Tn;
    *bin_evals = ev;
    *did = true;
    return ACSFIT_OK;
}

// ---------------------------------------------------------------------------------------------
// fused scale-up tick: get_pods_to_schedule + get_pending_pods + fulfill_pending
// (reference cluster.py:169-175, :206-215) on DEVICE buffers
// ---------------------------------------------------------------------------------------------
namespace {
// placed_all[p] = -2 (infeasible) | -1 (pending) | node ; from the feasible list and its placements
__global__ void expand_placed_kernel(const uint8_t *feasible, int64_t P, int32_t *placed_all)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < P; i += (int64_t)gridDim.x * blockDim.x)
        placed_all[i] = feasible[i] ? -1 : -2;
}
__global__ void scatter_i32_kernel(const int32_t *list, const int32_t *vals, int64_t n, int32_t *out)
{
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
        out[list[i]] = vals[i];
}
struct NegPred {
    const int32_t *v;
    __device__ bool operator()(int64_t i) const { return v[i] < 0; }
};
}  // namespace

static size_t scale_up_scratch(const acsfit_ctx *ctx, int64_t P, int64_t N, int T, int D)
{
    const size_t nblocks = (size_t)((P + kCompactChunk - 1) / kCompactChunk) + 1;
    return first_fit_scratch(ctx, P, N) + fulfill_scratch(P, T, D) + rank_scratch(P, D) + sizeof(int32_t) * (size_t)P * 8 +
           sizeof(double) * (size_t)(N + 1) * D /*used backup of the chained launch*/ +
           sizeof(int) * (nblocks + kMaxStagesPerPass + 16) + sizeof(double) * (size_t)T * D * 2 + 65536;
}

static acsfit_status scale_up_impl(acsfit_ctx *ctx, const double *req, int64_t P, int D, const double *unit_all_host,
                                   const double *unit_ordered_host, const int32_t *pool_actual,
                                   const int32_t *pool_max, const uint8_t *pool_ignored, int T, int64_t over_provision,
                                   const double *cap_type, const int32_t *node_type, double *used, int64_t N,
                                   uint8_t *out_feasible, int32_t *out_placed, int64_t *out_new_size,
                                   int64_t *out_units_needed, int64_t *out_bins_opened, int32_t *out_acc_pool,
                                   uint64_t *out_counters, cudaStream_t st, const acsfit_selectors *sel = nullptr)
{
    const int nblocks = (int)((P + kCompactChunk - 1) / kCompactChunk) + 1;
    const uint8_t *pod_class = sel ? sel->pod_class : nullptr;
    const unsigned long long *node_match = sel ? reinterpret_cast<const unsigned long long *>(sel->node_match) : nullptr;
    TAKE(flag, int, 1);
    TAKE(unit_all_dev, double, (size_t)T * D);
    TAKE(list_f, int32_t, P);      // pods to schedule (feasible), in order
    TAKE(placed_f, int32_t, P);    // their placements
    TAKE(list_p, int32_t, P);      // pending pods (pod numbers), in order
    TAKE(acc_p, int32_t, P);
    TAKE(bin_p, int32_t, P);
    TAKE(block_counts, int, nblocks);
    TAKE(total_dev, int64_t, 1);
    TAKE(evals_dev, unsigned long long, 2);

    uint64_t decisions = 0;
    TRY(check_domain(ctx, req, P * D, flag, st, "req"));
    TRY(build_ranks(ctx, req, P, D, st));
    if (T > 0) CUDA_TRY(cudaMemcpyAsync(unit_all_dev, unit_all_host, sizeof(double) * T * D, cudaMemcpyHostToDevice, st));
    // get_pods_to_schedule (cluster.py:217-240)
    CUDA_TRY(cudaMemsetAsync(evals_dev, 0, 2 * sizeof(unsigned long long), st));
    int64_t F = 0;
    if (P > 0 && sel) {
        TAKE(match_all_dev, unsigned long long, T);
        if (T > 0) CUDA_TRY(cudaMemcpyAsync(match_all_dev, sel->pool_match_all, sizeof(uint64_t) * T, cudaMemcpyHostToDevice, st));
        feasible_mask_sel_kernel<<<grid_for(ctx, P, 256), 256, (sizeof(double) * D + sizeof(uint64_t)) * std::max(1, T), st>>>(
            req, P, D, unit_all_dev, match_all_dev, T, pod_class, out_feasible, evals_dev);
        ++ctx->launches;
    } else if (P > 0) {
        feasible_mask_kernel<<<grid_for(ctx, P, 256), 256, sizeof(double) * std::max(1, T * D), st>>>(
            req, P, D, unit_all_dev, T, out_feasible, evals_dev);
        ++ctx->launches;
    }
    if (P > 0) {
        expand_placed_kernel<<<grid_for(ctx, P, 256), 256, 0, st>>>(out_feasible, P, out_placed);
        fill_i32_kernel<<<grid_for(ctx, P, 256), 256, 0, st>>>(out_acc_pool, P, -1);
        ctx->launches += 2;
        TRY(compact(ctx, FlagPred{out_feasible}, P, nullptr, list_f, block_counts, total_dev, &F, st));
    }
    // get_pending_pods (cluster.py:184-204); when every pod to schedule is eligible for the first pool the
    // scaler will visit, that pool's bin packing is chained behind it on a second stream
    int64_t Pn = 0;
    FirstPassDone pre;
    bool chained = false;
    if (F > 0) {
        int t0 = 0;
        while (t0 < T && pool_ignored[t0]) ++t0;
        if (ctx->overlap && ctx->prune != 1 && N > 0 && t0 < T && ctx->world == 1) {  // (cluster mode: the ranks chain instead)  // (forced pruning changes the node kernel: no chaining)
            TAKE(unit_ord_dev, double, (size_t)T * D);
            TAKE(bins_f, int32_t, F);
            TAKE(j_of_p, int32_t, F);
            TAKE(cur_bin_p, int32_t, F);
            TAKE(inel_dev, unsigned long long, 1);
            CUDA_TRY(cudaMemcpyAsync(unit_ord_dev, unit_ordered_host, sizeof(double) * T * D, cudaMemcpyHostToDevice, st));
            CUDA_TRY(cudaMemsetAsync(inel_dev, 0, sizeof(unsigned long long), st));
            if (sel)
                count_ineligible_sel_kernel<<<grid_for(ctx, P, 256), 256, 0, st>>>(
                    out_feasible, req, P, D, unit_ord_dev + (size_t)t0 * D,
                    (unsigned long long)sel->pool_match_ordered[t0], pod_class, inel_dev);
            else
                count_ineligible_kernel<<<grid_for(ctx, P, 256), 256, 0, st>>>(out_feasible, req, P, D,
                                                                              unit_ord_dev + (size_t)t0 * D, inel_dev);
            ++ctx->launches;
            unsigned long long inel = 1;
            CUDA_TRY(cudaMemcpyAsync(&inel, inel_dev, sizeof inel, cudaMemcpyDeviceToHost, st));
            CUDA_TRY(cudaStreamSynchronize(st));
            if (inel == 0) {
                int64_t covered = 0;
                uint64_t bev = 0;
                // The chained launch needs every stage CTA of both grids resident at once; the occupancy query cannot see
                // SMs another context holds (a shared GPU, MPS).  If the watchdog fires, the node state is restored from
                // this copy and the tick is redone unchained (and the ctx stops chaining) instead of failing.
                TAKE(used_backup, double, (size_t)N * D);
                CUDA_TRY(cudaMemcpyAsync(used_backup, used, sizeof(double) * (size_t)N * D, cudaMemcpyDeviceToDevice, st));
                acsfit_status cs = first_fit_chained(ctx, req, list_f, F, D, cap_type, node_type, used, N, placed_f, evals_dev + 1,
                                                     t0, unit_ord_dev + (size_t)t0 * D, bins_f, &covered, &bev, &chained, st,
                                                     pod_class, node_match);
                if (cs == ACSFIT_OK && chained && ctx->inject_chain_timeout > 0) {  // test hook: exercise the recovery path
                    --ctx->inject_chain_timeout;
                    cs = ACSFIT_E_TIMEOUT;
                }
                if (cs == ACSFIT_E_TIMEOUT) {
                    CUDA_TRY(cudaStreamSynchronize(ctx->side));
                    CUDA_TRY(cudaMemcpyAsync(used, used_backup, sizeof(double) * (size_t)N * D, cudaMemcpyDeviceToDevice, st));
                    ctx->overlap = false;
                    ++ctx->chain_fallbacks;
                    chained = false;
                    reset_stats(ctx);
                } else if (cs != ACSFIT_OK) {
                    return cs;
                }
                if (chained) {
                    // pending pods in list order: their feasible positions, pod numbers and first-pass bins
                    TRY(compact(ctx, NegPred{placed_f}, F, nullptr, j_of_p, block_counts, total_dev, &Pn, st));
                    if (Pn > 0) {
                        gather_i32_kernel<<<grid_for(ctx, Pn, 256), 256, 0, st>>>(list_f, j_of_p, Pn, list_p);
                        gather_i32_kernel<<<grid_for(ctx, Pn, 256), 256, 0, st>>>(bins_f, j_of_p, Pn, cur_bin_p);
                        ctx->launches += 2;
                    }
                    pre.pool = t0;
                    pre.cur_bin = cur_bin_p;
                    pre.bins_covered = covered;
                    pre.evals = bev;
                }
            }
        }
        if (!chained) {
            TRY(first_fit_impl(ctx, req, list_f, F, D, cap_type, node_type, used, N, placed_f, evals_dev + 1, st,
                               pod_class, node_match));
            TRY(compact(ctx, NegPred{placed_f}, F, list_f, list_p, block_counts, total_dev, &Pn, st));
        }
        scatter_i32_kernel<<<grid_for(ctx, F, 256), 256, 0, st>>>(list_f, placed_f, F, out_placed);
        ++ctx->launches;
    }
    unsigned long long ev[2] = {0, 0};
    CUDA_TRY(cudaMemcpyAsync(ev, evals_dev, sizeof ev, cudaMemcpyDeviceToHost, st));
    CUDA_TRY(cudaStreamSynchronize(st));
    decisions += ev[0] + ev[1];
    // scale(): fulfill_pending only when something is pending (cluster.py:214-215)
    int64_t unaccounted = 0;
    for (int t = 0; t < T; ++t) {
        out_new_size[t] = pool_actual[t];
        out_units_needed[t] = -1;
        out_bins_opened[t] = 0;
    }
    if (Pn > 0) {
        uint64_t fe = 0;
        TRY(fulfill_impl(ctx, req, list_p, Pn, Pn, D, unit_ordered_host, pool_actual, pool_max, pool_ignored, T,
                         over_provision, out_new_size, out_units_needed, out_bins_opened, acc_p, bin_p, &unaccounted,
                         &fe, st, chained ? &pre : nullptr, pod_class, sel ? sel->pool_match_ordered : nullptr));
        decisions += fe;
        scatter_i32_kernel<<<grid_for(ctx, Pn, 256), 256, 0, st>>>(list_p, acc_p, Pn, out_acc_pool);
        ++ctx->launches;
        CUDA_TRY(cudaGetLastError());
    }
    out_counters[0] = (uint64_t)F;
    out_counters[1] = (uint64_t)Pn;
    out_counters[2] = (uint64_t)unaccounted;
    out_counters[3] = decisions;
    return ACSFIT_OK;
}

static acsfit_status scale_up_check(acsfit_ctx *ctx, const void *req, int64_t P, int D, const void *unit_all,
                                    const void *unit_ordered, const void *pa, const void *pm, const void *pi, int T,
                                    const void *cap_type, const void *node_type, const void *used, int64_t N,
                                    const void *o1, const void *o2, const void *o3, const void *o4, const void *o5,
                                    const void *o6, const void *o7)
{
    if (P < 0 || N < 0 || P > INT32_MAX || N > INT32_MAX || T < 0 || T > ACSFIT_MAX_POOLS ||
        (P > 0 && (!req || !o1 || !o2 || !o6)) || (T > 0 && (!unit_all || !unit_ordered || !pa || !pm || !pi || !o3 || !o4 || !o5)) ||
        (N > 0 && (!cap_type || !node_type || !used)) || !o7)
        return fail(ctx, ACSFIT_E_INVALID, "scale_up: bad arguments");
    if (!pipeline_dims_ok(D))
        return fail(ctx, ACSFIT_E_INVALID, "scale_up: D=%d, need 2/4/8/16 (zero columns are neutral)", D);
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_scale_up(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                         const double *unit_all, const double *unit_ordered,
                                         const int32_t *pool_actual, const int32_t *pool_max,
                                         const uint8_t *pool_ignored, int T, int64_t over_provision,
                                         const double *cap_type, const int32_t *node_type, double *used_inout,
                                         int64_t N, uint8_t *out_feasible, int32_t *out_placed,
                                         int64_t *out_new_size, int64_t *out_units_needed, int64_t *out_bins_opened,
                                         int32_t *out_acc_pool, uint64_t *out_counters, acsfit_stream_t stream)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(scale_up_check(ctx, req, P, D, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, T, cap_type,
                       node_type, used_inout, N, out_feasible, out_placed, out_new_size, out_units_needed,
                       out_bins_opened, out_acc_pool, out_counters));
    TRY(check_req_aligned(ctx, req, "scale_up"));
    reset_stats(ctx);
    TRY(arena_reserve(ctx, scale_up_scratch(ctx, P, N, T, D), st));
    ctx->arena_off = 0;
    return scale_up_impl(ctx, req, P, D, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, T,
                         over_provision, cap_type, node_type, used_inout, N, out_feasible, out_placed, out_new_size,
                         out_units_needed, out_bins_opened, out_acc_pool, out_counters, st);
}

// ---------------------------------------------------------------------------------------------
// node selectors (include/acsfit.h, acsfit_selectors): the *_sel entry points
// ---------------------------------------------------------------------------------------------
enum { kSelNodes = 1, kSelPoolsAll = 2, kSelPoolsOrdered = 4 };

// host-side checks of the fields `need` names (pod_class is always needed when there are rows)
static acsfit_status check_selectors_host(acsfit_ctx *ctx, const acsfit_selectors *sel, int64_t rows, int64_t N, int T,
                                          int need, const char *what)
{
    if (!sel) return fail(ctx, ACSFIT_E_INVALID, "%s: selectors missing", what);
    if (ctx->world > 1) return fail(ctx, ACSFIT_E_INVALID, "%s: node selectors are not supported in cluster mode", what);
    if (sel->classes < 1 || sel->classes > ACSFIT_MAX_CLASSES)
        return fail(ctx, ACSFIT_E_INVALID, "%s: %d selector classes, need 1..%d", what, sel->classes, ACSFIT_MAX_CLASSES);
    if ((rows > 0 && !sel->pod_class) || ((need & kSelNodes) && N > 0 && !sel->node_match) ||
        ((need & kSelPoolsAll) && T > 0 && !sel->pool_match_all) ||
        ((need & kSelPoolsOrdered) && T > 0 && !sel->pool_match_ordered))
        return fail(ctx, ACSFIT_E_INVALID, "%s: selector field missing", what);
    for (int t = 0; t < T; ++t)  // class 0 (no selector) matches every pool
        if (((need & kSelPoolsAll) && !(sel->pool_match_all[t] & 1u)) ||
            ((need & kSelPoolsOrdered) && !(sel->pool_match_ordered[t] & 1u)))
            return fail(ctx, ACSFIT_E_INVALID, "%s: bit 0 (no selector) must be set in every pool mask", what);
    return ACSFIT_OK;
}

// device-side checks: every class < sel->classes (the kernels shift a 64-bit mask by it) and, when node masks are
// given, bit 0 (no selector) set in each of them
static acsfit_status check_classes(acsfit_ctx *ctx, const uint8_t *pod_class, int64_t rows, int classes, int *flag_dev,
                                   cudaStream_t st, const char *what, const uint64_t *node_match = nullptr,
                                   int64_t N = 0)
{
    if (rows <= 0 && N <= 0) return ACSFIT_OK;
    CUDA_TRY(cudaMemsetAsync(flag_dev, 0, sizeof(int), st));
    if (rows > 0) {
        class_check_kernel<<<grid_for(ctx, rows, 256), 256, 0, st>>>(pod_class, rows, classes, flag_dev);
        ++ctx->launches;
    }
    if (node_match && N > 0) {
        node_mask_check_kernel<<<grid_for(ctx, N, 256), 256, 0, st>>>(
            reinterpret_cast<const unsigned long long *>(node_match), N, flag_dev);
        ++ctx->launches;
    }
    int flag = 0;
    TRY(flag_to_host(ctx, flag_dev, st, &flag));
    CUDA_TRY(cudaGetLastError());
    if (flag & 1) return fail(ctx, ACSFIT_E_INVALID, "%s: a pod_class is >= classes (%d)", what, classes);
    if (flag & 2) return fail(ctx, ACSFIT_E_INVALID, "%s: bit 0 (no selector) must be set in every node mask", what);
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_feasible_mask_sel(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                                  const double *unit, int T, const acsfit_selectors *sel,
                                                  uint8_t *out_mask, uint64_t *out_evals, acsfit_stream_t stream)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    if (P < 0 || T < 0 || T > ACSFIT_MAX_POOLS || (P > 0 && (!req || !out_mask)) || (T > 0 && !unit))
        return fail(ctx, ACSFIT_E_INVALID, "feasible_mask_sel: bad arguments");
    TRY(check_selectors_host(ctx, sel, P, 0, T, kSelPoolsAll, "feasible_mask_sel"));
    if (out_evals) CUDA_TRY(cudaMemsetAsync(out_evals, 0, sizeof(uint64_t), st));
    if (P == 0) return ACSFIT_OK;
    TRY(arena_reserve(ctx, sizeof(uint64_t) * (size_t)T + 4096, st));
    ctx->arena_off = 0;
    TAKE(flag, int, 1);
    TAKE(match_dev, unsigned long long, T);
    TRY(check_classes(ctx, sel->pod_class, P, sel->classes, flag, st, "feasible_mask_sel"));
    if (T > 0) CUDA_TRY(cudaMemcpyAsync(match_dev, sel->pool_match_all, sizeof(uint64_t) * T, cudaMemcpyHostToDevice, st));
    feasible_mask_sel_kernel<<<grid_for(ctx, P, 256), 256, (sizeof(double) * D + sizeof(uint64_t)) * std::max(1, T), st>>>(
        req, P, D, unit, match_dev, T, sel->pod_class, out_mask, reinterpret_cast<unsigned long long *>(out_evals));
    ++ctx->launches;
    CUDA_TRY(cudaGetLastError());
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_first_fit_nodes_sel(acsfit_ctx *ctx, const double *req, int64_t req_rows,
                                                    const int32_t *pod_idx, int64_t P, int D, const double *cap_type,
                                                    const int32_t *node_type, double *used_inout, int64_t N,
                                                    const acsfit_selectors *sel, int32_t *out_placed,
                                                    uint64_t *out_decisions, acsfit_stream_t stream)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(check_first_fit_args(ctx, "first_fit_nodes_sel", req, req_rows, pod_idx, P, D, cap_type, node_type, used_inout,
                             N, out_placed));
    TRY(check_selectors_host(ctx, sel, req_rows, N, 0, kSelNodes, "first_fit_nodes_sel"));
    reset_stats(ctx);
    TRY(arena_reserve(ctx, first_fit_scratch(ctx, P, N) + rank_scratch(req_rows, D) + 1024, st));
    ctx->arena_off = 0;
    TAKE(flag, int, 1);
    TRY(check_domain(ctx, req, req_rows * D, flag, st, "req"));
    TRY(check_classes(ctx, sel->pod_class, req_rows, sel->classes, flag, st, "first_fit_nodes_sel", sel->node_match, N));
    if (P > 0 && N > 0) TRY(build_ranks(ctx, req, req_rows, D, st));
    return first_fit_impl(ctx, req, pod_idx, P, D, cap_type, node_type, used_inout, N, out_placed,
                          reinterpret_cast<unsigned long long *>(out_decisions), st, sel->pod_class,
                          reinterpret_cast<const unsigned long long *>(sel->node_match));
}

extern "C" acsfit_status acsfit_fulfill_pending_sel(acsfit_ctx *ctx, const double *req, int64_t Pp,
                                                    int64_t num_listed, int D, const double *unit,
                                                    const int32_t *pool_actual, const int32_t *pool_max,
                                                    const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                    const acsfit_selectors *sel, int64_t *out_new_size,
                                                    int64_t *out_units_needed, int64_t *out_bins_opened,
                                                    int32_t *out_acc_pool, int32_t *out_bin_of,
                                                    int64_t *out_unaccounted, uint64_t *out_evals,
                                                    acsfit_stream_t stream)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(check_fulfill_args(ctx, "fulfill_pending_sel", req, Pp, num_listed, D, unit, pool_actual, pool_max,
                           pool_ignored, T, out_new_size, out_units_needed, out_bins_opened, out_acc_pool, out_bin_of,
                           out_unaccounted));
    TRY(check_selectors_host(ctx, sel, Pp, 0, T, kSelPoolsOrdered, "fulfill_pending_sel"));
    reset_stats(ctx);
    TRY(arena_reserve(ctx, fulfill_scratch(Pp, T, D) + rank_scratch(Pp, D) + 1024, st));
    ctx->arena_off = 0;
    TAKE(flag, int, 1);
    TRY(check_domain(ctx, req, Pp * D, flag, st, "req"));
    TRY(check_classes(ctx, sel->pod_class, Pp, sel->classes, flag, st, "fulfill_pending_sel"));
    TRY(build_ranks(ctx, req, Pp, D, st));
    return fulfill_impl(ctx, req, nullptr, Pp, num_listed, D, unit, pool_actual, pool_max, pool_ignored, T,
                        over_provision, out_new_size, out_units_needed, out_bins_opened, out_acc_pool, out_bin_of,
                        out_unaccounted, out_evals, st, nullptr, sel->pod_class, sel->pool_match_ordered);
}

extern "C" acsfit_status acsfit_scale_up_sel(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                             const double *unit_all, const double *unit_ordered,
                                             const int32_t *pool_actual, const int32_t *pool_max,
                                             const uint8_t *pool_ignored, int T, int64_t over_provision,
                                             const double *cap_type, const int32_t *node_type, double *used_inout,
                                             int64_t N, const acsfit_selectors *sel, uint8_t *out_feasible,
                                             int32_t *out_placed, int64_t *out_new_size, int64_t *out_units_needed,
                                             int64_t *out_bins_opened, int32_t *out_acc_pool,
                                             uint64_t *out_counters, acsfit_stream_t stream)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(scale_up_check(ctx, req, P, D, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, T, cap_type,
                       node_type, used_inout, N, out_feasible, out_placed, out_new_size, out_units_needed,
                       out_bins_opened, out_acc_pool, out_counters));
    TRY(check_req_aligned(ctx, req, "scale_up_sel"));
    TRY(check_selectors_host(ctx, sel, P, N, T, kSelNodes | kSelPoolsAll | kSelPoolsOrdered, "scale_up_sel"));
    reset_stats(ctx);
    TRY(arena_reserve(ctx, scale_up_scratch(ctx, P, N, T, D) + sizeof(uint64_t) * (size_t)T + 1024, st));
    ctx->arena_off = 0;
    TAKE(flag, int, 1);
    TRY(check_classes(ctx, sel->pod_class, P, sel->classes, flag, st, "scale_up_sel", sel->node_match, N));
    return scale_up_impl(ctx, req, P, D, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, T,
                         over_provision, cap_type, node_type, used_inout, N, out_feasible, out_placed, out_new_size,
                         out_units_needed, out_bins_opened, out_acc_pool, out_counters, st, sel);
}

// ---------------------------------------------------------------------------------------------
// required pod anti-affinity (include/acsfit.h, acsfit_anti_affinity): the *_aa entry points
// ---------------------------------------------------------------------------------------------
static acsfit_status check_aa_host(acsfit_ctx *ctx, const acsfit_anti_affinity *aa, int64_t rows, int64_t N,
                                   const char *what)
{
    if (!aa) return fail(ctx, ACSFIT_E_INVALID, "%s: anti-affinity masks missing", what);
    if (ctx->world > 1) return fail(ctx, ACSFIT_E_INVALID, "%s: pod anti-affinity is not supported in cluster mode", what);
    if ((rows > 0 && (!aa->pod_carries || !aa->pod_matches)) || (N > 0 && (!aa->node_carries || !aa->node_matches)))
        return fail(ctx, ACSFIT_E_INVALID, "%s: anti-affinity field missing", what);
    return ACSFIT_OK;
}

// pod affinity (include/acsfit.h, acsfit_pod_affinity): the *_pa entry points share the *_aa ones' implementation
static acsfit_status check_pa_host(acsfit_ctx *ctx, const acsfit_pod_affinity *pa, int64_t rows, int64_t N,
                                   int *flag_dev, cudaStream_t st, const char *what)
{
    if (!pa) return fail(ctx, ACSFIT_E_INVALID, "%s: pod-affinity masks missing", what);
    if (ctx->world > 1) return fail(ctx, ACSFIT_E_INVALID, "%s: pod affinity is not supported in cluster mode", what);
    if ((rows > 0 && (!pa->pod_requires || !pa->pod_self || !pa->pod_matches)) || (N > 0 && !pa->node_has))
        return fail(ctx, ACSFIT_E_INVALID, "%s: pod-affinity field missing", what);
    if (rows <= 0) return ACSFIT_OK;
    CUDA_TRY(cudaMemsetAsync(flag_dev, 0, sizeof(int), st));
    pa_check_kernel<<<grid_for(ctx, rows, 256), 256, 0, st>>>(reinterpret_cast<const unsigned long long *>(pa->pod_requires),
                                                              reinterpret_cast<const unsigned long long *>(pa->pod_self),
                                                              rows, flag_dev);
    ++ctx->launches;
    int flag = 0;
    TRY(flag_to_host(ctx, flag_dev, st, &flag));
    CUDA_TRY(cudaGetLastError());
    if (flag & 4) return fail(ctx, ACSFIT_E_INVALID, "%s: a pod_requires has more than one bit, or pod_self is not inside it", what);
    return ACSFIT_OK;
}

// zero anti-affinity masks for a pod-affinity call without `aa` (rows pods, N nodes), from the arena
static acsfit_status zero_aa(acsfit_ctx *ctx, int64_t rows, int64_t N, acsfit_anti_affinity *out, cudaStream_t st)
{
    TAKE(z, uint64_t, (size_t)2 * rows + (size_t)2 * N);
    CUDA_TRY(cudaMemsetAsync(z, 0, sizeof(uint64_t) * std::max<size_t>(1, (size_t)2 * rows + (size_t)2 * N), st));
    *out = {z, z + rows, z + 2 * rows, z + 2 * rows + N};
    return ACSFIT_OK;
}

// topology spread (include/acsfit.h, acsfit_topology_spread): the *_ts entry points share the *_pa ones'
// implementation.  rows: request rows, N: nodes (0: fulfill, which reads neither counts nor domains)
static acsfit_status check_ts_host(acsfit_ctx *ctx, const acsfit_topology_spread *ts, int64_t rows, int64_t N,
                                   int *flag_dev, cudaStream_t st, const char *what)
{
    if (!ts) return fail(ctx, ACSFIT_E_INVALID, "%s: topology-spread arrays missing", what);
    if (ctx->world > 1) return fail(ctx, ACSFIT_E_INVALID, "%s: topology spread is not supported in cluster mode", what);
    if (ts->keys < 0 || ts->keys > ACSFIT_MAX_TS_KEYS)
        return fail(ctx, ACSFIT_E_INVALID, "%s: %d spread keys, at most %d", what, ts->keys, ACSFIT_MAX_TS_KEYS);
    if ((rows > 0 && (!ts->pod_key || !ts->pod_skew || !ts->pod_matches)) ||
        (N > 0 && ts->keys > 0 && (!ts->node_count || !ts->node_domain)) || (N > 0 && ts->keys > 0 && !ts->floor))
        return fail(ctx, ACSFIT_E_INVALID, "%s: topology-spread field missing", what);
    for (int k = 0; N > 0 && k < ts->keys; ++k)
        if (ts->floor[k] < 0) return fail(ctx, ACSFIT_E_INVALID, "%s: floor[%d] = %d is negative", what, k, ts->floor[k]);
    const int64_t counts = N > 0 ? N * ts->keys : 0;
    if (rows <= 0 && counts <= 0) return ACSFIT_OK;
    CUDA_TRY(cudaMemsetAsync(flag_dev, 0, sizeof(int), st));
    ts_check_kernel<<<grid_for(ctx, std::max(rows, counts), 256), 256, 0, st>>>(
        ts->pod_key, ts->pod_skew, reinterpret_cast<const unsigned long long *>(ts->pod_matches), rows, ts->keys,
        ts->node_count, counts, flag_dev);
    ++ctx->launches;
    int flag = 0;
    TRY(flag_to_host(ctx, flag_dev, st, &flag));
    CUDA_TRY(cudaGetLastError());
    if (flag & 8)
        return fail(ctx, ACSFIT_E_INVALID, "%s: a pod_key is >= keys, a pod_skew is negative, or a pod_matches names a "
                    "key >= keys", what);
    if (flag & 16) return fail(ctx, ACSFIT_E_INVALID, "%s: a node count is negative", what);
    return ACSFIT_OK;
}

// zero pod-affinity masks for a topology-spread call without `pa` (rows pods, N nodes), from the arena
static acsfit_status zero_pa(acsfit_ctx *ctx, int64_t rows, int64_t N, acsfit_pod_affinity *out, cudaStream_t st)
{
    TAKE(z, uint64_t, (size_t)3 * rows + (size_t)N);
    CUDA_TRY(cudaMemsetAsync(z, 0, sizeof(uint64_t) * std::max<size_t>(1, (size_t)3 * rows + (size_t)N), st));
    *out = {z, z + rows, z + 2 * rows, z + 3 * rows};
    return ACSFIT_OK;
}

// pa == nullptr and ts == nullptr: the *_aa form (aa required); otherwise the *_pa / *_ts form (aa, and for *_ts pa,
// may be NULL)
static acsfit_status first_fit_nodes_aa_pa(acsfit_ctx *ctx, const double *req, int64_t req_rows, const int32_t *pod_idx,
                                           int64_t P, int D, const double *cap_type, const int32_t *node_type,
                                           double *used_inout, int64_t N, const acsfit_selectors *sel,
                                           const acsfit_anti_affinity *aa, const acsfit_pod_affinity *pa,
                                           int32_t *out_placed, uint64_t *out_decisions, acsfit_stream_t stream,
                                           const char *what, const acsfit_topology_spread *ts = nullptr)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(check_first_fit_args(ctx, what, req, req_rows, pod_idx, P, D, cap_type, node_type, used_inout, N, out_placed));
    if ((!pa && !ts) || aa) TRY(check_aa_host(ctx, aa, req_rows, N, what));
    if (sel) TRY(check_selectors_host(ctx, sel, req_rows, N, 0, kSelNodes, what));
    if (ts && ctx->world > 1) return fail(ctx, ACSFIT_E_INVALID, "%s: topology spread is not supported in cluster mode", what);
    reset_stats(ctx);
    // without selectors: class 0 for every row and all-ones node masks, from the arena
    const size_t trivial = sel ? 0 : align_up((size_t)req_rows, 256) + sizeof(uint64_t) * (size_t)N + 512;
    // pod affinity, which topology spread runs on too (with zero masks without `pa`): zero anti-affinity masks
    // without `aa`, the needs, and the saved node state of a rerun
    const size_t pa_bytes = !pa && !ts ? 0 : (aa ? 0 : sizeof(uint64_t) * 2 * (size_t)(req_rows + N) + 256) +
                                                 sizeof(uint64_t) * (size_t)P + sizeof(double) * (size_t)N * D +
                                                 sizeof(uint64_t) * 3 * (size_t)N + 2048;
    // topology spread: zero pod-affinity masks without `pa`, the limits, the saved counts of a rerun
    const size_t ts_bytes = !ts ? 0 : (pa ? 0 : sizeof(uint64_t) * (size_t)(3 * req_rows + N) + 256) +
                                          ts_scratch(P) + sizeof(int32_t) * (size_t)N * std::max(0, ts->keys) + 256;
    TRY(arena_reserve(ctx, first_fit_scratch(ctx, P, N) + rank_scratch(req_rows, D) + trivial + pa_bytes + ts_bytes + 1024, st));
    ctx->arena_off = 0;
    TAKE(flag, int, 1);
    TRY(check_domain(ctx, req, req_rows * D, flag, st, "req"));
    if (pa) TRY(check_pa_host(ctx, pa, req_rows, N, flag, st, what));
    if (ts) TRY(check_ts_host(ctx, ts, req_rows, N, flag, st, what));
    acsfit_pod_affinity zero_p;
    if (ts && !pa) {
        TRY(zero_pa(ctx, req_rows, N, &zero_p, st));
        pa = &zero_p;
    }
    acsfit_anti_affinity zero;
    if (pa && !aa) {
        TRY(zero_aa(ctx, req_rows, N, &zero, st));
        aa = &zero;
    }
    const uint8_t *pod_class;
    const unsigned long long *node_match;
    if (sel) {
        TRY(check_classes(ctx, sel->pod_class, req_rows, sel->classes, flag, st, what, sel->node_match, N));
        pod_class = sel->pod_class;
        node_match = reinterpret_cast<const unsigned long long *>(sel->node_match);
    } else {
        TAKE(cls0, uint8_t, req_rows);
        TAKE(all, unsigned long long, N);
        if (req_rows > 0) CUDA_TRY(cudaMemsetAsync(cls0, 0, (size_t)req_rows, st));
        if (N > 0) CUDA_TRY(cudaMemsetAsync(all, 0xFF, sizeof(unsigned long long) * (size_t)N, st));
        pod_class = cls0;
        node_match = all;
    }
    if (P > 0 && N > 0) TRY(build_ranks(ctx, req, req_rows, D, st));
    return first_fit_impl(ctx, req, pod_idx, P, D, cap_type, node_type, used_inout, N, out_placed,
                          reinterpret_cast<unsigned long long *>(out_decisions), st, pod_class, node_match, aa, pa, ts);
}

extern "C" acsfit_status acsfit_first_fit_nodes_aa(acsfit_ctx *ctx, const double *req, int64_t req_rows,
                                                   const int32_t *pod_idx, int64_t P, int D, const double *cap_type,
                                                   const int32_t *node_type, double *used_inout, int64_t N,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   int32_t *out_placed, uint64_t *out_decisions,
                                                   acsfit_stream_t stream)
{
    return first_fit_nodes_aa_pa(ctx, req, req_rows, pod_idx, P, D, cap_type, node_type, used_inout, N, sel, aa,
                                 nullptr, out_placed, out_decisions, stream, "first_fit_nodes_aa");
}

extern "C" acsfit_status acsfit_first_fit_nodes_pa(acsfit_ctx *ctx, const double *req, int64_t req_rows,
                                                   const int32_t *pod_idx, int64_t P, int D, const double *cap_type,
                                                   const int32_t *node_type, double *used_inout, int64_t N,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   const acsfit_pod_affinity *pa, int32_t *out_placed,
                                                   uint64_t *out_decisions, acsfit_stream_t stream)
{
    if (ctx && !pa) return fail(ctx, ACSFIT_E_INVALID, "first_fit_nodes_pa: pod-affinity masks missing");
    return first_fit_nodes_aa_pa(ctx, req, req_rows, pod_idx, P, D, cap_type, node_type, used_inout, N, sel, aa, pa,
                                 out_placed, out_decisions, stream, "first_fit_nodes_pa");
}

static acsfit_status fulfill_pending_aa_pa(acsfit_ctx *ctx, const double *req, int64_t Pp, int64_t num_listed, int D,
                                           const double *unit, const int32_t *pool_actual, const int32_t *pool_max,
                                           const uint8_t *pool_ignored, int T, int64_t over_provision,
                                           const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                           const acsfit_pod_affinity *pa, uint64_t present, int64_t *out_new_size,
                                           int64_t *out_units_needed, int64_t *out_bins_opened, int32_t *out_acc_pool,
                                           int32_t *out_bin_of, int64_t *out_unaccounted, uint64_t *out_evals,
                                           acsfit_stream_t stream, const char *what,
                                           const acsfit_topology_spread *ts = nullptr)
{
    TRY(enter(ctx, D));
    cudaStream_t st = (cudaStream_t)stream;
    TRY(check_fulfill_args(ctx, what, req, Pp, num_listed, D, unit, pool_actual, pool_max, pool_ignored, T,
                           out_new_size, out_units_needed, out_bins_opened, out_acc_pool, out_bin_of,
                           out_unaccounted));
    if ((!pa && !ts) || aa) TRY(check_aa_host(ctx, aa, Pp, 0, what));
    if (sel) TRY(check_selectors_host(ctx, sel, Pp, 0, T, kSelPoolsOrdered, what));
    if (ts && ctx->world > 1) return fail(ctx, ACSFIT_E_INVALID, "%s: topology spread is not supported in cluster mode", what);
    reset_stats(ctx);
    const size_t pa_bytes = !pa && !ts ? 0 : (aa ? 0 : sizeof(uint64_t) * 2 * (size_t)Pp + 256) + sizeof(uint64_t) * (size_t)Pp + 2048;
    const size_t ts_bytes = !ts ? 0 : (pa ? 0 : sizeof(uint64_t) * 3 * (size_t)Pp + 256) + ts_scratch(Pp);
    TRY(arena_reserve(ctx, fulfill_scratch(Pp, T, D) + rank_scratch(Pp, D) + pa_bytes + ts_bytes + 1024, st));
    ctx->arena_off = 0;
    TAKE(flag, int, 1);
    TRY(check_domain(ctx, req, Pp * D, flag, st, "req"));
    if (pa) TRY(check_pa_host(ctx, pa, Pp, 0, flag, st, what));
    if (ts) TRY(check_ts_host(ctx, ts, Pp, 0, flag, st, what));
    acsfit_pod_affinity zero_p;
    if (ts && !pa) {
        TRY(zero_pa(ctx, Pp, 0, &zero_p, st));
        pa = &zero_p;
    }
    acsfit_anti_affinity zero;
    if (pa && !aa) {
        TRY(zero_aa(ctx, Pp, 0, &zero, st));
        aa = &zero;
    }
    if (sel) TRY(check_classes(ctx, sel->pod_class, Pp, sel->classes, flag, st, what));
    TRY(build_ranks(ctx, req, Pp, D, st));
    return fulfill_impl(ctx, req, nullptr, Pp, num_listed, D, unit, pool_actual, pool_max, pool_ignored, T,
                        over_provision, out_new_size, out_units_needed, out_bins_opened, out_acc_pool, out_bin_of,
                        out_unaccounted, out_evals, st, nullptr, sel ? sel->pod_class : nullptr,
                        sel ? sel->pool_match_ordered : nullptr, aa, pa, present, ts);
}

extern "C" acsfit_status acsfit_fulfill_pending_aa(acsfit_ctx *ctx, const double *req, int64_t Pp,
                                                   int64_t num_listed, int D, const double *unit,
                                                   const int32_t *pool_actual, const int32_t *pool_max,
                                                   const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   int64_t *out_new_size, int64_t *out_units_needed,
                                                   int64_t *out_bins_opened, int32_t *out_acc_pool,
                                                   int32_t *out_bin_of, int64_t *out_unaccounted,
                                                   uint64_t *out_evals, acsfit_stream_t stream)
{
    return fulfill_pending_aa_pa(ctx, req, Pp, num_listed, D, unit, pool_actual, pool_max, pool_ignored, T,
                                 over_provision, sel, aa, nullptr, 0, out_new_size, out_units_needed, out_bins_opened,
                                 out_acc_pool, out_bin_of, out_unaccounted, out_evals, stream, "fulfill_pending_aa");
}

extern "C" acsfit_status acsfit_fulfill_pending_pa(acsfit_ctx *ctx, const double *req, int64_t Pp,
                                                   int64_t num_listed, int D, const double *unit,
                                                   const int32_t *pool_actual, const int32_t *pool_max,
                                                   const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   const acsfit_pod_affinity *pa, uint64_t present,
                                                   int64_t *out_new_size, int64_t *out_units_needed,
                                                   int64_t *out_bins_opened, int32_t *out_acc_pool,
                                                   int32_t *out_bin_of, int64_t *out_unaccounted,
                                                   uint64_t *out_evals, acsfit_stream_t stream)
{
    if (ctx && !pa) return fail(ctx, ACSFIT_E_INVALID, "fulfill_pending_pa: pod-affinity masks missing");
    return fulfill_pending_aa_pa(ctx, req, Pp, num_listed, D, unit, pool_actual, pool_max, pool_ignored, T,
                                 over_provision, sel, aa, pa, present, out_new_size, out_units_needed, out_bins_opened,
                                 out_acc_pool, out_bin_of, out_unaccounted, out_evals, stream, "fulfill_pending_pa");
}

extern "C" acsfit_status acsfit_first_fit_nodes_ts(acsfit_ctx *ctx, const double *req, int64_t req_rows,
                                                   const int32_t *pod_idx, int64_t P, int D, const double *cap_type,
                                                   const int32_t *node_type, double *used_inout, int64_t N,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   const acsfit_pod_affinity *pa, const acsfit_topology_spread *ts,
                                                   int32_t *out_placed, uint64_t *out_decisions, acsfit_stream_t stream)
{
    if (ctx && !ts) return fail(ctx, ACSFIT_E_INVALID, "first_fit_nodes_ts: topology-spread arrays missing");
    return first_fit_nodes_aa_pa(ctx, req, req_rows, pod_idx, P, D, cap_type, node_type, used_inout, N, sel, aa, pa,
                                 out_placed, out_decisions, stream, "first_fit_nodes_ts", ts);
}

extern "C" acsfit_status acsfit_fulfill_pending_ts(acsfit_ctx *ctx, const double *req, int64_t Pp,
                                                   int64_t num_listed, int D, const double *unit,
                                                   const int32_t *pool_actual, const int32_t *pool_max,
                                                   const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                   const acsfit_selectors *sel, const acsfit_anti_affinity *aa,
                                                   const acsfit_pod_affinity *pa, uint64_t present,
                                                   const acsfit_topology_spread *ts, int64_t *out_new_size,
                                                   int64_t *out_units_needed, int64_t *out_bins_opened,
                                                   int32_t *out_acc_pool, int32_t *out_bin_of,
                                                   int64_t *out_unaccounted, uint64_t *out_evals,
                                                   acsfit_stream_t stream)
{
    if (ctx && !ts) return fail(ctx, ACSFIT_E_INVALID, "fulfill_pending_ts: topology-spread arrays missing");
    return fulfill_pending_aa_pa(ctx, req, Pp, num_listed, D, unit, pool_actual, pool_max, pool_ignored, T,
                                 over_provision, sel, aa, pa, present, out_new_size, out_units_needed, out_bins_opened,
                                 out_acc_pool, out_bin_of, out_unaccounted, out_evals, stream, "fulfill_pending_ts", ts);
}

// ---------------------------------------------------------------------------------------------
// host-buffer entry points
// ---------------------------------------------------------------------------------------------
static acsfit_status hbuf_reserve(acsfit_ctx *ctx, size_t bytes)
{
    ctx->hbuf_off = 0;
    if (bytes <= ctx->hbuf_cap) return ACSFIT_OK;
    CUDA_TRY(cudaDeviceSynchronize());
    if (ctx->hbuf) CUDA_TRY(cudaFree(ctx->hbuf));
    ctx->hbuf = nullptr;
    ctx->hbuf_cap = 0;
    const size_t cap = align_up(bytes + bytes / 4, 1 << 20);
    CUDA_TRY(cudaMalloc(&ctx->hbuf, cap));
    ctx->hbuf_cap = cap;
    return ACSFIT_OK;
}

template <typename T>
static T *hbuf_take(acsfit_ctx *ctx, size_t count)
{
    const size_t off = align_up(ctx->hbuf_off, 256);
    const size_t bytes = sizeof(T) * std::max<size_t>(count, 1);
    if (off + bytes > ctx->hbuf_cap) return nullptr;
    ctx->hbuf_off = off + bytes;
    return reinterpret_cast<T *>(ctx->hbuf + off);
}

#define HTAKE(var, T, count)                                                                \
    T *var = hbuf_take<T>(ctx, (count));                                                    \
    if (!var) return fail(ctx, ACSFIT_E_NOMEM, "host-entry device buffer too small for %s", #var)

#define H2D(dst, src, bytes)                                                                \
    do {                                                                                    \
        if ((bytes) > 0) CUDA_TRY(cudaMemcpyAsync((dst), (src), (bytes), cudaMemcpyHostToDevice, st)); \
    } while (0)
#define D2H(dst, src, bytes)                                                                \
    do {                                                                                    \
        if ((bytes) > 0) CUDA_TRY(cudaMemcpyAsync((dst), (src), (bytes), cudaMemcpyDeviceToHost, st)); \
    } while (0)

extern "C" acsfit_status acsfit_scale_up_host(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                              const double *unit_all, const double *unit_ordered,
                                              const int32_t *pool_actual, const int32_t *pool_max,
                                              const uint8_t *pool_ignored, int T, int64_t over_provision,
                                              const double *cap_type, int K, const int32_t *node_type,
                                              double *used_inout, int64_t N, uint8_t *out_feasible,
                                              int32_t *out_placed, int64_t *out_new_size,
                                              int64_t *out_units_needed, int64_t *out_bins_opened,
                                              int32_t *out_acc_pool, uint64_t *out_counters)
{
    TRY(enter(ctx, D));
    cudaStream_t st = nullptr;
    if (K < 0) return fail(ctx, ACSFIT_E_INVALID, "scale_up_host: K < 0");
    TRY(scale_up_check(ctx, req, P, D, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, T, cap_type,
                       node_type, used_inout, N, out_feasible, out_placed, out_new_size, out_units_needed,
                       out_bins_opened, out_acc_pool, out_counters));
    for (int i = 0; i < K * D; ++i)
        if (!std::isfinite(cap_type[i])) return fail(ctx, ACSFIT_E_DOMAIN, "scale_up_host: non-finite capacity");
    reset_stats(ctx);
    const size_t bytes = sizeof(double) * ((size_t)P * D + (size_t)K * D + (size_t)N * D) +
                         sizeof(int32_t) * ((size_t)N + 2 * (size_t)P) + (size_t)P + 16 * 256;
    TRY(hbuf_reserve(ctx, bytes));
    HTAKE(d_req, double, (size_t)P * D);
    HTAKE(d_cap, double, (size_t)K * D);
    HTAKE(d_used, double, (size_t)N * D);
    HTAKE(d_type, int32_t, N);
    HTAKE(d_placed, int32_t, P);
    HTAKE(d_acc, int32_t, P);
    HTAKE(d_feas, uint8_t, P);
    H2D(d_req, req, sizeof(double) * (size_t)P * D);
    H2D(d_cap, cap_type, sizeof(double) * (size_t)K * D);
    H2D(d_used, used_inout, sizeof(double) * (size_t)N * D);
    H2D(d_type, node_type, sizeof(int32_t) * (size_t)N);
    TRY(arena_reserve(ctx, scale_up_scratch(ctx, P, N, T, D), st));
    ctx->arena_off = 0;
    TRY(scale_up_impl(ctx, d_req, P, D, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, T, over_provision,
                      d_cap, d_type, d_used, N, d_feas, d_placed, out_new_size, out_units_needed, out_bins_opened,
                      d_acc, out_counters, st));
    D2H(out_feasible, d_feas, (size_t)P);
    D2H(out_placed, d_placed, sizeof(int32_t) * (size_t)P);
    D2H(out_acc_pool, d_acc, sizeof(int32_t) * (size_t)P);
    D2H(used_inout, d_used, sizeof(double) * (size_t)N * D);
    CUDA_TRY(cudaStreamSynchronize(st));
    return ACSFIT_OK;
}

// the same with node selectors; sel->pod_class and sel->node_match are host pointers here
extern "C" acsfit_status acsfit_scale_up_sel_host(acsfit_ctx *ctx, const double *req, int64_t P, int D,
                                                  const double *unit_all, const double *unit_ordered,
                                                  const int32_t *pool_actual, const int32_t *pool_max,
                                                  const uint8_t *pool_ignored, int T, int64_t over_provision,
                                                  const double *cap_type, int K, const int32_t *node_type,
                                                  double *used_inout, int64_t N, const acsfit_selectors *sel,
                                                  uint8_t *out_feasible, int32_t *out_placed,
                                                  int64_t *out_new_size, int64_t *out_units_needed,
                                                  int64_t *out_bins_opened, int32_t *out_acc_pool,
                                                  uint64_t *out_counters)
{
    TRY(enter(ctx, D));
    cudaStream_t st = nullptr;
    if (K < 0) return fail(ctx, ACSFIT_E_INVALID, "scale_up_sel_host: K < 0");
    TRY(scale_up_check(ctx, req, P, D, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, T, cap_type,
                       node_type, used_inout, N, out_feasible, out_placed, out_new_size, out_units_needed,
                       out_bins_opened, out_acc_pool, out_counters));
    TRY(check_selectors_host(ctx, sel, P, N, T, kSelNodes | kSelPoolsAll | kSelPoolsOrdered, "scale_up_sel_host"));
    for (int i = 0; i < K * D; ++i)
        if (!std::isfinite(cap_type[i])) return fail(ctx, ACSFIT_E_DOMAIN, "scale_up_sel_host: non-finite capacity");
    reset_stats(ctx);
    const size_t bytes = sizeof(double) * ((size_t)P * D + (size_t)K * D + (size_t)N * D) +
                         sizeof(int32_t) * ((size_t)N + 2 * (size_t)P) + 2 * (size_t)P + sizeof(uint64_t) * (size_t)N +
                         16 * 256;
    TRY(hbuf_reserve(ctx, bytes));
    HTAKE(d_req, double, (size_t)P * D);
    HTAKE(d_cap, double, (size_t)K * D);
    HTAKE(d_used, double, (size_t)N * D);
    HTAKE(d_type, int32_t, N);
    HTAKE(d_placed, int32_t, P);
    HTAKE(d_acc, int32_t, P);
    HTAKE(d_feas, uint8_t, P);
    HTAKE(d_class, uint8_t, P);
    HTAKE(d_match, uint64_t, N);
    H2D(d_req, req, sizeof(double) * (size_t)P * D);
    H2D(d_cap, cap_type, sizeof(double) * (size_t)K * D);
    H2D(d_used, used_inout, sizeof(double) * (size_t)N * D);
    H2D(d_type, node_type, sizeof(int32_t) * (size_t)N);
    H2D(d_class, sel->pod_class, (size_t)P);
    H2D(d_match, sel->node_match, sizeof(uint64_t) * (size_t)N);
    acsfit_selectors dsel = *sel;
    dsel.pod_class = d_class;
    dsel.node_match = d_match;
    TRY(arena_reserve(ctx, scale_up_scratch(ctx, P, N, T, D) + sizeof(uint64_t) * (size_t)T + 1024, st));
    ctx->arena_off = 0;
    TAKE(flag, int, 1);
    TRY(check_classes(ctx, d_class, P, sel->classes, flag, st, "scale_up_sel_host", d_match, N));
    TRY(scale_up_impl(ctx, d_req, P, D, unit_all, unit_ordered, pool_actual, pool_max, pool_ignored, T, over_provision,
                      d_cap, d_type, d_used, N, d_feas, d_placed, out_new_size, out_units_needed, out_bins_opened,
                      d_acc, out_counters, st, &dsel));
    D2H(out_feasible, d_feas, (size_t)P);
    D2H(out_placed, d_placed, sizeof(int32_t) * (size_t)P);
    D2H(out_acc_pool, d_acc, sizeof(int32_t) * (size_t)P);
    D2H(used_inout, d_used, sizeof(double) * (size_t)N * D);
    CUDA_TRY(cudaStreamSynchronize(st));
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_occupancy_host(acsfit_ctx *ctx, const int64_t *row_ptr, const int32_t *run_idx,
                                               const double *req_run, int64_t R, int64_t N, int D, double *used_inout)
{
    TRY(enter(ctx, D));
    cudaStream_t st = nullptr;
    if (N < 0 || R < 0 || (N > 0 && (!row_ptr || !used_inout)) || (R > 0 && !req_run))
        return fail(ctx, ACSFIT_E_INVALID, "occupancy_host: bad arguments");
    if (N == 0) return ACSFIT_OK;
    const int64_t nnz = row_ptr[N];
    if (nnz < 0) return fail(ctx, ACSFIT_E_INVALID, "occupancy_host: bad CSR");
    TRY(hbuf_reserve(ctx, sizeof(int64_t) * ((size_t)N + 1) + sizeof(int32_t) * (size_t)nnz +
                              sizeof(double) * ((size_t)R * D + (size_t)N * D) + 8 * 256));
    HTAKE(d_ptr, int64_t, (size_t)N + 1);
    HTAKE(d_req, double, (size_t)R * D);
    HTAKE(d_used, double, (size_t)N * D);
    HTAKE(d_idx, int32_t, nnz);
    H2D(d_ptr, row_ptr, sizeof(int64_t) * ((size_t)N + 1));
    H2D(d_req, req_run, sizeof(double) * (size_t)R * D);
    H2D(d_used, used_inout, sizeof(double) * (size_t)N * D);
    if (run_idx) H2D(d_idx, run_idx, sizeof(int32_t) * (size_t)nnz);
    TRY(acsfit_occupancy(ctx, d_ptr, run_idx ? d_idx : nullptr, d_req, N, D, d_used, st));
    D2H(used_inout, d_used, sizeof(double) * (size_t)N * D);
    CUDA_TRY(cudaStreamSynchronize(st));
    return ACSFIT_OK;
}

extern "C" acsfit_status acsfit_maintain_host(acsfit_ctx *ctx, const int64_t *row_ptr, const int32_t *run_idx,
                                              const double *req_run, const uint8_t *flags_run, int64_t R,
                                              const double *cap_type, int K, const int32_t *node_type,
                                              const uint8_t *node_flags, const int64_t *node_age,
                                              const int32_t *node_pool, int64_t N, int D, int any_pending,
                                              int64_t idle_threshold, const int64_t *budget0,
                                              const uint8_t *pool_scalable, int T, int dry_run,
                                              uint8_t *out_state, uint8_t *out_action)
{
    TRY(enter(ctx, D));
    cudaStream_t st = nullptr;
    if (N < 0 || R < 0 || K < 0 || T < 0 || T > ACSFIT_MAX_POOLS ||
        (N > 0 && (!row_ptr || !cap_type || !node_type || !node_flags || !node_age || !node_pool || !out_state || !out_action)) ||
        (R > 0 && (!req_run || !flags_run)) || (T > 0 && (!budget0 || !pool_scalable)))
        return fail(ctx, ACSFIT_E_INVALID, "maintain_host: bad arguments");
    if (N == 0) return ACSFIT_OK;
    const int64_t nnz = row_ptr[N];
    if (nnz < 0) return fail(ctx, ACSFIT_E_INVALID, "maintain_host: bad CSR");
    const size_t bytes = sizeof(int64_t) * (2 * (size_t)N + 2) + sizeof(int32_t) * ((size_t)nnz + 2 * (size_t)N) +
                         sizeof(double) * ((size_t)R * D + (size_t)K * D) + (size_t)R + 3 * (size_t)N + 16 * 256;
    TRY(hbuf_reserve(ctx, bytes));
    HTAKE(d_ptr, int64_t, (size_t)N + 1);
    HTAKE(d_age, int64_t, N);
    HTAKE(d_thr, int64_t, 1);
    HTAKE(d_req, double, (size_t)R * D);
    HTAKE(d_cap, double, (size_t)K * D);
    HTAKE(d_idx, int32_t, nnz);
    HTAKE(d_type, int32_t, N);
    HTAKE(d_pool, int32_t, N);
    HTAKE(d_pflags, uint8_t, R);
    HTAKE(d_nflags, uint8_t, N);
    HTAKE(d_state, uint8_t, N);
    HTAKE(d_action, uint8_t, N);
    H2D(d_ptr, row_ptr, sizeof(int64_t) * ((size_t)N + 1));
    H2D(d_age, node_age, sizeof(int64_t) * (size_t)N);
    H2D(d_thr, &idle_threshold, sizeof(int64_t));
    H2D(d_req, req_run, sizeof(double) * (size_t)R * D);
    H2D(d_cap, cap_type, sizeof(double) * (size_t)K * D);
    if (run_idx) H2D(d_idx, run_idx, sizeof(int32_t) * (size_t)nnz);
    H2D(d_type, node_type, sizeof(int32_t) * (size_t)N);
    H2D(d_pool, node_pool, sizeof(int32_t) * (size_t)N);
    H2D(d_pflags, flags_run, (size_t)R);
    H2D(d_nflags, node_flags, (size_t)N);
    TRY(run_node_states(ctx, d_ptr, run_idx ? d_idx : nullptr, d_req, d_pflags, d_cap, d_type, d_nflags, d_age, N, D, any_pending, d_thr, 1,
                        d_state, st));
    TRY(arena_reserve(ctx, maintain_scratch(N, T), st));
    ctx->arena_off = 0;
    TRY(maintain_actions_impl(ctx, d_state, d_pool, N, budget0, pool_scalable, T, dry_run, d_action, st));
    D2H(out_state, d_state, (size_t)N);
    D2H(out_action, d_action, (size_t)N);
    CUDA_TRY(cudaStreamSynchronize(st));
    return ACSFIT_OK;
}
