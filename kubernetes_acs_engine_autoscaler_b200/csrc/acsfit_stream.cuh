// acsfit_stream.cuh -- K1 / K6 for a CONTIGUOUS running-pod table (run_idx == NULL: the pods of node n are rows
// row_ptr[n] .. row_ptr[n+1] of req_run, which is how the host layer lays them out).  Same work split and the
// same ordered float64 sums as node_stream_kernel (acsfit.cu); what changes is how bytes reach the SM:
//
//   * a warp owns a contiguous range of 32-node groups, hence ONE contiguous byte range of req_run / flags_run.
//     It streams that range through two shared-memory buffers with Hopper TMA bulk copies: one
//     `cp.async.bulk.shared.global` per chunk for the rows and one for the flag bytes, issued by a single lane and
//     completed on an mbarrier -- no per-lane address arithmetic, no index gather, no
//     16-byte cp.async fan-out;
//   * chunk boundaries are multiples of 16 entries from the start of the table, so every copy is 16-byte aligned
//     in global and shared memory (the first chunk may start a few entries before the warp's range: ignored) --
//     provided req_run and flags_run themselves are 16-byte aligned, which plan_scan (acsfit_scan_plan.h) checks
//     before it picks this form;
//   * the consume loop is branch-free: a pod that does not count (a mirrored pod in get_node_state) adds +0.0,
//     which leaves a non-negative float64 sum bit-identical, so lanes never diverge on the flag test.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "../../include/acsfit.h"
#include "acsfit_scan_plan.h"

namespace acsfit {

// Lane = node: a warp is only fully busy while the chunk in shared memory holds entries of all 32 nodes of the
// group it is summing.  With ~10 running pods per node that takes >= 320 entries per chunk, so the chunks are
// large and the CTA has few warps; with small chunks the consume loop is issue-bound on idle lanes.
// The two pull against each other (fewer warps hide less latency), so the geometry is a template pair
// <warps per CTA, staging bytes per warp> chosen from measurements on H100 (DESIGN.md section 6): 16 warps x 8 KB
// = 128 KB of staging per SM, all of it in flight.

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((unsigned)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, unsigned bytes, uint64_t *bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     (unsigned)__cvta_generic_to_shared(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"((unsigned)__cvta_generic_to_shared(bar))
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity)
{
    const unsigned addr = (unsigned)__cvta_generic_to_shared(bar);
    unsigned done;
    do {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
    } while (!done);
}

template <int D, bool STATES, int kBytesPerWarp, int kBulkWarps>
__global__ void __launch_bounds__(kBulkWarps * 32)
node_stream_bulk_kernel(const int64_t *__restrict__ row_ptr, const double *__restrict__ req_run,
                        const uint8_t *__restrict__ flags_run, const double *__restrict__ cap_type,
                        const int32_t *__restrict__ node_type, const uint8_t *__restrict__ node_flags,
                        const int64_t *__restrict__ node_age, int64_t N, int any_pending,
                        const int64_t *__restrict__ idle_threshold, int S, uint8_t *__restrict__ out_state,
                        double *__restrict__ used_inout)
{
    constexpr int kChunk = kBytesPerWarp / 2 / (8 * D);  // entries per chunk
    static_assert(kChunk >= 16 && kChunk % 16 == 0, "chunks are multiples of 16 entries (16-byte aligned flag copies)");
    extern __shared__ __align__(128) unsigned char bulk_smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double *rows_s = reinterpret_cast<double *>(bulk_smem) + (size_t)warp * 2 * kChunk * D;
    uint8_t *flags_s = bulk_smem + (size_t)kBulkWarps * kBytesPerWarp + (size_t)warp * 2 * kChunk;
    uint64_t *bars = reinterpret_cast<uint64_t *>(bulk_smem + (size_t)kBulkWarps * kBytesPerWarp + (size_t)kBulkWarps * 2 * kChunk) + warp * 2;

    const int64_t groups = (N + 31) / 32;
    const int64_t n_warps = (int64_t)gridDim.x * kBulkWarps;
    const int64_t per = (groups + n_warps - 1) / n_warps;
    const int64_t g0 = ((int64_t)blockIdx.x * kBulkWarps + warp) * per;
    const int64_t g1 = min(groups, g0 + per);
    if (g0 >= g1) return;  // (whole warps only: no CTA-wide barrier below)
    const int64_t K0 = row_ptr[g0 * 32], K1 = row_ptr[min(g1 * 32, N)], Rtot = row_ptr[N];
    const int64_t base = K0 & ~(int64_t)15;
    const int64_t n_chunks = K1 > base ? (K1 - base + kChunk - 1) / kChunk : 0;

    if (lane == 0) {
        mbar_init(bars + 0, 1);
        mbar_init(bars + 1, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncwarp();

    auto issue = [&](int64_t c, int buf) {
        const int64_t kc = base + c * kChunk;
        const int ne = (int)min((int64_t)kChunk, Rtot - kc);
        if (lane == 0) {
            const unsigned row_bytes = (unsigned)ne * 8u * D;
            const unsigned flag_bytes = STATES ? (unsigned)(ne & ~15) : 0u;
            mbar_expect_tx(bars + buf, row_bytes + flag_bytes);
            bulk_g2s(rows_s + (size_t)buf * kChunk * D, req_run + (size_t)kc * D, row_bytes, bars + buf);
            if (flag_bytes) bulk_g2s(flags_s + buf * kChunk, flags_run + kc, flag_bytes, bars + buf);
        }
        if (STATES && (ne & 15)) {  // the table's last few flag bytes (not a multiple of 16): plain loads
            const int e = (ne & ~15) + lane;
            if (lane < 16 && e < ne) flags_s[buf * kChunk + e] = flags_run[kc + e];
        }
    };

    int64_t g = g0;
    int64_t lo, hi, lo_n = 0, hi_n = 0;
    double acc[D], acc_n[D];
    bool busy = false, undrainable = false;
    // per-node inputs of the state decision, fetched a group ahead like the row pointers (no exposed latency)
    int32_t ntype = 0, ntype_n = 0;
    uint8_t nflags = 0, nflags_n = 0;
    int64_t nage = 0, nage_n = 0;
    auto fetch_group = [&](int64_t gg, int64_t &l, int64_t &h, double (&a0)[D], int32_t &ty, uint8_t &fl, int64_t &ag) {
        const int64_t nn = gg * 32 + lane;
        l = row_ptr[min(nn, N)];
        h = row_ptr[min(nn + 1, N)];  // lanes past N get an empty range
#pragma unroll
        for (int d = 0; d < D; ++d) a0[d] = (!STATES && nn < N) ? used_inout[(size_t)nn * D + d] : 0.0;
        if (STATES && nn < N) {
            ty = node_type[nn];
            fl = node_flags[nn];
            ag = node_age[nn];
        }
    };
    fetch_group(g0, lo, hi, acc, ntype, nflags, nage);
    if (g0 + 1 < g1) fetch_group(g0 + 1, lo_n, hi_n, acc_n, ntype_n, nflags_n, nage_n);
    int64_t group_end = __shfl_sync(0xFFFFFFFFu, hi, 31);

    auto finalize = [&]() {
        const int64_t n = g * 32 + lane;
        if (n >= N) return;
        if (!STATES) {
#pragma unroll
            for (int d = 0; d < D; ++d) used_inout[(size_t)n * D + d] = acc[d];
            return;
        }
        const double *cap = cap_type + (size_t)ntype * D;
        bool under = true;
#pragma unroll
        for (int d = 0; d < D; ++d) {
            // (UTIL_THRESHOLD * capacity - utilization).possible: multiply THEN subtract, no FMA (scaler.py:86-87)
            const double left = __dsub_rn(__dmul_rn(cap[d], 0.3), acc[d]);
            under = under && (left >= 0.0);
        }
        const bool unsched = nflags & ACSFIT_NODEF_UNSCHEDULABLE;
        const bool pending = any_pending && !(nflags & ACSFIT_NODEF_NO_PENDING_MATCH);
        const int64_t age = nage;
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

    if (n_chunks > 0) issue(0, 0);
    if (n_chunks > 1) issue(1, 1);
    unsigned phase[2] = {0u, 0u};
    for (int64_t c = 0;; ++c) {
        const int buf = (int)(c & 1);
        const bool has_chunk = c < n_chunks;
        const int64_t kc = base + c * kChunk;
        const int64_t chunk_end = has_chunk ? min(kc + kChunk, K1) : K1;
        if (has_chunk) {
            mbar_wait(bars + buf, phase[buf]);
            phase[buf] ^= 1u;
            __syncwarp();  // the tail flag bytes written with plain stores by other lanes
        }
        const double *rows_b = rows_s + (size_t)buf * kChunk * D;
        const uint8_t *flags_b = flags_s + buf * kChunk;
        while (g < g1) {
            if (has_chunk) {
                const int ea = (int)(max(lo, kc) - kc), eb = (int)(min(hi, chunk_end) - kc);
                for (int e = ea; e < eb; ++e) {
                    bool take = true;
                    if (STATES) {
                        const uint8_t f = flags_b[e];
                        undrainable = undrainable || (f & ACSFIT_PODF_UNDRAINABLE);
                        take = f & ACSFIT_PODF_BUSY;
                        busy = busy || take;
                    }
                    const double2 *r = reinterpret_cast<const double2 *>(rows_b + (size_t)e * D);
#pragma unroll
                    for (int d = 0; d < D / 2; ++d) {
                        const double2 v = r[d];
                        // ordered sum, pod-list order; a pod that does not count adds +0.0 (bit-neutral on a sum >= +0)
                        acc[2 * d] = __dadd_rn(acc[2 * d], take ? v.x : 0.0);
                        acc[2 * d + 1] = __dadd_rn(acc[2 * d + 1], take ? v.y : 0.0);
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
            ntype = ntype_n;
            nflags = nflags_n;
            nage = nage_n;
            busy = false;
            undrainable = false;
            group_end = __shfl_sync(0xFFFFFFFFu, hi, 31);
            if (g + 1 < g1) fetch_group(g + 1, lo_n, hi_n, acc_n, ntype_n, nflags_n, nage_n);
        }
        if (g >= g1) break;
        __syncwarp();  // every lane is done with this buffer before it is refilled
        if (c + 2 < n_chunks) issue(c + 2, buf);
    }
}

template <int D, bool STATES, int kBytesPerWarp, int kBulkWarps>
static cudaError_t launch_node_stream_bulk(int grid, cudaStream_t st, const int64_t *row_ptr, const double *req_run,
                                           const uint8_t *flags_run, const double *cap_type, const int32_t *node_type,
                                           const uint8_t *node_flags, const int64_t *node_age, int64_t N, int any_pending,
                                           const int64_t *thr, int S, uint8_t *out_state, double *used, ScanLaunch *rec)
{
    constexpr int kChunk = kBytesPerWarp / 2 / (8 * D);
    const size_t smem = (size_t)kBulkWarps * kBytesPerWarp + (size_t)kBulkWarps * 2 * kChunk + (size_t)kBulkWarps * 2 * sizeof(uint64_t);
    auto kern = node_stream_bulk_kernel<D, STATES, kBytesPerWarp, kBulkWarps>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    int per_sm = 0, dev = 0, sms = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kBulkWarps * 32, smem) == cudaSuccess && per_sm > 0 &&
        cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess)
        grid = per_sm * sms;  // persistent: exactly the resident CTAs (each warp takes a contiguous range of groups)
    kern<<<grid, kBulkWarps * 32, smem, st>>>(row_ptr, req_run, flags_run, cap_type, node_type, node_flags, node_age, N,
                                              any_pending, thr, S, out_state, used);
    *rec = {STATES ? 2 : 1, kScanBulk, D, kBytesPerWarp, kBulkWarps, kChunk, grid, S};
    return cudaGetLastError();
}

}  // namespace acsfit
