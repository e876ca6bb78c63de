// ubench7.cu -- cost of ONE placing step of the resolver, two formulations, on sm_90a:
//   vote:     lane = node, every lane tests the SAME entry, a ballot names the first fitting lane, that lane's state
//             changes (the loop of firstfit_pipeline_kernel today);
//   systolic: lane = node, lane i tests entry (step - i): the entry stream moves one lane per step, the only
//             cross-lane traffic is the "still alive" bit (shfl_up), each lane's state recurrence is local.
// Reports cycles per step for one active warp per CTA (the frontier is one warp) and for 8.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -o tools/ubench7 tools/ubench7.cu && tools/ubench7
#include <cstdio>
#include <cuda_runtime.h>

template <int D>
__device__ __forceinline__ void load_row(double (&r)[D], const double *p)
{
#pragma unroll
    for (int d = 0; d < D; d += 2) {
        const double2 v = *reinterpret_cast<const double2 *>(p + d);
        r[d] = v.x;
        r[d + 1] = v.y;
    }
}

// INTCMP: the comparisons on the bit patterns (sign bits clear: order of non-negative doubles = order of their bits);
// nodes: fl(C - t) >= 0  <=>  t <= C for finite values, so the literal test is one add and one compare
template <int D, bool BINS, bool INTCMP>
__device__ __forceinline__ bool fits(const double (&S)[D], const double (&C)[D], const double (&r)[D], double (&t)[D])
{
    bool ok = true, ok2 = true;
#pragma unroll
    for (int d = 0; d < D; ++d) {
        bool f;
        if (BINS) {
            t[d] = __dsub_rn(S[d], r[d]);
            f = INTCMP ? __double_as_longlong(r[d]) <= __double_as_longlong(S[d]) : r[d] <= S[d];
        } else {
            t[d] = __dadd_rn(S[d], r[d]);
            f = INTCMP ? __double_as_longlong(t[d]) <= __double_as_longlong(C[d]) : __dsub_rn(C[d], t[d]) >= 0.0;
        }
        if (d < D / 2) ok = ok & f; else ok2 = ok2 & f;
    }
    return ok & ok2;
}

// dependent-chain latencies (one warp): cycles per link
template <int V>
__global__ void chain_kernel(double a, double b, long long *cyc, double *sink)
{
    const int lane = threadIdx.x & 31;
    double x = a + lane, y = b;
    unsigned m = 0;
    const int N = 4096;
    const long long t0 = clock64();
#pragma unroll 16
    for (int i = 0; i < N; ++i) {
        if (V == 0) x = __dadd_rn(x, y);                                  // DADD -> DADD
        if (V == 1) x = (x <= y) ? __longlong_as_double(__double_as_longlong(x) + 8) : y;   // DSETP -> SEL/IADD -> DSETP
        if (V == 2) x = (__double_as_longlong(x) <= __double_as_longlong(y)) ? __longlong_as_double(__double_as_longlong(x) + 8) : y;  // ISETP64 -> ...
        if (V == 3) { m = __ballot_sync(0xFFFFFFFFu, (m >> lane) & 1u ? false : true); }     // vote -> shift/test -> vote
        if (V == 4) { m = __shfl_up_sync(0xFFFFFFFFu, m + 1u, 1); }                           // shfl -> IADD -> shfl
        if (V == 5) { const bool p = __any_sync(0xFFFFFFFFu, x <= y); x = p ? __longlong_as_double(__double_as_longlong(x) + 8) : y; }  // DSETP -> vote.any -> SEL
    }
    const long long t1 = clock64();
    if (lane == 0) cyc[V] = t1 - t0;
    if (x == 1.2345e300 || m == 0x1234567u) sink[0] = x;
}

// rows: n_entries x D in shared memory (copied from global), found: byte per entry
template <int D, bool BINS, bool SYSTOLIC, bool INTCMP>
__global__ void step_kernel(const double *rows_g, int n_entries, int active_warps, unsigned *out, long long *cyc)
{
    extern __shared__ __align__(16) unsigned char smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    double *rows = reinterpret_cast<double *>(smem);                          // n_entries x D (shared by the warps)
    double *ring = rows + (size_t)n_entries * D + (size_t)warp * 64 * D;      // 64 rows per warp
    unsigned char *found = smem + ((size_t)n_entries * D + (size_t)(blockDim.x >> 5) * 64 * D) * 8 + (size_t)warp * n_entries;
    for (int i = threadIdx.x; i < n_entries * D; i += blockDim.x) rows[i] = rows_g[i];
    for (int i = lane; i < n_entries; i += 32) found[i] = 255;
    __syncthreads();
    if (warp >= active_warps) return;
    double S[D], C[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
        S[d] = BINS ? 10.0 : 0.0;
        C[d] = 10.0;
    }
    unsigned n_taken = 0;
    const long long t0 = clock64();
    if (!SYSTOLIC) {
        const unsigned me = 1u << lane, le = (me << 1) - 1u;
        double r[D];
        load_row<D>(r, rows);
        for (int k0 = 0; k0 < n_entries; k0 += 4) {
#pragma unroll
            for (int k = k0; k < k0 + 4; ++k) {
                double rn[D], t[D];
                load_row<D>(rn, rows + (size_t)((k + 1) % n_entries) * D);
                const bool ok = fits<D, BINS, INTCMP>(S, C, r, t);
                const bool any = __any_sync(0xFFFFFFFFu, ok);
                const unsigned m = __ballot_sync(0xFFFFFFFFu, ok);
                if (any) {
                    if ((m & le) == me) {
#pragma unroll
                        for (int d = 0; d < D; ++d) S[d] = t[d];
                        found[k] = (unsigned char)lane;
                        ++n_taken;
                    }
                }
#pragma unroll
                for (int d = 0; d < D; ++d) r[d] = rn[d];
            }
        }
    } else {
        // the stream is fed in blocks of 32 steps: lane s stages row (block*32 + s) into the ring, then 32 steps;
        // 31 never-fitting rows drain the pipe at the end
        const double inf = __longlong_as_double(0x7FF0000000000000ll);
        bool alive = false;
        int T = 0;
        const int n_blocks = n_entries / 32 + 1;
        for (int b = 0; b < n_blocks; ++b, T += 32) {
            {
                const int k = b * 32 + lane;
                double own[D];
                if (k < n_entries) load_row<D>(own, rows + (size_t)k * D);
                else {
#pragma unroll
                    for (int d = 0; d < D; ++d) own[d] = d == 0 ? inf : 0.0;
                }
                double *dst = ring + (size_t)((T + lane) & 63) * D;
#pragma unroll
                for (int d = 0; d < D; d += 2) *reinterpret_cast<double2 *>(dst + d) = make_double2(own[d], own[d + 1]);
            }
            __syncwarp();
            double r[D];
            load_row<D>(r, ring + (size_t)((T - lane) & 63) * D);
#pragma unroll 4
            for (int s = 0; s < 32; ++s) {
                double rn[D], t[D];
                if (s + 1 < 32) load_row<D>(rn, ring + (size_t)((T + s + 1 - lane) & 63) * D);
                const bool fit = fits<D, BINS, INTCMP>(S, C, r, t);
                const bool in = lane == 0 ? true : alive;
                const bool take = in & fit & (T + s - lane >= 0);
                if (take) {
#pragma unroll
                    for (int d = 0; d < D; ++d) S[d] = t[d];
                    const int k = T + s - lane;
                    if (k < n_entries) found[k] = (unsigned char)lane;
                    ++n_taken;
                }
                const unsigned oa = (in & !fit) ? 1u : 0u;
                alive = __shfl_up_sync(0xFFFFFFFFu, oa, 1) != 0u;
#pragma unroll
                for (int d = 0; d < D; ++d) r[d] = rn[d];
            }
        }
    }
    const long long t1 = clock64();
    unsigned tot = __reduce_add_sync(0xFFFFFFFFu, n_taken);
    if (lane == 0) {
        cyc[blockIdx.x * 8 + warp] = t1 - t0;
        atomicAdd(out, tot);
    }
    double acc = 0;
#pragma unroll
    for (int d = 0; d < D; ++d) acc += S[d];
    if (acc == 1.2345e300) out[1] = 1;
}

template <int D, bool BINS, bool SYSTOLIC, bool INTCMP>
void run(const char *name, int active_warps)
{
    const int n = 512;
    double *h = new double[(size_t)n * D];
    unsigned long long s = 88172645463325252ull;
    for (int i = 0; i < n * D; ++i) {
        s ^= s << 13; s ^= s >> 7; s ^= s << 17;
        h[i] = 0.5 + (double)(s % 4000) / 1000.0;   // 0.5 .. 4.5 of capacity 10 -> 2-4 entries per lane
    }
    double *rows;
    unsigned *out;
    long long *cyc;
    cudaMalloc(&rows, sizeof(double) * n * D);
    cudaMalloc(&out, 8);
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    cudaMalloc(&cyc, sizeof(long long) * sms * 8);
    cudaMemcpy(rows, h, sizeof(double) * n * D, cudaMemcpyHostToDevice);
    const size_t smem = ((size_t)n * D + 8 * 64 * D) * 8 + 8 * n;
    auto k = step_kernel<D, BINS, SYSTOLIC, INTCMP>;
    cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    long long hc[8];
    unsigned ho[2];
    for (int rep = 0; rep < 2; ++rep) {
        cudaMemset(out, 0, 8);
        k<<<sms, 256, smem>>>(rows, n, active_warps, out, cyc);
        cudaDeviceSynchronize();
    }
    cudaMemcpy(hc, cyc, sizeof(hc), cudaMemcpyDeviceToHost);
    cudaMemcpy(ho, out, 8, cudaMemcpyDeviceToHost);
    const int steps = SYSTOLIC ? (n / 32 + 1) * 32 : n;
    printf("%-28s D=%d warps=%d: %7lld cycles for %d entries = %6.1f cycles/entry (%d steps, %5.1f cycles/step), taken/warp %.1f  [%s]\n",
           name, D, active_warps, hc[0], n, (double)hc[0] / n, steps, (double)hc[0] / steps,
           (double)ho[0] / ((double)sms * active_warps), cudaGetErrorString(cudaGetLastError()));
    delete[] h;
}

int main()
{
    {
        long long *cyc, hc[6];
        double *sink;
        cudaMalloc(&cyc, 48);
        cudaMalloc(&sink, 8);
        chain_kernel<0><<<1, 32>>>(1.0, 1e-9, cyc, sink);
        chain_kernel<1><<<1, 32>>>(1.0, 1e300, cyc, sink);
        chain_kernel<2><<<1, 32>>>(1.0, 1e300, cyc, sink);
        chain_kernel<3><<<1, 32>>>(1.0, 1e300, cyc, sink);
        chain_kernel<4><<<1, 32>>>(1.0, 1e300, cyc, sink);
        chain_kernel<5><<<1, 32>>>(1.0, 1e300, cyc, sink);
        cudaDeviceSynchronize();
        cudaMemcpy(hc, cyc, 48, cudaMemcpyDeviceToHost);
        const char *names[6] = {"DADD->DADD", "DSETP->SEL+IADD64", "ISETP64->SEL+IADD64", "ballot->shift/test", "shfl_up->IADD", "DSETP->vote.any->SEL+IADD64"};
        for (int i = 0; i < 6; ++i) printf("chain %-30s %.1f cycles per link\n", names[i], (double)hc[i] / 4096.0);
    }
    for (int w : {1, 8}) {
        run<4, false, false, false>("nodes vote fp64", w);
        run<4, false, false, true>("nodes vote intcmp", w);
        run<4, true, false, false>("bins vote fp64", w);
        run<4, true, false, true>("bins vote intcmp", w);
        run<8, false, false, false>("nodes vote fp64", w);
        run<8, false, false, true>("nodes vote intcmp", w);
        run<8, true, false, false>("bins vote fp64", w);
        run<8, true, false, true>("bins vote intcmp", w);
        run<4, false, true, true>("nodes systolic intcmp", w);
        run<4, true, true, true>("bins systolic intcmp", w);
    }
    return 0;
}
