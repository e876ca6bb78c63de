// developer micro-benchmark of the resolver's inner loop (one warp, lane = bin, D = 4):
// cycles per entry for several formulations.  nvcc -gencode arch=compute_90a,code=sm_90a -O3
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int D = 4;
constexpr int NE = 256;

__device__ __forceinline__ void load_row(double (&r)[D], const double *src)
{
    double2 a = *reinterpret_cast<const double2 *>(src), b = *reinterpret_cast<const double2 *>(src + 2);
    r[0] = a.x; r[1] = a.y; r[2] = b.x; r[3] = b.y;
}

template <int V>
__global__ void resolver(const double *rows_g, double unit0, double unit1, double unit2, double unit3, long long *cyc,
                         int *out_placed, int reps)
{
    __shared__ __align__(16) double rows[NE * D];
    __shared__ unsigned outq_all[8][NE + 1];
    unsigned *outq = outq_all[threadIdx.x >> 5];
    for (int i = threadIdx.x; i < NE * D; i += blockDim.x) rows[i] = rows_g[i];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    long long total = 0;
    int placed_sum = 0;
    for (int rep = 0; rep < reps; ++rep) {
        double S[D] = {unit0, unit1, unit2, unit3};
        unsigned out = 0, touched = 0;
        int n_placed = 0;
        unsigned long long evals = 0;
        long long t0 = clock64();
        for (int base = 0; base < NE; base += 32) {
            int placed_here = -1;
            double r[D];
            load_row(r, rows + (size_t)base * D);
#pragma unroll 2
            for (int k = 0; k < 32; ++k) {
                double rn[D];
                load_row(rn, rows + (size_t)(base + (k + 1 < 32 ? k + 1 : 31)) * D);
                int found = -1;
                unsigned m;
                if (V == 0) {
                    bool ok = true;
#pragma unroll
                    for (int d = 0; d < D; ++d) ok = ok & (r[d] <= S[d]);
                    m = __ballot_sync(0xFFFFFFFFu, ok);
                } else if (V == 1) {  // independent compares, masks and-ed
                    m = 0xFFFFFFFFu;
#pragma unroll
                    for (int d = 0; d < D; ++d) m &= __ballot_sync(0xFFFFFFFFu, r[d] <= S[d]);
                } else {  // integer: non-negative finite doubles order like their bit patterns
                    long long bad = 0;
#pragma unroll
                    for (int d = 0; d < D; ++d) bad |= (__double_as_longlong(S[d]) - __double_as_longlong(r[d]));
                    m = __ballot_sync(0xFFFFFFFFu, bad >= 0);
                }
                if (m) {
                    found = __ffs(m) - 1;
                    if (V == 3) {
#pragma unroll
                        for (int d = 0; d < D; ++d) { double s2 = __dsub_rn(S[d], r[d]); S[d] = lane == found ? s2 : S[d]; }
                    } else if (lane == found) {
#pragma unroll
                        for (int d = 0; d < D; ++d) S[d] = __dsub_rn(S[d], r[d]);
                    }
                    evals += (unsigned long long)found + ((touched >> found) & 1u);
                    touched |= 1u << found;
                    if (lane == k) placed_here = found;
                    ++n_placed;
                } else {
                    if (lane == k) outq[out] = base + k + 1;
                    ++out;
                }
#pragma unroll
                for (int d = 0; d < D; ++d) r[d] = rn[d];
            }
            if (placed_here >= 0) out_placed[(threadIdx.x >> 5) * 0 + base + lane] = placed_here;
        }
        total += clock64() - t0;
        placed_sum += n_placed + (int)(evals & 1) + (int)out;
        __syncwarp();
    }
    if (threadIdx.x == 0) { *cyc = total; out_placed[NE] = placed_sum; }
}

int main()
{
    double h[NE * D];
    unsigned s = 12345;
    const double cpus[6] = {0.1, 0.25, 0.5, 1.0, 1.5, 2.0};
    for (int i = 0; i < NE; ++i) {
        s = s * 1664525u + 1013904223u;
        h[i * D + 0] = 0.0; h[i * D + 1] = cpus[(s >> 16) % 6];
        s = s * 1664525u + 1013904223u;
        h[i * D + 2] = (double)(64 << ((s >> 16) % 6)) * 1048576.0; h[i * D + 3] = 1.0;
    }
    double *d; long long *cyc; int *pl;
    cudaMalloc(&d, sizeof h); cudaMalloc(&cyc, 8); cudaMalloc(&pl, 4 * (NE + 1));
    cudaMemcpy(d, h, sizeof h, cudaMemcpyHostToDevice);
    const int reps = 200;
    for (int nw = 1; nw <= 8; nw *= 2)
    for (int v = 0; v < 1; ++v) {
        long long c = 0;
        for (int it = 0; it < 2; ++it) {
            if (v == 0) resolver<0><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, pl, reps);
            if (v == 1) resolver<1><<<1, 32>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, pl, reps);
            if (v == 2) resolver<2><<<1, 32>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, pl, reps);
            if (v == 3) resolver<3><<<1, 32>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, pl, reps);
            cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
        }
        int ps; cudaMemcpy(&ps, pl + NE, 4, cudaMemcpyDeviceToHost);
        printf("warps %d variant %d: %.1f cycles / entry  (checksum %d) %s\n", nw, v, (double)c / (reps * NE), ps, cudaGetErrorString(cudaGetLastError()));
    }
    return 0;
}
