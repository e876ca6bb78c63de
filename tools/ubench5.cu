// developer micro-benchmark: throughput of the scan's inner loop (compare-only, thresholds in registers,
// pod rows broadcast from shared memory) in DSETP per cycle per SM, for 8 and 16 warps per SM.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o build_tmp/ubench5 tools/ubench5.cu
#include <cstdio>
#include <cuda_runtime.h>

template <int D, int K, int PODS, bool SIGN>
__global__ void scan(const double *rows_g, int n_rows, int reps, long long *cyc, unsigned *sink)
{
    extern __shared__ __align__(16) double rows[];
    for (int i = threadIdx.x; i < n_rows * D; i += blockDim.x) rows[i] = rows_g[i];
    __syncthreads();
    double t[K][D];
    for (int k = 0; k < K; ++k)
        for (int d = 0; d < D; ++d) t[k][d] = 0.5 + 0.001 * ((threadIdx.x * 7 + k * 3 + d) % 13);
    unsigned hits = 0;
    long long t0 = clock64();
    for (int rep = 0; rep < reps; ++rep)
        for (int q = 0; q < n_rows; q += PODS) {
            double r[PODS][D];
#pragma unroll
            for (int p = 0; p < PODS; ++p)
#pragma unroll
                for (int d = 0; d < D; d += 2) {
                    double2 v = *reinterpret_cast<const double2 *>(rows + (size_t)(q + p) * D + d);
                    r[p][d] = v.x; r[p][d + 1] = v.y;
                }
#pragma unroll
            for (int k = 0; k < K; ++k)
#pragma unroll
                for (int p = 0; p < PODS; ++p) {
                    bool ok = true;
                    if (SIGN) {
                        int neg = 0;
#pragma unroll
                        for (int d = 0; d < D; ++d) neg |= __double2hiint(__dsub_rn(t[k][d], r[p][d]));
                        ok = neg >= 0;
                    } else {
#pragma unroll
                        for (int d = 0; d < D; ++d) ok = ok & (r[p][d] <= t[k][d]);
                    }
                    if (ok) hits += k + p + 1;
                }
        }
    long long t1 = clock64();
    if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
    sink[blockIdx.x * blockDim.x + threadIdx.x] = hits;
}

template <int D, int K, int PODS, bool SIGN>
void run(const double *d_rows, int n_rows, int warps, long long *cyc, unsigned *sink)
{
    const int reps = 50;
    auto kern = scan<D, K, PODS, SIGN>;
    for (int it = 0; it < 2; ++it) kern<<<1, warps * 32, n_rows * D * 8>>>(d_rows, n_rows, reps, cyc, sink);
    long long c; cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
    const double cmp = (double)reps * n_rows * K * D * warps * 32;
    printf("%s D=%d K=%d pods/iter=%d warps=%2d: %.1f compare lane-ops / cycle / SM (%s)\n", SIGN ? "DADD+sign" : "DSETP    ", D, K, PODS, warps, cmp / c,
           cudaGetErrorString(cudaGetLastError()));
}

int main()
{
    const int n_rows = 256;
    double h[256 * 8];
    for (int i = 0; i < 256 * 8; ++i) h[i] = 0.6 + 0.0001 * (i % 97);   // almost never all dims <= t
    double *d; long long *cyc; unsigned *sink;
    cudaMalloc(&d, sizeof h); cudaMalloc(&cyc, 8 * 8); cudaMalloc(&sink, 4 * 1024);
    cudaMemcpy(d, h, sizeof h, cudaMemcpyHostToDevice);
    for (int w = 8; w <= 16; w += 8) {
        run<4, 4, 2, false>(d, n_rows, w, cyc, sink); run<4, 4, 2, true>(d, n_rows, w, cyc, sink);
        run<4, 4, 4, false>(d, n_rows, w, cyc, sink); run<4, 4, 4, true>(d, n_rows, w, cyc, sink);
        run<8, 2, 2, false>(d, n_rows, w, cyc, sink); run<8, 2, 2, true>(d, n_rows, w, cyc, sink);
        run<8, 2, 4, false>(d, n_rows, w, cyc, sink); run<8, 2, 4, true>(d, n_rows, w, cyc, sink);
        run<8, 1, 4, false>(d, n_rows, w, cyc, sink); run<8, 1, 4, true>(d, n_rows, w, cyc, sink);
    }
    return 0;
}
