// ubench6.cu -- issue rate of the packed-rank scan's inner operation on sm_90a:
//     miss |= ((tg - r) & g) ^ g            (one IADD + one three-input LOP3 per packed word, acsfit_kernels.cuh)
// measured as int32 lane-operations per clock and SM with every SM full of resident warps.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench6 tools/ubench6.cu && tools/ubench6
#include <cstdio>
#include <cuda_runtime.h>

template <int ILP>
__global__ void scan_op_kernel(unsigned *out, unsigned g, int iters)
{
    unsigned tg[ILP], miss[ILP], r = threadIdx.x * 2654435761u;
#pragma unroll
    for (int i = 0; i < ILP; ++i) {
        tg[i] = (r >> i) | g;
        miss[i] = 0;
    }
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < ILP; ++i) miss[i] |= ((tg[i] - r) & g) ^ g;
        r = r * 3u + 1u;  // one extra op per ILP pairs keeps the compiler from hoisting
    }
    unsigned acc = 0;
#pragma unroll
    for (int i = 0; i < ILP; ++i) acc ^= miss[i];
    if (acc == 0x12345u) out[0] = acc;
}

int main()
{
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, 0);
    unsigned *out;
    cudaMalloc(&out, 4);
    const int iters = 1 << 14, ILP = 16;
    for (int warps_per_sm : {8, 16, 32, 64}) {
        const int blocks = prop.multiProcessorCount * warps_per_sm / 8;
        scan_op_kernel<ILP><<<blocks, 256>>>(out, 0x88888888u, 16);
        cudaDeviceSynchronize();
        cudaEvent_t a, b;
        cudaEventCreate(&a);
        cudaEventCreate(&b);
        cudaEventRecord(a);
        scan_op_kernel<ILP><<<blocks, 256>>>(out, 0x88888888u, iters);
        cudaEventRecord(b);
        cudaEventSynchronize(b);
        float ms;
        cudaEventElapsedTime(&ms, a, b);
        int clk_khz;
        cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
        const double pairs = (double)blocks * 256 * iters * ILP;
        const double clocks = ms * 1e-3 * clk_khz * 1e3;
        printf("warps/SM %2d: %.3f ms, %.1f pair-ops (IADD+LOP3) per clock per SM = %.1f int32 lane-ops/clk/SM (nominal clock %d MHz)\n",
               warps_per_sm, ms, pairs / clocks / prop.multiProcessorCount, 2.0 * pairs / clocks / prop.multiProcessorCount,
               clk_khz / 1000);
    }
    return 0;
}
