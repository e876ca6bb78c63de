// developer micro-benchmark: latency of the dependent steps a sequential placement loop is made of
// (one warp, dependent chain of N iterations, cycles per iteration).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -o build_tmp/ubench4 tools/ubench4.cu
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int N = 2048;

template <int V>
__global__ void chain(double seed, double step, long long *cyc, double *sink)
{
    const int lane = threadIdx.x & 31;
    double x = seed + lane, y = step;
    unsigned u = (unsigned)lane * 2654435761u + 12345u;
    long long t0 = clock64();
#pragma unroll 8
    for (int i = 0; i < N; ++i) {
        if (V == 0) {  // DADD -> DADD
            x = __dadd_rn(x, y);
        } else if (V == 1) {  // DADD -> integer op on the high word -> DADD
            x = __dadd_rn(x, y);
            int hi = __double2hiint(x) ^ 1;
            x = __hiloint2double(hi ^ 1, __double2loint(x));
        } else if (V == 2) {  // DADD -> DSETP -> select -> DADD
            double z = __dadd_rn(x, y);
            x = (z >= 0.0) ? z : x;
        } else if (V == 3) {  // DADD -> sign test (ISETP) -> select
            double z = __dadd_rn(x, y);
            x = (__double2hiint(z) >= 0) ? z : x;
        } else if (V == 4) {  // ISETP -> VOTE -> integer
            const unsigned m = __ballot_sync(0xFFFFFFFFu, (int)u >= 0);
            u = u * 3u + m;
        } else if (V == 5) {  // REDUX.MIN -> integer
            const unsigned m = __reduce_min_sync(0xFFFFFFFFu, u);
            u = (u ^ m) * 3u + 1u;
        } else if (V == 6) {  // SHFL -> integer
            const unsigned m = __shfl_up_sync(0xFFFFFFFFu, u, 1);
            u = (u ^ m) * 3u + 1u;
        } else if (V == 7) {  // integer only (reference for 4..6): IMAD chain
            u = (u ^ (u >> 3)) * 3u + 1u;
        } else if (V == 8) {  // DADD -> sign -> VOTE -> lane compare -> select -> DADD  (the literal chain, minimal)
            double z = __dadd_rn(x, y);
            const unsigned m = __ballot_sync(0xFFFFFFFFu, __double2hiint(z) >= 0);
            x = ((m & (0u - m)) == (1u << lane)) ? z : x;
        } else if (V == 9) {  // same with DSETP
            double z = __dadd_rn(x, y);
            const unsigned m = __ballot_sync(0xFFFFFFFFu, z >= 0.0);
            x = ((m & (0u - m)) == (1u << lane)) ? z : x;
        } else if (V == 10) {  // 4 chained DSETP (the and-chain the compiler emits for 4 dims)
            bool ok = (x <= y);
            ok = ok & (x + 1.0 <= y);
            ok = ok & (x + 2.0 <= y);
            ok = ok & (x + 3.0 <= y);
            x = ok ? x : __dadd_rn(x, -1.0);
        } else if (V == 11) {  // match.any as a cross-lane step
            const unsigned m = __match_any_sync(0xFFFFFFFFu, u & 3u);
            u = u * 3u + m;
        }
    }
    long long t1 = clock64();
    if (threadIdx.x == 0) *cyc = t1 - t0;
    sink[threadIdx.x] = x + (double)u;
}

int main()
{
    long long *cyc; double *sink;
    cudaMalloc(&cyc, 8); cudaMalloc(&sink, 8 * 32);
    const char *names[12] = {"DADD->DADD", "DADD->LOP(hi)->DADD", "DADD->DSETP->SEL", "DADD->ISETP(hi)->SEL", "ISETP->VOTE->IMAD",
                             "REDUX.MIN->IMAD", "SHFL->IMAD", "LOP/IMAD only", "DADD->ISETP->VOTE->ISETP->SEL", "DADD->DSETP->VOTE->ISETP->SEL",
                             "4 DSETP and-chain -> SEL/DADD", "MATCH.ANY->IMAD"};
    for (int v = 0; v < 12; ++v) {
        long long c = 0;
        for (int it = 0; it < 2; ++it) {
            switch (v) {
            case 0: chain<0><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            case 1: chain<1><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            case 2: chain<2><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            case 3: chain<3><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            case 4: chain<4><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            case 5: chain<5><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            case 6: chain<6><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            case 7: chain<7><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            case 8: chain<8><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            case 9: chain<9><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            case 10: chain<10><<<1, 32>>>(1.0, 1e9, cyc, sink); break;
            case 11: chain<11><<<1, 32>>>(1.0, 0.5, cyc, sink); break;
            }
            cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
        }
        printf("%-36s %.1f cycles / iteration  %s\n", names[v], (double)c / N, cudaGetErrorString(cudaGetLastError()));
    }
    return 0;
}
