// developer micro-benchmark: the resolver's sequential loop, literal form versus the speculative form
// (both outcomes of the next test are prepared off the critical chain; the chain is ballot -> select).
// one CTA, nw warps each running its own copy; lane = bin (or node), D = 4.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -fmad=false -o /tmp/ubench3 tools/ubench3.cu
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

// V = 0 literal loop (as in the round-1 kernel), V = 1 speculative.  BINS: S = remaining, test r <= S, S -= r.
// NODES: S = used, test C - (S + r) >= 0, S += r.
template <int V, bool BINS>
__global__ void resolver(const double *rows_g, double u0, double u1, double u2, double u3, long long *cyc, unsigned *out_sum,
                         int reps)
{
    __shared__ __align__(16) double rows[(NE + 8) * D];
    __shared__ unsigned char fnd_all[8][NE];
    for (int i = threadIdx.x; i < NE * D; i += blockDim.x) rows[i] = rows_g[i];
    for (int i = threadIdx.x; i < 8 * D; i += blockDim.x) rows[NE * D + i] = (i % D == 0) ? __longlong_as_double(0x7FF0000000000000ll) : 0.0;
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1u;
    volatile unsigned char *fnd = fnd_all[threadIdx.x >> 5];
    long long total = 0;
    unsigned check = 0;
    for (int rep = 0; rep < reps; ++rep) {
        const double C[D] = {u0, u1, u2, u3};
        double S[D];
#pragma unroll
        for (int d = 0; d < D; ++d) S[d] = BINS ? C[d] : 0.0;
        long long t0 = clock64();
        for (int base = 0; base < NE; base += 32) {
            const double *brow = rows + (size_t)base * D;
            unsigned took = 0, mymask = 0;
#pragma unroll
            for (int d = 0; d < D; ++d) S[d] = BINS ? C[d] : 0.0;
            double r[D];
            load_row(r, brow);
            if (V == 0) {
                for (int k0 = 0; k0 < 32; k0 += 4)
#pragma unroll
                for (int k = k0; k < k0 + 4; ++k) {
                    double rn[D];
                    load_row(rn, brow + (size_t)(k + 1) * D);
                    bool ok = true;
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        if (BINS) ok = ok & (r[d] <= S[d]);
                        else ok = ok & (__dsub_rn(C[d], __dadd_rn(S[d], r[d])) >= 0.0);
                    }
                    const unsigned m = __ballot_sync(0xFFFFFFFFu, ok);
                    if (m) {
                        const int found = __ffs(m) - 1;
                        if (lane == found) {
#pragma unroll
                            for (int d = 0; d < D; ++d) S[d] = BINS ? __dsub_rn(S[d], r[d]) : __dadd_rn(S[d], r[d]);
                        }
                        if (lane == 0) fnd[k] = (unsigned char)found;
                        took |= 1u << k;
                    }
#pragma unroll
                    for (int d = 0; d < D; ++d) r[d] = rn[d];
                }
            } else if (V == 2) {  // literal order, unchained: new state first, one sign test over all dims
                for (int k0 = 0; k0 < 32; k0 += 4)
#pragma unroll
                for (int k = k0; k < k0 + 4; ++k) {
                    double rn[D], X[D];
                    load_row(rn, brow + (size_t)(k + 1) * D);
                    int neg = 0;
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        X[d] = BINS ? __dsub_rn(S[d], r[d]) : __dadd_rn(S[d], r[d]);
                        neg |= __double2hiint(BINS ? X[d] : __dsub_rn(C[d], X[d]));
                    }
                    const bool ok = neg >= 0;
                    const unsigned m = __ballot_sync(0xFFFFFFFFu, ok);
                    const bool mine = ok && !(m & lt);
#pragma unroll
                    for (int d = 0; d < D; ++d) S[d] = mine ? X[d] : S[d];
                    mymask |= (mine ? 1u : 0u) << k;
#pragma unroll
                    for (int d = 0; d < D; ++d) r[d] = rn[d];
                }
            } else if (V == 4) {  // literal order, integer-only chain: sign words -> REDUX.MIN -> bitwise select
                int myfound = 32;
                for (int k0 = 0; k0 < 32; k0 += 4)
#pragma unroll
                for (int k = k0; k < k0 + 4; ++k) {
                    double rn[D], X[D];
                    load_row(rn, brow + (size_t)(k + 1) * D);
                    int neg = 0;
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        X[d] = BINS ? __dsub_rn(S[d], r[d]) : __dadd_rn(S[d], r[d]);
                        neg |= __double2hiint(BINS ? X[d] : __dsub_rn(C[d], X[d]));
                    }
                    const unsigned val = (unsigned)lane | (((unsigned)neg >> 31) << 5);  // lane if it fits, else >= 32
                    const unsigned found = __reduce_min_sync(0xFFFFFFFFu, val);
                    const int sel = (int)((found ^ (unsigned)lane) - 1u) >> 31;  // all ones on the taking lane
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        const long long xs = __double_as_longlong(X[d]), ss = __double_as_longlong(S[d]);
                        const int lo = (__double2loint(X[d]) & sel) | (__double2loint(S[d]) & ~sel);
                        const int hi = (__double2hiint(X[d]) & sel) | (__double2hiint(S[d]) & ~sel);
                        (void)xs; (void)ss;
                        S[d] = __hiloint2double(hi, lo);
                    }
                    if (lane == k) myfound = (int)found;
#pragma unroll
                    for (int d = 0; d < D; ++d) r[d] = rn[d];
                }
                took = __ballot_sync(0xFFFFFFFFu, myfound < 32);
                check = check * 31u + took + (myfound < 32 ? (unsigned)myfound : 0u);
            } else if (V == 5) {  // speculative, integer-only chain
                int myfound = 32;
                double X[D];
                int neg = 0;
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    X[d] = BINS ? __dsub_rn(S[d], r[d]) : __dadd_rn(S[d], r[d]);
                    neg |= __double2hiint(BINS ? X[d] : __dsub_rn(C[d], X[d]));
                }
                unsigned val = (unsigned)lane | (((unsigned)neg >> 31) << 5);
                for (int k0 = 0; k0 < 32; k0 += 4)
#pragma unroll
                for (int k = k0; k < k0 + 4; ++k) {
                    double rn[D], XA[D], XB[D];
                    load_row(rn, brow + (size_t)(k + 1) * D);
                    int negA = 0, negB = 0;
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        XA[d] = BINS ? __dsub_rn(S[d], rn[d]) : __dadd_rn(S[d], rn[d]);
                        XB[d] = BINS ? __dsub_rn(X[d], rn[d]) : __dadd_rn(X[d], rn[d]);
                        negA |= __double2hiint(BINS ? XA[d] : __dsub_rn(C[d], XA[d]));
                        negB |= __double2hiint(BINS ? XB[d] : __dsub_rn(C[d], XB[d]));
                    }
                    const unsigned valA = (unsigned)lane | (((unsigned)negA >> 31) << 5);
                    const unsigned valB = (unsigned)lane | (((unsigned)negB >> 31) << 5);
                    const unsigned found = __reduce_min_sync(0xFFFFFFFFu, val);
                    const int sel = (int)((found ^ (unsigned)lane) - 1u) >> 31;
                    val = (valB & sel) | (valA & ~sel);
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        const int slo = (__double2loint(X[d]) & sel) | (__double2loint(S[d]) & ~sel);
                        const int shi = (__double2hiint(X[d]) & sel) | (__double2hiint(S[d]) & ~sel);
                        const int xlo = (__double2loint(XB[d]) & sel) | (__double2loint(XA[d]) & ~sel);
                        const int xhi = (__double2hiint(XB[d]) & sel) | (__double2hiint(XA[d]) & ~sel);
                        S[d] = __hiloint2double(shi, slo);
                        X[d] = __hiloint2double(xhi, xlo);
                    }
                    if (lane == k) myfound = (int)found;
                }
                took = __ballot_sync(0xFFFFFFFFu, myfound < 32);
                check = check * 31u + took + (myfound < 32 ? (unsigned)myfound : 0u);
            } else if (V == 6) {  // pairs: entries a,b per step; b's test is prepared against S and against S-after-a
                for (int k0 = 0; k0 < 32; k0 += 4)
#pragma unroll
                for (int k = k0; k < k0 + 4; k += 2) {
                    double ra[D], rb[D], Xa[D], Xb[D], Xab[D];
                    load_row(ra, brow + (size_t)k * D);
                    load_row(rb, brow + (size_t)(k + 1) * D);
                    int na = 0, nb = 0, nab = 0;
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        Xa[d] = BINS ? __dsub_rn(S[d], ra[d]) : __dadd_rn(S[d], ra[d]);
                        Xb[d] = BINS ? __dsub_rn(S[d], rb[d]) : __dadd_rn(S[d], rb[d]);
                        Xab[d] = BINS ? __dsub_rn(Xa[d], rb[d]) : __dadd_rn(Xa[d], rb[d]);
                        na |= __double2hiint(BINS ? Xa[d] : __dsub_rn(C[d], Xa[d]));
                        nb |= __double2hiint(BINS ? Xb[d] : __dsub_rn(C[d], Xb[d]));
                        nab |= __double2hiint(BINS ? Xab[d] : __dsub_rn(C[d], Xab[d]));
                    }
                    const unsigned ma = __ballot_sync(0xFFFFFFFFu, na >= 0);
                    const unsigned mb = __ballot_sync(0xFFFFFFFFu, nb >= 0);
                    const unsigned mab = __ballot_sync(0xFFFFFFFFu, nab >= 0);
                    const unsigned bit_a = ma & (0u - ma);            // lowest set bit (0 if none)
                    const unsigned mb2 = (mb & ~bit_a) | (mab & bit_a);
                    const unsigned bit_b = mb2 & (0u - mb2);
                    const unsigned me = 1u << lane;
                    const bool ta = (bit_a & me) != 0, tb = (bit_b & me) != 0;
#pragma unroll
                    for (int d = 0; d < D; ++d) S[d] = ta ? (tb ? Xab[d] : Xa[d]) : (tb ? Xb[d] : S[d]);
                    if (lane == 0) { fnd[k] = (unsigned char)(__ffs(bit_a) - 1); fnd[k + 1] = (unsigned char)(__ffs(bit_b) - 1); }
                    took |= ((bit_a ? 1u : 0u) << k) | ((bit_b ? 2u : 0u) << k);
                }
                __syncwarp();
                check = check * 31u + took + (((took >> lane) & 1u) ? fnd[lane] : 0u);
            } else if (V == 7 || V == 8) {  // 7: one entry per step, 8: pairs; per-lane masks, bookkeeping after the loop
                if (V == 7) {
                    for (int k0 = 0; k0 < 32; k0 += 4)
#pragma unroll
                    for (int k = k0; k < k0 + 4; ++k) {
                        double rn[D], X[D];
                        load_row(rn, brow + (size_t)(k + 1) * D);
                        int neg = 0;
#pragma unroll
                        for (int d = 0; d < D; ++d) {
                            X[d] = BINS ? __dsub_rn(S[d], r[d]) : __dadd_rn(S[d], r[d]);
                            neg |= __double2hiint(BINS ? X[d] : __dsub_rn(C[d], X[d]));
                        }
                        const unsigned m = __ballot_sync(0xFFFFFFFFu, neg >= 0);
                        const bool mine = (m & (0u - m)) == (1u << lane);
#pragma unroll
                        for (int d = 0; d < D; ++d) S[d] = mine ? X[d] : S[d];
                        mymask |= (mine ? 1u : 0u) << k;
#pragma unroll
                        for (int d = 0; d < D; ++d) r[d] = rn[d];
                    }
                } else {
                    for (int k0 = 0; k0 < 32; k0 += 4)
#pragma unroll
                    for (int k = k0; k < k0 + 4; k += 2) {
                        double ra[D], rb[D], Xa[D], Xb[D], Xab[D];
                        load_row(ra, brow + (size_t)k * D);
                        load_row(rb, brow + (size_t)(k + 1) * D);
                        int na = 0, nb = 0, nab = 0;
#pragma unroll
                        for (int d = 0; d < D; ++d) {
                            Xa[d] = BINS ? __dsub_rn(S[d], ra[d]) : __dadd_rn(S[d], ra[d]);
                            Xb[d] = BINS ? __dsub_rn(S[d], rb[d]) : __dadd_rn(S[d], rb[d]);
                            Xab[d] = BINS ? __dsub_rn(Xa[d], rb[d]) : __dadd_rn(Xa[d], rb[d]);
                            na |= __double2hiint(BINS ? Xa[d] : __dsub_rn(C[d], Xa[d]));
                            nb |= __double2hiint(BINS ? Xb[d] : __dsub_rn(C[d], Xb[d]));
                            nab |= __double2hiint(BINS ? Xab[d] : __dsub_rn(C[d], Xab[d]));
                        }
                        const unsigned ma = __ballot_sync(0xFFFFFFFFu, na >= 0);
                        const unsigned mb = __ballot_sync(0xFFFFFFFFu, nb >= 0);
                        const unsigned mab = __ballot_sync(0xFFFFFFFFu, nab >= 0);
                        const unsigned bit_a = ma & (0u - ma);
                        const unsigned mb2 = (mb & ~bit_a) | (mab & bit_a);
                        const unsigned bit_b = mb2 & (0u - mb2);
                        const unsigned me = 1u << lane;
                        const bool ta = bit_a == me, tb = bit_b == me;
#pragma unroll
                        for (int d = 0; d < D; ++d) S[d] = ta ? (tb ? Xab[d] : Xa[d]) : (tb ? Xb[d] : S[d]);
                        mymask |= ((ta ? 1u : 0u) | (tb ? 2u : 0u)) << k;
                    }
                }
                took = __reduce_or_sync(0xFFFFFFFFu, mymask);
                for (unsigned t = mymask; t; t &= t - 1) fnd[__ffs(t) - 1] = (unsigned char)lane;
                __syncwarp();
                check = check * 31u + took + (((took >> lane) & 1u) ? fnd[lane] : 0u);
            } else if (V == 9 || V == 10) {  // like 7 / 8 with the next group's rows fetched a whole group ahead
                double g[4][D];
#pragma unroll
                for (int j = 0; j < 4; ++j) load_row(g[j], brow + (size_t)j * D);
                for (int k0 = 0; k0 < 32; k0 += 4) {
                    double gn[4][D];
#pragma unroll
                    for (int j = 0; j < 4; ++j) load_row(gn[j], brow + (size_t)(k0 + 4 + j) * D);
                    if (V == 9) {
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            double X[D];
                            int neg = 0;
#pragma unroll
                            for (int d = 0; d < D; ++d) {
                                X[d] = BINS ? __dsub_rn(S[d], g[j][d]) : __dadd_rn(S[d], g[j][d]);
                                neg |= __double2hiint(BINS ? X[d] : __dsub_rn(C[d], X[d]));
                            }
                            const unsigned m = __ballot_sync(0xFFFFFFFFu, neg >= 0);
                            const bool mine = (m & (0u - m)) == (1u << lane);
#pragma unroll
                            for (int d = 0; d < D; ++d) S[d] = mine ? X[d] : S[d];
                            mymask |= (mine ? 1u : 0u) << (k0 + j);
                        }
                    } else {
#pragma unroll
                        for (int j = 0; j < 4; j += 2) {
                            double Xa[D], Xb[D], Xab[D];
                            int na = 0, nb = 0, nab = 0;
#pragma unroll
                            for (int d = 0; d < D; ++d) {
                                Xa[d] = BINS ? __dsub_rn(S[d], g[j][d]) : __dadd_rn(S[d], g[j][d]);
                                Xb[d] = BINS ? __dsub_rn(S[d], g[j + 1][d]) : __dadd_rn(S[d], g[j + 1][d]);
                                Xab[d] = BINS ? __dsub_rn(Xa[d], g[j + 1][d]) : __dadd_rn(Xa[d], g[j + 1][d]);
                                na |= __double2hiint(BINS ? Xa[d] : __dsub_rn(C[d], Xa[d]));
                                nb |= __double2hiint(BINS ? Xb[d] : __dsub_rn(C[d], Xb[d]));
                                nab |= __double2hiint(BINS ? Xab[d] : __dsub_rn(C[d], Xab[d]));
                            }
                            const unsigned ma = __ballot_sync(0xFFFFFFFFu, na >= 0);
                            const unsigned mb = __ballot_sync(0xFFFFFFFFu, nb >= 0);
                            const unsigned mab = __ballot_sync(0xFFFFFFFFu, nab >= 0);
                            const unsigned bit_a = ma & (0u - ma);
                            const unsigned mb2 = (mb & ~bit_a) | (mab & bit_a);
                            const unsigned bit_b = mb2 & (0u - mb2);
                            const unsigned me = 1u << lane;
                            const bool ta = bit_a == me, tb = bit_b == me;
#pragma unroll
                            for (int d = 0; d < D; ++d) S[d] = ta ? (tb ? Xab[d] : Xa[d]) : (tb ? Xb[d] : S[d]);
                            mymask |= ((ta ? 1u : 0u) | (tb ? 2u : 0u)) << (k0 + j);
                        }
                    }
#pragma unroll
                    for (int j = 0; j < 4; ++j)
#pragma unroll
                        for (int d = 0; d < D; ++d) g[j][d] = gn[j][d];
                }
                took = __reduce_or_sync(0xFFFFFFFFu, mymask);
                for (unsigned t = mymask; t; t &= t - 1) fnd[__ffs(t) - 1] = (unsigned char)lane;
                __syncwarp();
                check = check * 31u + took + (((took >> lane) & 1u) ? fnd[lane] : 0u);
            } else if (V == 3) {  // speculative + sign test: X = state if the current entry is taken here
                double X[D];
                int neg = 0;
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    X[d] = BINS ? __dsub_rn(S[d], r[d]) : __dadd_rn(S[d], r[d]);
                    neg |= __double2hiint(BINS ? X[d] : __dsub_rn(C[d], X[d]));
                }
                bool ok = neg >= 0;
                for (int k0 = 0; k0 < 32; k0 += 4)
#pragma unroll
                for (int k = k0; k < k0 + 4; ++k) {
                    double rn[D], XA[D], XB[D];
                    load_row(rn, brow + (size_t)(k + 1) * D);
                    int negA = 0, negB = 0;
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        XA[d] = BINS ? __dsub_rn(S[d], rn[d]) : __dadd_rn(S[d], rn[d]);
                        XB[d] = BINS ? __dsub_rn(X[d], rn[d]) : __dadd_rn(X[d], rn[d]);
                        negA |= __double2hiint(BINS ? XA[d] : __dsub_rn(C[d], XA[d]));
                        negB |= __double2hiint(BINS ? XB[d] : __dsub_rn(C[d], XB[d]));
                    }
                    const unsigned m = __ballot_sync(0xFFFFFFFFu, ok);
                    const bool mine = ok && !(m & lt);
#pragma unroll
                    for (int d = 0; d < D; ++d) { S[d] = mine ? X[d] : S[d]; X[d] = mine ? XB[d] : XA[d]; }
                    ok = (mine ? negB : negA) >= 0;
                    mymask |= (mine ? 1u : 0u) << k;
                }
            } else {
                bool ok = true;
#pragma unroll
                for (int d = 0; d < D; ++d) {
                    if (BINS) ok = ok & (r[d] <= S[d]);
                    else ok = ok & (__dsub_rn(C[d], __dadd_rn(S[d], r[d])) >= 0.0);
                }
                for (int k0 = 0; k0 < 32; k0 += 4)
#pragma unroll
                for (int k = k0; k < k0 + 4; ++k) {
                    double rn[D], S2[D];
                    load_row(rn, brow + (size_t)(k + 1) * D);
                    bool okA = true, okB = true;
#pragma unroll
                    for (int d = 0; d < D; ++d) {
                        S2[d] = BINS ? __dsub_rn(S[d], r[d]) : __dadd_rn(S[d], r[d]);
                        if (BINS) {
                            okA = okA & (rn[d] <= S[d]);
                            okB = okB & (rn[d] <= S2[d]);
                        } else {
                            okA = okA & (__dsub_rn(C[d], __dadd_rn(S[d], rn[d])) >= 0.0);
                            okB = okB & (__dsub_rn(C[d], __dadd_rn(S2[d], rn[d])) >= 0.0);
                        }
                    }
                    const unsigned m = __ballot_sync(0xFFFFFFFFu, ok);
                    const bool mine = ok && !(m & lt);
#pragma unroll
                    for (int d = 0; d < D; ++d) S[d] = mine ? S2[d] : S[d];
                    ok = mine ? okB : okA;
                    if (m) {
                        if (lane == 0) fnd[k] = (unsigned char)(__ffs(m) - 1);
                        took |= 1u << k;
                    }
#pragma unroll
                    for (int d = 0; d < D; ++d) r[d] = rn[d];
                }
            }
            if (V >= 4) {} else if (V >= 2) {  // who took entry `lane`?  one ballot per placed entry, off the dependent chain
                took = __reduce_or_sync(0xFFFFFFFFu, mymask);
                unsigned f = 0;
                for (unsigned t = took; t; t &= t - 1) {
                    const int k = __ffs(t) - 1;
                    const unsigned b = __ballot_sync(0xFFFFFFFFu, (mymask >> k) & 1u);
                    if (lane == k) f = __ffs(b) - 1;
                }
                check = check * 31u + took + f;
            } else {
            __syncwarp();
            check = check * 31u + took + (((took >> lane) & 1u) ? fnd[lane] : 0u);
            }
        }
        total += clock64() - t0;
#pragma unroll
        for (int d = 0; d < D; ++d) check += (unsigned)(__double_as_longlong(S[d]) >> 20);
        __syncwarp();
    }
    for (int o = 16; o > 0; o >>= 1) check += __shfl_xor_sync(0xFFFFFFFFu, check, o);
    if (threadIdx.x == 0) { *cyc = total; *out_sum = check; }
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
    double *d; long long *cyc; unsigned *chk;
    cudaMalloc(&d, sizeof h); cudaMalloc(&cyc, 8); cudaMalloc(&chk, 4);
    cudaMemcpy(d, h, sizeof h, cudaMemcpyHostToDevice);
    const int reps = 200;
    for (int bins = 1; bins >= 0; --bins)
    for (int nw = 1; nw <= 8; nw *= 8)
    for (int v = 0; v < 11; v += (v == 0 ? 7 : 1)) {
        long long c = 0;
        for (int it = 0; it < 2; ++it) {
            if (v == 0 && bins) resolver<0, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 1 && bins) resolver<1, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 2 && bins) resolver<2, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 3 && bins) resolver<3, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 2 && !bins) resolver<2, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 3 && !bins) resolver<3, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 4 && bins) resolver<4, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 5 && bins) resolver<5, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 4 && !bins) resolver<4, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 5 && !bins) resolver<5, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 6 && bins) resolver<6, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 6 && !bins) resolver<6, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 7 && bins) resolver<7, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 7 && !bins) resolver<7, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 8 && bins) resolver<8, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 8 && !bins) resolver<8, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 9 && bins) resolver<9, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 9 && !bins) resolver<9, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 10 && bins) resolver<10, true><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 10 && !bins) resolver<10, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 0 && !bins) resolver<0, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            if (v == 1 && !bins) resolver<1, false><<<1, 32 * nw>>>(d, 0.0, 2.0, 7096762368.0, 110.0, cyc, chk, reps);
            cudaMemcpy(&c, cyc, 8, cudaMemcpyDeviceToHost);
        }
        unsigned ps; cudaMemcpy(&ps, chk, 4, cudaMemcpyDeviceToHost);
        printf("%s warps %d variant %d: %.1f cycles / entry  (checksum %08x) %s\n", bins ? "bins " : "nodes", nw, v,
               (double)c / (reps * NE), ps, cudaGetErrorString(cudaGetLastError()));
    }
    return 0;
}
