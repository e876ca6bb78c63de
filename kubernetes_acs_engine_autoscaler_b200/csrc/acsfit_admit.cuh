// acsfit_admit.cuh -- the pending-pod admission test of node states with pod anti-affinity, pod affinity and hostname
// topology spread (acsfit_pending_admit, acsfit_pending_admit_pa, acsfit_pending_admit_ts, include/acsfit.h): which
// nodes some pod to schedule could land on, given the pods already there.
#pragma once
#include <cstdint>

namespace acsfit {

constexpr int kAdmitBlock = 256;  // threads per CTA = nodes per CTA = signatures per shared-memory tile
constexpr int kAdmitSmem = kAdmitBlock * (2 * 8 + 1);  // static shared bytes per CTA: one tile of the table
constexpr int kAdmitSmemPa = kAdmitBlock * (8 + 1);    // ... of the pod-affinity-only form (class, need)
constexpr int kAdmitSmemAaPa = kAdmitBlock * (3 * 8 + 1);  // ... of the combined form (class, carries, matches, need)
// ... of the topology-spread forms: the columns of the AA / PA form plus key (1 byte) and limit (4 bytes)
constexpr int admit_smem_ts(bool aa, bool pa) { return kAdmitBlock * ((aa ? 16 : 0) + (pa ? 8 : 0) + 1 + 1 + 4); }
constexpr uint8_t kNodeNoPendingMatch = 2u;  // ACSFIT_NODEF_NO_PENDING_MATCH
constexpr uint8_t kAdmitNoKey = 0xFFu;       // a signature without a spread constraint

// One thread per node.  The thread ORs the masks of the node's CSR slice (rows row_ptr[n] .. row_ptr[n+1], absolute):
// carries / matches into NC / NX with AA, has into HAS with PA.  It then walks the signature table, which the CTA
// stages through shared memory one tile at a time.  A signature (class, carries, matches, need) admits the node when
// the node matches the class, with AA (carries & NX) | (matches & NC) == 0, and with PA need == 0 or
// (need & HAS) != 0.  A thread stops testing once a signature admits its node, and the CTA stops loading tiles once
// every node of it is admitted.  Nodes no signature admits gain the flag bit; no other bit changes.  A form reads only
// the arrays of its tests (the PA-only form never touches the anti-affinity masks).  With TS a signature with a key
// (key != 0xFF) also needs node_count[key * N + n] <= limit, its skew plus the key's minimum (the host computes it);
// that global load comes after the shared-memory tests, so it runs only for signatures that pass them.  The TS form
// without AA and PA never reads the row table.  New arrays come last so that the earlier forms keep their parameter
// layout.
template <bool AA, bool PA, bool TS>
__global__ void __launch_bounds__(kAdmitBlock)
pending_admit_kernel(const int64_t *__restrict__ row_ptr, const unsigned long long *__restrict__ run_carries,
                     const unsigned long long *__restrict__ run_matches, int64_t N,
                     const unsigned long long *__restrict__ node_match, const uint8_t *__restrict__ sig_class,
                     const unsigned long long *__restrict__ sig_carries,
                     const unsigned long long *__restrict__ sig_matches, int U, uint8_t *__restrict__ node_flags,
                     const unsigned long long *__restrict__ run_has, const unsigned long long *__restrict__ sig_need,
                     const uint8_t *__restrict__ sig_key, const int32_t *__restrict__ sig_limit,
                     const int32_t *__restrict__ node_count)
{
    __shared__ unsigned long long s_carries[AA ? kAdmitBlock : 1], s_matches[AA ? kAdmitBlock : 1];
    __shared__ unsigned long long s_need[PA ? kAdmitBlock : 1];
    __shared__ uint8_t s_class[kAdmitBlock];
    __shared__ int32_t s_limit[TS ? kAdmitBlock : 1];
    __shared__ uint8_t s_key[TS ? kAdmitBlock : 1];
    const int t = threadIdx.x;
    const int64_t n = (int64_t)blockIdx.x * kAdmitBlock + t;
    unsigned long long nc = 0, nx = 0, has = 0, classes = ~0ull;
    bool open = n < N;  // no signature has admitted the node yet
    if (open) {
        if constexpr (AA || PA)
            for (int64_t k = row_ptr[n], e = row_ptr[n + 1]; k < e; ++k) {
                if constexpr (AA) {
                    nc |= run_carries[k];
                    nx |= run_matches[k];
                }
                if constexpr (PA) has |= run_has[k];
            }
        if (node_match) classes = node_match[n];
    }
    for (int base = 0; base < U; base += kAdmitBlock) {
        if (!__syncthreads_or(open)) break;  // also the barrier before the tile is overwritten
        const int cnt = min(kAdmitBlock, U - base);
        if (t < cnt) {
            s_class[t] = sig_class[base + t];
            if constexpr (AA) {
                s_carries[t] = sig_carries[base + t];
                s_matches[t] = sig_matches[base + t];
            }
            if constexpr (PA) s_need[t] = sig_need[base + t];
            if constexpr (TS) {
                s_key[t] = sig_key[base + t];
                s_limit[t] = sig_limit[base + t];
            }
        }
        __syncthreads();
        for (int j = 0; open && j < cnt; ++j)
            if (((classes >> s_class[j]) & 1ull) && (!AA || ((s_carries[j] & nx) | (s_matches[j] & nc)) == 0) &&
                (!PA || s_need[j] == 0 || (s_need[j] & has) != 0) &&
                (!TS || s_key[j] == kAdmitNoKey || node_count[(int64_t)s_key[j] * N + n] <= s_limit[j]))
                open = false;
    }
    if (open) node_flags[n] |= kNodeNoPendingMatch;
}

}  // namespace acsfit
