/*
 * ts_states_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, single-threaded statement of the pending-pod admission rule of node states with hostname topology spread
 * (include/acsfit.h, acsfit_pending_admit_ts), per node and per pod to schedule, without deduplicating the pods:
 *   admits(n, p)  the rule of tests/pa_states_oracle.c (the affinity part only when run_has is not NULL)
 *                 and pod_key[p] == 0xFF or node_count[pod_key[p] * N + n] <= pod_skew[p] + min(pod_key[p])
 *   min(k)        min(floor[k], node_count[k * N + m] over the nodes m with bit k in node_domain), computed here from
 *                 the counts, domains and floor (not handed in), in 64 bits
 *   node n gains ACSFIT_NODEF_NO_PENDING_MATCH (bit 1) when no p admits it; no other bit changes.
 * With every key 0xFF it is tests/pa_states_oracle.c.  tests/ts_states_oracle.py compiles it with the flags of
 * oracle/Makefile.
 */
#include <stdint.h>

#define ORACLE_API __attribute__((visibility("default")))
#define NODEF_NO_PENDING_MATCH 2u

static long long key_min(const int32_t *node_count, const uint64_t *node_domain, const int32_t *floor, int64_t N,
                         int k)
{
    long long m = floor[k];
    for (int64_t n = 0; n < N; ++n)
        if (((node_domain[n] >> k) & 1u) && node_count[(int64_t)k * N + n] < m) m = node_count[(int64_t)k * N + n];
    return m;
}

ORACLE_API void oracle_pending_admit_ts(const int64_t *row_ptr, const uint64_t *run_carries,
                                        const uint64_t *run_matches, const uint64_t *run_has, int64_t N,
                                        const uint64_t *node_match, const uint8_t *pod_class,
                                        const uint64_t *pod_carries, const uint64_t *pod_matches,
                                        const uint64_t *pod_need, const uint8_t *pod_key, const int32_t *pod_skew,
                                        int64_t P, const int32_t *node_count, const uint64_t *node_domain,
                                        const int32_t *floor, uint8_t *node_flags)
{
    long long mins[64];
    for (int64_t p = 0; p < P; ++p)
        if (pod_key[p] != 0xFF) mins[pod_key[p]] = key_min(node_count, node_domain, floor, N, pod_key[p]);
    for (int64_t n = 0; n < N; ++n) {
        uint64_t nc = 0, nx = 0, has = 0;
        for (int64_t k = row_ptr[n]; k < row_ptr[n + 1]; ++k) {
            if (run_carries) {
                nc |= run_carries[k];
                nx |= run_matches[k];
            }
            if (run_has) has |= run_has[k];
        }
        int admitted = 0;
        for (int64_t p = 0; p < P && !admitted; ++p) {
            const int match = node_match == 0 || ((node_match[n] >> pod_class[p]) & 1u);
            const int blocked = run_carries && ((pod_carries[p] & nx) | (pod_matches[p] & nc)) != 0;
            const int affine = !run_has || pod_need[p] == 0 || (pod_need[p] & has) != 0;
            const int k = pod_key[p];
            const int spread = k == 0xFF || (long long)node_count[(int64_t)k * N + n] <=
                                                (long long)pod_skew[p] + mins[k];
            admitted = match && !blocked && affine && spread;
        }
        if (!admitted) node_flags[n] |= NODEF_NO_PENDING_MATCH;
    }
}
