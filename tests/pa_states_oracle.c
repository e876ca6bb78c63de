/*
 * pa_states_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, single-threaded statement of the pending-pod admission rule of node states with required pod affinity
 * (include/acsfit.h, acsfit_pending_admit_pa), per node and per pod to schedule, without deduplicating the pods:
 *   NC(n), NX(n), HAS(n)  the OR of carries / matches / has over the rows row_ptr[n] .. row_ptr[n+1]
 *   admits(n, p)  bit pod_class[p] of node_match[n] is set (always, when node_match is NULL)
 *                 and, when run_carries is not NULL, (pod_carries[p] & NX(n)) | (pod_matches[p] & NC(n)) == 0
 *                 and pod_need[p] == 0 or (pod_need[p] & HAS(n)) != 0
 *   node n gains ACSFIT_NODEF_NO_PENDING_MATCH (bit 1) when no p admits it; no other bit changes.
 * With every need 0 it is tests/aa_states_oracle.c.  tests/pa_states_oracle.py compiles it with the flags of
 * oracle/Makefile.
 */
#include <stdint.h>

#define ORACLE_API __attribute__((visibility("default")))
#define NODEF_NO_PENDING_MATCH 2u

ORACLE_API void oracle_pending_admit_pa(const int64_t *row_ptr, const uint64_t *run_carries,
                                        const uint64_t *run_matches, const uint64_t *run_has, int64_t N,
                                        const uint64_t *node_match, const uint8_t *pod_class,
                                        const uint64_t *pod_carries, const uint64_t *pod_matches,
                                        const uint64_t *pod_need, int64_t P, uint8_t *node_flags)
{
    for (int64_t n = 0; n < N; ++n) {
        uint64_t nc = 0, nx = 0, has = 0;
        for (int64_t k = row_ptr[n]; k < row_ptr[n + 1]; ++k) {
            if (run_carries) {
                nc |= run_carries[k];
                nx |= run_matches[k];
            }
            has |= run_has[k];
        }
        int admitted = 0;
        for (int64_t p = 0; p < P && !admitted; ++p) {
            const int match = node_match == 0 || ((node_match[n] >> pod_class[p]) & 1u);
            const int blocked = run_carries && ((pod_carries[p] & nx) | (pod_matches[p] & nc)) != 0;
            const int affine = pod_need[p] == 0 || (pod_need[p] & has) != 0;
            admitted = match && !blocked && affine;
        }
        if (!admitted) node_flags[n] |= NODEF_NO_PENDING_MATCH;
    }
}
