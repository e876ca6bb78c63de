/*
 * aa_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, single-threaded restatement of the node pass and the bin pass WITH required pod anti-affinity (the opt-in
 * mode of include/acsfit.h, acsfit_anti_affinity), on the layout and with the arithmetic of tests/sel_oracle.c.  The
 * block test is evaluated first (with the selector match) and short-circuits; it is not an extra evaluation:
 *   blocked(p, x) = (carries[p] & x.matches) | (matches[p] & x.carries) != 0
 *   first fit   : the first node with  !blocked and match(node) and node.can_fit(req); the node's masks then gain
 *                 the pod's                                                      (one call per node visited)
 *   bin packing : pool gate  match(pool) and (unit - req).possible; the first bin with !blocked and a fit, else a new
 *                 bin with both masks 0; the bin's masks then gain the pod's      (one per gate and bin test)
 * With every mask 0 each function is exactly its counterpart in tests/sel_oracle.c.  tests/aa_oracle.py compiles it
 * with the same flags as oracle/Makefile.
 */
#include <stdint.h>
#include <stdlib.h>

#define ORACLE_API __attribute__((visibility("default")))

static int sub_possible(const double *a, const double *b, int D)
{
    for (int d = 0; d < D; ++d) {
        double diff = a[d] - b[d];
        if (!(diff >= 0)) return 0;
    }
    return 1;
}

static int node_can_fit(const double *cap, const double *used, const double *req, int D)
{
    for (int d = 0; d < D; ++d) {
        double s = used[d] + req[d];
        double left = cap[d] - s;
        if (!(left >= 0)) return 0;
    }
    return 1;
}

static int match(uint64_t mask, uint8_t cls) { return (int)((mask >> cls) & 1u); }

static int blocked(uint64_t pc, uint64_t pm, uint64_t xc, uint64_t xm) { return ((pc & xm) | (pm & xc)) != 0; }

ORACLE_API uint64_t oracle_first_fit_nodes_aa(const double *req, int64_t P, int D, const double *cap_type,
                                              const int32_t *node_type, double *used, int64_t N,
                                              const uint64_t *node_match, const uint8_t *pod_class,
                                              const uint64_t *pod_carries, const uint64_t *pod_matches,
                                              uint64_t *node_carries, uint64_t *node_matches, int32_t *placed)
{
    uint64_t calls = 0;
    for (int64_t p = 0; p < P; ++p) {
        const double *r = req + (size_t)p * D;
        int64_t hit = -1;
        for (int64_t n = 0; n < N; ++n) {
            ++calls;
            if (!blocked(pod_carries[p], pod_matches[p], node_carries[n], node_matches[n]) &&
                match(node_match[n], pod_class[p]) &&
                node_can_fit(cap_type + (size_t)node_type[n] * D, used + (size_t)n * D, r, D)) {
                hit = n;
                break;
            }
        }
        placed[p] = (int32_t)hit;
        if (hit >= 0) {
            for (int d = 0; d < D; ++d) {
                double s = used[(size_t)hit * D + d] + r[d];
                used[(size_t)hit * D + d] = s;
            }
            node_carries[hit] |= pod_carries[p];
            node_matches[hit] |= pod_matches[p];
        }
    }
    return calls;
}

ORACLE_API uint64_t oracle_fulfill_pending_aa(const double *req, int64_t Pp, int64_t num_listed, int D,
                                              const double *unit, const int32_t *pool_actual,
                                              const int32_t *pool_max, const uint8_t *pool_ignored, int T,
                                              int64_t over_provision, const uint64_t *pool_match,
                                              const uint8_t *pod_class, const uint64_t *pod_carries,
                                              const uint64_t *pod_matches, int64_t *new_size, int64_t *units_needed,
                                              int64_t *bins_opened, int32_t *acc_pool, int32_t *bin_of,
                                              int64_t *out_unaccounted)
{
    uint64_t evals = 0;
    int64_t num_unaccounted = num_listed;
    const size_t cap = (size_t)(Pp > 0 ? Pp : 1);
    double *bins = (double *)malloc(sizeof(double) * cap * D);
    uint64_t *bin_c = (uint64_t *)malloc(sizeof(uint64_t) * cap);
    uint64_t *bin_m = (uint64_t *)malloc(sizeof(uint64_t) * cap);
    int32_t *cur_bin = (int32_t *)malloc(sizeof(int32_t) * cap);
    for (int64_t p = 0; p < Pp; ++p) { acc_pool[p] = -1; bin_of[p] = -1; }

    for (int t = 0; t < T; ++t) {
        const double *u = unit + (size_t)t * D;
        new_size[t] = pool_actual[t];
        units_needed[t] = -1;
        bins_opened[t] = 0;
        if (pool_ignored[t] || !num_unaccounted) continue;

        int64_t nb = 0;
        for (int64_t p = 0; p < Pp; ++p) {
            cur_bin[p] = -1;
            if (acc_pool[p] >= 0) continue;
            const double *r = req + (size_t)p * D;
            ++evals;
            if (!(match(pool_match[t], pod_class[p]) && sub_possible(u, r, D))) continue;
            int64_t hit = -1;
            for (int64_t i = 0; i < nb; ++i) {
                ++evals;
                if (!blocked(pod_carries[p], pod_matches[p], bin_c[i], bin_m[i]) &&
                    sub_possible(bins + (size_t)i * D, r, D)) {
                    hit = i;
                    break;
                }
            }
            if (hit < 0) {
                hit = nb++;
                for (int d = 0; d < D; ++d) bins[(size_t)hit * D + d] = u[d];
                bin_c[hit] = 0;
                bin_m[hit] = 0;
            }
            for (int d = 0; d < D; ++d) {
                double left = bins[(size_t)hit * D + d] - r[d];
                bins[(size_t)hit * D + d] = left;
            }
            bin_c[hit] |= pod_carries[p];
            bin_m[hit] |= pod_matches[p];
            cur_bin[p] = (int32_t)hit;
            bin_of[p] = (int32_t)hit;
        }
        int64_t needed = nb + over_provision;
        int64_t room = (int64_t)pool_max[t] - (int64_t)pool_actual[t];
        int64_t unavailable = needed - room > 0 ? needed - room : 0;
        int64_t requested = needed - unavailable;
        units_needed[t] = needed;
        bins_opened[t] = nb;
        new_size[t] = (int64_t)pool_actual[t] + requested;
        int64_t take = nb < requested ? nb : requested;
        for (int64_t p = 0; p < Pp; ++p)
            if (cur_bin[p] >= 0 && cur_bin[p] < take) {
                acc_pool[p] = t;
                --num_unaccounted;
            }
    }
    free(bins);
    free(bin_c);
    free(bin_m);
    free(cur_bin);
    *out_unaccounted = num_unaccounted;
    return evals;
}
