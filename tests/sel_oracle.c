/*
 * sel_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, single-threaded restatement of the scale-up decision path WITH node selectors (the opt-in mode of
 * include/acsfit.h, acsfit_selectors), on the dense float64 layout of oracle/acsfit_oracle.c and with the same
 * arithmetic in the same order.  The only addition is the match test, evaluated first:
 *   feasibility : some pool with  match(pool) and (unit - req).possible          (one evaluation per pool visited)
 *   first fit   : the first node with  match(node) and node.can_fit(req)           (one call per node visited)
 *   bin packing : pool gate  match(pool) and (unit - req).possible; bins unchanged  (one per gate and bin test)
 * match(x) = bit pod_class[p] of x's mask.  With every pod in class 0 each function is exactly its counterpart in
 * oracle/acsfit_oracle.c.  tests/sel_oracle.py compiles it with the same flags as oracle/Makefile.
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

ORACLE_API uint64_t oracle_feasible_mask_sel(const double *req, int64_t P, int D, const double *unit, int T,
                                             const uint64_t *pool_match, const uint8_t *pod_class,
                                             uint8_t *out_mask)
{
    uint64_t evals = 0;
    for (int64_t p = 0; p < P; ++p) {
        uint8_t ok = 0;
        for (int t = 0; t < T; ++t) {
            ++evals;
            if (match(pool_match[t], pod_class[p]) && sub_possible(unit + (size_t)t * D, req + (size_t)p * D, D)) {
                ok = 1;
                break;
            }
        }
        out_mask[p] = ok;
    }
    return evals;
}

ORACLE_API uint64_t oracle_first_fit_nodes_sel(const double *req, int64_t P, int D, const double *cap_type,
                                               const int32_t *node_type, double *used, int64_t N,
                                               const uint64_t *node_match, const uint8_t *pod_class,
                                               int32_t *placed)
{
    uint64_t calls = 0;
    for (int64_t p = 0; p < P; ++p) {
        const double *r = req + (size_t)p * D;
        int64_t hit = -1;
        for (int64_t n = 0; n < N; ++n) {
            ++calls;
            if (match(node_match[n], pod_class[p]) &&
                node_can_fit(cap_type + (size_t)node_type[n] * D, used + (size_t)n * D, r, D)) {
                hit = n;
                break;
            }
        }
        placed[p] = (int32_t)hit;
        if (hit >= 0)
            for (int d = 0; d < D; ++d) {
                double s = used[(size_t)hit * D + d] + r[d];
                used[(size_t)hit * D + d] = s;
            }
    }
    return calls;
}

ORACLE_API uint64_t oracle_fulfill_pending_sel(const double *req, int64_t Pp, int64_t num_listed, int D,
                                               const double *unit, const int32_t *pool_actual,
                                               const int32_t *pool_max, const uint8_t *pool_ignored, int T,
                                               int64_t over_provision, const uint64_t *pool_match,
                                               const uint8_t *pod_class, int64_t *new_size, int64_t *units_needed,
                                               int64_t *bins_opened, int32_t *acc_pool, int32_t *bin_of,
                                               int64_t *out_unaccounted)
{
    uint64_t evals = 0;
    int64_t num_unaccounted = num_listed;
    double *bins = (double *)malloc(sizeof(double) * (size_t)(Pp > 0 ? Pp : 1) * D);
    int32_t *cur_bin = (int32_t *)malloc(sizeof(int32_t) * (size_t)(Pp > 0 ? Pp : 1));
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
                if (sub_possible(bins + (size_t)i * D, r, D)) { hit = i; break; }
            }
            if (hit < 0) {
                hit = nb++;
                for (int d = 0; d < D; ++d) bins[(size_t)hit * D + d] = u[d];
            }
            for (int d = 0; d < D; ++d) {
                double left = bins[(size_t)hit * D + d] - r[d];
                bins[(size_t)hit * D + d] = left;
            }
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
    free(cur_bin);
    *out_unaccounted = num_unaccounted;
    return evals;
}
