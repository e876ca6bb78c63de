/*
 * pa_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, single-threaded restatement of the node pass and the bin pass WITH required pod affinity (the opt-in mode of
 * include/acsfit.h, acsfit_pod_affinity), on top of node selectors and anti-affinity as tests/aa_oracle.c states them.
 * It keeps one boolean per signature ("some pod anywhere matches it"), updated at every placement: no flip positions,
 * no reruns, so it checks the GPU's scheme independently.
 *   affine(p, has) = requires[p] == 0 || (requires[p] & has) != 0 || (self[p] != 0 && !present[sig of p])
 *   first fit   : the first node with affine and !blocked and match and can_fit; the node's has mask and `present`
 *                 then gain matches[p]                                          (one call per node visited)
 *   bin packing : pool gate as in aa_oracle.c; the first bin with affine and !blocked and a fit, else a new bin when
 *                 affine(p, 0) holds, else the pod is left out of this pool's bins.  Credited tests: a placed pod's
 *                 bins before its bin, plus its bin unless it opened it; a pod left out is credited none.
 *                 `present` starts from the argument and carries from pool to pool
 * Flips: for each pass (the node pass, each pool's packing) the signatures absent at its start that some pod of the
 * call matches itself are watched; the first placement of a pod matching one is reported as (signature, position),
 * sorted by position, then signature -- the order in which the GPU fixes them.
 * With every affinity mask 0 each function is exactly its counterpart in tests/aa_oracle.c.
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

static int affine(uint64_t requires, uint64_t self, uint64_t has, uint64_t present)
{
    return requires == 0 || (requires & has) != 0 || (self != 0 && (self & present) == 0);
}

/* flips: record the first placement of each watched signature; out holds (sig, pos) pairs in placement order, which
 * is position order; pairs of one position come in signature order */
static void note_placed(uint64_t matches, uint64_t *watch, int64_t pos, int64_t *flips, int64_t *n_flips)
{
    uint64_t w = matches & *watch;
    for (int s = 0; s < 64; ++s)
        if ((w >> s) & 1u) {
            flips[2 * *n_flips] = s;
            flips[2 * *n_flips + 1] = pos;
            ++*n_flips;
        }
    *watch &= ~w;
}

ORACLE_API uint64_t oracle_first_fit_nodes_pa(const double *req, int64_t P, int D, const double *cap_type,
                                              const int32_t *node_type, double *used, int64_t N,
                                              const uint64_t *node_match, const uint8_t *pod_class,
                                              const uint64_t *pod_carries, const uint64_t *pod_matches,
                                              uint64_t *node_carries, uint64_t *node_matches,
                                              const uint64_t *pod_requires, const uint64_t *pod_self,
                                              const uint64_t *pod_aff_matches, uint64_t *node_has, int32_t *placed,
                                              int64_t *flips, int64_t *n_flips)
{
    uint64_t calls = 0, present = 0, selfs = 0;
    for (int64_t n = 0; n < N; ++n) present |= node_has[n];
    for (int64_t p = 0; p < P; ++p) selfs |= pod_self[p];
    uint64_t watch = selfs & ~present;
    *n_flips = 0;
    for (int64_t p = 0; p < P; ++p) {
        const double *r = req + (size_t)p * D;
        int64_t hit = -1;
        for (int64_t n = 0; n < N; ++n) {
            ++calls;
            if (affine(pod_requires[p], pod_self[p], node_has[n], present) &&
                !blocked(pod_carries[p], pod_matches[p], node_carries[n], node_matches[n]) &&
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
            node_has[hit] |= pod_aff_matches[p];
            present |= pod_aff_matches[p];
            note_placed(pod_aff_matches[p], &watch, p, flips, n_flips);
        }
    }
    return calls;
}

/* flips: room for 64 pairs per pool */
ORACLE_API uint64_t oracle_fulfill_pending_pa(const double *req, int64_t Pp, int64_t num_listed, int D,
                                              const double *unit, const int32_t *pool_actual,
                                              const int32_t *pool_max, const uint8_t *pool_ignored, int T,
                                              int64_t over_provision, const uint64_t *pool_match,
                                              const uint8_t *pod_class, const uint64_t *pod_carries,
                                              const uint64_t *pod_matches, const uint64_t *pod_requires,
                                              const uint64_t *pod_self, const uint64_t *pod_aff_matches,
                                              uint64_t present, int64_t *new_size, int64_t *units_needed,
                                              int64_t *bins_opened, int32_t *acc_pool, int32_t *bin_of,
                                              int64_t *out_unaccounted, int64_t *flips, int64_t *n_flips)
{
    uint64_t evals = 0, selfs = 0;
    int64_t num_unaccounted = num_listed;
    const size_t cap = (size_t)(Pp > 0 ? Pp : 1);
    double *bins = (double *)malloc(sizeof(double) * cap * D);
    uint64_t *bin_c = (uint64_t *)malloc(sizeof(uint64_t) * cap);
    uint64_t *bin_m = (uint64_t *)malloc(sizeof(uint64_t) * cap);
    uint64_t *bin_h = (uint64_t *)malloc(sizeof(uint64_t) * cap);
    int32_t *cur_bin = (int32_t *)malloc(sizeof(int32_t) * cap);
    for (int64_t p = 0; p < Pp; ++p) { acc_pool[p] = -1; bin_of[p] = -1; selfs |= pod_self[p]; }
    *n_flips = 0;

    for (int t = 0; t < T; ++t) {
        const double *u = unit + (size_t)t * D;
        new_size[t] = pool_actual[t];
        units_needed[t] = -1;
        bins_opened[t] = 0;
        if (pool_ignored[t] || !num_unaccounted) continue;

        uint64_t watch = selfs & ~present;
        int64_t nb = 0;
        for (int64_t p = 0; p < Pp; ++p) {
            cur_bin[p] = -1;
            if (acc_pool[p] >= 0) continue;
            const double *r = req + (size_t)p * D;
            ++evals;
            if (!(match(pool_match[t], pod_class[p]) && sub_possible(u, r, D))) continue;
            int64_t hit = -1;
            for (int64_t i = 0; i < nb; ++i) {
                if (affine(pod_requires[p], pod_self[p], bin_h[i], present) &&
                    !blocked(pod_carries[p], pod_matches[p], bin_c[i], bin_m[i]) &&
                    sub_possible(bins + (size_t)i * D, r, D)) {
                    hit = i;
                    evals += (uint64_t)i + 1;
                    break;
                }
            }
            if (hit < 0) {
                if (!affine(pod_requires[p], pod_self[p], 0, present)) continue;  /* opens no bin */
                evals += (uint64_t)nb;
                hit = nb++;
                for (int d = 0; d < D; ++d) bins[(size_t)hit * D + d] = u[d];
                bin_c[hit] = 0;
                bin_m[hit] = 0;
                bin_h[hit] = 0;
            }
            for (int d = 0; d < D; ++d) {
                double left = bins[(size_t)hit * D + d] - r[d];
                bins[(size_t)hit * D + d] = left;
            }
            bin_c[hit] |= pod_carries[p];
            bin_m[hit] |= pod_matches[p];
            bin_h[hit] |= pod_aff_matches[p];
            present |= pod_aff_matches[p];
            note_placed(pod_aff_matches[p], &watch, p, flips, n_flips);
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
    free(bin_h);
    free(cur_bin);
    *out_unaccounted = num_unaccounted;
    return evals;
}
