/*
 * ts_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Plain-C, single-threaded restatement of the node pass and the bin pass WITH hostname topology spread (the opt-in
 * mode of include/acsfit.h, acsfit_topology_spread), on top of node selectors, anti-affinity and pod affinity as
 * tests/pa_oracle.c states them.  It recomputes each key's minimum from the current counts at every pod: no levels,
 * no rises fixed ahead, no reruns, so it checks the GPU's scheme independently.
 *   spread(p, n)  pod_key[p] == 0xFF || cnt[key][n] + self - min(key) <= maxSkew, i.e. cnt[key][n] <= pod_skew[p] +
 *                 min(key); min(key) = min(floor[key], cnt[key][m] over the nodes m with bit key in node_domain)
 *   first fit   : the first node with spread, affine, !blocked, match and can_fit; the node's counts of every key of
 *                 ts_matches[p] then grow by 1                                      (one call per node visited)
 *   bin packing : as tests/pa_oracle.c, with spread(p, bin) for min = 0: cnt[key][bin] <= pod_skew[p]; a new bin
 *                 starts with count 0 and so always admits
 * Rises: every time a placement raises a key's minimum, (key, position) is reported, in position order then key order
 * -- the order in which the GPU fixes them.  The node pass follows `follow` rises at most (< 0: all): once that many
 * are reported no key's minimum moves again, as the GPU keeps its levels after its last fixed rise; flips are still
 * followed.  With every pod_key 0xFF each function is exactly its counterpart in tests/pa_oracle.c (flips included).
 */
#include <limits.h>
#include <stdint.h>
#include <stdlib.h>

#define ORACLE_API __attribute__((visibility("default")))
#define NO_KEY 0xFF

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

/* the minimum of key k now: floor[k] and the counts of its domains among the N nodes */
static long long key_min(const int32_t *count, const uint64_t *domain, const int32_t *floor, int64_t N, int k)
{
    long long m = floor[k];
    for (int64_t n = 0; n < N; ++n)
        if (((domain[n] >> k) & 1u) && count[(size_t)k * N + n] < m) m = count[(size_t)k * N + n];
    return m;
}

/* rises: room for `max_rises` pairs; `follow` (< 0: no limit) as above */
ORACLE_API uint64_t oracle_first_fit_nodes_ts(const double *req, int64_t P, int D, const double *cap_type,
                                              const int32_t *node_type, double *used, int64_t N,
                                              const uint64_t *node_match, const uint8_t *pod_class,
                                              const uint64_t *pod_carries, const uint64_t *pod_matches,
                                              uint64_t *node_carries, uint64_t *node_matches,
                                              const uint64_t *pod_requires, const uint64_t *pod_self,
                                              const uint64_t *pod_aff_matches, uint64_t *node_has, int keys,
                                              const uint8_t *pod_key, const int32_t *pod_skew,
                                              const uint64_t *ts_matches, int32_t *node_count,
                                              const uint64_t *node_domain, const int32_t *floor, int32_t *placed,
                                              int64_t *flips, int64_t *n_flips, int64_t *rises, int64_t *n_rises,
                                              int64_t max_rises, int64_t follow)
{
    uint64_t calls = 0, present = 0, selfs = 0;
    long long cur[64];
    for (int64_t n = 0; n < N; ++n) present |= node_has[n];
    for (int64_t p = 0; p < P; ++p) selfs |= pod_self[p];
    for (int k = 0; k < keys; ++k) cur[k] = key_min(node_count, node_domain, floor, N, k);
    uint64_t watch = selfs & ~present;
    *n_flips = 0;
    *n_rises = 0;
    for (int64_t p = 0; p < P; ++p) {
        const double *r = req + (size_t)p * D;
        const int k = pod_key[p];
        int64_t hit = -1;
        for (int64_t n = 0; n < N; ++n) {
            ++calls;
            if ((k == NO_KEY || (long long)node_count[(size_t)k * N + n] <= (long long)pod_skew[p] + cur[k]) &&
                affine(pod_requires[p], pod_self[p], node_has[n], present) &&
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
            for (int b = 0; b < keys; ++b) {
                if (!((ts_matches[p] >> b) & 1u)) continue;
                ++node_count[(size_t)b * N + hit];
                if (follow >= 0 && *n_rises >= follow) continue;  /* past the last followed rise */
                const long long m = key_min(node_count, node_domain, floor, N, b);
                if (m > cur[b] && *n_rises < max_rises) {
                    rises[2 * *n_rises] = b;
                    rises[2 * *n_rises + 1] = p;
                    ++*n_rises;
                }
                cur[b] = m;
            }
        }
    }
    return calls;
}

/* flips: room for 64 pairs per pool */
ORACLE_API uint64_t oracle_fulfill_pending_ts(const double *req, int64_t Pp, int64_t num_listed, int D,
                                              const double *unit, const int32_t *pool_actual,
                                              const int32_t *pool_max, const uint8_t *pool_ignored, int T,
                                              int64_t over_provision, const uint64_t *pool_match,
                                              const uint8_t *pod_class, const uint64_t *pod_carries,
                                              const uint64_t *pod_matches, const uint64_t *pod_requires,
                                              const uint64_t *pod_self, const uint64_t *pod_aff_matches,
                                              uint64_t present, int keys, const uint8_t *pod_key,
                                              const int32_t *pod_skew, const uint64_t *ts_matches,
                                              int64_t *new_size, int64_t *units_needed, int64_t *bins_opened,
                                              int32_t *acc_pool, int32_t *bin_of, int64_t *out_unaccounted,
                                              int64_t *flips, int64_t *n_flips)
{
    uint64_t evals = 0, selfs = 0;
    int64_t num_unaccounted = num_listed;
    const size_t cap = (size_t)(Pp > 0 ? Pp : 1);
    const size_t kk = (size_t)(keys > 0 ? keys : 1);
    double *bins = (double *)malloc(sizeof(double) * cap * D);
    uint64_t *bin_c = (uint64_t *)malloc(sizeof(uint64_t) * cap);
    uint64_t *bin_m = (uint64_t *)malloc(sizeof(uint64_t) * cap);
    uint64_t *bin_h = (uint64_t *)malloc(sizeof(uint64_t) * cap);
    int32_t *bin_n = (int32_t *)malloc(sizeof(int32_t) * cap * kk);  /* [bin][key] */
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
            const int k = pod_key[p];
            ++evals;
            if (!(match(pool_match[t], pod_class[p]) && sub_possible(u, r, D))) continue;
            int64_t hit = -1;
            for (int64_t i = 0; i < nb; ++i) {
                if ((k == NO_KEY || bin_n[(size_t)i * kk + k] <= pod_skew[p]) &&
                    affine(pod_requires[p], pod_self[p], bin_h[i], present) &&
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
                for (size_t b = 0; b < kk; ++b) bin_n[(size_t)hit * kk + b] = 0;
            }
            for (int d = 0; d < D; ++d) {
                double left = bins[(size_t)hit * D + d] - r[d];
                bins[(size_t)hit * D + d] = left;
            }
            bin_c[hit] |= pod_carries[p];
            bin_m[hit] |= pod_matches[p];
            bin_h[hit] |= pod_aff_matches[p];
            for (int b = 0; b < keys; ++b)
                if ((ts_matches[p] >> b) & 1u) ++bin_n[(size_t)hit * kk + b];
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
    free(bin_n);
    free(cur_bin);
    *out_unaccounted = num_unaccounted;
    return evals;
}
