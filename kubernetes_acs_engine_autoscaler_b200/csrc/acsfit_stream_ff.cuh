// acsfit_stream_ff.cuh -- firstfit_stream_kernel: the first-fit stage pipeline WITHOUT CTA-wide barriers.
//
// Same algorithm, same stages, same results as firstfit_pipeline_kernel (acsfit_kernels.cuh): the node (bin) list
// is cut into stages of Tn nodes, a CTA owns a stage, pods flow through in tiles of 256, per (stage, tile) a
// parallel candidate scan in rank space is followed by an in-order resolve through a chain of warps (warp w owns
// nodes 32w..32w+31 of the stage, lane = node, literal float64 reference expression).  What changes is the
// schedule inside the CTA.  In the barrier form every tile is load -> scan -> resolve -> refresh -> publish with
// __syncthreads between the phases, so the warp chain DRAINS before the next tile may enter it: a frontier tile
// costs several times the work of its busiest warp.  Here every warp
// runs its own loop and tiles stream through the chain:
//
//   warp w, iteration i:   scan share of tile i      (its 32 pods against ALL nodes of the stage, packed ranks)
//                          resolve share of tile i-1 (its 32 nodes, entries arriving from warp w-1's queue)
//                          [last warp] publish tile i-1
//
// Per-tile data lives in a ring of kSlots = 4 shared-memory slots; warps synchronise through tagged flags
// (scan_ready[slot][warp], tile_tag[slot], the self-validating queue words of the barrier form) and never through
// a CTA barrier.  Why this stays exact:
//   * scanning tile i before tile i-1 is resolved uses STALE node thresholds.  Nodes only fill up (requests >= 0,
//     rounding monotone), so a stale threshold admits a superset of the pods that still fit, and a candidate found
//     under it is still a lower bound of the first fitting node; the resolver decides with the literal expression.
//   * a packed threshold row is replaced word by word with single 32-bit stores; a reader sees old (looser) or new
//     fields, never an invalid one.
//   * slot reuse: warp 0 starts resolving tile i-1 only after EVERY warp flagged its scan share of tile i-1, which a
//     warp does at the top of its iteration i-1, i.e. after it completed iteration i-2 (resolve + publish of tile
//     i-3).  So when any warp writes slot (i % 4) for tile i, tile i-4 has been published.
// Used for D <= 8 with a rank layout (RW > 0) and stages of a multiple of 32 nodes; everything else runs the
// barrier form.  Both forms pass the same parity suite (knob "stream").
#pragma once
#include "acsfit_kernels.cuh"

namespace acsfit {

constexpr int kSlots = 4;

template <int D, bool BINS, int RW>
struct StreamSmem {
    static __host__ __device__ size_t bytes(int Tn)
    {
        return sizeof(double) * ((size_t)(BINS ? 1 : 3) * D * Tn + (size_t)kSlots * kTile * D + (size_t)8 * 36 * D)
               + sizeof(unsigned) * ((size_t)RW * Tn + (size_t)kSlots * kTile * RW + (size_t)kSlots * kTile /*cand*/ +
                                     (size_t)kSlots * (kTile + 1) /*hitlist*/ + (size_t)kSlots * 7 * (kTile + 1) /*queues*/ +
                                     (size_t)kSlots * (8 + 8 + 8 + 8) /*alive, hitword, scan_ready, alive_cnt*/ +
                                     (size_t)kSlots * 4 /*hit_count, tile_tag, placed_cnt, pad*/ + 8 /*opened*/ + 8 /*misc*/ + 4)
               + 8 * 32 /*found*/ + 16;
    }
};

template <int D, bool BINS, int RW>
__global__ void __launch_bounds__(256)
firstfit_stream_kernel(const PipelineParams p)
{
    static_assert(RW > 0 && D <= 8, "streaming form: packed-rank scan, D <= 8");
    constexpr int NW = 8;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int Tn = p.Tn;
    double *state_s = reinterpret_cast<double *>(smem_raw);                     // [D][Tn] used (nodes) / remaining (bins)
    double *thr_s = BINS ? state_s : state_s + (size_t)D * Tn;                  // [D][Tn] scan thresholds (nodes)
    double *cap_s = BINS ? state_s : thr_s + (size_t)D * Tn;                    // [D][Tn] capacity (nodes)
    double *rows_s = state_s + (size_t)(BINS ? 1 : 3) * D * Tn;                 // [kSlots][kTile][D] rows of the HIT pods only
    double *brows = rows_s + (size_t)kSlots * kTile * D;                        // [NW][36][D] rows of a resolver batch
    unsigned *tw_s = reinterpret_cast<unsigned *>(brows + (size_t)NW * 36 * D); // [Tn][RW] packed node rows
    unsigned *rw_s = tw_s + (size_t)RW * Tn;                                    // [kSlots][kTile][RW] packed pod rows
    unsigned *cand_s = rw_s + (size_t)kSlots * kTile * RW;                      // [kSlots][kTile]
    unsigned *hitlist = cand_s + (size_t)kSlots * kTile;                        // [kSlots][kTile+1]
    unsigned *queue = hitlist + (size_t)kSlots * (kTile + 1);                   // [kSlots][7][kTile+1]
    unsigned *alive_w = queue + (size_t)kSlots * 7 * (kTile + 1);               // [kSlots][8]
    unsigned *hitword = alive_w + kSlots * 8;                                   // [kSlots][8]
    unsigned *scan_ready = hitword + kSlots * 8;                                // [kSlots][8] tile + 1 once the share is done
    unsigned *alive_cnt = scan_ready + kSlots * 8;                              // [kSlots][8]
    unsigned *hit_count = alive_cnt + kSlots * 8;                               // [kSlots]
    unsigned *tile_tag = hit_count + kSlots;                                    // [kSlots] tile + 1 once hitlist / hit_count are valid
    unsigned *placed_cnt = tile_tag + kSlots;                                   // [kSlots]
    unsigned *opened = placed_cnt + 2 * kSlots;                                 // [8] bins: bin already holds a pod (bit per lane)
    unsigned *misc = opened + 8;                                                // 0 stage, 1 abort, 2 tiles published by this stage
    unsigned char *found_s = reinterpret_cast<unsigned char *>(misc + 8);       // [NW][32]

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) {
        misc[0] = (unsigned)atomicAdd(p.ticket, 1);
        misc[1] = 0;
        misc[2] = 0;
    }
    for (int i = tid; i < kSlots * (8 * (kTile + 1)) + kSlots * 32 + kSlots * 4 + 8; i += 256) hitlist[i] = 0;  // hitlists .. opened
    __syncthreads();
    const int stage = (int)misc[0];
    const int64_t stage_lo = p.node_lo + (int64_t)stage * Tn;
    const int n_valid = (int)max((int64_t)0, min((int64_t)Tn, p.node_hi - stage_lo));
    const int n_warps = Tn >> 5;                          // resolver warps (every warp also scans)
    const int n_k = Tn >> 5;                              // node words per scanning lane
    const bool remote_in = stage == 0 && p.alive_in != nullptr;
    const bool sys_out = p.sys_scope && stage == (int)gridDim.x - 1;
    const int T = p.num_tiles;

    // ---- stage start: state, thresholds and packed rows of the stage's nodes ------------------------------
    for (int i = tid; i < Tn * D; i += 256) {
        const int n = i / D, d = i - n * D;
        if (BINS) {
            state_s[(size_t)d * Tn + n] = n < n_valid ? p.unit[d] : -1.0;
        } else {
            double u = 0.0, c = -1.0, t = -1.0;
            if (n < n_valid) {
                const int64_t gn = stage_lo + n;
                u = p.used[(size_t)gn * D + d];
                c = p.cap_type[(size_t)p.node_type[gn] * D + d];
                t = node_threshold(c, u);
            }
            state_s[(size_t)d * Tn + n] = u;
            cap_s[(size_t)d * Tn + n] = c;
            thr_s[(size_t)d * Tn + n] = t;
        }
    }
    for (int i = tid; i < Tn * RW; i += 256) tw_s[i] = 0;
    __syncthreads();
    for (int i = tid; i < Tn * D; i += 256) {
        const int d = i / Tn, n = i - d * Tn;
        const double thr = BINS ? state_s[i] : thr_s[i];
        atomicOr(&tw_s[n * RW + p.rk.word[d]], rank_upper(p.rk.sorted + (size_t)d * kRankCap, p.rk.count[d], thr) << p.rk.shift[d]);
    }
    __syncthreads();  // the last CTA-wide barrier

    volatile unsigned *vmisc = misc;
    const unsigned long long t_start = global_timer_ns();
    auto aborted = [&]() { return vmisc[1] != 0; };
    auto give_up = [&](int code) {
        atomicExch(p.status, code);
        vmisc[1] = 1;
    };
    unsigned g[RW];
#pragma unroll
    for (int w = 0; w < RW; ++w) g[w] = p.rk.guard[w];

    // ---- persistent resolver state of this lane's node ------------------------------------------------------
    const int my_lo = warp << 5;
    const int n = my_lo + lane;
    const bool resolver = warp < n_warps;
    const bool last = warp == n_warps - 1;
    double S[D], C[D];
#pragma unroll
    for (int d = 0; d < D; ++d) {
        S[d] = resolver ? state_s[(size_t)d * Tn + n] : (BINS ? -1.0 : 0.0);
        C[d] = (!BINS && resolver) ? cap_s[(size_t)d * Tn + n] : -1.0;
    }
    unsigned touched_or_open = 0u;  // bins: this warp's bins that already hold a pod
    unsigned long long my_evals = 0;
    long long forwarded = 0;        // (last warp) pods this stage passed on
    bool state_dirty = false;       // this lane's node changed since the stage started

    // ---- scanner state: upstream progress, the ring of alive words, the prefetched row index of this lane's pod
    int known = 0, ring_base = 0, ring_hi = 0;
    unsigned ring_word = 0u;  // lane l < 8: alive word of this warp's pods in tile ring_base + l
    bool drained_seen = false;
    int64_t pre_row = -1;
    unsigned prew[RW];
    auto prefetch_pod = [&](int tile) {
        pre_row = -1;
        const int64_t j = (int64_t)(p.tile_lo + tile) * kTile + tid;
        if (tile < T && j < p.M) {
            int64_t row = p.pod_idx ? (int64_t)__ldg(p.pod_idx + j) : j;
            if (p.row_map) row = (int64_t)__ldg(p.row_map + row);
            pre_row = row;
#pragma unroll
            for (int w = 0; w < RW; ++w) prew[w] = __ldg(p.rk.packed + (size_t)row * RW + w);
        }
    };
    prefetch_pod(0);

    auto publish = [&](int tiles_done) {
        if (sys_out) {
            __threadfence_system();
            st_release_sys(p.progress + stage, tiles_done);
        } else {
            st_release(p.progress + stage, tiles_done);
        }
    };

    for (int it = 0; it <= T; ++it) {
        // =================== scan share of tile `it` ===================================================
        if (it < T) {
            const int slot = it % kSlots;
            // slot reuse guard (resolver warps satisfy it by construction; scan-only warps of narrow stages wait here)
            for (unsigned spins = 0; (int)vmisc[2] < it - kSlots + 1 && !aborted();)
                if ((++spins & 1023u) == 0 && global_timer_ns() - t_start > p.watchdog_ns) give_up(1);
            if (known <= it && !drained_seen) {
                int seen = known;
                if (lane == 0) {
                    if (!(stage > 0 || p.upstream)) {
                        seen = T;
                    } else {
                        const int *flag = stage > 0 ? p.progress + (stage - 1) : p.upstream;
                        unsigned spins = 0;
                        for (;;) {
                            if (stage > 0 && *(volatile int *)p.drained) {
                                seen = -1;  // an earlier stage finished with nothing left alive
                                break;
                            }
                            seen = (p.sys_scope && stage == 0) ? ld_acquire_sys(flag) : ld_acquire(flag);
                            if (seen > it || aborted()) break;
                            if ((++spins & 63u) == 0 &&
                                (*(volatile int *)p.status != 0 || global_timer_ns() - t_start > p.watchdog_ns)) {
                                give_up(1);
                                break;
                            }
                            __nanosleep(20);
                        }
                    }
                }
                seen = __shfl_sync(0xFFFFFFFFu, seen, 0);
                if (seen < 0) {
                    drained_seen = true;
                    known = T;
                } else {
                    known = seen;
                }
            }
            if (aborted()) break;
            unsigned word = 0u;
            if (!drained_seen) {
                if (it >= ring_hi) {  // refill: this warp's alive word of every tile known to be published (<= 8 ahead)
                    const int hi_t = min(known, it + 8);
                    ring_word = 0u;
                    if (lane < hi_t - it) {
                        const int64_t wj = (int64_t)(p.tile_lo + it + lane) * (kTile / 32) + warp;
                        if (wj * 32 < p.M) ring_word = remote_in ? ld_relaxed_sys_u32(p.alive_in + wj) : __ldcg(p.alive + wj);
                    }
                    ring_base = it;
                    ring_hi = hi_t;
                }
                word = __shfl_sync(0xFFFFFFFFu, ring_word, it - ring_base);
            }
            const bool is_alive = (word >> lane) & 1u;
            const int q = my_lo + lane;  // pod position inside the tile
            if (is_alive) {
#pragma unroll
                for (int w = 0; w < RW; ++w) rw_s[((size_t)slot * kTile + q) * RW + w] = prew[w];
            }
            __syncwarp();
            unsigned hitbits = 0u;
            bool all_hit = false;
            if (BINS) {
                int n_open = 0;
#pragma unroll
                for (int w = 0; w < NW; ++w) n_open += __popc(((volatile unsigned *)opened)[w]);
                all_hit = n_open < n_valid;  // an untouched bin takes any eligible pod (scaler.py:134 is the same test)
            }
            if (all_hit) {
                hitbits = word;
                if (is_alive) cand_s[slot * kTile + q] = 0u;
            } else if (word) {
                unsigned tg[8][RW];
#pragma unroll
                for (int k = 0; k < 8; ++k)
#pragma unroll
                    for (int w = 0; w < RW; ++w) tg[k][w] = (k < n_k ? ((volatile unsigned *)tw_s)[(lane + 32 * k) * RW + w] : 0u) | g[w];
                for (unsigned bits = word; bits; bits &= bits - 1) {
                    const int b = __ffs(bits) - 1;
                    unsigned r[RW];
#pragma unroll
                    for (int w = 0; w < RW; ++w) r[w] = rw_s[((size_t)slot * kTile + my_lo + b) * RW + w];
                    unsigned fitk = 0u;  // bit k: node lane + 32k fits (in rank space, under possibly stale thresholds)
#pragma unroll
                    for (int k = 0; k < 8; ++k) {
                        unsigned miss = 0u;
#pragma unroll
                        for (int w = 0; w < RW; ++w) miss |= ((tg[k][w] - r[w]) & g[w]) ^ g[w];
                        fitk |= (miss == 0u ? 1u : 0u) << k;
                    }
                    if (__any_sync(0xFFFFFFFFu, fitk != 0u)) {
                        unsigned c = kNoCand;
#pragma unroll
                        for (int k = 0; k < 8; ++k) {
                            const unsigned bk = __ballot_sync(0xFFFFFFFFu, (fitk >> k) & 1u);
                            if (c == kNoCand && bk) c = 32u * k + (unsigned)__ffs(bk) - 1u;
                        }
                        hitbits |= 1u << b;
                        if (lane == 0) cand_s[slot * kTile + my_lo + b] = c;
                    }
                }
            }
            if ((hitbits >> lane) & 1u) {  // the float64 rows of the hit pods, for the resolvers
                const double *src = p.req + (size_t)pre_row * D;
                double *dst = rows_s + ((size_t)slot * kTile + q) * D;
#pragma unroll
                for (int d = 0; d < D; d += 2) *reinterpret_cast<double2 *>(dst + d) = __ldg(reinterpret_cast<const double2 *>(src + d));
            }
            prefetch_pod(it + 1);
            __syncwarp();
            if (lane == 0) {
                alive_w[slot * 8 + warp] = word;
                alive_cnt[slot * 8 + warp] = (unsigned)__popc(word);
                hitword[slot * 8 + warp] = hitbits;
                __threadfence_block();
                ((volatile unsigned *)scan_ready)[slot * 8 + warp] = (unsigned)it + 1u;
            }
        }
        // =================== resolve share of tile `it - 1` ============================================
        if (it >= 1 && resolver) {
            const int tj = it - 1;
            const int slot = tj % kSlots;
            unsigned H = 0;
            if (warp == 0) {
                for (unsigned spins = 0;; ++spins) {
                    const unsigned tag = lane < NW ? ((volatile unsigned *)scan_ready)[slot * 8 + lane] : (unsigned)tj + 1u;
                    if (__all_sync(0xFFFFFFFFu, tag == (unsigned)tj + 1u) || aborted()) break;
                    if ((spins & 1023u) == 1023u && global_timer_ns() - t_start > p.watchdog_ns) give_up(1);
                }
                __threadfence_block();
                unsigned base = 0;
                unsigned *hl = hitlist + (size_t)slot * (kTile + 1);
#pragma unroll
                for (int v = 0; v < NW; ++v) {
                    const unsigned hw = hitword[slot * 8 + v];
                    if ((hw >> lane) & 1u) hl[base + __popc(hw & ((1u << lane) - 1u))] = 32u * v + lane + 1u;
                    base += __popc(hw);
                }
                H = base;
                __syncwarp();
                if (lane == 0) {
                    hl[H] = kQueueEnd;
                    hit_count[slot] = H;
                    __threadfence_block();
                    ((volatile unsigned *)tile_tag)[slot] = (unsigned)tj + 1u;
                }
                __syncwarp();
            } else {
                for (unsigned spins = 0; ((volatile unsigned *)tile_tag)[slot] != (unsigned)tj + 1u && !aborted(); ++spins)
                    if ((spins & 1023u) == 1023u && global_timer_ns() - t_start > p.watchdog_ns) give_up(1);
                __threadfence_block();
                H = ((volatile unsigned *)hit_count)[slot];
            }
            if (aborted()) break;
            unsigned touched_tile = 0u;
            if (H > 0) {
                double Mx[D];
#pragma unroll
                for (int d = 0; d < D; ++d) Mx[d] = warp_upper_bound(BINS ? S[d] : thr_s[(size_t)d * Tn + n]);
                const volatile unsigned *in_q = warp == 0 ? hitlist + (size_t)slot * (kTile + 1)
                                                          : queue + ((size_t)slot * 7 + (warp - 1)) * (kTile + 1);
                volatile unsigned *out_q = queue + ((size_t)slot * 7 + (last ? 0 : warp)) * (kTile + 1);  // (unused when last)
                const double *rows = rows_s + (size_t)slot * kTile * D;
                const unsigned *cand = cand_s + slot * kTile;
                unsigned ev_local = 0, head = 0, out = 0;
                int n_placed = 0;
                bool done = false;
                while (!done) {
                    const unsigned idx = head + lane <= (unsigned)kTile ? head + lane : (unsigned)kTile;
                    unsigned e, present;
                    int nb;
                    for (unsigned spins = 0;; ++spins) {
                        e = in_q[idx];
                        if (head + lane > (unsigned)kTile) e = 0;
                        present = __ballot_sync(0xFFFFFFFFu, e != 0);
                        nb = __ffs(~present) ? __ffs(~present) - 1 : 32;  // written entries form a prefix
                        const bool has_end = __any_sync(0xFFFFFFFFu, lane < nb && e == kQueueEnd);
                        if (has_end || nb >= kMinBatch) break;
                        __nanosleep(64);
                        if (aborted() || ((spins & 4095u) == 4095u && global_timer_ns() - t_start > p.watchdog_ns)) {
                            give_up(2);
                            e = lane == 0 ? kQueueEnd : 0u;
                            nb = 1;
                            break;
                        }
                    }
                    const unsigned endmask = __ballot_sync(0xFFFFFFFFu, lane < nb && e == kQueueEnd);
                    const int n_ent = endmask ? __ffs(endmask) - 1 : nb;
                    // consumed words (the end marker included) go back to "not written" for the slot's next tile
                    if (lane < n_ent + (endmask ? 1 : 0) && head + lane <= (unsigned)kTile)
                        const_cast<volatile unsigned *>(in_q)[head + lane] = 0u;
                    const bool mine = lane < n_ent;
                    const unsigned q_l = mine ? e - 1 : 0;
                    const unsigned c_l = mine ? cand[q_l] : kNoCand;
                    const unsigned testmask = __ballot_sync(0xFFFFFFFFu, mine && (int)c_l < my_lo + 32);
                    int placed_here = -1;
                    double *brow = brows + (size_t)warp * 36 * D;
                    volatile unsigned char *fnd = found_s + warp * 32;
                    double own[D];
                    load_row<D>(own, rows + (size_t)q_l * D);
                    bool poss = (testmask >> lane) & 1u;
#pragma unroll
                    for (int d = 0; d < D; ++d) poss = poss & (own[d] <= Mx[d]);
                    const unsigned possmask = __ballot_sync(0xFFFFFFFFu, poss);
                    const int n_poss = __popc(possmask);
                    const int my_rank = __popc(possmask & ((1u << lane) - 1u));
                    if (poss) {
#pragma unroll
                        for (int d = 0; d < D; d += 2)
                            *reinterpret_cast<double2 *>(brow + (size_t)my_rank * D + d) = make_double2(own[d], own[d + 1]);
                    }
                    if (lane < 4) {
                        double *pad = brow + (size_t)(n_poss + lane) * D;
                        pad[0] = __longlong_as_double(0x7FF0000000000000ll);
#pragma unroll
                        for (int d = 1; d < D; ++d) pad[d] = 0.0;
                    }
                    __syncwarp();
                    double r[D];
                    load_row<D>(r, brow);
                    unsigned took = 0;    // bit k: dense entry k of the batch was placed by this warp
                    unsigned mymask = 0;  // bit k: ... by THIS lane's node
                    const unsigned me = 1u << lane, le = (me << 1) - 1u;  // this lane's bit, and all bits up to it
                    // The placement chain.  Entry k's test needs the state left by entry k-1, which is only known once
                    // the vote of entry k-1 has named its taker.  Instead of waiting for it, both outcomes are computed
                    // while that vote is in flight: fit_keep = "entry k fits this node as it is", fit_took = "... after
                    // this node took entry k-1" (the same float64 expressions, same rounding), and the vote's answer
                    // merely selects one.  What stays on the vote-to-vote path is a predicate select and a mask
                    // compare; the float64 adds and compares run beside it.
                    auto fits = [&](const double (&st)[D], const double (&row)[D]) {
                        bool ok = true, ok2 = true;  // two independent and-chains over the dimensions
#pragma unroll
                        for (int d = 0; d < D / 2; ++d) {
                            if (BINS) ok = ok & (row[d] <= st[d]);   // == (st - row >= 0) for finite values (scaler.py:139)
                            else ok = ok & (__dsub_rn(C[d], __dadd_rn(st[d], row[d])) >= 0.0);  // kube.py:175
                        }
#pragma unroll
                        for (int d = D / 2; d < D; ++d) {
                            if (BINS) ok2 = ok2 & (row[d] <= st[d]);
                            else ok2 = ok2 & (__dsub_rn(C[d], __dadd_rn(st[d], row[d])) >= 0.0);
                        }
                        return ok & ok2;
                    };
                    // It pays for the bins at D = 8.  Not used where it loses: the D = 8 node test is 24 float64
                    // instructions per entry and issue-bound; at D <= 4 the extra registers cost the second stage CTA
                    // per SM, and with it the nodes -> bins chaining of the c2 tick.
                    constexpr bool kSpeculate = BINS && D >= 8;
                    if constexpr (!kSpeculate) {
                        for (int k0 = 0; k0 < n_poss; k0 += 4)
#pragma unroll
                        for (int k = k0; k < k0 + 4; ++k) {  // slots past n_poss hold never-fitting rows
                            double r_next[D];
                            load_row<D>(r_next, brow + (size_t)(k + 1) * D);
                            const bool ok = fits(S, r);
                            // two votes issued back to back: the predicate one steers the (uniform) branch without an
                            // integer compare on the chain, the ballot names the first fitting node
                            const bool any = __any_sync(0xFFFFFFFFu, ok);
                            const unsigned m = __ballot_sync(0xFFFFFFFFu, ok);
                            if (any) {
                                if ((m & le) == me) {  // the first fitting node of the warp takes the pod
#pragma unroll
                                    for (int d = 0; d < D; ++d)
                                        S[d] = BINS ? __dsub_rn(S[d], r[d]) : __dadd_rn(S[d], r[d]);  // scaler.py:140 / kube.py:171
                                    mymask |= 1u << k;
                                }
                                took |= 1u << k;
                            }
#pragma unroll
                            for (int d = 0; d < D; ++d) r[d] = r_next[d];
                        }
                    } else {
                    double Sm[D];  // the state this node would have after taking the previous entry
#pragma unroll
                    for (int d = 0; d < D; ++d) Sm[d] = S[d];
                    bool prev_mine = false;
                    bool fit_keep = fits(S, r), fit_took = fit_keep;
                    for (int k0 = 0; k0 < n_poss; k0 += 4)
#pragma unroll
                    for (int k = k0; k < k0 + 4; ++k) {  // slots past n_poss hold never-fitting rows
                        double r_next[D];
                        load_row<D>(r_next, brow + (size_t)(k + 1) * D);
                        const bool ok = prev_mine ? fit_took : fit_keep;
                        if (prev_mine) {
#pragma unroll
                            for (int d = 0; d < D; ++d) S[d] = Sm[d];
                        }
                        const unsigned m = __ballot_sync(0xFFFFFFFFu, ok);
                        // beside the vote: the state after taking THIS entry, and the next entry's test either way
#pragma unroll
                        for (int d = 0; d < D; ++d)
                            Sm[d] = BINS ? __dsub_rn(S[d], r[d])   // bins[i] - pod.resources   scaler.py:140
                                         : __dadd_rn(S[d], r[d]);  // used += pod.resources     kube.py:171
                        fit_keep = fits(S, r_next);
                        fit_took = fits(Sm, r_next);
                        prev_mine = (m & le) == me;  // the first fitting node of the warp takes the pod
                        if (prev_mine) mymask |= 1u << k;
                        if (m) took |= 1u << k;
#pragma unroll
                        for (int d = 0; d < D; ++d) r[d] = r_next[d];
                    }
                    if (prev_mine) {  // the last entry's taker
#pragma unroll
                        for (int d = 0; d < D; ++d) S[d] = Sm[d];
                    }
                    }  // kSpeculate
                    for (unsigned t = mymask; t; t &= t - 1) fnd[__ffs(t) - 1] = (unsigned char)lane;
                    if (mymask) state_dirty = true;
                    __syncwarp();
                    if (took) {
                        n_placed += __popc(took);
                        const bool got = poss && ((took >> my_rank) & 1u);
                        const int found = got ? (int)fnd[my_rank] : -1;
                        placed_here = found;
                        const unsigned acc_lanes = __reduce_or_sync(0xFFFFFFFFu, got ? (1u << found) : 0u);
                        ev_local += __reduce_add_sync(0xFFFFFFFFu, got ? (unsigned)found + 1u : 0u) -
                                    (unsigned)__popc(acc_lanes & ~touched_or_open);
                        touched_or_open |= acc_lanes;
                        touched_tile |= acc_lanes;
                        if (BINS) {
#pragma unroll
                            for (int d = 0; d < D; ++d) Mx[d] = warp_upper_bound(S[d]);
                        }
                    }
                    if (!last) {
                        const unsigned fwd = __ballot_sync(0xFFFFFFFFu, mine && placed_here < 0);
                        if (mine && placed_here < 0) out_q[out + __popc(fwd & ((1u << lane) - 1u))] = e;
                        out += __popc(fwd);
                    }
                    if (placed_here >= 0) {
                        p.placed[(int64_t)(p.tile_lo + tj) * kTile + q_l] = (int32_t)(stage_lo + my_lo + placed_here);
                        atomicAnd(&alive_w[slot * 8 + (q_l >> 5)], ~(1u << (q_l & 31)));
                    }
                    head += (unsigned)n_ent;
                    done = endmask != 0;
                }
                if (n_placed) {
                    if (BINS) my_evals += (unsigned long long)ev_local + (unsigned long long)n_placed * (unsigned long long)(stage_lo + my_lo);
                    if (lane == 0) {
                        atomicAdd(&placed_cnt[slot], (unsigned)n_placed);
                        if (BINS) ((volatile unsigned *)opened)[warp] = touched_or_open;
                    }
                }
                __syncwarp();
                if (!last && lane == 0) {
                    __threadfence_block();  // placements of this warp (alive bits, placed_cnt) before the end marker
                    out_q[out] = kQueueEnd;
                }
                // ---- thresholds and packed rows of the nodes that took a pod (this warp's nodes only) -------
                if (touched_tile) {
                    if ((touched_tile >> lane) & 1u) {
#pragma unroll
                        for (int d = 0; d < D; ++d) state_s[(size_t)d * Tn + n] = S[d];
                    }
                    __syncwarp();
                    constexpr int NPR = 32 / D;  // nodes per round: lane = (node j of the round, dimension d)
                    const int nd = __popc(touched_tile);
                    for (int base = 0; base < nd; base += NPR) {
                        const int j = base + lane / D, d = lane % D;
                        unsigned val[RW];
#pragma unroll
                        for (int w = 0; w < RW; ++w) val[w] = 0u;
                        int nn = 0;
                        if (j < nd) {
                            nn = my_lo + (int)__fns(touched_tile, 0, j + 1);
                            const size_t i = (size_t)d * Tn + nn;
                            double thr;
                            if (BINS) {
                                thr = state_s[i];
                            } else {
                                thr = node_threshold(cap_s[i], state_s[i]);
                                thr_s[i] = thr;
                            }
                            const unsigned t = rank_upper(p.rk.sorted + (size_t)d * kRankCap, p.rk.count[d], thr);
#pragma unroll
                            for (int w = 0; w < RW; ++w) val[w] = p.rk.word[d] == w ? t << p.rk.shift[d] : 0u;
                        }
#pragma unroll
                        for (int o = 1; o < D; o <<= 1) {
#pragma unroll
                            for (int w = 0; w < RW; ++w) val[w] |= __shfl_xor_sync(0xFFFFFFFFu, val[w], o);
                        }
                        if (j < nd && d == 0) {
#pragma unroll
                            for (int w = 0; w < RW; ++w) ((volatile unsigned *)tw_s)[nn * RW + w] = val[w];  // one 32-bit store per word
                        }
                    }
                    __syncwarp();
                }
            }
            // ---- the last resolver warp retires the tile ---------------------------------------------------
            if (last) {
                __threadfence_block();
                const unsigned n_pl = ((volatile unsigned *)placed_cnt)[slot];
                unsigned alive_total = 0;
#pragma unroll
                for (int v = 0; v < NW; ++v) alive_total += alive_cnt[slot * 8 + v];
                forwarded += (long long)alive_total - (long long)n_pl;
                if (lane < kTile / 32 && (n_pl || remote_in)) {
                    const int64_t wj = (int64_t)(p.tile_lo + tj) * (kTile / 32) + lane;
                    if (wj * 32 < p.M) __stcg(p.alive + wj, ((volatile unsigned *)alive_w)[slot * 8 + lane]);
                }
                __syncwarp();
                if (lane == 0) {
                    placed_cnt[slot] = 0;
                    if (n_pl || remote_in) __threadfence();
                    publish(tj + 1);
                    __threadfence_block();
                    vmisc[2] = (unsigned)tj + 1u;
                }
            }
        }
        if (aborted()) break;
    }
    if (aborted()) return;
    // ---- stage end: write the mutated node state back -------------------------------------------------------
    if (!BINS && resolver && state_dirty && n < n_valid) {
#pragma unroll
        for (int d = 0; d < D; ++d) p.used[(size_t)(stage_lo + n) * D + d] = S[d];
    }
    if (BINS && resolver && lane == 0 && my_evals) atomicAdd(p.evals, my_evals);
    if (last && lane == 0 && forwarded == 0) atomicExch(p.drained, 1);
}

}  // namespace acsfit
