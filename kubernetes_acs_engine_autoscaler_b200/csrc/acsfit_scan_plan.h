// acsfit_scan_plan.h -- which kernel form and staging geometry K1 (occupancy) / K6 (node states) run with.
// Plain C++ (no CUDA): the launch code in acsfit.cu dispatches on it, and tests/cpp/test_scan_plan.cpp checks
// the whole table with g++ on a machine without a GPU.
//
//   form 2, bulk copy  (node_stream_bulk_kernel, acsfit_stream.cuh): contiguous table (run_idx == NULL),
//           D in {2,4,8,16}.  `cp.async.bulk` needs 16-byte aligned global addresses: req_run and, for K6,
//           flags_run must be 16-byte aligned (chunks start at multiples of 16 entries from those pointers).
//   form 1, index gather (node_stream_kernel, acsfit.cu): run_idx given, D in {2,4,8,16}.  Its 16-byte
//           `cp.async` row pieces need req_run 16-byte aligned (flag bytes are plain loads).
//   form 0, per thread (occupancy_kernel / node_states_kernel): any D in [1,16], any layout, scalar loads.
//           Also the fall-back for tables the two other forms cannot read: same result, only slower.
#pragma once
#include <cstdint>

namespace acsfit {

enum ScanForm { kScanPerThread = 0, kScanGather = 1, kScanBulk = 2 };

constexpr int kStreamWarps = 8;       // warps per CTA of the gather form
constexpr int kPerThreadBlock = 128;  // threads per CTA of the per-thread form

struct ScanPlan {
    int form;            // ScanForm
    int bytes_per_warp;  // staging bytes per warp (0: per-thread form)
    int warps;           // warps per CTA
    int chunk;           // table entries per staging chunk, bytes_per_warp / 2 / (8 D) (0: per-thread form)
};

// one acsfit_last_scan_launch record (ACSFIT_SCAN_FIELDS ints, in this order), written where the kernel is launched
struct ScanLaunch {
    int kernel;  // 0 none, 1 occupancy (K1), 2 node states (K6), 3 pending admission (acsfit_pending_admit),
                 // 4 pending admission with pod affinity (acsfit_pending_admit_pa),
                 // 5 pending admission with topology spread (acsfit_pending_admit_ts; form: 1 anti-affinity | 2 pod
                 // affinity)
    int form, D, bytes_per_warp, warps, chunk;
    int grid;    // CTAs launched
    int S;       // idle thresholds (0 for K1)
};

// bulk-copy geometry <bytes per warp, warps per CTA> for developer knob bulk_cfg (ACSFIT_BULK_CFG); D = 16 has
// one geometry, every other value of bulk_cfg (4 included) is the default measured on H100 (DESIGN.md section 6)
inline void bulk_geometry(int D, int bulk_cfg, int *bytes, int *warps)
{
    if (D > 8) { *bytes = 16384; *warps = 8; return; }
    switch (bulk_cfg) {
    case 0: *bytes = 8192; *warps = 8; return;
    case 1: *bytes = 16384; *warps = 12; return;
    case 2: *bytes = 16384; *warps = 8; return;
    case 3: *bytes = 32768; *warps = 6; return;
    default: *bytes = 8192; *warps = 16; return;
    }
}

// gather staging bytes per warp for developer knob stream_bytes (ACSFIT_STREAM_BYTES): the smallest of
// 2048 (D <= 4) / 4096 (D <= 8) / 8192 that is >= the knob; a chunk must hold at least 32 entries
inline int gather_bytes(int D, int stream_bytes)
{
    if (D <= 4 && stream_bytes <= 2048) return 2048;
    if (D <= 8 && stream_bytes <= 4096) return 4096;
    return 8192;
}

inline bool aligned16(const void *p) { return ((uintptr_t)p & 15u) == 0; }

// states: K6 (reads flags_run) rather than K1
inline ScanPlan plan_scan(int D, bool states, const void *run_idx, const void *req_run, const void *flags_run,
                          int bulk_cfg, int stream_bytes)
{
    ScanPlan p = {kScanPerThread, 0, kPerThreadBlock / 32, 0};
    if (!(D == 2 || D == 4 || D == 8 || D == 16) || !aligned16(req_run)) return p;
    if (!run_idx) {
        if (states && !aligned16(flags_run)) return p;
        p.form = kScanBulk;
        bulk_geometry(D, bulk_cfg, &p.bytes_per_warp, &p.warps);
    } else {
        p.form = kScanGather;
        p.bytes_per_warp = gather_bytes(D, stream_bytes);
        p.warps = kStreamWarps;
    }
    p.chunk = p.bytes_per_warp / 2 / (8 * D);
    return p;
}

}  // namespace acsfit
