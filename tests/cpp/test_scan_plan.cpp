// host-side table test of acsfit::plan_scan (csrc/acsfit_scan_plan.h): which K1 / K6 kernel form and staging
// geometry every (D, table layout, alignment, knob) combination gets.  The -m gpu tests check from the launch
// records that the library runs what this table says.
// Build: g++ -O2 -I<csrc> test_scan_plan.cpp -o test_scan_plan
#include <cstdio>
#include <initializer_list>
#include "acsfit_scan_plan.h"

using namespace acsfit;

static long failures = 0, checks = 0;

static void expect(int D, bool states, const void *idx, const void *req, const void *flags, int cfg, int sb, int form,
                   int bytes, int warps)
{
    const ScanPlan p = plan_scan(D, states, idx, req, flags, cfg, sb);
    const int chunk = form == kScanPerThread ? 0 : bytes / 2 / (8 * D);
    ++checks;
    if (p.form != form || p.bytes_per_warp != bytes || p.warps != warps || p.chunk != chunk) {
        ++failures;
        std::printf("FAIL D=%d states=%d idx=%p req=%p flags=%p cfg=%d sb=%d: got form %d %d B x %d warps chunk %d, "
                    "want form %d %d B x %d warps chunk %d\n", D, (int)states, idx, req, flags, cfg, sb, p.form,
                    p.bytes_per_warp, p.warps, p.chunk, form, bytes, warps, chunk);
    }
}

int main()
{
    alignas(16) static unsigned char buf[256];
    const void *a16 = buf + 16, *a8 = buf + 8, *idx = buf + 64;
    const unsigned char *fl = buf + 128;
    const int pipeline_dims[] = {2, 4, 8, 16};

    for (int states = 0; states < 2; ++states) {
        for (int D : pipeline_dims) {
            // bulk copy: every bulk_cfg, out-of-range values take the default (cfg 4); D = 16 has one geometry
            const int cfgs[] = {-1, 0, 1, 2, 3, 4, 5, 1000};
            for (int cfg : cfgs) {
                int bytes = 8192, warps = 16;
                if (D == 16) { bytes = 16384; warps = 8; }
                else if (cfg == 0) { bytes = 8192; warps = 8; }
                else if (cfg == 1) { bytes = 16384; warps = 12; }
                else if (cfg == 2) { bytes = 16384; warps = 8; }
                else if (cfg == 3) { bytes = 32768; warps = 6; }
                expect(D, states, nullptr, a16, fl, cfg, 8192, kScanBulk, bytes, warps);
            }
            // index gather: 2048 only for D <= 4, 4096 only for D <= 8, else clamped up; bulk_cfg plays no part
            const int sbs[] = {-5, 0, 1024, 2048, 2049, 4096, 4097, 8192, 1 << 20};
            for (int sb : sbs) {
                int bytes = 8192;
                if (D <= 4 && sb <= 2048) bytes = 2048;
                else if (D <= 8 && sb <= 4096) bytes = 4096;
                expect(D, states, idx, a16, fl, 0, sb, kScanGather, bytes, kStreamWarps);
            }
            // the clamps named in the knob's documentation
            if (D == 8) expect(D, states, idx, a16, fl, 4, 2048, kScanGather, 4096, 8);
            if (D == 16) expect(D, states, idx, a16, fl, 4, 2048, kScanGather, 8192, 8);
            // misaligned tables: the per-thread form
            expect(D, states, nullptr, a8, fl, 4, 8192, kScanPerThread, 0, 4);
            expect(D, states, idx, a8, fl, 4, 8192, kScanPerThread, 0, 4);
            expect(D, states, idx, buf + 3, fl, 4, 2048, kScanPerThread, 0, 4);
            for (int off : {1, 7, 8, 15}) {
                // flag bytes matter to the bulk copy of K6 only; the gather form loads them one by one
                if (states) expect(D, states, nullptr, a16, fl + off, 4, 8192, kScanPerThread, 0, 4);
                else expect(D, states, nullptr, a16, fl + off, 4, 8192, kScanBulk, D == 16 ? 16384 : 8192, D == 16 ? 8 : 16);
                expect(D, states, idx, a16, fl + off, 4, 8192, kScanGather, 8192, 8);
            }
            // a table that is 16-byte aligned, wherever it starts
            expect(D, states, nullptr, buf + 48, fl + 32, 4, 8192, kScanBulk, D == 16 ? 16384 : 8192, D == 16 ? 8 : 16);
        }
        // every other D: the per-thread form, whatever the layout and knobs
        for (int D = 1; D <= 16; ++D) {
            if (D == 2 || D == 4 || D == 8 || D == 16) continue;
            for (int cfg : {0, 3, 4}) {
                expect(D, states, nullptr, a16, fl, cfg, 2048, kScanPerThread, 0, 4);
                expect(D, states, idx, a16, fl, cfg, 2048, kScanPerThread, 0, 4);
                expect(D, states, idx, a8, fl + 1, cfg, 8192, kScanPerThread, 0, 4);
            }
        }
    }
    // chunk sizes stay multiples of 16 entries for every bulk geometry (16-byte aligned flag copies) and hold at
    // least one entry per lane in the gather form
    for (int D : pipeline_dims)
        for (int cfg = 0; cfg <= 4; ++cfg) {
            const ScanPlan b = plan_scan(D, true, nullptr, a16, fl, cfg, 8192);
            ++checks;
            if (b.chunk < 16 || b.chunk % 16) { ++failures; std::printf("FAIL bulk chunk D=%d cfg=%d: %d\n", D, cfg, b.chunk); }
            for (int sb : {2048, 4096, 8192}) {
                const ScanPlan g = plan_scan(D, true, idx, a16, fl, cfg, sb);
                ++checks;
                if (g.chunk < 32) { ++failures; std::printf("FAIL gather chunk D=%d sb=%d: %d\n", D, sb, g.chunk); }
            }
        }
    std::printf("checked %ld plans, failures=%ld\n", checks, failures);
    return failures ? 1 : 0;
}
