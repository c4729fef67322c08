// Host build of context_assign_batch_kernel (online decoding, csrc/unfilter.cuh) under the SIMT emulator
// (tests/emu/simt.h): test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/unfilter.cuh"

using namespace pngb200;

// One launch over n ranges, range k being rows [r0[k], r1[k]) of pass z[k] of the image whose filtered stream (rows
// already holding their pixels) is filtered[k] and whose storage is pixels[k], planned by plan_assign_batch as the library
// plans it, with a budget of `max_ctas` CTAs.  y[2k], y[2k + 1]: the storage rows range k writes.  Returns the number of
// CTAs.
extern "C" int emu_context_assign_batch(int n, const int* z, const uint64_t* r0, const uint64_t* r1,
                                        const uint8_t* const* filtered, uint8_t* const* pixels, const uint32_t* geometry,
                                        const int* overdraw, unsigned max_ctas, int order, uint64_t* y)
{
    std::vector<AssignRange> ranges(n);
    for (int k = 0; k < n; ++k) {
        const uint32_t* g = geometry + 5 * k;   // width, height, volume, depth, interlaced
        ranges[k] = {z[k], r0[k], r1[k], filtered[k], pixels[k], g[0], g[1], g[2], g[3], g[4] != 0, overdraw[k] != 0};
    }
    std::vector<AssignJob> jobs;
    std::vector<uint32_t>  cta_base;
    std::vector<uint64_t>  rows;
    const uint32_t ctas = plan_assign_batch(ranges, max_ctas, jobs, cta_base, rows);
    simt::launch(ctas, ASSIGN_THREADS, 0, [&]() { context_assign_batch_kernel(jobs.data(), cta_base.data(), (uint32_t)n); },
                 order);
    std::copy(rows.begin(), rows.end(), y);
    return (int)ctas;
}

// The same range alone, through context_assign_kernel with at most `max_ctas` CTAs
extern "C" int emu_context_assign_one(int z, uint64_t r0, uint64_t r1, const uint8_t* filtered, uint8_t* pixels,
                                      const uint32_t* g, int overdraw, unsigned max_ctas, int order, uint64_t* y)
{
    AssignJob j;
    const uint32_t ctas = plan_assign(z, r0, r1, filtered, pixels, g[0], g[1], g[2], g[3], g[4] != 0, overdraw != 0,
                                      max_ctas, &j, y, y + 1);
    simt::launch(ctas, ASSIGN_THREADS, 0, [&]() { context_assign_kernel(j); }, order);
    return (int)ctas;
}
