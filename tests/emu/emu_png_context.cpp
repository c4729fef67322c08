// Host build of context_assign_kernel (online decoding, csrc/unfilter.cuh) under the SIMT emulator (tests/emu/simt.h):
// test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/unfilter.cuh"

using namespace pngb200;

// Rows [r0, r1) of pass z of `filtered` (whose rows already hold their pixels) assigned, and with `overdraw` painted, into
// `pixels`, in one launch planned by plan_assign as the library plans it, with at most `max_ctas` CTAs.  y[0], y[1]: the
// storage rows the launch writes.  Returns the number of CTAs.
extern "C" int emu_context_assign(int z, uint64_t r0, uint64_t r1, const uint8_t* filtered, uint8_t* pixels, uint32_t w,
                                  uint32_t h, uint32_t volume, uint32_t depth, int interlaced, int overdraw, unsigned max_ctas,
                                  int order, uint64_t* y)
{
    AssignJob j;
    const uint32_t ctas = plan_assign(z, r0, r1, filtered, pixels, w, h, volume, depth, interlaced != 0, overdraw != 0,
                                      max_ctas, &j, y, y + 1);
    simt::launch(ctas, ASSIGN_THREADS, 0, [&]() { context_assign_kernel(j); }, order);
    return (int)ctas;
}
