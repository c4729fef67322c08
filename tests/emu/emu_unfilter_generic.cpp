// Host build of unfilter_generic_kernel under the SIMT emulator (tests/emu/simt.h): test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/unfilter.cuh"

using namespace pngb200;

// one image, one 128-thread CTA as run_unfilter launches it; `filtered` is reconstructed in place
extern "C" int emu_unfilter_generic(uint8_t* filtered, uint64_t filtered_len, uint8_t* pixels, uint32_t w, uint32_t h,
                                    uint32_t volume, uint32_t depth, uint32_t interlaced)
{
    GenericJob job{};
    job.filtered = filtered; job.pixels = pixels; job.inflated = nullptr; job.filtered_len = filtered_len;
    job.width = w; job.height = h; job.volume = (uint8_t)volume; job.depth = (uint8_t)depth;
    job.interlaced = (uint8_t)interlaced; job.bpp = (uint8_t)((volume + 7) >> 3);
    simt::launch(1, 128, 0, [&]() { unfilter_generic_kernel(&job, 1); });
    return 0;
}
