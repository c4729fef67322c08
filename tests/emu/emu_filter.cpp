// Host build of filter_rows_kernel under the SIMT emulator (tests/emu/simt.h): test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/filter.cuh"

#include <vector>

using namespace pngb200;

// a batch of images, one warp per filtered row: row_base and the grid as pngb200_filter_batch
// (csrc/pngb200_api.cu) builds them; rows are independent, so the CTAs run one after the other
extern "C" void emu_filter_batch(int n, const uint8_t* const* pixels, uint8_t* const* filtered, const uint32_t* w,
                                 const uint32_t* h, const uint8_t* volume, const uint8_t* depth, const uint8_t* interlaced,
                                 int order)
{
    std::vector<FilterJob> jobs(n);
    std::vector<uint32_t>  row_base(n + 1);
    uint64_t rows = 0;
    for (int i = 0; i < n; ++i) {
        jobs[i].pixels = pixels[i];
        jobs[i].filtered = filtered[i];
        jobs[i].width = w[i];
        jobs[i].height = h[i];
        jobs[i].volume = volume[i];
        jobs[i].depth = depth[i];
        jobs[i].interlaced = interlaced[i];
        jobs[i].bpp = (uint8_t)((volume[i] + 7) >> 3);
        row_base[i] = (uint32_t)rows;
        rows += filter_rows(w[i], h[i], interlaced[i]);
    }
    row_base[n] = (uint32_t)rows;
    const unsigned grid = (unsigned)std::max<uint64_t>(1, (rows + FILTER_WARPS - 1) / FILTER_WARPS);
    simt::launch(grid, FILTER_WARPS * 32, 0,
                 [&]() { filter_rows_kernel(jobs.data(), row_base.data(), (uint32_t)n, (uint32_t)rows); }, order);
}
