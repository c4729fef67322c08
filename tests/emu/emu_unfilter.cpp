// Host build of unfilter_wave_kernel under the SIMT emulator (tests/emu/simt.h): test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/unfilter.cuh"

using namespace pngb200;

// one image, `grid` CTAs resident at once (bands wait for each other through the progress words)
extern "C" int emu_unfilter(const uint8_t* filtered, uint64_t filtered_len, uint8_t* pixels, uint32_t w, uint32_t h,
                            uint32_t bpp, uint32_t depth, unsigned grid, int order)
{
    ImageJob job{};
    job.filtered = filtered; job.pixels = pixels; job.inflated = nullptr; job.filtered_len = filtered_len;
    job.width = w; job.height = h; job.pitch = w * bpp; job.volume = (uint8_t)(8 * bpp); job.depth = (uint8_t)depth;
    job.interlaced = 0; job.bpp = (uint8_t)bpp;
    const uint32_t bands = (h + 31) / 32;
    uint32_t band_base[2] = {0, bands};
    std::vector<uint32_t> progress(bands + 1, 0);
    uint32_t ticket = 0;
    WaveParams p{};
    p.jobs = &job; p.band_base = band_base; p.progress = progress.data(); p.ticket = &ticket;
    p.njobs = 1; p.total_bands = bands; p.hist = nullptr;
    simt::launch(grid, WAVE_WARPS * 32, WAVE_SMEM, [&]() { unfilter_wave_kernel(p); }, order, true);
    return 0;
}
// several images, planned by plan_bands as run_unfilter plans them: tickets level by level, or job by job past 4096 bands
extern "C" int emu_unfilter_multi(int n, const uint8_t* const* filtered, const uint64_t* filtered_len, uint8_t* const* pixels,
                                  const uint32_t* w, const uint32_t* h, uint32_t bpp, uint32_t depth, unsigned grid, int order)
{
    std::vector<ImageJob> jobs(n);
    for (int i = 0; i < n; ++i) {
        ImageJob& job = jobs[i];
        job = ImageJob{};
        job.filtered = filtered[i]; job.pixels = pixels[i]; job.inflated = nullptr; job.filtered_len = filtered_len[i];
        job.width = w[i]; job.height = h[i]; job.pitch = w[i] * bpp; job.volume = (uint8_t)(8 * bpp); job.depth = (uint8_t)depth;
        job.interlaced = 0; job.bpp = (uint8_t)bpp;
    }
    std::vector<uint32_t> band_base, level_start;
    const uint32_t bands = (uint32_t)plan_bands(jobs, band_base, level_start);
    std::vector<uint32_t> progress(bands + 1, 0);
    WaveParams p{};
    p.jobs = jobs.data(); p.band_base = band_base.data(); p.progress = progress.data(); p.ticket = &progress[bands];
    p.njobs = (uint32_t)n; p.total_bands = bands; p.hist = nullptr;
    p.level_start = level_start.data(); p.levels = level_start.empty() ? 0u : (uint32_t)level_start.size() - 1;
    simt::launch(grid, WAVE_WARPS * 32, WAVE_SMEM, [&]() { unfilter_wave_kernel(p); }, order, true);
    return 0;
}
