// Host build of the pass path (unfilter_pass_kernel, then unfilter_interleave_kernel) under the SIMT emulator
// (tests/emu/simt.h): test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/unfilter.cuh"

using namespace pngb200;

// One decode of n images, planned by plan_passes and plan_bands as run_unfilter plans the pass path, in one launch of
// `grid` CTAs that are all resident, then the interleave kernel over `igrid` CTAs.  `filtered[i]` is reconstructed in
// place.  status[i] < 0 stands for an inflate error (the kernels see a StreamResult with that status).
extern "C" int emu_unfilter_passes(int n, uint8_t* const* filtered, const uint64_t* filtered_len, uint8_t* const* pixels,
                                   const uint32_t* w, const uint32_t* h, const uint32_t* volume, const uint32_t* depth,
                                   const uint32_t* interlaced, const int32_t* status, unsigned grid, unsigned igrid, int order)
{
    std::vector<StreamResult> results(n);
    std::vector<PassJob>      jobs;
    std::vector<InterleaveJob> inter;
    uint64_t blocks = 0;
    for (int i = 0; i < n; ++i) {
        results[i] = StreamResult{};
        results[i].status = status[i];
        results[i].produced = filtered_len[i];
        InterleaveJob t{};
        t.filtered = filtered[i]; t.pixels = pixels[i]; t.inflated = &results[i]; t.filtered_len = 0;
        t.width = w[i]; t.height = h[i]; t.volume = (uint8_t)volume[i]; t.depth = (uint8_t)depth[i];
        t.interlaced = (uint8_t)interlaced[i]; t.bpp = (uint8_t)((volume[i] + 7) >> 3);
        plan_passes(t, jobs, inter, blocks);
    }
    std::vector<uint32_t> band_base, level_start;
    const uint32_t bands = (uint32_t)plan_bands(jobs, band_base, level_start);
    std::vector<uint32_t> progress(bands + 1, 0);
    WaveParams p{};
    p.jobs = jobs.data(); p.band_base = band_base.data(); p.progress = progress.data(); p.ticket = &progress[bands];
    p.njobs = (uint32_t)jobs.size(); p.total_bands = bands; p.hist = nullptr;
    p.level_start = level_start.data(); p.levels = level_start.empty() ? 0u : (uint32_t)level_start.size() - 1;
    if (bands) simt::launch(grid, WAVE_WARPS * 32, WAVE_SMEM, [&]() { unfilter_pass_kernel(p); }, order, true);
    // one CTA after the other: the kernel's pass table is a __shared__ array, which the emulator keeps per kernel
    simt::launch(igrid, INTERLEAVE_THREADS, 0, [&]() { unfilter_interleave_kernel(inter.data(), (uint32_t)n, blocks); }, order);
    return 0;
}
