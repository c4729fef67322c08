// Host build of the pass path (unfilter_pass_kernel, then unfilter_interleave_kernel) under the SIMT emulator
// (tests/emu/simt.h): test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/unfilter.cuh"

using namespace pngb200;

static const int ADAM7[7][4] = {{0, 0, 3, 3}, {4, 0, 3, 3}, {0, 4, 2, 3}, {2, 0, 2, 2}, {0, 2, 1, 2}, {1, 0, 1, 1}, {0, 1, 0, 1}};

// One decode of n images, planned as run_unfilter plans the pass path: a PassJob per non-empty Adam7 pass (one for a
// non-interlaced image), jobs sorted by band count and their bands handed out level by level in one launch of `grid`
// CTAs that are all resident, then the interleave kernel over `igrid` CTAs.  `filtered[i]` is reconstructed in place.
// status[i] < 0 stands for an inflate error (the kernels see a StreamResult with that status).
extern "C" int emu_unfilter_passes(int n, uint8_t* const* filtered, const uint64_t* filtered_len, uint8_t* const* pixels,
                                   const uint32_t* w, const uint32_t* h, const uint32_t* volume, const uint32_t* depth,
                                   const uint32_t* interlaced, const int32_t* status, unsigned grid, unsigned igrid, int order)
{
    std::vector<StreamResult> results(n);
    std::vector<PassJob>      jobs;
    std::vector<InterleaveJob> inter(n);
    uint64_t blocks = 0;
    for (int i = 0; i < n; ++i) {
        results[i] = StreamResult{};
        results[i].status = status[i];
        results[i].produced = filtered_len[i];
        const uint32_t bpp = (volume[i] + 7) >> 3;
        uint64_t off = 0;
        for (int z = 0; z < (interlaced[i] ? 7 : 1); ++z) {
            uint64_t sw = w[i], sh = h[i];
            if (interlaced[i]) {
                sw = ((uint64_t)w[i] + (1u << ADAM7[z][2]) - ADAM7[z][0] - 1) >> ADAM7[z][2];
                sh = ((uint64_t)h[i] + (1u << ADAM7[z][3]) - ADAM7[z][1] - 1) >> ADAM7[z][3];
                if (sw == 0 || sh == 0) continue;
            }
            PassJob j{};
            j.pitch = (uint32_t)((sw * volume[i] + 7) >> 3);
            j.filtered = filtered[i] + off;
            j.inflated = &results[i];
            j.filtered_len = 0;
            j.offset = off;
            j.height = (uint32_t)sh;
            j.bpp = bpp;
            jobs.push_back(j);
            off += sh * ((uint64_t)j.pitch + 1);
        }
        InterleaveJob& t = inter[i];
        t = InterleaveJob{};
        t.filtered = filtered[i]; t.pixels = pixels[i]; t.inflated = &results[i]; t.filtered_len = 0;
        t.block_base = blocks; t.width = w[i]; t.height = h[i];
        t.volume = (uint8_t)volume[i]; t.depth = (uint8_t)depth[i]; t.interlaced = (uint8_t)interlaced[i]; t.bpp = (uint8_t)bpp;
        const uint64_t chunks = (15 + (uint64_t)w[i] * h[i] * bpp + 15) / 16;
        blocks += (chunks + INTERLEAVE_THREADS - 1) / INTERLEAVE_THREADS;
    }
    auto nb = [](const PassJob& j) { return (j.height + 31) / 32; };
    std::stable_sort(jobs.begin(), jobs.end(), [&](const PassJob& a, const PassJob& b) { return nb(a) > nb(b); });
    std::vector<uint32_t> band_base(jobs.size() + 1, 0);
    for (size_t k = 0; k < jobs.size(); ++k) band_base[k + 1] = band_base[k] + nb(jobs[k]);
    const uint32_t maxb = jobs.empty() ? 0 : nb(jobs[0]);
    std::vector<uint32_t> level_start(maxb + 1, 0);
    for (uint32_t b = 0; b < maxb; ++b) {
        uint32_t alive = 0;
        for (const PassJob& j : jobs) alive += nb(j) > b;
        level_start[b + 1] = level_start[b] + alive;
    }
    const uint32_t bands = band_base[jobs.size()];
    std::vector<uint32_t> progress(bands + 1, 0);
    WaveParams p{};
    p.jobs = jobs.data(); p.band_base = band_base.data(); p.progress = progress.data(); p.ticket = &progress[bands];
    p.njobs = (uint32_t)jobs.size(); p.total_bands = bands; p.hist = nullptr;
    p.level_start = level_start.data(); p.levels = maxb;
    if (bands) simt::launch(grid, WAVE_WARPS * 32, WAVE_SMEM, [&]() { unfilter_pass_kernel(p); }, order, true);
    // one CTA after the other: the kernel's pass table is a __shared__ array, which the emulator keeps per kernel
    simt::launch(igrid, INTERLEAVE_THREADS, 0, [&]() { unfilter_interleave_kernel(inter.data(), (uint32_t)n, blocks); }, order);
    return 0;
}
