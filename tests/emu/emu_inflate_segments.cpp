// Host build of the segmented-stream pipeline (block_search_kernel, inflate_cells_kernel in symbolic mode,
// window_propagate_kernel, marker_resolve_kernel) under the SIMT emulator: test infrastructure.  The driver
// below restates run_segments() of pngb200_api.cu without the CUDA runtime.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/inflate_wave.cuh"
#include "../../swift-png_b200/csrc/block_search.cuh"
#include "../../swift-png_b200/csrc/inflate_segments.cuh"
#include "../../swift-png_b200/csrc/inflate_cells.cuh"

using namespace pngb200;

// returns 0 and fills dst when every segment lined up; 1 = the pipeline asked for the whole-stream fallback;
// `plant`: if nonzero, a forged split point (bit offset) is added to check that step 3 rejects it
extern "C" int emu_inflate_segmented(const uint8_t* src, uint64_t len, uint8_t* dst, uint64_t cap, int format, uint32_t nseg,
                                     uint64_t plant, uint64_t* produced, uint32_t* segments_used)
{
    const uint64_t bits = 8 * len, step = bits / nseg;
    std::vector<SearchJob> sj;
    for (uint32_t k = 1; k < nseg; ++k) sj.push_back(SearchJob{src, len, k * step, k + 1 < nseg ? (k + 1) * step : bits, ~0ull});
    if (!sj.empty()) simt::launch((unsigned)sj.size(), 256, 0, [&]() { block_search_kernel(sj.data(), (uint32_t)sj.size()); }, 0, false, 256 << 10, BS_CTAS);
    std::vector<uint64_t> at{0};
    for (auto& q : sj)
        if (q.found != ~0ull) at.push_back(q.found);
    if (plant) { at.push_back(plant); std::sort(at.begin(), at.end()); }
    const size_t n = at.size();
    std::vector<StreamJob> sg(n);
    std::vector<std::vector<uint16_t>> sym(n);
    for (size_t k = 0; k < n; ++k) {
        const uint64_t end = k + 1 < n ? at[k + 1] : bits;
        StreamJob s{};
        s.src = src; s.src_len = len; s.format = format;
        s.start_bit = at[k]; s.start_out = 0; s.phase = k == 0 ? 0 : 1;
        s.stop_bit = k + 1 < n ? at[k + 1] : 0;
        s.symbolic = 1;
        s.dst_cap = (uint64_t)((double)cap * 1.5 * (double)(end - at[k]) / (double)bits) + (64u << 10);
        sym[k].assign(s.dst_cap + 64, 0xDEAD);
        s.dst = (uint8_t*)sym[k].data();
        sg[k] = s;
    }
    std::vector<StreamResult> sr(n);
    memset(sr.data(), 0, sizeof(StreamResult) * n);
    uint32_t ticket = 0;
    WvParams P{};
    P.jobs = sg.data(); P.results = sr.data(); P.order = nullptr; P.ticket = &ticket; P.count = (int)n;
    const unsigned grid = (unsigned)std::min<size_t>(n, 3);   // fewer CTAs than segments: the ticket loop is exercised
    P.scratch_stride = CL_SCRATCH;
    std::vector<uint8_t> scratch(P.scratch_stride * grid + 256, 0);
    P.scratch = scratch.data();
    simt::launch(grid, WV_THREADS, sizeof(ClShared), [&]() { inflate_cells_kernel(P); });
    *segments_used = (uint32_t)n;
    bool ok = true;
    uint64_t total = 0;
    for (size_t k = 0; k < n && ok; ++k) {
        const bool last = k + 1 == n;
        ok = sr[k].status == PNGB200_OK && (last ? sr[k].phase == 2 : (sr[k].phase == 1 && sr[k].consumed_bits == sg[k].stop_bit));
        total += sr[k].produced;
    }
    if (!ok || total > cap) return 1;
    std::vector<SegmentRecord> recs(n);
    std::vector<uint64_t> chunk_base(n);
    uint64_t off = 0, chunks = 0;
    for (size_t k = 0; k < n; ++k) {
        recs[k] = SegmentRecord{sym[k].data(), dst + off, sr[k].produced, 0, k == 0 ? 1u : 0u};
        chunk_base[k] = chunks;
        chunks += (sr[k].produced + 4095) / 4096;
        off += sr[k].produced;
    }
    std::vector<uint32_t> stream_first{0, (uint32_t)n};
    std::vector<uint8_t> windows((size_t)SEG_WINDOW * n, 0xEE);
    simt::launch(1, 256, 0, [&]() { window_propagate_kernel(recs.data(), stream_first.data(), 1, windows.data()); });
    if (chunks) simt::launch((unsigned)chunks, 256, 0, [&]() { marker_resolve_kernel(recs.data(), (uint32_t)n, windows.data(), chunk_base.data()); });
    *produced = total;
    return 0;
}
