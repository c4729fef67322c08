// Host build of png_walk_kernel under the SIMT emulator (tests/emu/simt.h): test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/png_walk.cuh"

#include <vector>

using namespace pngb200;

extern "C" size_t emu_walk_summary_size() { return sizeof(WalkSummary); }
extern "C" size_t emu_chunk_rec_size() { return sizeof(ChunkRec); }

// both passes over a batch of files, as pngb200_png_inspect_files / pngb200_png_decode_files launch them: pass 1 fills
// `sums` (count of them), the record bases follow from its chunk counts, pass 2 writes the records into `recs`
// (`recs_cap` of them); returns the number of records, or -1 when they do not fit
extern "C" long long emu_png_walk(int n, const uint8_t* const* files, const uint64_t* lens, WalkSummary* sums,
                                  ChunkRec* recs, uint64_t recs_cap, int order)
{
    std::vector<WalkFile> fs(n);
    for (int i = 0; i < n; ++i) fs[i] = {files[i], lens[i]};
    const unsigned grid = (unsigned)std::max(1, (n + WALK_WARPS - 1) / WALK_WARPS);
    simt::launch(grid, WALK_WARPS * 32, 0, [&]() { png_walk_kernel(fs.data(), (uint32_t)n, sums, nullptr, nullptr); }, order);
    std::vector<uint64_t> base(n + 1, 0);
    for (int i = 0; i < n; ++i) base[i + 1] = base[i] + sums[i].head.chunks;
    if (base[n] > recs_cap) return -1;
    simt::launch(grid, WALK_WARPS * 32, 0, [&]() { png_walk_kernel(fs.data(), (uint32_t)n, sums, recs, base.data()); }, order);
    return (long long)base[n];
}
