// Host build of the head + tail pipeline with a tail that may leave symbolic mode (StreamJob.may_switch), as
// run_split() of pngb200_api.cu launches it: block_search_kernel, inflate_wave_kernel, split_resolve_kernel and
// split_finish_kernel under the SIMT emulator.  Test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/inflate_wave.cuh"
#include "../../swift-png_b200/csrc/block_search.cuh"
#include "../../swift-png_b200/csrc/inflate_segments.cuh"

using namespace pngb200;

extern "C" int emu_switch_result_size() { return (int)sizeof(StreamResult); }

// Cuts the zlib stream at the first plausible header at or after `share` of its bits (or at bit `plant` when nonzero)
// and runs both pieces through one launch of two CTAs.  The tail's scratch holds `tail_cap` symbols (2 tail_cap bytes;
// 0 = `cap`).  Returns 1 when split_finish_kernel accepted the stream (dst and *res then hold what a whole-stream
// decode gives), 0 when it asked for the whole-stream fallback, -1 when the search found no split point.  sw[0..1]: the
// tail's SwitchRecord (where it left symbolic mode, where its bytes start); 0, 0 when may_switch is 0.
extern "C" int emu_inflate_switch(const uint8_t* src, uint64_t len, uint8_t* dst, uint64_t cap, double share, uint64_t plant,
                                  uint64_t tail_cap, uint32_t may_switch, StreamResult* res, uint64_t* split_bit,
                                  StreamResult* pieces, uint64_t* sw)
{
    const uint64_t bits = 8 * len;
    uint64_t at = plant;
    if (!at) {
        SearchJob sj{src, len, (uint64_t)(share * (double)bits), bits, ~0ull};
        simt::launch(1, 256, 0, [&]() { block_search_kernel(&sj, 1); }, 0, false, 256 << 10, BS_CTAS);
        if (sj.found == ~0ull) return -1;
        at = sj.found;
    }
    *split_bit = at;
    if (!tail_cap) tail_cap = cap;
    std::vector<uint16_t> sym(tail_cap + 64, 0xDEAD);
    StreamJob jobs[2] = {};
    jobs[0].src = src; jobs[0].src_len = len; jobs[0].dst = dst; jobs[0].dst_cap = cap; jobs[0].format = PNGB200_FORMAT_ZLIB;
    jobs[1] = jobs[0];
    jobs[0].stop_bit = at;
    jobs[1].start_bit = at;
    jobs[1].phase = 1;
    jobs[1].symbolic = 1;
    jobs[1].may_switch = may_switch;
    jobs[1].dst = (uint8_t*)sym.data();
    jobs[1].dst_cap = tail_cap;
    StreamResult sr[2];
    memset(sr, 0, sizeof sr);
    uint32_t ticket = 0;
    WvParams P{};
    P.jobs = jobs; P.results = sr; P.order = nullptr; P.ticket = &ticket; P.count = 2;
    P.bitmap_words = wv_bitmap_words(cap);
    P.scratch_stride = wv_scratch_stride(P.bitmap_words);
    std::vector<uint8_t> scratch(P.scratch_stride * 2 + 256, 0);
    P.scratch = scratch.data();
    SwitchRecord switched[2] = {};
    P.switched = switched;
    simt::launch(2, WV_THREADS, sizeof(WvShared), [&]() { inflate_wave_kernel(P); });
    pieces[0] = sr[0];
    pieces[1] = sr[1];
    memset(res, 0, sizeof(StreamResult));
    SplitRecord rec{&sr[0], &sr[1], sym.data(), dst, cap, at, res, may_switch ? &switched[1] : nullptr};
    sw[0] = switched[1].out;
    sw[1] = switched[1].bytes;
    std::vector<uint32_t> partial(2 * SPLIT_CTAS, 0xFFFFFFFFu);
    uint32_t accept = 7;
    simt::launch(1, 256, 0, [&]() { split_resolve_kernel(&rec, partial.data()); }, 0, false, 256 << 10, SPLIT_CTAS);
    simt::launch(1, 128, 0, [&]() { split_finish_kernel(&rec, 1, partial.data(), &accept); });
    return (int)accept;
}
