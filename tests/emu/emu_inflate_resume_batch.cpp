// Host build of the streaming inflator's two kernels under the SIMT emulator (tests/emu/simt.h), for one launch over a
// table of jobs with resume records, as pngb200_inflator_push_batch launches them: test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/inflate_wave.cuh"

using namespace pngb200;

// n jobs in one launch: job k is the first len[k] bytes of src[k], resumed at (start_bit[k], start_out[k], phase[k])
// with the record at[k], into dst[k] of cap[k] bytes.  engine 0: inflate_serial_kernel, one CTA per job; 1:
// inflate_wave_kernel on `grid` CTAs pulling jobs from a ticket.  Results in res[k].
extern "C" void emu_inflate_resume_batch(int engine, int n, const uint8_t* const* src, const uint64_t* len,
                                         uint8_t* const* dst, const uint64_t* cap, const int* format,
                                         const uint64_t* start_bit, const uint64_t* start_out, const int* phase,
                                         ResumePoint* at, StreamResult* res, unsigned grid, int order)
{
    std::vector<StreamJob> jobs(n);
    uint64_t max_cap = 0;
    for (int k = 0; k < n; ++k) {
        StreamJob& j = jobs[k];
        j = StreamJob{};
        j.src = src[k]; j.src_len = len[k]; j.dst = dst[k]; j.dst_cap = cap[k]; j.format = format[k];
        j.start_bit = start_bit[k]; j.start_out = start_out[k]; j.phase = phase[k]; j.resume = &at[k];
        memset(&res[k], 0, sizeof res[k]);
        at[k].bits = at[k].bytes = at[k].serial_bytes = 0;
        max_cap = std::max(max_cap, cap[k]);
    }
    if (engine == 0) {
        simt::launch((unsigned)n, 32, 0, [&]() { inflate_serial_kernel(jobs.data(), res, nullptr, n); }, order);
        return;
    }
    WvParams P{};
    P.jobs = jobs.data(); P.results = res; P.order = nullptr; P.count = n;
    P.bitmap_words = wv_bitmap_words(max_cap);
    P.scratch_stride = wv_scratch_stride(P.bitmap_words);
    std::vector<uint8_t> scratch(P.scratch_stride * grid + 256, 0);
    P.scratch = scratch.data();
    P.ticket = (uint32_t*)(scratch.data() + P.scratch_stride * grid);
    simt::launch(grid, WV_THREADS, sizeof(WvShared), [&]() { inflate_wave_kernel(P); }, order);
}
