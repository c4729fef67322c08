// Host build of the streaming inflator's two kernels, inflate_serial_kernel and inflate_wave_kernel, under the SIMT
// emulator (tests/emu/simt.h), for one launch of a job with a resume record: test infrastructure.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/inflate_wave.cuh"

using namespace pngb200;

// One launch as pngb200_inflator_push makes it: the stream's first `len` bytes, resumed at (start_bit, start_out,
// phase) with the record `at` (read in phase 3, rewritten by the kernel).  engine 0: the serial kernel, 1: the ring
// kernel.  `cap`: bytes of dst.
extern "C" int emu_inflate_resume(int engine, const uint8_t* src, uint64_t len, uint8_t* dst, uint64_t cap, int format,
                                  uint64_t start_bit, uint64_t start_out, int phase, ResumePoint* at, StreamResult* res,
                                  int order)
{
    StreamJob job{};
    job.src = src; job.src_len = len; job.dst = dst; job.dst_cap = cap; job.format = format;
    job.start_bit = start_bit; job.start_out = start_out; job.phase = phase; job.resume = at;
    memset(res, 0, sizeof *res);
    at->bits = at->bytes = at->serial_bytes = 0;
    if (engine == 0) {
        simt::launch(1, 32, 0, [&]() { inflate_serial_kernel(&job, res, nullptr, 1); }, order);
        return res->status;
    }
    uint32_t ticket = 0;
    WvParams P{};
    P.jobs = &job; P.results = res; P.order = nullptr; P.ticket = &ticket; P.count = 1;
    P.bitmap_words = wv_bitmap_words(cap);
    P.scratch_stride = wv_scratch_stride(P.bitmap_words);
    std::vector<uint8_t> scratch(P.scratch_stride + 256, 0);
    P.scratch = scratch.data();
    simt::launch(1, WV_THREADS, sizeof(WvShared), [&]() { inflate_wave_kernel(P); }, order);
    return res->status;
}
extern "C" size_t emu_result_size() { return sizeof(StreamResult); }
extern "C" size_t emu_resume_size() { return sizeof(ResumePoint); }
extern "C" uint32_t emu_wave_bits() { return WV_BITS; }
