// Host build of the online encoder's two device steps under the SIMT emulator (tests/emu/simt.h): test infrastructure.
// filter_resume_kernel over the new scanlines of every handle of a push call, then deflate_resume_kernel with each
// handle's scanline ends (DfEnds), as pngb200_png_encoder_push_batch launches them.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/filter.cuh"
#include "../../swift-png_b200/csrc/deflate.cuh"

using namespace pngb200;

extern "C" size_t emu_encoder_filter_job_size() { return sizeof(FilterResumeJob); }
extern "C" size_t emu_encoder_carry_size() { return sizeof(DfCarry); }
extern "C" void   emu_encoder_carry_init(DfCarry* c) { df_carry_init(*c); }

// the warps of a launch are independent, so its CTAs run one after the other
extern "C" void emu_encoder_filter(const FilterResumeJob* jobs, const uint32_t* line_base, uint32_t njobs, uint32_t lines,
                                   int order)
{
    const unsigned grid = (lines + FILTER_WARPS - 1) / FILTER_WARPS;
    simt::launch(grid ? grid : 1, FILTER_WARPS * 32, 0,
                 [&]() { filter_resume_kernel(jobs, line_base, njobs, lines); }, order);
}

// one CTA takes every job through the kernel's grid-stride loop, as emu_deflate_resume.cpp does
extern "C" void emu_encoder_deflate(const DfResumeJob* jobs, int n, const DfEnds* ends, int order)
{
    simt::launch(1, 32, sizeof(DfShared), [&]() { deflate_resume_kernel(jobs, n, ends); }, order);
}
