// Host build of deflate_resume_kernel under the SIMT emulator (tests/emu/simt.h): test infrastructure.
//
// One CTA takes every job of a launch through the kernel's grid-stride loop, for the reason emu_deflate.cpp gives.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/deflate.cuh"

using namespace pngb200;

extern "C" size_t emu_deflate_carry_size() { return sizeof(DfCarry); }
extern "C" void   emu_deflate_carry_init(DfCarry* c) { df_carry_init(*c); }

extern "C" void emu_deflate_resume(const DfResumeJob* jobs, int n, int order)
{
    simt::launch(1, 32, sizeof(DfShared), [&]() { deflate_resume_kernel(jobs, n); }, order);
}
