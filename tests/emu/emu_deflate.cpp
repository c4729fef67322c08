// Host build of deflate_kernel under the SIMT emulator (tests/emu/simt.h): test infrastructure.
//
// One CTA (one warp slot) takes every job of the batch through the kernel's ticket loop, so a slot's
// scratch and shared memory carry over from one stream to the next exactly as on the device.  One CTA
// is also a necessity here: simt.h turns the kernel's function-local __shared__ arrays (syms_s, mfreq,
// cl) into process-wide statics, which several CTAs would share.
#define PNGB200_EMU 1
#include "../../swift-png_b200/csrc/deflate.cuh"

#include <algorithm>
#include <vector>

using namespace pngb200;

// graph capacity and slot stride as run_deflate (csrc/pngb200_api.cu) sizes them
extern "C" void emu_deflate_batch(const DeflateJob* jobs, int n, DeflateResult* results, int order)
{
    uint64_t verts = 2;
    for (int i = 0; i < n; ++i)
        if (jobs[i].level >= 8) verts = std::max<uint64_t>(verts, std::min<uint64_t>(jobs[i].n, DF_GRAPH_CAP) + 2);
    DfParams P{};
    P.jobs = jobs;
    P.results = results;
    P.graph_vertices = verts;
    P.scratch_stride = df_scratch_stride(verts);
    std::vector<uint8_t> scratch(P.scratch_stride, 0xCD);   // the device workspace is not cleared either
    uint32_t ticket = 0;
    P.scratch = scratch.data();
    P.ticket = &ticket;
    P.count = n;
    std::fill(results, results + n, DeflateResult{});
    simt::launch(1, 32, sizeof(DfShared), [&]() { deflate_kernel(P); }, order);
}
