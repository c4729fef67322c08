// common.cuh -- device-side job/result records and small helpers shared by all kernels.
#pragma once

#ifdef PNGB200_EMU
// host-side SIMT emulation of the kernels (tests/emu/simt.h): test infrastructure, never the product
#include "simt.h"
#else
#include <cuda_runtime.h>
#define PNGB200_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif
#include <stdint.h>

#include "../../include/pngb200.h"

namespace pngb200 {

// Where a streaming decode stopped inside a fixed or dynamic block, and the work one launch did.  Only the streaming
// handle passes one (StreamJob.resume); the kernel reads the position when the job starts in phase 3 and writes it
// when it stops inside a Huffman block for want of input (StreamResult.phase 3).
struct ResumePoint {
    uint64_t header_bit;   // the block's header
    uint64_t symbol_bit;   // its next undecoded symbol
    uint64_t out;          // output size at symbol_bit
    uint32_t final;        // the block's BFINAL
    uint32_t pad_;
    // the launch's work, set by the kernel: input bits decoded (a bit decoded twice counts twice), output bytes
    // written, and how many of those the one-warp serial decoder wrote
    uint64_t bits, bytes, serial_bytes;
};

// One DEFLATE stream to inflate (device-resident record).
struct StreamJob {
    const uint8_t* src;
    uint64_t       src_len;
    uint8_t*       dst;
    uint64_t       dst_cap;
    uint64_t       start_bit;   // resume point (bit offset of a block header, or of a symbol in phase 3), 0 = the top
    uint64_t       start_out;   // bytes already produced before start_bit
    int32_t        format;      // pngb200_format
    int32_t        phase;       // where to resume: 0 stream header, 1 block header, 2 trailer, 3 inside the Huffman
                                // block whose header is at resume->header_bit (its header is parsed again)
    // segments of a stream that several CTAs decode side by side (inflate_wave_kernel only):
    uint64_t       stop_bit;    // 0 = to the end of the stream; else stop at the first block boundary >= stop_bit
    uint32_t       symbolic;    // 1: dst is uint16_t[dst_cap]; a byte copied from in front of the segment becomes
                                // the marker 0x8000 | index into the 32 KiB window that precedes the segment
    uint32_t       may_switch;  // symbolic tails of a stream cut in two: once the last 32 KiB hold no marker, go on
                                // in bytes behind the symbols (dst then holds 2 dst_cap bytes; SwitchRecord)
    // host-side planning only (no kernel reads them): a device buffer of `scratch_cap` bytes that is dead while the
    // stream is inflated (the image's pixel buffer, written by unfilter afterwards), or null
    uint8_t*       scratch;
    uint64_t       scratch_cap;
    // the streaming handle's resume record (serial and ring kernels only), or null: then a decode that runs out of
    // input inside a block resumes at the block's header
    ResumePoint*   resume;
};

struct StreamResult {
    int32_t  status;
    uint32_t err_a, err_b;
    uint32_t checksum;
    uint32_t blocks;
    uint32_t declared;        // trailer checksum as read from the stream
    uint64_t produced;
    uint64_t consumed_bits;
    uint64_t resume_bit;      // start of the last block header not yet completed
    uint64_t resume_out;      // output size at resume_bit
    uint32_t trailer_seen;    // 1 when the final block and trailer were parsed
    uint32_t phase;           // phase to resume in at resume_bit (see StreamJob.phase)
    // device-side counters (the reference's -DDUMP_LZ77_BLOCKS style statistics)
    uint32_t stat_waves, stat_sync_rounds, stat_resolve_rounds, stat_fallback;
    uint64_t stat_tokens, stat_matches, stat_deferred;  // tokens / LZ77 matches on the stream, matches that had to wait
    uint32_t ck_done;         // 1: `checksum` was computed (and compared) by the inflate kernel itself
    uint32_t pad_;
    // SM cycles thread 0 of the stream's CTA spent per phase of the wave kernel (each ends at a barrier):
    // 0 header+tables 1 stage 2 speculate 3 walk 4 chain 5 count+scan 6 emit 7 resolve 8 store 9 stored blocks
    uint64_t stat_cycles[12];
};

// Where a symbolic job with may_switch left symbolic mode (inflate_wave_kernel, WvParams.switched): output [0, out)
// is symbols at dst, [out, produced) bytes that start at byte `bytes` of dst.  out = produced: it never switched.
struct SwitchRecord {
    uint64_t out;
    uint64_t bytes;
};

// One image for the unfilter stage.
struct ImageJob {
    const uint8_t*      filtered;   // inflated IDAT stream
    uint8_t*            pixels;     // PNG.Image.storage
    const StreamResult* inflated;   // producer's result (rows available = produced / (pitch+1)); may be null
    uint64_t            filtered_len;  // used when `inflated` is null
    uint32_t            width, height;
    uint32_t            pitch;      // bytes per row (non-interlaced)
    uint8_t             volume, depth, interlaced, bpp;
};

// bytes of filtered stream that may be consumed: nothing after an inflate error (the reference
// throws out of Inflator.push before any row is pulled), everything produced otherwise
__device__ __forceinline__ uint64_t usable_bytes(const StreamResult* r, uint64_t fallback)
{
    if (r == nullptr) return fallback;
    return r->status < 0 ? 0 : r->produced;
}

__device__ __forceinline__ unsigned lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p)
{
#ifdef PNGB200_EMU
    return *(const volatile uint32_t*)p;
#else
    uint32_t v;
    asm volatile("ld.volatile.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
#endif
}
__device__ __forceinline__ void st_volatile_u32(uint32_t* p, uint32_t v)
{
#ifdef PNGB200_EMU
    *(volatile uint32_t*)p = v;
#else
    asm volatile("st.volatile.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#endif
}

}  // namespace pngb200
