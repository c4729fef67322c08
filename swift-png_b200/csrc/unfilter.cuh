// unfilter.cuh -- PNG scanline reconstruction (None/Sub/Up/Average/Paeth) + PNG.Image.assign.
//
// Replaces PNG.Decoder.defilter (Sources/PNG/Decoding/PNG.Decoder.swift:152-196), PNG.paeth
// (Sources/PNG/PNG.swift:124-147), the row loop of PNG.Decoder.push (:113-140) and the straight
// copy cases of PNG.Image.assign (Sources/PNG/PNG.Image.swift:218-283).
//
// unfilter_wave_kernel (the fast path: non-interlaced, >= 8 bits per sample):
//   Average and Paeth make byte x of row y depend on (x-bpp, y), (x, y-1), (x-bpp, y-1); that is
//   a 2-D wavefront, not a scan.  A warp owns a band of 32 consecutive rows, lane l = row y0+l,
//   and sweeps left to right in 16-byte chunks with lane l one chunk behind lane l-1; the chunk a
//   lane has just reconstructed is handed to the lane below with one shuffle (it is that lane's
//   "previous row").  Bands are pipelined the same way through HBM/L2: the last row of band k is
//   the previous row of band k+1, published chunk-by-chunk with a progress counter.  Bands are
//   handed out by an atomic ticket in row order, so a band's predecessor is always already
//   running (no deadlock whatever the residency).  Each lane stages its own row through a
//   shared-memory ring in 16-byte chunks (see WAVE_DEPTH) and writes its chunks in pairs: two
//   back-to-back 16-byte stores that fill a whole 32-byte sector (see wave_band).
//
// unfilter_pass_kernel (Adam7 and 1/2/4-bit images whose filtered stream is longer than UNFILTER_GENERIC_MAX):
//   the same wavefront over PassJobs.  An Adam7 pass is an ordinary filtered image of its own width and height with
//   the image's filter distance, and the rows of a 1/2/4-bit image are byte rows with filter distance 1, so each pass
//   (or the whole sub-byte image) is one job.  Rows are reconstructed in place in the library's private copy of the
//   filtered stream; unfilter_interleave_kernel then writes PNG.Image.storage from the pass rows.
//
// unfilter_generic_kernel: the same formats when the filtered stream is short; one CTA per image.
#pragma once

#include <algorithm>
#include <type_traits>
#include <vector>

#include "common.cuh"

namespace pngb200 {

// ---- per-byte SIMD-in-word arithmetic ----
__device__ __forceinline__ uint32_t avg_floor4(uint32_t a, uint32_t b)
{
    return (a & b) + (((a ^ b) & 0xfefefefeu) >> 1);
}
// PNG.paeth on four byte lanes at once.  With pa=|b-c|, pb=|a-c|: pc=|a+b-2c| equals pa+pb when
// (b-c) and (a-c) have the same sign and |pa-pb| otherwise; a saturating add is enough because a
// saturated pc (255) still compares >= pa and >= pb exactly as the true value does.
__device__ __forceinline__ uint32_t paeth4(uint32_t a, uint32_t b, uint32_t c)
{
    uint32_t pa   = __vabsdiffu4(b, c);
    uint32_t pb   = __vabsdiffu4(a, c);
    uint32_t same = ~(__vcmpgeu4(b, c) ^ __vcmpgeu4(a, c));
    uint32_t pc   = (same & __vaddus4(pa, pb)) | (~same & __vabsdiffu4(pa, pb));
    uint32_t sa   = __vcmpleu4(pa, pb) & __vcmpleu4(pa, pc);
    uint32_t sb   = ~sa & __vcmpleu4(pb, pc);
    return (a & sa) | (b & sb) | (c & ~(sa | sb));
}
__device__ __forceinline__ uint32_t paeth1(uint32_t a, uint32_t b, uint32_t c)
{
    int pa = abs((int)b - (int)c), pb = abs((int)a - (int)c), pc = abs((int)a + (int)b - 2 * (int)c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}
__device__ __forceinline__ uint32_t predict4(uint32_t type, uint32_t a, uint32_t b, uint32_t c, bool any_paeth)
{
    uint32_t p = type == 1 ? a : type == 2 ? b : type == 3 ? avg_floor4(a, b) : 0u;
    if (any_paeth) {
        uint32_t pp = paeth4(a, b, c);
        p = type == 4 ? pp : p;
    }
    return p;
}

// 16 bytes starting `m` bytes into the 32-byte window (lo, hi)
__device__ __forceinline__ uint4 shift_bytes(uint4 lo, uint4 hi, uint32_t m)
{
    uint32_t w[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
    uint32_t mw = m >> 2;
    if (mw & 2) {
#pragma unroll
        for (int i = 0; i < 6; ++i) w[i] = w[i + 2];
    }
    if (mw & 1) {
#pragma unroll
        for (int i = 0; i < 5; ++i) w[i] = w[i + 1];
    }
    uint32_t sel = 0x3210u + 0x1111u * (m & 3);
    uint4    r;
    r.x = __byte_perm(w[0], w[1], sel);
    r.y = __byte_perm(w[1], w[2], sel);
    r.z = __byte_perm(w[2], w[3], sel);
    r.w = __byte_perm(w[3], w[4], sel);
    return r;
}

__device__ __forceinline__ uint4 load16_any(const uint8_t* p, bool l2_only)
{
    uintptr_t a = (uintptr_t)p;
    uint32_t  m = a & 15;
    const uint4* q = (const uint4*)(a - m);
    if (l2_only) {
        uint4 lo = __ldcg(q);
        if (m == 0) return lo;
        return shift_bytes(lo, __ldcg(q + 1), m);
    }
    uint4 lo = *q;
    if (m == 0) return lo;
    return shift_bytes(lo, q[1], m);
}

__device__ __forceinline__ void store16_partial(uint8_t* p, uint4 v, int nbytes)
{
    if (nbytes >= 16 && (((uintptr_t)p) & 15) == 0) {
        *(uint4*)p = v;
        return;
    }
    uint32_t w[4] = {v.x, v.y, v.z, v.w};
    if ((((uintptr_t)p) & 3) == 0) {
        int i = 0;
        for (; i + 4 <= nbytes && i < 16; i += 4) *(uint32_t*)(p + i) = w[i >> 2];
        for (; i < nbytes && i < 16; ++i) p[i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
    } else {
        for (int i = 0; i < nbytes && i < 16; ++i) p[i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
    }
}

// ---- the layout of a filtered stream, shared by every scanline kernel and the host ----
// Adam7 (PNG.adam7, PNG.Decoder.swift:6-15): pass z holds the pixels (bx + (i << ex), by + (r << ey)), as
// {bx, by, ex, ey}.  The host reads h_adam7, the device its copy in constant memory.  The copy is defined here, after
// the inflate and deflate tables (huffman.cuh, deflate.cuh), so that it does not move their constant-bank addresses.
struct Adam7Table {
    int p[7][4];
};
constexpr Adam7Table h_adam7 = {{{0, 0, 3, 3}, {4, 0, 3, 3}, {0, 4, 2, 3}, {2, 0, 2, 2}, {0, 2, 1, 2}, {1, 0, 1, 1}, {0, 1, 0, 1}}};
__constant__ Adam7Table c_adam7 = h_adam7;

// One pass of a filtered stream: Adam7 pass z of an interlaced image, or for z = 0 the whole of a non-interlaced one,
// whose passes 1 to 6 are empty.  Its rows lie back to back, each a filter byte and `pitch` bytes; an empty Adam7 pass
// has width = height = 0.  Sizes are 64-bit: a pass's width * volume passes 2^32 long before geometry()'s limits.
struct Pass {
    uint32_t bx, by, ex, ey;  // row r holds the pixels (bx + (i << ex), by + (r << ey)), i < width
    uint64_t width, height;   // pixels per row, rows
    uint64_t pitch;           // bytes per row, not counting the filter byte
};

__host__ __device__ __forceinline__ Pass stream_pass(int z, uint32_t w, uint32_t h, uint64_t volume, bool interlaced)
{
    Pass s = {0, 0, 0, 0, z == 0 ? w : 0u, z == 0 ? h : 0u, 0};
    if (interlaced) {
#ifdef __CUDA_ARCH__
        const int* a = c_adam7.p[z];
#else
        const int* a = h_adam7.p[z];
#endif
        s.bx = a[0]; s.by = a[1]; s.ex = a[2]; s.ey = a[3];
        s.width  = ((uint64_t)w + (1u << s.ex) - s.bx - 1) >> s.ex;
        s.height = ((uint64_t)h + (1u << s.ey) - s.by - 1) >> s.ey;
        if (s.width == 0 || s.height == 0) s.width = s.height = 0;
    }
    s.pitch = (s.width * volume + 7) >> 3;
    return s;
}

// bytes of the filtered stream in front of pass z; z = 7 gives the length of the whole stream.  The loop has a fixed
// trip count so that the compiler unrolls it: a loop up to z costs unfilter_interleave_kernel 8 more registers.
__host__ __device__ __forceinline__ uint64_t stream_pass_offset(int z, uint32_t w, uint32_t h, uint64_t volume, bool interlaced)
{
    uint64_t off = 0;
    for (int k = 0; k < 7; ++k) {
        const Pass s = stream_pass(k, w, h, volume, interlaced);
        if (k < z) off += s.height * (s.pitch + 1);
    }
    return off;
}

// One Adam7 pass of an image, or the whole of a non-interlaced 1/2/4-bit image, for unfilter_pass_kernel.  Its rows are
// reconstructed in place: the pixels of row y overwrite that row's filtered bytes, at stride pitch + 1, offset 1.
struct PassJob {
    uint8_t*            filtered;      // the pass's first filter byte in the image's private (mutable) filtered stream
    const StreamResult* inflated;      // the image's producer result, as ImageJob; may be null
    uint64_t            filtered_len;  // used when `inflated` is null
    uint64_t            offset;        // bytes of the image's stream in front of the pass
    uint32_t            height, pitch; // rows and bytes per row of the pass
    uint32_t            bpp;           // filter distance
};

struct WaveParams {
    const void*     jobs;       // ImageJob[] (unfilter_wave_kernel) or PassJob[] (unfilter_pass_kernel)
    const uint32_t* band_base;  // [njobs + 1] exclusive prefix of ceil(h/32)
    uint32_t*       progress;   // [total_bands]
    uint32_t*       ticket;
    uint32_t        njobs;
    uint32_t        total_bands;
    // Ticket order.  levels == 0: image after image (ticket = band_base[image] + band).  Otherwise band LEVEL after
    // level: jobs[] is sorted by band count (descending), level_start[b] = tickets in front of level b = sum over
    // b' < b of the images that have more than b' bands, and ticket level_start[b] + r is band b of image r.  A band
    // follows the band above it by ~40 steps, so of one image's bands only duration / 40 can be busy at a time; handed
    // out image by image the resident warps hold ALL bands of a few images and most of them wait for their turn;
    // handed out level by level they hold a few bands of every image.
    const uint32_t* level_start;   // [levels + 1]
    uint32_t        levels;
    unsigned long long* hist;   // [6]: scanlines per filter type 0..4, [5] = invalid filter bytes (the reference's
                                // -DDUMP_FILTERED_SCANLINES view of a decode, PNG.Decoder.swift:96-98,128); may be null
};

// Asynchronous staging of a lane's own row (cp.async = LDGSTS: global -> shared memory without a register in
// between).  Every lane keeps a private ring of WAVE_DEPTH aligned 16-byte chunks of its row in shared memory: the
// first WAVE_DEPTH chunks are issued before the sweep, and step j issues chunk j + WAVE_DEPTH into the slot chunk j
// has just left.  Reconstructed chunks are stored from registers, two at a time.  The rings are the CTA's whole shared
// memory (WAVE_SMEM, 32 KiB); a deeper ring, or a second one for the output or for lane 0's row above, costs resident
// warps, and the kernel's throughput follows resident warps, not lookahead per warp (DESIGN §4.3).
constexpr int      WAVE_WARPS   = 4;    // warps per CTA
constexpr int      WAVE_DEPTH   = 16;   // ring slots per lane
constexpr int      WAVE_PUBLISH = 8;    // publish progress every this many chunks
static_assert(WAVE_PUBLISH % 2 == 0, "progress must only ever count chunk pairs that have been stored");
constexpr unsigned WAVE_POLL_NS = 64;   // lane 0's back-off while the band above has not published the chunk it needs
constexpr size_t   WAVE_SMEM    = sizeof(uint4) * 32 * (size_t)WAVE_WARPS * WAVE_DEPTH;
__device__ __forceinline__ void cp_async16(uint4* smem, const uint4* gmem)
{
#ifdef PNGB200_EMU
    *smem = *gmem;
#else
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem)), "l"(gmem) : "memory");
#endif
}
__device__ __forceinline__ void cp_async_commit()
{
#ifndef PNGB200_EMU
    asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
template <int N>
__device__ __forceinline__ void cp_async_wait()   // at most N of this thread's groups still in flight
{
#ifndef PNGB200_EMU
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
#endif
}

// Where wave_band writes the pixels of a row: an ImageJob's go to PNG.Image.storage at stride pitch, a PassJob's over the
// row's own filtered bytes, at stride pitch + 1 from offset 1.
__device__ __forceinline__ uint8_t* wave_out(const ImageJob& job) { return job.pixels; }
__device__ __forceinline__ uint32_t wave_out_stride(const ImageJob& job) { return job.pitch; }
__device__ __forceinline__ uint8_t* wave_out(const PassJob& job) { return job.filtered + 1; }
__device__ __forceinline__ uint32_t wave_out_stride(const PassJob& job) { return job.pitch + 1; }
// Rows of the job the stream delivered in full (wave_band also stops at the job's height).  A pass starts `offset`
// bytes into its image's stream: when the stream ends in front of it, or after an inflate error, it has none.
__device__ __forceinline__ uint64_t wave_rows(const ImageJob& job, uint32_t pitch)
{
    return usable_bytes(job.inflated, job.filtered_len) / (pitch + 1);
}
__device__ __forceinline__ uint64_t wave_rows(const PassJob& job, uint32_t pitch)
{
    const uint64_t usable = usable_bytes(job.inflated, job.filtered_len);
    return usable > job.offset ? (usable - job.offset) / (pitch + 1) : 0;
}

// Job is ImageJob or PassJob.  In place (PassJob), the rows of a job lie back to back, so the aligned 16-byte chunk a
// lane stages first also holds the tail of the row above, and the last one it stages the head of the row below; lane 0
// reading the band above's last row through load16_any reads the head of its own row with it.  Those neighbours may be
// rewriting the bytes in the meantime: they lie outside the row and are read and discarded.  A lane's own input bytes
// are never rewritten before they are read: output chunk j covers aligned input chunks j and j + 1, and it is stored
// at step j or j + 1, after the ring has taken both (cp_async_wait below).
template <int BPP, typename Job>
__device__ void wave_band(const Job& job, uint32_t band, uint32_t* prog_prev, uint32_t* prog_mine, uint4 (*ring)[32],
                          unsigned long long* hist)
{
    constexpr bool in_place = std::is_same<Job, PassJob>::value;
    const unsigned lane   = lane_id();
    const uint32_t y      = band * 32 + lane;
    const uint32_t pitch  = job.pitch;
    const uint64_t rows   = wave_rows(job, pitch);
    const bool     active = y < job.height && y < rows;
    const int      nchunk = (int)((pitch + 15) >> 4);
    const uint8_t* row    = job.filtered + (uint64_t)(active ? y : 0) * (pitch + 1);
    uint32_t       type   = active ? row[0] : 0;
    if (hist != nullptr) {   // filter-type histogram of the batch: one atomic per type per band
        const uint32_t raw = active ? min(type, 5u) : 6u;
#pragma unroll
        for (uint32_t k = 0; k < 6; ++k) {
            const unsigned m = __ballot_sync(0xffffffffu, raw == k);
            if (lane == 0 && m) atomicAdd(hist + k, (unsigned long long)__popc(m));
        }
    }
    if (type > 4) type = 0;  // invalid filter byte: row unchanged (PNG.Decoder.swift:193-194)
    const bool any_paeth = __any_sync(0xffffffffu, type == 4);
    const uint8_t* in    = row + 1;
    const uint32_t m     = (uint32_t)((uintptr_t)in & 15);
    const uint4*   inq   = (const uint4*)(in - m);
    const int      nq    = (int)(((uint64_t)m + pitch + 15) >> 4);  // aligned chunks that hold row bytes
    uint8_t*       out   = wave_out(job) + (uint64_t)(active ? y : 0) * wave_out_stride(job);
    const uint8_t* above = band == 0 ? nullptr : wave_out(job) + (uint64_t)(band * 32 - 1) * wave_out_stride(job);
    const bool     publish = lane == 31 && prog_mine != nullptr;
    // rows the stream did not deliver (a complete zlib stream that is shorter than the image is not an error in
    // the reference: the rows simply stay as PNG.Image.storage was initialised, zero -- PNG.Image.swift:84).  In
    // place they are left alone: unfilter_interleave_kernel writes their zeros, and the stream may end inside them.
    if constexpr (!in_place) {
        if (!active && y < job.height) {
            uint8_t* z = job.pixels + (uint64_t)y * pitch;
            for (uint32_t k = 0; k < pitch; ++k) z[k] = 0;
        }
    }

    uint4    qcur  = make_uint4(0, 0, 0, 0);
    uint4    mine  = make_uint4(0, 0, 0, 0);  // my last reconstructed chunk
    uint4    held  = make_uint4(0, 0, 0, 0);  // even chunk j, stored together with chunk j + 1
    uint32_t a0 = 0, a1 = 0, c0 = 0, c1 = 0;  // BPP 4/8 histories (words)
    uint64_t ah = 0, ch = 0;                  // generic byte histories
    uint32_t seen = 0;
    uint4    upn = make_uint4(0, 0, 0, 0);  // lane 0: the chunk of the row above for the next step
    bool     upn_ok = false;
    // input chunk k of my row is cp.async group k of this thread: WAVE_DEPTH groups are opened here, one more per
    // step, so when chunk j is consumed the groups up to j + 1 must have landed = at most WAVE_DEPTH - 2 in flight
    if (active) {
#pragma unroll
        for (int k = 0; k < WAVE_DEPTH; ++k) {
            if (k < nq) cp_async16(&ring[k][lane], inq + k);
            cp_async_commit();
        }
    }

    for (int S = 0; S < nchunk + 32; ++S) {
        const int j = S - (int)lane;
        uint4     up = mine;
        up.x = __shfl_up_sync(0xffffffffu, mine.x, 1);
        up.y = __shfl_up_sync(0xffffffffu, mine.y, 1);
        up.z = __shfl_up_sync(0xffffffffu, mine.z, 1);
        up.w = __shfl_up_sync(0xffffffffu, mine.w, 1);
        if (lane == 0) {
            // the band above publishes its last row chunk by chunk; its chunk j + 1 is fetched while chunk j
            // is being used, so the L2 round trip of that load is off the warp's critical path
            up = make_uint4(0, 0, 0, 0);
            if (active && above != nullptr && j < nchunk) {
                if (upn_ok) {
                    up = upn;
                } else {
                    const uint32_t want = min((uint32_t)j + 1u, (uint32_t)nchunk);   // chunks the band above must have published
                    while (seen < want) {
                        seen = ld_volatile_u32(prog_prev);
                        if (seen < want) __nanosleep(WAVE_POLL_NS);
                    }
                    up = load16_any(above + 16 * (uint64_t)j, true);
                }
                upn_ok = false;
                if (j + 1 < nchunk) {
                    if (seen <= (uint32_t)(j + 1)) seen = ld_volatile_u32(prog_prev);
                    if (seen > (uint32_t)(j + 1)) {
                        upn = load16_any(above + 16 * (uint64_t)(j + 1), true);
                        upn_ok = true;
                    }
                }
            }
        }
        if (active && j >= 0 && j < nchunk) {
            cp_async_wait<WAVE_DEPTH - 2>();
            qcur = ring[j % WAVE_DEPTH][lane];
            const uint4 qnext = ring[(j + 1) % WAVE_DEPTH][lane];
            uint4 x = m == 0 ? qcur : shift_bytes(qcur, qnext, m);
            // chunk j + WAVE_DEPTH takes the slot chunk j just left (x depends on the loads above: they are done)
            if (j + WAVE_DEPTH < nq) cp_async16(&ring[j % WAVE_DEPTH][lane], inq + j + WAVE_DEPTH);
            cp_async_commit();
            uint4 o;
            if (BPP == 4) {
                o.x = __vadd4(x.x, predict4(type, a1, up.x, c1, any_paeth));
                o.y = __vadd4(x.y, predict4(type, o.x, up.y, up.x, any_paeth));
                o.z = __vadd4(x.z, predict4(type, o.y, up.z, up.y, any_paeth));
                o.w = __vadd4(x.w, predict4(type, o.z, up.w, up.z, any_paeth));
                a1 = o.w;
                c1 = up.w;
            } else if (BPP == 8) {
                o.x = __vadd4(x.x, predict4(type, a0, up.x, c0, any_paeth));
                o.y = __vadd4(x.y, predict4(type, a1, up.y, c1, any_paeth));
                o.z = __vadd4(x.z, predict4(type, o.x, up.z, up.x, any_paeth));
                o.w = __vadd4(x.w, predict4(type, o.y, up.w, up.y, any_paeth));
                a0 = o.z; a1 = o.w;
                c0 = up.z; c1 = up.w;
            } else {
                uint32_t xs[4] = {x.x, x.y, x.z, x.w}, us[4] = {up.x, up.y, up.z, up.w}, os[4];
#pragma unroll
                for (int w = 0; w < 4; ++w) {
                    uint32_t ow = 0;
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        uint32_t xb = (xs[w] >> (8 * k)) & 0xff, b = (us[w] >> (8 * k)) & 0xff;
                        uint32_t a = (uint32_t)(ah >> (8 * (BPP - 1))) & 0xff;
                        uint32_t c = (uint32_t)(ch >> (8 * (BPP - 1))) & 0xff;
                        uint32_t p = type == 1 ? a : type == 2 ? b : type == 3 ? (a + b) >> 1
                                   : type == 4 ? paeth1(a, b, c) : 0u;
                        uint32_t ob = (xb + p) & 0xff;
                        ow |= ob << (8 * k);
                        ah = (ah << 8) | ob;
                        ch = (ch << 8) | b;
                    }
                    os[w] = ow;
                }
                o = make_uint4(os[0], os[1], os[2], os[3]);
            }
            // Chunks 2k and 2k + 1 are stored back to back, one step late for the even one: a lone 16-byte store
            // leaves half a 32-byte sector dirty in L2 for a whole step (thousands of cycles, ~100 K rows in flight),
            // and on the H100 those half-written sectors cost the kernel half its bandwidth.  The band below reads
            // this row only up to the published progress, which always counts pairs that have been stored.
            if ((j & 1) == 0 && j + 1 < nchunk) {
                held = o;
            } else {
                if (j & 1) store16_partial(out + 16 * (uint64_t)(j - 1), held, 16);
                // bytes of the row from chunk j on, capped at 16 before the narrowing: pitch can pass 2^31
                store16_partial(out + 16 * (uint64_t)j, o, (int)min(pitch - 16u * (uint32_t)j, 16u));
            }
            mine = o;
            if (publish && (((j + 1) % WAVE_PUBLISH) == 0 || j + 1 == nchunk)) {
                __threadfence();
                st_volatile_u32(prog_mine, (uint32_t)(j + 1));
            }
        }
    }
    cp_async_wait<0>();   // nothing of this band may still land in the ring when the warp takes its next band
    __syncwarp();
}

template <typename Job>
__device__ __forceinline__ void wave_run(const WaveParams& p)
{
    PNGB200_DYN_SMEM(wave_smem);   // [warp][slot][lane] input rings: conflict-free 16-byte accesses
    uint4 (*ring)[32] = reinterpret_cast<uint4 (*)[32]>(wave_smem) + (threadIdx.x >> 5) * WAVE_DEPTH;
    const unsigned lane = lane_id();
    for (;;) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd(p.ticket, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= p.total_bands) return;
        uint32_t lo = 0, band, gidx;
        if (p.levels) {
            // level of ticket t: last b with level_start[b] <= t
            uint32_t hi = p.levels;
            while (hi - lo > 1) {
                uint32_t mid = (lo + hi) >> 1;
                if (p.level_start[mid] <= t) lo = mid;
                else hi = mid;
            }
            band = lo;
            lo   = t - p.level_start[band];          // image (rank in the sorted job list)
            gidx = p.band_base[lo] + band;
        } else {
            // image owning ticket t: last index with band_base[i] <= t
            uint32_t hi = p.njobs;
            while (hi - lo > 1) {
                uint32_t mid = (lo + hi) >> 1;
                if (p.band_base[mid] <= t) lo = mid;
                else hi = mid;
            }
            band = t - p.band_base[lo];
            gidx = t;
        }
        const Job      job   = static_cast<const Job*>(p.jobs)[lo];
        const uint32_t nband = p.band_base[lo + 1] - p.band_base[lo];
        uint32_t*      prev  = band == 0 ? nullptr : p.progress + gidx - 1;
        uint32_t*      mine  = band + 1 < nband ? p.progress + gidx : nullptr;
        switch (job.bpp) {
        case 1: wave_band<1>(job, band, prev, mine, ring, p.hist); break;
        case 2: wave_band<2>(job, band, prev, mine, ring, p.hist); break;
        case 3: wave_band<3>(job, band, prev, mine, ring, p.hist); break;
        case 4: wave_band<4>(job, band, prev, mine, ring, p.hist); break;
        case 6: wave_band<6>(job, band, prev, mine, ring, p.hist); break;
        default: wave_band<8>(job, band, prev, mine, ring, p.hist); break;
        }
    }
}

__global__ void __launch_bounds__(WAVE_WARPS * 32) unfilter_wave_kernel(WaveParams p) { wave_run<ImageJob>(p); }

// p.hist must be null: the filter histogram counts the non-interlaced images of 8 bits or more only
__global__ void __launch_bounds__(WAVE_WARPS * 32) unfilter_pass_kernel(WaveParams p) { wave_run<PassJob>(p); }

// An Adam7 or 1/2/4-bit image for unfilter_generic_kernel, which reconstructs its rows in place and assigns them, or
// for unfilter_interleave_kernel, which assigns the passes unfilter_pass_kernel reconstructed in place.
struct PassImageJob {
    uint8_t*            filtered;      // the image's private (mutable) filtered stream
    uint8_t*            pixels;        // PNG.Image.storage
    const StreamResult* inflated;      // may be null
    uint64_t            filtered_len;  // used when `inflated` is null
    uint64_t            block_base;    // the image's first CTA block of the launch (unfilter_interleave_kernel only)
    uint32_t            width, height;
    uint8_t             volume, depth, interlaced, bpp;
};
using GenericJob    = PassImageJob;   // each kernel's name for its job
using InterleaveJob = PassImageJob;

// ---- generic path: Adam7 and sub-byte depths.  One CTA per image; defilters in place. ----
__global__ void __launch_bounds__(128) unfilter_generic_kernel(const GenericJob* jobs, int count)
{
    if ((int)blockIdx.x >= count) return;
    const GenericJob job = jobs[blockIdx.x];
    const int        tid = threadIdx.x, nt = blockDim.x;
    const uint32_t   bpp = job.bpp;
    uint8_t*         at  = job.filtered;
    // PNG.Image.storage starts out zeroed (PNG.Image.swift:84): pixels no row reaches stay zero
    {
        const uint64_t total = (uint64_t)job.width * job.height * bpp;
        for (uint64_t k = tid; k < total; k += nt) job.pixels[k] = 0;
        __syncthreads();
    }
    const uint8_t*   end = job.filtered + usable_bytes(job.inflated, job.filtered_len);
    for (int z = 0; z < 7; ++z) {
        const Pass ps = stream_pass(z, job.width, job.height, job.volume, job.interlaced);
        // the pitch fits 32 bits (geometry() caps it at 0xfffffff0); the byte loops below count in 64 bits so that
        // i + nt cannot wrap
        const uint32_t sw = (uint32_t)ps.width, shh = (uint32_t)ps.height, pitch = (uint32_t)ps.pitch;
        uint8_t*       last  = nullptr;
        for (uint32_t y = 0; y < shh; ++y) {
            if (at + pitch + 1 > end) return;  // inflator.pull(pitch + 1) == nil
            uint8_t*      line = at + 1;
            const uint8_t type = at[0];
            if (type == 2) {
                if (last)
                    for (uint64_t i = tid; i < pitch; i += nt) line[i] = (uint8_t)(line[i] + last[i]);
            } else if (type == 1 || type == 3 || type == 4) {
                if ((uint32_t)tid < bpp) {  // channels are independent chains
                    for (uint64_t i = tid; i < pitch; i += bpp) {
                        uint32_t a = i >= bpp ? line[i - bpp] : 0;
                        uint32_t b = last ? last[i] : 0;
                        uint32_t c = (last && i >= bpp) ? last[i - bpp] : 0;
                        uint32_t p = type == 1 ? a : type == 3 ? (a + b) >> 1 : paeth1(a, b, c);
                        line[i] = (uint8_t)(line[i] + p);
                    }
                }
            }
            __syncthreads();
            // PNG.Image.assign
            const uint32_t oy = ps.by + (y << ps.ey);
            if (job.depth < 8) {
                const uint32_t per = 8 / job.depth, mask = (1u << job.depth) - 1;
                for (uint32_t i = tid; i < sw; i += nt) {
                    uint32_t sh = ((~i) & (per - 1)) * job.depth;
                    job.pixels[(uint64_t)oy * job.width + ps.bx + ((uint64_t)i << ps.ex)] =
                        (uint8_t)((line[i / per] >> sh) & mask);
                }
            } else {
                for (uint64_t k = tid; k < pitch; k += nt) {   // depth >= 8: sw * bpp == pitch
                    uint32_t i = (uint32_t)k / bpp, c = (uint32_t)k - i * bpp;
                    job.pixels[((uint64_t)oy * job.width + ps.bx + ((uint64_t)i << ps.ex)) * bpp + c] = line[k];
                }
            }
            last = line;
            at += pitch + 1;
            __syncthreads();
        }
    }
}

// ---- the pass path's second kernel: PNG.Image.assign from the rows unfilter_pass_kernel reconstructed in place ----
constexpr int INTERLEAVE_THREADS = 256;   // one aligned 16-byte chunk of storage per thread and block

// Every byte of an image's storage, in output order: a block writes 4 KiB that are contiguous in memory, a thread one
// aligned 16-byte chunk of it with a single store, so that every store fills whole 32-byte sectors.  A pixel takes its
// sample from its pass row (Adam7 origin and step per c_adam7; a 1/2/4-bit sample MSB-first, one byte per pixel), or
// zero where that row was not reconstructed: storage starts out zeroed in the reference (PNG.Image.swift:84).  Rows
// per pass follow wave_rows: the stream up to the first incomplete row, none after an inflate error.
__global__ void __launch_bounds__(INTERLEAVE_THREADS) unfilter_interleave_kernel(const InterleaveJob* jobs, uint32_t count,
                                                                                 uint64_t blocks)
{
    __shared__ const uint8_t* s_line[7];   // pixel bytes of the pass's row 0
    __shared__ uint64_t       s_stride[7]; // pitch + 1
    __shared__ uint64_t       s_rows[7];   // rows reconstructed
    for (uint64_t b = blockIdx.x; b < blocks; b += gridDim.x) {
        uint32_t lo = 0, hi = count;   // image owning block b: last index with block_base <= b
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (jobs[mid].block_base <= b) lo = mid;
            else hi = mid;
        }
        const InterleaveJob job = jobs[lo];
        __syncthreads();   // the previous block's threads are done with the pass table
        if (threadIdx.x < 7) {
            const int      z      = threadIdx.x;
            const Pass     ps     = stream_pass(z, job.width, job.height, job.volume, job.interlaced);
            const uint64_t off    = stream_pass_offset(z, job.width, job.height, job.volume, job.interlaced);
            const uint64_t usable = usable_bytes(job.inflated, job.filtered_len);
            const uint64_t rows   = usable > off ? (usable - off) / (ps.pitch + 1) : 0;
            s_line[z]   = job.filtered + off + 1;
            s_stride[z] = ps.pitch + 1;
            s_rows[z]   = rows < ps.height ? rows : ps.height;
        }
        __syncthreads();
        const uint32_t bpp   = job.bpp;
        const uint32_t lper  = job.depth == 1 ? 3 : job.depth == 2 ? 2 : 1;
        const uint64_t bytes = (uint64_t)job.width * job.height * bpp;
        const uint32_t mis   = (uint32_t)((uintptr_t)job.pixels & 15);
        // chunk k of the image covers storage bytes [16 k - mis, 16 k - mis + 16)
        const uint64_t k     = (b - job.block_base) * INTERLEAVE_THREADS + threadIdx.x;
        const int64_t  first = (int64_t)(16 * k) - mis;
        if (first >= (int64_t)bytes) continue;
        const uint64_t s  = first < 0 ? 0 : (uint64_t)first;
        const uint64_t e  = min((uint64_t)(first + 16), bytes);
        const uint64_t px = s / bpp;
        uint32_t       c  = (uint32_t)(s - px * bpp);
        uint64_t       y  = px / job.width;
        uint32_t       x  = (uint32_t)(px - y * job.width);
        uint32_t       w0 = 0, w1 = 0, w2 = 0, w3 = 0;
        for (uint64_t at = s; at < e; ++at) {
            int z = 0;   // Adam7 pass of pixel (x, y)
            if (job.interlaced)
                z = (y & 1) ? 6 : (x & 1) ? 5 : (y & 2) ? 4 : (x & 2) ? 3 : (y & 4) ? 2 : (x & 4) ? 1 : 0;
            const int      ex = job.interlaced ? c_adam7.p[z][2] : 0, ey = job.interlaced ? c_adam7.p[z][3] : 0;
            const uint64_t r  = y >> ey;   // (y - origin) >> step: the origin's bits sit below the step
            const uint64_t i  = x >> ex;
            uint32_t       v  = 0;
            if (r < s_rows[z]) {
                const uint8_t* line = s_line[z] + r * s_stride[z];
                if (job.depth < 8) {   // 1, 2 or 4 bits: 8 >> lper samples a byte
                    const uint32_t sh = ((~(uint32_t)i) & ((1u << lper) - 1)) * job.depth;
                    v = (line[i >> lper] >> sh) & ((1u << job.depth) - 1);
                } else {
                    v = line[i * bpp + c];
                }
            }
            const uint32_t slot = (uint32_t)(at - (uint64_t)first), sv = v << (8 * (slot & 3));
            w0 |= slot < 4 ? sv : 0u;   // selects, not w[slot >> 2]: a dynamically indexed array goes to local memory
            w1 |= slot >> 2 == 1 ? sv : 0u;
            w2 |= slot >> 2 == 2 ? sv : 0u;
            w3 |= slot >= 12 ? sv : 0u;
            if (++c == bpp) {
                c = 0;
                if (++x == job.width) {
                    x = 0;
                    ++y;
                }
            }
        }
        uint8_t* dst = job.pixels + (int64_t)first;   // aligned: 16 k - mis bytes past the start of the storage
        if (first >= 0 && e - s == 16) {
            *(uint4*)dst = make_uint4(w0, w1, w2, w3);
        } else {   // the image's first or last chunk
            for (uint64_t at = s; at < e; ++at) {
                const uint32_t slot = (uint32_t)(at - (uint64_t)first);
                const uint32_t word = slot < 4 ? w0 : slot < 8 ? w1 : slot < 12 ? w2 : w3;
                job.pixels[at] = (uint8_t)(word >> (8 * (slot & 3)));
            }
        }
    }
}

// ---- host planning of the wavefront and the pass path ----

// The wavefront's ticket order over `jobs` (ImageJob or PassJob, `height` rows each).  Tickets go out band level by band
// level (see WaveParams): jobs sorted by band count, descending; level_start[b] = tickets in front of level b.  (Jobs of
// more than 4096 bands -- 131072 rows -- keep the job-major order and leave level_start empty.)  band_base[i] = the
// first band of job i.  Returns the number of bands.
template <typename Job>
uint64_t plan_bands(std::vector<Job>& jobs, std::vector<uint32_t>& band_base, std::vector<uint32_t>& level_start)
{
    auto nb = [&](const Job& j) { return (j.height + 31) / 32; };
    level_start.clear();
    std::vector<uint32_t> idx(jobs.size());
    for (size_t i = 0; i < idx.size(); ++i) idx[i] = (uint32_t)i;
    std::stable_sort(idx.begin(), idx.end(), [&](uint32_t a, uint32_t b) { return nb(jobs[a]) > nb(jobs[b]); });
    const uint32_t maxb = jobs.empty() ? 0 : nb(jobs[idx[0]]);
    if (!jobs.empty() && maxb <= 4096) {
        std::vector<Job> sorted(jobs.size());
        for (size_t i = 0; i < idx.size(); ++i) sorted[i] = jobs[idx[i]];
        jobs.swap(sorted);
        level_start.assign(maxb + 1, 0);
        size_t alive = jobs.size();          // jobs with more than b bands: a prefix of the sorted list
        for (uint32_t b = 0; b < maxb; ++b) {
            while (alive && nb(jobs[alive - 1]) <= b) --alive;
            level_start[b + 1] = level_start[b] + (uint32_t)alive;
        }
    }
    band_base.assign(jobs.size() + 1, 0);
    uint64_t bands = 0;
    for (size_t i = 0; i < jobs.size(); ++i) {
        band_base[i] = (uint32_t)std::min<uint64_t>(bands, UINT32_MAX);
        bands += nb(jobs[i]);
    }
    band_base[jobs.size()] = (uint32_t)std::min<uint64_t>(bands, UINT32_MAX);
    return bands;
}

// The pass path's work for one image: a PassJob per non-empty pass, reconstructed in place in `image.filtered`, then
// the image itself for unfilter_interleave_kernel, its blocks numbered from `blocks` on (advanced past them).
inline void plan_passes(InterleaveJob image, std::vector<PassJob>& passes, std::vector<InterleaveJob>& images, uint64_t& blocks)
{
    for (int z = 0; z < 7; ++z) {
        const Pass ps = stream_pass(z, image.width, image.height, image.volume, image.interlaced);
        if (ps.height == 0) continue;
        const uint64_t off = stream_pass_offset(z, image.width, image.height, image.volume, image.interlaced);
        passes.push_back({image.filtered + off, image.inflated, image.filtered_len, off, (uint32_t)ps.height,
                          (uint32_t)ps.pitch, image.bpp});
    }
    image.block_base = blocks;
    images.push_back(image);
    const uint64_t chunks = (15 + (uint64_t)image.width * image.height * image.bpp + 15) / 16;   // any misalignment of the pixels
    blocks += (chunks + INTERLEAVE_THREADS - 1) / INTERLEAVE_THREADS;
}

}  // namespace pngb200
