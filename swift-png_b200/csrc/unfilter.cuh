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
//   shared-memory ring in 16-byte chunks (see WAVE_DEPTH) and writes 16-byte stores.
//
// unfilter_generic_kernel: every other format (Adam7, 1/2/4-bit samples); one CTA per image.
#pragma once

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

struct WaveParams {
    const ImageJob* jobs;
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
// has just left.  Reconstructed chunks are stored straight from registers.  The rings are the CTA's whole shared
// memory (WAVE_SMEM, 32 KiB); a deeper ring, or a second one for the output or for lane 0's row above, costs resident
// warps, and the kernel's throughput follows resident warps, not lookahead per warp (DESIGN §4.3).
constexpr int      WAVE_WARPS   = 4;    // warps per CTA
constexpr int      WAVE_DEPTH   = 16;   // ring slots per lane
constexpr int      WAVE_PUBLISH = 8;    // publish progress every this many chunks
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

template <int BPP>
__device__ void wave_band(const ImageJob& job, uint32_t band, uint32_t* prog_prev, uint32_t* prog_mine, uint4 (*ring)[32],
                          unsigned long long* hist)
{
    const unsigned lane   = lane_id();
    const uint32_t y      = band * 32 + lane;
    const uint32_t pitch  = job.pitch;
    const uint64_t rows   = usable_bytes(job.inflated, job.filtered_len) / (pitch + 1);
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
    const int      nq    = (int)((m + pitch + 15) >> 4);  // aligned chunks that hold row bytes
    uint8_t*       out   = job.pixels + (uint64_t)(active ? y : 0) * pitch;
    const uint8_t* above = band == 0 ? nullptr : job.pixels + (uint64_t)(band * 32 - 1) * pitch;
    const bool     publish = lane == 31 && prog_mine != nullptr;
    // rows the stream did not deliver (a complete zlib stream that is shorter than the image is not an error in
    // the reference: the rows simply stay as PNG.Image.storage was initialised, zero -- PNG.Image.swift:84)
    if (!active && y < job.height) {
        uint8_t* z = job.pixels + (uint64_t)y * pitch;
        for (uint32_t k = 0; k < pitch; ++k) z[k] = 0;
    }

    uint4    qcur  = make_uint4(0, 0, 0, 0);
    uint4    mine  = make_uint4(0, 0, 0, 0);  // my last reconstructed chunk
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
            store16_partial(out + 16 * (uint64_t)j, o, (int)pitch - 16 * j);
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

__global__ void __launch_bounds__(WAVE_WARPS * 32) unfilter_wave_kernel(WaveParams p)
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
        const ImageJob job   = p.jobs[lo];
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

// ---- generic path: Adam7 and sub-byte depths.  One CTA per image; defilters in place. ----
__constant__ int c_adam7[7][4] = {{0, 0, 3, 3}, {4, 0, 3, 3}, {0, 4, 2, 3}, {2, 0, 2, 2},
                                  {0, 2, 1, 2}, {1, 0, 1, 1}, {0, 1, 0, 1}};

struct GenericJob {
    uint8_t*            filtered;  // mutable: rows are reconstructed in place
    uint8_t*            pixels;
    const StreamResult* inflated;
    uint64_t            filtered_len;
    uint32_t width, height;
    uint8_t  volume, depth, interlaced, bpp;
};

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
    const int npass = job.interlaced ? 7 : 1;
    for (int z = 0; z < npass; ++z) {
        int      bx = 0, by = 0, ex = 0, ey = 0;
        uint32_t sw = job.width, shh = job.height;
        if (job.interlaced) {
            bx = c_adam7[z][0]; by = c_adam7[z][1]; ex = c_adam7[z][2]; ey = c_adam7[z][3];
            sw  = (job.width + (1u << ex) - bx - 1) >> ex;
            shh = (job.height + (1u << ey) - by - 1) >> ey;
            if (sw == 0 || shh == 0) continue;
        }
        const uint32_t pitch = (sw * job.volume + 7) >> 3;
        uint8_t*       last  = nullptr;
        for (uint32_t y = 0; y < shh; ++y) {
            if (at + pitch + 1 > end) return;  // inflator.pull(pitch + 1) == nil
            uint8_t*      line = at + 1;
            const uint8_t type = at[0];
            if (type == 2) {
                if (last)
                    for (uint32_t i = tid; i < pitch; i += nt) line[i] = (uint8_t)(line[i] + last[i]);
            } else if (type == 1 || type == 3 || type == 4) {
                if ((uint32_t)tid < bpp) {  // channels are independent chains
                    for (uint32_t i = tid; i < pitch; i += bpp) {
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
            const uint32_t oy = by + (y << ey);
            if (job.depth < 8) {
                const uint32_t per = 8 / job.depth, mask = (1u << job.depth) - 1;
                for (uint32_t i = tid; i < sw; i += nt) {
                    uint32_t sh = ((~i) & (per - 1)) * job.depth;
                    job.pixels[(uint64_t)oy * job.width + bx + ((uint64_t)i << ex)] =
                        (uint8_t)((line[i / per] >> sh) & mask);
                }
            } else {
                for (uint32_t k = tid; k < sw * bpp; k += nt) {
                    uint32_t i = k / bpp, c = k - i * bpp;
                    job.pixels[((uint64_t)oy * job.width + bx + ((uint64_t)i << ex)) * bpp + c] = line[k];
                }
            }
            last = line;
            at += pitch + 1;
            __syncthreads();
        }
    }
}

}  // namespace pngb200
