// filter.cuh -- encode-side stage 1: PNG.Image.collect + PNG.Encoder.filter for every row.
//
// Replaces PNG.Encoder.filter / score (Sources/PNG/Encoding/PNG.Encoder.swift:132-204,230-234)
// and the gather of PNG.Image.collect (Sources/PNG/PNG.Image.swift:431-544).  All five candidate
// rows are functions of the UNFILTERED current and previous rows only, so every row of every
// image is independent: one warp per row computes the five sum|int8| scores in a single pass
// (warp-shuffle reduction), picks the first minimum in the order None, Sub, Up, Average, Paeth
// (strict <), and writes the winning candidate behind its filter-type byte.
#pragma once

#include "common.cuh"
#include "unfilter.cuh"

namespace pngb200 {

struct FilterJob {
    const uint8_t* pixels;    // PNG.Image.storage
    uint8_t*       filtered;  // out
    uint32_t       width, height;
    uint8_t        volume, depth, interlaced, bpp;
};

constexpr int      FILTER_WARPS = 8;
constexpr uint32_t FILTER_SLICE = 1u << 29;   // bytes of a row a warp scores in 32-bit lane sums (see filter_rows_kernel)

inline uint64_t filter_rows(uint32_t w, uint32_t h, int interlaced)
{
    uint64_t rows = 0;
    for (int z = 0; z < 7; ++z) rows += stream_pass(z, w, h, 1, interlaced).height;
    return rows;
}

// a scanline of one (sub)image, addressed bytewise as PNG.Image.collect would have packed it
struct RowView {
    const uint8_t* storage;
    uint32_t       width;     // full image width
    uint32_t       oy;        // storage row
    uint32_t       bx, ex;    // first column, log2 column stride
    uint32_t       sw;        // pixels in this scanline
    uint32_t       depth, bpp;
    bool           valid;     // false: the all-zero reference row above the first row of a pass

    __device__ __forceinline__ uint32_t byte(uint32_t i) const
    {
        if (!valid) return 0;
        if (depth >= 8) {
            uint32_t px = i / bpp, c = i - px * bpp;
            return storage[((uint64_t)oy * width + bx + ((uint64_t)px << ex)) * bpp + c];
        }
        uint32_t per = 8 / depth, mask = (1u << depth) - 1, v = 0;
        for (uint32_t k = 0; k < per; ++k) {
            uint32_t px = i * per + k;
            if (px < sw) {
                uint32_t s = storage[(uint64_t)oy * width + bx + ((uint64_t)px << ex)] & mask;
                v |= s << (((~px) & (per - 1)) * depth);
            }
        }
        return v;
    }
};

__device__ __forceinline__ uint32_t abs_i8(uint32_t b) { return b & 0x80 ? 256 - b : b; }

// Where stream scanline r of an image lies: its pass, its row y in that pass and its offset in the filtered stream
// (only an interlaced image walks its passes: walking them for every image cost filter_batch 1 % on an H100 80GB HBM3
// at 700 W, 8K and 512x512 RGBA8 alike)
__device__ __forceinline__ Pass filter_locate(uint32_t width, uint32_t height, uint32_t volume, bool interlaced, uint32_t r,
                                              uint32_t* y, uint64_t* out_off)
{
    *y = r;
    *out_off = 0;
    Pass ps = stream_pass(0, width, height, volume, false);
    if (interlaced) {
        for (int z = 0; z < 7; ++z) {
            ps = stream_pass(z, width, height, volume, true);
            if (*y < ps.height) break;
            *y -= (uint32_t)ps.height;
            *out_off += ps.height * (ps.pitch + 1);
        }
    }
    *out_off += (uint64_t)*y * (ps.pitch + 1);
    return ps;
}

// PNG.Encoder.filter of one scanline by the whole warp: scores the five candidates of `cur` against `prev` (filter
// delay d) and writes the winner behind its filter-type byte at out[0 .. pitch].
__device__ __forceinline__ void filter_scanline(const RowView& cur, const RowView& prev, uint32_t pitch, uint32_t d,
                                                uint8_t* out, unsigned lane)
{
    // A row scores up to 128 * pitch, past 2^32 from pitch 2^25 on (the reference sums in Swift Int): the scores are
    // 64-bit.  Each lane sums a slice of FILTER_SLICE bytes in 32 bits (at most FILTER_SLICE / 32 * 128 = 2^31) and
    // folds it into its 64-bit totals; slice offsets also keep the byte index from wrapping on a 4 GiB row.
    uint64_t t0 = 0, t1 = 0, t2 = 0, t3 = 0, t4 = 0;
    for (uint64_t base = 0; base < pitch; base += FILTER_SLICE) {
        const uint32_t n = (uint32_t)min((uint64_t)FILTER_SLICE, pitch - base);
        uint32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0;
        for (uint32_t k = lane; k < n; k += 32) {
            const uint32_t i = (uint32_t)base + k;
            uint32_t x = cur.byte(i), b = prev.byte(i);
            uint32_t a = i >= d ? cur.byte(i - d) : 0, c = i >= d ? prev.byte(i - d) : 0;
            s0 += abs_i8(x);
            s1 += abs_i8((x - a) & 0xff);
            s2 += abs_i8((x - b) & 0xff);
            s3 += abs_i8((x - ((a + b) >> 1)) & 0xff);
            s4 += abs_i8((x - paeth1(a, b, c)) & 0xff);
        }
        t0 += s0; t1 += s1; t2 += s2; t3 += s3; t4 += s4;
    }
    for (int o = 16; o; o >>= 1) {
        t0 += __shfl_xor_sync(0xffffffffu, t0, o);
        t1 += __shfl_xor_sync(0xffffffffu, t1, o);
        t2 += __shfl_xor_sync(0xffffffffu, t2, o);
        t3 += __shfl_xor_sync(0xffffffffu, t3, o);
        t4 += __shfl_xor_sync(0xffffffffu, t4, o);
    }
    uint32_t best = 0;
    uint64_t minimum = t0;
    if (t1 < minimum) { minimum = t1; best = 1; }
    if (t2 < minimum) { minimum = t2; best = 2; }
    if (t3 < minimum) { minimum = t3; best = 3; }
    if (t4 < minimum) { minimum = t4; best = 4; }
    if (lane == 0) out[0] = (uint8_t)best;
    for (uint64_t i = lane; i < pitch; i += 32) {
        uint32_t x = cur.byte(i), p = 0;
        if (best) {
            uint32_t b = prev.byte(i);
            uint32_t a = i >= d ? cur.byte(i - d) : 0, c = i >= d ? prev.byte(i - d) : 0;
            p = best == 1 ? a : best == 2 ? b : best == 3 ? (a + b) >> 1 : paeth1(a, b, c);
        }
        out[1 + i] = (uint8_t)(x - p);
    }
}

__global__ void __launch_bounds__(FILTER_WARPS * 32)
filter_rows_kernel(const FilterJob* jobs, const uint32_t* row_base, uint32_t njobs, uint32_t total_rows)
{
    const unsigned lane = lane_id();
    const uint32_t t    = blockIdx.x * FILTER_WARPS + (threadIdx.x >> 5);
    if (t >= total_rows) return;
    uint32_t lo = 0, hi = njobs;
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (row_base[mid] <= t) lo = mid;
        else hi = mid;
    }
    const FilterJob job = jobs[lo];
    uint32_t y;
    uint64_t out_off;
    const Pass ps = filter_locate(job.width, job.height, job.volume, job.interlaced, t - row_base[lo], &y, &out_off);
    RowView cur{job.pixels, job.width, ps.by + (y << ps.ey), ps.bx, ps.ex, (uint32_t)ps.width, job.depth, job.bpp, true};
    RowView prev = cur;
    prev.valid = y > 0;
    prev.oy = ps.by + ((y ? y - 1 : 0) << ps.ey);
    filter_scanline(cur, prev, (uint32_t)ps.pitch, job.bpp, job.filtered + out_off, lane);   // geometry() caps a pitch at 0xfffffff0
}

// ---- the online encoder (pngb200_png_encoder_push_batch): the scanlines a push completes, one warp each ----
//
// A push brings the next storage rows of an image; the scanlines it completes, in stream order, are filtered straight
// onto the end of the handle's deflator input.  A non-interlaced scanline y reads storage row y from the push (`rows`
// holds rows row0, row0 + 1, ...) and row y - 1 from the push or, for y == row0, from the handle's carried copy of the
// previous push's last row.  An Adam7 scanline reads both rows from the handle's copy of the whole storage (`rows` is
// then its row 0), since later passes reread rows that pass 0 used.
struct FilterResumeJob {
    const uint8_t* rows;
    const uint8_t* carried;    // non-interlaced: storage row row0 - 1
    uint8_t*       out;        // where scanline `first` goes
    uint64_t       out_off0;   // stream offset of scanline `first`
    uint32_t       width, height;
    uint32_t       first, row0;
    uint8_t        volume, depth, interlaced, bpp;
};

__global__ void __launch_bounds__(FILTER_WARPS * 32)
filter_resume_kernel(const FilterResumeJob* jobs, const uint32_t* line_base, uint32_t njobs, uint32_t total_lines)
{
    const unsigned lane = lane_id();
    const uint32_t t    = blockIdx.x * FILTER_WARPS + (threadIdx.x >> 5);
    if (t >= total_lines) return;
    uint32_t lo = 0, hi = njobs;
    while (hi - lo > 1) {
        uint32_t mid = (lo + hi) >> 1;
        if (line_base[mid] <= t) lo = mid;
        else hi = mid;
    }
    const FilterResumeJob job = jobs[lo];
    uint32_t y;
    uint64_t out_off;
    const Pass ps = filter_locate(job.width, job.height, job.volume, job.interlaced, job.first + (t - line_base[lo]), &y, &out_off);
    RowView cur{job.rows, job.width, ps.by + (y << ps.ey), ps.bx, ps.ex, (uint32_t)ps.width, job.depth, job.bpp, true};
    RowView prev = cur;
    prev.valid = y > 0;
    if (job.interlaced) {
        prev.oy = ps.by + ((y ? y - 1 : 0) << ps.ey);
    } else {
        cur.oy = y - job.row0;
        if (y > job.row0) prev.oy = y - 1 - job.row0;
        else prev.storage = job.carried, prev.oy = 0;
    }
    filter_scanline(cur, prev, (uint32_t)ps.pitch, job.bpp, job.out + (out_off - job.out_off0), lane);
}

}  // namespace pngb200
