// color.cuh -- colour targets on the device: PNG.Image.storage <-> [PNG.RGBA<T>] / [PNG.VA<T>]
// (SURVEY.md section 8f row N1: the unpack that sits inside the reference's own timed decode loop,
// Benchmarks/Decompression/Swift/Main.swift:105-106, and its inverse used by PNG.Image.init(packing:)).
//
// The reference expresses these as generic closures over convolve / deconvolve
// (Sources/PNG/PNG.swift:149-1285, ColorTargets/PNG.RGBA.swift:262-478, ColorTargets/PNG.VA.swift,
// ColorTargets/PNG.Color.swift).  Here each is one elementwise, HBM-bound map: one thread per pixel
// per iteration, the format switch uniform across the CTA, palettes staged in shared memory.
// Algorithmic bytes per pixel: storage bytes read + target bytes written (or the reverse).
#pragma once

#include "common.cuh"

namespace pngb200 {

constexpr int COLOR_THREADS = 256;
constexpr int COLOR_TILE    = 8 * COLOR_THREADS;  // pixels per CTA iteration

struct ColorJob {
    uint8_t*  storage;      // PNG.Image.storage (unpack: read, pack: written)
    uint8_t*  pixels;       // target array, native-endian T components
    uint64_t  count;        // pixels
    uint32_t  palette_off;  // first entry of this job's palette in ColorParams::palettes
    uint16_t  palette_count;
    uint16_t  key[3];
    uint8_t   color, depth, bgr, has_key;
    int32_t   status;
};

struct ColorParams {
    ColorJob*       jobs;
    const uint32_t* palettes;  // r | g << 8 | b << 16 | a << 24
    uint32_t        count;
    int             target;      // PNGB200_TARGET_*
    int             alpha_mode;  // PNGB200_ALPHA_*
};

__device__ __forceinline__ int color_channels(int color) { return color == 0 || color == 3 ? 1 : color == 2 ? 3 : color == 4 ? 2 : 4; }

// PNG.quantum + the transform closures of convolve(_:of:depth:kernel:) (PNG.swift:255-261, 494-523)
__device__ __forceinline__ uint32_t color_widen(uint32_t v, int depth, int tbits)
{
    if (tbits == depth) return v;
    if (tbits > depth) return v * (((1u << tbits) - 1u) / ((1u << depth) - 1u));
    return v >> (depth - tbits);
}
// the transform closures of deconvolve(_:as:depth:kernel:) (PNG.swift:1063-1095)
__device__ __forceinline__ uint32_t color_narrow(uint32_t v, int tbits, int depth)
{
    if (tbits == depth) return v;
    if (tbits < depth) return v * (((1u << depth) - 1u) / ((1u << tbits) - 1u));
    return v >> (tbits - depth);
}
// PNG.premultiply (PNG.swift:54-66)
template <int BITS> __device__ __forceinline__ uint32_t color_premultiply(uint32_t c, uint32_t a)
{
    constexpr uint32_t MAX = (1u << BITS) - 1u;
    return (c * a + (MAX >> 1)) / MAX;
}
// PNG.straighten (PNG.swift:100-120); saturates where the reference's dividingFullWidth traps
template <int BITS> __device__ __forceinline__ uint32_t color_straighten(uint32_t p, uint32_t a)
{
    constexpr uint32_t MAX = (1u << BITS) - 1u;
    if (a == 0) return p;
    return min((MAX * p + (a >> 1)) / a, MAX);
}

template <int TBITS>
__device__ __forceinline__ void color_alpha(uint32_t& r, uint32_t& g, uint32_t& b, uint32_t& a, int mode)
{
    if (mode == PNGB200_ALPHA_PREMULTIPLIED) {
        r = color_premultiply<TBITS>(r, a), g = color_premultiply<TBITS>(g, a), b = color_premultiply<TBITS>(b, a);
    } else if (mode == PNGB200_ALPHA_STRAIGHTENED) {
        r = color_straighten<TBITS>(r, a), g = color_straighten<TBITS>(g, a), b = color_straighten<TBITS>(b, a);
    } else if (TBITS == 16 && (mode == PNGB200_ALPHA_PREMULTIPLIED_AS8 || mode == PNGB200_ALPHA_STRAIGHTENED_AS8)) {
        // premultiplied(as: UInt8.self) / straightened(as: UInt8.self) (PNG.RGBA.swift:141-155, 187-201)
        const uint32_t a8 = a >> 8;
        if (mode == PNGB200_ALPHA_PREMULTIPLIED_AS8) {
            r = color_premultiply<8>(r >> 8, a8) * 257u, g = color_premultiply<8>(g >> 8, a8) * 257u;
            b = color_premultiply<8>(b >> 8, a8) * 257u;
        } else {
            r = color_straighten<8>(r >> 8, a8) * 257u, g = color_straighten<8>(g >> 8, a8) * 257u;
            b = color_straighten<8>(b >> 8, a8) * 257u;
        }
        a = a8 * 257u;
    }
}

// the bytes of pixel i (bpp = 1..8), first sample in the low bits
__device__ __forceinline__ uint64_t color_load_pixel(const uint8_t* storage, uint64_t i, int bpp, bool aligned)
{
    const uint8_t* p = storage + i * bpp;
    if (aligned) {
        if (bpp == 8) { uint2 v = *(const uint2*)p; return (uint64_t)v.y << 32 | v.x; }
        if (bpp == 4) return *(const uint32_t*)p;
        if (bpp == 2) return *(const uint16_t*)p;
    }
    uint64_t v = 0;
    for (int k = 0; k < bpp; ++k) v |= (uint64_t)p[k] << (8 * k);
    return v;
}
__device__ __forceinline__ void color_store_pixel(uint8_t* storage, uint64_t i, int bpp, bool aligned, uint64_t v)
{
    uint8_t* p = storage + i * bpp;
    if (aligned) {
        if (bpp == 8) { *(uint2*)p = make_uint2((uint32_t)v, (uint32_t)(v >> 32)); return; }
        if (bpp == 4) { *(uint32_t*)p = (uint32_t)v; return; }
        if (bpp == 2) { *(uint16_t*)p = (uint16_t)v; return; }
    }
    for (int k = 0; k < bpp; ++k) p[k] = (uint8_t)(v >> (8 * k));
}

template <int TBITS, bool VA>
__device__ void unpack_image(const ColorJob& job, ColorJob* slot, const uint32_t* palette, int alpha_mode)
{
    const int  ch      = color_channels(job.color);
    const int  bpp     = ch * (job.depth == 16 ? 2 : 1);
    const bool wide    = job.depth == 16;
    const bool aligned = (((uintptr_t)job.storage) & 7) == 0;
    constexpr uint32_t TMAX = (1u << TBITS) - 1u;
    for (uint64_t base = (uint64_t)blockIdx.x * COLOR_TILE; base < job.count; base += (uint64_t)gridDim.x * COLOR_TILE) {
#pragma unroll 2
        for (uint64_t i = base + threadIdx.x; i < min(base + COLOR_TILE, job.count); i += COLOR_THREADS) {
            const uint64_t bits = color_load_pixel(job.storage, i, bpp, aligned);
            uint32_t raw[4];
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                // A(bigEndian:) (PNG.swift:152-204)
                raw[c] = wide ? __byte_perm((uint32_t)(bits >> (16 * c)), 0, 0x4401) & 0xffffu
                              : (uint32_t)(bits >> (8 * c)) & 0xffu;
            }
            uint32_t r, g, b, a;
            if (job.color == 3) {
                if (raw[0] >= job.palette_count) {  // palette[i] traps in the reference
                    atomicMin(&slot->status, (int32_t)PNGB200_ERR_PNG_PALETTE_INDEX);
                    continue;
                }
                const uint32_t e = palette[raw[0]];
                r = color_widen(e & 0xff, 8, TBITS), g = color_widen((e >> 8) & 0xff, 8, TBITS);
                b = color_widen((e >> 16) & 0xff, 8, TBITS), a = color_widen(e >> 24, 8, TBITS);
            } else if (job.color == 0 || job.color == 4) {
                r = g = b = color_widen(raw[0], job.depth, TBITS);
                a = job.color == 4 ? color_widen(raw[1], job.depth, TBITS)
                                   : (job.has_key && raw[0] == job.key[0]) ? 0u : TMAX;
            } else {
                const uint32_t c0 = color_widen(raw[0], job.depth, TBITS), c1 = color_widen(raw[1], job.depth, TBITS),
                               c2 = color_widen(raw[2], job.depth, TBITS);
                r = job.bgr ? c2 : c0, g = c1, b = job.bgr ? c0 : c2;
                a = job.color == 6 ? color_widen(raw[3], job.depth, TBITS)
                                   : (job.has_key && raw[0] == job.key[0] && raw[1] == job.key[1] && raw[2] == job.key[2]) ? 0u : TMAX;
            }
            color_alpha<TBITS>(r, g, b, a, alpha_mode);
            if (VA) {
                if (TBITS == 8) ((uint16_t*)job.pixels)[i] = (uint16_t)(r | a << 8);
                else ((uint32_t*)job.pixels)[i] = r | a << 16;
            } else {
                if (TBITS == 8) ((uint32_t*)job.pixels)[i] = r | g << 8 | b << 16 | a << 24;
                else ((uint2*)job.pixels)[i] = make_uint2(r | g << 16, b | a << 16);
            }
        }
    }
}

__global__ void __launch_bounds__(COLOR_THREADS) unpack_kernel(ColorParams p)
{
    __shared__ uint32_t palette[256];
    for (uint32_t j = blockIdx.y; j < p.count; j += gridDim.y) {
        const ColorJob job = p.jobs[j];
        if (job.color == 3) {
            __syncthreads();
            if (threadIdx.x < job.palette_count) palette[threadIdx.x] = p.palettes[job.palette_off + threadIdx.x];
            __syncthreads();
        }
        switch (p.target) {
        case PNGB200_TARGET_RGBA8:  unpack_image<8, false>(job, p.jobs + j, palette, p.alpha_mode); break;
        case PNGB200_TARGET_RGBA16: unpack_image<16, false>(job, p.jobs + j, palette, p.alpha_mode); break;
        case PNGB200_TARGET_VA8:    unpack_image<8, true>(job, p.jobs + j, palette, p.alpha_mode); break;
        default:                    unpack_image<16, true>(job, p.jobs + j, palette, p.alpha_mode); break;
        }
    }
}

template <int TBITS, bool VA>
__device__ void pack_image(const ColorJob& job, const uint32_t* palette)
{
    const int  ch      = color_channels(job.color);
    const int  bpp     = ch * (job.depth == 16 ? 2 : 1);
    const bool wide    = job.depth == 16;
    const bool aligned = (((uintptr_t)job.storage) & 7) == 0;
    for (uint64_t base = (uint64_t)blockIdx.x * COLOR_TILE; base < job.count; base += (uint64_t)gridDim.x * COLOR_TILE) {
#pragma unroll 2
        for (uint64_t i = base + threadIdx.x; i < min(base + COLOR_TILE, job.count); i += COLOR_THREADS) {
            uint32_t r, g, b, a;
            if (VA) {
                if (TBITS == 8) { uint32_t v = ((const uint16_t*)job.pixels)[i]; r = v & 0xff, a = v >> 8; }
                else { uint32_t v = ((const uint32_t*)job.pixels)[i]; r = v & 0xffff, a = v >> 16; }
                g = b = r;
            } else {
                if (TBITS == 8) { uint32_t v = ((const uint32_t*)job.pixels)[i]; r = v & 0xff, g = (v >> 8) & 0xff, b = (v >> 16) & 0xff, a = v >> 24; }
                else { uint2 v = ((const uint2*)job.pixels)[i]; r = v.x & 0xffff, g = v.x >> 16, b = v.y & 0xffff, a = v.y >> 16; }
            }
            if (job.color == 3) {
                // default indexer (PNG.Color.swift): palette -> index hash table, missing colours -> 0
                const uint32_t q = color_narrow(r, TBITS, 8) | color_narrow(g, TBITS, 8) << 8 |
                                   color_narrow(b, TBITS, 8) << 16 | color_narrow(a, TBITS, 8) << 24;
                uint32_t idx = 0;
                for (uint32_t k = 0; k < job.palette_count; ++k)
                    if (palette[k] == q) { idx = k; break; }
                job.storage[i] = (uint8_t)idx;
                continue;
            }
            uint32_t s[4] = {0, 0, 0, 0};
            if (job.color == 0) s[0] = r;
            else if (job.color == 4) s[0] = r, s[1] = a;
            else s[0] = job.bgr ? b : r, s[1] = g, s[2] = job.bgr ? r : b, s[3] = a;
            uint64_t bits = 0;
#pragma unroll
            for (int c = 0; c < 4; ++c) {
                const uint32_t v = color_narrow(s[c], TBITS, job.depth);
                if (c < ch) bits |= wide ? (uint64_t)(__byte_perm(v, 0, 0x4401) & 0xffffu) << (16 * c) : (uint64_t)(v & 0xffu) << (8 * c);
            }
            color_store_pixel(job.storage, i, bpp, aligned, bits);
        }
    }
}

__global__ void __launch_bounds__(COLOR_THREADS) pack_kernel(ColorParams p)
{
    __shared__ uint32_t palette[256];
    for (uint32_t j = blockIdx.y; j < p.count; j += gridDim.y) {
        const ColorJob job = p.jobs[j];
        if (job.color == 3) {
            __syncthreads();
            if (threadIdx.x < job.palette_count) palette[threadIdx.x] = p.palettes[job.palette_off + threadIdx.x];
            __syncthreads();
        }
        switch (p.target) {
        case PNGB200_TARGET_RGBA8:  pack_image<8, false>(job, palette); break;
        case PNGB200_TARGET_RGBA16: pack_image<16, false>(job, palette); break;
        case PNGB200_TARGET_VA8:    pack_image<8, true>(job, palette); break;
        default:                    pack_image<16, true>(job, palette); break;
        }
    }
}

// ---- RGBA<UInt32 / UInt64>, VA<UInt32 / UInt64> and the scalar targets [UInt8 ... UInt64] ----
// image.unpack(as: T.self) / PNG.Image(packing: [T]) (Sources/PNG/PNG.Image.swift:681-833, 1126-1145)
// and the wide specialisations of PNG.RGBA / PNG.VA (PNG.RGBA.swift:253-257).  Each (T, shape) pair
// is its own kernel, so the 64-bit arithmetic here never reaches unpack_kernel / pack_kernel.
// Components are carried as uint64_t; stores and loads are 16 bytes (RGBA32, VA64, two for RGBA64),
// 8 bytes (VA32, V64), 4 bytes (V32) or, for V8 / V16, one 32-bit word of 4 / 2 adjacent pixels.
enum ColorShape { COLOR_RGBA, COLOR_VA, COLOR_V };

template <int BITS> __host__ __device__ constexpr uint64_t color_max() { return ~0ull >> (64 - BITS); }  // no 1 << 64

// PNG.premultiply (PNG.swift:54-66) at any width up to 64 bits: (c * a + T.max >> 1) / T.max
template <int BITS> __device__ __forceinline__ uint64_t color_premultiply_wide(uint64_t c, uint64_t a)
{
    constexpr uint64_t MAX = color_max<BITS>();
    if constexpr (BITS <= 32) {
        return (c * a + (MAX >> 1)) / MAX;
    } else {
        // x / (2^64 - 1) without a 128-bit divide: x = hi * 2^64 + lo = hi * MAX + (hi + lo),
        // and hi + lo <= 2 * MAX, so at most two corrections
        const unsigned __int128 x = (unsigned __int128)c * a + (MAX >> 1);
        const uint64_t hi = (uint64_t)(x >> 64);
        unsigned __int128 s = (unsigned __int128)hi + (uint64_t)x;
        uint64_t q = hi;
        if (s >= MAX) s -= MAX, ++q;
        if (s >= MAX) ++q;
        return q;
    }
}
// PNG.straighten (PNG.swift:100-120) at any width up to 64 bits; saturates where the reference traps
template <int BITS> __device__ __forceinline__ uint64_t color_straighten_wide(uint64_t p, uint64_t a)
{
    constexpr uint64_t MAX = color_max<BITS>();
    if (a == 0) return p;
    if constexpr (BITS <= 32) {
        const uint64_t q = (MAX * p + (a >> 1)) / a;
        return q < MAX ? q : MAX;
    } else {
        if (p >= a) return MAX;  // the quotient is at least MAX
        return (uint64_t)(((unsigned __int128)MAX * p + (a >> 1)) / a);
    }
}
// premultiplied(as: U.self) / straightened(as: U.self) of a T color, U narrower than T
// (PNG.RGBA.swift:146-206, PNG.VA.swift:79, 120): shift = T - U, q = T.max / (T.max >> shift)
template <int T, int U>
__device__ __forceinline__ void color_alpha_as(uint64_t& r, uint64_t& g, uint64_t& b, uint64_t& a, bool straighten)
{
    static_assert(T > U, "premultiplied(as:) needs a narrower type");
    constexpr int      SHIFT = T - U;
    constexpr uint64_t Q     = color_max<T>() / (color_max<T>() >> SHIFT);
    const uint64_t     au    = a >> SHIFT;
    if (straighten) {
        r = color_straighten_wide<U>(r >> SHIFT, au) * Q, g = color_straighten_wide<U>(g >> SHIFT, au) * Q;
        b = color_straighten_wide<U>(b >> SHIFT, au) * Q;
    } else {
        r = color_premultiply_wide<U>(r >> SHIFT, au) * Q, g = color_premultiply_wide<U>(g >> SHIFT, au) * Q;
        b = color_premultiply_wide<U>(b >> SHIFT, au) * Q;
    }
    a = au * Q;
}
template <int T>
__device__ __forceinline__ void color_alpha_wide(uint64_t& r, uint64_t& g, uint64_t& b, uint64_t& a, int mode)
{
    switch (mode) {
    case PNGB200_ALPHA_PREMULTIPLIED:
        r = color_premultiply_wide<T>(r, a), g = color_premultiply_wide<T>(g, a), b = color_premultiply_wide<T>(b, a);
        break;
    case PNGB200_ALPHA_STRAIGHTENED:
        r = color_straighten_wide<T>(r, a), g = color_straighten_wide<T>(g, a), b = color_straighten_wide<T>(b, a);
        break;
    case PNGB200_ALPHA_PREMULTIPLIED_AS8:  color_alpha_as<T, 8>(r, g, b, a, false); break;
    case PNGB200_ALPHA_STRAIGHTENED_AS8:   color_alpha_as<T, 8>(r, g, b, a, true); break;
    case PNGB200_ALPHA_PREMULTIPLIED_AS16: color_alpha_as<T, 16>(r, g, b, a, false); break;
    case PNGB200_ALPHA_STRAIGHTENED_AS16:  color_alpha_as<T, 16>(r, g, b, a, true); break;
    default:
        if constexpr (T > 32) {
            if (mode == PNGB200_ALPHA_PREMULTIPLIED_AS32) color_alpha_as<T, 32>(r, g, b, a, false);
            else if (mode == PNGB200_ALPHA_STRAIGHTENED_AS32) color_alpha_as<T, 32>(r, g, b, a, true);
        }
        break;
    }
}

template <int TBITS> struct ColorWord;
template <> struct ColorWord<8>  { using type = uint8_t; };
template <> struct ColorWord<16> { using type = uint16_t; };
template <> struct ColorWord<32> { using type = uint32_t; };
template <> struct ColorWord<64> { using type = uint64_t; };

// V8 / V16: pixels per 32-bit word; every other target: 1
template <int TBITS, int SHAPE> __host__ __device__ constexpr int color_group() { return SHAPE == COLOR_V && TBITS < 32 ? 32 / TBITS : 1; }

// Calls f(i) for every pixel index i of a scalar head / tail that a grouped target cannot cover with
// whole aligned words, and returns the number of leading pixels before the first aligned word.
template <int TBITS, int SHAPE, typename F>
__device__ __forceinline__ uint64_t color_edges(const ColorJob& job, uint64_t& groups, F f)
{
    constexpr int G = color_group<TBITS, SHAPE>();
    if (G == 1) { groups = job.count; return 0; }
    const uint64_t head = min((uint64_t)(((4u - ((uintptr_t)job.pixels & 3u)) & 3u) / (TBITS / 8)), job.count);
    groups = (job.count - head) / G;
    const uint64_t body_end = head + groups * G;
    if (blockIdx.x == 0 && threadIdx.x < head + (job.count - body_end))
        f(threadIdx.x < head ? (uint64_t)threadIdx.x : body_end + threadIdx.x - head);
    return head;
}

template <int TBITS, int SHAPE>
__device__ void unpack_wide_image(const ColorJob& job, ColorJob* slot, const uint32_t* palette, int alpha_mode)
{
    using T = typename ColorWord<TBITS>::type;
    constexpr int      G    = color_group<TBITS, SHAPE>();
    constexpr uint64_t TMAX = color_max<TBITS>();
    constexpr uint64_t Q8   = TMAX / 255u;  // palette entries are 8-bit
    const int  ch      = color_channels(job.color);
    const bool wide    = job.depth == 16;
    const int  bpp     = ch * (wide ? 2 : 1);
    const bool aligned = (((uintptr_t)job.storage) & 7) == 0;
    // PNG.quantum / the convolve transforms (PNG.swift:255-261, 494-523), hoisted per image
    const bool     up = TBITS >= job.depth;
    const uint64_t q  = up ? TMAX / (~0ull >> (64 - job.depth)) : 0;
    const int      sh = up ? 0 : job.depth - TBITS;
    auto widen = [&](uint32_t v) -> uint64_t { return up ? v * q : v >> sh; };
    // pixel i as (r, g, b, a) in T's range; false (and the job's status set) on a bad palette index
    auto fetch = [&](uint64_t i, uint64_t& r, uint64_t& g, uint64_t& b, uint64_t& a) -> bool {
        const uint64_t bits = color_load_pixel(job.storage, i, bpp, aligned);
        uint32_t raw[4];
#pragma unroll
        for (int c = 0; c < 4; ++c)
            raw[c] = wide ? __byte_perm((uint32_t)(bits >> (16 * c)), 0, 0x4401) & 0xffffu : (uint32_t)(bits >> (8 * c)) & 0xffu;
        if (job.color == 3) {
            if (raw[0] >= job.palette_count) {  // palette[i] traps in the reference
                atomicMin(&slot->status, (int32_t)PNGB200_ERR_PNG_PALETTE_INDEX);
                return false;
            }
            const uint32_t e = palette[raw[0]];
            r = (e & 0xff) * Q8, g = ((e >> 8) & 0xff) * Q8, b = ((e >> 16) & 0xff) * Q8, a = (e >> 24) * Q8;
        } else if (job.color == 0 || job.color == 4) {
            r = g = b = widen(raw[0]);
            a = job.color == 4 ? widen(raw[1]) : (job.has_key && raw[0] == job.key[0]) ? 0u : TMAX;
        } else {
            const uint64_t c0 = widen(raw[0]), c1 = widen(raw[1]), c2 = widen(raw[2]);
            r = job.bgr ? c2 : c0, g = c1, b = job.bgr ? c0 : c2;
            a = job.color == 6 ? widen(raw[3])
                               : (job.has_key && raw[0] == job.key[0] && raw[1] == job.key[1] && raw[2] == job.key[2]) ? 0u : TMAX;
        }
        if constexpr (SHAPE != COLOR_V) color_alpha_wide<TBITS>(r, g, b, a, alpha_mode);
        return true;
    };
    // the scalar target is the red sample (PNG.Image.swift:681-758): v, the v of va, r of rgb(a),
    // c.2 of bgr(a)8, palette[i].r -- which is what fetch returns in r, chroma key ignored
    auto put = [&](uint64_t i) {
        uint64_t r, g, b, a;
        if (!fetch(i, r, g, b, a)) return;
        if constexpr (SHAPE == COLOR_V) {
            ((T*)job.pixels)[i] = (T)r;
        } else if constexpr (SHAPE == COLOR_VA) {
            if constexpr (TBITS == 32) ((uint2*)job.pixels)[i] = make_uint2((uint32_t)r, (uint32_t)a);
            else ((ulonglong2*)job.pixels)[i] = make_ulonglong2(r, a);
        } else {
            if constexpr (TBITS == 32) ((uint4*)job.pixels)[i] = make_uint4((uint32_t)r, (uint32_t)g, (uint32_t)b, (uint32_t)a);
            else ((ulonglong2*)job.pixels)[2 * i] = make_ulonglong2(r, g), ((ulonglong2*)job.pixels)[2 * i + 1] = make_ulonglong2(b, a);
        }
    };
    uint64_t groups;
    const uint64_t head = color_edges<TBITS, SHAPE>(job, groups, put);
    constexpr uint64_t TILE = COLOR_TILE / G;
    for (uint64_t base = (uint64_t)blockIdx.x * TILE; base < groups; base += (uint64_t)gridDim.x * TILE) {
#pragma unroll 2
        for (uint64_t u = base + threadIdx.x; u < min(base + TILE, groups); u += COLOR_THREADS) {
            if constexpr (G == 1) {
                put(u);
            } else {
                uint32_t w = 0;
#pragma unroll
                for (int k = 0; k < G; ++k) {
                    uint64_t r, g, b, a;
                    if (fetch(head + u * G + k, r, g, b, a)) w |= (uint32_t)r << (TBITS * k);
                }
                ((uint32_t*)(job.pixels + head * (TBITS / 8)))[u] = w;
            }
        }
    }
}

template <int TBITS, int SHAPE>
__global__ void __launch_bounds__(COLOR_THREADS) unpack_wide_kernel(ColorParams p)
{
    __shared__ uint32_t palette[256];
    for (uint32_t j = blockIdx.y; j < p.count; j += gridDim.y) {
        const ColorJob job = p.jobs[j];
        if (job.color == 3) {
            __syncthreads();
            if (threadIdx.x < job.palette_count) palette[threadIdx.x] = p.palettes[job.palette_off + threadIdx.x];
            __syncthreads();
        }
        unpack_wide_image<TBITS, SHAPE>(job, p.jobs + j, palette, p.alpha_mode);
    }
}

template <int TBITS, int SHAPE>
__device__ void pack_wide_image(const ColorJob& job, const uint32_t* palette)
{
    using T = typename ColorWord<TBITS>::type;
    constexpr int      G    = color_group<TBITS, SHAPE>();
    constexpr uint64_t TMAX = color_max<TBITS>();
    const int  ch      = color_channels(job.color);
    const bool wide    = job.depth == 16;
    const int  bpp     = ch * (wide ? 2 : 1);
    const bool aligned = (((uintptr_t)job.storage) & 7) == 0;
    // the deconvolve transforms (PNG.swift:1063-1097), hoisted per image: T -> depth
    const bool     down = TBITS >= job.depth;
    const int      sh   = down ? TBITS - job.depth : 0;
    const uint32_t q    = down ? 0u : (uint32_t)((~0ull >> (64 - job.depth)) / TMAX);
    auto narrow = [&](uint64_t v) -> uint32_t { return down ? (uint32_t)(v >> sh) : (uint32_t)v * q; };
    // pixel i of storage from (r, g, b, a); the scalar target packs (v, v, v, T.max) (PNG.Image.swift:760-833)
    auto store = [&](uint64_t i, uint64_t r, uint64_t g, uint64_t b, uint64_t a) {
        if (job.color == 3) {
            // default indexer (PNG.Color.swift, PNG.Image.swift:1126-1145): first equal palette entry, else 0
            constexpr int S8 = TBITS - 8;
            const uint32_t key = (uint32_t)(r >> S8) | (uint32_t)(g >> S8) << 8 | (uint32_t)(b >> S8) << 16 | (uint32_t)(a >> S8) << 24;
            uint32_t idx = 0;
            for (uint32_t k = 0; k < job.palette_count; ++k)
                if (palette[k] == key) { idx = k; break; }
            job.storage[i] = (uint8_t)idx;
            return;
        }
        uint64_t s[4] = {0, 0, 0, 0};
        if (job.color == 0) s[0] = r;
        else if (job.color == 4) s[0] = r, s[1] = a;
        else s[0] = job.bgr ? b : r, s[1] = g, s[2] = job.bgr ? r : b, s[3] = a;
        uint64_t bits = 0;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const uint32_t v = narrow(s[c]);
            if (c < ch) bits |= wide ? (uint64_t)(__byte_perm(v, 0, 0x4401) & 0xffffu) << (16 * c) : (uint64_t)(v & 0xffu) << (8 * c);
        }
        color_store_pixel(job.storage, i, bpp, aligned, bits);
    };
    auto get = [&](uint64_t i) {
        if constexpr (SHAPE == COLOR_V) {
            const uint64_t v = ((const T*)job.pixels)[i];
            store(i, v, v, v, TMAX);
        } else if constexpr (SHAPE == COLOR_VA) {
            if constexpr (TBITS == 32) { const uint2 v = ((const uint2*)job.pixels)[i]; store(i, v.x, v.x, v.x, v.y); }
            else { const ulonglong2 v = ((const ulonglong2*)job.pixels)[i]; store(i, v.x, v.x, v.x, v.y); }
        } else {
            if constexpr (TBITS == 32) { const uint4 v = ((const uint4*)job.pixels)[i]; store(i, v.x, v.y, v.z, v.w); }
            else {
                const ulonglong2 v0 = ((const ulonglong2*)job.pixels)[2 * i], v1 = ((const ulonglong2*)job.pixels)[2 * i + 1];
                store(i, v0.x, v0.y, v1.x, v1.y);
            }
        }
    };
    uint64_t groups;
    const uint64_t head = color_edges<TBITS, SHAPE>(job, groups, get);
    constexpr uint64_t TILE = COLOR_TILE / G;
    for (uint64_t base = (uint64_t)blockIdx.x * TILE; base < groups; base += (uint64_t)gridDim.x * TILE) {
#pragma unroll 2
        for (uint64_t u = base + threadIdx.x; u < min(base + TILE, groups); u += COLOR_THREADS) {
            if constexpr (G == 1) {
                get(u);
            } else {
                const uint32_t w = ((const uint32_t*)(job.pixels + head * (TBITS / 8)))[u];
#pragma unroll
                for (int k = 0; k < G; ++k) {
                    const uint64_t v = (w >> (TBITS * k)) & TMAX;
                    store(head + u * G + k, v, v, v, TMAX);
                }
            }
        }
    }
}

template <int TBITS, int SHAPE>
__global__ void __launch_bounds__(COLOR_THREADS) pack_wide_kernel(ColorParams p)
{
    __shared__ uint32_t palette[256];
    for (uint32_t j = blockIdx.y; j < p.count; j += gridDim.y) {
        const ColorJob job = p.jobs[j];
        if (job.color == 3) {
            __syncthreads();
            if (threadIdx.x < job.palette_count) palette[threadIdx.x] = p.palettes[job.palette_off + threadIdx.x];
            __syncthreads();
        }
        pack_wide_image<TBITS, SHAPE>(job, palette);
    }
}

}  // namespace pngb200
