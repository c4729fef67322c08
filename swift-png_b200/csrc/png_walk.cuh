// png_walk.cuh -- the chunk walk of a whole PNG file, compiled for the host and the device: lexing, IHDR / PLTE /
// tRNS parsing and the ordering rules of the reference's decompress(stream:) (Sources/PNG/PNG.Image.swift:298-401;
// PNG.Header.init(parsing:standard:), Parsing/PNG.Header.swift:40-98; PNG.Palette.init(parsing:pixel:),
// PNG.Palette.swift:27-55; PNG.Transparency.init(parsing:pixel:palette:), PNG.Transparency.swift:68-122; ordering
// rules of Decoding/PNG.Metadata.swift:70-92 and PNG.Context.swift:51-81).  It reads the chunk headers and the
// bodies of IHDR, PLTE and tRNS; every other payload byte (CRCs, IDAT) is left to the device stages behind it.
//
// walk_png is the one statement of those rules.  pngb200_png_inspect_batch and pngb200_png_decode_batch run it on
// the host over host files (png_file.cuh, walk_file); png_walk_kernel runs it on the device, one warp per file, over
// files that already sit in device memory.  Inside an IDAT run the warp walks speculatively: lane j loads the header
// that would follow if the next j chunks all had the current chunk's length, and the walk takes the longest prefix
// of lanes that pass the checks lex() makes (type IDAT, same length, body and CRC inside the file) in one step.
// Records and summaries are the scalar walk's, bit for bit (tests/emu/emu_png_walk.cpp).
#pragma once

#include "common.cuh"

namespace pngb200 {

#define PNGB200_HD __host__ __device__

constexpr uint32_t fourcc(char a, char b, char c, char d)
{
    return (uint32_t)(uint8_t)a << 24 | (uint32_t)(uint8_t)b << 16 | (uint32_t)(uint8_t)c << 8 | (uint32_t)(uint8_t)d;
}
constexpr uint32_t CK_CgBI = fourcc('C', 'g', 'B', 'I'), CK_IHDR = fourcc('I', 'H', 'D', 'R'), CK_PLTE = fourcc('P', 'L', 'T', 'E'),
                   CK_IDAT = fourcc('I', 'D', 'A', 'T'), CK_IEND = fourcc('I', 'E', 'N', 'D'), CK_tRNS = fourcc('t', 'R', 'N', 'S'),
                   CK_bKGD = fourcc('b', 'K', 'G', 'D'), CK_hIST = fourcc('h', 'I', 'S', 'T'), CK_cHRM = fourcc('c', 'H', 'R', 'M'),
                   CK_gAMA = fourcc('g', 'A', 'M', 'A'), CK_sRGB = fourcc('s', 'R', 'G', 'B'), CK_iCCP = fourcc('i', 'C', 'C', 'P'),
                   CK_sBIT = fourcc('s', 'B', 'I', 'T'), CK_pHYs = fourcc('p', 'H', 'Y', 's'), CK_sPLT = fourcc('s', 'P', 'L', 'T'),
                   CK_tIME = fourcc('t', 'I', 'M', 'E'), CK_iTXt = fourcc('i', 'T', 'X', 't'), CK_tEXt = fourcc('t', 'E', 'X', 't'),
                   CK_zTXt = fourcc('z', 'T', 'X', 't');
constexpr uint32_t PNG_SIGNATURE_HI = 0x89504E47u, PNG_SIGNATURE_LO = 0x0D0A1A0Au;  // 137 P N G \r \n 26 \n

PNGB200_HD inline uint32_t load_be32(const uint8_t* p) { return (uint32_t)p[0] << 24 | (uint32_t)p[1] << 16 | (uint32_t)p[2] << 8 | p[3]; }
PNGB200_HD inline uint32_t load_be16(const uint8_t* p) { return (uint32_t)p[0] << 8 | p[1]; }

// PNG.Chunk.init(validating:) (Lexing/PNG.Chunk.swift:39-58)
PNGB200_HD inline bool chunk_type_ok(uint32_t name)
{
    switch (name) {
    case CK_CgBI: case CK_IHDR: case CK_PLTE: case CK_IDAT: case CK_IEND: case CK_cHRM: case CK_gAMA: case CK_iCCP:
    case CK_sBIT: case CK_sRGB: case CK_bKGD: case CK_hIST: case CK_tRNS: case CK_pHYs: case CK_sPLT: case CK_tIME:
    case CK_iTXt: case CK_tEXt: case CK_zTXt:
        return true;
    default:
        return (name & 0x20002000u) == 0x20000000u;
    }
}

// PNG.Format.Pixel.recognize(code:): whether (color, depth, bgr) is a pixel format (bgr, the iOS byte order: 8-bit
// RGB and RGBA only), and the channels of colour type `color` (4 for a type that does not exist)
struct PixelRule { bool valid; int channels; };
PNGB200_HD inline PixelRule pixel_rule(int color, int depth, bool bgr)
{
    bool ok;
    switch (color) {
    case 0: ok = depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16; break;
    case 3: ok = depth == 1 || depth == 2 || depth == 4 || depth == 8; break;
    case 2: case 4: case 6: ok = depth == 8 || depth == 16; break;
    default: ok = false;
    }
    if (bgr && (depth != 8 || (color != 2 && color != 6))) ok = false;
    return {ok, color == 0 || color == 3 ? 1 : color == 2 ? 3 : color == 4 ? 2 : 4};
}

struct ChunkRec {
    uint64_t off;       // offset of the chunk's length field in the file
    uint32_t len;       // body bytes
    uint32_t type;
    uint32_t declared;  // CRC-32 stored behind the body
};

constexpr uint64_t WALK_NONE = ~0ull;

// What the walk learned about one file (POD: the device walk hands it to the host as it is).  `stop` is the index of
// the chunk at which the reference would have thrown for a structural reason (WALK_NONE if none); `stop_before_crc`
// tells whether that happens before the chunk's own CRC check (lexing) or after it (parsing / ordering).
// [first_idat, idat_end) is the contiguous IDAT run.  format.palette is left null: the palette is written to the
// walk's `palette` argument, `palette_entries` entries of it.
struct WalkHead {
    int32_t              status;
    uint32_t             a, b;
    uint32_t             stop_before_crc;
    uint64_t             stop, first_idat, idat_end;
    uint64_t             chunks;
    uint32_t             width, height;
    uint8_t              depth, color, interlaced, standard;
    uint32_t             idat_chunks;
    pngb200_pixel_format format;
    uint64_t             storage_size, idat_bytes;
    uint32_t             palette_entries;
    uint32_t             pad_;
};
struct WalkSummary {
    WalkHead head;
    uint8_t  palette_rgba[1024];
};

// A record sink over an array; null: count only
struct RecordArray {
    ChunkRec* p;
    PNGB200_HD void put(uint64_t k, const ChunkRec& r) const
    {
        if (p) p[k] = r;
    }
};

// Walks file `f` of `n` bytes.  `sink.put(k, rec)` takes chunk k's record in order; `palette` receives the RGBA
// palette (alpha 255 until the first IDAT merges tRNS in).  `writer`: this thread writes the palette and the records
// the scalar steps lex.  Warp: all 32 lanes of a warp call this with the same arguments (lane 0 the writer) and take
// the IDAT runs in speculative steps of 32 chunks; every lane ends with the same `s`.
template <bool Warp, class Sink>
PNGB200_HD void walk_png(const uint8_t* f, uint64_t n, WalkHead& s, uint8_t* palette, const Sink& sink, bool writer)
{
    s = WalkHead{};
    s.stop = s.first_idat = WALK_NONE;
    if (n < 8) {
        s.status = PNGB200_ERR_LEX_TRUNCATED_SIGNATURE, s.stop = 0, s.stop_before_crc = 1;
        return;
    }
    if (load_be32(f) != PNG_SIGNATURE_HI || load_be32(f + 4) != PNG_SIGNATURE_LO) {
        s.status = PNGB200_ERR_LEX_INVALID_SIGNATURE, s.a = load_be32(f), s.b = load_be32(f + 4), s.stop = 0, s.stop_before_crc = 1;
        return;
    }
    auto stop = [&](int status, uint32_t a, uint32_t b, bool before_crc) {
        s.status = status, s.a = a, s.b = b;
        s.stop = s.chunks - (before_crc ? 0 : 1);
        s.stop_before_crc = before_crc;
    };
    uint64_t at = 8;
    ChunkRec c{};  // the last chunk lexed
    // lexes one chunk header; false = stopped
    auto lex = [&]() -> bool {
        if (n - at < 8) { stop(PNGB200_ERR_LEX_TRUNCATED_CHUNK_HEADER, 0, 0, true); return false; }
        const uint32_t len = load_be32(f + at), name = load_be32(f + at + 4);
        if (!chunk_type_ok(name)) { stop(PNGB200_ERR_LEX_INVALID_CHUNK_TYPE, name, 0, true); return false; }
        if ((uint64_t)(n - at - 8) < (uint64_t)len + 4) { stop(PNGB200_ERR_LEX_TRUNCATED_CHUNK_BODY, len + 4, 0, true); return false; }
        c = {at, len, name, load_be32(f + at + 8 + len)};
        if (writer) sink.put(s.chunks, c);
        s.chunks++;
        at += 12 + (uint64_t)len;
        return true;
    };
    if (!lex()) return;
    if (c.type == CK_CgBI) {
        s.standard = 1;
        if (!lex()) return;
    }
    {
        if (c.type != CK_IHDR) return stop(PNGB200_ERR_DECODE_REQUIRED_CHUNK, CK_IHDR, c.type, false);
        const uint8_t* h = f + c.off + 8;
        if (c.len != 13) return stop(PNGB200_ERR_PARSE_HEADER_CHUNK_LENGTH, c.len, 0, false);
        const int depth = h[8], color = h[9];
        const PixelRule rule = pixel_rule(color, depth, false);
        if (!rule.valid) return stop(PNGB200_ERR_PARSE_HEADER_PIXEL_FORMAT_CODE, (uint32_t)depth, (uint32_t)color, false);
        if (s.standard == 1 && !pixel_rule(color, depth, true).valid)
            return stop(PNGB200_ERR_PARSE_HEADER_PIXEL_FORMAT, (uint32_t)depth, (uint32_t)color, false);
        if (h[10]) return stop(PNGB200_ERR_PARSE_HEADER_COMPRESSION_CODE, h[10], 0, false);
        if (h[11]) return stop(PNGB200_ERR_PARSE_HEADER_FILTER_CODE, h[11], 0, false);
        if (h[12] > 1) return stop(PNGB200_ERR_PARSE_HEADER_INTERLACING_CODE, h[12], 0, false);
        s.width = load_be32(h), s.height = load_be32(h + 4);
        if (!s.width || !s.height) return stop(PNGB200_ERR_PARSE_HEADER_SIZE, s.width, s.height, false);
        // the reference traps when the storage size overflows (PNG.Image.swift:84); refuse such a file here
        // (w * h < 2^62, so w * h * bpp > 2^46, overflowing or not, is w * h > 2^46 / bpp)
        const uint64_t bpp = (uint64_t)((depth * rule.channels + 7) >> 3);
        if (s.width > 0x7fffffffu || s.height > 0x7fffffffu || (uint64_t)s.width * s.height > (1ull << 46) / (bpp ? bpp : 1))
            return stop(PNGB200_ERR_PARSE_HEADER_SIZE, s.width, s.height, false);
        s.depth = (uint8_t)depth, s.color = (uint8_t)color, s.interlaced = h[12];
        s.format.color = s.color, s.format.depth = s.depth, s.format.bgr = s.standard;
        s.storage_size = (uint64_t)s.width * s.height * bpp;
    }
    bool     have_palette = false, have_background = false, have_transparency = false;
    uint32_t npal = 0, nalpha = 0;
    uint64_t alpha_at = 0;  // tRNS body of an indexed file: merged into the palette at the first IDAT
    for (;;) {  // up to the first IDAT
        if (!lex()) return;
        const uint8_t* body = f + c.off + 8;
        if (c.type == CK_IHDR) return stop(PNGB200_ERR_DECODE_DUPLICATE_CHUNK, CK_IHDR, 0, false);
        if (c.type == CK_PLTE) {
            if (have_palette) return stop(PNGB200_ERR_DECODE_DUPLICATE_CHUNK, CK_PLTE, 0, false);
            if (have_background) return stop(PNGB200_ERR_DECODE_UNEXPECTED_CHUNK, CK_PLTE, CK_bKGD, false);
            if (have_transparency) return stop(PNGB200_ERR_DECODE_UNEXPECTED_CHUNK, CK_PLTE, CK_tRNS, false);
            if (s.color == 0 || s.color == 4) return stop(PNGB200_ERR_PARSE_UNEXPECTED_PALETTE, 0, 0, false);
            if (c.len % 3) return stop(PNGB200_ERR_PARSE_PALETTE_CHUNK_LENGTH, c.len, 0, false);
            const uint32_t max = 1u << (s.depth < 8 ? s.depth : 8);
            if (c.len / 3 < 1 || c.len / 3 > max) return stop(PNGB200_ERR_PARSE_PALETTE_COUNT, c.len / 3, max, false);
            have_palette = true, npal = c.len / 3;
            if (s.color == 3) {
                s.palette_entries = npal;
                if (writer)
                    for (uint32_t i = 0; i < npal; ++i) {
                        palette[4 * i] = body[3 * i], palette[4 * i + 1] = body[3 * i + 1], palette[4 * i + 2] = body[3 * i + 2];
                        palette[4 * i + 3] = 255;
                    }
            }
        } else if (c.type == CK_tRNS) {
            if (have_transparency) return stop(PNGB200_ERR_DECODE_DUPLICATE_CHUNK, CK_tRNS, 0, false);
            const uint32_t max = 0xffffu >> (16 - s.depth);
            if (s.color == 0) {
                if (c.len != 2) return stop(PNGB200_ERR_PARSE_TRANSPARENCY_CHUNK_LENGTH, c.len, 2, false);
                if (load_be16(body) > max) return stop(PNGB200_ERR_PARSE_TRANSPARENCY_SAMPLE, load_be16(body), max, false);
                s.format.has_key = 1, s.format.key[0] = (uint16_t)load_be16(body);
            } else if (s.color == 2) {
                if (c.len != 6) return stop(PNGB200_ERR_PARSE_TRANSPARENCY_CHUNK_LENGTH, c.len, 6, false);
                const uint32_t r = load_be16(body), g = load_be16(body + 2), b = load_be16(body + 4);
                const uint32_t top = r > g ? (r > b ? r : b) : (g > b ? g : b);
                if (top > max) return stop(PNGB200_ERR_PARSE_TRANSPARENCY_SAMPLE, top, max, false);
                s.format.has_key = 1;  // Format.recognize keeps a bgr8 key in (b, g, r) order (PNG.Format.swift:228-240)
                s.format.key[0] = (uint16_t)(s.standard ? b : r), s.format.key[1] = (uint16_t)g, s.format.key[2] = (uint16_t)(s.standard ? r : b);
            } else if (s.color == 3) {
                if (!have_palette) return stop(PNGB200_ERR_DECODE_REQUIRED_CHUNK, CK_PLTE, CK_tRNS, false);
                if (c.len > npal) return stop(PNGB200_ERR_PARSE_TRANSPARENCY_COUNT, c.len, npal, false);
                alpha_at = c.off + 8, nalpha = c.len;
            } else
                return stop(PNGB200_ERR_PARSE_UNEXPECTED_TRANSPARENCY, 0, 0, false);
            have_transparency = true;
        } else if (c.type == CK_bKGD) {
            if (have_background) return stop(PNGB200_ERR_DECODE_DUPLICATE_CHUNK, CK_bKGD, 0, false);
            if (s.color == 3 && !have_palette) return stop(PNGB200_ERR_DECODE_REQUIRED_CHUNK, CK_PLTE, CK_bKGD, false);
            have_background = true;
        } else if (c.type == CK_cHRM || c.type == CK_gAMA || c.type == CK_sRGB || c.type == CK_iCCP || c.type == CK_sBIT) {
            if (have_palette) return stop(PNGB200_ERR_DECODE_UNEXPECTED_CHUNK, c.type, CK_PLTE, false);
        } else if (c.type == CK_hIST) {
            if (!have_palette) return stop(PNGB200_ERR_DECODE_REQUIRED_CHUNK, CK_PLTE, CK_hIST, false);
        } else if (c.type == CK_IDAT) {
            if (s.color == 3 && !have_palette) return stop(PNGB200_ERR_DECODE_REQUIRED_CHUNK, CK_PLTE, CK_IDAT, false);
            if (writer)
                for (uint32_t i = 0; i < nalpha; ++i) palette[4 * i + 3] = f[alpha_at + i];
            s.format.palette_count = s.color == 3 ? (uint16_t)npal : 0;
            break;
        } else if (c.type == CK_IEND) {
            return stop(PNGB200_ERR_DECODE_REQUIRED_CHUNK, CK_IDAT, CK_IEND, false);
        }
    }
    s.first_idat = s.chunks - 1;
    while (c.type == CK_IDAT) {
        s.idat_bytes += c.len, s.idat_chunks++;
        s.idat_end = s.chunks;
#if defined(__CUDA_ARCH__) || defined(PNGB200_EMU)
        if (Warp) {
            // speculative steps: lane j checks the header 12 + len bytes * j behind `at`
            const uint32_t lane = threadIdx.x & 31u;
            const uint64_t step = 12 + (uint64_t)c.len;
            for (;;) {
                const uint64_t h = at + lane * step;
                bool     ok = false;
                uint32_t declared = 0;
                if (h < n && n - h >= 8 && load_be32(f + h) == c.len && load_be32(f + h + 4) == CK_IDAT &&
                    n - h - 8 >= (uint64_t)c.len + 4) {
                    ok = true;
                    declared = load_be32(f + h + 8 + c.len);
                }
                const uint32_t pass = __ballot_sync(0xffffffffu, ok);
                const uint32_t m = pass == 0xffffffffu ? 32u : (uint32_t)(__ffs(~pass) - 1);
                if (m == 0) break;
                if (lane < m) sink.put(s.chunks + lane, ChunkRec{h, c.len, CK_IDAT, declared});
                c.off = at + (uint64_t)(m - 1) * step;
                c.declared = __shfl_sync(0xffffffffu, declared, m - 1);
                s.chunks += m, s.idat_chunks += m, s.idat_bytes += (uint64_t)m * c.len;
                s.idat_end = s.chunks;
                at += (uint64_t)m * step;
                if (m < 32) break;
            }
        }
#endif
        if (!lex()) return;
    }
    for (;;) {  // Context.push(ancillary:) until IEND
        const uint32_t t = c.type;
        if (t == CK_IEND) return;
        switch (t) {
        case CK_CgBI: case CK_IHDR: case CK_PLTE: case CK_bKGD: case CK_tRNS: case CK_IDAT: case CK_hIST: case CK_cHRM:
        case CK_gAMA: case CK_sRGB: case CK_iCCP: case CK_sBIT: case CK_pHYs: case CK_sPLT:
            return stop(PNGB200_ERR_DECODE_UNEXPECTED_CHUNK, t, CK_IDAT, false);
        default: break;
        }
        if (!lex()) return;
    }
}

struct WalkFile {
    const uint8_t* file;
    uint64_t       len;
};

constexpr int WALK_WARPS = 4;

// One warp per file.  Pass 1 (recs null): summaries only.  Pass 2: also the records, file i's at recs + rec_base[i].
__global__ void __launch_bounds__(WALK_WARPS * 32)
    png_walk_kernel(const WalkFile* files, uint32_t count, WalkSummary* sums, ChunkRec* recs, const uint64_t* rec_base)
{
    const uint32_t i = blockIdx.x * WALK_WARPS + (threadIdx.x >> 5);
    if (i >= count) return;
    const bool lead = (threadIdx.x & 31) == 0;
    WalkHead   h;
    walk_png<true>(files[i].file, files[i].len, h, sums[i].palette_rgba, RecordArray{recs ? recs + rec_base[i] : nullptr}, lead);
    if (lead) sums[i].head = h;
}

}  // namespace pngb200
