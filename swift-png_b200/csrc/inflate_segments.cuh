// inflate_segments.cuh -- more than one CTA per DEFLATE stream (SURVEY section 7 "Stage B").
//
// The reference's token loop is serial per stream (Stream.readBlock(with:),
// Sources/LZ77/Inflator/LZ77.InflatorBuffers.Stream.swift:266-381) and so is one CTA of
// inflate_wave_kernel.  A batch with fewer streams than CTA slots (BASELINE configs 4 and 5: 8 images
// per GPU, one 1 GiB gzip stream) would leave the GPU idle, so such streams are cut into SEGMENTS:
//
//   1. block_search_kernel (block_search.cuh) finds, for every wanted split point, the next bit offset
//      that holds a plausible dynamic-block header (a pure function of the offset; false positives are
//      caught in step 3).
//   2. inflate_wave_kernel decodes every segment with its own CTA into 16-bit symbols: bytes copied from
//      in front of the segment are markers 0x8000 | window index (see emit_token_sym).
//   3. the host accepts a stream only if every segment ended exactly where the next one starts (on a
//      block boundary) -- otherwise the stream is simply decoded whole; correct by construction.
//   4. window_propagate_kernel resolves, segment by segment, the 32 KiB window in front of each segment
//      (a serial chain per stream, 32 KiB per link), marker_resolve_kernel then replaces the markers of
//      all segments in parallel and packs the symbols into the byte stream at their final offsets.
#pragma once

#include "common.cuh"
#include "inflate_stream.cuh"   // shared pieces: Adler-32 helpers

namespace pngb200 {

constexpr uint32_t SEG_WINDOW = 32768;

struct SegmentRecord {         // one per segment, in stream order; segments of one stream are adjacent
    const uint16_t* sym;       // the segment's symbols
    uint8_t*        out;       // final position of the segment's first byte
    uint64_t        produced;  // symbols in the segment
    uint32_t        stream;    // index of the stream (window chain) it belongs to
    uint32_t        first;     // 1: first segment of its stream (no window in front, no markers)
};

// window[k] (32 KiB of bytes) = the output in front of segment k.  One CTA per stream walks the chain:
// window[k+1] = last 32 KiB of (window[k] ++ resolved segment k).
__global__ void __launch_bounds__(256) window_propagate_kernel(const SegmentRecord* segs, const uint32_t* stream_first,
                                                               uint32_t nstreams, uint8_t* windows)
{
    if (blockIdx.x >= nstreams) return;
    const uint32_t lo = stream_first[blockIdx.x], hi = stream_first[blockIdx.x + 1];
    for (uint32_t k = lo; k + 1 < hi; ++k) {
        const SegmentRecord s  = segs[k];
        const uint8_t*      w  = windows + (size_t)k * SEG_WINDOW;        // window in front of segment k
        uint8_t*            wn = windows + (size_t)(k + 1) * SEG_WINDOW;  // window in front of segment k + 1
        const uint64_t      n  = s.produced;
        for (uint32_t i = threadIdx.x; i < SEG_WINDOW; i += blockDim.x) {
            // byte i of the next window is byte (n - 32768 + i) of this segment, or, if the segment is shorter
            // than the window, byte (i + n) of this segment's own window
            uint8_t v;
            if (n + i >= SEG_WINDOW) {
                const uint16_t x = s.sym[n + i - SEG_WINDOW];
                v = (x & 0x8000u) ? (s.first ? 0 : w[x & 0x7fffu]) : (uint8_t)x;
            } else {
                v = s.first ? 0 : w[i + n];
            }
            wn[i] = v;
        }
        __threadfence();
        __syncthreads();
    }
}

// every symbol of every segment -> its byte at its final place; 16 bytes per thread-iteration
__global__ void __launch_bounds__(256) marker_resolve_kernel(const SegmentRecord* segs, uint32_t nsegs, const uint8_t* windows,
                                                             const uint64_t* chunk_base)
{
    // chunk_base[k]: exclusive prefix of ceil(produced / 4096) over the segments; one CTA per 4096-symbol chunk
    const uint64_t chunk = blockIdx.x;
    uint32_t lo = 0, hi = nsegs;
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (chunk_base[mid] <= chunk) lo = mid;
        else hi = mid;
    }
    const SegmentRecord s = segs[lo];
    const uint8_t*      w = windows + (size_t)lo * SEG_WINDOW;
    const uint64_t base = (chunk - chunk_base[lo]) * 4096;
    for (uint32_t j = threadIdx.x; j < 4096; j += blockDim.x) {
        const uint64_t i = base + j;
        if (i >= s.produced) break;
        const uint16_t x = s.sym[i];
        s.out[i] = (x & 0x8000u) ? (s.first ? 0 : w[x & 0x7fffu]) : (uint8_t)x;
    }
}

// ---- a stream cut in two (DESIGN.md section 4.2 "head and tail") ----
// The HEAD decodes bits [0, split) straight into the stream's output and folds Adler-32 as a whole stream does;
// the TAIL decodes from the block header at `split` to the trailer into symbols.  The 32 KiB in front of the tail
// is the end of the head's output, already final, so no window chain is needed: one pass replaces the markers,
// writes the tail's bytes behind the head's and folds their Adler-32 partial sums.
struct SplitRecord {
    const StreamResult* head;      // head's result: produced = n1, checksum = Adler-32 of bytes [0, n1)
    const StreamResult* tail;      // tail's result: produced = n2, declared = the stream's trailer
    const uint16_t*     sym;       // the tail's symbols
    uint8_t*            out;       // the stream's output (the head's dst)
    uint64_t            dst_cap;
    uint64_t            split_bit; // where the tail starts (the head's stop_bit)
    StreamResult*       final_;    // the stream's result record, written only when the split is accepted
    const SwitchRecord* sw = nullptr;   // where the tail left symbolic mode; null: it did not (all n2 are symbols)
};

// tail bytes [0, m) are symbols, [m, n2) bytes (SwitchRecord)
__device__ __forceinline__ uint64_t split_switch_out(const SplitRecord& s, uint64_t n2) { return s.sw ? s.sw->out : n2; }

constexpr uint32_t SPLIT_CTAS = 64;  // resolve CTAs per split stream (blockIdx.y)

// the pieces line up: the head ended on the tail's first block header, the tail reached the trailer, and the
// head is long enough to hold every byte a marker can refer to
__device__ __forceinline__ bool split_lines_up(const SplitRecord& s, uint64_t n1, uint64_t n2)
{
    return s.head->status == PNGB200_OK && s.head->phase == 1 && s.head->consumed_bits == s.split_bit &&
           s.tail->status == PNGB200_OK && s.tail->phase == 2 && n1 >= SEG_WINDOW && n1 + n2 <= s.dst_cap &&
           split_switch_out(s, n2) <= n2;
}

// grid (splits, SPLIT_CTAS): CTA y takes the 4096-byte chunks y, y + SPLIT_CTAS, ... of its stream's tail and leaves
// the tail's Adler-32 partial sums (sum of b, sum of (n2 - i) b, both mod 65521) in partial[2 * (k * SPLIT_CTAS + y)].
// Tail bytes [0, m) are symbols; [m, n2) are bytes the tail wrote after it left symbolic mode (SplitRecord.sw)
__global__ void __launch_bounds__(256) split_resolve_kernel(const SplitRecord* recs, uint32_t* partial)
{
    const SplitRecord s  = recs[blockIdx.x];
    const uint64_t    n1 = s.head->produced, n2 = s.tail->produced;
    uint32_t*         pp = partial + 2 * ((size_t)blockIdx.x * SPLIT_CTAS + blockIdx.y);
    if (!split_lines_up(s, n1, n2)) return;
    const uint64_t m = split_switch_out(s, n2);
    const uint8_t* w = s.out + n1 - SEG_WINDOW;   // marker index -> byte in front of the tail
    uint8_t*       o = s.out + n1;
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(s.sym) + (s.sw ? s.sw->bytes : 0);   // tail byte m
    uint64_t a = 0, b = 0;
    for (uint64_t base = (uint64_t)blockIdx.y * 4096; base < n2; base += (uint64_t)SPLIT_CTAS * 4096) {
        const uint64_t end = min(base + 4096, n2);
        for (uint64_t i = base + threadIdx.x; i < min(end, m); i += blockDim.x) {
            const uint16_t x = s.sym[i];
            const uint8_t  v = (x & 0x8000u) ? w[x & 0x7fffu] : (uint8_t)x;
            o[i] = v;
            a += v;
            b += (n2 - i) * v;
        }
        if (end > m) {
            // bytes [lo, end): 16-byte stores aligned in the output; the source (any relative alignment) is read as
            // five aligned words per store and shifted into place
            const uint64_t  lo = max(base, m);
            const uintptr_t g0 = (uintptr_t)(o + lo) & ~(uintptr_t)15;
            const uint64_t  ng = ((uintptr_t)(o + end) - g0 + 15) / 16;
            for (uint64_t g = threadIdx.x; g < ng; g += blockDim.x) {
                const int64_t i0 = (int64_t)(g0 + 16 * g - (uintptr_t)o);   // tail offset of the group's first byte
                if (i0 >= (int64_t)lo && (uint64_t)i0 + 16 <= end) {
                    const uint8_t*  src = bytes + ((uint64_t)i0 - m);
                    const uint32_t* sw  = reinterpret_cast<const uint32_t*>((uintptr_t)src & ~(uintptr_t)3);
                    const uint32_t  sh  = 8 * (uint32_t)((uintptr_t)src & 3);
                    const uint32_t  w0 = sw[0], w1 = sw[1], w2 = sw[2], w3 = sw[3], w4 = sw[4];
                    uint4 x;
                    x.x = __funnelshift_r(w0, w1, sh);
                    x.y = __funnelshift_r(w1, w2, sh);
                    x.z = __funnelshift_r(w2, w3, sh);
                    x.w = __funnelshift_r(w3, w4, sh);
                    *reinterpret_cast<uint4*>(o + i0) = x;
                    adler_chunk16(x, n2 - (uint64_t)i0, a, b);
                } else {
                    for (int64_t i = max(i0, (int64_t)lo); i < min(i0 + 16, (int64_t)end); ++i) {
                        const uint8_t v = bytes[i - m];
                        o[i] = v;
                        a += v;
                        b += (n2 - i) * v;
                    }
                }
            }
        }
        b %= ADLER_MOD32;
    }
    uint32_t a32 = (uint32_t)(a % ADLER_MOD32), b32 = (uint32_t)b;
    for (int k = 16; k; k >>= 1) {
        a32 += __shfl_down_sync(0xffffffffu, a32, k);
        b32 += __shfl_down_sync(0xffffffffu, b32, k);
    }
    __shared__ uint32_t red[2][8];
    const unsigned warp = threadIdx.x >> 5;
    if (lane_id() == 0) { red[0][warp] = a32 % ADLER_MOD32; red[1][warp] = b32 % ADLER_MOD32; }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t sa = 0, sb = 0;
        for (unsigned k = 0; k < blockDim.x / 32; ++k) { sa += red[0][k]; sb += red[1][k]; }
        pp[0] = sa % ADLER_MOD32;
        pp[1] = sb % ADLER_MOD32;
    }
}

// one thread per split stream: Adler-32 of head ++ tail from the head's checksum and the tail's partial sums, checked
// against the trailer.  A stream whose pieces line up and whose checksum matches gets its final result record and
// accept[k] = 1; any other stream keeps an untouched record (accept[k] = 0) and is decoded whole afterwards.
__global__ void __launch_bounds__(128) split_finish_kernel(const SplitRecord* recs, uint32_t count, const uint32_t* partial,
                                                           uint32_t* accept)
{
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= count) return;
    const SplitRecord s  = recs[k];
    const uint64_t    n1 = s.head->produced, n2 = s.tail->produced;
    bool ok = split_lines_up(s, n1, n2) && s.head->ck_done;
    uint32_t computed = 0;
    if (ok) {
        uint64_t ta = 0, tb = 0;
        for (uint32_t y = 0; y < SPLIT_CTAS; ++y) {
            ta += partial[2 * ((size_t)k * SPLIT_CTAS + y)];
            tb += partial[2 * ((size_t)k * SPLIT_CTAS + y) + 1];
        }
        // adler(H ++ T): A = A_H + sum T, B = B_H + |T| A_H + sum (|T| - i) T_i  (the zlib adler32_combine arithmetic)
        const uint64_t ah = s.head->checksum & 0xffffu, bh = s.head->checksum >> 16;
        const uint64_t A = (ah + ta) % ADLER_MOD32;
        const uint64_t B = (bh + (n2 % ADLER_MOD32) * ah + tb) % ADLER_MOD32;
        computed = (uint32_t)(B << 16 | A);
        ok = computed == s.tail->declared;
    }
    accept[k] = ok ? 1u : 0u;
    if (!ok) return;
    // what a whole-stream decode reports: trailer fields from the tail, counts over both pieces
    StreamResult f = *s.tail;
    const StreamResult& h = *s.head;
    f.produced   = n1 + n2;
    f.resume_out = n1 + f.resume_out;
    f.blocks     = h.blocks + f.blocks;
    f.checksum   = computed;
    f.ck_done    = 1;
    f.stat_waves += h.stat_waves;
    f.stat_sync_rounds += h.stat_sync_rounds;
    f.stat_resolve_rounds = max(f.stat_resolve_rounds, h.stat_resolve_rounds);
    f.stat_fallback |= h.stat_fallback;
    f.stat_tokens += h.stat_tokens;
    f.stat_matches += h.stat_matches;
    f.stat_deferred += h.stat_deferred;
    for (int q = 0; q < 12; ++q) f.stat_cycles[q] += h.stat_cycles[q];
    *s.final_ = f;
}

}  // namespace pngb200
