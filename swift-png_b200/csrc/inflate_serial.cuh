// inflate_serial.cuh -- one warp per DEFLATE stream: the latency-tolerant, fully general inflate.
//
// Every lane holds the same bit-reader state and walks the token loop in lock step (loads are
// warp broadcasts), so literal/length/distance decoding costs one instruction stream; the 32
// lanes then split each LZ77 copy.  This kernel is the correctness anchor (all block types,
// truncation, every error of LZ77.DecompressionError), the resume-capable back end of the
// streaming pngb200_inflator, and the fallback for tiny streams.  Throughput on big batches comes
// from inflate_parallel.cuh.
//
// Replaces LZ77.InflatorBuffers.advance + Stream.readBlock* (Sources/LZ77/Inflator/
// LZ77.InflatorBuffers.swift:25-230, LZ77.InflatorBuffers.Stream.swift:59-399) and
// LZ77.InflatorOut.append/expand (LZ77.InflatorOut.swift:114-140).
#pragma once

#include "huffman.cuh"

namespace pngb200 {

struct SerialShared {
    uint32_t    lit[LIT_CAP];
    uint32_t    dist[DIST_CAP];
    uint32_t    meta[META_CAP];
    uint8_t     lens[320 + 140];
    HuffScratch scratch;
};

// LSB-first bit reader over 32-bit aligned words; bytes outside [src, src+len) read as zero,
// which reproduces the reference's 48 zero pad bits (LZ77.InflatorIn.swift:47-138).
struct BitReader {
    const uint32_t* words;
    uint64_t        lead_bits;  // bits in the first aligned word that precede the stream
    uint64_t        total_bits; // lead_bits + 8 * len
    uint64_t        wi;         // next word to load
    uint64_t        buf;
    int             cnt;
    uint64_t        pos;        // absolute position in `words` bit space (includes lead_bits)

    __device__ void init(const uint8_t* src, uint64_t len, uint64_t start_bit)
    {
        uintptr_t a = (uintptr_t)src;
        words       = (const uint32_t*)(a & ~(uintptr_t)3);
        lead_bits   = (a & 3) * 8;
        total_bits  = lead_bits + 8 * len;
        seek(lead_bits + start_bit);
    }
    __device__ void seek(uint64_t p)
    {
        pos = p;
        wi  = p >> 5;
        buf = 0;
        cnt = 0;
        refill();
        int skip = (int)(p & 31);
        buf >>= skip;
        cnt -= skip;
    }
    __device__ __forceinline__ uint32_t load_word(uint64_t i) const
    {
        uint64_t lo = i << 5;
        if (lo >= total_bits) return 0;
        uint32_t w = __ldg(words + i);
        if (lo < lead_bits) w &= ~0u << (lead_bits - lo);           // only i == 0
        if (lo + 32 > total_bits) w &= ~0u >> (lo + 32 - total_bits);
        return w;
    }
    __device__ __forceinline__ void refill()
    {
        while (cnt <= 32) {
            buf |= (uint64_t)load_word(wi) << cnt;
            cnt += 32;
            ++wi;
        }
    }
    __device__ __forceinline__ uint32_t peek() const { return (uint32_t)buf; }
    __device__ __forceinline__ void     consume(int n)
    {
        buf >>= n;
        cnt -= n;
        pos += n;
    }
    __device__ __forceinline__ uint32_t take(int n)
    {
        uint32_t v = (uint32_t)buf & (n >= 32 ? ~0u : ((1u << n) - 1u));
        consume(n);
        return v;
    }
    // stream-relative bit position and size
    __device__ __forceinline__ uint64_t at() const { return pos - lead_bits; }
    __device__ __forceinline__ uint64_t size() const { return total_bits - lead_bits; }
    __device__ __forceinline__ bool     have(uint64_t n) const { return pos + n <= total_bits; }
};

__device__ __forceinline__ int fail(StreamResult* r, int code, uint32_t a = 0, uint32_t b = 0)
{
    if (lane_id() == 0) {
        r->status = code;
        r->err_a  = a;
        r->err_b  = b;
    }
    return code;
}

// zlib / gzip stream headers.  LZ77.StreamHeader.read (LZ77.StreamHeader.swift:16-54),
// Gzip.StreamHeader.read + .strings (Gzip.StreamHeader.swift:19-83, InflatorBuffers.swift:153-197)
__device__ int read_stream_header(BitReader& br, int format, StreamResult* r)
{
    if (format == PNGB200_FORMAT_ZLIB) {
        if (!br.have(16)) return PNGB200_NEED_MORE_INPUT;
        br.refill();
        uint32_t v = br.take(16);
        uint32_t method = v & 15, e = (v >> 4) & 15, flags = v >> 8;
        if (method != 8) return fail(r, PNGB200_ERR_ZLIB_METHOD, method);
        if (e >= 8) return fail(r, PNGB200_ERR_ZLIB_WINDOW, e + 8);
        if ((((e << 12) | (8u << 8)) + flags) % 31 != 0) return fail(r, PNGB200_ERR_ZLIB_CHECK_BITS);
        if (flags & 0x20) return fail(r, PNGB200_ERR_ZLIB_DICTIONARY);
    } else if (format == PNGB200_FORMAT_GZIP) {
        if (!br.have(80)) return PNGB200_NEED_MORE_INPUT;
        br.refill();
        uint32_t sig = br.take(16);
        if (sig != 0x8b1f) return fail(r, PNGB200_ERR_GZIP_SIGIL);
        br.refill();
        uint32_t method = br.take(8);
        if (method != 8) return fail(r, PNGB200_ERR_GZIP_METHOD, method);
        uint32_t flags = br.take(8);
        if (flags & 0xe0) return fail(r, PNGB200_ERR_GZIP_FLAG_BITS, flags);
        if (flags & 0x02) return fail(r, PNGB200_ERR_GZIP_HEADER_CHECKSUM_UNSUPPORTED);
        br.refill();
        br.consume(32);  // MTIME
        br.refill();
        br.consume(16);  // XFL, OS
        if (flags & 0x04) {
            if (!br.have(16)) return PNGB200_NEED_MORE_INPUT;
            br.refill();
            uint64_t xlen = br.take(16);
            if (!br.have(8 * xlen)) return PNGB200_NEED_MORE_INPUT;
            br.seek(br.pos + 8 * xlen);
        }
        int strings = ((flags & 0x08) ? 1 : 0) + ((flags & 0x10) ? 1 : 0);
        while (strings > 0) {
            uint32_t byte;
            do {
                if (!br.have(8)) return PNGB200_NEED_MORE_INPUT;
                br.refill();
                byte = br.take(8);
            } while (byte != 0);
            --strings;
        }
    }
    return PNGB200_OK;
}

// Block header, part 1 (ONE warp, lock step): BFINAL/BTYPE, stored LEN/NLEN, or the code lengths
// of a fixed/dynamic block written to sh->lens (literal/length codes first, then distance codes).
// Returns PNGB200_OK with *type/*final/*stored_len/*nlit/*ndist set, PNGB200_NEED_MORE_INPUT, or
// an error.  Stream.readBlockMetadata / readBlockTables (LZ77.InflatorBuffers.Stream.swift:59-263).
template <typename Reader, typename Shared>
__device__ int parse_block_header(Reader& br, Shared* sh, StreamResult* r, int lane, int* type, int* final,
                                  uint32_t* stored_len, int* nlit_out, int* ndist_out)
{
    if (!br.have(3)) return PNGB200_NEED_MORE_INPUT;
    br.refill();
    uint32_t hdr = br.take(3);
    *final = hdr & 1;
    *type  = hdr >> 1;
    if (*type == 0) {
        uint64_t boundary = (br.pos + 7) & ~(uint64_t)7;
        if (boundary + 32 > br.total_bits) return PNGB200_NEED_MORE_INPUT;
        br.seek(boundary);
        uint32_t v = br.take(32);
        uint32_t l = v & 0xffff, m = v >> 16;
        if (l != (~m & 0xffffu)) return fail(r, PNGB200_ERR_BLOCK_COUNT_PARITY, l, m);
        br.refill();
        *stored_len = l;
        return PNGB200_OK;
    }
    if (*type == 3) return fail(r, PNGB200_ERR_BLOCK_TYPE, 3);
    int nlit, ndist;
    __syncwarp();
    if (*type == 1) {
        nlit = 288;
        ndist = 32;
        for (int s = lane; s < 320; s += 32)
            sh->lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : s < 288 ? 8 : 5;
    } else {
        if (!br.have(14)) return PNGB200_NEED_MORE_INPUT;
        br.refill();
        uint32_t v = br.take(14);
        nlit  = 257 + (int)(v & 31);
        ndist = 1 + (int)((v >> 5) & 31);
        int nclen = 4 + (int)(v >> 10);
        if (!br.have(3 * (uint64_t)nclen)) return PNGB200_NEED_MORE_INPUT;
        if (nlit > 286) return fail(r, PNGB200_ERR_RUNLITERAL_SYMBOL_COUNT, (uint32_t)nlit);
        if (lane < 19) sh->lens[lane] = 0;
        __syncwarp();
        for (int i = 0; i < nclen; ++i) {
            br.refill();
            uint32_t l = br.take(3);
            if (lane == 0) sh->lens[c_clen_order[i]] = (uint8_t)l;
        }
        __syncwarp();
        build_table<META_ROOT, META_CAP>(sh->meta, sh->lens, 19, ALPHA_META, &sh->scratch, lane, 32);
        if (sh->scratch.status) return fail(r, sh->scratch.status);
        // code lengths: sequential, replicated in every lane; lane 0 records them
        int total = nlit + ndist, have = 0;
        uint32_t prev = 0;
        __syncwarp();
        while (have < total) {
            if (!br.have(1)) return PNGB200_NEED_MORE_INPUT;
            br.refill();
            uint32_t e = sh->meta[br.peek() & (META_CAP - 1)];
            uint32_t len = e_len(e), sym = e_value(e);
            if (!br.have(len)) return PNGB200_NEED_MORE_INPUT;
            if (sym < 16) {
                br.consume((int)len);
                if (lane == 0) sh->lens[have] = (uint8_t)sym;
                prev = sym;
                ++have;
                continue;
            }
            uint32_t element, extra, base;
            if (sym == 16) {
                if (have == 0) return fail(r, PNGB200_ERR_CODELENGTH_SEQUENCE);
                element = prev; extra = 2; base = 3;
            } else if (sym == 17) {
                element = 0; extra = 3; base = 3;
            } else {
                element = 0; extra = 7; base = 11;
            }
            if (!br.have(len + extra)) return PNGB200_NEED_MORE_INPUT;
            br.consume((int)len);
            uint32_t reps = base + br.take((int)extra);
            for (uint32_t k = lane; k < reps; k += 32) sh->lens[have + k] = (uint8_t)element;
            prev = element;
            have += (int)reps;
        }
        if (have != total) return fail(r, PNGB200_ERR_CODELENGTH_SEQUENCE);
    }
    __syncwarp();
    *nlit_out  = nlit;
    *ndist_out = ndist;
    return PNGB200_OK;
}

// Block header, part 2 (cooperative, `nt` threads: 32 = calling warp, else the whole CTA): the
// literal/length and distance decode tables from sh->lens.
template <typename Shared>
__device__ int build_block_tables(Shared* sh, StreamResult* r, int nlit, int ndist, int tid, int nt)
{
    build_table<LIT_ROOT, LIT_CAP>(sh->lit, sh->lens, nlit, ALPHA_LITLEN, &sh->scratch, tid, nt);
    if (sh->scratch.status) return fail(r, sh->scratch.status);
    if (nt == 32) __syncwarp();
    else __syncthreads();
    build_table<DIST_ROOT, DIST_CAP>(sh->dist, sh->lens + nlit, ndist, ALPHA_DIST, &sh->scratch, tid, nt);
    if (sh->scratch.status) return fail(r, sh->scratch.status);
    return PNGB200_OK;
}

// zlib / gzip trailer: byte-align, read the 4-byte checksum (big-endian Adler-32 or little-endian
// CRC-32 followed by ISIZE).  The comparison happens in the checksum kernel.
// LZ77.InflatorBuffers.advance(.checksum) (LZ77.InflatorBuffers.swift:109-130, :206-223)
__device__ int read_trailer(BitReader& br, int format, StreamResult* r)
{
    if (format == PNGB200_FORMAT_IOS) {
        if (lane_id() == 0) r->trailer_seen = 1;
        return PNGB200_OK;
    }
    uint64_t boundary = (br.pos + 7) & ~(uint64_t)7;
    if (boundary + 32 > br.total_bits) return PNGB200_NEED_MORE_INPUT;
    br.seek(boundary);
    uint32_t v = br.take(32);
    uint32_t declared = format == PNGB200_FORMAT_GZIP ? v : __byte_perm(v, 0, 0x0123);
    if (lane_id() == 0) {
        r->declared     = declared;
        r->trailer_seen = 1;  // the checksum comparison outranks a missing ISIZE, as in the reference
    }
    if (format == PNGB200_FORMAT_GZIP) {
        if (!br.have(32)) return PNGB200_NEED_MORE_INPUT;  // ISIZE: read, never validated
        br.refill();
        br.consume(32);
    }
    return PNGB200_OK;
}

// The whole serial decode of one stream by one warp, from (start_bit, start_out, phase).  In phase 3, start_bit is a
// symbol inside the Huffman block whose header is at `header_bit`: the header is parsed again and decoding goes on at
// start_bit.  With a resume record (job.resume), input that ends inside a Huffman block leaves the resume point at
// the last complete symbol (phase 3), and the launch's work is added to the record's counters.
// `r` must have been zeroed (status 0) by the caller.
__device__ void serial_inflate(SerialShared& sh, const StreamJob& job, StreamResult* r, uint64_t start_bit,
                               uint64_t start_out, uint32_t phase, uint32_t blocks, uint64_t header_bit = 0)
{
    const unsigned lane = lane_id();
    BitReader      br;
    br.init(job.src, job.src_len, phase == 3 ? header_bit : start_bit);
    uint64_t out = start_out;
    int      st  = PNGB200_OK;
    uint64_t resume_bit = start_bit, resume_out = start_out;
    uint64_t reparsed = 0;          // header bits parsed again to resume inside a block
    bool     inside = phase == 3;   // the next header is that of the block to resume in
    uint64_t hdr_bit = header_bit;  // the current block's header and BFINAL (for a phase-3 resume point)
    int      final = 0;

    if (phase == 0) {
        st = read_stream_header(br, job.format, r);
        if (st == PNGB200_OK) {
            resume_bit = br.at();
            phase = 1;
        }
    }
    uint8_t* dst = job.dst;
    if (st == PNGB200_OK && phase == 2) st = read_trailer(br, job.format, r);
    while (st == PNGB200_OK && (phase == 1 || phase == 3)) {
        int      type;
        uint32_t stored = 0;
        int nlit = 0, ndist = 0;
        hdr_bit = br.at();
        st = parse_block_header(br, &sh, r, (int)lane, &type, &final, &stored, &nlit, &ndist);
        if (st == PNGB200_OK && type != 0) st = build_block_tables(&sh, r, nlit, ndist, (int)lane, 32);
        if (st != PNGB200_OK) break;
        if (inside) {
            reparsed = br.at() - hdr_bit;
            br.seek(br.lead_bits + start_bit);
            inside = false;
        }
        if (type == 0) {
            // Stream.readBlock(upTo:), Stream.swift:384-399 -- byte-aligned copy
            if (!br.have(8 * (uint64_t)stored)) { st = PNGB200_NEED_MORE_INPUT; break; }
            if (out + stored > job.dst_cap) { st = fail(r, PNGB200_ERR_OUTPUT_CAPACITY); break; }
            const uint8_t* s = job.src + (br.at() >> 3);
            for (uint32_t k = lane; k < stored; k += 32) dst[out + k] = s[k];
            out += stored;
            br.seek(br.pos + 8 * (uint64_t)stored);
            __syncwarp();
        } else {
            // Stream.readBlock(with:), Stream.swift:266-381
            uint64_t sym_bit = br.at();   // the symbol being decoded starts here
            for (;;) {
                sym_bit = br.at();
                br.refill();
                uint32_t e   = lookup<LIT_ROOT>(sh.lit, br.peek());
                uint32_t len = e_len(e), kind = e_kind(e);
                if (kind == K_LIT) {
                    if (!br.have(len)) { st = PNGB200_NEED_MORE_INPUT; break; }
                    if (out >= job.dst_cap) { st = fail(r, PNGB200_ERR_OUTPUT_CAPACITY); break; }
                    br.consume((int)len);
                    if (lane == 0) dst[out] = (uint8_t)e_value(e);
                    ++out;
                } else if (kind == K_BASE) {
                    uint64_t start = br.pos;
                    br.consume((int)len);
                    uint32_t run = e_value(e) + br.take((int)e_extra(e));
                    br.refill();
                    uint32_t d = lookup<DIST_ROOT>(sh.dist, br.peek());
                    if (e_kind(d) != K_BASE) {
                        // beyond the end the zero padding decodes as *something*: the reference
                        // reports "need more input" before looking at validity
                        if (start + len + e_extra(e) + e_len(d) > br.total_bits) st = PNGB200_NEED_MORE_INPUT;
                        else st = fail(r, PNGB200_ERR_INVALID_SYMBOL, e_value(d), 1);
                        break;
                    }
                    br.consume((int)e_len(d));
                    uint32_t offset = e_value(d) + br.take((int)e_extra(d));
                    if (br.pos > br.total_bits) { st = PNGB200_NEED_MORE_INPUT; break; }
                    if (offset > out) { st = fail(r, PNGB200_ERR_STRING_REFERENCE); break; }
                    if (out + run > job.dst_cap) { st = fail(r, PNGB200_ERR_OUTPUT_CAPACITY); break; }
                    __syncwarp();
                    // InflatorOut.expand: forward copy; an overlapping copy repeats the last
                    // `offset` bytes, so byte k comes from (k mod offset) of the existing tail
                    const uint8_t* from = dst + out - offset;
                    for (uint32_t k = lane; k < run; k += 32) dst[out + k] = from[offset >= run ? k : k % offset];
                    out += run;
                    __syncwarp();
                } else if (kind == K_EOB) {
                    if (!br.have(len)) { st = PNGB200_NEED_MORE_INPUT; break; }
                    br.consume((int)len);
                    break;
                } else {
                    if (!br.have(len ? len : 1)) st = PNGB200_NEED_MORE_INPUT;
                    else st = fail(r, PNGB200_ERR_INVALID_SYMBOL, e_value(e), 0);
                    break;
                }
            }
            if (st == PNGB200_NEED_MORE_INPUT && job.resume) {
                // stop at the last complete symbol: `out` holds exactly the bytes of the symbols before sym_bit
                resume_bit = sym_bit;
                resume_out = out;
                phase      = 3;
                br.seek(br.lead_bits + sym_bit);
            }
            if (st != PNGB200_OK) break;
        }
        ++blocks;
        resume_bit = br.at();
        resume_out = out;
        phase = 1;
        if (final) {
            phase = 2;
            st = read_trailer(br, job.format, r);
            break;
        }
    }
    if (lane == 0) {
        if (r->status == 0) r->status = st;
        r->produced      = out;
        r->consumed_bits = br.at();
        r->blocks        = blocks;
        r->resume_bit    = resume_bit;
        r->resume_out    = resume_out;
        r->phase         = phase;
        if (job.resume) {
            if (phase == 3) *job.resume = ResumePoint{hdr_bit, resume_bit, resume_out, (uint32_t)final, 0,
                                                      job.resume->bits, job.resume->bytes, job.resume->serial_bytes};
            const uint64_t to = br.at() < br.size() ? br.at() : br.size();
            job.resume->bits += reparsed + (to > start_bit ? to - start_bit : 0);
            job.resume->bytes += out - start_out;
            job.resume->serial_bytes += out - start_out;
        }
    }
}

__global__ void __launch_bounds__(32) inflate_serial_kernel(const StreamJob* jobs, StreamResult* results,
                                                            const uint32_t* order, int count)
{
    __shared__ SerialShared sh;
    if ((int)blockIdx.x >= count) return;
    const int j = order ? (int)order[blockIdx.x] : (int)blockIdx.x;
    const StreamJob job = jobs[j];
    serial_inflate(sh, job, results + j, job.start_bit, job.start_out, (uint32_t)job.phase, 0,
                   job.phase == 3 ? job.resume->header_bit : 0);
}

}  // namespace pngb200
