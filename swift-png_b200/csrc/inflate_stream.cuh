// inflate_stream.cuh -- what the three wave kernels (inflate_wave.cuh, inflate_cells.cuh, inflate_parallel.cuh) share:
// the PTX wrappers, the bit reader and token decoder of the wave phases, the block-header parsers, the running
// Adler-32 and the stream driver around the LZ77 half of each kernel.
#pragma once

#include "inflate_serial.cuh"

namespace pngb200 {

constexpr int      WV_THREADS      = 256;
constexpr int      WV_WARPS        = WV_THREADS / 32;
constexpr uint32_t WV_SUB_BITS     = 256;
constexpr uint32_t WV_BITS         = WV_THREADS * WV_SUB_BITS;          // 65536 bits per wave
constexpr uint32_t WV_WORDS        = WV_BITS / 32 + 8;                  // + look-ahead for the last token
constexpr uint32_t WV_SMEM_WORDS   = WV_WORDS + WV_WORDS / 8 + 1;
constexpr uint32_t WV_WINDOW       = 32768;                             // DEFLATE's largest distance
constexpr uint32_t WV_HDR_WORDS    = 192;                               // block header staging (<= 566 bytes)
constexpr uint32_t ADLER_MOD32     = 65521;
constexpr uint32_t WV_WALK_K       = 8;                                 // tokens per walk in round 0 (doubles)

// cost model instrumentation (emulator builds only): loop trips per thread and per warp (max over lanes)
#if defined(PNGB200_EMU) && defined(WV_PROFILE)
struct WvProfile { uint64_t thread_iters[8], warp_iters[8]; };
inline WvProfile& wv_profile() { static WvProfile p; return p; }
inline void wv_count(int phase, uint32_t iters)
{
    uint32_t m = iters;
    for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
    wv_profile().thread_iters[phase] += iters;
    if ((threadIdx.x & 31) == 0) wv_profile().warp_iters[phase] += m;
}
#define WV_COUNT(phase, iters) wv_count(phase, iters)
#else
#define WV_COUNT(phase, iters)
#endif

enum : uint32_t { PF_EOB = 1, PF_BAD = 2 };
// how a thread's walk ended
enum : uint32_t { WK_SYNC = 0, WK_END = 1, WK_EOB = 2, WK_BAD = 3, WK_OWN_EOB = 4, WK_OWN_BAD = 5, WK_RUNNING = 6 };

struct WvHeader {  // block header as parsed by warp 0, broadcast to the CTA
    int32_t  status, type, final, nlit, ndist;
    uint32_t stored;
    uint64_t pos;     // reader position after the header
};

struct WvParams {
    const StreamJob* jobs;
    StreamResult*    results;
    const uint32_t*  order;
    uint32_t*        ticket;       // global work counter (zeroed before launch)
    uint8_t*         scratch;      // per-CTA: deferred copy list + unresolved bitmap for oversized waves
    uint64_t         scratch_stride;
    uint64_t         bitmap_words; // size of the HBM bitmap of each CTA
    int              count;
    SwitchRecord*    switched = nullptr;   // per job, or null: where a job with may_switch left symbolic mode
};

struct CopyItem { uint32_t o; uint32_t run_dist; };  // run | (dist - 1) << 16; run == 0: empty slot

#ifdef PNGB200_EMU
typedef uintptr_t saddr_t;
inline uint32_t lds32(saddr_t addr) { return *(const uint32_t*)addr; }
inline uint32_t bfe32(uint32_t x, uint32_t pos, uint32_t len);
inline saddr_t smem_addr(const void* p) { return (uintptr_t)p; }
inline saddr_t opaque(saddr_t a) { return a; }
inline uint32_t bmsk(uint32_t pos, uint32_t width)   // PTX bmsk.clamp.b32: `width` one bits starting at bit `pos`
{
    pos &= 0xff; width &= 0xff;
    if (pos > 31 || width == 0) return 0;
    const uint32_t m = width >= 32 ? ~0u : (1u << width) - 1u;
    return m << pos;
}
inline uint32_t bfe32(uint32_t x, uint32_t pos, uint32_t len) { return pos > 31 ? 0 : (x >> pos) & bmsk(0, len); }
#else
typedef uint32_t saddr_t;
__device__ __forceinline__ uint32_t lds32(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t bmsk(uint32_t pos, uint32_t width)   // `width` one bits starting at bit `pos`
{
    uint32_t r;
    asm("bmsk.clamp.b32 %0, %1, %2;" : "=r"(r) : "r"(pos), "r"(width));
    return r;
}
// bits [pos, pos + len) of x (pos <= 31).  sm_90 has no BFE instruction (ptxas expands bfe.u32 into several);
// shift + BMSK + AND is three
__device__ __forceinline__ uint32_t bfe32(uint32_t x, uint32_t pos, uint32_t len)
{
    return (x >> pos) & bmsk(0, len);
}
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// a value the compiler cannot rematerialise: it stays in a register (a shared-window address is otherwise rebuilt from
// SR_CgaCtaId wherever registers are short -- an S2R at the top of a decode loop, ncu r02)
__device__ __forceinline__ uint32_t opaque(uint32_t a)
{
    asm volatile("" : "+r"(a));
    return a;
}
#endif

// ---- bulk asynchronous copy (TMA, 1-D) global -> shared memory, completion on an mbarrier ----
// The next wave's 8 KiB of compressed words are fetched by the copy engine while this wave is still being emitted,
// resolved and stored: the HBM round trip of the stage phase (8.4 K cycles per wave, round-2 counters) leaves the
// critical path.  One elected thread issues, everybody waits on the mbarrier's phase parity.
#ifdef PNGB200_EMU
inline void mbar_init(uint64_t*, uint32_t) {}
inline void mbar_expect_tx(uint64_t*, uint32_t) {}
inline void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t*) { memcpy(dst, src, bytes); }
inline bool mbar_try_wait(uint64_t*, uint32_t) { return true; }
inline void fence_proxy_async() {}
inline void bulk_prefetch_l2(const void*, uint32_t) {}
#else
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     (uint32_t)__cvta_generic_to_shared(dst)),
                 "l"(src), "r"(bytes), "r"((uint32_t)__cvta_generic_to_shared(bar))
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok)
                 : "r"((uint32_t)__cvta_generic_to_shared(bar)), "r"(parity)
                 : "memory");
    return ok != 0;
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// bulk prefetch of `bytes` (multiple of 16, 16-byte aligned) into L2: one instruction for the copy engine, no completion to wait for
__device__ __forceinline__ void bulk_prefetch_l2(const void* src, uint32_t bytes)
{
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(src), "r"(bytes) : "memory");
}
#endif
constexpr uint32_t WV_PF_WORDS = WV_WORDS + 4;   // prefetched words: the wave + up to 3 words of 16-byte alignment slack

// register look-ahead bit reader over the staged (padded) words
struct FastBits {
    saddr_t  wbase;     // shared-memory address of the staged words
    uint32_t wi;        // next word to fetch
    uint32_t cur, nxt;
    uint32_t off;       // < 32 at every peek
    uint32_t pos;
    __device__ __forceinline__ void init(saddr_t words_addr, uint32_t start)
    {
        wbase = words_addr;
        const uint32_t W = start >> 5;
        cur = lds32(wbase + ((W + (W >> 3)) << 2));
        nxt = lds32(wbase + ((W + 1 + ((W + 1) >> 3)) << 2));
        wi  = W + 2;
        off = start & 31;
        pos = start;
    }
    __device__ __forceinline__ uint32_t peek() const { return __funnelshift_r(cur, nxt, off); }
    __device__ __forceinline__ void skip(uint32_t n)  // n <= 32
    {
        off += n;
        pos += n;
        if (off >= 32) {
            cur = nxt;
            nxt = lds32(wbase + ((wi + (wi >> 3)) << 2));
            ++wi;
            off -= 32;
        }
    }
};

// one table lookup of the decode passes: root entry, subtable entry behind a pointer (rare)
template <int ROOT>
__device__ __forceinline__ uint32_t fast_lookup(saddr_t table_addr, uint32_t bits)
{
    uint32_t e = lds32(table_addr + ((bits & ((1u << ROOT) - 1u)) << 2));
    if ((e & (E_SPECIAL | E_PTR | E_INVALID)) == (E_SPECIAL | E_PTR))
        e = lds32(table_addr + (((e >> 16) + bfe32(bits, ROOT, e_skip(e) - ROOT)) << 2));
    return e;
}

// Decode one token at the reader's position.  Literal and copy tokens run through ONE predicated
// body: in a warp some lanes always hold a literal while others hold a copy, so two divergent paths
// would cost their sum every iteration.  Returns 0, PF_EOB (consumed) or PF_BAD (reader not advanced
// past the offending code).  `run`: bytes the token produces; `dist`: 0 for a literal (then `lit_byte`
// is the byte), else the LZ77 distance (only computed when WANT_DIST).
template <bool WANT_DIST>
__device__ __forceinline__ uint32_t wv_decode(FastBits& b, saddr_t lit, saddr_t dst, uint32_t& run, uint32_t& dist,
                                              uint32_t& is_copy)
{
    const uint32_t bits = b.peek();
    const uint32_t e = fast_lookup<LIT_ROOT>(lit, bits);
    if (e & E_SPECIAL) {  // end of block, or an invalid code: rare, leave the loop
        if (e & E_INVALID) return PF_BAD;
        b.skip(e_len(e));
        return PF_EOB;
    }
    const uint32_t len = e & 15u, skipn = (e >> 4) & 31u;
    run = (e >> 16) + bfe32(bits, len, skipn - len);  // literals: width 0, value = the byte
    b.skip(skipn);
    is_copy = (e >> 9) & 1u;
    const uint32_t dbits = b.peek();
    const uint32_t d = fast_lookup<DIST_ROOT>(dst, dbits);  // ignored for literals
    if (is_copy && (d & E_SPECIAL)) return PF_BAD;
    const uint32_t dlen = d & 15u, dskip = (d >> 4) & 31u;
    if (WANT_DIST) dist = (d >> 16) + bfe32(dbits, dlen, dskip - dlen);
    b.skip(is_copy ? dskip : 0u);
    return 0;
}

// Block headers are parsed out of a shared-memory copy of the next 768 bytes of the stream (a
// dynamic header is at most 566 bytes), same interface as BitReader.
struct StagedReader {
    const uint32_t* w;
    uint64_t        base_bit, total_bits, pos;
    uint32_t        wi;
    uint64_t        buf;
    int             cnt;
    __device__ void init(const uint32_t* words, uint64_t base, uint64_t total, uint64_t p)
    {
        w = words; base_bit = base; total_bits = total;
        seek(p);
    }
    __device__ void seek(uint64_t p)
    {
        pos = p;
        wi  = (uint32_t)((p - base_bit) >> 5);
        buf = 0;
        cnt = 0;
        refill();
        int skip = (int)(p & 31);
        buf >>= skip;
        cnt -= skip;
    }
    __device__ __forceinline__ void refill()
    {
        while (cnt <= 32) {
            buf |= (uint64_t)(wi < WV_HDR_WORDS ? w[wi] : 0u) << cnt;
            cnt += 32;
            ++wi;
        }
    }
    __device__ __forceinline__ uint32_t peek() const { return (uint32_t)buf; }
    __device__ __forceinline__ void consume(int n) { buf >>= n; cnt -= n; pos += n; }
    __device__ __forceinline__ uint32_t take(int n)
    {
        uint32_t v = (uint32_t)buf & (n >= 32 ? ~0u : ((1u << n) - 1u));
        consume(n);
        return v;
    }
    __device__ __forceinline__ bool have(uint64_t n) const { return pos + n <= total_bits; }
};

// ---- unresolved-byte bitmap (bit i = output byte i of the wave is not final yet) ----
__device__ __forceinline__ uint32_t bit_mask(uint32_t lo, uint32_t hi)  // bits [lo, hi) of a word, hi <= 32
{
    return (hi >= 32 ? ~0u : ((1u << hi) - 1u)) & ~((1u << lo) - 1u);
}

// Block header, fast path (warp 0): a valid header that lies completely inside the input.  The
// code-length-code lengths are picked out lane-parallel, the code lengths themselves are decoded by
// lane 0 with a register bit buffer over the staged words (this loop is the serial part of every
// block: ~100 cycles per symbol instead of ~250 for the lock-step general parser).  Anything irregular
// -- block type 3, a bad count, an invalid code-length code, a repeat without a predecessor, too many
// lengths, truncation -- returns false and the caller runs parse_block_header, which owns the exact
// error semantics of the reference (Stream.readBlockMetadata / readBlockTables,
// LZ77.InflatorBuffers.Stream.swift:59-263).
template <class Shared>
__device__ bool wv_fast_header(Shared& sh, uint64_t hbase_bit, uint64_t pos, uint64_t total_bits, int lane, WvHeader& out)
{
    const uint32_t* const W = sh.words;
    auto get = [&](uint32_t rel, uint32_t n) -> uint32_t {   // n <= 32 bits at staged bit `rel`
        const uint32_t w = rel >> 5;
        const uint32_t v = __funnelshift_r(W[w], W[w + 1], rel & 31u);
        return n >= 32 ? v : v & ((1u << n) - 1u);
    };
    uint32_t rel = (uint32_t)(pos - hbase_bit);
    if (pos + 3 > total_bits) return false;
    const uint32_t h3 = get(rel, 3);
    rel += 3;
    out.status = PNGB200_OK;
    out.final = (int32_t)(h3 & 1u);
    out.type = (int32_t)(h3 >> 1);
    out.stored = 0;
    out.nlit = out.ndist = 0;
    if (out.type == 3) return false;
    if (out.type == 0) {
        const uint64_t boundary = (pos + 3 + 7) & ~(uint64_t)7;
        if (boundary + 32 > total_bits) return false;
        const uint32_t v = get((uint32_t)(boundary - hbase_bit), 32);
        const uint32_t l = v & 0xffffu, m = v >> 16;
        if (l != (~m & 0xffffu)) return false;
        out.stored = l;
        out.pos = boundary + 32;
        return true;
    }
    uint8_t* const lens = sh.ser.lens;
    if (out.type == 1) {
        for (int k = lane; k < 320; k += 32) lens[k] = k < 144 ? 8 : k < 256 ? 9 : k < 280 ? 7 : k < 288 ? 8 : 5;
        out.nlit = 288;
        out.ndist = 32;
        out.pos = pos + 3;
        __syncwarp();
        return true;
    }
    if (pos + 17 > total_bits) return false;
    const uint32_t v = get(rel, 14);
    rel += 14;
    const int nlit = 257 + (int)(v & 31u), ndist = 1 + (int)((v >> 5) & 31u), nclen = 4 + (int)(v >> 10);
    if (nlit > 286) return false;
    if (lane < 19) lens[lane] = 0;
    __syncwarp();
    if (lane < nclen) lens[c_clen_order[lane]] = (uint8_t)get(rel + 3u * (uint32_t)lane, 3);
    rel += 3u * (uint32_t)nclen;
    __syncwarp();
    build_table<META_ROOT, META_CAP>(sh.ser.meta, lens, 19, ALPHA_META, &sh.ser.scratch, lane, 32);
    if (sh.ser.scratch.status) return false;
    __syncwarp();
    uint32_t ok = 1, end_rel = 0;
    if (lane == 0) {
        const uint32_t* const meta = sh.ser.meta;
        uint32_t wi  = rel >> 5;
        uint64_t buf = ((uint64_t)W[wi + 1] << 32 | W[wi]) >> (rel & 31u);
        int      cnt = 64 - (int)(rel & 31u);
        wi += 2;
        const int total = nlit + ndist;
        int       have = 0;
        uint32_t  prev = 0;
        while (have < total) {
            if (cnt < 32) {
                buf |= (uint64_t)(wi < WV_HDR_WORDS ? W[wi] : 0u) << cnt;
                cnt += 32;
                ++wi;
            }
            const uint32_t e = meta[(uint32_t)buf & (META_CAP - 1)];
            if (e & E_SPECIAL) { ok = 0; break; }
            const uint32_t len = e & 15u, sym = e >> 16;
            buf >>= len;
            cnt -= (int)len;
            if (sym < 16) {
                lens[have++] = (uint8_t)sym;
                prev = sym;
                continue;
            }
            uint32_t element, extra, base;
            if (sym == 16) {
                if (have == 0) { ok = 0; break; }
                element = prev; extra = 2; base = 3;
            } else if (sym == 17) {
                element = 0; extra = 3; base = 3;
            } else {
                element = 0; extra = 7; base = 11;
            }
            const int reps = (int)(base + ((uint32_t)buf & ((1u << extra) - 1u)));
            buf >>= extra;
            cnt -= (int)extra;
            if (have + reps > total) { ok = 0; break; }
            for (int k = 0; k < reps; ++k) lens[have + k] = (uint8_t)element;
            prev = element;
            have += reps;
        }
        end_rel = (wi << 5) - (uint32_t)cnt;
    }
    ok = __shfl_sync(0xffffffffu, ok, 0);
    end_rel = __shfl_sync(0xffffffffu, end_rel, 0);
    if (!ok || hbase_bit + end_rel > total_bits) return false;
    out.nlit = nlit;
    out.ndist = ndist;
    out.pos = hbase_bit + end_rel;
    __syncwarp();
    return true;
}

// Adler-32 partial sums of bytes [0, n) at `p` for a piece whose first byte has weight `wt` (weights
// fall by one per byte): a += sum b, bw += sum (wt - i) b_i.  64-bit accumulators, any alignment.
__device__ __forceinline__ void adler_bytes(const uint8_t* p, uint64_t n, uint64_t wt, uint64_t& a, uint64_t& bw)
{
    for (uint64_t i = 0; i < n; ++i) {
        a += p[i];
        bw += (wt - i) * p[i];
    }
}
// the same with 32-bit accumulators: enough for one thread's chunks of a wave that fits the shared-memory image
// (<= 9 chunks x weight <= 32784 x byte sum <= 4080 < 2^31)
__device__ __forceinline__ void adler_chunk16_u32(uint4 x, uint32_t wt, uint32_t& a, uint32_t& bw)
{
    const uint32_t s = __vsadu4(x.x, 0) + __vsadu4(x.y, 0) + __vsadu4(x.z, 0) + __vsadu4(x.w, 0);
    const uint32_t wsum = __dp4a(x.x, 0x03020100u, 0u) + __dp4a(x.y, 0x07060504u, 0u) +
                          __dp4a(x.z, 0x0b0a0908u, 0u) + __dp4a(x.w, 0x0f0e0d0cu, 0u);
    a += s;
    bw += wt * s - wsum;
}
__device__ __forceinline__ void adler_chunk16(uint4 x, uint64_t wt, uint64_t& a, uint64_t& bw)
{
    const uint32_t s = __vsadu4(x.x, 0) + __vsadu4(x.y, 0) + __vsadu4(x.z, 0) + __vsadu4(x.w, 0);
    // sum (wt - i) b_i = wt * s - sum i * b_i
    const uint32_t wsum = __dp4a(x.x, 0x03020100u, 0u) + __dp4a(x.y, 0x07060504u, 0u) +
                          __dp4a(x.z, 0x0b0a0908u, 0u) + __dp4a(x.w, 0x0f0e0d0cu, 0u);
    a += s;
    bw += wt * s - wsum;
}

// ==== the stream driver of the wave kernels ====
// Each kernel keeps its own shared-memory layout (`Shared`); the pieces below use its members ser, words[], hdr,
// anomaly, ticket, cyc[12], tick, warp_sums[WV_WARPS + 1] and adler_a / adler_b[WV_WARPS], and the wave front end
// further down also mask[], pf_bar, exc[], valid[], next_[], kind_[], last and term.

// Claims the CTA's next stream and resets its anomaly flag and phase timers.  Returns the job index, -1 once the
// batch is done.  Every thread calls it.
template <class Shared>
__device__ __forceinline__ int next_stream(Shared& sh, const WvParams& P)
{
    __syncthreads();
    if (threadIdx.x == 0) {
        sh.ticket = atomicAdd(P.ticket, 1u);
        sh.anomaly = 0;
        for (int k = 0; k < 12; ++k) sh.cyc[k] = 0;
        sh.tick = (uint64_t)clock64();
    }
    __syncthreads();
    if (sh.ticket >= (uint32_t)P.count) return -1;
    return P.order ? (int)P.order[sh.ticket] : (int)sh.ticket;
}

// phase timer: thread 0 charges the cycles since the last tick to phase `i` (StreamResult.stat_cycles)
template <class Shared>
__device__ __forceinline__ void phase_tick(Shared& sh, int i)
{
    if (threadIdx.x == 0) {
        const uint64_t now = (uint64_t)clock64();
        sh.cyc[i] += now - sh.tick;
        sh.tick = now;
    }
}

// Running Adler-32 of a stream decoded from its first byte, folded piece by piece (a stored block, a wave) from the
// per-warp partial sums the piece leaves in sh.adler_a / adler_b: no second pass over the inflated bytes.  Only
// thread 0's copy is meaningful; it lives in registers or in shared memory, as the kernel declares it.
struct AdlerRun {
    uint64_t pend_len;   // bytes of the piece whose partial sums wait in sh.adler_* (pend != 0)
    uint32_t s1, s2, pend;
    __device__ __forceinline__ void reset()
    {
        s1 = 1;
        s2 = 0;
        pend = 0;
    }
    // fold the pending piece into (s1, s2): every thread calls it right after a barrier
    template <class Shared>
    __device__ __forceinline__ void fold(const Shared& sh)
    {
        if (threadIdx.x == 0 && pend) {
            uint64_t A = 0, B = 0;
            for (int w = 0; w < WV_WARPS; ++w) { A += sh.adler_a[w]; B += sh.adler_b[w]; }
            s2 = (uint32_t)((s2 + (pend_len % ADLER_MOD32) * s1 + B) % ADLER_MOD32);
            s1 = (uint32_t)((s1 + A) % ADLER_MOD32);
            pend = 0;
        }
    }
    // a piece of `n` bytes whose partial sums (a, bw), see adler_bytes, every thread holds for its part: warp sums
    // into sh.adler_*, folded after the next barrier
    template <class Shared>
    __device__ __forceinline__ void piece_from_partials(Shared& sh, uint32_t a, uint32_t bw, uint64_t n)
    {
        for (int o = 16; o; o >>= 1) {
            a += __shfl_down_sync(0xffffffffu, a, o);
            bw += __shfl_down_sync(0xffffffffu, bw, o);
        }
        if (lane_id() == 0) { sh.adler_a[threadIdx.x >> 5] = a; sh.adler_b[threadIdx.x >> 5] = bw; }
        if (threadIdx.x == 0) { pend = 1; pend_len = n; }
    }
    // a finished piece of `n` bytes at HBM address `p` (stored blocks, waves written to HBM directly): every thread
    // sums its share
    template <class Shared>
    __device__ __forceinline__ void piece_from_hbm(Shared& sh, const uint8_t* p, uint64_t n)
    {
        uint64_t a = 0, bw = 0;
        const uint64_t per = (n + WV_THREADS - 1) / WV_THREADS;
        const uint64_t lo = min((uint64_t)threadIdx.x * per, n), hi = min(lo + per, n);
        adler_bytes(p + lo, hi - lo, n - lo, a, bw);
        piece_from_partials(sh, (uint32_t)(a % ADLER_MOD32), (uint32_t)(bw % ADLER_MOD32), n);
    }
    // LZ77.InflatorBuffers.advance(.checksum): compare with the trailer (InflatorBuffers.swift:109-130).  Thread 0.
    __device__ __forceinline__ void check_trailer(StreamResult* r, int32_t format) const
    {
        if (format == PNGB200_FORMAT_GZIP) return;
        const uint32_t computed = s2 << 16 | s1;
        r->checksum = computed;
        r->ck_done  = 1;
        if (r->trailer_seen && format != PNGB200_FORMAT_IOS && r->status >= 0 && r->declared != computed) {
            r->status = PNGB200_ERR_STREAM_CHECKSUM;
            r->err_a  = r->declared;
            r->err_b  = computed;
        }
    }
};

// One stream as a CTA decodes it: the reader, where the output and the resume point stand, and the status.  The block
// loops of the ring and cell kernels advance it; open(), end_block(), copy_stored() and finish() are the parts of those
// loops they share.  (The round-1 kernel keeps these parts inline: as a struct they cost its 64-register build spills.)
struct StreamRun {
    StreamJob     job;
    StreamResult* r;
    BitReader     br;
    uint64_t      out, resume_bit, resume_out;
    uint32_t      blocks, phase;
    int           st;
    bool          fallback;   // the serial decoder redoes the stream from the resume point
    // With a resume record (job.resume), thread 0 keeps the block being decoded there: its header, and the last wave
    // checkpoint inside it (symbol_bit, out; symbol_bit = 0: none yet), where the serial decoder takes over.  The
    // checkpoints live in the record rather than in registers, which the ring kernel has none to spare of.

    // job `j` of the batch: its stream header, or its trailer when the job starts there
    __device__ __forceinline__ void open(const WvParams& P, int j)
    {
        job = P.jobs[j];
        r   = P.results + j;
        br.init(job.src, job.src_len, job.start_bit);
        out        = job.start_out;
        resume_bit = job.start_bit;
        resume_out = job.start_out;
        blocks     = 0;
        phase      = (uint32_t)job.phase;
        st         = PNGB200_OK;
        fallback   = false;
        if (phase == 3) {
            // inside a Huffman block: its header is parsed again (begin_block), then the first wave starts at start_bit
            br.seek(br.lead_bits + job.resume->header_bit);
            phase = 1;
        }
        if (phase == 0) {
            st = read_stream_header(br, job.format, r);
            if (st == PNGB200_OK) {
                resume_bit = br.at();
                phase = 1;
            }
        }
        if (st == PNGB200_OK && phase == 2) st = read_trailer(br, job.format, r);
    }

    // The header of a Huffman block, parsed at `hdr` (reader space), ends at the reader.  Every thread calls it; when the
    // job resumes inside this block, the reader moves on to the resume symbol, and the header bits count as decoded.
    __device__ __forceinline__ void begin_block(uint64_t hdr, int final)
    {
        if (!job.resume) return;
        const bool resumed = job.phase == 3 && blocks == 0;
        if (threadIdx.x == 0) {
            job.resume->header_bit = hdr - br.lead_bits;
            job.resume->final = (uint32_t)final;
            if (resumed) job.resume->bits = br.pos - hdr;
            else job.resume->symbol_bit = 0;
        }
        if (resumed) br.seek(br.lead_bits + job.start_bit);
    }
    // A wave of the current Huffman block ended at the reader, on a symbol boundary, with `out` bytes decoded
    __device__ __forceinline__ void wave_done()
    {
        if (threadIdx.x == 0 && job.resume) {
            job.resume->symbol_bit = br.at();
            job.resume->out = out;
        }
    }
    // The wave that starts at the reader cannot be decoded here: the serial decoder takes over.  The wave counts as
    // decoded up to the end of the input.
    __device__ __forceinline__ void fall_back()
    {
        fallback = true;
        if (threadIdx.x == 0 && job.resume) job.resume->bits += min(br.at() + WV_BITS, br.size()) - job.start_bit;
    }

    // After a block: the resume point moves behind it.  True when the block loop ends there: at the end of a
    // segment, or after the final block (then the trailer is read).
    __device__ __forceinline__ bool end_block(bool final)
    {
        ++blocks;
        resume_bit = br.at();
        resume_out = out;
        if (job.stop_bit && !final && br.at() >= job.stop_bit) return true;   // end of my segment (the host checks ==)
        if (final) {
            phase = 2;
            st = read_trailer(br, job.format, r);
            return true;
        }
        return false;
    }

    // A stored block of `stored` bytes at the reader (which is past its header): copied to dst as bytes, or as 16-bit
    // symbols for a segment, and taken into the running Adler-32.  Every thread calls it; false: st holds the error.
    template <class Shared>
    __device__ __forceinline__ bool copy_stored(Shared& sh, uint8_t* dst, uint64_t dst_cap, bool sym, uint32_t stored,
                                                AdlerRun& adler, bool adler_on)
    {
        if (!br.have(8 * (uint64_t)stored)) { st = PNGB200_NEED_MORE_INPUT; return false; }
        if (out + stored > dst_cap) { st = fail(r, PNGB200_ERR_OUTPUT_CAPACITY); return false; }
        const uint8_t* s = job.src + (br.at() >> 3);
        if (sym) for (uint32_t k = threadIdx.x; k < stored; k += WV_THREADS) reinterpret_cast<uint16_t*>(dst)[out + k] = s[k];
        else for (uint32_t k = threadIdx.x; k < stored; k += WV_THREADS) dst[out + k] = s[k];
        if (adler_on && stored) adler.piece_from_hbm(sh, s, stored);
        out += stored;
        br.seek(br.pos + 8 * (uint64_t)stored);
        __syncthreads();
        adler.fold(sh);
        return true;
    }

    // The end of the stream, every thread: the last Adler-32 fold, the kernel's statistics (`stats`, called by every
    // thread; sh.adler_* and sh.warp_sums are free again), then the result record.  A segment that fell back reports
    // `seg_status` (a segment cannot go through the byte-wise serial decoder: the host decodes the stream whole);
    // any other fallback hands the stream to the serial decoder, which owns the result record.
    template <class Shared, class Stats>
    __device__ __forceinline__ void finish(Shared& sh, AdlerRun& adler, bool adler_on, int seg_status, Stats&& stats)
    {
        __syncthreads();
        adler.fold(sh);
        __syncthreads();   // thread 0 has read the last piece's sums before the statistics reuse sh.adler_*
        stats();
        const uint32_t t = threadIdx.x;
        if (fallback && job.symbolic) {
            if (t == 0) {
                r->status = seg_status;
                r->produced = out;
                r->consumed_bits = br.at();
                r->blocks = blocks;
            }
        } else if (fallback) {
            if (t == 0 && job.resume) job.resume->bytes = out - job.start_out;
            __syncthreads();
            // with a resume record, from the last wave checkpoint of the block: at most one wave is decoded again
            if (t < 32) {
                const ResumePoint at = job.resume ? *job.resume : ResumePoint{};
                const bool mid = at.symbol_bit != 0;
                serial_inflate(sh.ser, job, r, mid ? at.symbol_bit : resume_bit, mid ? at.out : resume_out, mid ? 3 : 1,
                               blocks, at.header_bit);
            }
        } else if (t == 0) {
            if (r->status == 0) r->status = st;
            r->produced      = out;
            r->consumed_bits = br.at();
            r->blocks        = blocks;
            r->resume_bit    = resume_bit;
            r->resume_out    = resume_out;
            r->phase         = phase;
            if (adler_on) adler.check_trailer(r, job.format);
            if (job.resume) {
                job.resume->bits += br.at() - job.start_bit;
                job.resume->bytes = out - job.start_out;
            }
        }
        if (t == 0) r->stat_fallback = fallback ? 1u : 0u;
    }
};

// Per-stream statistics of the ring and cell kernels (the reference's -DDUMP_LZ77_BLOCKS style counters): CTA sums of
// each thread's `tokens`, `deferred` and `walk_tokens` (the last two clamped to 32 bits per warp), the largest
// `rounds`.  Every thread calls it; thread 0 writes them.
template <class Shared>
__device__ __forceinline__ void report_wave_stats(Shared& sh, StreamResult* r, uint32_t waves, uint64_t matches, uint64_t tokens,
                                                  uint64_t deferred, uint64_t walk_tokens, uint32_t rounds)
{
    const unsigned warp = threadIdx.x >> 5;
    for (int o = 16; o; o >>= 1) {
        tokens += __shfl_down_sync(0xffffffffu, tokens, o);
        deferred += __shfl_down_sync(0xffffffffu, deferred, o);
        walk_tokens += __shfl_down_sync(0xffffffffu, walk_tokens, o);
        rounds = max(rounds, __shfl_down_sync(0xffffffffu, rounds, o));
    }
    if (lane_id() == 0) {
        sh.warp_sums[warp] = tokens;
        sh.adler_a[warp] = (uint32_t)min(deferred, (uint64_t)0xffffffffu);
        sh.adler_b[warp] = (uint32_t)min(walk_tokens, (uint64_t)0xffffffffu);
        sh.exc[warp] = rounds;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t tk = 0, df = 0, wt = 0;
        uint32_t rr = 0;
        for (int w = 0; w < WV_WARPS; ++w) {
            tk += sh.warp_sums[w];
            df += sh.adler_a[w];
            wt += sh.adler_b[w];
            rr = max(rr, sh.exc[w]);
        }
        r->stat_waves          = waves;
        r->stat_sync_rounds    = (uint32_t)min(wt, (uint64_t)0xffffffffu);   // tokens decoded by walks
        r->stat_resolve_rounds = rr;
        r->stat_tokens         = tk;
        r->stat_matches        = matches;
        r->stat_deferred       = df;
        for (int k = 0; k < 12; ++k) r->stat_cycles[k] = sh.cyc[k];
    }
}

// The general block-header parser over the words stage_header_words staged (warp 0); it owns the reference's error
// semantics (Stream.readBlockMetadata / readBlockTables, LZ77.InflatorBuffers.Stream.swift:59-263)
template <class Shared>
__device__ WvHeader general_block_header(Shared& sh, const BitReader& br, StreamResult* r)
{
    int      type = 0, final = 0, nlit = 0, ndist = 0;
    uint32_t stored = 0;
    StagedReader sr;
    sr.init(sh.words, (br.pos >> 5) << 5, br.total_bits, br.pos);
    const int st = parse_block_header(sr, &sh.ser, r, (int)lane_id(), &type, &final, &stored, &nlit, &ndist);
    return WvHeader{st, type, final, nlit, ndist, stored, sr.pos};
}

// the WV_HDR_WORDS words from the one that holds the reader's position, into sh.words; every thread, ends with a barrier
template <class Shared>
__device__ __forceinline__ void stage_header_words(Shared& sh, const BitReader& br)
{
    const uint64_t hbase = br.pos >> 5;
    for (uint32_t k = threadIdx.x; k < WV_HDR_WORDS; k += WV_THREADS) sh.words[k] = br.load_word(hbase + k);
    __syncthreads();
}

// The header of the block at the reader: warp 0 walks the header bits alone (the fast parser, the general one where
// that declines), the CTA then builds the tables together.  Every thread calls it and gets the header.
template <class Shared>
__device__ __forceinline__ WvHeader read_block_header(Shared& sh, const BitReader& br, StreamResult* r)
{
    stage_header_words(sh, br);
    if (threadIdx.x < 32) {
        WvHeader h;
        if (!wv_fast_header(sh, (br.pos >> 5) << 5, br.pos, br.total_bits, (int)lane_id(), h)) h = general_block_header(sh, br, r);
        if (lane_id() == 0) sh.hdr = h;
    }
    __syncthreads();
    return sh.hdr;
}

// CTA-wide exclusive scan of one packed count per thread (copies << 40 | bytes): returns the thread's exclusive prefix
// and leaves the wave's totals in sh.warp_sums[WV_WARPS].  Every thread calls it; two barriers.
template <class Shared>
__device__ __forceinline__ uint64_t cta_scan_packed(Shared& sh, uint64_t mine)
{
    const unsigned lane = lane_id(), warp = threadIdx.x >> 5;
    uint64_t incl = mine;
    for (int o = 1; o < 32; o <<= 1) {
        uint64_t v = __shfl_up_sync(0xffffffffu, incl, o);
        if ((int)lane >= o) incl += v;
    }
    if (lane == 31) sh.warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint64_t ws = lane < WV_WARPS ? sh.warp_sums[lane] : 0, wi = ws;
        for (int o = 1; o < 32; o <<= 1) {
            uint64_t v = __shfl_up_sync(0xffffffffu, wi, o);
            if ((int)lane >= o) wi += v;
        }
        if (lane < WV_WARPS) sh.warp_sums[lane] = wi - ws;        // exclusive
        if (lane == WV_WARPS - 1) sh.warp_sums[WV_WARPS] = wi;   // wave totals
    }
    __syncthreads();
    return sh.warp_sums[warp] + incl - mine;
}

// ==== the wave front end of the ring and cell kernels ====

// The next wave's words, fetched by the copy engine (bulk async copy) into the token maps' memory -- mask[] and what
// follows it, dead from the end of phase D until the next phase A -- while this wave is emitted, resolved and stored:
// the HBM round trip of the stage phase (8.4 K cycles per wave, round-2 counters) leaves the critical path.
struct WavePrefetch {
    uint32_t parity;    // phase of the mbarrier the next wait looks for
    bool     pending;   // a bulk prefetch is in flight / has landed
    uint64_t first;     // first word (reader space) of the prefetched range

    // wait until the prefetch, if one is in flight, has landed
    template <class Shared>
    __device__ __forceinline__ void drain(Shared& sh)
    {
        if (pending) {
            while (!mbar_try_wait(&sh.pf_bar, parity)) {}
            parity ^= 1;
            pending = false;
        }
    }
    // the words from `nbase` on, the predicted first staged word of the next wave; every thread calls it
    template <class Shared>
    __device__ __forceinline__ void start(Shared& sh, const BitReader& br, uint64_t nbase)
    {
        const uint64_t f = nbase - ((((uintptr_t)br.words >> 2) + nbase) & 3);   // 16-byte aligned address
        if (f >= 1 && (f + WV_PF_WORDS + 1) * 32 <= br.total_bits) {
            if (threadIdx.x == 0) {
                fence_proxy_async();   // the maps were read and written through the generic proxy
                mbar_expect_tx(&sh.pf_bar, sizeof(uint32_t) * WV_PF_WORDS);
                bulk_g2s(sh.mask, br.words + f, sizeof(uint32_t) * WV_PF_WORDS, &sh.pf_bar);
            }
            pending = true;
            first = f;
        }
    }
    // Stages the wave whose first staged word is `wbase` in sh.words (padded 9/8): the prefetched words when the
    // prediction held, else straight from the input.  Every thread calls it right after a barrier.  A prefetch in
    // flight is always waited for: its landing zone is about to become the token maps again.
    template <class Shared>
    __device__ __forceinline__ void stage(Shared& sh, const BitReader& br, uint64_t wbase)
    {
        const bool had = pending;
        drain(sh);
        if (had && wbase >= first && wbase - first < 4) {
            const uint32_t* lin = sh.mask + (uint32_t)(wbase - first);
            for (uint32_t k = threadIdx.x; k < WV_WORDS; k += WV_THREADS) sh.words[k + (k >> 3)] = lin[k];
        } else {
            for (uint32_t k = threadIdx.x; k < WV_WORDS; k += WV_THREADS) sh.words[k + (k >> 3)] = br.load_word(wbase + k);
        }
    }
};

// C. the true chain: the orbit of thread 0 under "t -> subsequence where t's walk joined".  Thread 0 follows it with
// the exception words (sh.exc: walks that did not simply join the next subsequence) in registers, one shared-memory
// load per such walk, and leaves the chain's members in sh.valid, its last thread in sh.last and how that thread's
// walk ended in sh.term.
template <class Shared>
__device__ __forceinline__ void follow_chain(Shared& sh)
{
    uint32_t E[WV_WARPS];
#pragma unroll
    for (int w = 0; w < WV_WARPS; ++w) E[w] = sh.exc[w];
    uint32_t cur = 0, x = 0;
    bool     done = false;
#pragma unroll
    for (int w = 0; w < WV_WARPS; ++w) {
        uint32_t v = 0;
        while (!done && cur < 32u * (w + 1)) {   // cur >= 32 w here
            const uint32_t lo = cur - 32u * w;
            const uint32_t m = E[w] & (~0u << lo);
            if (m == 0) {                        // the rest of this word joins its neighbour
                v |= ~0u << lo;
                cur = 32u * (w + 1);
                break;
            }
            const uint32_t b = (uint32_t)__ffs((int)m) - 1;
            x = 32u * w + b;
            v |= bit_mask(lo, b + 1);            // threads cur .. x are on the chain
            const uint32_t nx = sh.next_[x];
            if (nx == 0xffffu) done = true;      // thread 255 never joins anybody: always reached
            else cur = nx;                       // > x + 1: the walk crossed subsequences
        }
        sh.valid[w] = v;
    }
    sh.last = x;
    sh.term = sh.kind_[x];
}

// per-CTA HBM scratch of the ring and round-1 kernels: a copy list of `list_cap` items, then the unresolved bitmap of
// waves too big for shared memory
inline uint64_t wave_bitmap_words(uint64_t max_dst_cap, uint32_t list_cap)
{
    const uint64_t max_wave_out = (uint64_t)list_cap * 258;
    const uint64_t bytes = max_dst_cap < max_wave_out ? max_dst_cap : max_wave_out;
    return (bytes + 31) / 32 + 8;
}
inline uint64_t wave_scratch_stride(uint64_t bitmap_words, uint32_t list_cap)
{
    const uint64_t s = sizeof(CopyItem) * (uint64_t)list_cap + 4 * bitmap_words;
    return (s + 255) / 256 * 256;
}

}  // namespace pngb200
