// inflate_wave.cuh -- intra-stream parallel DEFLATE inflate, second generation ("chain walk").
//
// One CTA of 256 threads eats a DEFLATE block in WAVES of 256 subsequences x 256 bits (8 KiB of
// compressed data staged in shared memory, padded 9/8 so lane-strided word reads do not conflict).
// The last 32 KiB of output -- the LZ77 window -- and the wave's own output live in a 64 KiB RING in
// shared memory (index = stream offset mod 65536), so no token of a wave ever waits for HBM: literals,
// window copies and the unresolved-copy sweep are shared-memory traffic; HBM sees the compressed words
// once (coalesced) and the output once (16-byte coalesced stores out of the ring).
//
// DEFLATE has no sync markers, but Huffman codes self-synchronise: a decoder started at a wrong bit
// falls into step with the true token sequence after a few tokens (median 6, 1 % beyond 40 for PNG
// data).  Round 1 exploited that with CTA-wide re-decode rounds (3.2 decode passes per bit, ~20
// barriers per wave).  Here:
//
//   A. speculate  thread t decodes subsequence t from a guessed start (thread 0's is exact) until it
//                 leaves the subsequence.  It records a 256-bit map of the token start positions it
//                 visited, byte / copy counts at every 32-bit boundary of the map, and its exit position.
//   B. walk       a walk continues from each exit through the following subsequences until it lands on
//                 a position the owner of that subsequence also visited (from there on the two decodes
//                 are identical), or on end-of-block / the end of the wave.  Walk lengths are heavy
//                 tailed, so walks run in rounds of 8, 16, 32 ... tokens and the unfinished ones are
//                 compacted onto the lowest threads: a round costs what it still has to do.
//   C. chain      the true token chain is the orbit of thread 0 under "t -> subsequence where t's walk
//                 joined".  One thread follows it in registers, stepping only where a walk crossed a
//                 subsequence without joining.
//   D. count      a thread on the chain owns the tokens that START in its subsequence: from its
//                 predecessor's exit to its own exit.  Their byte / copy counts = the predecessor's walk
//                 + own totals - the garbage prefix (checkpoint + at most 31 bits decoded again);
//                 CTA scan -> output offsets and list slots.
//   E. emit       every thread decodes its share once more and writes it: literals into the ring; an
//                 LZ77 copy runs immediately when its source is final -- behind the wave (the window:
//                 in PNG the distance is about one scanline) or inside the thread's own finished bytes
//                 (distance of a pixel or two).  Only copies that read another thread's bytes of THIS
//                 wave are deferred to a list sorted by output offset, their destination bytes flagged
//                 in an "unresolved" bitmap.
//   F. resolve    barrier-free sweep of the deferred list (a copy runs once none of its source bytes
//                 is flagged; the smallest open item is always ready).
//   G. store      ring -> HBM with 16-byte coalesced stores; the Adler-32 of the wave is taken from
//                 the same registers (reassociated sums, folded per wave), so zlib streams need no
//                 separate checksum pass over the inflated bytes.
//
// Waves that expand beyond 32 KiB (flat graphics: 8 KiB -> megabytes) write HBM directly, read their
// sources from HBM and keep their bitmap in HBM scratch; the ring is refilled from HBM afterwards.
// Anything irregular (invalid symbol on the chain, truncation, output overflow, distance before the
// start of the output) is not handled here: warp 0 re-runs the block with the serial decoder
// (inflate_serial.cuh), which owns the exact error semantics of the reference.
//
// CTAs are persistent: each takes streams from an atomic ticket (the host orders streams longest
// first), so per-CTA scratch in HBM is bounded by the number of resident CTAs.
//
// Replaces the reference's serial token loop Stream.readBlock(with:) and InflatorOut.expand
// (Sources/LZ77/Inflator/LZ77.InflatorBuffers.Stream.swift:266-381, LZ77.InflatorOut.swift:124-140),
// the window of LZ77.InflatorOut (LZ77.InflatorOut.swift:86-110) and, for zlib streams, the running
// MRC32 (Sources/LZ77/Wrappers/LZ77.MRC32.swift:26-47).
#pragma once

#include "inflate_serial.cuh"

namespace pngb200 {

#ifndef WV_CTAS
#define WV_CTAS 2
#endif
constexpr int      WV_THREADS      = 256;
constexpr int      WV_CTAS_PER_SM  = WV_CTAS;
constexpr int      WV_WARPS        = WV_THREADS / 32;
constexpr uint32_t WV_SUB_BITS     = 256;
constexpr uint32_t WV_BITS         = WV_THREADS * WV_SUB_BITS;          // 65536 bits per wave
constexpr uint32_t WV_WORDS        = WV_BITS / 32 + 8;                  // + look-ahead for the last token
constexpr uint32_t WV_SMEM_WORDS   = WV_WORDS + WV_WORDS / 8 + 1;
constexpr uint32_t WV_RING         = 65536;                             // window + wave output (uint16 index wraps)
constexpr uint32_t WV_WINDOW       = 32768;                             // DEFLATE's largest distance
constexpr uint32_t WV_OUT_BYTES    = WV_RING - WV_WINDOW;               // largest wave the ring can take
constexpr uint32_t WV_BITMAP_WORDS = WV_OUT_BYTES / 32;
constexpr uint32_t WV_LIST_CAP     = WV_BITS / 2 + 64;                  // >= copies per wave (2 bits min each)
constexpr uint64_t WV_MAX_WAVE_OUT = (uint64_t)WV_LIST_CAP * 258;
constexpr uint32_t WV_HDR_WORDS    = 192;                               // block header staging (<= 566 bytes)
constexpr uint32_t ADLER_MOD32     = 65521;
#ifndef WV_POLL_NS
#define WV_POLL_NS 20
#endif
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

struct WvShared {
    SerialShared ser;
    uint32_t     words[WV_SMEM_WORDS];
    uint32_t     mask[8 * WV_THREADS];          // [k][t]: token starts in bits 32k .. 32k+31 of subsequence t
    uint32_t     ck[8 * WV_THREADS];            // [k][t]: bytes (low 16 bits) and copies produced by thread t's tokens that
                                                //         start before map word k (written for words that hold a start)
    uint32_t     exit_[WV_THREADS];             // where thread t's own decode left its subsequence
    uint32_t     wpos_[WV_THREADS];             // where thread t's walk is / ended (wave-relative bit)
    uint32_t     wn_[WV_THREADS];               // bytes produced by the walk
    uint64_t     cross_[WV_THREADS];            // where the walk first crossed into the subsequence after the one it
                                                // started in: 1 << 63 | position << 40 | copies << 24 | bytes (0: it did not)
    uint16_t     wc_[WV_THREADS];               // copies among the walk's tokens
    uint16_t     next_[WV_THREADS];             // subsequence the walk joined, 0xffff: the chain ends with thread t
    uint8_t      kind_[WV_THREADS];             // WK_*
    uint8_t      wlist[2][WV_THREADS];          // unfinished walks of a round, compacted
    uint16_t     dpre_[WV_THREADS];             // deferred copies of the threads below t (exclusive prefix)
    uint16_t     cst_[WV_THREADS];              // first list slot of thread t
    uint32_t     dsum[WV_WARPS];
    uint32_t     wcount[3];
    uint32_t     bitmap[WV_BITMAP_WORDS];
    uint8_t      ring[WV_RING] __align__(16);
    uint64_t     warp_sums[WV_WARPS + 1];
    uint32_t     adler_a[WV_WARPS], adler_b[WV_WARPS];
    uint32_t     exc[WV_WARPS], valid[WV_WARPS];
    uint32_t     mark[WV_WARPS];                // symbolic wave: 1 + the last wave offset holding a marker, per warp
    uint32_t     last, term, anomaly, ticket;
    uint64_t     cyc[12], tick;                 // phase timers (thread 0)
    uint64_t     pf_bar;                        // mbarrier of the bulk prefetch (lands in mask[] .. ck[], dead by then)
    WvHeader     hdr;
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
// set / clear / test the bits [o, o + run) (run >= 1): one or two words for run <= 32, the common case
__device__ __forceinline__ void bits_set(uint32_t* U, uint32_t o, uint32_t run)
{
    const uint32_t a = o & 31u;
    uint32_t*      w = U + (o >> 5);
    if (a + run <= 32u) { atomicOr(w, bmsk(a, run)); return; }
    atomicOr(w, ~0u << a);
    uint32_t rem = run - (32u - a);
    for (++w; rem >= 32u; ++w, rem -= 32u) atomicOr(w, ~0u);
    if (rem) atomicOr(w, bmsk(0, rem));
}
__device__ __forceinline__ void bits_clear(uint32_t* U, uint32_t o, uint32_t run)
{
    const uint32_t a = o & 31u;
    uint32_t*      w = U + (o >> 5);
    if (a + run <= 32u) { atomicAnd(w, ~bmsk(a, run)); return; }
    atomicAnd(w, ~(~0u << a));
    uint32_t rem = run - (32u - a);
    for (++w; rem >= 32u; ++w, rem -= 32u) atomicAnd(w, 0u);
    if (rem) atomicAnd(w, ~bmsk(0, rem));
}
__device__ __forceinline__ bool bits_all_clear(const uint32_t* U, uint32_t o, uint32_t run)
{
    const volatile uint32_t* w = U + (o >> 5);
    const uint32_t a = o & 31u;
    uint32_t any;
    if (a + run <= 32u) any = *w & bmsk(a, run);
    else {
        any = *w & (~0u << a);
        uint32_t rem = run - (32u - a);
        for (++w; rem >= 32u; ++w, rem -= 32u) any |= *w;
        if (rem) any |= *w & bmsk(0, rem);
    }
    __threadfence_block();
    return any == 0;
}

// One LZ77 copy inside the ring (d, s: ring positions of destination and source, taken mod 65536 per
// byte; the source is final or is produced by this very loop when the ranges overlap).
__device__ __forceinline__ void ring_copy(uint8_t* ring, uint32_t d, uint32_t s, uint32_t run, uint32_t dist)
{
    d &= 0xffffu;
    s &= 0xffffu;
    if (dist >= 4 && max(d, s) + run + 3 < WV_RING) {
        // four bytes per step: byte k+3 reads k+3-dist < k, so the loads of a step never depend on its stores;
        // the loads may run up to 3 bytes past the run (still inside the ring), the stores may not
        const uint8_t* sp = ring + s;
        uint8_t*       dp = ring + d;
        for (uint32_t k = 0; k < run; k += 4) {
            const uint8_t b0 = sp[k], b1 = sp[k + 1], b2 = sp[k + 2], b3 = sp[k + 3];
            dp[k] = b0;
            if (k + 1 < run) dp[k + 1] = b1;
            if (k + 2 < run) dp[k + 2] = b2;
            if (k + 3 < run) dp[k + 3] = b3;
        }
    } else {
        for (uint32_t k = 0; k < run; ++k) ring[(d + k) & 0xffffu] = ring[(s + k) & 0xffffu];
    }
}

// The same for an oversized wave, whose output and sources live in HBM (`hbm` = address of wave
// offset 0; the source is final or produced by this very loop).
template <typename T>
__device__ __forceinline__ void hbm_copy(T* hbm, uint32_t o, uint32_t run, uint32_t dist)
{
    T*       to   = hbm + o;
    const T* from = to - dist;
    if (dist >= 4) {
        uint32_t k = 0;
        for (; k + 4 <= run; k += 4) {
            const T b0 = from[k], b1 = from[k + 1], b2 = from[k + 2], b3 = from[k + 3];
            to[k] = b0; to[k + 1] = b1; to[k + 2] = b2; to[k + 3] = b3;
        }
        for (; k < run; ++k) to[k] = from[k];
    } else {
        uint32_t q = 0;
        for (uint32_t k = 0; k < run; ++k) {
            to[k] = from[q];
            if (++q == dist) q = 0;
        }
    }
}

// per-thread emit state: where the next byte goes, which of the thread's own bytes are final
struct EmitState {
    uint8_t*  ring;      // shared-memory ring
    uint32_t  rbase;     // ring position of wave offset 0
    uint8_t*  hbm;       // HBM address of wave offset 0 (oversized waves write here directly)
    uint32_t* U;         // unresolved bitmap
    CopyItem* list;
    uint32_t  reach;     // stream offset of wave offset 0 (saturated: 2^31 - 1 once the window is full)
    uint32_t  o;         // next output byte (wave-relative)
    uint32_t  first;     // my first output byte: only I flag bytes of [first, o) before the resolve sweep
    uint32_t  clean;     // my bytes in [clean, o) are final
    uint32_t  c_next;    // my next list slot
    bool      bad_ref;   // invalidStringReference seen
};

template <bool IN_HBM>
__device__ __forceinline__ void emit_token(EmitState& S, uint32_t run, uint32_t dist, uint32_t is_copy)
{
    const uint32_t o = S.o;
    if (!is_copy) {
        if (IN_HBM) S.hbm[o] = (uint8_t)run;
        else S.ring[(S.rbase + o) & 0xffffu] = (uint8_t)run;
        S.o = o + 1;
        return;
    }
    if (dist > S.reach + o) {  // invalidStringReference: the serial decoder reports it
        S.bad_ref = true;
        return;
    }
    const int32_t src = (int32_t)o - (int32_t)dist;
    bool final = src + (int32_t)run <= 0 || src >= (int32_t)S.clean;
    if (!final && src >= (int32_t)S.first)   // inside my own bytes, below a deferred copy: final unless it overlaps one
        final = bits_all_clear(S.U, (uint32_t)src, min(run, dist));
    if (final) {
        // source is final: behind the wave (the window), or inside this thread's own finished bytes
        if (IN_HBM) hbm_copy(S.hbm, o, run, dist);
        else ring_copy(S.ring, S.rbase + o, S.rbase + o - dist, run, dist);
    } else {
        bits_set(S.U, o, run);                                      // [o, o + run) is unresolved
        S.list[S.c_next++] = CopyItem{o, run | (dist - 1) << 16};  // list is sorted by o
        S.clean = o + run;
    }
    S.o = o + run;
}

// A token of a SEGMENT (a piece of a stream that starts at a block boundary somewhere inside it and is decoded
// by its own CTA): the output is 16-bit symbols in HBM.  Bytes that an LZ77 copy takes from in front of the
// segment are not known yet; they become markers 0x8000 | index into the 32 KiB window that precedes the
// segment, travel through later copies like any other symbol, and are replaced once the segment in front
// has been resolved (window_propagate_kernel / marker_resolve_kernel in inflate_segments.cuh).
__device__ __forceinline__ void emit_token_sym(EmitState& S, uint32_t run, uint32_t dist, uint32_t is_copy)
{
    uint16_t* const h = reinterpret_cast<uint16_t*>(S.hbm);
    uint32_t o = S.o;
    if (!is_copy) {
        h[o] = (uint16_t)run;
        S.o = o + 1;
        return;
    }
    const uint32_t have = S.reach + o;              // bytes of the segment in front of this copy (saturated)
    if (dist > have) {
        const uint32_t pre = min(dist - have, run);  // this many bytes come from in front of the segment
        const uint32_t idx = WV_WINDOW - (dist - have);
        for (uint32_t k = 0; k < pre; ++k) h[o + k] = (uint16_t)(0x8000u | (idx + k));
        o += pre;
        run -= pre;
        if (run == 0) { S.o = o; return; }
    }
    const int32_t src = (int32_t)o - (int32_t)dist;
    bool final = src + (int32_t)run <= 0 || src >= (int32_t)S.clean;
    if (!final && src >= (int32_t)S.first) final = bits_all_clear(S.U, (uint32_t)src, min(run, dist));
    if (final) {
        hbm_copy(h, o, run, dist);
    } else {
        bits_set(S.U, o, run);
        S.list[S.c_next++] = CopyItem{o, run | (dist - 1) << 16};
        S.clean = o + run;
    }
    S.o = o + run;
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

__global__ void __launch_bounds__(WV_THREADS, WV_CTAS_PER_SM) inflate_wave_kernel(WvParams P)
{
    PNGB200_DYN_SMEM(wv_smem);
    WvShared& sh = *reinterpret_cast<WvShared*>(wv_smem);
    const uint32_t t    = threadIdx.x;
    const unsigned lane = lane_id(), warp = t >> 5;
    CopyItem* const list    = reinterpret_cast<CopyItem*>(P.scratch + blockIdx.x * P.scratch_stride);
    uint32_t* const gbitmap = reinterpret_cast<uint32_t*>(P.scratch + blockIdx.x * P.scratch_stride +
                                                         sizeof(CopyItem) * WV_LIST_CAP);
    for (uint32_t k = t; k < WV_BITMAP_WORDS; k += WV_THREADS) sh.bitmap[k] = 0;
    if (t == 0) mbar_init(&sh.pf_bar, 1);
    static_assert(offsetof(WvShared, ck) == offsetof(WvShared, mask) + sizeof(uint32_t) * 8 * WV_THREADS, "prefetch area = mask ++ ck");
    static_assert(sizeof(uint32_t) * WV_PF_WORDS <= 2 * sizeof(uint32_t) * 8 * WV_THREADS && offsetof(WvShared, mask) % 16 == 0, "prefetch area");
    uint32_t pf_parity = 0;          // phase of the mbarrier the next wait looks for
    const saddr_t words_addr = smem_addr(sh.words);
    const saddr_t lit = smem_addr(sh.ser.lit), dstt = smem_addr(sh.ser.dist);
    uint32_t* const mk = sh.mask;

    for (;;) {
        __syncthreads();
        if (t == 0) {
            sh.ticket = atomicAdd(P.ticket, 1u);
            sh.anomaly = 0;
            for (int k = 0; k < 12; ++k) sh.cyc[k] = 0;
            sh.tick = (uint64_t)clock64();
        }
        __syncthreads();
        if (sh.ticket >= (uint32_t)P.count) return;
        const int       j   = P.order ? (int)P.order[sh.ticket] : (int)sh.ticket;
        const StreamJob job = P.jobs[j];
        StreamResult*   r   = P.results + j;

        BitReader br;
        br.init(job.src, job.src_len, job.start_bit);
        uint64_t out    = job.start_out;
        uint32_t blocks = 0, waves = 0, resolve_rounds = 0;
        uint64_t n_tokens = 0, n_matches = 0, n_deferred = 0, walk_tokens = 0;
        int      st     = PNGB200_OK;
        uint32_t phase  = (uint32_t)job.phase;
        uint64_t resume_bit = job.start_bit, resume_out = job.start_out;
        uint8_t* dst     = job.dst;
        uint64_t dst_cap = job.dst_cap;
        bool     sym     = job.symbolic != 0;         // segment: 16-bit symbols, always written straight to HBM
        uint32_t esz     = sym ? 2u : 1u;
        uint32_t mis     = (uint32_t)((uintptr_t)dst & 15);  // ring position = stream offset + mis (mod 65536)
        // a tail that may leave symbolic mode: 1 + the last offset that holds a marker (tracked while symbolic), and
        // where it switched (~0: it did not) / the byte offset in job.dst of its byte `sw_out`
        const bool may_switch = sym && job.may_switch;
        uint64_t   mark_end = 0, sw_out = ~0ull, sw_bytes = 0;
        bool fallback = false, over_cap = false;
        bool ring_stale = job.start_out != 0;   // the ring does not hold the window [out - 32768, out)
        bool     pf_pending = false;            // a bulk prefetch is in flight / has landed
        uint64_t pf_first = 0;                  // first word (reader space) of the prefetched range
        // running Adler-32 (thread 0): valid when this launch sees the stream from its first byte
        const bool adler_on = job.start_out == 0 && !sym;
        uint32_t   s1 = 1, s2 = 0;
        uint64_t   pend_len = 0;       // a finished piece whose partial sums wait in sh.adler_*
        bool       pend = false;
        // fold the pending piece into (s1, s2): called by every thread right after a barrier
        auto fold_adler = [&]() {
            if (pend && t == 0) {
                uint64_t A = 0, B = 0;
                for (int w = 0; w < WV_WARPS; ++w) { A += sh.adler_a[w]; B += sh.adler_b[w]; }
                s2 = (uint32_t)((s2 + (pend_len % ADLER_MOD32) * s1 + B) % ADLER_MOD32);
                s1 = (uint32_t)((s1 + A) % ADLER_MOD32);
            }
            pend = false;
        };
        // CTA-wide partial sums of a finished piece of `n` bytes at HBM address `p` (stored blocks,
        // oversized waves); every thread calls it, results land in sh.adler_* for the next fold
        auto adler_hbm = [&](const uint8_t* p, uint64_t n) {
            uint64_t a = 0, bw = 0;
            const uint64_t per = (n + WV_THREADS - 1) / WV_THREADS;
            const uint64_t lo = min((uint64_t)t * per, n), hi = min(lo + per, n);
            adler_bytes(p + lo, hi - lo, n - lo, a, bw);
            uint32_t a32 = (uint32_t)(a % ADLER_MOD32), b32 = (uint32_t)(bw % ADLER_MOD32);
            for (int o = 16; o; o >>= 1) {
                a32 += __shfl_down_sync(0xffffffffu, a32, o);
                b32 += __shfl_down_sync(0xffffffffu, b32, o);
            }
            if (lane == 0) { sh.adler_a[warp] = a32; sh.adler_b[warp] = b32; }
            pend = true;
            pend_len = n;
        };
        // phase timer: thread 0 charges the cycles since the last tick to phase `i`
        auto tick = [&](int i) {
            if (t == 0) {
                const uint64_t now = (uint64_t)clock64();
                sh.cyc[i] += now - sh.tick;
                sh.tick = now;
            }
        };
        // A symbolic tail whose last 32 KiB hold no marker: DEFLATE distances are at most 32768, so no later byte can
        // depend on the output in front of the tail, and the rest is decoded as a head decodes it.  The window goes,
        // as bytes, in front of a byte area behind the symbols, so that the ring refill (ring_stale), oversized waves
        // and stored blocks find it where a direct decode has it.  Every thread calls it, right after a barrier.
        auto try_switch = [&]() {
            if (!may_switch || !sym || out < mark_end + WV_WINDOW) return;
            const uint64_t area = (2 * out + 15) & ~(uint64_t)15;   // byte offset in job.dst of the window's copy
            const uint64_t room = 2 * job.dst_cap;                   // bytes of job.dst (the store slack lies behind)
            if (area + WV_WINDOW > room) return;                     // no room: stay symbolic
            const uint16_t* const s16 = reinterpret_cast<const uint16_t*>(job.dst);
            uint8_t* const        nd  = job.dst + area + WV_WINDOW - out;   // nd[x] = byte x, x >= out - 32768
            for (uint64_t x = out - WV_WINDOW + t; x < out; x += WV_THREADS) nd[x] = (uint8_t)s16[x];
            __syncthreads();
            sym        = false;
            esz        = 1;
            dst        = nd;
            dst_cap    = room - area - WV_WINDOW + out;
            mis        = (uint32_t)((uintptr_t)nd & 15);
            ring_stale = true;
            sw_out     = out;
            sw_bytes   = area + WV_WINDOW;
        };

        if (phase == 0) {
            st = read_stream_header(br, job.format, r);
            if (st == PNGB200_OK) {
                resume_bit = br.at();
                phase = 1;
            }
        }
        if (st == PNGB200_OK && phase == 2) st = read_trailer(br, job.format, r);

        while (st == PNGB200_OK && phase == 1) {
            // warp 0 walks the header bits alone; the CTA then builds the tables together
            __syncthreads();
            fold_adler();
            {
                const uint64_t hbase = br.pos >> 5;
                for (uint32_t k = t; k < WV_HDR_WORDS; k += WV_THREADS) sh.words[k] = br.load_word(hbase + k);
                __syncthreads();
                if (warp == 0) {
                    WvHeader h;
                    if (!wv_fast_header(sh, hbase << 5, br.pos, br.total_bits, (int)lane, h)) {
#ifdef PNGB200_EMU
                        if (lane == 0 && getenv("WV_TRACE_HDR")) fprintf(stderr, "slow header at bit %llu\n", (unsigned long long)br.pos);
#endif
                        int      type0 = 0, final0 = 0, nlit0 = 0, ndist0 = 0;
                        uint32_t stored0 = 0;
                        StagedReader sr;
                        sr.init(sh.words, hbase << 5, br.total_bits, br.pos);
                        int st0 = parse_block_header(sr, &sh.ser, r, (int)lane, &type0, &final0, &stored0, &nlit0, &ndist0);
                        h = WvHeader{st0, type0, final0, nlit0, ndist0, stored0, sr.pos};
                    }
                    if (lane == 0) sh.hdr = h;
                }
            }
            __syncthreads();
            const WvHeader hdr = sh.hdr;
            st = hdr.status;
            if (st != PNGB200_OK) break;
            const int      type = hdr.type, final = hdr.final;
            const uint32_t stored = hdr.stored;
            br.seek(hdr.pos);
            if (type != 0) {
                st = build_block_tables(&sh.ser, r, hdr.nlit, hdr.ndist, (int)t, WV_THREADS);
                if (st != PNGB200_OK) break;
            }
            tick(0);
            if (type == 0) {
                if (!br.have(8 * (uint64_t)stored)) { st = PNGB200_NEED_MORE_INPUT; break; }
                if (out + stored > dst_cap) { st = fail(r, PNGB200_ERR_OUTPUT_CAPACITY); break; }
                const uint8_t* s = job.src + (br.at() >> 3);
                if (sym) for (uint32_t k = t; k < stored; k += WV_THREADS) reinterpret_cast<uint16_t*>(dst)[out + k] = s[k];
                else for (uint32_t k = t; k < stored; k += WV_THREADS) dst[out + k] = s[k];
                if (adler_on && stored) adler_hbm(s, stored);
                if (stored) ring_stale = true;
                out += stored;
                br.seek(br.pos + 8 * (uint64_t)stored);
                __syncthreads();
                fold_adler();
                try_switch();
                tick(9);
            } else {
                bool block_done = false;
                while (!block_done) {
                    ++waves;
                    // ---- stage the wave's bits in shared memory ----
                    const uint64_t wstart = br.pos;                       // absolute bit (reader space)
                    const uint64_t wbase  = (wstart >> 5) & ~(uint64_t)7; // first staged word
                    __syncthreads();
                    bool staged = false;
                    if (pf_pending) {
                        // the words the copy engine fetched while the previous wave was emitted (always waited
                        // for: the landing zone is about to become the token maps again)
                        while (!mbar_try_wait(&sh.pf_bar, pf_parity)) {}
                        pf_parity ^= 1;
                        pf_pending = false;
                        if (wbase >= pf_first && wbase - pf_first < 4) {
                            const uint32_t* lin = sh.mask + (uint32_t)(wbase - pf_first);
                            for (uint32_t k = t; k < WV_WORDS; k += WV_THREADS) sh.words[k + (k >> 3)] = lin[k];
                            staged = true;
                        }
                    }
                    if (!staged)
                        for (uint32_t k = t; k < WV_WORDS; k += WV_THREADS)
                            sh.words[k + (k >> 3)] = br.load_word(wbase + k);
                    if (t == 0) sh.wcount[0] = 0;
                    __syncthreads();                                      // (1)
                    fold_adler();
                    tick(1);
                    const uint32_t rel0  = (uint32_t)(wstart - (wbase << 5));  // < 256
                    const uint32_t base  = t * WV_SUB_BITS;
                    const uint32_t limit = base + WV_SUB_BITS;

                    // ---- A. speculative decode of my subsequence: token-start map, checkpoints, totals ----
                    uint32_t nout = 0, ncopy = 0, flags = 0, exit_bit;
                    {
#pragma unroll
                        for (int k = 0; k < 8; ++k) mk[k * WV_THREADS + t] = 0;
                        sh.ck[t] = 0;
                        FastBits b;
                        b.init(words_addr, t == 0 ? rel0 : base);
                        uint32_t mi = 0, mw = 0, n = 0;
                        while (b.pos < limit) {
                            const uint32_t rr = b.pos - base, wi = rr >> 5;
                            if (wi != mi) {
                                mk[mi * WV_THREADS + t] = mw;
                                mw = 0;
                                mi = wi;
                                sh.ck[wi * WV_THREADS + t] = nout | ncopy << 16;   // checkpoint of map word wi
                            }
                            mw |= 1u << (rr & 31);
                            uint32_t run = 0, dist = 0, cp = 0;
                            const uint32_t s = wv_decode<false>(b, lit, dstt, run, dist, cp);
                            if (s) { flags = s; break; }
                            nout += cp ? run : 1u;
                            ncopy += cp;
                            ++n;
                        }
                        mk[mi * WV_THREADS + t] = mw;
                        exit_bit = b.pos;
                        WV_COUNT(0, n);
                    }
                    sh.exit_[t] = exit_bit;
                    sh.cross_[t] = 0;
                    __syncthreads();                                      // (2) maps complete
                    tick(2);

                    // ---- B. walks: from each exit until the walk joins a subsequence owner's decode.  Walk
                    //      lengths are heavy-tailed (median 6 tokens, 1 % beyond 40), so they run in rounds of
                    //      8, 16, 32 ... tokens; the unfinished walks of a round are compacted onto the lowest
                    //      threads (state in shared memory), so that a round costs what it still has to do ----
                    {
                        uint32_t u = t, pos = exit_bit, wn = 0, wc = 0;
                        bool     active = flags == 0;
                        if (!active) {
                            sh.kind_[t] = (uint8_t)(flags == PF_EOB ? WK_OWN_EOB : WK_OWN_BAD);
                            sh.wpos_[t] = exit_bit;
                            sh.wn_[t] = 0;
                            sh.wc_[t] = 0;
                        }
                        for (uint32_t round = 0;; ++round) {
                            const uint32_t K = WV_WALK_K << min(round, 6u);
                            bool     still = false;
                            uint32_t iters = 0;
                            if (active) {
                                FastBits b;
                                b.init(words_addr, pos);
                                uint32_t kind = WK_RUNNING;
                                const uint32_t first_sub = sh.exit_[u] >> 8;
                                bool     crossed = sh.cross_[u] != 0;
                                for (; iters < K; ++iters) {
                                    const uint32_t p = b.pos;
                                    if (p >= WV_BITS) { kind = WK_END; break; }
                                    const uint32_t s = p >> 8, rr = p & 255u;
                                    if (!crossed && s > first_sub) {
                                        // a walk that leaves a subsequence without joining: the skipped owner
                                        // can take the part of the walk that lies in its subsequence (phase D)
                                        sh.cross_[u] = 1ull << 63 | (uint64_t)p << 40 | (uint64_t)(wc & 0xffu) << 24 | (wn & 0xffffffu);
                                        crossed = true;
                                    }
                                    if ((mk[(rr >> 5) * WV_THREADS + s] >> (rr & 31)) & 1u) { kind = WK_SYNC; break; }
                                    uint32_t run = 0, dist = 0, cp = 0;
                                    const uint32_t e = wv_decode<false>(b, lit, dstt, run, dist, cp);
                                    if (e) { kind = e == PF_EOB ? WK_EOB : WK_BAD; break; }
                                    wn += cp ? run : 1u;
                                    wc += cp;
                                }
                                sh.wpos_[u] = b.pos;
                                sh.wn_[u]   = wn;
                                sh.wc_[u]   = (uint16_t)wc;
                                sh.kind_[u] = (uint8_t)kind;
                                still = kind == WK_RUNNING;
                                walk_tokens += iters;
                            }
                            WV_COUNT(1, iters);
                            if (t == 0) sh.wcount[(round + 1) % 3] = 0;
                            const unsigned bal = __ballot_sync(0xffffffffu, still);
                            if (still) {
                                uint32_t at = 0;
                                const int leader = __ffs((int)bal) - 1;
                                if ((int)lane == leader) at = atomicAdd(&sh.wcount[round % 3], (uint32_t)__popc(bal));
                                at = __shfl_sync(bal, at, leader);
                                sh.wlist[round & 1][at + __popc(bal & ((1u << lane) - 1u))] = (uint8_t)u;
                            }
                            __syncthreads();
                            const uint32_t cnt = sh.wcount[round % 3];
                            if (cnt == 0) break;
                            active = t < cnt;
                            if (active) {
                                u   = sh.wlist[round & 1][t];
                                pos = sh.wpos_[u];
                                wn  = sh.wn_[u];
                                wc  = sh.wc_[u];
                            }
                        }
                    }
                    tick(3);
                    const uint32_t kind = sh.kind_[t], wpos = sh.wpos_[t];
                    {
                        const bool joins_next = kind == WK_SYNC && (wpos >> 8) == t + 1;
                        sh.next_[t] = (uint16_t)(kind == WK_SYNC ? wpos >> 8 : 0xffffu);
                        const unsigned e = __ballot_sync(0xffffffffu, !joins_next);
                        if (lane == 0) sh.exc[warp] = e;
                    }
                    __syncthreads();                                      // (3)

                    // ---- C. the true chain: orbit of thread 0.  One thread, exception words in registers, one
                    //      shared-memory load per walk that did not simply join the next subsequence ----
                    if (t == 0) {
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
                    __syncthreads();                                      // (4)
                    tick(4);

                    // ---- D. my share of the chain: the tokens that START in my subsequence, i.e. from the exit
                    //      of my predecessor on the chain to my own exit (the last thread adds its own walk) ----
                    const bool     on_chain = (sh.valid[warp] >> lane) & 1u;
                    const uint32_t last = sh.last, term = sh.term;
                    uint32_t from = rel0, to = exit_bit;   // my share of the chain: the tokens that start in [from, to)
                    uint32_t my_nout = 0, my_ncopy = 0;
                    bool     adopted = false;              // not on the chain, but I take a piece of my left neighbour's walk
                    if (on_chain) {
                        uint32_t pn = 0, pc = 0, pre_n = 0, pre_c = 0;
                        if (t > 0) {
                            uint32_t w = warp, m = sh.valid[w] & ((1u << lane) - 1u);
                            while (m == 0) m = sh.valid[--w];
                            const uint32_t pred = w * 32 + 31 - (uint32_t)__clz((int)m);
                            const uint32_t p0 = sh.wpos_[pred];       // where the predecessor's walk joined me
                            from = sh.exit_[pred];
                            pn = sh.wn_[pred];
                            pc = sh.wc_[pred];
                            if (pred + 1 < t) {
                                // the walk crossed the subsequences pred+1 .. t-1 without joining; thread pred+1
                                // takes the tokens that start in its subsequence, I take the rest
                                const uint64_t cr = sh.cross_[pred];
                                if (cr) {
                                    from = (uint32_t)(cr >> 40) & 0x1ffffu;
                                    pn -= (uint32_t)cr & 0xffffffu;
                                    pc -= (uint32_t)(cr >> 24) & 0xffu;
                                }
                            }
                            // my garbage prefix: tokens of mine that start before p0 = checkpoint of p0's map
                            // word + the tokens between the first start in that word and p0
                            const uint32_t rr = p0 - base, q = rr >> 5;
                            const uint32_t ck = sh.ck[q * WV_THREADS + t];
                            pre_n = ck & 0xffffu;
                            pre_c = ck >> 16;
                            const uint32_t first = (uint32_t)__ffs((int)mk[q * WV_THREADS + t]) - 1;
                            if (first != (rr & 31)) {
                                FastBits b;
                                b.init(words_addr, base + 32 * q + first);
                                while (b.pos != p0 && b.pos < limit) {
                                    uint32_t run = 0, dist = 0, cp = 0;
                                    if (wv_decode<false>(b, lit, dstt, run, dist, cp)) break;
                                    pre_n += cp ? run : 1u;
                                    pre_c += cp;
                                }
                            }
                        }
                        my_nout  = pn + nout - pre_n;
                        my_ncopy = pc + ncopy - pre_c;
                        if (t == last) {
                            to = wpos;
                            my_nout += sh.wn_[t];
                            my_ncopy += sh.wc_[t];
                            // ---- anomalies on the chain -> serial decoder ----
                            if (term == WK_BAD || term == WK_OWN_BAD || (wbase << 5) + wpos > br.total_bits)
                                sh.anomaly = 1;
                        }
                    }
                    else if (t > 0 && ((sh.valid[(t - 1) >> 5] >> ((t - 1) & 31)) & 1u) && sh.kind_[t - 1] == WK_SYNC) {
                        const uint64_t cr = sh.cross_[t - 1];
                        if (cr) {
                            adopted  = true;
                            from     = sh.exit_[t - 1];
                            to       = (uint32_t)(cr >> 40) & 0x1ffffu;
                            my_nout  = (uint32_t)cr & 0xffffffu;
                            my_ncopy = (uint32_t)(cr >> 24) & 0xffu;
                        }
                    }
                    // ---- scan of output byte counts and copy counts (packed: copies << 40 | bytes) ----
                    const uint64_t mine = (uint64_t)my_ncopy << 40 | my_nout;
                    uint64_t incl = mine;
                    for (int o = 1; o < 32; o <<= 1) {
                        uint64_t v = __shfl_up_sync(0xffffffffu, incl, o);
                        if ((int)lane >= o) incl += v;
                    }
                    if (lane == 31) sh.warp_sums[warp] = incl;
                    __syncthreads();                                      // (5)
                    if (warp == 0) {
                        uint64_t ws = lane < WV_WARPS ? sh.warp_sums[lane] : 0, wi = ws;
                        for (int o = 1; o < 32; o <<= 1) {
                            uint64_t v = __shfl_up_sync(0xffffffffu, wi, o);
                            if ((int)lane >= o) wi += v;
                        }
                        if (lane < WV_WARPS) sh.warp_sums[lane] = wi - ws;  // exclusive
                        if (lane == WV_WARPS - 1) sh.warp_sums[WV_WARPS] = wi;  // wave totals
                    }
                    __syncthreads();                                      // (6)
                    tick(5);
                    const uint64_t excl    = sh.warp_sums[warp] + incl - mine;
                    const uint32_t o_start = (uint32_t)(excl & 0xffffffffffull);
                    const uint32_t c_start = (uint32_t)(excl >> 40);           // my first list slot
                    const uint64_t total64 = sh.warp_sums[WV_WARPS] & 0xffffffffffull;
                    const uint32_t np      = (uint32_t)(sh.warp_sums[WV_WARPS] >> 40);
                    if (sh.anomaly || out + total64 > dst_cap || total64 > P.bitmap_words * 32) {
                        fallback = true;
                        over_cap = out + total64 > dst_cap;
                        break;
                    }
                    const uint32_t  total  = (uint32_t)total64;
                    // ---- the next wave will almost always start in the word after this one's last: fetch its words
                    //      now (bulk async copy into the token maps' memory, which is dead until the next phase A) ----
                    {
                        const uint64_t nbase = wbase + WV_BITS / 32;                       // predicted first staged word
                        const uint64_t first = nbase - ((((uintptr_t)br.words >> 2) + nbase) & 3);   // 16-byte aligned address
                        if (first >= 1 && (first + WV_PF_WORDS + 1) * 32 <= br.total_bits) {
                            if (t == 0) {
                                fence_proxy_async();   // the maps were read and written through the generic proxy
                                mbar_expect_tx(&sh.pf_bar, sizeof(uint32_t) * WV_PF_WORDS);
                                bulk_g2s(sh.mask, br.words + first, sizeof(uint32_t) * WV_PF_WORDS, &sh.pf_bar);
                            }
                            pf_pending = true;
                            pf_first = first;
                        }
                    }
                    // ---- E. emit: decode my share once more and write it ----
                    uint8_t* const  wdst   = dst + out * esz;     // HBM address of wave offset 0
                    const bool      in_hbm = sym || total > WV_OUT_BYTES;
                    const uint32_t  rbase  = (uint32_t)(out + mis) & 0xffffu;  // ring position of wave offset 0
                    uint32_t* const U      = total > WV_OUT_BYTES ? gbitmap : sh.bitmap;   // (a segment's wave may fit the shared-memory bitmap)
                    if (!in_hbm && ring_stale) {
                        // the window [out - 32768, out) was written to HBM behind the ring's back: fetch it
                        const uint64_t lo = out > WV_WINDOW ? out - WV_WINDOW : 0;
                        for (uint64_t x = lo + t; x < out; x += WV_THREADS) sh.ring[(x + mis) & 0xffffu] = dst[x];
                        __syncthreads();
                    }
                    ring_stale = in_hbm;
                    uint32_t deferred = 0, emitted = 0;
                    if (on_chain || adopted) {
                        EmitState S;
                        S.ring = sh.ring; S.rbase = rbase; S.hbm = wdst; S.U = U; S.list = list;
                        S.reach = out >= WV_WINDOW ? 0x7fffffffu : (uint32_t)out;
                        S.o = o_start; S.first = o_start; S.clean = o_start; S.c_next = c_start;
                        S.bad_ref = false;
                        FastBits b;
                        b.init(words_addr, from);
                        if (sym) {
                            while (b.pos != to && b.pos < WV_BITS + 64) {
                                uint32_t run = 0, dist = 0, cp = 0;
                                if (wv_decode<true>(b, lit, dstt, run, dist, cp)) break;
                                emit_token_sym(S, run, dist, cp);
                                ++emitted;
                            }
                        } else if (in_hbm) {
                            while (b.pos != to && b.pos < WV_BITS + 64) {
                                uint32_t run = 0, dist = 0, cp = 0;
                                if (wv_decode<true>(b, lit, dstt, run, dist, cp)) break;
                                emit_token<true>(S, run, dist, cp);
                                ++emitted;
                            }
                        } else {
                            while (b.pos != to && b.pos < WV_BITS + 64) {
                                uint32_t run = 0, dist = 0, cp = 0;
                                if (wv_decode<true>(b, lit, dstt, run, dist, cp)) break;
                                emit_token<false>(S, run, dist, cp);
                                ++emitted;
                            }
                        }
                        if (S.bad_ref) sh.anomaly = 1;
                        deferred = S.c_next - c_start;
                    }
                    WV_COUNT(2, emitted);
                    // ---- F. resolve the deferred copies.  Their list is sparse (slots were handed out for ALL
                    //      copies before anybody knew which ones would wait), so a scan of the per-thread counts
                    //      numbers them densely in output order; item g lives in the region of the last thread
                    //      whose prefix is <= g ----
                    uint32_t dincl = deferred;
                    for (int o = 1; o < 32; o <<= 1) {
                        const uint32_t v = __shfl_up_sync(0xffffffffu, dincl, o);
                        if ((int)lane >= o) dincl += v;
                    }
                    if (lane == 31) sh.dsum[warp] = dincl;
                    __threadfence_block();
                    __syncthreads();                                      // (7)
                    tick(6);
                    uint32_t nd = 0;
                    {
                        uint32_t below = 0;
#pragma unroll
                        for (int w = 0; w < WV_WARPS; ++w) {
                            const uint32_t v = sh.dsum[w];
                            below += w < (int)warp ? v : 0u;
                            nd += v;
                        }
                        sh.dpre_[t] = (uint16_t)(below + dincl - deferred);
                        sh.cst_[t]  = (uint16_t)c_start;
                    }
                    __syncthreads();                                      // (7b)
                    // No CTA barriers from here.  The numbering is sorted by output offset and a copy only depends
                    // on smaller offsets, so a lane may simply block on its current item (items t, t + 256, ...
                    // in order): the smallest open item is always somebody's current item and it is ready.
                    if (!sh.anomaly && nd) {
                        auto slot_of = [&](uint32_t g) -> uint32_t {   // list slot of dense item g
                            uint32_t lo = 0, hi = WV_THREADS;          // last u with dpre_[u] <= g
                            while (hi - lo > 1) {
                                const uint32_t mid = (lo + hi) >> 1;
                                if (sh.dpre_[mid] <= g) lo = mid;
                                else hi = mid;
                            }
                            return (uint32_t)sh.cst_[lo] + g - sh.dpre_[lo];
                        };
                        uint32_t g = t, rounds = 0;
                        CopyItem it = CopyItem{0, 0}, n1 = it, n2 = it;   // fetched from L2 two items ahead
                        if (g < nd) it = list[slot_of(g)];
                        if (g + WV_THREADS < nd) n1 = list[slot_of(g + WV_THREADS)];
                        if (g + 2 * WV_THREADS < nd) n2 = list[slot_of(g + 2 * WV_THREADS)];
                        for (;;) {
                            bool progressed = false;
                            if (g < nd) {
                                const uint32_t run = it.run_dist & 0xffff, dist = (it.run_dist >> 16) + 1;
                                const int32_t  src = (int32_t)it.o - (int32_t)dist;
                                const int32_t  hi  = src + (int32_t)min(run, dist);
                                bool ready = true;
                                if (hi > 0) {
                                    const uint32_t lo = (uint32_t)max(src, 0);
                                    ready = bits_all_clear(U, lo, (uint32_t)hi - lo);
                                }
                                if (ready) {
                                    if (sym) hbm_copy(reinterpret_cast<uint16_t*>(wdst), it.o, run, dist);
                                    else if (in_hbm) hbm_copy(wdst, it.o, run, dist);
                                    else ring_copy(sh.ring, rbase + it.o, rbase + it.o - dist, run, dist);
                                    __threadfence_block();
                                    bits_clear(U, it.o, run);
                                    g += WV_THREADS;
                                    it = n1;
                                    n1 = n2;
                                    if (g + 2 * WV_THREADS < nd) n2 = list[slot_of(g + 2 * WV_THREADS)];
                                    progressed = true;
                                }
                            }
                            ++rounds;
                            if (!__any_sync(0xffffffffu, g < nd)) break;
                            if (!__any_sync(0xffffffffu, progressed)) __nanosleep(WV_POLL_NS);
                        }
                        resolve_rounds += rounds;
                        WV_COUNT(4, rounds);
                    }
                    __threadfence_block();
                    __syncthreads();                                      // (8)
                    tick(7);
                    if (sh.anomaly) {
                        // leave the bitmap clean for whoever uses it next
                        for (uint32_t k = t; k < (total + 31) / 32; k += WV_THREADS) U[k] = 0;
                        fallback = true;
                        break;
                    }
                    if (may_switch && sym) {
                        // the wave's last marker, read back from L2 (only while the tail is still symbolic)
                        const uint16_t* const ws = reinterpret_cast<const uint16_t*>(wdst);
                        uint32_t lm = 0;
                        for (uint32_t k = t; k < total; k += WV_THREADS)
                            if (ws[k] & 0x8000u) lm = k + 1;
                        for (int o = 16; o; o >>= 1) lm = max(lm, __shfl_xor_sync(0xffffffffu, lm, o));
                        if (lane == 0) sh.mark[warp] = lm;
                        __syncthreads();
                        uint32_t wm = 0;
#pragma unroll
                        for (int w = 0; w < WV_WARPS; ++w) wm = max(wm, sh.mark[w]);
                        if (wm) mark_end = out + wm;
                    }
                    // ---- G. store: ring -> HBM, 16-byte coalesced; Adler-32 partial sums from the same registers ----
                    if (!in_hbm && total) {
                        const uint32_t shift = rbase & 15u;                  // == (uintptr_t)wdst & 15
                        uint8_t* const gbase = wdst - shift;                 // 16-byte aligned
                        const uint32_t rb16  = rbase - shift;                // ring position of gbase
                        const uint32_t end   = shift + total;                // bytes [shift, end) are ours
                        const uint32_t nq    = (end + 15) >> 4;
                        uint32_t a = 0, bw = 0;
                        for (uint32_t c = t; c < nq; c += WV_THREADS) {
                            const uint32_t lo = c << 4, hi = lo + 16;
                            if (lo >= shift && hi <= end) {
                                const uint4 x = *reinterpret_cast<const uint4*>(sh.ring + ((rb16 + lo) & 0xffffu));
                                reinterpret_cast<uint4*>(gbase)[c] = x;
                                adler_chunk16_u32(x, end - lo, a, bw);
                            } else {
                                for (uint32_t k = max(lo, shift); k < min(hi, end); ++k) {
                                    const uint8_t v = sh.ring[(rb16 + k) & 0xffffu];
                                    gbase[k] = v;
                                    a += v;
                                    bw += (end - k) * v;
                                }
                            }
                        }
                        if (adler_on) {
                            uint32_t a32 = a, b32 = bw % ADLER_MOD32;
                            for (int o = 16; o; o >>= 1) {
                                a32 += __shfl_down_sync(0xffffffffu, a32, o);
                                b32 += __shfl_down_sync(0xffffffffu, b32, o);
                            }
                            if (lane == 0) { sh.adler_a[warp] = a32; sh.adler_b[warp] = b32; }
                            pend = true;
                            pend_len = total;
                        }
                    } else if (in_hbm && adler_on) {
                        adler_hbm(wdst, total);
                    }
                    tick(8);
                    out += total;
                    if (t == 0) n_matches += np;
                    n_tokens += emitted;
                    n_deferred += deferred;
                    br.seek((wbase << 5) + sh.wpos_[last]);
                    if (term == WK_EOB || term == WK_OWN_EOB) block_done = true;
                    try_switch();
                }
                if (fallback) break;
            }
            ++blocks;
            resume_bit = br.at();
            resume_out = out;
            if (job.stop_bit && !final && br.at() >= job.stop_bit) break;   // end of my segment (the host checks ==)
            if (final) {
                phase = 2;
                st = read_trailer(br, job.format, r);
                break;
            }
        }
        if (pf_pending) {   // nothing may still land in shared memory when the CTA turns to its next stream
            while (!mbar_try_wait(&sh.pf_bar, pf_parity)) {}
            pf_parity ^= 1;
            pf_pending = false;
        }
        __syncthreads();
        fold_adler();
        __syncthreads();   // thread 0 has read the last piece's sums before the statistics reuse sh.adler_*
        // per-stream statistics (the reference's -DDUMP_LZ77_BLOCKS style counters): CTA sums
        {
            uint64_t v0 = n_tokens, v1 = n_deferred, v2 = walk_tokens;
            uint32_t v3 = resolve_rounds;
            for (int o = 16; o; o >>= 1) {
                v0 += __shfl_down_sync(0xffffffffu, v0, o);
                v1 += __shfl_down_sync(0xffffffffu, v1, o);
                v2 += __shfl_down_sync(0xffffffffu, v2, o);
                v3 = max(v3, __shfl_down_sync(0xffffffffu, v3, o));
            }
            if (lane == 0) {
                sh.warp_sums[warp] = v0;
                sh.adler_a[warp] = (uint32_t)min(v1, (uint64_t)0xffffffffu);
                sh.adler_b[warp] = (uint32_t)min(v2, (uint64_t)0xffffffffu);
                sh.exc[warp] = v3;
            }
            __syncthreads();
            if (t == 0) {
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
                r->stat_matches        = n_matches;
                r->stat_deferred       = df;
                for (int k = 0; k < 12; ++k) r->stat_cycles[k] = sh.cyc[k];
            }
        }
        if (fallback && job.symbolic) {
            // a segment cannot go through the byte-wise serial decoder: report it, the host decodes the stream whole
            // (a tail whose bytes ran out of room behind its symbols says so)
            if (t == 0) {
                r->status = sw_out != ~0ull && over_cap ? PNGB200_ERR_OUTPUT_CAPACITY : PNGB200_ERR_INTERNAL;
                r->produced = out;
                r->consumed_bits = br.at();
                r->blocks = blocks;
            }
        } else if (fallback) {
            // the serial decoder redoes this block (and whatever follows) and owns the result record
            __syncthreads();
            if (warp == 0) serial_inflate(sh.ser, job, r, resume_bit, resume_out, 1, blocks);
        } else if (t == 0) {
            if (r->status == 0) r->status = st;
            r->produced      = out;
            r->consumed_bits = br.at();
            r->blocks        = blocks;
            r->resume_bit    = resume_bit;
            r->resume_out    = resume_out;
            r->phase         = phase;
            if (adler_on && job.format != PNGB200_FORMAT_GZIP) {
                // LZ77.InflatorBuffers.advance(.checksum): compare with the trailer (InflatorBuffers.swift:109-130)
                const uint32_t computed = s2 << 16 | s1;
                r->checksum = computed;
                r->ck_done  = 1;
                if (r->trailer_seen && job.format != PNGB200_FORMAT_IOS && r->status >= 0 && r->declared != computed) {
                    r->status = PNGB200_ERR_STREAM_CHECKSUM;
                    r->err_a  = r->declared;
                    r->err_b  = computed;
                }
            }
        }
        if (t == 0) r->stat_fallback = fallback ? 1u : 0u;
        if (t == 0 && may_switch && P.switched) P.switched[j] = SwitchRecord{sw_out != ~0ull ? sw_out : out, sw_bytes};
    }
}

#ifndef PNGB200_EMU
// host side: opt in to the large dynamic shared memory on the current device (once per context)
inline int configure_inflate_wave()
{
    return (int)cudaFuncSetAttribute(inflate_wave_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)sizeof(WvShared));
}
#endif

inline uint64_t wv_bitmap_words(uint64_t max_dst_cap)
{
    uint64_t bytes = max_dst_cap < WV_MAX_WAVE_OUT ? max_dst_cap : WV_MAX_WAVE_OUT;
    return (bytes + 31) / 32 + 8;
}
inline uint64_t wv_scratch_stride(uint64_t bitmap_words)
{
    uint64_t s = sizeof(CopyItem) * (uint64_t)WV_LIST_CAP + 4 * bitmap_words;
    return (s + 255) / 256 * 256;
}

}  // namespace pngb200
