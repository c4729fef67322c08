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
// (inflate_serial.cuh), which owns the exact error semantics of the reference.  A job with a resume record (the
// streaming handle) hands it only the rest of the block from the last wave that completed.
//
// CTAs are persistent: each takes streams from an atomic ticket (the host orders streams longest
// first), so per-CTA scratch in HBM is bounded by the number of resident CTAs.
//
// Replaces the reference's serial token loop Stream.readBlock(with:) and InflatorOut.expand
// (Sources/LZ77/Inflator/LZ77.InflatorBuffers.Stream.swift:266-381, LZ77.InflatorOut.swift:124-140),
// the window of LZ77.InflatorOut (LZ77.InflatorOut.swift:86-110) and, for zlib streams, the running
// MRC32 (Sources/LZ77/Wrappers/LZ77.MRC32.swift:26-47).
#pragma once

#include "inflate_stream.cuh"

namespace pngb200 {

constexpr int      WV_CTAS_PER_SM  = 2;
constexpr uint32_t WV_RING         = 65536;                             // window + wave output (uint16 index wraps)
constexpr uint32_t WV_OUT_BYTES    = WV_RING - WV_WINDOW;               // largest wave the ring can take
constexpr uint32_t WV_BITMAP_WORDS = WV_OUT_BYTES / 32;
constexpr uint32_t WV_LIST_CAP     = WV_BITS / 2 + 64;                  // >= copies per wave (2 bits min each)
constexpr unsigned WV_POLL_NS      = 20;

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
    WavePrefetch pf{0, false, 0};
    const saddr_t words_addr = smem_addr(sh.words);
    const saddr_t lit = smem_addr(sh.ser.lit), dstt = smem_addr(sh.ser.dist);
    uint32_t* const mk = sh.mask;

    for (;;) {
        const int j = next_stream(sh, P);
        if (j < 0) return;
        StreamRun S;
        S.open(P, j);
        const StreamJob& job = S.job;
        StreamResult* const r = S.r;
        BitReader& br = S.br;
        uint64_t&  out = S.out;
        uint32_t waves = 0, resolve_rounds = 0;
        uint64_t n_tokens = 0, n_matches = 0, n_deferred = 0, walk_tokens = 0;
        uint8_t* dst     = job.dst;
        uint64_t dst_cap = job.dst_cap;
        bool     sym     = job.symbolic != 0;         // segment: 16-bit symbols, always written straight to HBM
        uint32_t esz     = sym ? 2u : 1u;
        uint32_t mis     = (uint32_t)((uintptr_t)dst & 15);  // ring position = stream offset + mis (mod 65536)
        // a tail that may leave symbolic mode: 1 + the last offset that holds a marker (tracked while symbolic), and
        // where it switched (~0: it did not) / the byte offset in job.dst of its byte `sw_out`
        const bool may_switch = sym && job.may_switch;
        uint64_t   mark_end = 0, sw_out = ~0ull, sw_bytes = 0;
        bool over_cap = false;
        bool ring_stale = job.start_out != 0;   // the ring does not hold the window [out - 32768, out)
        // running Adler-32: valid when this launch sees the stream from its first byte
        const bool adler_on = job.start_out == 0 && !sym;
        AdlerRun   adler;
        adler.reset();
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

        while (S.st == PNGB200_OK && S.phase == 1) {
            __syncthreads();
            adler.fold(sh);
            const uint64_t hpos = br.pos;
            const WvHeader hdr = read_block_header(sh, br, r);
            S.st = hdr.status;
            if (S.st != PNGB200_OK) break;
            const int      type = hdr.type, final = hdr.final;
            const uint32_t stored = hdr.stored;
            br.seek(hdr.pos);
            if (type != 0) {
                S.st = build_block_tables(&sh.ser, r, hdr.nlit, hdr.ndist, (int)t, WV_THREADS);
                if (S.st != PNGB200_OK) break;
                S.begin_block(hpos, final);
            }
            phase_tick(sh, 0);
            if (type == 0) {
                if (!S.copy_stored(sh, dst, dst_cap, sym, stored, adler, adler_on)) break;
                if (stored) ring_stale = true;
                try_switch();
                phase_tick(sh, 9);
            } else {
                bool block_done = false;
                while (!block_done) {
                    ++waves;
                    // ---- stage the wave's bits in shared memory ----
                    const uint64_t wstart = br.pos;                       // absolute bit (reader space)
                    const uint64_t wbase  = (wstart >> 5) & ~(uint64_t)7; // first staged word
                    __syncthreads();
                    pf.stage(sh, br, wbase);
                    if (t == 0) sh.wcount[0] = 0;
                    __syncthreads();                                      // (1)
                    adler.fold(sh);
                    phase_tick(sh, 1);
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
                    phase_tick(sh, 2);

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
                    phase_tick(sh, 3);
                    const uint32_t kind = sh.kind_[t], wpos = sh.wpos_[t];
                    {
                        const bool joins_next = kind == WK_SYNC && (wpos >> 8) == t + 1;
                        sh.next_[t] = (uint16_t)(kind == WK_SYNC ? wpos >> 8 : 0xffffu);
                        const unsigned e = __ballot_sync(0xffffffffu, !joins_next);
                        if (lane == 0) sh.exc[warp] = e;
                    }
                    __syncthreads();                                      // (3)

                    // ---- C. the true chain ----
                    if (t == 0) follow_chain(sh);
                    __syncthreads();                                      // (4)
                    phase_tick(sh, 4);

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
                    // ---- scan of output byte counts and copy counts ----
                    const uint64_t excl    = cta_scan_packed(sh, (uint64_t)my_ncopy << 40 | my_nout);   // (5), (6)
                    phase_tick(sh, 5);
                    const uint32_t o_start = (uint32_t)(excl & 0xffffffffffull);
                    const uint32_t c_start = (uint32_t)(excl >> 40);           // my first list slot
                    const uint64_t total64 = sh.warp_sums[WV_WARPS] & 0xffffffffffull;
                    const uint32_t np      = (uint32_t)(sh.warp_sums[WV_WARPS] >> 40);
                    // (bit 1 only: a thread already in phase E may have set bit 2 for this wave -- read after barrier (7))
                    if ((sh.anomaly & 1u) || out + total64 > dst_cap || total64 > P.bitmap_words * 32) {
                        S.fall_back();
                        over_cap = out + total64 > dst_cap;
                        break;
                    }
                    const uint32_t  total  = (uint32_t)total64;
                    // ---- the next wave will almost always start in the word after this one's last: fetch its words ----
                    pf.start(sh, br, wbase + WV_BITS / 32);
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
                        if (S.bad_ref) sh.anomaly = 2;
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
                    phase_tick(sh, 6);
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
                    phase_tick(sh, 7);
                    if (sh.anomaly) {
                        // leave the bitmap clean for whoever uses it next
                        for (uint32_t k = t; k < (total + 31) / 32; k += WV_THREADS) U[k] = 0;
                        S.fall_back();
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
                        if (adler_on) adler.piece_from_partials(sh, a, bw % ADLER_MOD32, total);
                    } else if (in_hbm && adler_on) {
                        adler.piece_from_hbm(sh, wdst, total);
                    }
                    phase_tick(sh, 8);
                    out += total;
                    if (t == 0) n_matches += np;
                    n_tokens += emitted;
                    n_deferred += deferred;
                    br.seek((wbase << 5) + sh.wpos_[last]);
                    if (term == WK_EOB || term == WK_OWN_EOB) block_done = true;
                    else S.wave_done();
                    try_switch();
                }
                if (S.fallback) break;
            }
            if (S.end_block(final)) break;
        }
        pf.drain(sh);   // nothing may still land in shared memory when the CTA turns to its next stream
        // a segment that falls back reports it; a tail whose bytes ran out of room behind its symbols says so
        const int seg_status = sw_out != ~0ull && over_cap ? PNGB200_ERR_OUTPUT_CAPACITY : PNGB200_ERR_INTERNAL;
        S.finish(sh, adler, adler_on, seg_status,
                 [&] { report_wave_stats(sh, r, waves, n_matches, n_tokens, n_deferred, walk_tokens, resolve_rounds); });
        if (t == 0 && may_switch && P.switched) P.switched[j] = SwitchRecord{sw_out != ~0ull ? sw_out : out, sw_bytes};
    }
}

// per-CTA HBM scratch of inflate_wave_kernel (see wave_bitmap_words)
inline uint64_t wv_bitmap_words(uint64_t max_dst_cap) { return wave_bitmap_words(max_dst_cap, WV_LIST_CAP); }
inline uint64_t wv_scratch_stride(uint64_t bitmap_words) { return wave_scratch_stride(bitmap_words, WV_LIST_CAP); }

}  // namespace pngb200
