// deflate.cuh -- encode-side stage 2: LZ77.Deflator on the GPU, bit-exact with the reference.
//
// The reference's compressed bytes are a function of a long chain of order-dependent rules
// (SURVEY.md "hard part 2"): exact 4-byte-key dictionary with window expiry, attempts/goal
// cut-offs, per-decade first-wins edges, the skip-after-long-match rule, strict-< relaxation order,
// quarter-bit cost tables carried across blocks, a specific binary heap for the Huffman build.
// This first version keeps that sequential structure intact per stream and spends the GPU on
// (a) many streams at once -- one warp per stream, persistent warps pulling streams from a ticket --
// and (b) the lanes of the warp inside the hot inner loops:
//   * match extension: 32 bytes compared per step (ballot for the first mismatch)
//   * min-cost path relaxation ("explore"): lane = match length, all <= 256 targets of a vertex
//     relaxed in parallel against a shared-memory ring of path costs; the 30 distance decades of a
//     vertex arrive as one coalesced 128-byte row
//   * Adler-32 / CRC-32 of the input, table fills
// Everything else (dictionary update, greedy/lazy control flow, heap-based length-limited Huffman
// construction, code-length RLE, bit packing) runs in lock step on all lanes.
//
// Replaces Sources/LZ77/Deflator/* (DeflatorBuffers.Stream.swift:30-709, DeflatorWindow.swift:59-212,
// DeflatorMatches.swift:55-379, DeflatorMatches.Depths.swift:32-99, DeflatorSearch.swift:13-34),
// HuffmanCoding/LZ77.HuffmanTree.swift:206-404, LZ77.Heap.swift, DeflatorOut.swift:105-145.
#pragma once

#include "checksum.cuh"
#include "common.cuh"
#include "huffman.cuh"

namespace pngb200 {

struct DeflateJob {
    const uint8_t* src;
    uint64_t       n;
    uint8_t*       dst;
    uint64_t       cap;
    int32_t        format, level, exponent, pad;
};
struct DeflateResult {
    int32_t  status;
    uint32_t checksum, blocks, pad;
    uint64_t produced;
};

constexpr int      DF_HASH_BITS = 16;
constexpr uint32_t DF_MAX_DEPTH = 40;       // Huffman level-vector capacity (total weight <= 2^21 => depth <= 31)
constexpr uint32_t DF_RING      = 1024;     // path-cost ring (targets reach <= 258 ahead)
constexpr uint64_t DF_GRAPH_CAP = 1ull << 21;

__constant__ uint8_t c_zpos[19] = {3, 17, 15, 13, 11, 9, 7, 5, 4, 6, 8, 10, 12, 14, 16, 18, 0, 1, 2};

struct DfTree {            // LZ77.HuffmanTree: symbols ordered by (length, symbol), level ranges
    uint16_t symbols[288];
    uint16_t lo[15], hi[15];
};
struct DfShared {
    DfTree   rl, dist, meta;
    uint32_t freq[320];
    uint8_t  lengths[320];
    uint16_t cw_bits[288 + 32 + 19];
    uint8_t  cw_len[288 + 32 + 19];
    uint8_t  depths[542], dflt[542];
    uint8_t  mt_sym[320], mt_bits[320];
    // heap scratch for the Huffman build
    uint32_t hkey[288];
    uint16_t hid[288];
    uint16_t hn[288];
    uint16_t hvec[288][DF_MAX_DEPTH];
    uint32_t ring[DF_RING];
    uint32_t win[768];      // upstream window for the path walks
    uint32_t terms[2048];   // greedy/lazy term vector: run << 16 | (dist - 1) or 0x80000000 | literal
};

struct DfParams {
    const DeflateJob* jobs;
    DeflateResult*    results;
    uint32_t*         ticket;
    uint8_t*          scratch;         // per warp slot: head, prevh, next, graph
    uint64_t          scratch_stride;
    uint64_t          graph_vertices;  // capacity of each slot's graph (vertices)
    int               count;
};

__device__ __forceinline__ uint32_t df_run_decade(uint32_t run)
{
    if (run == 258) return 29;
    if (run <= 10) return run - 2;
    uint32_t v = run - 3, e = 29 - __clz(v);  // extra bits: floor(log2(v)) - 2
    return 4 * e + 1 + (v >> e) ;
}
__device__ __forceinline__ uint32_t df_dist_decade(uint32_t dist)
{
    if (dist <= 4) return dist - 1;
    uint32_t v = dist - 1, e = 30 - __clz(v);  // floor(log2(v)) - 1
    return 2 * e + 2 + ((v >> e) & 1);
}

// ---- bit writer (all lanes hold the same state; lane 0 stores) ----
struct DfOut {
    uint8_t* p;
    uint64_t cap, bytes;
    uint64_t acc;
    int      nacc;
    int      overflow;
    __device__ __forceinline__ void put(uint32_t v, int count)
    {
        acc |= (uint64_t)v << nacc;
        nacc += count;
        while (nacc >= 8) {
            if (bytes < cap) { if (lane_id() == 0) p[bytes] = (uint8_t)acc; }
            else overflow = 1;
            ++bytes;
            acc >>= 8;
            nacc -= 8;
        }
    }
    __device__ __forceinline__ void pad() { if (nacc) put(0, 8 - nacc); }
};

// ---- LZ77.HuffmanTree.init(frequencies:limit:) with the reference's heap (lock step, shared mem) ----
__device__ int df_heap_lowest(DfShared& S, int count, int parent)
{
    int r = (parent << 1) + 1, l = parent << 1, end = 1 + count;
    if (l >= end) return 0;
    if (r >= end) return S.hkey[l - 1] < S.hkey[parent - 1] ? l : 0;
    int c = S.hkey[r - 1] < S.hkey[l - 1] ? r : l;
    return S.hkey[c - 1] < S.hkey[parent - 1] ? c : 0;
}
__device__ void df_heap_swap(DfShared& S, int i, int j)
{
    __syncwarp();   // every lane has read the keys (df_heap_lowest, df_sift_up, the dequeue) before lane 0 moves them
    if (lane_id() == 0) {
        uint32_t k = S.hkey[i - 1]; S.hkey[i - 1] = S.hkey[j - 1]; S.hkey[j - 1] = k;
        uint16_t d = S.hid[i - 1]; S.hid[i - 1] = S.hid[j - 1]; S.hid[j - 1] = d;
    }
    __syncwarp();
}
__device__ void df_sift_down(DfShared& S, int count, int i)
{
    int c;
    while ((c = df_heap_lowest(S, count, i)) != 0) { df_heap_swap(S, i, c); i = c; }
}
__device__ void df_sift_up(DfShared& S, int i)
{
    for (;;) {
        int p = i >> 1;
        if (p < 1 || !(S.hkey[i - 1] < S.hkey[p - 1])) return;
        df_heap_swap(S, i, p);
        i = p;
    }
}

// returns 0, or PNGB200_ERR_INTERNAL if a level vector would outgrow DF_MAX_DEPTH
__device__ int df_build_tree(DfShared& S, DfTree& T, const uint32_t* freq, int n, int limit)
{
    const unsigned lane = lane_id();
    __shared__ uint16_t syms_s[288];
    int ns = 0;
    for (int i = 0; i < n; ++i)
        if (freq[i] > 0) { if (lane == 0) syms_s[ns] = (uint16_t)i; ++ns; }
    __syncwarp();
    // stable insertion sort by decreasing frequency (lane 0)
    if (lane == 0)
        for (int i = 1; i < ns; ++i) {
            uint16_t s = syms_s[i];
            int j = i;
            while (j > 0 && freq[syms_s[j - 1]] < freq[s]) { syms_s[j] = syms_s[j - 1]; --j; }
            syms_s[j] = s;
        }
    __syncwarp();
    if (lane < 15) { T.lo[lane] = 0; T.hi[lane] = 0; }
    __syncwarp();
    if (ns <= 1) {  // HuffmanTree.init(stub:)
        if (lane == 0) {
            if (ns == 1) T.symbols[0] = syms_s[0];
            T.lo[0] = 0; T.hi[0] = (uint16_t)ns;
            for (int i = 1; i < 15; ++i) { T.lo[i] = (uint16_t)ns; T.hi[i] = (uint16_t)ns; }
        }
        __syncwarp();
        return 0;
    }
    int count = ns;
    for (int i = (int)lane; i < ns; i += 32) {  // symbols.reversed().map { (freq, [1]) }
        S.hkey[i] = freq[syms_s[ns - 1 - i]];
        S.hid[i]  = (uint16_t)i;
        S.hn[i]   = 1;
        S.hvec[i][0] = 1;
    }
    __syncwarp();
    for (int i = count >> 1; i >= 1; --i) df_sift_down(S, count, i);
    int      nl = 0;
    uint16_t leaves[DF_MAX_DEPTH];
    for (;;) {
        // dequeue first
        uint32_t k1 = S.hkey[0]; uint16_t id1 = S.hid[0];
        if (count > 1) { df_heap_swap(S, 1, count); --count; df_sift_down(S, count, 1); }
        else { count = 0; }
        if (count == 0) {
            nl = S.hn[id1] - 1;  // first.value.dropLast().reversed()
            for (int i = 0; i < nl; ++i) leaves[i] = S.hvec[id1][nl - 1 - i];
            break;
        }
        uint32_t k2 = S.hkey[0]; uint16_t id2 = S.hid[0];
        if (count > 1) { df_heap_swap(S, 1, count); --count; df_sift_down(S, count, 1); }
        else { count = 0; }
        uint16_t big = S.hn[id1] > S.hn[id2] ? id1 : id2, small = S.hn[id1] > S.hn[id2] ? id2 : id1;
        int nb = S.hn[big], nsm = S.hn[small];
        if (nb + 1 > (int)DF_MAX_DEPTH) return PNGB200_ERR_INTERNAL;
        __syncwarp();
        for (int i = (int)lane; i < nsm; i += 32) S.hvec[big][nb - 1 - i] += S.hvec[small][nsm - 1 - i];
        if (lane == 0) { S.hvec[big][nb] = 0; S.hn[big] = (uint16_t)(nb + 1); }
        __syncwarp();
        if (lane == 0) { S.hkey[count] = k1 + k2; S.hid[count] = big; }
        __syncwarp();
        ++count;
        df_sift_up(S, count);
    }
    // limitHeight
    int levels[DF_MAX_DEPTH];
    for (int i = 0; i < nl; ++i) levels[i] = leaves[i];
    if (nl > limit) {
        long unhoused = 0;
        for (int l = nl - 1; l >= limit; --l) {
            int pairs = levels[l] >> 1;
            unhoused += pairs;
            levels[l - 1] += pairs;
        }
        nl = limit;
        int split = limit - 2;
        while (unhoused > 0) {
            if (levels[split] <= 0) { split -= 1; continue; }
            long res = levels[split] < unhoused ? levels[split] : unhoused;
            unhoused -= res;
            levels[split] -= (int)res;
            levels[split + 1] += (int)(2 * res);
            if (split < limit - 2) split += 1;
        }
    }
    if (lane == 0) {
        int base = 0;
        for (int i = 0; i < 15; ++i) {
            int c = i < nl ? levels[i] : 0;
            T.lo[i] = (uint16_t)base; T.hi[i] = (uint16_t)(base + c);
            // symbols of this level, ascending (insertion sort of the slice)
            for (int a = base; a < base + c; ++a) {
                uint16_t s = syms_s[a];
                int j = a;
                while (j > base && T.symbols[j - 1] > s) { T.symbols[j] = T.symbols[j - 1]; --j; }
                T.symbols[j] = s;
            }
            base += c;
        }
    }
    __syncwarp();
    return 0;
}

// HuffmanTree.codewords: canonical codes, bit-reversed for the LSB-first writer
__device__ void df_codewords(const DfTree& T, uint16_t* bits, uint8_t* len, int count)
{
    const unsigned lane = lane_id();
    for (int i = (int)lane; i < count; i += 32) { bits[i] = 0; len[i] = 0; }
    __syncwarp();
    if (lane == 0) {
        uint32_t counter = 0;
        for (int l = 1; l <= 15; ++l) {
            for (int i = T.lo[l - 1]; i < T.hi[l - 1]; ++i) {
                bits[T.symbols[i]] = (uint16_t)(__brev(counter) >> (32 - l));
                len[T.symbols[i]]  = (uint8_t)l;
                ++counter;
            }
            counter <<= 1;
        }
    }
    __syncwarp();
}

struct DfState {
    const uint8_t* x;
    int64_t  n, mask, end_index, dequeued;
    int32_t *head, *prevh, *next;
    uint32_t* graph;   // 32 x u32 per vertex: (unused), (unused), 30 edges: distance << 16 | longest run
    uint32_t* up;      // upstream word per vertex (+1 for the sink)
    int64_t  limit, capacity, count, skip_until;
    int      mode, goal, iterations, generic;
    long     attempts;
};

__device__ __forceinline__ uint32_t df_key(const DfState& z, int64_t p)
{
    uint32_t k = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) k = k << 8 | (uint32_t)((p + i >= 0 && p + i < z.n) ? z.x[p + i] : 0);
    return k;
}
__device__ __forceinline__ int64_t df_input_count(const DfState& z) { return z.n - z.dequeued; }

// DeflatorWindow.update: position entering the window; *next = previous position with the same key
__device__ int64_t df_window_update(DfState& z, int64_t* next)
{
    int64_t  a = z.end_index;
    uint32_t k = df_key(z, a), h = (k * 2654435761u) >> (32 - DF_HASH_BITS);
    int64_t  p = z.head[h], found = -1;
    while (p >= 0 && a - p <= z.mask) {
        if (df_key(z, p) == k) { found = p; break; }
        p = z.prevh[p & z.mask];
    }
    __syncwarp();
    if (lane_id() == 0) {
        z.next[a & z.mask]  = (int32_t)found;
        z.prevh[a & z.mask] = z.head[h];
        z.head[h]           = (int32_t)a;
    }
    __syncwarp();
    z.end_index += 1;
    z.dequeued += 1;
    if (next) *next = found;
    return a;
}

// run = 4 + common prefix of x[current+4...] and x[a+4...], capped at limit (lanes compare 32 bytes/step)
__device__ __forceinline__ int df_extend(const DfState& z, int64_t a, int64_t current, int limit)
{
    const unsigned lane = lane_id();
    int run = 4;
    while (run < limit) {
        int  k = run + (int)lane;
        bool eq = k < limit && z.x[current + k] == z.x[a + k];
        unsigned m = __ballot_sync(0xffffffffu, !eq);
        if (m) { run += __ffs(m) - 1; break; }
        run += 32;
    }
    return run < limit ? run : limit;
}

// DeflatorWindow.match with a per-candidate callback expressed as a functor
template <typename F>
__device__ void df_window_match(const DfState& z, int64_t a, int64_t next, F&& delegate)
{
    if (next < 0) return;
    int64_t lookahead = df_input_count(z);
    int     limit = (int)(lookahead + 4 < 258 ? lookahead + 4 : 258);
    int64_t current = next, distance = a - current;
    long    remaining = z.attempts;
    for (;;) {
        int run = df_extend(z, a, current, limit);
        if (run < 4) run = 4;
        delegate(run, (int)distance);
        remaining -= 1;
        if (!(remaining > 0 && z.goal > run)) break;
        int64_t nx = z.next[current & z.mask];
        if (nx < 0) break;
        distance += current - nx;
        current = nx;
        if (!(distance < z.mask)) break;
    }
}
__device__ bool df_window_best(const DfState& z, int64_t a, int64_t next, int* brun, int* bdist)
{
    int br = 5, bd = 1;
    df_window_match(z, a, next, [&](int run, int dist) { if (br < run) { br = run; bd = dist; } });
    *brun = br; *bdist = bd;
    return br > 5;
}
__device__ __forceinline__ uint8_t df_literal(const DfState& z, int64_t a) { return a >= 0 && a < z.n ? z.x[a] : 0; }
__device__ __forceinline__ int64_t df_unfilled(const DfState& z) { return z.limit - 1 - z.count; }

__device__ void df_store_vertex(DfState& z, uint8_t lit)
{
    uint32_t* v = z.graph + (z.count << 5);
    v[lane_id()] = lane_id() == 0 ? lit : 0;   // upstream = literal; depth slot and 30 edges cleared
    __syncwarp();
    z.count += 1;
}

// Stream.compress(all:), Stream.swift:195-404; returns true when the match buffer is full.  `lookahead` is 0 for
// compress(all: true), else 258 (greedy, full) or 259 (lazy): a head is taken only while more input than that is
// pending (:210, :269, :345), so a key and a 258-byte compare never reach past z.n, and only all: true runs the epilogue.
__device__ bool df_compress(DfState& z, DfShared& S, int64_t lookahead)
{
    const unsigned lane = lane_id();
    while (z.end_index < 0 && df_input_count(z) > lookahead) { z.end_index += 1; z.dequeued += 1; }
    int64_t next;
    if (z.mode == 0) {
        while (df_input_count(z) > lookahead) {
            if (df_unfilled(z) <= 0) return true;
            int64_t a = df_window_update(z, &next);
            int run, dist;
            if (df_window_best(z, a, next, &run, &dist)) {
                for (int k = 1; k < run; ++k) df_window_update(z, nullptr);
                if (lane == 0) S.terms[z.count] = (uint32_t)run << 16 | (uint32_t)(dist - 1);
            } else if (lane == 0) S.terms[z.count] = 0x80000000u | df_literal(z, a);
            z.count += 1;
        }
    } else if (z.mode == 1) {
        while (df_input_count(z) > lookahead) {
            if (df_unfilled(z) <= 1) return true;
            int64_t a = df_window_update(z, &next);
            uint8_t first = df_literal(z, a);
            int er, ed, lr, ld;
            if (df_window_best(z, a, next, &er, &ed)) {
                int64_t a1 = df_window_update(z, &next);
                if (df_window_best(z, a1, next, &lr, &ld) && er < lr) {
                    if (lane == 0) {
                        S.terms[z.count]     = 0x80000000u | first;
                        S.terms[z.count + 1] = (uint32_t)lr << 16 | (uint32_t)(ld - 1);
                    }
                    z.count += 2;
                    for (int k = 1; k < lr; ++k) df_window_update(z, nullptr);
                } else {
                    if (lane == 0) S.terms[z.count] = (uint32_t)er << 16 | (uint32_t)(ed - 1);
                    z.count += 1;
                    for (int k = 2; k < er; ++k) df_window_update(z, nullptr);
                }
            } else {
                if (lane == 0) S.terms[z.count] = 0x80000000u | first;
                z.count += 1;
            }
        }
    } else {
        // Full mode, 32 positions per step (lane = position).  Every position becomes a vertex and
        // enters the dictionary whatever the parse does, and its candidate chain is a pure function
        // of the dictionary state at that position, so a batch does: (D) all 32 dictionary look-ups
        // against the pre-batch state in parallel, in-batch predecessors by warp match, one batched
        // update; (M) 32 independent chain walks; (S) the order-dependent skip rule over the lanes.
        // A position is taken as a head while more than `lookahead` bytes are pending, and as a skip vertex of a long
        // match whatever is pending (:376): `take` positions from a0 on qualify before this batch sets skip_until.
        uint32_t* g = z.graph;
        for (;;) {
            const int64_t a0 = z.end_index, left = df_input_count(z);
            int64_t take = left - lookahead > z.skip_until - a0 ? left - lookahead : z.skip_until - a0;
            if (take > left) take = left;
            if (take <= 0) break;
            const int64_t unf = df_unfilled(z);
            if (unf <= 0) return true;
            const int     nb = (int)(unf < 32 ? (unf < take ? unf : take) : (take < 32 ? take : 32));
            const bool    act = (int)lane < nb;
            const int64_t a = a0 + lane;
            // ---- (D) ----
            const uint32_t key = act ? df_key(z, a) : 0u;
            const uint32_t h = (key * 2654435761u) >> (32 - DF_HASH_BITS);
            const int32_t  oldhead = act ? z.head[h] : -1;
            int64_t p = oldhead, found = -1;
            if (act)
                while (p >= 0 && a - p <= z.mask) {
                    if (df_key(z, p) == key) { found = p; break; }
                    p = z.prevh[p & z.mask];
                }
            const unsigned actmask = __ballot_sync(0xffffffffu, act);
            const unsigned below = (1u << lane) - 1u;
            const unsigned pk = __match_any_sync(0xffffffffu, key) & actmask;
            const unsigned ph = __match_any_sync(0xffffffffu, h) & actmask;
            const int64_t nxt = (pk & below) ? a0 + (31 - __clz(pk & below)) : found;
            const int64_t prv = (ph & below) ? a0 + (31 - __clz(ph & below)) : (int64_t)oldhead;
            // the window slots this batch overwrites still belong to positions one window back,
            // which an earlier lane's chain walk may yet have to read: keep their links
            if (act) S.win[lane] = (uint32_t)z.next[a & z.mask];
            __syncwarp();
            if (act) {
                z.next[a & z.mask]  = (int32_t)nxt;
                z.prevh[a & z.mask] = (int32_t)prv;
                if ((int)lane == 31 - __clz(ph)) z.head[h] = (int32_t)a;
            }
            for (int r = 0; r < nb; ++r)  // DeflatorMatches.store(vertex:) for the batch, one row per store
                g[((z.count + r) << 5) + lane] = lane == 0 ? (uint32_t)z.x[a0 + r] : 0u;
            __syncwarp();
            // ---- (M) ----
            int extent = 1;
            if (act && nxt >= 0) {
                const int limit = (int)(z.n - a < 258 ? z.n - a : 258);
                int64_t   current = nxt, distance = a - current;
                long      remaining = z.attempts;
                uint32_t* edges = g + ((z.count + lane) << 5) + 2;
                for (;;) {
                    int run = 4;
                    while (run < limit && z.x[current + run] == z.x[a + run]) ++run;
                    if (run > extent) extent = run;
                    const uint32_t dd = df_dist_decade((uint32_t)distance);
                    if ((uint32_t)run > (edges[dd] & 0xffffu)) edges[dd] = (uint32_t)distance << 16 | (uint32_t)run;
                    remaining -= 1;
                    if (!(remaining > 0 && z.goal > run)) break;
                    const int64_t q = current + z.mask + 1 - a0;  // lane that overwrote this slot, if any
                    const int64_t nx = (q > (int64_t)lane && q < nb) ? (int64_t)(int32_t)S.win[q]
                                                                    : (int64_t)z.next[current & z.mask];
                    if (nx < 0) break;
                    distance += current - nx;
                    current = nx;
                    if (!(distance < z.mask)) break;
                }
            }
            __syncwarp();
            // ---- (S) skip rule: after a match longer than 100 the next min(extent - 100, unfilled)
            //      vertices carry no edges (and do not trigger the rule themselves) ----
            for (int l = 0; l < nb; ++l) {
                const int     ext = __shfl_sync(0xffffffffu, extent, l);
                const int64_t al = a0 + l;
                if (al < z.skip_until) {
                    if (lane >= 2) g[((z.count + l) << 5) + lane] = 0u;
                } else if (ext > 100) {
                    const int64_t unf_after = z.limit - 1 - (z.count + l + 1);
                    z.skip_until = al + 1 + (ext - 100 < unf_after ? ext - 100 : unf_after);
                }
            }
            __syncwarp();
            z.count += nb;
            z.end_index += nb;
            z.dequeued += nb;
        }
    }
    if (lookahead > 0) return false;
    int64_t epilogue = -3 - (z.end_index < 0 ? z.end_index : 0);
    while (df_input_count(z) > epilogue) {
        if (df_unfilled(z) <= 0) return true;
        int64_t a = df_window_update(z, nullptr);
        if (z.mode == 2) df_store_vertex(z, df_literal(z, a));
        else { if (lane == 0) S.terms[z.count] = 0x80000000u | df_literal(z, a); z.count += 1; }
    }
    __syncwarp();
    return false;
}

// DeflatorMatches.minimize: forward relaxation (explore) + backward walk with frequency tally
__device__ void df_minimize(DfState& z, DfShared& S)
{
    const unsigned lane = lane_id();
    uint32_t* g  = z.graph;   // 32 words per vertex; words 2..31 = best edge per distance decade
    uint32_t* up = z.up;      // upstream word per vertex: length << 16 | decade << 8
    const int64_t  count = z.count;
    const uint8_t* lits  = z.x + (z.end_index - z.count);  // vertex v is input position pos0 + v
    for (uint32_t i = lane; i < DF_RING; i += 32) S.ring[i] = 0xffffffffu;
    for (uint32_t i = lane; i < 320; i += 32) S.freq[i] = 0;
    __syncwarp();
    if (lane == 0) S.ring[0] = 0;
    __syncwarp();
    // ---- explore every vertex in order; path costs live in the shared-memory ring, upstream words
    //      are write-only here; edge rows are prefetched four vertices ahead ----
    uint32_t r0 = 0 < count ? g[(0 << 5) + lane] : 0, r1 = 1 < count ? g[(1 << 5) + lane] : 0;
    uint32_t r2 = 2 < count ? g[(2 << 5) + lane] : 0, r3 = 3 < count ? g[(3 << 5) + lane] : 0;
    for (int64_t s = 0; s < count; ++s) {
        const uint32_t row = r0;
        r0 = r1; r1 = r2; r2 = r3;
        r3 = s + 4 < count ? g[((s + 4) << 5) + lane] : 0;
        const uint32_t cur_depth = S.ring[s & (DF_RING - 1)];
        const int64_t  remaining = count - s;
        if (lane == 0) {
            S.ring[(s + 512) & (DF_RING - 1)] = 0xffffffffu;  // recycle a slot far ahead
            const uint32_t ld = cur_depth + S.depths[lits[s]];   // literal edge (length 1)
            uint32_t& nd = S.ring[(s + 1) & (DF_RING - 1)];
            if (ld < nd) {
                nd = ld;
                up[s + 1] = 0x0001ff00u;
            }
        }
        uint32_t myrun = (lane >= 2 && remaining >= 3) ? (row & 0xffffu) : 0;
        if ((int64_t)myrun > remaining) myrun = (uint32_t)remaining;
        const unsigned present = __ballot_sync(0xffffffffu, myrun > 0);
        if (present) {
            uint32_t maxrun = myrun;
            for (int o = 16; o; o >>= 1) maxrun = max(maxrun, __shfl_xor_sync(0xffffffffu, maxrun, o));
            for (uint32_t base = 3; base <= maxrun; base += 32) {
                const uint32_t len = base + lane;
                uint32_t best = 0xffffffffu, bdec = 0;
                unsigned m = present;
                while (m) {   // decades ascending: a later decade must be strictly cheaper to win
                    const int dl = __ffs(m) - 1;
                    m &= m - 1;
                    const uint32_t r = __shfl_sync(0xffffffffu, myrun, dl);
                    if (len <= r) {
                        const uint32_t d = cur_depth + S.depths[512 + dl - 2] + S.depths[253 + len];
                        if (d < best) { best = d; bdec = (uint32_t)(dl - 2); }
                    }
                }
                if (len <= maxrun && best != 0xffffffffu) {
                    uint32_t& nd = S.ring[(s + len) & (DF_RING - 1)];
                    if (best < nd) {
                        nd = best;
                        up[s + len] = len << 16 | bdec << 8;
                    }
                }
            }
        }
        __syncwarp();
    }
    __syncwarp();
    // ---- walk back from the sink, reverse the links, tally symbol frequencies ----
    if (count > 0) {
        int64_t  ci = count;
        uint32_t cu = up[ci];
        int64_t  wlo = -1;  // window [wlo, wlo + 768) of upstream words in shared memory
        do {
            const int64_t length = cu >> 16;
            const int64_t ni = ci - length;
            if (wlo < 0 || ni < wlo) {
                __syncwarp();
                wlo = ni - 767 > 0 ? ni - 767 : 0;
                for (int64_t k = wlo + lane; k <= ni; k += 32) S.win[k - wlo] = up[k];
                __syncwarp();
            }
            const uint32_t nu = S.win[ni - wlo];
            if (lane == 0) {
                up[ni] = cu;
                if (length == 1) S.freq[lits[ni]] += 1;
                else {
                    S.freq[256 | df_run_decade((uint32_t)length)] += 1;
                    S.freq[288 + ((cu >> 8) & 0xff)] += 1;
                }
            }
            ci = ni;
            cu = nu;
        } while (ci > 0);
    }
    __syncwarp();
    if (lane == 0) S.freq[256] = 1;
    __syncwarp();
}

// Depths.update / generalize
__device__ void df_depths_update(DfShared& S)
{
    if (lane_id() == 0) {
        for (int l = 1; l <= 15; ++l)
            for (int i = S.rl.lo[l - 1]; i < S.rl.hi[l - 1]; ++i) {
                int sym = S.rl.symbols[i];
                if (sym < 256) S.depths[sym] = (uint8_t)(l << 2);
                else if (sym > 256) {
                    int dec = sym - 257, len = l + c_len_extra[dec], base = 253 + c_len_base[dec], cnt = 1 << c_len_extra[dec];
                    for (int k = base; k < base + cnt; ++k) S.depths[k] = (uint8_t)(len << 2);
                }
            }
        for (int l = 1; l <= 15; ++l)
            for (int i = S.dist.lo[l - 1]; i < S.dist.hi[l - 1]; ++i) {
                int sym = S.dist.symbols[i];
                S.depths[512 + sym] = (uint8_t)((l + c_dist_extra[sym]) << 2);
            }
    }
    __syncwarp();
}

// Stream.writeBlock(final:): trees, code-length RLE, header, tables, terms.  returns 0 or error
__device__ int df_write_block(DfState& z, DfShared& S, DfOut& out, bool final)
{
    const unsigned lane = lane_id();
    int rc;
    if (z.mode != 2) {  // DeflatorMatches.trees()
        for (uint32_t i = lane; i < 320; i += 32) S.freq[i] = 0;
        __syncwarp();
        if (lane == 0) {
            for (int64_t i = 0; i < z.count; ++i) {
                uint32_t t = S.terms[i];
                if (t & 0x80000000u) { S.freq[t & 0xff] += 1; }
                else { S.freq[256 | df_run_decade(t >> 16)] += 1; S.freq[288 + df_dist_decade((t & 0xffff) + 1)] += 1; }
            }
            S.freq[256] = 1;
        }
        __syncwarp();
        if ((rc = df_build_tree(S, S.rl, S.freq, 286, 15))) return rc;
        if ((rc = df_build_tree(S, S.dist, S.freq + 288, 30, 15))) return rc;
    } else {            // DeflatorMatches.trees(iterations:)
        z.limit = 2 * z.limit < z.capacity ? 2 * z.limit : z.capacity;
        int i = z.generic ? -z.iterations : 0;
        for (;;) {
            df_minimize(z, S);
            if ((rc = df_build_tree(S, S.rl, S.freq, 286, 15))) return rc;
            if ((rc = df_build_tree(S, S.dist, S.freq + 288, 30, 15))) return rc;
            i += 1;
            if (!(i < z.iterations)) break;
            df_depths_update(S);
            z.generic = 0;
        }
    }
    // code lengths
    for (uint32_t i = lane; i < 320; i += 32) S.lengths[i] = 0;
    __syncwarp();
    int r = 257, d = 1;
    if (lane == 0) {
        for (int l = 1; l <= 15; ++l)
            for (int i = S.rl.lo[l - 1]; i < S.rl.hi[l - 1]; ++i) S.lengths[S.rl.symbols[i]] = (uint8_t)l;
    }
    __syncwarp();
    {
        int rr = 286;
        while (rr > 0 && S.lengths[rr - 1] == 0) --rr;
        r = rr < 257 ? 257 : rr;
    }
    __syncwarp();
    if (lane == 0) {
        for (int l = 1; l <= 15; ++l)
            for (int i = S.dist.lo[l - 1]; i < S.dist.hi[l - 1]; ++i) S.lengths[r + S.dist.symbols[i]] = (uint8_t)l;
    }
    __syncwarp();
    {
        int dd = 32;
        while (dd > 0 && S.lengths[r + dd - 1] == 0) --dd;
        d = dd < 1 ? 1 : dd;
    }
    // run-length terms of the code lengths (Stream.swift:482-543); lock step, lane 0 stores
    int nmt = 0;
    {
        int repetitions = 1;
        uint8_t last = S.lengths[0];
        auto emit = [&](uint8_t sym, uint8_t bits) {
            if (lane == 0) { S.mt_sym[nmt] = sym; S.mt_bits[nmt] = bits; }
            ++nmt;
        };
        for (int at = 1;; ++at) {
            bool have = at < r + d;
            if (have && S.lengths[at] == last) { repetitions += 1; continue; }
            if (last == 0) {
                while (repetitions > 138) { emit(18, 138 - 11); repetitions -= 138; }
                if (repetitions > 2) {
                    if (repetitions < 11) emit(17, (uint8_t)(repetitions - 3));
                    else emit(18, (uint8_t)(repetitions - 11));
                } else for (int k = 0; k < repetitions; ++k) emit(0, 0);
            } else {
                emit(last, 0);
                repetitions -= 1;
                while (repetitions > 6) { emit(16, 3); repetitions -= 6; }
                if (repetitions > 2) emit(16, (uint8_t)(repetitions - 3));
                else for (int k = 0; k < repetitions; ++k) emit(last, 0);
            }
            if (!have) break;
            last = S.lengths[at];
            repetitions = 1;
        }
    }
    __syncwarp();
    __shared__ uint32_t mfreq[19];
    if (lane < 19) mfreq[lane] = 0;
    __syncwarp();
    if (lane == 0) for (int i = 0; i < nmt; ++i) mfreq[S.mt_sym[i]] += 1;
    __syncwarp();
    if ((rc = df_build_tree(S, S.meta, mfreq, 19, 7))) return rc;
    df_codewords(S.rl, S.cw_bits, S.cw_len, 288);
    df_codewords(S.dist, S.cw_bits + 288, S.cw_len + 288, 32);
    df_codewords(S.meta, S.cw_bits + 320, S.cw_len + 320, 19);
    // writeBlockMetadata
    __shared__ uint8_t cl[19];
    if (lane < 19) cl[lane] = 0;
    __syncwarp();
    if (lane == 0)
        for (int l = 1; l <= 8; ++l)
            for (int i = S.meta.lo[l - 1]; i < S.meta.hi[l - 1]; ++i) cl[c_zpos[S.meta.symbols[i]]] = (uint8_t)l;
    __syncwarp();
    int ncl = 19;
    while (ncl > 0 && cl[ncl - 1] == 0) --ncl;
    if (ncl < 4) ncl = 4;
    out.put(final ? 5 : 4, 3);
    out.put((uint32_t)(r - 257), 5);
    out.put((uint32_t)(d - 1), 5);
    out.put((uint32_t)(ncl - 4), 4);
    for (int i = 0; i < ncl; ++i) out.put(cl[i], 3);
    // writeBlockTables
    for (int i = 0; i < nmt; ++i) {
        uint8_t sym = S.mt_sym[i];
        out.put(S.cw_bits[320 + sym], S.cw_len[320 + sym]);
        int extra = sym == 18 ? 7 : sym == 17 ? 3 : sym == 16 ? 2 : 0;
        out.put(S.mt_bits[i], extra);
    }
    // writeBlock(with:)
    if (z.mode != 2) {
        for (int64_t i = 0; i < z.count; ++i) {
            uint32_t t = S.terms[i];
            if (t & 0x80000000u) out.put(S.cw_bits[t & 0xff], S.cw_len[t & 0xff]);
            else {
                uint32_t run = t >> 16, dist = (t & 0xffff) + 1, rd = df_run_decade(run), dd = df_dist_decade(dist);
                out.put(S.cw_bits[256 | rd], S.cw_len[256 | rd]);
                out.put(run - c_len_base[rd - 1], c_len_extra[rd - 1]);
                out.put(S.cw_bits[288 + dd], S.cw_len[288 + dd]);
                out.put(dist - c_dist_base[dd], c_dist_extra[dd]);
            }
        }
        out.put(S.cw_bits[256], S.cw_len[256]);
        z.count = 0;
    } else {
        uint32_t* g = z.graph;
        const uint32_t* up = z.up;
        const uint8_t*  lits = z.x + (z.end_index - z.count);
        int64_t index = 0, whi = -1;  // window [wlo, whi) of upstream words
        int64_t wlo = 0;
        while (index < z.count) {
            if (index >= whi) {
                __syncwarp();
                wlo = index;
                whi = index + 768 < z.count ? index + 768 : z.count;
                for (int64_t k = wlo + lane; k < whi; k += 32) S.win[k - wlo] = up[k];
                __syncwarp();
            }
            uint32_t upw = S.win[index - wlo];
            int64_t  cnt = upw >> 16;
            if (cnt == 1) { const uint32_t lit = lits[index]; out.put(S.cw_bits[lit], S.cw_len[lit]); }
            else {
                uint32_t rd = df_run_decade((uint32_t)cnt), dd = (upw >> 8) & 0xff;
                uint32_t offset = g[(index << 5) + 2 + dd] >> 16;
                out.put(S.cw_bits[256 | rd], S.cw_len[256 | rd]);
                out.put((uint32_t)cnt - c_len_base[rd - 1], c_len_extra[rd - 1]);
                out.put(S.cw_bits[288 + dd], S.cw_len[288 + dd]);
                out.put(offset - c_dist_base[dd], c_dist_extra[dd]);
            }
            index += cnt;
        }
        out.put(S.cw_bits[256], S.cw_len[256]);
        z.count = 0;
        for (uint32_t i = lane; i < 542; i += 32) {  // Depths.generalize
            uint8_t s = S.depths[i], gg = S.dflt[i];
            S.depths[i] = (uint8_t)((s & gg) + ((s ^ gg) >> 1));
        }
        __syncwarp();
    }
    return 0;
}

// DeflatorSearch.init(level:) and the match buffer's capacity
__device__ void df_search(DfState& z, int level)
{
    const int lv = level <= 0 ? 0 : level;
    const long AT[13] = {1, 2, 4, 40, 20, 40, 64, 100, 14, 20, 30, 60, 100};
    const int  GO[13] = {6, 8, 10, 24, 32, 54, 80, 160, 20, 32, 50, 80, 133};
    if (lv <= 12) { z.mode = lv <= 3 ? 0 : lv <= 7 ? 1 : 2; z.attempts = AT[lv]; z.goal = GO[lv]; z.iterations = lv >= 8 ? lv - 7 : 0; }
    else { z.mode = 2; z.attempts = 0x7fffffffffffffffL; z.goal = 258; z.iterations = 6; }
    z.capacity = z.mode == 2 ? (int64_t)DF_GRAPH_CAP : (1 << 15);
}

// Depths.default into S.dflt, and into S.depths when `reset`
__device__ void df_default_depths(DfShared& S, bool reset)
{
    for (uint32_t i = lane_id(); i < 542; i += 32) {
        uint8_t v;
        if (i < 256) v = 33;
        else if (i < 512) { uint32_t run = i - 253; v = (uint8_t)(30 + (c_len_extra[df_run_decade(run) - 1] << 2)); }
        else v = (uint8_t)(19 + (c_dist_extra[i - 512] << 2));
        S.dflt[i] = v;
        if (reset) S.depths[i] = v;
    }
    __syncwarp();
}

// the stored final block of a stream shorter than 3 bytes, Stream.swift:45-60, :417-435
__device__ void df_write_stored(DfOut& out, const uint8_t* x, int64_t n)
{
    out.put(1, 3);
    out.pad();
    out.put((uint32_t)n, 16);
    out.put(~(uint32_t)n & 0xffff, 16);
    for (int64_t i = 0; i < n; ++i) out.put(x[i], 8);
}

__global__ void __launch_bounds__(32) deflate_kernel(DfParams P)
{
    PNGB200_DYN_SMEM(df_smem);
    DfShared& S = *reinterpret_cast<DfShared*>(df_smem);
    const unsigned lane = lane_id();
    uint8_t* slot = P.scratch + blockIdx.x * P.scratch_stride;
    for (;;) {
        uint32_t t = 0;
        if (lane == 0) t = atomicAdd(P.ticket, 1u);
        t = __shfl_sync(0xffffffffu, t, 0);
        if (t >= (uint32_t)P.count) return;
        const DeflateJob job = P.jobs[t];
        DeflateResult*   res = P.results + t;
        DfState z;
        z.x = job.src; z.n = (int64_t)job.n;
        int exponent = job.format == PNGB200_FORMAT_IOS ? 15 : job.exponent;
        z.mask = ((int64_t)1 << exponent) - 1;
        z.end_index = -3; z.dequeued = 0; z.count = 0; z.limit = 2048; z.generic = 1; z.skip_until = 0;
        z.head  = reinterpret_cast<int32_t*>(slot);
        z.prevh = z.head + (1 << DF_HASH_BITS);
        z.next  = z.prevh + 32768;
        z.graph = reinterpret_cast<uint32_t*>(z.next + 32768);
        z.up    = z.graph + 32 * P.graph_vertices;
        df_search(z, job.level);
        int status = PNGB200_OK;
        if (z.mode == 2 && (uint64_t)(z.n < (int64_t)DF_GRAPH_CAP ? z.n : (int64_t)DF_GRAPH_CAP) + 2 > P.graph_vertices)
            status = PNGB200_ERR_INTERNAL;
        for (uint32_t i = lane; i < (1u << DF_HASH_BITS); i += 32) z.head[i] = -1;
        df_default_depths(S, true);
        DfOut out;
        out.p = job.dst; out.cap = job.cap; out.bytes = 0; out.acc = 0; out.nacc = 0; out.overflow = 0;
        uint32_t blocks = 0;
        if (status == PNGB200_OK) {
            if (job.format == PNGB200_FORMAT_ZLIB) {
                uint32_t unpaired = (uint32_t)(exponent - 8) << 4 | 8;
                uint32_t check = ~(((unpaired << 8) | (unpaired >> 8)) % 31) & 31;
                out.put(check << 8 | unpaired, 16);
            } else if (job.format == PNGB200_FORMAT_GZIP) {
                out.put(0x8b1f, 16); out.put(0x0008, 16); out.put(0, 16); out.put(0, 16); out.put(0xff00, 16);
            }
            if (z.n >= 3) {
                for (;;) {
                    bool full = df_compress(z, S, 0);
                    int rc = df_write_block(z, S, out, !full);
                    ++blocks;
                    if (rc) { status = rc; break; }
                    if (!full) break;
                }
            } else {
                df_write_stored(out, z.x, z.n);
                ++blocks;
            }
        }
        // checksum of the input: Adler-32 (zlib) or CRC-32 (gzip), lanes in parallel
        uint32_t checksum = 0;
        if (status == PNGB200_OK && job.format == PNGB200_FORMAT_ZLIB) {
            uint64_t s1 = 0, s2 = 0;
            for (int64_t base = 0; base < z.n; base += 32 * 4096) {
                uint64_t a = 0, b = 0;
                int64_t hi = base + 32 * 4096 < z.n ? base + 32 * 4096 : z.n;
                for (int64_t k = base + lane; k < hi; k += 32) { a += z.x[k]; b += (uint64_t)(z.n - k) * z.x[k]; }
                s1 = (s1 + a) % ADLER_MOD;
                s2 = (s2 + b) % ADLER_MOD;
            }
            for (int o = 16; o; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2 += __shfl_xor_sync(0xffffffffu, s2, o); }
            s1 = (s1 + 1) % ADLER_MOD;
            s2 = (s2 + (uint64_t)z.n % ADLER_MOD) % ADLER_MOD;
            checksum = (uint32_t)(s2 << 16 | s1);
            out.pad();
            out.put(checksum >> 24, 8); out.put((checksum >> 16) & 0xff, 8); out.put((checksum >> 8) & 0xff, 8); out.put(checksum & 0xff, 8);
        } else if (status == PNGB200_OK && job.format == PNGB200_FORMAT_GZIP) {
            uint32_t crc = 0xffffffffu;  // bytewise, lock step (gzip streams are the secondary path)
            for (int64_t k = 0; k < z.n; ++k) crc = crc32_byte_table((crc ^ z.x[k]) & 0xff) ^ (crc >> 8);
            checksum = ~crc;
            out.pad();
            out.put(checksum & 0xffff, 16); out.put(checksum >> 16, 16);
            out.put((uint32_t)z.n & 0xffff, 16); out.put(((uint32_t)z.n >> 16) & 0xffff, 16);
        }
        out.pad();
        if (lane == 0) {
            res->status = status != PNGB200_OK ? status : (out.overflow ? PNGB200_ERR_OUTPUT_CAPACITY : PNGB200_OK);
            res->produced = out.bytes;
            res->checksum = checksum;
            res->blocks = blocks;
        }
        __syncwarp();
    }
}

// ---- the online deflator (pngb200_deflator_create_online): one launch per push batch, one warp per handle ----
//
// LZ77.DeflatorBuffers.push(_:last:) compresses whenever more than 4096 bytes are pending or `last` is set
// (DeflatorBuffers.swift:68-137): compressBlocks(final: false) writes every block that fills while more input than the
// lookahead is pending, and leaves the rest for a later push.  Everything that push carries lives in DfCarry and the
// handle's device buffers.  Positions are relative to `base`, the absolute stream position of the handle's input byte 0;
// after each non-final launch the base moves forward by a multiple of 32 768 (the dictionary slots `pos & mask` stay
// put), so no position exceeds the unfinished block + the window + the pending input whatever the stream length.
struct DfCarry {
    int64_t  end_index, count, limit, skip_until;   // relative to base
    uint64_t base;                                  // absolute position of input byte 0
    uint64_t summed;                                // input bytes folded into the checksum (absolute)
    uint64_t acc;                                   // the bit writer's partial byte
    int32_t  nacc, generic, fresh, status;
    uint32_t s1, s2, crc, pad;                      // running Adler-32 (s1, s2) and CRC-32
    uint8_t  depths[544];                           // Depths carried across blocks (542 used)
    uint32_t terms[2048];                           // greedy / lazy: the unfinished block's terms
};
struct DfResumeJob {
    DfCarry*  carry;
    uint8_t*  in;              // input from `base` on: n bytes
    uint64_t  n;
    int32_t*  dict;            // head, prevh, next
    uint32_t* graph;           // full mode: the unfinished block's vertices, 32 words each
    uint32_t* up;              // full mode: graph_vertices + 1 words, not carried
    uint64_t  graph_vertices;
    uint8_t*  dst;             // device: this launch's complete bytes, up to cap
    uint64_t  cap;
    uint8_t*  host_dst;        // where the warp copies them (pinned host memory)
    struct DfResumeResult* result;   // pinned host memory
    int32_t   format, level, exponent, last;
};
// The scanline ends of a push (pngb200_png_encoder_push_batch), positions relative to the carry's base in increasing
// order, the last one the job's n.  PNG.Encoder.pull pushes one scanline at a time into its deflator, and each of those
// pushes compresses when more than 4096 bytes are pending (DeflatorBuffers.swift:74): the kernel walks the ends and does
// the same at each, so it releases blocks no earlier than the reference.  It is an array beside the jobs, so that a
// DfResumeJob keeps its layout.
struct DfEnds {
    const uint64_t* at;
    uint64_t        count;
};
struct DfResumeResult {
    int32_t  status;
    uint32_t blocks;           // blocks written by this launch
    uint64_t produced;         // complete bytes written by this launch
    uint64_t base;             // the carry's base after it
    int64_t  end_index, count; // relative to that base
};
// the carry of a handle that has compressed nothing yet
inline void df_carry_init(DfCarry& c)
{
    memset(&c, 0, sizeof c);
    c.end_index = -3;
    c.limit = 2048;   // DeflatorMatches.init ignores its `limit:` argument
    c.generic = 1;
    c.fresh = 1;
    c.s1 = 1;
    c.crc = 0xffffffffu;
}
constexpr size_t DF_DICT_WORDS = (1u << DF_HASH_BITS) + 2 * 32768;

// `ends`: null, or one DfEnds per job; a job whose ends are null, or a launch without them, has one end at n.
__global__ void __launch_bounds__(32) deflate_resume_kernel(const DfResumeJob* jobs, int count, const DfEnds* ends = nullptr)
{
    PNGB200_DYN_SMEM(df_smem);
    DfShared& S = *reinterpret_cast<DfShared*>(df_smem);
    const unsigned lane = lane_id();
    for (int t = blockIdx.x; t < count; t += gridDim.x) {
        const DfResumeJob job = jobs[t];
        DfCarry&          c = *job.carry;
        DfState z;
        z.x = job.in; z.n = (int64_t)job.n;
        const int exponent = job.format == PNGB200_FORMAT_IOS ? 15 : job.exponent;
        z.mask = ((int64_t)1 << exponent) - 1;
        z.end_index = c.end_index; z.dequeued = c.end_index + 3;   // the window has dequeued 3 bytes past its end
        z.count = c.count; z.limit = c.limit; z.skip_until = c.skip_until; z.generic = c.generic;
        z.head  = job.dict;
        z.prevh = z.head + (1 << DF_HASH_BITS);
        z.next  = z.prevh + 32768;
        z.graph = job.graph;
        z.up    = job.up;
        df_search(z, job.level);
        const bool fresh = c.fresh != 0;
        if (fresh)
            for (uint32_t i = lane; i < (1u << DF_HASH_BITS); i += 32) z.head[i] = -1;
        df_default_depths(S, fresh);
        if (!fresh)
            for (uint32_t i = lane; i < 542; i += 32) S.depths[i] = c.depths[i];
        if (z.mode != 2)
            for (int64_t i = lane; i < z.count; i += 32) S.terms[i] = c.terms[i];
        __syncwarp();
        int status = c.status;
        if (z.mode == 2 && (uint64_t)(z.count + (z.n - z.end_index)) + 2 > job.graph_vertices &&
            (uint64_t)DF_GRAPH_CAP + 2 > job.graph_vertices)
            status = PNGB200_ERR_INTERNAL;
        // fold the bytes that arrived since the last launch into the checksum
        uint32_t s1 = c.s1, s2 = c.s2, crc = c.crc;
        const int64_t from = (int64_t)(c.summed - c.base);
        if (job.format == PNGB200_FORMAT_ZLIB) {
            for (int64_t b0 = from; b0 < z.n; b0 += 32 * 4096) {
                const int64_t len = z.n - b0 < 32 * 4096 ? z.n - b0 : 32 * 4096;
                uint64_t a = 0, b = 0;
                for (int64_t k = lane; k < len; k += 32) { a += z.x[b0 + k]; b += (uint64_t)(len - k) * z.x[b0 + k]; }
                for (int o = 16; o; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
                s2 = (uint32_t)((s2 + (uint64_t)len % ADLER_MOD * s1 + b % ADLER_MOD) % ADLER_MOD);
                s1 = (uint32_t)((s1 + a % ADLER_MOD) % ADLER_MOD);
            }
        } else if (job.format == PNGB200_FORMAT_GZIP) {
            for (int64_t k = from; k < z.n; ++k) crc = crc32_byte_table((crc ^ z.x[k]) & 0xff) ^ (crc >> 8);
        }
        DfOut out;
        out.p = job.dst; out.cap = job.cap; out.bytes = 0; out.acc = c.acc; out.nacc = c.nacc; out.overflow = 0;
        uint32_t blocks = 0;
        if (status == PNGB200_OK) {
            const uint64_t total = c.base + (uint64_t)z.n;
            if (job.last && total < 3) {
                df_write_stored(out, z.x, z.n);   // never compacted: a stream this short has base 0
                ++blocks;
            } else {
                const DfEnds  e = ends ? ends[t] : DfEnds{nullptr, 0};
                const uint64_t nends = e.at ? e.count : 1;
                for (uint64_t k = 0; k < nends && status == PNGB200_OK; ++k) {
                    const bool last = job.last && k + 1 == nends;
                    if (e.at) {
                        z.n = (int64_t)e.at[k];
                        if (!last && df_input_count(z) <= 4096) continue;   // DeflatorBuffers.swift:74
                    }
                    const int64_t lookahead = last ? 0 : z.mode == 1 ? 259 : 258;
                    for (;;) {
                        const bool full = df_compress(z, S, lookahead);
                        if (!full && !last) break;
                        const int rc = df_write_block(z, S, out, !full);
                        ++blocks;
                        if (rc) { status = rc; break; }
                        if (!full) break;
                    }
                }
                z.n = (int64_t)job.n;
            }
            if (job.last && job.format == PNGB200_FORMAT_ZLIB) {
                const uint32_t ck = s2 << 16 | s1;
                out.pad();
                out.put(ck >> 24, 8); out.put((ck >> 16) & 0xff, 8); out.put((ck >> 8) & 0xff, 8); out.put(ck & 0xff, 8);
            } else if (job.last && job.format == PNGB200_FORMAT_GZIP) {
                const uint32_t ck = ~crc;
                out.pad();
                out.put(ck & 0xffff, 16); out.put(ck >> 16, 16);
                out.put((uint32_t)total & 0xffff, 16); out.put(((uint32_t)total >> 16) & 0xffff, 16);
            }
            if (job.last) out.pad();
            if (out.overflow) status = PNGB200_ERR_OUTPUT_CAPACITY;
        }
        // Move the base past what no later push reads: window look-ups and compares reach back to end_index - mask, and
        // full mode reads the unfinished block's literals from end_index - count.
        int64_t shift = 0;
        if (status == PNGB200_OK && !job.last) {
            int64_t keep = z.end_index - z.mask;
            if (z.mode == 2 && z.end_index - z.count < keep) keep = z.end_index - z.count;
            shift = keep > 0 ? keep >> 15 << 15 : 0;
        }
        if (shift) {
            // positions that fall out of the window become -1, which ends a chain walk exactly as expiry does
            uint4* d = reinterpret_cast<uint4*>(z.head);
            const int32_t sh = (int32_t)shift;
            auto rebase = [sh](uint32_t w) { return (int32_t)w >= sh ? (uint32_t)((int32_t)w - sh) : 0xffffffffu; };
            for (uint32_t i = lane; i < DF_DICT_WORDS / 4; i += 32) {
                uint4 v = d[i];
                v.x = rebase(v.x); v.y = rebase(v.y); v.z = rebase(v.z); v.w = rebase(v.w);
                d[i] = v;
            }
            // slide the live input down; a step moves 512 bytes, less than the shift, so a step reads nothing an
            // earlier step wrote
            const int64_t live = z.n - shift, vec = live >> 4;
            uint4* dv = reinterpret_cast<uint4*>(job.in);
            const uint4* sv = reinterpret_cast<const uint4*>(job.in + shift);
            for (int64_t i0 = 0; i0 < vec; i0 += 32) {
                if (i0 + lane < vec) dv[i0 + lane] = sv[i0 + lane];
                __syncwarp();
            }
            for (int64_t i = (vec << 4) + lane; i < live; i += 32) job.in[i] = job.in[i + shift];
            z.end_index -= shift;
            z.skip_until -= shift;
        }
        __syncwarp();
        // the complete bytes to the host
        for (uint64_t i = lane; i < out.bytes && i < job.cap; i += 32) job.host_dst[i] = job.dst[i];
        if (z.mode != 2)
            for (int64_t i = lane; i < z.count; i += 32) c.terms[i] = S.terms[i];
        for (uint32_t i = lane; i < 542; i += 32) c.depths[i] = S.depths[i];
        __syncwarp();
        if (lane == 0) {
            c.end_index = z.end_index; c.count = z.count; c.limit = z.limit; c.skip_until = z.skip_until;
            c.generic = z.generic; c.fresh = 0; c.status = status;
            c.base += (uint64_t)shift;
            c.summed = c.base + (uint64_t)(z.n - shift);
            c.acc = out.acc; c.nacc = out.nacc;
            c.s1 = s1; c.s2 = s2; c.crc = crc;
            DfResumeResult r;
            r.status = status; r.blocks = blocks; r.produced = out.bytes < job.cap ? out.bytes : job.cap;
            r.base = c.base; r.end_index = z.end_index; r.count = z.count;
            *job.result = r;
        }
        __syncwarp();
    }
}

inline uint64_t df_scratch_stride(uint64_t graph_vertices)
{
    uint64_t s = 4ull * ((1u << DF_HASH_BITS) + 2 * 32768) + 132ull * graph_vertices;
    return (s + 255) / 256 * 256;
}

}  // namespace pngb200
