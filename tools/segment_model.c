/*
 * tools/segment_model.c -- CPU model of the segment-parallel inflate planned in DESIGN.md section 8
 * item 1: split points -> speculative block-boundary search (block_probe.c) -> every segment decoded on
 * its own with the 32 KiB window in front of it unknown (bytes that depend on it are kept as symbolic
 * markers and propagate through copies) -> segments chained by "the predecessor's decode arrives exactly
 * at my first bit on a block boundary" -> markers resolved segment by segment.  Measures how many output
 * bytes stay symbolic (that decides the data structure on the GPU) and proves the result bit-exact.
 * A measurement tool: not product code, not the oracle.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

int probe_dynamic_header(const uint8_t* in, size_t n, uint64_t p, uint64_t* header_bits);

typedef struct {
    const uint8_t* p;
    size_t         n;
    uint64_t       at;
} bitsrc;
static inline uint32_t peek(const bitsrc* b, int count)
{
    uint64_t v = 0;
    size_t   byte = (size_t)(b->at >> 3);
    for (int k = 0; k < 8 && byte + (size_t)k < b->n; ++k) v |= (uint64_t)b->p[byte + k] << (8 * k);
    return (uint32_t)((v >> (b->at & 7)) & ((1ull << count) - 1));
}
static inline uint32_t take(bitsrc* b, int count)
{
    uint32_t v = peek(b, count);
    b->at += (uint64_t)count;
    return v;
}

typedef struct {
    uint16_t count[16], symbol[320];
} huff;
static int build(huff* h, const uint8_t* lens, int n)
{
    memset(h->count, 0, sizeof h->count);
    for (int i = 0; i < n; ++i) h->count[lens[i]]++;
    h->count[0] = 0;
    uint16_t offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = (uint16_t)(offs[l] + h->count[l]);
    for (int i = 0; i < n; ++i)
        if (lens[i]) h->symbol[offs[lens[i]]++] = (uint16_t)i;
    return 0;
}
static int decode(bitsrc* b, const huff* h)
{
    int code = 0, first = 0, index = 0;
    for (int l = 1; l <= 15; ++l) {
        code |= (int)take(b, 1);
        int c = h->count[l];
        if (code - c < first) return h->symbol[index + (code - first)];
        index += c, first += c, first <<= 1, code <<= 1;
    }
    return -1;
}
static const uint16_t LBASE[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
static const uint8_t  LEXT[29]  = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
static const uint16_t DBASE[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
static const uint8_t  DEXT[30]  = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};
static const uint8_t  ORDER[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

/* symbols: 0..255 a byte; 256 + i = "byte i of the unknown 32 KiB window in front of the segment" */
typedef struct {
    uint16_t* sym;
    size_t    n, cap;
} symbuf;
static void push(symbuf* o, uint16_t v)
{
    if (o->n == o->cap) o->sym = (uint16_t*)realloc(o->sym, (o->cap = o->cap ? o->cap * 2 : 1 << 16) * sizeof(uint16_t));
    o->sym[o->n++] = v;
}

/* Decode blocks from `start` until a block boundary that is one of stops[0..nstops) (returns its
 * index), or the final block ends (returns nstops), or an error (-1).  Candidates that the decode runs
 * past without landing on them are simply not joined. */
static int decode_segment(const uint8_t* in, size_t n, uint64_t start, const uint64_t* stops, int nstops, int known_window,
                          symbuf* out, uint64_t* end_bit)
{
    bitsrc b = {in, n, start};
    for (;;) {
        for (int s = 0; s < nstops; ++s)
            if (stops[s] == b.at && b.at != start) { *end_bit = b.at; return s; }
        if (b.at + 3 > (uint64_t)n * 8) return -1;
        int final = (int)take(&b, 1), type = (int)take(&b, 2);
        if (type == 0) {
            b.at = (b.at + 7) & ~(uint64_t)7;
            uint32_t len = take(&b, 16), nlen = take(&b, 16);
            if (len != (~nlen & 0xffffu)) return -1;
            for (uint32_t k = 0; k < len; ++k) push(out, (uint16_t)take(&b, 8));
        } else if (type == 1 || type == 2) {
            huff    lit, dist;
            uint8_t lens[320];
            if (type == 1) {
                for (int i = 0; i < 288; ++i) lens[i] = i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8;
                build(&lit, lens, 288);
                for (int i = 0; i < 30; ++i) lens[i] = 5;
                build(&dist, lens, 30);
            } else {
                int     hlit = (int)take(&b, 5) + 257, hdist = (int)take(&b, 5) + 1, hclen = (int)take(&b, 4) + 4;
                uint8_t cl[19] = {0};
                huff    meta;
                for (int i = 0; i < hclen; ++i) cl[ORDER[i]] = (uint8_t)take(&b, 3);
                build(&meta, cl, 19);
                for (int i = 0; i < hlit + hdist;) {
                    int s = decode(&b, &meta);
                    if (s < 0) return -1;
                    if (s < 16) { lens[i++] = (uint8_t)s; continue; }
                    int rep, val = 0;
                    if (s == 16) { if (!i) return -1; val = lens[i - 1]; rep = 3 + (int)take(&b, 2); }
                    else if (s == 17) rep = 3 + (int)take(&b, 3);
                    else rep = 11 + (int)take(&b, 7);
                    if (i + rep > hlit + hdist) return -1;
                    while (rep--) lens[i++] = (uint8_t)val;
                }
                build(&lit, lens, hlit);
                build(&dist, lens + hlit, hdist);
            }
            for (;;) {
                int s = decode(&b, &lit);
                if (s < 0 || b.at > (uint64_t)n * 8) return -1;
                if (s < 256) { push(out, (uint16_t)s); continue; }
                if (s == 256) break;
                if (s > 285) return -1;
                uint32_t run = LBASE[s - 257] + take(&b, LEXT[s - 257]);
                int      d = decode(&b, &dist);
                if (d < 0 || d > 29) return -1;
                uint32_t back = DBASE[d] + take(&b, DEXT[d]);
                for (uint32_t k = 0; k < run; ++k) {
                    if (back <= out->n) push(out, out->sym[out->n - back]);       /* may copy a marker */
                    else if (known_window) return -1;                             /* invalidStringReference */
                    else push(out, (uint16_t)(256 + 32768 - (back - out->n)));    /* window byte 32768 - reach */
                }
            }
        } else
            return -1;
        if (final) { *end_bit = b.at; return nstops; }
    }
}

/* The tail of a stream cut in two (DESIGN.md section 4.2): decoded from the block header at `start` to the end of
 * the stream with the 32 KiB in front unknown.  out[0] output bytes; out[1] the first output offset whose last
 * 32 KiB hold no marker (from there on nothing can depend on the head; out[0] if the tail never gets there);
 * out[2] markers.  Returns 0, or -1 when the decode fails (`start` is not a real block boundary). */
int tail_model(const uint8_t* in, size_t n, uint64_t start, uint64_t* out)
{
    symbuf   s = {0};
    uint64_t end, last = 0, markers = 0;   /* last: 1 + offset of the last marker */
    const int rc = decode_segment(in, n, start, NULL, 0, 0, &s, &end);
    if (rc >= 0)
        for (size_t i = 0; i < s.n; ++i)
            if (s.sym[i] >= 256) { last = i + 1; ++markers; }
    out[0] = s.n;
    out[1] = last + 32768 < s.n ? last + 32768 : s.n;
    out[2] = markers;
    free(s.sym);
    return rc >= 0 ? 0 : -1;
}

/* Whole model.  stats[4 * k + ...] per accepted segment: start bit, symbols, markers, markers beyond
 * the first 32 KiB.  Returns output length (0 on failure); *nsegments = segments actually joined. */
size_t segment_model(const uint8_t* in, size_t n, int want, uint8_t* out, size_t cap, uint64_t* stats, int* nsegments,
                     uint64_t* scanned_bits)
{
    const uint64_t total = (uint64_t)n * 8, first = 16;
    uint64_t cand[256];
    int      nc = 0;
    *scanned_bits = 0;
    if (want > 256) want = 256;
    for (int k = 1; k < want; ++k) {  /* the search a GPU thread per bit offset would run */
        uint64_t t = first + (total - first) * (uint64_t)k / (uint64_t)want, hb;
        for (uint64_t p = t; p + 17 <= total; ++p) {
            ++*scanned_bits;
            if (probe_dynamic_header(in, n, p, &hb) == 0) {
                if (!nc || cand[nc - 1] != p) cand[nc++] = p;
                break;
            }
        }
    }
    /* every segment is decoded independently (in parallel on the GPU) ... */
    symbuf*   seg = (symbuf*)calloc((size_t)nc + 1, sizeof(symbuf));
    int*      joins = (int*)malloc(sizeof(int) * ((size_t)nc + 1));
    uint64_t* ends = (uint64_t*)malloc(sizeof(uint64_t) * ((size_t)nc + 1));
    for (int k = 0; k <= nc; ++k) {
        uint64_t start = k ? cand[k - 1] : first;
        joins[k] = decode_segment(in, n, start, cand + k, nc - k, k == 0, &seg[k], &ends[k]);
        if (joins[k] >= 0) joins[k] += k;  /* index into cand[] of the boundary reached, nc = end of stream */
    }
    /* ... and chained afterwards: follow the joins from segment 0; segments nobody arrives at are dropped */
    size_t o = 0;
    int    k = 0, used = 0;
    for (;;) {
        if (joins[k] < 0) { o = 0; break; }
        const symbuf* s = &seg[k];
        uint64_t markers = 0, late = 0;
        if (o + s->n > cap) { o = 0; break; }
        for (size_t i = 0; i < s->n; ++i) {
            uint16_t v = s->sym[i];
            if (v >= 256) {
                const size_t reach = 32768u - (size_t)(v - 256);  /* bytes in front of the segment start */
                if (reach > o) { o = 0; goto done; }
                v = out[o - reach];
                ++markers;
                if (i >= 32768) ++late;
            }
            out[o + i] = (uint8_t)v;
        }
        stats[4 * used] = k ? cand[k - 1] : first, stats[4 * used + 1] = s->n, stats[4 * used + 2] = markers, stats[4 * used + 3] = late;
        ++used;
        o += s->n;
        if (joins[k] == nc) break;  /* reached the end of the stream */
        k = joins[k] + 1;           /* cand[joins[k]] is where segment joins[k] + 1 started */
    }
done:
    *nsegments = used;
    for (int i = 0; i <= nc; ++i) free(seg[i].sym);
    free(seg), free(joins), free(ends);
    return o;
}
