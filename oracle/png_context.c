/*
 * oracle/png_context.c -- CPU restatement of swift-png's online decoding.  TEST INFRASTRUCTURE ONLY (see oracle.h).
 *
 * Follows (paths relative to the reference checkout):
 *   Sources/PNG/Decoding/PNG.Context.swift:55-100     PNG.Context.init / push(data:overdraw:)   (create, push)
 *   Sources/PNG/Decoding/PNG.Context.swift:134-141    push(ancillary:) with IEND                 (end)
 *   Sources/PNG/Decoding/PNG.Decoder.swift:47-149     PNG.Decoder.push: the resumable row loop   (push)
 *   Sources/PNG/PNG.Image.swift:133-183               PNG.Image.overdraw                         (overdraw)
 *   Sources/PNG/PNG.Image.swift:186-285               PNG.Image.assign                           (assign)
 *
 * What the reference's inflator makes available after a push depends only on the bytes pushed so far, so it is taken
 * from the one-shot orc_inflate of that prefix (its status NEED_MORE_INPUT, its `produced`); orc_inflate releases a
 * stored block's payload byte by byte as Stream.readBlock(upTo:) does (Stream.swift:384-399).
 */
#include "oracle.h"

#include <stdlib.h>
#include <string.h>

/* Entry points (bound by tests/png_context_cases.py):
 *   orc_png_context* orc_png_context_create(w, h, volume, depth, interlaced, standard)   standard 0 zlib, 1 ios
 *   int  orc_png_context_push(c, data, n, overdraw)    ORC_OK or an error; an inflate error is sticky
 *   int  orc_png_context_end(c)                        ORC_OK iff the stream is complete
 *   void orc_png_context_progress(c, out[6])           next pass (7 when done), next row, filtered bytes consumed,
 *                                                      stream complete, storage rows [out[4], out[5]) the last push wrote
 *   const uint8_t* orc_png_context_storage(c)          PNG.Image.storage, w * h * ((volume + 7) >> 3) bytes
 *   void orc_png_context_error(c, &status, &a, &b), orc_png_context_destroy(c) */
typedef struct orc_png_context orc_png_context;

static const int ADAM7[7][4] = {/* base.x, base.y, exponent.x, exponent.y, PNG.Decoder.swift:6-15 */
                                {0, 0, 3, 3}, {4, 0, 3, 3}, {0, 4, 2, 3}, {2, 0, 2, 2},
                                {0, 2, 1, 2}, {1, 0, 1, 1}, {0, 1, 0, 1}};

struct orc_png_context {
    uint32_t w, h;
    int      volume, depth, interlaced, format;
    uint8_t* storage;
    uint8_t* input;       /* everything pushed */
    size_t   input_len, input_cap;
    uint8_t* filtered;    /* the inflated prefix */
    size_t   filtered_cap;
    size_t   consumed;    /* filtered bytes pulled */
    int      pass;        /* PNG.Decoder.pass: 7 once every row is assigned */
    uint64_t row;         /* PNG.Decoder.row.index */
    uint8_t* last;        /* PNG.Decoder.row.reference (pitch + 1 bytes of the current pass) */
    int      terminal;    /* continue == nil */
    int      status;
    uint32_t a, b;
    uint64_t band0, band1;
};

typedef struct { int bx, by, ex, ey; uint64_t w, h, pitch; } cpass;

static cpass pass_of(const orc_png_context* c, int z)
{
    cpass p = {0, 0, 0, 0, 0, 0, 0};
    if (!c->interlaced) {
        if (z == 0) p.w = c->w, p.h = c->h;
    } else {
        p.bx = ADAM7[z][0], p.by = ADAM7[z][1], p.ex = ADAM7[z][2], p.ey = ADAM7[z][3];
        p.w = ((uint64_t)c->w + (1u << p.ex) - (uint64_t)p.bx - 1) >> p.ex;
        p.h = ((uint64_t)c->h + (1u << p.ey) - (uint64_t)p.by - 1) >> p.ey;
        if (p.w == 0 || p.h == 0) p.w = p.h = 0;
    }
    p.pitch = (p.w * (uint64_t)c->volume + 7) >> 3;
    return p;
}

orc_png_context* orc_png_context_create(uint32_t w, uint32_t h, int volume, int depth, int interlaced, int standard)
{
    orc_png_context* c = (orc_png_context*)calloc(1, sizeof *c);
    c->w = w, c->h = h, c->volume = volume, c->depth = depth, c->interlaced = interlaced;
    c->format = standard ? ORC_FORMAT_IOS : ORC_FORMAT_ZLIB;
    c->storage = (uint8_t*)calloc((size_t)w * h * (size_t)((volume + 7) >> 3) + 1, 1);   /* uninitialized: false */
    return c;
}

void orc_png_context_destroy(orc_png_context* c)
{
    if (!c) return;
    free(c->storage), free(c->input), free(c->filtered), free(c->last);
    free(c);
}

/* PNG.Image.assign, PNG.Image.swift:186-285 (scanline without its filter byte) */
static void assign(orc_png_context* c, const uint8_t* scanline, int bx, uint64_t y, int stride)
{
    size_t i = 0, bpp = (size_t)((c->volume + 7) >> 3);
    for (uint64_t x = (uint64_t)bx; x < c->w; x += (uint64_t)stride, ++i) {
        uint8_t* dst = c->storage + bpp * (y * c->w + x);
        if (c->depth < 8) {
            int per = 8 / c->depth;
            *dst = (uint8_t)((scanline[i / (size_t)per] >> ((int)((~i) & (size_t)(per - 1)) * c->depth)) &
                             ((1 << c->depth) - 1));
        } else {
            memcpy(dst, scanline + bpp * i, bpp);
        }
    }
}

/* PNG.Image.overdraw(at:brush:), PNG.Image.swift:133-183: the element is the pixel's (volume + 7) >> 3 bytes */
static void overdraw(orc_png_context* c, int bx, uint64_t by, uint64_t brx, uint64_t bry)
{
    if (brx * bry <= 1) return;
    size_t bpp = (size_t)((c->volume + 7) >> 3);
    for (uint64_t y = by; y < by + bry && y < c->h; ++y)
        for (uint64_t x = (uint64_t)bx; x < c->w; x += brx) {
            const uint8_t* src = c->storage + bpp * (by * c->w + x);
            for (uint64_t x2 = x; x2 < x + brx && x2 < c->w; ++x2)
                memmove(c->storage + bpp * (y * c->w + x2), src, bpp);
        }
}

int orc_png_context_push(orc_png_context* c, const uint8_t* data, size_t n, int draw)
{
    c->band0 = c->band1 = 0;
    if (c->status < 0) return c->status;
    if (c->terminal) return ORC_ERR_PNG_EXTRANEOUS_COMPRESSED_DATA; /* PNG.Decoder.swift:51-55 */
    if (c->input_len + n > c->input_cap) {
        c->input_cap = 2 * (c->input_len + n) + 64;
        c->input = (uint8_t*)realloc(c->input, c->input_cap);
    }
    if (n) memcpy(c->input + c->input_len, data, n);
    c->input_len += n;
    /* self.continue = try self.inflator.push(data) */
    orc_inflate_result r;
    if (!c->filtered) { /* a null output would measure instead of decoding */
        c->filtered_cap = 65536;
        c->filtered = (uint8_t*)malloc(c->filtered_cap);
    }
    for (;;) {
        orc_inflate(c->format, c->input, c->input_len, c->filtered, c->filtered_cap, &r);
        if (r.status != ORC_ERR_OUTPUT_CAPACITY) break;
        c->filtered_cap *= 2;
        c->filtered = (uint8_t*)realloc(c->filtered, c->filtered_cap);
    }
    if (r.status < 0) {
        c->a = r.a, c->b = r.b;
        return c->status = r.status;
    }
    c->terminal = r.status == ORC_OK;
    const size_t avail = (size_t)r.produced;
    const int    delay = (c->volume + 7) >> 3;
    uint64_t     lo = c->h, hi = 0;
    for (; c->pass < 7; ++c->pass, c->row = 0) {
        const cpass p = pass_of(c, c->pass);
        if (p.h == 0) continue;
        const size_t count = (size_t)p.pitch + 1;
        if (c->row == 0) {
            free(c->last);
            c->last = (uint8_t*)calloc(count, 1);
        }
        uint8_t* line = (uint8_t*)malloc(count);
        for (; c->row < p.h; ++c->row) {
            if (c->consumed + count > avail) break; /* inflator.pull(count) == nil */
            memcpy(line, c->filtered + c->consumed, count);
            c->consumed += count;
            orc_defilter(line, c->last, count, delay);
            const uint64_t y = (uint64_t)p.by + (c->row << p.ey);
            assign(c, line + 1, p.bx, y, 1 << p.ex);
            uint64_t end = y + 1;
            if (draw) { /* PNG.Context.swift:89-95 */
                const uint64_t brx = (1u << p.ex) >> (p.bx != 0), bry = (1u << p.ey) >> ((y & 7) != 0);
                overdraw(c, p.bx, y, brx, bry);
                if (brx * bry > 1) end = y + bry < c->h ? y + bry : c->h;
            }
            if (y < lo) lo = y;
            if (end > hi) hi = end;
            memcpy(c->last, line, count);
        }
        free(line);
        if (c->row < p.h) break;
    }
    if (hi) c->band0 = lo, c->band1 = hi;
    if (c->pass == 7) {
        c->row = 0;
        if (avail > c->consumed) { /* guard self.inflator.pull().isEmpty, PNG.Decoder.swift:142-147 */
            c->consumed = avail;
            return ORC_ERR_PNG_EXTRANEOUS_IMAGE_DATA;
        }
    }
    return ORC_OK;
}

int orc_png_context_end(const orc_png_context* c)
{
    return c->terminal ? ORC_OK : ORC_ERR_PNG_INCOMPLETE_DATASTREAM; /* PNG.Context.swift:134-141 */
}

void orc_png_context_progress(const orc_png_context* c, uint64_t out[6])
{
    out[0] = (uint64_t)c->pass, out[1] = c->row, out[2] = c->consumed, out[3] = (uint64_t)c->terminal;
    out[4] = c->band0, out[5] = c->band1;
}

const uint8_t* orc_png_context_storage(const orc_png_context* c) { return c->storage; }

void orc_png_context_error(const orc_png_context* c, int* status, uint32_t* a, uint32_t* b)
{
    *status = c->status < 0 ? c->status : ORC_OK, *a = c->a, *b = c->b;
}
