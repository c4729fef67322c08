/*
 * tests/deflate_stream.c -- CPU restatement of LZ77.Deflator's *streaming* behaviour: push(_:last:), pop(), pull()
 * (Sources/LZ77/Deflator/LZ77.Deflator.swift:8-44).  Test infrastructure only, next to the one-shot orc_deflate of
 * oracle/lz77_deflate.c, whose window, match, graph, tree and block writer it shares by including that file; only
 * the input queue, compress(all:) with its lookahead and the chunk queue are restated here.  Built by
 * tests/deflate_stream.py together with oracle/lz77_inflate.c (Adler-32, CRC-32).
 *
 * The compressed bytes do not depend on push granularity (SURVEY.md section 8a E4), so the concatenated chunks equal
 * orc_deflate's stream; what this pins is *when* each byte becomes available.
 */
#include "../oracle/lz77_deflate.c"

typedef struct orc_deflator {
    deflator z;                /* z.x / z.n: every byte pushed so far */
    int      format;
    size_t   chunk;            /* DeflatorOut queues 2 x capacity bytes at a time */
    uint8_t* in;
    size_t   in_cap;
    size_t   graph_cap;        /* vertices allocated in z.graph */
    size_t   at;               /* output bytes handed out */
    uint64_t blocks;
    int      finished;
} orc_deflator;

/* DeflatorBuffers.init (DeflatorBuffers.swift:50-65, Gzip :100-112): the stream header is written at creation */
orc_deflator* orc_deflator_create(int format, int level, int exponent, size_t chunk)
{
    init_tables();
    if (exponent < 8 || exponent > 15 || format < 0 || format > 2 || !chunk) return NULL;
    if (format == ORC_FORMAT_IOS) exponent = 15;
    orc_deflator* d = (orc_deflator*)calloc(1, sizeof *d);
    deflator*     z = &d->z;
    d->format = format;
    d->chunk = chunk;
    z->search = search_for(level);
    z->mask = ((int64_t)1 << exponent) - 1;
    z->end_index = -3;
    z->limit = 2048;
    if (z->search.mode == MODE_FULL) {
        z->capacity = (int64_t)1 << 21;
        depths_init(&z->depths);
    } else {
        z->capacity = 1 << 15;
        z->terms = (term_t*)malloc(sizeof(term_t) * 2048);
    }
    z->head = (int32_t*)malloc(sizeof(int32_t) << HASH_BITS);
    for (size_t i = 0; i < ((size_t)1 << HASH_BITS); ++i) z->head[i] = -1;
    z->prevh = (int32_t*)malloc(sizeof(int32_t) * (size_t)(z->mask + 1));
    z->next = (int32_t*)malloc(sizeof(int32_t) * (size_t)(z->mask + 1));
    z->out.cap = 4096;
    z->out.p = (uint8_t*)malloc(z->out.cap);
    if (format == ORC_FORMAT_ZLIB) {
        uint32_t unpaired = (uint32_t)(exponent - 8) << 4 | 8;
        uint32_t check = ~(((unpaired << 8) | (unpaired >> 8)) % 31) & 31;
        put_bits(&z->out, check << 8 | unpaired, 16);
    } else if (format == ORC_FORMAT_GZIP) {
        put_bits(&z->out, 0x8b1f, 16); put_bits(&z->out, 0x0008, 16);
        put_bits(&z->out, 0, 16); put_bits(&z->out, 0, 16); put_bits(&z->out, 0xff00, 16);
    }
    return d;
}

void orc_deflator_destroy(orc_deflator* d)
{
    if (!d) return;
    free(d->z.head); free(d->z.prevh); free(d->z.next); free(d->z.terms); free(d->z.graph);
    free(d->z.out.p); free(d->in);
    free(d);
}

/* Stream.compress(all:), Stream.swift:195-404 with lookahead = all ? 0 : 258 (greedy, full) or 259 (lazy) (:210, :269,
 * :345).  The lookahead is tested at a head position only: full mode consumes a long match's skip vertices (:376)
 * whatever is pending, and a buffer that fills exactly as the lookahead is reached waits for a later push (:219, :277,
 * :353).  Returns 1 when the match buffer is full. */
static int compress_stream(deflator* z, int all)
{
    const int64_t lookahead = all ? 0 : z->search.mode == MODE_LAZY ? 259 : 258;
    while (z->end_index < 0 && input_count(z) > lookahead) { /* DeflatorWindow.initialize */
        z->end_index += 1;
        z->dequeued += 1;
    }
    int64_t next;
    if (z->search.mode == MODE_GREEDY) {
        while (input_count(z) > lookahead) {
            if (unfilled(z) <= 0) return 1;
            int64_t a = window_update(z, &next);
            best_t  m;
            if (window_best(z, a, next, &m)) {
                for (int k = 1; k < m.run; ++k) window_update(z, NULL);
                store_match(z, m.run, m.distance);
            } else {
                store_literal(z, literal_at(z, a));
            }
        }
    } else if (z->search.mode == MODE_LAZY) {
        while (input_count(z) > lookahead) {
            if (unfilled(z) <= 1) return 1;
            int64_t a = window_update(z, &next);
            uint8_t first = literal_at(z, a);
            best_t  eager, lazy;
            if (window_best(z, a, next, &eager)) {
                int64_t a1 = window_update(z, &next);
                if (window_best(z, a1, next, &lazy) && eager.run < lazy.run) {
                    store_literal(z, first);
                    store_match(z, lazy.run, lazy.distance);
                    for (int k = 1; k < lazy.run; ++k) window_update(z, NULL);
                } else {
                    store_match(z, eager.run, eager.distance);
                    for (int k = 2; k < eager.run; ++k) window_update(z, NULL);
                }
            } else {
                store_literal(z, first);
            }
        }
    } else {
        while (input_count(z) > lookahead) {
            if (unfilled(z) <= 0) return 1;
            int64_t  a = window_update(z, &next);
            edge_ctx e = {z, store_vertex(z, literal_at(z, a)), 1};
            window_match(z, a, next, edge_delegate, &e);
            int64_t skip = e.extent - 100 < unfilled(z) ? e.extent - 100 : unfilled(z);
            for (int64_t k = 0; k < skip; ++k) {
                int64_t b = window_update(z, NULL);
                store_vertex(z, literal_at(z, b));
            }
        }
    }
    if (!all) return 0; /* guard all else { return nil } */
    int64_t epilogue = -3 - (z->end_index < 0 ? z->end_index : 0);
    while (input_count(z) > epilogue) {
        if (unfilled(z) <= 0) return 1;
        int64_t a = window_update(z, NULL);
        if (z->search.mode == MODE_FULL) store_vertex(z, literal_at(z, a));
        else store_literal(z, literal_at(z, a));
    }
    return 0;
}

static void reserve_out(bitout* o, size_t more)
{
    size_t need = (size_t)(o->bits >> 3) + more + 64;
    if (need <= o->cap) return;
    o->cap = need * 2;
    o->p = (uint8_t*)realloc(o->p, o->cap);
}

/* DeflatorBuffers.push(_:last:), DeflatorBuffers.swift:68-137.  Returns 0, or -1 after push(last: true). */
int orc_deflator_push(orc_deflator* d, const uint8_t* data, size_t n, int last)
{
    deflator* z = &d->z;
    if (d->finished) return -1;
    if (n) { /* input.enqueue(contentsOf:) */
        size_t have = (size_t)z->n;
        if (have + n > d->in_cap) {
            d->in_cap = (have + n) * 2;
            d->in = (uint8_t*)realloc(d->in, d->in_cap);
        }
        memcpy(d->in + have, data, n);
        z->n = (int64_t)(have + n);
    }
    z->x = d->in;
    /* guard self.stream.input.count > 4096 || last (:74, :120) */
    if (!(input_count(z) > 4096 || last)) return 0;
    if (z->search.mode == MODE_FULL) { /* a graph for every vertex this push can add to the block */
        size_t want = (size_t)(z->count + z->n - z->end_index);
        if (want > (size_t)z->capacity) want = (size_t)z->capacity;
        if (want + 2 > d->graph_cap) {
            d->graph_cap = want + 2;
            z->graph = (vertex_t*)realloc(z->graph, sizeof(vertex_t) * d->graph_cap);
        }
    }
    reserve_out(&z->out, orc_deflate_bound((size_t)(z->count * 8 + z->n - z->end_index)));
    /* Stream.compressBlocks(final:), Stream.swift:30-60 */
    if (!last) {
        while (compress_stream(z, 0)) write_block(z, 0), d->blocks++;
        return 0;
    }
    if (z->n >= 3) {
        while (compress_stream(z, 1)) write_block(z, 0), d->blocks++;
        write_block(z, 1);
    } else { /* stored final block, :45-60 and :417-435, whichever pushes brought the bytes */
        put_bits(&z->out, 1, 3);
        pad_to_byte(&z->out);
        put_bits(&z->out, (uint32_t)z->n, 16);
        put_bits(&z->out, ~(uint32_t)z->n & 0xffff, 16);
        for (int64_t i = 0; i < z->n; ++i) put_bits(&z->out, d->in[i], 8);
    }
    d->blocks++;
    /* trailers, :80-91 and :123-136 */
    if (d->format == ORC_FORMAT_ZLIB) put_be32(&z->out, orc_adler32(1, d->in, (size_t)z->n));
    else if (d->format == ORC_FORMAT_GZIP) {
        put_le32(&z->out, orc_crc32(0, d->in, (size_t)z->n));
        put_le32(&z->out, (uint32_t)z->n);
    }
    pad_to_byte(&z->out);
    d->finished = 1;
    return 0;
}

/* DeflatorOut (DeflatorOut.swift:105-135) queues a chunk the moment its buffer fills: pop() hands out complete chunks */
int orc_deflator_pop(orc_deflator* d, const uint8_t** chunk, size_t* n)
{
    size_t complete = (size_t)(d->z.out.bits >> 3);
    if (complete - d->at < d->chunk) return 0;
    *chunk = d->z.out.p + d->at;
    *n = d->chunk;
    d->at += d->chunk;
    return 1;
}

/* pull(): a complete chunk, else after push(last: true) the flushed rest, else nothing.  Before `last` the reference
 * flushes a byte-padded partial buffer (DeflatorOut.swift:96-101), which corrupts the rest of the stream; this
 * restatement, like the library, hands out nothing there. */
int orc_deflator_pull(orc_deflator* d, const uint8_t** chunk, size_t* n)
{
    if (orc_deflator_pop(d, chunk, n)) return 1;
    size_t complete = (size_t)(d->z.out.bits >> 3);
    if (!d->finished || d->at >= complete) return 0;
    *chunk = d->z.out.p + d->at;
    *n = complete - d->at;
    d->at = complete;
    return 1;
}

/* out[0] input bytes dequeued, out[1] complete bytes written (header included), out[2] blocks, out[3] pending input */
void orc_deflator_progress(const orc_deflator* d, uint64_t out[4])
{
    const int64_t taken = d->z.dequeued < d->z.n ? d->z.dequeued : d->z.n; /* the epilogue dequeues 3 bytes past the end */
    out[0] = (uint64_t)taken;
    out[1] = d->z.out.bits >> 3;
    out[2] = d->blocks;
    out[3] = (uint64_t)(d->z.n - taken);
}
