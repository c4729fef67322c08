// png_file.cuh -- file-level entry points (SURVEY.md section 8f row N2): whole PNG files in, pixels out,
// and back.  Included at the end of pngb200_api.cu (uses the context internals defined there).
//
// The reference's PNG.Image.decompress(stream:) (Sources/PNG/PNG.Image.swift:298-401) interleaves
// lexing, per-chunk CRC-32, chunk parsing and decoding, one chunk at a time, on the host.  Here the
// host only walks chunk HEADERS (8 bytes per chunk); every payload byte is touched on the device:
// the file goes to HBM once, crc_regions_kernel checks all chunks of all files in one launch,
// segment_copy_kernel concatenates IDAT bodies when a file has more than one, and the batch decode
// path runs on the result.  Errors are reported in the order the reference's streaming loop would
// meet them (see resolve order below).  Encode mirrors compress(stream:level:hint:) (:576-670).
// Files already in device memory take the same path with the walk on the device (png_walk.cuh): nothing is staged
// but the gathered IDAT run, and an encoded file is written where the caller wants it.
#pragma once

namespace {

const uint8_t PNG_SIGNATURE[8] = {137, 80, 78, 71, 13, 10, 26, 10};

inline void store_be32(uint8_t* p, uint32_t v) { p[0] = (uint8_t)(v >> 24), p[1] = (uint8_t)(v >> 16), p[2] = (uint8_t)(v >> 8), p[3] = (uint8_t)v; }

// What the chunk walk (png_walk.cuh) learned about one file, with every lexed chunk's record
struct FileWalk {
    std::vector<ChunkRec> chunks;
    int      status = PNGB200_OK;
    uint32_t a = 0, b = 0;
    size_t   stop = (size_t)-1;
    bool     stop_before_crc = false;
    size_t   first_idat = (size_t)-1, idat_end = 0;  // [first_idat, idat_end): the contiguous IDAT run
};

// the out fields of `d` and the scalars of `w` from a walk's summary; `palette`: the palette the walk wrote, null when
// it wrote into d.palette_rgba itself
void take_walk(const WalkHead& h, const uint8_t* palette, pngb200_png_desc& d, FileWalk& w)
{
    d.width = h.width, d.height = h.height;
    d.depth = h.depth, d.color = h.color, d.interlaced = h.interlaced, d.standard = h.standard;
    d.format = h.format;
    d.format.palette = d.palette_rgba;
    if (palette) memcpy(d.palette_rgba, palette, 4 * (size_t)h.palette_entries);
    d.storage_size = h.storage_size, d.idat_bytes = h.idat_bytes;
    d.idat_chunks = h.idat_chunks, d.chunks = (uint32_t)h.chunks;
    w.status = h.status, w.a = h.a, w.b = h.b;
    w.stop = (size_t)h.stop, w.stop_before_crc = h.stop_before_crc != 0;
    w.first_idat = (size_t)h.first_idat, w.idat_end = (size_t)h.idat_end;
}

// one chunk onto `h`: length, type, body and CRC-32 (these few bytes are CRC'd where they are built)
void put_chunk(std::vector<uint8_t>& h, uint32_t type, const uint8_t* body, size_t n)
{
    const size_t at = h.size();
    h.resize(at + 12 + n);
    store_be32(h.data() + at, (uint32_t)n), store_be32(h.data() + at + 4, type);
    if (n) memcpy(h.data() + at + 8, body, n);
    uint32_t c = 0xffffffffu;
    for (size_t k = at + 4; k < at + 8 + n; ++k) {
        c ^= h[k];
        for (int b = 0; b < 8; ++b) c = (c & 1) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    }
    store_be32(h.data() + at + 8 + n, ~c);
}

// Everything in front of the first IDAT, built on the host (a few hundred bytes): signature, [CgBI], IHDR, [PLTE],
// [tRNS]  (PNG.Image.swift:580-629, PNG.Image.encode :416-423, Layout.palette / Layout.transparency,
// Formats/PNG.Layout.swift:43-135)
void png_head(const pngb200_pixel_format& f, uint32_t width, uint32_t height, int interlaced, std::vector<uint8_t>& h)
{
    h.assign(PNG_SIGNATURE, PNG_SIGNATURE + 8);
    if (f.bgr) {
        const uint8_t cgbi[4] = {48, 0, 32, (uint8_t)(f.color == 2 ? 6 : 2)};
        put_chunk(h, CK_CgBI, cgbi, 4);
    }
    uint8_t ihdr[13];
    store_be32(ihdr, width), store_be32(ihdr + 4, height);
    ihdr[8] = f.depth, ihdr[9] = f.color, ihdr[10] = 0, ihdr[11] = 0, ihdr[12] = interlaced ? 1 : 0;
    put_chunk(h, CK_IHDR, ihdr, 13);
    if (f.color == 3) {
        uint8_t rgb[768], alpha[256];
        int last = -1;
        for (int k = 0; k < f.palette_count; ++k) {
            memcpy(rgb + 3 * k, f.palette + 4 * k, 3);
            alpha[k] = f.palette[4 * k + 3];
            if (alpha[k] != 255) last = k;
        }
        put_chunk(h, CK_PLTE, rgb, 3 * (size_t)f.palette_count);
        if (last >= 0) put_chunk(h, CK_tRNS, alpha, (size_t)last + 1);
    } else if (f.has_key && (f.color == 0 || f.color == 2)) {
        uint8_t k[6];
        if (f.color == 0) {
            k[0] = (uint8_t)(f.key[0] >> 8), k[1] = (uint8_t)f.key[0];
            put_chunk(h, CK_tRNS, k, 2);
        } else {
            const uint16_t r = f.bgr ? f.key[2] : f.key[0], g = f.key[1], b = f.bgr ? f.key[0] : f.key[2];
            k[0] = (uint8_t)(r >> 8), k[1] = (uint8_t)r, k[2] = (uint8_t)(g >> 8), k[3] = (uint8_t)g, k[4] = (uint8_t)(b >> 8), k[5] = (uint8_t)b;
            put_chunk(h, CK_tRNS, k, 6);
        }
    }
}

// the format checks of pngb200_png_encode_files: a pixel format the PNG layout allows, a palette that fits its depth
bool encode_format_ok(const pngb200_pixel_format& f, uint32_t width, uint32_t height)
{
    return pixel_rule(f.color, f.depth, f.bgr).valid && width && height &&
           !(f.color == 3 && (!f.palette || !f.palette_count || f.palette_count > (1u << f.depth)));
}

struct RecordVector {
    std::vector<ChunkRec>* v;
    void put(uint64_t, const ChunkRec& r) const { v->push_back(r); }
};

// the walk of a host file, on the host
void walk_file(pngb200_png_desc& d, FileWalk& w)
{
    WalkHead h;
    w.chunks.clear();
    walk_png<false>(d.file, d.file_len, h, d.palette_rgba, RecordVector{&w.chunks}, true);
    take_walk(h, nullptr, d, w);
}

// The walk of device files, on the device (png_walk_kernel): pass 1 fills the out fields of `d` and the scalars of
// `walks`; with `records`, pass 2 brings every chunk's record back too (24 bytes a chunk), into record arrays sized
// from pass 1's counts.  The summaries and records pass through the file arena, which a device-file batch does not
// otherwise use.
int walk_device_files(pngb200_ctx* ctx, pngb200_png_desc* d, size_t count, std::vector<FileWalk>& walks, bool records)
{
    std::vector<WalkFile> files(count);
    for (size_t i = 0; i < count; ++i) {
        if (!d[i].file && d[i].file_len) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "file %zu: null pointer", i);
        files[i] = {d[i].file, d[i].file_len};
    }
    if (count == 0) return PNGB200_OK;
    if (count > 0xffffffffu) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "batch too large");
    const unsigned grid = (unsigned)((count + WALK_WARPS - 1) / WALK_WARPS);
    const size_t   sum_bytes = sizeof(WalkSummary) * count;
    std::vector<uint64_t> base(count + 1, 0);
    {
        Tables t(ctx->h_genjobs, ctx->d_file);
        const size_t off_files = t.host(files.data(), sizeof(WalkFile) * count);
        const size_t off_sums = t.device(sum_bytes, false);
        if (int rc = t.upload(ctx, t.end)) return rc;
        png_walk_kernel<<<grid, WALK_WARPS * 32, 0, ctx->stream>>>(t.dev<WalkFile>(off_files), (uint32_t)count,
                                                                   t.dev<WalkSummary>(off_sums), nullptr, nullptr);
        ctx->launches++;
        CU(cudaGetLastError());
        CU(cudaMemcpyAsync(t.pin<WalkSummary>(off_sums), t.dev<WalkSummary>(off_sums), sum_bytes, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        for (size_t i = 0; i < count; ++i) {
            const WalkSummary& s = t.pin<WalkSummary>(off_sums)[i];
            take_walk(s.head, s.palette_rgba, d[i], walks[i]);
            base[i + 1] = base[i] + s.head.chunks;
        }
    }
    if (!records || base[count] == 0) return PNGB200_OK;
    Tables t(ctx->h_genjobs, ctx->d_file);
    const size_t off_files = t.host(files.data(), sizeof(WalkFile) * count);
    const size_t off_base = t.host(base.data(), sizeof(uint64_t) * (count + 1));
    const size_t off_sums = t.device(sum_bytes, false);
    const size_t off_recs = t.device(sizeof(ChunkRec) * base[count], false);
    if (int rc = t.upload(ctx, t.end)) return rc;
    png_walk_kernel<<<grid, WALK_WARPS * 32, 0, ctx->stream>>>(t.dev<WalkFile>(off_files), (uint32_t)count, t.dev<WalkSummary>(off_sums),
                                                               t.dev<ChunkRec>(off_recs), t.dev<uint64_t>(off_base));
    ctx->launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(t.pin<ChunkRec>(off_recs), t.dev<ChunkRec>(off_recs), sizeof(ChunkRec) * base[count], cudaMemcpyDeviceToHost,
                       ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < count; ++i)
        walks[i].chunks.assign(t.pin<ChunkRec>(off_recs) + base[i], t.pin<ChunkRec>(off_recs) + base[i + 1]);
    return PNGB200_OK;
}

// CRC-32 of `regions` (device pointers) in three enqueue steps, so that a caller can put the small
// table upload in front of its bulk H2D copies and the small result download behind its kernels (copies
// of one direction are served in issue order across all streams: a few KB queued behind another lane's
// gigabyte would stall this lane for its whole duration).
struct CrcPlan {
    CrcParams p;
    size_t    acc_bytes = 0, off_acc = 0;
    bool      any = false;
};
// The first piece of each item (CrcRegion or CopySegment: CRC_PIECE bytes a piece, at least one per item), then the
// total, in `base`; false when the pieces do not fit a launch
template <typename Item>
bool piece_bases(const std::vector<Item>& items, std::vector<uint32_t>& base)
{
    base.resize(items.size() + 1);
    uint64_t pieces = 0;
    for (size_t i = 0; i < items.size(); ++i) {
        base[i] = (uint32_t)pieces;
        pieces += std::max<uint64_t>(1, (items[i].len + CRC_PIECE - 1) / CRC_PIECE);
    }
    base[items.size()] = (uint32_t)pieces;
    return pieces < (1ull << 31);
}
int crc_upload(pngb200_ctx* ctx, const std::vector<CrcRegion>& regions, uint32_t* d_acc_out, CrcPlan* plan)
{
    const size_t count = regions.size();
    plan->any = count != 0;
    if (count == 0) return PNGB200_OK;
    int rc = ensure_crc_tables(ctx);
    if (rc != PNGB200_OK) return rc;
    std::vector<uint32_t> base;
    if (!piece_bases(regions, base)) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "batch too large");
    const size_t ab = sizeof(uint32_t) * count;
    Tables t(ctx->h_crc, ctx->d_crc);
    const size_t off_regions = t.host(regions.data(), sizeof(CrcRegion) * count);
    const size_t off_base = t.host(base.data(), sizeof(uint32_t) * (count + 1));
    const size_t off_acc = t.device(ab, false);
    if ((rc = t.upload(ctx, t.end)) != PNGB200_OK) return rc;   // crc_fetch brings the results back behind the tables
    uint32_t* acc = d_acc_out ? d_acc_out : t.dev<uint32_t>(off_acc);
    CU(cudaMemsetAsync(acc, 0, ab, ctx->stream));
    plan->p.regions = t.dev<CrcRegion>(off_regions);
    plan->p.piece_base = t.dev<uint32_t>(off_base);
    plan->p.acc = acc;
    plan->p.tables = ctx->d_crctab.as<uint32_t>();
    plan->p.count = (uint32_t)count;
    plan->p.total_pieces = base[count];
    plan->acc_bytes = ab, plan->off_acc = off_acc;
    return PNGB200_OK;
}
int crc_launch(pngb200_ctx* ctx, const CrcPlan& plan)
{
    if (!plan.any) return PNGB200_OK;
    crc_regions_kernel<<<plan.p.total_pieces, CRC_THREADS, 0, ctx->stream>>>(plan.p);
    ctx->launches++;
    CU(cudaGetLastError());
    return PNGB200_OK;
}
// enqueue the download of the results into pinned memory; valid after the stream's next synchronisation
int crc_fetch(pngb200_ctx* ctx, const CrcPlan& plan, const uint32_t** pinned_out)
{
    *pinned_out = nullptr;
    if (!plan.any) return PNGB200_OK;
    CU(cudaMemcpyAsync((char*)ctx->h_crc.p + plan.off_acc, plan.p.acc, plan.acc_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    *pinned_out = (const uint32_t*)((char*)ctx->h_crc.p + plan.off_acc);
    return PNGB200_OK;
}
// all three at once; host_out: wait for the results
int run_crc(pngb200_ctx* ctx, const std::vector<CrcRegion>& regions, uint32_t* d_acc_out, std::vector<uint32_t>* host_out)
{
    CrcPlan plan;
    int rc = crc_upload(ctx, regions, d_acc_out, &plan);
    if (rc == PNGB200_OK) rc = crc_launch(ctx, plan);
    if (rc != PNGB200_OK || !host_out || !plan.any) return rc;
    const uint32_t* pinned = nullptr;
    rc = crc_fetch(ctx, plan, &pinned);
    if (rc != PNGB200_OK) return rc;
    CU(cudaStreamSynchronize(ctx->stream));
    host_out->assign(pinned, pinned + regions.size());
    return PNGB200_OK;
}

struct CopyPlan {
    CopyParams p;
    bool       any = false;
};
int copy_upload(pngb200_ctx* ctx, const std::vector<CopySegment>& segs, CopyPlan* plan)
{
    const size_t count = segs.size();
    plan->any = count != 0;
    if (count == 0) return PNGB200_OK;
    std::vector<uint32_t> base;
    if (!piece_bases(segs, base)) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "batch too large");
    Tables t(ctx->h_seg, ctx->d_seg);
    const size_t off_segs = t.host(segs.data(), sizeof(CopySegment) * count);
    const size_t off_base = t.host(base.data(), sizeof(uint32_t) * (count + 1));
    if (int rc = t.upload(ctx)) return rc;
    plan->p.segments = t.dev<CopySegment>(off_segs);
    plan->p.piece_base = t.dev<uint32_t>(off_base);
    plan->p.count = (uint32_t)count;
    plan->p.total_pieces = base[count];
    return PNGB200_OK;
}
int copy_launch(pngb200_ctx* ctx, const CopyPlan& plan)
{
    if (!plan.any) return PNGB200_OK;
    segment_copy_kernel<<<plan.p.total_pieces, CRC_THREADS, 0, ctx->stream>>>(plan.p);
    ctx->launches++;
    CU(cudaGetLastError());
    return PNGB200_OK;
}
int run_segment_copy(pngb200_ctx* ctx, const std::vector<CopySegment>& segs)
{
    CopyPlan plan;
    int rc = copy_upload(ctx, segs, &plan);
    return rc != PNGB200_OK ? rc : copy_launch(ctx, plan);
}

// One chunk of a png_decode batch on one context.  `optimistic`: the chunk CRCs are computed on the
// device while the decode is already running on the assumption that they all match (no host round trip
// between the two); the rare file whose CRC failure changes what the decoder may see -- a bad chunk
// before the end of its IDAT run -- is put through the exact order once more (`optimistic` = false:
// CRCs first, then the decode of just the IDAT chunks lexed before the failure).
// `device_files`: every d[i].file is device memory.  The walk then runs on the device, CRC regions point into the
// files themselves and the IDAT run is gathered device to device; nothing else changes.
int png_decode_some(pngb200_ctx* ctx, pngb200_png_desc* d, size_t count, int memspace, bool device_files, bool optimistic = true)
{
    DeviceGuard guard(ctx->device);
    const bool host_pixels = memspace == PNGB200_MEM_HOST;
    std::vector<FileWalk> walks(count);
    if (device_files)
        if (int rc = walk_device_files(ctx, d, count, walks, true)) return rc;
    // Device image of a file: [bytes in front of the first IDAT | bytes behind the IDAT run] in the file
    // arena, and the bodies of the IDAT run back to back in the payload arena.  The H2D copy itself
    // does the concatenation: a run of equal-sized IDAT chunks (what every encoder writes, the reference
    // included) is one pitched copy (cudaMemcpy2DAsync: row = body, source pitch = body + 12).
    std::vector<size_t> f_off(count), g_off(count), pre_len(count), post_at(count), post_len(count);
    Slots files{16}, payloads{16};
    for (size_t i = 0; i < count; ++i) {
        FileWalk& w = walks[i];
        if (!device_files) {
            if (!d[i].file && d[i].file_len) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "file %zu: null pointer", i);
            walk_file(d[i], w);
        }
        d[i].status = PNGB200_OK, d[i].err_a = d[i].err_b = 0;
        d[i].checksum = d[i].blocks = 0, d[i].produced = 0;
        if (w.first_idat != (size_t)-1 && (!d[i].pixels || d[i].pixels_cap < d[i].storage_size))
            return set_error(ctx, PNGB200_ERR_OUTPUT_CAPACITY, "file %zu: pixels_cap %zu < %llu", i, d[i].pixels_cap,
                             (unsigned long long)d[i].storage_size);
        const size_t lexed = w.chunks.empty() ? 0 : (size_t)(w.chunks.back().off + 12 + w.chunks.back().len);
        if (device_files) {
            pre_len[i] = post_at[i] = post_len[i] = 0;  // nothing staged: the CRC pass reads the file where it is
        } else if (w.first_idat == (size_t)-1) {
            pre_len[i] = lexed, post_at[i] = lexed, post_len[i] = 0;
        } else {
            pre_len[i] = (size_t)w.chunks[w.first_idat].off;
            post_at[i] = w.idat_end < w.chunks.size() ? (size_t)w.chunks[w.idat_end].off : lexed;
            post_len[i] = lexed - post_at[i];
        }
        if (!device_files) f_off[i] = files.add(pre_len[i] + post_len[i]);
        g_off[i] = payloads.add(d[i].idat_bytes);
    }
    if (!device_files) CU(ctx->d_file.reserve(std::max<size_t>(files.total, 256)));
    CU(ctx->d_in.reserve(std::max<size_t>(payloads.total, 256)));
    // every lexed chunk's CRC region (type + body): in the device file; else in the file arena, or -- IDAT run -- the
    // body in the payload arena with the type folded in as a prefix
    std::vector<CrcRegion> regions;
    std::vector<size_t>    region_base(count + 1);
    for (size_t i = 0; i < count; ++i) {
        region_base[i] = regions.size();
        const FileWalk& w = walks[i];
        uint8_t* const  meta = ctx->d_file.as<uint8_t>() + f_off[i];
        uint8_t*        body = ctx->d_in.as<uint8_t>() + g_off[i];
        for (size_t k = 0; k < w.chunks.size(); ++k) {
            const ChunkRec& c = w.chunks[k];
            if (device_files) {
                regions.push_back({d[i].file + c.off + 4, (uint64_t)c.len + 4, 0, 0});
            } else if (w.first_idat != (size_t)-1 && k >= w.first_idat && k < w.idat_end) {
                regions.push_back({body, (uint64_t)c.len, CK_IDAT, 1});
                body += c.len;
            } else {
                const size_t at = c.off < pre_len[i] ? (size_t)c.off : pre_len[i] + ((size_t)c.off - post_at[i]);
                regions.push_back({meta + at + 4, (uint64_t)c.len + 4, 0, 0});
            }
        }
    }
    region_base[count] = regions.size();
    const cudaMemcpyKind kind = device_files ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    auto upload_files = [&]() -> int {
        for (size_t i = 0; i < count; ++i) {
            const FileWalk& w = walks[i];
            uint8_t* const  meta = ctx->d_file.as<uint8_t>() + f_off[i];
            if (pre_len[i]) CU(cudaMemcpyAsync(meta, d[i].file, pre_len[i], kind, ctx->stream));
            if (post_len[i]) CU(cudaMemcpyAsync(meta + pre_len[i], d[i].file + post_at[i], post_len[i], kind, ctx->stream));
            if (w.first_idat == (size_t)-1) continue;
            uint8_t* body = ctx->d_in.as<uint8_t>() + g_off[i];
            for (size_t k = w.first_idat; k < w.idat_end;) {
                const uint32_t len = w.chunks[k].len;
                size_t run = 1;
                while (k + run < w.idat_end && w.chunks[k + run].len == len) ++run;
                const uint8_t* src = d[i].file + w.chunks[k].off + 8;
                if (len == 0) {
                } else if (run == 1) {
                    CU(cudaMemcpyAsync(body, src, len, kind, ctx->stream));
                } else {
                    CU(cudaMemcpy2DAsync(body, len, src, (size_t)len + 12, len, run, kind, ctx->stream));
                }
                body += (size_t)len * run;
                k += run;
            }
        }
        return PNGB200_OK;
    };
    std::vector<uint32_t> crc;
    const uint32_t*       crc_late = nullptr;
    int rc = PNGB200_OK;
    if (!optimistic) {
        if ((rc = upload_files()) != PNGB200_OK) return rc;
        if ((rc = run_crc(ctx, regions, nullptr, &crc)) != PNGB200_OK) return rc;
    }
    // Resolve where the reference's loop would have stopped lexing: the first chunk, in file order, with
    // a bad CRC or a structural error (a lexing error precedes that chunk's CRC check, a parsing /
    // ordering error follows it).
    struct Plan { size_t stop; int status; uint32_t a, b; size_t idat_lo, idat_hi; };
    std::vector<Plan> plans(count);
    std::vector<pngb200_image_desc> images;
    std::vector<size_t>             owner;
    std::vector<size_t>             o_off(count);
    Slots outs{16};
    for (size_t i = 0; i < count; ++i) {
        const FileWalk& w = walks[i];
        Plan& p = plans[i];
        p.stop = w.stop, p.status = w.status, p.a = w.a, p.b = w.b;
        for (size_t k = 0; k < w.chunks.size(); ++k) {
            if (optimistic || k > w.stop || (k == w.stop && w.stop_before_crc)) break;
            if (crc[region_base[i] + k] != w.chunks[k].declared) {
                p.stop = k, p.status = PNGB200_ERR_LEX_INVALID_CHUNK_CHECKSUM, p.a = w.chunks[k].declared, p.b = crc[region_base[i] + k];
                break;
            }
        }
        // IDAT chunks pushed into the decoder before lexing stopped
        p.idat_lo = p.idat_hi = 0;
        if (w.first_idat != (size_t)-1 && p.stop > w.first_idat) {
            p.idat_lo = w.first_idat;
            p.idat_hi = std::min(w.idat_end, p.stop);
        }
        if (p.idat_hi == p.idat_lo) continue;
        uint64_t payload = 0;
        for (size_t k = p.idat_lo; k < p.idat_hi; ++k) payload += w.chunks[k].len;
        pngb200_image_desc im;
        memset(&im, 0, sizeof im);
        im.idat = ctx->d_in.as<uint8_t>() + g_off[i];  // the chunks pushed so far are a prefix of the gathered run
        im.idat_len = payload;
        if (host_pixels)
            o_off[i] = outs.add(d[i].storage_size);
        else
            im.pixels = (uint8_t*)d[i].pixels;
        im.pixels_cap = d[i].storage_size;
        im.width = d[i].width, im.height = d[i].height;
        im.volume = (uint8_t)(d[i].depth * pixel_rule(d[i].color, d[i].depth, false).channels), im.depth = d[i].depth;
        im.interlaced = d[i].interlaced;
        im.format = d[i].standard ? PNGB200_FORMAT_IOS : PNGB200_FORMAT_ZLIB;
        images.push_back(im);
        owner.push_back(i);
    }
    if (outs.total) CU(ctx->d_out.reserve(outs.total));
    if (host_pixels)
        for (size_t j = 0; j < images.size(); ++j) images[j].pixels = ctx->d_out.as<uint8_t>() + o_off[owner[j]];
    CrcPlan crc_plan;
    if (optimistic) {
        // issue order: small table, bulk files, kernels, decode, and only then the small CRC download
        if ((rc = crc_upload(ctx, regions, nullptr, &crc_plan)) != PNGB200_OK) return rc;
        if ((rc = upload_files()) != PNGB200_OK) return rc;
        if ((rc = crc_launch(ctx, crc_plan)) != PNGB200_OK) return rc;
    }
    if (!images.empty()) {
        rc = pngb200_decode_batch_enqueue(ctx, images.data(), images.size(), PNGB200_MEM_DEVICE);
        if (rc != PNGB200_OK) return rc;
    }
    if (optimistic && (rc = crc_fetch(ctx, crc_plan, &crc_late)) != PNGB200_OK) return rc;
    if (!images.empty()) {
        rc = pngb200_decode_batch_finish(ctx, images.data(), images.size());
        if (rc != PNGB200_OK) return rc;
    }
    std::vector<size_t> redo;
    std::vector<char>   skip(count, 0);
    if (optimistic) {
        CU(cudaStreamSynchronize(ctx->stream));  // the CRCs have landed in pinned memory
        for (size_t i = 0; i < count; ++i) {
            const FileWalk& w = walks[i];
            for (size_t k = 0; k < w.chunks.size(); ++k) {
                if (k > w.stop || (k == w.stop && w.stop_before_crc)) break;
                const uint32_t computed = crc_late[region_base[i] + k];
                if (computed == w.chunks[k].declared) continue;
                if (k < plans[i].idat_hi && k > plans[i].idat_lo) {
                    redo.push_back(i), skip[i] = 1;  // the decoder was shown IDAT chunks it should not have seen
                } else {
                    plans[i].stop = k, plans[i].status = PNGB200_ERR_LEX_INVALID_CHUNK_CHECKSUM;
                    plans[i].a = w.chunks[k].declared, plans[i].b = computed;
                    if (k <= plans[i].idat_lo && plans[i].idat_hi > plans[i].idat_lo) skip[i] = 2;  // failed before any IDAT
                }
                break;
            }
        }
    }
    for (size_t j = 0; j < images.size(); ++j) {
        const size_t i = owner[j];
        if (skip[i]) continue;
        d[i].checksum = images[j].checksum, d[i].blocks = images[j].blocks, d[i].produced = images[j].produced;
        const bool hard = images[j].status < 0 && images[j].status != PNGB200_ERR_PNG_INCOMPLETE_DATASTREAM;
        if (hard) {
            // the decoder throws while the offending IDAT is pushed, before any later chunk is lexed
            plans[i].status = images[j].status, plans[i].a = images[j].err_a, plans[i].b = images[j].err_b;
        } else if (plans[i].status == PNGB200_OK && images[j].status != PNGB200_OK) {
            plans[i].status = images[j].status;  // IEND while the decoder still expects data
        }
        if (plans[i].status == PNGB200_OK && host_pixels)
            CU(cudaMemcpyAsync(d[i].pixels, images[j].pixels, d[i].storage_size, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < count; ++i) {
        d[i].status = plans[i].status, d[i].err_a = plans[i].a, d[i].err_b = plans[i].b;
        if (skip[i] == 2) d[i].checksum = d[i].blocks = 0, d[i].produced = 0;
    }
    if (!redo.empty()) {
        std::vector<pngb200_png_desc> again(redo.size());
        for (size_t r = 0; r < redo.size(); ++r) again[r] = d[redo[r]];
        rc = png_decode_some(ctx, again.data(), again.size(), memspace, device_files, false);
        if (rc != PNGB200_OK) return rc;
        for (size_t r = 0; r < redo.size(); ++r) {
            d[redo[r]] = again[r];
            d[redo[r]].format.palette = d[redo[r]].palette_rgba;
        }
    }
    return PNGB200_OK;
}

}  // namespace

extern "C" {

int pngb200_png_inspect_files(pngb200_ctx* ctx, pngb200_png_desc* d, size_t count, int file_memspace)
{
    if (!d && count) return PNGB200_ERR_BAD_ARGUMENT;
    std::vector<FileWalk> walks(count);
    auto report = [&](size_t i) {
        const FileWalk& w = walks[i];
        d[i].status = w.status, d[i].err_a = w.a, d[i].err_b = w.b;
        d[i].checksum = d[i].blocks = 0, d[i].produced = 0;
    };
    if (file_memspace == PNGB200_MEM_HOST) {
        for (size_t i = 0; i < count; ++i) {
            if (!d[i].file && d[i].file_len) return PNGB200_ERR_BAD_ARGUMENT;
            walk_file(d[i], walks[i]);
            report(i);
        }
        return PNGB200_OK;
    }
    if (file_memspace != PNGB200_MEM_DEVICE) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "file_memspace %d", file_memspace);
    if (!ctx) return PNGB200_ERR_BAD_ARGUMENT;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    DeviceGuard guard(ctx->device);
    if (int rc = walk_device_files(ctx, d, count, walks, false)) return rc;
    for (size_t i = 0; i < count; ++i) report(i);
    return PNGB200_OK;
}

int pngb200_png_inspect_batch(pngb200_png_desc* d, size_t count)
{
    return pngb200_png_inspect_files(nullptr, d, count, PNGB200_MEM_HOST);
}

int pngb200_png_decode_files(pngb200_ctx* ctx, pngb200_png_desc* d, size_t count, int file_memspace, int memspace)
{
    if (!ctx || (!d && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (file_memspace != PNGB200_MEM_HOST && file_memspace != PNGB200_MEM_DEVICE)
        return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "file_memspace %d", file_memspace);
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    if (count == 0) return PNGB200_OK;
    if (file_memspace == PNGB200_MEM_DEVICE) {   // no H2D copy to overlap
        start_unfilter_stats(ctx);
        return png_decode_some(ctx, d, count, memspace, true);
    }
    return run_over_lanes(ctx, count, memspace,
                          [&](size_t i) { return d[i].file_len + (size_t)0; },
                          [&](pngb200_ctx* lane, size_t lo, size_t n) { return png_decode_some(lane, d + lo, n, memspace, false); });
}

int pngb200_png_decode_batch(pngb200_ctx* ctx, pngb200_png_desc* d, size_t count, int memspace)
{
    return pngb200_png_decode_files(ctx, d, count, PNGB200_MEM_HOST, memspace);
}

size_t pngb200_png_encode_bound(uint32_t width, uint32_t height, const pngb200_pixel_format* f, int interlaced, uint32_t idat_chunk)
{
    if (!f) return 0;
    const size_t chunk = idat_chunk ? idat_chunk : 65544;
    const int    volume = f->depth * pixel_rule(f->color, f->depth, false).channels;
    const size_t z = pngb200_deflate_bound(pngb200_filtered_size(width, height, volume, interlaced));
    return 8 + 16 + 25 + (12 + 768) + (12 + 256) + z + 12 * (z / chunk + 2) + 12 + 64;
}

int pngb200_png_encode_files(pngb200_ctx* ctx, pngb200_png_encode_desc* d, size_t count, int memspace, int file_memspace)
{
    if (!ctx || (!d && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (file_memspace != PNGB200_MEM_HOST && file_memspace != PNGB200_MEM_DEVICE)
        return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "file_memspace %d", file_memspace);
    const bool host_files = file_memspace == PNGB200_MEM_HOST;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    if (count == 0) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    const bool host_pixels = memspace == PNGB200_MEM_HOST;
    // stage 1: filter + deflate on the device, payload left in HBM (pngb200_encode_batch, DEVICE memspace)
    std::vector<pngb200_encode_desc> enc(count);
    std::vector<size_t> p_off(count), z_off(count), head_len(count);
    std::vector<std::vector<uint8_t>> heads(count);
    Slots pixels{16}, payloads{16};
    for (size_t i = 0; i < count; ++i) {
        const pngb200_pixel_format& f = d[i].format;
        if (!encode_format_ok(f, d[i].width, d[i].height) || !d[i].pixels || !d[i].file)
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "image %zu: bad descriptor", i);
        const int    volume = f.depth * pixel_rule(f.color, f.depth, f.bgr).channels;
        const size_t storage = pngb200_storage_size(d[i].width, d[i].height, volume);
        if (d[i].pixels_len < storage) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "image %zu: pixels_len", i);
        if (d[i].file_cap < pngb200_png_encode_bound(d[i].width, d[i].height, &f, d[i].interlaced, d[i].idat_chunk))
            return set_error(ctx, PNGB200_ERR_OUTPUT_CAPACITY, "image %zu: file_cap below pngb200_png_encode_bound", i);
        p_off[i] = pixels.add(storage);
        z_off[i] = payloads.add(pngb200_deflate_bound(pngb200_filtered_size(d[i].width, d[i].height, volume, d[i].interlaced)));
    }
    if (host_pixels) CU(ctx->d_in.reserve(pixels.total));
    CU(ctx->d_out.reserve(payloads.total));
    for (size_t i = 0; i < count; ++i) {
        const pngb200_pixel_format& f = d[i].format;
        const int    volume = f.depth * pixel_rule(f.color, f.depth, f.bgr).channels;
        const size_t storage = pngb200_storage_size(d[i].width, d[i].height, volume);
        pngb200_encode_desc& e = enc[i];
        memset(&e, 0, sizeof e);
        if (host_pixels) {
            CU(cudaMemcpyAsync(ctx->d_in.as<uint8_t>() + p_off[i], d[i].pixels, storage, cudaMemcpyHostToDevice, ctx->stream));
            e.pixels = ctx->d_in.as<uint8_t>() + p_off[i];
        } else {
            e.pixels = (const uint8_t*)d[i].pixels;
        }
        e.pixels_len = storage;
        e.idat = ctx->d_out.as<uint8_t>() + z_off[i];
        e.idat_cap = pngb200_deflate_bound(pngb200_filtered_size(d[i].width, d[i].height, volume, d[i].interlaced));
        e.width = d[i].width, e.height = d[i].height;
        e.volume = (uint8_t)volume, e.depth = f.depth, e.interlaced = d[i].interlaced;
        e.format = f.bgr ? PNGB200_FORMAT_IOS : PNGB200_FORMAT_ZLIB;
        e.level = d[i].level;
        png_head(f, d[i].width, d[i].height, d[i].interlaced, heads[i]);
        const std::vector<uint8_t>& h = heads[i];
        head_len[i] = h.size();
    }
    int rc = pngb200_encode_batch(ctx, enc.data(), count, PNGB200_MEM_DEVICE);
    if (rc != PNGB200_OK) return rc;
    // stage 2: frame the payload into IDAT chunks inside a device image of the file (device files: the file itself),
    // CRC them there
    std::vector<size_t> file_off(count), file_len(count);
    Slots files{16};
    std::vector<FrameItem>   frames;
    std::vector<CrcRegion>   regions;
    std::vector<CopySegment> segs;
    for (size_t i = 0; i < count; ++i) {
        d[i].status = enc[i].status, d[i].checksum = enc[i].checksum, d[i].blocks = enc[i].blocks, d[i].produced = 0;
        if (enc[i].status != PNGB200_OK) continue;
        const size_t chunk = d[i].idat_chunk ? d[i].idat_chunk : 65544;
        const size_t z = enc[i].produced, nchunks = (z + chunk - 1) / chunk;
        file_len[i] = head_len[i] + z + 12 * nchunks + 12;
        if (host_files) file_off[i] = files.add(file_len[i]);
    }
    if (host_files) CU(ctx->d_file.reserve(std::max<size_t>(files.total, 256)));
    for (size_t i = 0; i < count; ++i) {
        if (enc[i].status != PNGB200_OK) continue;
        uint8_t* base = host_files ? ctx->d_file.as<uint8_t>() + file_off[i] : d[i].file;
        CU(cudaMemcpyAsync(base, heads[i].data(), head_len[i], cudaMemcpyHostToDevice, ctx->stream));
        const size_t chunk = d[i].idat_chunk ? d[i].idat_chunk : 65544;
        // Encoder.pull hands out DeflatorOut's queued buffers (2 x capacity bytes each), then the rest
        // (Encoding/PNG.Encoder.swift:33-129, Deflator/LZ77.DeflatorOut.swift:73-125)
        size_t at = head_len[i];
        for (size_t o = 0; o < enc[i].produced; o += chunk) {
            const size_t n = std::min(chunk, (size_t)enc[i].produced - o);
            frames.push_back({base + at, (uint32_t)n, CK_IDAT});
            segs.push_back({enc[i].idat + o, base + at + 8, n});
            regions.push_back({base + at + 8, n, CK_IDAT, 1});
            at += 12 + n;
        }
        frames.push_back({base + at, 0, CK_IEND});
        regions.push_back({base + at + 8, 0, CK_IEND, 1});
    }
    CU(cudaStreamSynchronize(ctx->stream));  // `heads` is pageable host memory read by the copies above
    rc = run_segment_copy(ctx, segs);
    if (rc != PNGB200_OK) return rc;
    if (!frames.empty()) {
        Tables t(ctx->h_genjobs, ctx->d_genjobs);
        const size_t off_frames = t.host(frames.data(), sizeof(FrameItem) * frames.size());
        const size_t off_crc = t.device(sizeof(uint32_t) * frames.size(), false);   // run_crc clears it
        if ((rc = t.upload(ctx)) != PNGB200_OK) return rc;
        FrameItem* d_frames = t.dev<FrameItem>(off_frames);
        uint32_t*  d_crc = t.dev<uint32_t>(off_crc);
        const unsigned blocks = (unsigned)((frames.size() + 255) / 256);
        frame_chunks_kernel<<<blocks, 256, 0, ctx->stream>>>(d_frames, d_crc, (uint32_t)frames.size(), 0);
        ctx->launches++;
        rc = run_crc(ctx, regions, d_crc, nullptr);  // the chunk type is folded in as a 4-byte prefix
        if (rc != PNGB200_OK) return rc;
        frame_chunks_kernel<<<blocks, 256, 0, ctx->stream>>>(d_frames, d_crc, (uint32_t)frames.size(), 1);
        ctx->launches++;
        CU(cudaGetLastError());
    }
    for (size_t i = 0; i < count; ++i) {
        if (enc[i].status != PNGB200_OK) continue;
        if (host_files)
            CU(cudaMemcpyAsync(d[i].file, ctx->d_file.as<uint8_t>() + file_off[i], file_len[i], cudaMemcpyDeviceToHost, ctx->stream));
        d[i].produced = file_len[i];
    }
    CU(cudaStreamSynchronize(ctx->stream));
    return PNGB200_OK;
}

int pngb200_png_encode_batch(pngb200_ctx* ctx, pngb200_png_encode_desc* d, size_t count, int memspace)
{
    return pngb200_png_encode_files(ctx, d, count, memspace, PNGB200_MEM_HOST);
}

}  // extern "C"

// ---------------- online encoding: PNG.Encoder.pull as the rows arrive ----------------
// The handle owns an online deflator; each push filters the scanlines it completes onto the end of the deflator's
// input, deflates them (scanline ends in DfEnds), CRCs the new payload bytes on the device and frames the chunks that
// the deflator's pop() / pull() now hand out.
struct pngb200_png_encoder {
    pngb200_ctx*      ctx = nullptr;
    pngb200_deflator* z = nullptr;
    uint32_t width = 0, height = 0;
    uint8_t  volume = 0, depth = 0, interlaced = 0, bpp = 0;
    uint64_t row_bytes = 0;            // storage bytes a row
    uint64_t rows = 0;                 // storage rows received
    uint64_t lines = 0;                // stream scanlines filtered
    DevBuf   d_rows;                   // non-interlaced: the last row received; Adam7: the whole storage
    DevBuf   d_header;                 // the deflate stream's header (zlib: 2 bytes), CRC'd with the first chunk
    uint64_t header = 0;
    int      status = PNGB200_OK;      // sticky: a failed launch leaves the device state unknown
    // IDAT CRC-32s: stream bytes CRC'd so far, the open chunk's CRC (its type included), the finished chunks' CRCs
    uint64_t crc_at = 0;
    uint32_t crc_open = 0;
    std::deque<uint32_t> crcs;
    std::deque<std::vector<uint8_t>> pieces;   // framed, not popped yet
    std::vector<uint8_t> popped;               // the piece pop() handed out last
    uint64_t idat_out = 0;
    bool     iend = false;
    size_t device_bytes() const { return z->device_bytes() + d_rows.cap + d_header.cap; }
    // the first stream scanline that needs a storage row at or past `r` (Adam7: pass z's scanline y reads row
    // by + y * sy), and the stream offset of scanline `line`
    uint64_t lines_complete(uint64_t r) const
    {
        uint64_t n = 0;
        for (int p = 0; p < 7; ++p) {
            const Pass ps = stream_pass(p, width, height, volume, interlaced);
            const uint64_t got = r > ps.by ? std::min<uint64_t>(ps.height, ((r - 1 - ps.by) >> ps.ey) + 1) : 0;
            n += got;
            if (got < ps.height) break;
        }
        return n;
    }
    uint64_t line_offset(uint64_t line) const
    {
        uint64_t off = 0;
        for (int p = 0; p < 7; ++p) {
            const Pass ps = stream_pass(p, width, height, volume, interlaced);
            const uint64_t k = std::min<uint64_t>(line, ps.height);
            off += k * (ps.pitch + 1);
            line -= k;
        }
        return off;
    }
    uint64_t line_end(uint64_t line) const { return line_offset(line + 1); }
};

namespace {

// crc(A || B) from crc(A), crc(B) and |B| (crc32.cuh: multiply crc(A) by x^(8|B|))
uint32_t crc_combine(uint32_t a, uint32_t b, uint64_t nb)
{
    static const std::vector<uint32_t> t = [] {
        std::vector<uint32_t> v(CRC_TABLE_WORDS);
        crc_build_tables(v.data());
        return v;
    }();
    for (int k = 0; nb && a; nb >>= 1, ++k) {
        if (!(nb & 1)) continue;
        uint32_t s = 0;
        for (int i = 0; i < 32; ++i)
            if (a >> i & 1) s ^= t[256 + 32 * k + i];
        a = s;
    }
    return a ^ b;
}

// one IDAT chunk from the deflator's bytes and the CRC the device computed for it
std::vector<uint8_t> frame_idat(const uint8_t* body, size_t n, uint32_t crc)
{
    std::vector<uint8_t> c(12 + n);
    store_be32(c.data(), (uint32_t)n), store_be32(c.data() + 4, CK_IDAT);
    memcpy(c.data() + 8, body, n);
    store_be32(c.data() + 8 + n, crc);
    return c;
}

// The pushes of one pngb200_png_encoder_push_batch call, on distinct encoders of `ctx`
int encoder_pushes(pngb200_ctx* ctx, pngb200_png_encoder_push_desc* pushes, size_t count)
{
    struct Item {
        pngb200_png_encoder_push_desc* d;
        pngb200_png_encoder* e;
        uint64_t rows, lines;          // after the push
        uint64_t filtered;             // bytes of the scanlines it completes
        bool     last;
        DfNeed   need;
        size_t   staged = 0;           // offset of its host rows in the staging
        size_t   ends = 0, job = (size_t)-1;
        uint64_t written = 0;          // the deflator's bytes before the launch
    };
    std::vector<Item> live;
    size_t staged = 0, nlines = 0, nends = 0, run = 0, host_out = 0, nfilter = 0;
    for (size_t i = 0; i < count; ++i) {
        pngb200_png_encoder_push_desc* d = &pushes[i];
        pngb200_png_encoder* e = d->encoder;
        const uint64_t add = d->n / e->row_bytes;
        if (e->status < 0) {
            d->status = e->status;
            continue;
        }
        if (e->rows == e->height)
            d->status = set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_encoder: push after the image is complete");
        else if (d->n % e->row_bytes || add > e->height - e->rows)
            d->status = set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_encoder: %zu bytes are not whole rows inside the image", d->n);
        if (e->rows == e->height || d->n % e->row_bytes || add > e->height - e->rows) continue;
        Item it;
        it.d = d, it.e = e;
        it.rows = e->rows + add;
        it.lines = e->lines_complete(it.rows);
        it.filtered = e->line_offset(it.lines) - e->line_offset(e->lines);
        it.last = it.rows == e->height;
        if (it.filtered > kMaxDeflatorPush) {
            d->status = set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_encoder: a push completes at most 1 GiB of scanlines");
            continue;
        }
        d->status = PNGB200_ERR_CUDA;   // until its push is answered
        it.need = df_need(e->z, it.filtered, it.last);
        if (d->memspace == PNGB200_MEM_HOST) it.staged = staged, staged += d->n;
        if (it.lines > e->lines) ++nfilter, nlines += it.lines - e->lines;
        if (it.need.run) {
            it.ends = nends, nends += it.lines - e->lines;
            host_out += align_up(it.need.out, 256), ++run;
        }
        live.push_back(it);
    }
    if (nlines >= (1ull << 31)) {
        for (Item& it : live) it.d->status = set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_encoder_push_batch: too many scanlines");
        return PNGB200_OK;
    }
    // the tables of the call, laid out now so that every allocation comes before any device work
    std::vector<FilterResumeJob> fjobs(nfilter);
    std::vector<uint32_t>        line_base(nfilter + 1, 0);
    std::vector<DfResumeJob>     djobs(run);
    std::vector<DfEnds>          dends(run);
    std::vector<uint64_t>        ends(nends);
    Tables t(ctx->h_st, ctx->d_st);
    const size_t off_f = t.host(fjobs.data(), sizeof(FilterResumeJob) * fjobs.size());
    const size_t off_lb = t.host(line_base.data(), sizeof(uint32_t) * line_base.size());
    const size_t off_dj = t.host(djobs.data(), sizeof(DfResumeJob) * djobs.size());
    const size_t off_de = t.host(dends.data(), sizeof(DfEnds) * dends.size());
    const size_t off_e = t.host(ends.data(), sizeof(uint64_t) * ends.size());
    PushCall call(ctx);
    const size_t res_off = align_up(host_out, 256);
    CU(ctx->h_dfout.reserve(res_off + sizeof(DfResumeResult) * std::max<size_t>(run, 1)));
    CU(ctx->h_st.reserve(t.host_end));
    CU(ctx->d_st.reserve(t.end));
    for (Item& it : live) df_grow(call, it.e->z, it.need);
    if (int rc = call.grow(staged)) return rc;
    // Everything up to the deflate launch.  A failure here leaves every handle of the call with a sticky error: a
    // deflator may have counted in input that was never written, so its input and the encoder's row counts no longer
    // agree.
    auto enqueue = [&]() -> int {
        // the host rows of every encoder with one upload; Adam7 rows into the encoder's storage
        if (int rc = call.pack(live.size(), [&](size_t k) {
                const pngb200_png_encoder_push_desc* d = live[k].d;
                return std::pair<const void*, size_t>(d->memspace == PNGB200_MEM_HOST ? d->rows : nullptr,
                                                      d->memspace == PNGB200_MEM_HOST ? d->n : 0);
            }))
            return rc;
        size_t f = 0, out_at = 0, j = 0;
        for (Item& it : live) {
            pngb200_png_encoder* e = it.e;
            pngb200_deflator* z = e->z;
            const uint8_t* rows = it.d->memspace == PNGB200_MEM_HOST ? ctx->d_stin.as<uint8_t>() + it.staged : (const uint8_t*)it.d->rows;
            if (e->interlaced && it.d->n)
                CU(cudaMemcpyAsync(e->d_rows.as<uint8_t>() + e->rows * e->row_bytes, rows, it.d->n, cudaMemcpyDeviceToDevice, ctx->stream));
            const uint64_t held = z->held(), off0 = e->line_offset(e->lines);
            if (it.lines > e->lines) {
                FilterResumeJob& fj = fjobs[f];
                fj.rows = e->interlaced ? e->d_rows.as<uint8_t>() : rows;
                fj.carried = e->d_rows.as<uint8_t>();
                fj.out = z->d_in.as<uint8_t>() + held;
                fj.out_off0 = off0;
                fj.width = e->width, fj.height = e->height;
                fj.first = (uint32_t)e->lines, fj.row0 = (uint32_t)e->rows;
                fj.volume = e->volume, fj.depth = e->depth, fj.interlaced = e->interlaced, fj.bpp = e->bpp;
                line_base[f + 1] = line_base[f] + (uint32_t)(it.lines - e->lines);
                ++f;
            }
            z->total += it.filtered;
            df_drop_popped(z);
            it.written = z->written;
            if (!it.need.run) continue;
            for (uint64_t k = e->lines; k < it.lines; ++k) ends[it.ends + (k - e->lines)] = held + (e->line_end(k) - off0);
            dends[j] = {it.lines > e->lines ? t.dev<uint64_t>(off_e) + it.ends : nullptr, it.lines - e->lines};
            djobs[j] = df_job(z, it.need, it.last, ctx->h_dfout.as<uint8_t>() + out_at,
                              (DfResumeResult*)(ctx->h_dfout.as<uint8_t>() + res_off) + j);
            out_at += align_up(it.need.out, 256);
            it.job = j++;
        }
        if (int rc = t.upload(ctx)) return rc;
        if (nlines) {
            filter_resume_kernel<<<(unsigned)((nlines + FILTER_WARPS - 1) / FILTER_WARPS), FILTER_WARPS * 32, 0, ctx->stream>>>(
                t.dev<FilterResumeJob>(off_f), t.dev<uint32_t>(off_lb), (uint32_t)nfilter, (uint32_t)nlines);
            ctx->launches++;
            CU(cudaGetLastError());
        }
        // a non-interlaced encoder carries its last row to the next push (behind the filter launch, which reads the old one)
        for (const Item& it : live) {
            const pngb200_png_encoder* e = it.e;
            if (e->interlaced || !it.d->n || it.last) continue;
            const uint8_t* rows = it.d->memspace == PNGB200_MEM_HOST ? ctx->d_stin.as<uint8_t>() + it.staged : (const uint8_t*)it.d->rows;
            CU(cudaMemcpyAsync(e->d_rows.p, rows + it.d->n - e->row_bytes, e->row_bytes, cudaMemcpyDeviceToDevice, ctx->stream));
        }
        return PNGB200_OK;
    };
    if (int rc = enqueue()) {
        for (Item& it : live) it.d->status = it.e->status = it.e->z->status = rc;
        return rc;
    }
    cudaError_t err = cudaSuccess;
    if (run) err = df_launch(ctx, t.dev<DfResumeJob>(off_dj), run, t.dev<DfEnds>(off_de));
    else err = cudaStreamSynchronize(ctx->stream);
    for (Item& it : live) {
        pngb200_png_encoder* e = it.e;
        int st = PNGB200_OK;
        if (it.job != (size_t)-1) st = df_take(ctx, e->z, djobs[it.job], err);
        else if (err != cudaSuccess) st = e->z->status = set_error(ctx, PNGB200_ERR_CUDA, "png_encoder: %s", cudaGetErrorString(err));
        e->rows = it.rows, e->lines = it.lines;
        it.d->status = e->status = st;
    }
    if (err != cudaSuccess) return PNGB200_ERR_CUDA;
    // The IDAT CRC-32s: every new payload byte on the device, cut at chunk edges, the chunk type folded into a chunk's
    // first piece; the stream header sits in d_header and the launch's bytes in d_out.
    struct Piece { pngb200_png_encoder* e; uint64_t len; bool first; };
    std::vector<CrcRegion> regions;
    std::vector<Piece>     pieces;
    for (Item& it : live) {
        pngb200_png_encoder* e = it.e;
        if (it.d->status != PNGB200_OK) continue;
        const uint64_t chunk = e->z->chunk;
        auto cut = [&](const uint8_t* p, uint64_t at, uint64_t len) {
            while (len) {
                const uint64_t take = std::min(len, (at / chunk + 1) * chunk - at);
                regions.push_back({p, take, CK_IDAT, at % chunk == 0 ? 1u : 0u});
                pieces.push_back({e, take, at % chunk == 0});
                p += take, at += take, len -= take;
            }
        };
        if (e->crc_at < e->header) cut(e->d_header.as<uint8_t>(), 0, e->header);
        cut(e->z->d_out.as<uint8_t>(), it.written, e->z->written - it.written);
    }
    if (!regions.empty()) {
        CrcPlan plan;
        const uint32_t* crc = nullptr;
        int rc = crc_upload(ctx, regions, nullptr, &plan);
        if (rc == PNGB200_OK) rc = crc_launch(ctx, plan);
        if (rc == PNGB200_OK) rc = crc_fetch(ctx, plan, &crc);
        if (rc == PNGB200_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess)
            rc = set_error(ctx, PNGB200_ERR_CUDA, "png_encoder: CRC-32 pass failed");
        if (rc != PNGB200_OK) {
            for (const Piece& p : pieces) p.e->status = rc;
            for (Item& it : live)
                if (it.e->status != PNGB200_OK) it.d->status = it.e->status;
            return rc;
        }
        for (size_t k = 0; k < pieces.size(); ++k) {
            pngb200_png_encoder* e = pieces[k].e;
            e->crc_open = pieces[k].first ? crc[k] : crc_combine(e->crc_open, crc[k], pieces[k].len);
            e->crc_at += pieces[k].len;
            if (e->crc_at % e->z->chunk == 0) e->crcs.push_back(e->crc_open);
        }
    }
    // frame what the deflator hands out now: pop() before each scanline, then after the last push([], last: true)
    // pull() until nil and IEND
    for (Item& it : live) {
        pngb200_png_encoder* e = it.e;
        if (it.d->status != PNGB200_OK) continue;
        pngb200_deflator* z = e->z;
        if (z->finished && e->crc_at % z->chunk) e->crcs.push_back(e->crc_open);
        const uint8_t* body;
        size_t         n;
        while (z->finished ? pngb200_deflator_pull(z, &body, &n) : pngb200_deflator_pop(z, &body, &n)) {
            e->pieces.push_back(frame_idat(body, n, e->crcs.front()));
            e->crcs.pop_front();
        }
        if (z->finished) {
            std::vector<uint8_t> iend;
            put_chunk(iend, CK_IEND, nullptr, 0);
            e->pieces.push_back(std::move(iend));
            e->iend = true;
        }
    }
    return call.done();
}

}  // namespace

extern "C" {

pngb200_png_encoder* pngb200_png_encoder_create(pngb200_ctx* ctx, const pngb200_png_encoder_desc* d)
{
    Geometry g;
    if (!ctx || !d || !encode_format_ok(d->format, d->width, d->height) || d->level < 0 || d->level > 13 ||
        !geometry(d->width, d->height, d->format.depth * pixel_rule(d->format.color, d->format.depth, d->format.bgr).channels,
                  d->format.depth, d->interlaced, &g)) {
        set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_encoder_create: bad descriptor");
        return nullptr;
    }
    // One push completes at most kMaxDeflatorPush filtered bytes.  A caller can always keep a non-interlaced push under
    // that by pushing fewer rows, unless one scanline is over it; an Adam7 image's last row completes passes 1 to 6 at
    // once (about 63/64 of its stream) whatever the schedule.  Such images are refused here, before any row is taken.
    if (d->interlaced ? g.filtered > kMaxDeflatorPush : (uint64_t)g.pitch + 1 > kMaxDeflatorPush) {
        set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_encoder_create: %s is over 1 GiB",
                  d->interlaced ? "the filtered stream of an Adam7 image" : "a filtered scanline");
        return nullptr;
    }
    const pngb200_pixel_format& f = d->format;
    pngb200_png_encoder* e = new pngb200_png_encoder();
    e->ctx = ctx;
    e->width = d->width, e->height = d->height;
    e->volume = (uint8_t)(f.depth * pixel_rule(f.color, f.depth, f.bgr).channels), e->depth = f.depth;
    e->interlaced = d->interlaced ? 1 : 0, e->bpp = g.bpp;
    e->row_bytes = (uint64_t)d->width * g.bpp;
    e->z = pngb200_deflator_create_online(ctx, f.bgr ? PNGB200_FORMAT_IOS : PNGB200_FORMAT_ZLIB, d->level, 15,
                                          d->idat_chunk ? d->idat_chunk : 65544);
    if (!e->z) {
        delete e;
        return nullptr;
    }
    DeviceGuard guard(ctx->device);
    e->header = e->z->output.size();
    if (e->d_rows.reserve(e->interlaced ? g.storage : e->row_bytes) != cudaSuccess ||
        e->d_header.reserve(std::max<uint64_t>(e->header, 1)) != cudaSuccess ||
        (e->header && cudaMemcpy(e->d_header.p, e->z->output.data(), e->header, cudaMemcpyHostToDevice) != cudaSuccess) ||
        ensure_crc_tables(ctx) != PNGB200_OK) {
        set_error(ctx, PNGB200_ERR_CUDA, "png_encoder_create: cannot allocate the device state");
        pngb200_deflator_destroy(e->z);
        delete e;
        return nullptr;
    }
    std::vector<uint8_t> head;
    png_head(f, d->width, d->height, e->interlaced, head);
    e->pieces.push_back(std::move(head));
    return e;
}

void pngb200_png_encoder_destroy(pngb200_png_encoder* e)
{
    if (!e) return;
    pngb200_deflator_destroy(e->z);   // synchronises the stream
    DeviceGuard guard(e->ctx->device);
    delete e;
}

int pngb200_png_encoder_push_batch(pngb200_ctx* ctx, pngb200_png_encoder_push_desc* pushes, size_t count)
{
    if (!ctx || (!pushes && count)) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_encoder_push_batch: null argument");
    std::vector<const void*> seen(count);
    for (size_t i = 0; i < count; ++i) {
        const pngb200_png_encoder* e = pushes[i].encoder;
        if (!e || e->ctx != ctx || (!pushes[i].rows && pushes[i].n) ||
            (pushes[i].memspace != PNGB200_MEM_HOST && pushes[i].memspace != PNGB200_MEM_DEVICE))
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_encoder_push_batch: item %zu has no encoder of this context, "
                             "no rows or no memspace", i);
        seen[i] = e;
    }
    std::sort(seen.begin(), seen.end());
    if (std::adjacent_find(seen.begin(), seen.end()) != seen.end())
        return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_encoder_push_batch: a handle appears twice");
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    if (!count) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    return encoder_pushes(ctx, pushes, count);
}

int pngb200_png_encoder_push(pngb200_png_encoder* e, const void* rows, size_t n, int memspace)
{
    if (!e) return PNGB200_ERR_BAD_ARGUMENT;
    pngb200_png_encoder_push_desc d{e, rows, n, memspace, 0};
    if (int rc = pngb200_png_encoder_push_batch(e->ctx, &d, 1)) return rc;
    return d.status;
}

int pngb200_png_encoder_pop(pngb200_png_encoder* e, const uint8_t** bytes, size_t* n)
{
    if (!e || !bytes || !n) return PNGB200_ERR_BAD_ARGUMENT;
    if (e->pieces.empty()) return 0;
    e->popped = std::move(e->pieces.front());
    e->pieces.pop_front();
    const bool idat = e->popped.size() >= 8 && memcmp(e->popped.data() + 4, "IDAT", 4) == 0;
    if (idat) e->idat_out++;
    *bytes = e->popped.data();
    *n = e->popped.size();
    return 1;
}

int pngb200_png_encoder_progress(const pngb200_png_encoder* e, uint64_t out[6])
{
    if (!e || !out) return PNGB200_ERR_BAD_ARGUMENT;
    out[0] = e->rows;
    out[1] = e->lines;
    out[2] = e->z->dequeued();
    out[3] = e->idat_out;
    out[4] = e->iend ? 1 : 0;
    out[5] = e->device_bytes();
    return PNGB200_OK;
}

void pngb200_png_encoder_error(const pngb200_png_encoder* e, int* status, uint32_t* a, uint32_t* b)
{
    if (status) *status = e ? e->status : PNGB200_ERR_BAD_ARGUMENT;
    if (a) *a = 0;
    if (b) *b = 0;
}

}  // extern "C"

// ---------------- cloning handles: the encoder and pngb200_clone_batch ----------------
namespace {

cudaError_t clone_encoder(const pngb200_png_encoder* s, pngb200_png_encoder* e, std::vector<CopySegment>& segs)
{
    e->ctx = s->ctx;
    e->width = s->width, e->height = s->height;
    e->volume = s->volume, e->depth = s->depth, e->interlaced = s->interlaced, e->bpp = s->bpp;
    e->row_bytes = s->row_bytes, e->rows = s->rows, e->lines = s->lines;
    e->header = s->header;
    e->status = s->status;
    e->crc_at = s->crc_at, e->crc_open = s->crc_open, e->crcs = s->crcs;
    e->pieces = s->pieces;   // each handle pops its own copy; `popped` starts empty
    e->idat_out = s->idat_out, e->iend = s->iend;
    e->z = new pngb200_deflator();
    cudaError_t err = clone_deflator(s->z, e->z, segs);
    // Adam7: the whole storage, of which the rows received are written; otherwise the row carried to the next push
    const uint64_t rows = e->interlaced ? s->row_bytes * s->height : s->row_bytes;
    const uint64_t keep = e->interlaced ? s->row_bytes * s->rows : s->rows ? s->row_bytes : 0;
    if (err == cudaSuccess) err = clone_buf(segs, e->d_rows, s->d_rows, rows, keep, false);
    if (err == cudaSuccess) err = clone_buf(segs, e->d_header, s->d_header, std::max<uint64_t>(s->header, 1), s->header, false);
    return err;
}

// the host bytes an item's clone copies: queues, tails, a buffered deflator's input, host storage
uint64_t clone_host_bytes(const pngb200_clone_desc& d)
{
    auto deflator = [](const pngb200_deflator* z) { return (uint64_t)(z->input.size() + z->output.size()); };
    if (d.inflator) return d.inflator->tail.size();
    if (d.deflator) return deflator(d.deflator);
    if (d.context) return d.context->z->tail.size() + (d.context->memspace == PNGB200_MEM_HOST ? d.context->storage : 0);
    uint64_t n = deflator(d.encoder->z) + sizeof(uint32_t) * d.encoder->crcs.size();
    for (const std::vector<uint8_t>& piece : d.encoder->pieces) n += piece.size();
    return n;
}

void destroy_clone(pngb200_clone_desc& d)
{
    if (!d.clone) return;
    if (d.inflator) pngb200_inflator_destroy((pngb200_inflator*)d.clone);
    else if (d.deflator) pngb200_deflator_destroy((pngb200_deflator*)d.clone);
    else if (d.context) pngb200_png_context_destroy((pngb200_png_context*)d.clone);
    else pngb200_png_encoder_destroy((pngb200_png_encoder*)d.clone);
    d.clone = nullptr;
}

// The checks of pngb200_clone_batch, made before any work
int check_clones(pngb200_ctx* ctx, const pngb200_clone_desc* items, size_t count)
{
    if (!ctx || (!items && count)) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "clone_batch: null argument");
    for (size_t i = 0; i < count; ++i) {
        const pngb200_clone_desc& d = items[i];
        const int sources = !!d.inflator + !!d.deflator + !!d.context + !!d.encoder;
        const pngb200_ctx* owner = d.inflator ? d.inflator->ctx : d.deflator ? d.deflator->ctx : d.context ? d.context->ctx
                                 : d.encoder ? d.encoder->ctx : nullptr;
        if (sources != 1 || owner != ctx)
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "clone_batch: item %zu has not exactly one source of this context", i);
        if (d.context) {
            const uintptr_t a = (uintptr_t)d.pixels, b = (uintptr_t)d.context->pixels, n = (uintptr_t)d.context->storage;
            if (!d.pixels || d.pixels_cap < d.context->storage || (n && a < b + n && b < a + n))
                return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "clone_batch: item %zu has no storage of %llu bytes apart from its "
                                 "source's", i, (unsigned long long)n);
        }
    }
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "clone_batch: a decode batch is pending");
    return PNGB200_OK;
}

}  // namespace

extern "C" {

int pngb200_clone_batch(pngb200_ctx* ctx, pngb200_clone_desc* items, size_t count)
{
    for (size_t i = 0; items && i < count; ++i) items[i].clone = nullptr;
    if (ctx) ctx->clone_bytes[0] = ctx->clone_bytes[1] = 0;
    if (int rc = check_clones(ctx, items, count)) return rc;
    if (!count) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    std::vector<CopySegment> segs;
    cudaError_t e = cudaSuccess;
    for (size_t i = 0; i < count && e == cudaSuccess; ++i) {
        pngb200_clone_desc& d = items[i];
        if (d.inflator) {
            pngb200_inflator* z = new pngb200_inflator();
            d.clone = z;
            e = clone_inflator(d.inflator, z, segs);
        } else if (d.deflator) {
            pngb200_deflator* z = new pngb200_deflator();
            d.clone = z;
            e = clone_deflator(d.deflator, z, segs);
        } else if (d.context) {
            pngb200_png_context* c = new pngb200_png_context();
            d.clone = c;
            e = clone_context(d.context, c, (uint8_t*)d.pixels, segs);
        } else {
            pngb200_png_encoder* c = new pngb200_png_encoder();
            d.clone = c;
            e = clone_encoder(d.encoder, c, segs);
        }
    }
    int rc = e == cudaSuccess ? PNGB200_OK
                              : set_error(ctx, PNGB200_ERR_CUDA, "clone_batch: cannot allocate a clone: %s", cudaGetErrorString(e));
    // One launch copies every segment.  Each starts at byte 0 of a DevBuf, which cudaMalloc aligns, so the kernel's
    // misaligned branch never runs for them -- except a context's device storage, at the caller's alignment: there the
    // last word that branch reads is the aligned word holding the segment's last byte, inside the same allocation.
    if (rc == PNGB200_OK && !segs.empty()) {
        CopyPlan plan;
        rc = copy_upload(ctx, segs, &plan);
        if (rc == PNGB200_OK) rc = copy_launch(ctx, plan);
        if (rc == PNGB200_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess)
            rc = set_error(ctx, PNGB200_ERR_CUDA, "clone_batch: the copy failed");
    }
    if (rc != PNGB200_OK) {
        for (size_t i = 0; i < count; ++i) destroy_clone(items[i]);
        return rc;
    }
    for (size_t i = 0; i < count; ++i) {
        if (items[i].context && items[i].context->memspace == PNGB200_MEM_HOST)
            memcpy(items[i].pixels, items[i].context->pixels, items[i].context->storage);
        ctx->clone_bytes[1] += clone_host_bytes(items[i]);
    }
    for (const CopySegment& s : segs) ctx->clone_bytes[0] += s.len;
    return PNGB200_OK;
}

pngb200_inflator* pngb200_inflator_clone(const pngb200_inflator* z)
{
    pngb200_clone_desc d{};
    d.inflator = const_cast<pngb200_inflator*>(z);
    return pngb200_clone_batch(z ? z->ctx : nullptr, &d, 1) ? nullptr : (pngb200_inflator*)d.clone;
}

pngb200_deflator* pngb200_deflator_clone(const pngb200_deflator* z)
{
    pngb200_clone_desc d{};
    d.deflator = const_cast<pngb200_deflator*>(z);
    return pngb200_clone_batch(z ? z->ctx : nullptr, &d, 1) ? nullptr : (pngb200_deflator*)d.clone;
}

pngb200_png_context* pngb200_png_context_clone(const pngb200_png_context* c, void* pixels, size_t pixels_cap)
{
    pngb200_clone_desc d{};
    d.context = const_cast<pngb200_png_context*>(c);
    d.pixels = pixels;
    d.pixels_cap = pixels_cap;
    return pngb200_clone_batch(c ? c->ctx : nullptr, &d, 1) ? nullptr : (pngb200_png_context*)d.clone;
}

pngb200_png_encoder* pngb200_png_encoder_clone(const pngb200_png_encoder* e)
{
    pngb200_clone_desc d{};
    d.encoder = const_cast<pngb200_png_encoder*>(e);
    return pngb200_clone_batch(e ? e->ctx : nullptr, &d, 1) ? nullptr : (pngb200_png_encoder*)d.clone;
}

}  // extern "C"
