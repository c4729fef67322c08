// pngb200_api.cu -- the C ABI declared in include/pngb200.h: contexts, batching, host glue.
//
// The library talks to the CUDA runtime directly (no torch types anywhere); callers that live in
// a PyTorch process pass raw device pointers (tensor.data_ptr()) with PNGB200_MEM_DEVICE.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <functional>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "checksum.cuh"
#include "common.cuh"
#include "deflate.cuh"
#include "filter.cuh"
#include "color.cuh"
#include "crc32.cuh"
#include "inflate_wave.cuh"
#include "inflate_parallel.cuh"
#include "inflate_cells.cuh"
#include "block_search.cuh"
#include "inflate_segments.cuh"
#include "inflate_serial.cuh"
#include "png_walk.cuh"
#include "unfilter.cuh"

using namespace pngb200;

namespace {

thread_local std::string g_last_error;

// A grow-only workspace that owns its memory: device memory (cudaMalloc) or pinned host memory (cudaHostAlloc).
// Movable, not copyable; a move assignment swaps, so the buffer moved from frees the old memory when it goes.
template <bool Pinned>
struct Buf {
    void*  p   = nullptr;
    size_t cap = 0;
    Buf() = default;
    Buf(Buf&& o) noexcept { std::swap(p, o.p), std::swap(cap, o.cap); }
    Buf& operator=(Buf&& o) noexcept
    {
        std::swap(p, o.p), std::swap(cap, o.cap);
        return *this;
    }
    ~Buf() { release(); }
    cudaError_t reserve(size_t n)
    {
        if (n <= cap) return cudaSuccess;
        release();
        size_t      want;
        cudaError_t e;
        if (Pinned) {
            want = std::max(n + n / 4, (size_t)1 << 12);
            e = cudaHostAlloc(&p, want, cudaHostAllocDefault);
        } else {
            want = std::max(n + std::min(n / 4, (size_t)1 << 30), (size_t)1 << 16);
            e = cudaMalloc(&p, want);
            if (e != cudaSuccess) {
                want = n;
                e = cudaMalloc(&p, want);
            }
        }
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release()
    {
        if (p) Pinned ? cudaFreeHost(p) : cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <typename T> T* as() const { return (T*)p; }
};
using DevBuf = Buf<false>;
using PinBuf = Buf<true>;

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Per-item staging slots of an arena: the item's bytes plus `pad`, rounded up to 256
struct Slots {
    size_t pad;
    size_t total = 0;
    size_t add(size_t bytes)   // the item's offset
    {
        const size_t off = total;
        total += align_up(bytes + pad, 256);
        return off;
    }
};

}  // namespace

struct pngb200_ctx {
    int          device = 0;
    cudaStream_t stream = nullptr;
    uint64_t     launches = 0;
    int          inflate_mode = 0;
    int          last_engine = -1;       // whole-stream engine of the last batch: 0 round-1, 1 ring, 2 cells, -1 none
    int          sm_count = 132;
    size_t       device_bytes = 0;     // global memory of the device (sizes the deflate scratch arena)
    std::string  error;
    bool         pending = false;
    int          pending_memspace = 0;
    // device workspaces (grow-only)
    DevBuf d_jobs, d_results, d_imgjobs, d_genjobs, d_misc, d_partial, d_filtered, d_in, d_out, d_order, d_scratch, d_dfscratch, d_dfjobs, d_dfres, d_enc,
           d_file, d_crc, d_seg, d_crctab, d_sgjobs, d_sgres, d_sgsym, d_sgsearch, d_sgrec, d_sgwin;
    // pinned host tables
    PinBuf h_jobs, h_results, h_imgjobs, h_genjobs, h_misc, h_order, h_crc, h_seg, h_sgsearch, h_sgjobs, h_sgres, h_sgrec;
    // the streaming handles' pushes (pngb200_inflator_push_batch, pngb200_png_context_push_batch): tables, checksum
    // bases and partials, and the staged input, apart from the decode batch's so that they may run while one is pending
    DevBuf d_st, d_stbase, d_stpartial, d_stin;
    PinBuf h_st, h_stin;
    PinBuf h_dfout;   // the online deflators' launch: the bytes each handle wrote and its result, written by the kernel
    uint64_t seg_streams = 0, seg_segments = 0, seg_fallbacks = 0;  // last batch: streams cut into segments, segments, rejected
    uint64_t split_stats[6] = {};      // last batch, streams cut in two: see pngb200_ctx_split_stats
    uint64_t clone_bytes[2] = {};      // last pngb200_clone_batch: device bytes, host bytes copied
    uint64_t scratch_stride = 0;       // layout of d_scratch the last inflate launch used
    size_t parallel_threshold = 8192;  // streams at least this long use the block-parallel kernel
    unsigned long long* d_hist = nullptr;   // filter-type histogram of the last wavefront-unfilter launch (in d_imgjobs)
    uint64_t unfilter_images[3] = {};  // images of the batch by unfilter path: wavefront, pass path, generic kernel
    size_t peer_streams = 0;           // lanes: streams of the whole host batch (its chunks run side by side on this GPU)
    bool   split = true;               // cut big streams into a head and a tail when that evens out the CTA slots (PNGB200_SPLIT=0: off)
    size_t plan_slots = 0;             // CTA slots the segment and split planners assume, 0 = the ring kernel's (PNGB200_PLAN_SLOTS:
                                       // lets a small test batch take the paths meant for a full GPU)
    cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};  // decode stage boundaries
    // geometry of the pending decode batch
    std::vector<uint64_t> expected;   // filtered bytes expected per image
    std::vector<size_t>   out_offset; // staging offsets (HOST memspace)
    std::vector<size_t>   out_bytes;
    // helper contexts (own stream + workspaces) that pipeline big host-memory batches: while one
    // lane's PCIe copies run, another lane's kernels do
    std::vector<pngb200_ctx*> lanes;
    // Bulk H2D copies of the call in flight, issued by run_inflate after its own small table uploads and
    // right before its first launch: copies of one direction are served in issue order across all
    // streams, so a table queued behind another lane's gigabyte would hold this lane's kernels back.
    std::function<int()> bulk_h2d;
};

namespace {

int set_error(pngb200_ctx* ctx, int code, const char* fmt, ...)
{
    char    buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (ctx) ctx->error = buf;
    g_last_error = buf;
    return code;
}

#define CU(call)                                                                                  \
    do {                                                                                          \
        cudaError_t e_ = (call);                                                                  \
        if (e_ != cudaSuccess)                                                                    \
            return set_error(ctx, PNGB200_ERR_CUDA, "%s failed: %s (%s:%d)", #call,               \
                             cudaGetErrorString(e_), __FILE__, __LINE__);                         \
    } while (0)

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev)
    {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard()
    {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// The small tables of a launch, uploaded with one H2D copy: host arrays, then device-only regions, each at a
// 256-byte-aligned offset of a device buffer.  upload() packs the host arrays into the pinned buffer, copies that
// part, and clears the device-only regions asked to be zero; it may move both buffers, so dev() and pin() are for
// after it.  A pinned buffer must not take a second table before a stream synchronise: the copy reads it when the
// stream gets there.
struct Tables {
    PinBuf& h;
    DevBuf& d;
    struct Part { const void* src; size_t off, bytes; bool zero; };
    std::vector<Part> parts;
    size_t host_end = 0, end = 0;
    Tables(PinBuf& h_, DevBuf& d_) : h(h_), d(d_) {}
    size_t host(const void* src, size_t bytes)   // src null: the region is copied unwritten
    {
        const size_t off = add(src, bytes, false);
        host_end = end;
        return off;
    }
    size_t device(size_t bytes, bool zero) { return add(nullptr, bytes, zero); }
    size_t add(const void* src, size_t bytes, bool zero)
    {
        const size_t off = align_up(end, 256);
        parts.push_back({src, off, bytes, zero});
        end = off + bytes;
        return off;
    }
    // `pinned`: bytes of pinned memory to reserve when a readback lands behind the host arrays
    int upload(pngb200_ctx* ctx, size_t pinned = 0)
    {
        CU(h.reserve(std::max(pinned, host_end)));
        CU(d.reserve(end));
        for (const Part& p : parts)
            if (p.src && p.bytes) memcpy((char*)h.p + p.off, p.src, p.bytes);
        CU(cudaMemcpyAsync(d.p, h.p, host_end, cudaMemcpyHostToDevice, ctx->stream));
        for (const Part& p : parts)
            if (p.zero) CU(cudaMemsetAsync((char*)d.p + p.off, 0, p.bytes, ctx->stream));
        return PNGB200_OK;
    }
    template <typename T> T* dev(size_t off) const { return (T*)((char*)d.p + off); }
    template <typename T> T* pin(size_t off) const { return (T*)((char*)h.p + off); }
};

// The buffers one push call grows and the input it stages.  grow() takes the buffers add() listed in two phases.
// Phase 1 allocates a replacement for each and room to stage `staged` pushed bytes; it touches no handle and enqueues
// no device work, so a failure leaves every handle as it was.  Phase 2 copies each buffer's first `keep` bytes into
// its replacement on the stream and swaps the replacement in.  The buffers replaced are freed with this object, after
// the call's last synchronise: done() says the call ended in one; on any other way out the destructor makes it, since
// the stream may still be reading them, the staging or the caller's memory.
struct PushCall {
    struct Grow { DevBuf* buf; size_t size, keep; DevBuf next; };
    pngb200_ctx*        ctx;
    std::vector<Grow>   list;
    std::vector<DevBuf> replaced;
    bool                synced = false;
    explicit PushCall(pngb200_ctx* c) : ctx(c) {}
    ~PushCall() { if (!synced) cudaStreamSynchronize(ctx->stream); }
    void add(DevBuf& b, size_t size, size_t keep) { list.push_back({&b, size, keep, DevBuf()}); }
    int grow(size_t staged)
    {
        CU(ctx->h_stin.reserve(staged));
        CU(ctx->d_stin.reserve(staged));
        for (Grow& g : list) CU(g.next.reserve(g.size));
        for (Grow& g : list) {
            if (g.keep) CU(cudaMemcpyAsync(g.next.p, g.buf->p, g.keep, cudaMemcpyDeviceToDevice, ctx->stream));
            std::swap(*g.buf, g.next);
            replaced.push_back(std::move(g.next));
        }
        list.clear();
        return PNGB200_OK;
    }
    // Packs the host byte ranges range(0 .. count - 1), each a (pointer, length) pair, back to back into the staging
    // and uploads them with one copy: range k lands in d_stin behind the lengths of the ranges before it.
    template <typename Range>
    int pack(size_t count, Range range)
    {
        size_t off = 0;
        for (size_t k = 0; k < count; ++k) {
            const std::pair<const void*, size_t> r = range(k);
            if (r.second) memcpy(ctx->h_stin.as<uint8_t>() + off, r.first, r.second), off += r.second;
        }
        if (off) CU(cudaMemcpyAsync(ctx->d_stin.p, ctx->h_stin.p, off, cudaMemcpyHostToDevice, ctx->stream));
        return PNGB200_OK;
    }
    // Packs and uploads the items' bytes and appends each item's at byte held() of its handle's d_in; `appended(d)`
    // counts them in once that copy is queued.
    template <typename Desc, typename Handle, typename Appended>
    int stage(const std::vector<Desc*>& items, Handle* Desc::*handle, Appended appended)
    {
        if (int rc = pack(items.size(), [&](size_t k) { return std::pair<const void*, size_t>(items[k]->data, items[k]->n); }))
            return rc;
        size_t off = 0;
        for (Desc* d : items) {
            Handle* z = d->*handle;
            if (d->n)
                CU(cudaMemcpyAsync((uint8_t*)z->d_in.p + z->held(), ctx->d_stin.as<uint8_t>() + off, d->n,
                                   cudaMemcpyDeviceToDevice, ctx->stream));
            off += d->n;
            appended(d);
        }
        return PNGB200_OK;
    }
    int done() { synced = true; return PNGB200_OK; }
};

// the CRC-32 byte table and shift operators (crc32.cuh), uploaded once per context
int ensure_crc_tables(pngb200_ctx* ctx)
{
    if (ctx->d_crctab.p) return PNGB200_OK;
    std::vector<uint32_t> t(CRC_TABLE_WORDS);
    crc_build_tables(t.data());
    CU(ctx->d_crctab.reserve(sizeof(uint32_t) * CRC_TABLE_WORDS));
    CU(cudaMemcpyAsync(ctx->d_crctab.p, t.data(), sizeof(uint32_t) * CRC_TABLE_WORDS, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return PNGB200_OK;
}

// a job that decodes a whole stream from its header into dst
StreamJob whole_stream_job(const uint8_t* src, uint64_t src_len, uint8_t* dst, uint64_t dst_cap, int32_t format)
{
    StreamJob j{};
    j.src = src;
    j.src_len = src_len;
    j.dst = dst;
    j.dst_cap = dst_cap;
    j.format = format;
    return j;
}

// The engines that decode big streams in waves of 256 subsequences, numbered as pngb200_ctx_last_inflate_engine reports them
enum Engine { ENG_PARALLEL = 0, ENG_WAVE = 1, ENG_CELLS = 2 };

// One launch of a wave engine: `grid` persistent CTAs pull the `count` jobs from a ticket, through `order` when it is
// not null.  `max_cap`: the largest dst_cap the per-CTA HBM bitmaps have to cover (the cell engine has none).
// `switched`: a SwitchRecord per job, for jobs with may_switch (ring engine), or null.  `before_launch`, when given,
// is enqueued after the scratch set-up and right before the kernel.
int launch_waves(pngb200_ctx* ctx, Engine engine, const StreamJob* jobs, StreamResult* results, const uint32_t* order, size_t count,
                 unsigned grid, uint64_t max_cap, SwitchRecord* switched, const std::function<int()>& before_launch = nullptr)
{
    const uint64_t bitmap_words = engine == ENG_WAVE ? wv_bitmap_words(max_cap) : engine == ENG_PARALLEL ? par_bitmap_words(max_cap) : 0;
    const uint64_t stride = engine == ENG_WAVE       ? wv_scratch_stride(bitmap_words)
                            : engine == ENG_PARALLEL ? par_scratch_stride(bitmap_words)
                                                     : CL_SCRATCH;
    // d_scratch holds `stride` bytes per CTA, then the ticket.  The per-CTA "unresolved" bitmaps must be all-zero when
    // a launch starts; the kernels leave them clean.  A different stride moves the bitmaps onto bytes that held copy
    // lists before, and a fresh allocation is garbage: zero the whole arena in both cases.
    const size_t need = (size_t)stride * grid + 256;
    if (need > ctx->d_scratch.cap || stride != ctx->scratch_stride) {
        CU(ctx->d_scratch.reserve(need));
        CU(cudaMemsetAsync(ctx->d_scratch.p, 0, ctx->d_scratch.cap, ctx->stream));
        ctx->scratch_stride = stride;
    }
    uint32_t* ticket = (uint32_t*)((char*)ctx->d_scratch.p + (size_t)stride * grid);
    CU(cudaMemsetAsync(ticket, 0, sizeof(uint32_t), ctx->stream));
    if (before_launch)
        if (int rc = before_launch()) return rc;
    const WvParams pp{jobs, results, order, ticket, ctx->d_scratch.as<uint8_t>(), stride, bitmap_words, (int)count, switched};
    if (engine == ENG_PARALLEL && count <= (size_t)ctx->sm_count * 3)
        inflate_parallel_kernel3<<<grid, PAR_THREADS, sizeof(ParShared), ctx->stream>>>(pp);
    else if (engine == ENG_PARALLEL)
        inflate_parallel_kernel<<<grid, PAR_THREADS, sizeof(ParShared), ctx->stream>>>(pp);
    else if (engine == ENG_CELLS)
        inflate_cells_kernel<<<grid, WV_THREADS, sizeof(ClShared), ctx->stream>>>(pp);
    else
        inflate_wave_kernel<<<grid, WV_THREADS, sizeof(WvShared), ctx->stream>>>(pp);
    ctx->launches++;
    return PNGB200_OK;
}

// the first plausible dynamic-block header of each of the n SearchJobs in h_sgsearch (found, or ~0), one host round trip
int search_blocks(pngb200_ctx* ctx, size_t n)
{
    CU(ctx->d_sgsearch.reserve(sizeof(SearchJob) * n));
    CU(cudaMemcpyAsync(ctx->d_sgsearch.p, ctx->h_sgsearch.p, sizeof(SearchJob) * n, cudaMemcpyHostToDevice, ctx->stream));
    block_search_kernel<<<dim3((unsigned)n, BS_CTAS), 256, 0, ctx->stream>>>(ctx->d_sgsearch.as<SearchJob>(), (uint32_t)n);
    ctx->launches++;
    CU(cudaMemcpyAsync(ctx->h_sgsearch.p, ctx->d_sgsearch.p, sizeof(SearchJob) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return PNGB200_OK;
}

// ---- more than one CTA per stream (inflate_segments.cuh) ----
// Streams of `par` that are worth cutting are decoded here, segment by segment; on return `par` holds the
// streams that still have to go through the whole-stream kernels (not cut, or a segment did not line up).
// Two host round trips (split points, segment results): the path exists for batches that would otherwise
// leave most of the GPU idle.
int run_segments(pngb200_ctx* ctx, const StreamJob* h_jobs, std::vector<uint32_t>& par)
{
    ctx->seg_streams = ctx->seg_segments = ctx->seg_fallbacks = 0;
    const size_t slots = (size_t)ctx->sm_count * CL_CTAS_PER_SM;
    constexpr uint64_t kMinSegment = 256u << 10;  // compressed bytes per segment, at least
    if (par.empty() || par.size() * 2 > slots) return PNGB200_OK;
    const size_t per_stream = std::max<size_t>(1, slots / par.size());
    struct Cut { uint32_t stream; uint32_t nseg; size_t first_search; };
    std::vector<Cut> cuts;
    size_t nsearch = 0;
    for (uint32_t i : par) {
        const size_t nseg = std::min<size_t>(per_stream, h_jobs[i].src_len / kMinSegment);
        if (nseg < 4 || h_jobs[i].start_bit != 0 || h_jobs[i].phase != 0 || h_jobs[i].dst_cap < (1u << 20)) continue;
        cuts.push_back(Cut{i, (uint32_t)nseg, nsearch});
        nsearch += nseg - 1;
    }
    if (cuts.empty()) return PNGB200_OK;
    // 1. split points: the first plausible dynamic-block header at or after k / nseg of the stream
    CU(ctx->h_sgsearch.reserve(sizeof(SearchJob) * nsearch));
    SearchJob* sj = ctx->h_sgsearch.as<SearchJob>();
    for (const Cut& c : cuts) {
        const StreamJob& j = h_jobs[c.stream];
        const uint64_t bits = 8 * j.src_len, step = bits / c.nseg;
        for (uint32_t k = 1; k < c.nseg; ++k) {
            SearchJob& q = sj[c.first_search + k - 1];
            q.src = j.src;
            q.src_len = j.src_len;
            q.from_bit = k * step;
            q.limit_bit = k + 1 < c.nseg ? (k + 1) * step : bits;
            q.found = ~0ull;
        }
    }
    if (int rc = search_blocks(ctx, nsearch)) return rc;
    // 2. one job per segment; symbols go to a scratch sized 1.5 x the segment's share of the output bound
    std::vector<StreamJob> sg;
    std::vector<uint32_t>  sg_stream, first_of;   // stream of each segment; first segment of each cut (+ end)
    size_t sym_total = 0;
    for (const Cut& c : cuts) {
        const StreamJob& j = h_jobs[c.stream];
        std::vector<uint64_t> at{0};
        for (uint32_t k = 1; k < c.nseg; ++k)
            if (sj[c.first_search + k - 1].found != ~0ull) at.push_back(sj[c.first_search + k - 1].found);
        first_of.push_back((uint32_t)sg.size());
        for (size_t k = 0; k < at.size(); ++k) {
            const uint64_t end = k + 1 < at.size() ? at[k + 1] : 8 * j.src_len;
            StreamJob s = j;
            s.start_bit = at[k];
            s.start_out = 0;
            s.phase = k == 0 ? 0 : 1;
            s.stop_bit = k + 1 < at.size() ? at[k + 1] : 0;
            s.symbolic = 1;
            s.dst_cap = (uint64_t)((double)j.dst_cap * 1.5 * (double)(end - at[k]) / (double)(8 * j.src_len)) + (64u << 10);
            s.dst = (uint8_t*)(uintptr_t)sym_total;  // offset for now (symbols)
            sym_total += align_up(s.dst_cap + 8, 128);
            sg.push_back(s);
            sg_stream.push_back(c.stream);
        }
    }
    first_of.push_back((uint32_t)sg.size());
    const size_t n = sg.size();
    CU(ctx->d_sgsym.reserve(sizeof(uint16_t) * sym_total));
    for (StreamJob& s : sg) s.dst = (uint8_t*)(ctx->d_sgsym.as<uint16_t>() + (size_t)(uintptr_t)s.dst);
    CU(ctx->h_sgjobs.reserve(sizeof(StreamJob) * n));
    CU(ctx->d_sgjobs.reserve(sizeof(StreamJob) * n));
    CU(ctx->d_sgres.reserve(sizeof(StreamResult) * n));
    CU(ctx->h_sgres.reserve(sizeof(StreamResult) * n));
    memcpy(ctx->h_sgjobs.p, sg.data(), sizeof(StreamJob) * n);
    CU(cudaMemcpyAsync(ctx->d_sgjobs.p, ctx->h_sgjobs.p, sizeof(StreamJob) * n, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_sgres.p, 0, sizeof(StreamResult) * n, ctx->stream));
    if (int rc = launch_waves(ctx, ENG_CELLS, ctx->d_sgjobs.as<StreamJob>(), ctx->d_sgres.as<StreamResult>(), nullptr, n,
                              (unsigned)std::min<size_t>(n, slots), 0, nullptr))
        return rc;
    CU(cudaMemcpyAsync(ctx->h_sgres.p, ctx->d_sgres.p, sizeof(StreamResult) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    // 3. a stream is accepted when every segment ended exactly where the next one starts
    const StreamResult* sr = ctx->h_sgres.as<StreamResult>();
    std::vector<SegmentRecord> recs;
    std::vector<uint32_t> stream_first{0};
    std::vector<uint64_t> chunk_base;
    std::vector<uint32_t> accepted;
    std::vector<StreamResult> finals;
    uint64_t chunks = 0;
    for (size_t c = 0; c < cuts.size(); ++c) {
        const uint32_t lo = first_of[c], hi = first_of[c + 1];
        const StreamJob& j = h_jobs[cuts[c].stream];
        bool ok = true;
        uint64_t total = 0, blocks = 0;
        for (uint32_t k = lo; k < hi && ok; ++k) {
            const bool last = k + 1 == hi;
            ok = sr[k].status == PNGB200_OK && (last ? sr[k].phase == 2 : (sr[k].phase == 1 && sr[k].consumed_bits == sg[k].stop_bit));
            total += sr[k].produced;
            blocks += sr[k].blocks;
        }
        if (ok && total > j.dst_cap) ok = false;
        ctx->seg_streams++;
        ctx->seg_segments += hi - lo;
        if (!ok) { ctx->seg_fallbacks++; continue; }
        uint64_t off = 0;
        for (uint32_t k = lo; k < hi; ++k) {
            SegmentRecord rec;
            rec.sym = (const uint16_t*)sg[k].dst;
            rec.out = j.dst + off;
            rec.produced = sr[k].produced;
            rec.stream = cuts[c].stream;
            rec.first = k == lo;
            chunk_base.push_back(chunks);
            chunks += (sr[k].produced + 4095) / 4096;
            off += sr[k].produced;
            recs.push_back(rec);
        }
        stream_first.push_back((uint32_t)recs.size());
        accepted.push_back(cuts[c].stream);
        StreamResult f = sr[hi - 1];   // trailer fields come from the last segment
        f.produced = total;
        f.blocks = (uint32_t)blocks;
        f.resume_out = total;
        f.ck_done = 0;
        f.stat_waves = 0;
        f.stat_tokens = f.stat_matches = f.stat_deferred = 0;
        for (int q = 0; q < 12; ++q) f.stat_cycles[q] = 0;
        for (uint32_t k = lo; k < hi; ++k) {
            f.stat_waves += sr[k].stat_waves;
            f.stat_tokens += sr[k].stat_tokens;
            f.stat_matches += sr[k].stat_matches;
            f.stat_deferred += sr[k].stat_deferred;
            for (int q = 0; q < 12; ++q) f.stat_cycles[q] += sr[k].stat_cycles[q];
        }
        finals.push_back(f);
    }
    if (!recs.empty()) {
        // 4. windows in front of the segments, then markers -> bytes at their final places
        const size_t nr = recs.size(), ns = stream_first.size() - 1;
        Tables t(ctx->h_sgrec, ctx->d_sgrec);
        const size_t off_recs = t.host(recs.data(), sizeof(SegmentRecord) * nr);
        const size_t off_first = t.host(stream_first.data(), sizeof(uint32_t) * (ns + 1));
        const size_t off_chunk = t.host(chunk_base.data(), sizeof(uint64_t) * nr);
        if (int rc = t.upload(ctx)) return rc;
        CU(ctx->d_sgwin.reserve((size_t)SEG_WINDOW * nr));
        const SegmentRecord* d_recs = t.dev<SegmentRecord>(off_recs);
        window_propagate_kernel<<<(unsigned)ns, 256, 0, ctx->stream>>>(d_recs, t.dev<uint32_t>(off_first), (uint32_t)ns,
                                                                       ctx->d_sgwin.as<uint8_t>());
        if (chunks)
            marker_resolve_kernel<<<(unsigned)chunks, 256, 0, ctx->stream>>>(d_recs, (uint32_t)nr, ctx->d_sgwin.as<uint8_t>(),
                                                                             t.dev<uint64_t>(off_chunk));
        ctx->launches += 2;
        CU(cudaGetLastError());
        // the streams' result records (the whole-stream kernels will not touch them)
        StreamResult* d_results = ctx->d_results.as<StreamResult>();
        StreamResult* hf = ctx->h_sgres.as<StreamResult>();  // reuse: the segment results have been consumed
        for (size_t a = 0; a < accepted.size(); ++a) {
            hf[a] = finals[a];
            CU(cudaMemcpyAsync(d_results + accepted[a], hf + a, sizeof(StreamResult), cudaMemcpyHostToDevice, ctx->stream));
        }
        std::vector<uint32_t> rest;
        for (uint32_t i : par)
            if (std::find(accepted.begin(), accepted.end(), i) == accepted.end()) rest.push_back(i);
        par.swap(rest);
    }
    return PNGB200_OK;
}

// CTA slots the segment and split planners fill
size_t plan_slots(const pngb200_ctx* ctx) { return ctx->plan_slots ? ctx->plan_slots : (size_t)ctx->sm_count * WV_CTAS_PER_SM; }

// ---- a stream cut in two: a direct head and a symbolic tail (inflate_segments.cuh, DESIGN.md section 4.2) ----
// Per output byte, a tail costs this many times what a head costs: stat_cycles over produced (tools/split_cost.py),
// 10.64 against 10.12 cycles per byte, for the 198 x 7680x4320 RGBA8 photo batch (bench.py's default) cut at
// h = 0.763, on an H100 80GB HBM3 at a 700 W power limit and 1980 MHz.  A tail decodes symbols (about 1.38x a head's
// cost per byte) only until its last 32 KiB hold no marker, 10.3 % of its bytes on that batch, and bytes like a head
// after that.
constexpr double kSymbolicCost = 1.05;

// B big streams on N CTA slots with N / 2 < B < N: one CTA per stream would leave N - B slots idle for the whole
// launch.  Each stream is cut at a block boundary instead: heads take the first B tickets, the N - B other CTAs
// work through the tails one after another.  Head share h = B rho / (N - B + B rho) gives a chain of B / (N - B)
// tails the cost of one head.  The tail's symbols go to the stream's scratch (the image's pixel buffer, dead until
// unfilter), and once the tail leaves symbolic mode its bytes go behind them (StreamJob.may_switch): 2m + 32 KiB +
// (n2 - m) bytes for a tail of n2 bytes that switched at m, at most the 2 n2 of a tail that never does, which is what
// the scratch guard below provides for (with a margin for tails longer than 1 - h of the stream); a switched tail
// that still runs out of room fails and its stream is decoded whole.  The head's bytes are final where they land.
// On return `par` holds the streams still to be decoded whole: not cut, or cut but not accepted (split_finish_kernel)
// -- so statuses and errors are those of the whole-stream path for every input.

// the head share h when the big streams `par` are to be cut, else 0
double split_head_share(const pngb200_ctx* ctx, const StreamJob* h_jobs, const std::vector<uint32_t>& par)
{
    constexpr uint64_t kMinSplit = 1u << 20;   // compressed bytes of a stream worth cutting, at least
    const size_t slots = plan_slots(ctx), nb = par.size();
    if (!ctx->split || ctx->peer_streams || nb * 2 <= slots || nb >= slots) return 0;
    const double h = nb * kSymbolicCost / ((double)(slots - nb) + nb * kSymbolicCost);
    if (h < 0.55 || h > 0.95) return 0;   // below: the tail would not fit its scratch; above: little to gain
    for (uint32_t i : par) {   // every big stream qualifies, or none is cut (a second launch would serialise them)
        const StreamJob& j = h_jobs[i];
        if (j.format != PNGB200_FORMAT_ZLIB || j.start_bit != 0 || j.phase != 0 || j.src_len < kMinSplit || j.dst_cap < kMinSplit ||
            !j.scratch || (uintptr_t)j.scratch % 16 || (double)j.scratch_cap < 2.5 * (1.0 - h) * (double)j.dst_cap + 4096)
            return 0;
    }
    return h;
}

int run_split(pngb200_ctx* ctx, const StreamJob* h_jobs, std::vector<uint32_t>& par, double h)
{
    const size_t slots = plan_slots(ctx), nb = par.size();
    // 1. split points: the first plausible dynamic-block header at or after h of the stream
    CU(ctx->h_sgsearch.reserve(sizeof(SearchJob) * nb));
    SearchJob* sj = ctx->h_sgsearch.as<SearchJob>();
    for (size_t k = 0; k < nb; ++k) {
        const StreamJob& j = h_jobs[par[k]];
        sj[k] = SearchJob{j.src, j.src_len, (uint64_t)(h * (double)(8 * j.src_len)), 8 * j.src_len, ~0ull};
    }
    if (int rc = search_blocks(ctx, nb)) return rc;
    // 2. heads (LPT order, first tickets), then the tails in the same order
    std::vector<uint32_t> cut, rest;
    for (size_t k = 0; k < nb; ++k) (sj[k].found != ~0ull ? cut : rest).push_back(par[k]);
    const size_t n = cut.size();
    if (n == 0) return PNGB200_OK;
    CU(ctx->h_sgjobs.reserve(sizeof(StreamJob) * 2 * n));
    CU(ctx->d_sgjobs.reserve(sizeof(StreamJob) * 2 * n));
    // the pieces' results, then where each job left symbolic mode (SwitchRecord; only the tails' are written)
    const size_t res_bytes = sizeof(StreamResult) * 2 * n + sizeof(SwitchRecord) * 2 * n;
    static_assert(sizeof(StreamResult) % alignof(SwitchRecord) == 0, "switch records behind the results");
    CU(ctx->d_sgres.reserve(res_bytes));
    StreamJob* sg = ctx->h_sgjobs.as<StreamJob>();
    uint64_t max_cap = 0;
    for (size_t k = 0, s = 0; k < nb; ++k) {
        if (sj[k].found == ~0ull) continue;
        const StreamJob& j = h_jobs[par[k]];
        StreamJob& hd = sg[s];
        StreamJob& tl = sg[n + s];
        ++s;
        hd = j;
        hd.stop_bit = sj[k].found;
        tl = j;
        tl.start_bit = sj[k].found;
        tl.phase = 1;
        tl.symbolic = 1;
        tl.may_switch = 1;
        tl.dst = j.scratch;
        tl.dst_cap = j.scratch_cap / 2 - 64;   // symbols, with the kernel's store slack behind them
        max_cap = std::max(max_cap, j.dst_cap);
    }
    CU(cudaMemcpyAsync(ctx->d_sgjobs.p, sg, sizeof(StreamJob) * 2 * n, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_sgres.p, 0, res_bytes, ctx->stream));
    SwitchRecord* d_switch = (SwitchRecord*)(ctx->d_sgres.as<StreamResult>() + 2 * n);
    if (int rc = launch_waves(ctx, ENG_WAVE, ctx->d_sgjobs.as<StreamJob>(), ctx->d_sgres.as<StreamResult>(), nullptr, 2 * n,
                              (unsigned)std::min<size_t>(2 * n, slots), max_cap, d_switch))
        return rc;
    // 3. tails -> bytes behind their heads, Adler-32 of the whole stream, acceptance; device-side, one host round trip
    std::vector<SplitRecord> rec(n);
    const StreamResult* d_sgres = ctx->d_sgres.as<StreamResult>();
    for (size_t s = 0; s < n; ++s) {
        const StreamJob& j = h_jobs[cut[s]];
        rec[s] = SplitRecord{d_sgres + s, d_sgres + n + s, (const uint16_t*)j.scratch, j.dst, j.dst_cap, sg[s].stop_bit,
                             ctx->d_results.as<StreamResult>() + cut[s], d_switch + n + s};
    }
    Tables t(ctx->h_sgrec, ctx->d_sgrec);
    const size_t off_rec = t.host(rec.data(), sizeof(SplitRecord) * n);
    const size_t off_accept = t.device(sizeof(uint32_t) * n, false);
    const size_t off_partial = t.device(sizeof(uint32_t) * 2 * SPLIT_CTAS * n, false);
    if (int rc = t.upload(ctx, off_partial)) return rc;   // the accept flags come back behind the records
    const SplitRecord* d_rec = t.dev<SplitRecord>(off_rec);
    uint32_t* d_accept  = t.dev<uint32_t>(off_accept);
    uint32_t* d_partial = t.dev<uint32_t>(off_partial);
    split_resolve_kernel<<<dim3((unsigned)n, SPLIT_CTAS), 256, 0, ctx->stream>>>(d_rec, d_partial);
    split_finish_kernel<<<(unsigned)((n + 127) / 128), 128, 0, ctx->stream>>>(d_rec, (uint32_t)n, d_partial, d_accept);
    ctx->launches += 2;
    CU(cudaGetLastError());
    uint32_t* accept = t.pin<uint32_t>(off_accept);
    CU(cudaMemcpyAsync(accept, d_accept, sizeof(uint32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CU(ctx->h_sgres.reserve(res_bytes));
    CU(cudaMemcpyAsync(ctx->h_sgres.p, d_sgres, res_bytes, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    ctx->seg_streams += n;
    ctx->seg_segments += 2 * n;
    const StreamResult* pieces = ctx->h_sgres.as<StreamResult>();
    const SwitchRecord* switched = (const SwitchRecord*)(pieces + 2 * n);
    for (size_t s = 0; s < n; ++s) {
        if (!accept[s]) {
            ctx->seg_fallbacks++;
            rest.push_back(cut[s]);
            continue;
        }
        const StreamResult &hd = pieces[s], &tl = pieces[n + s];
        ctx->split_stats[0] += hd.produced;
        ctx->split_stats[2] += tl.produced;
        for (int q = 0; q < 12; ++q) {
            ctx->split_stats[1] += hd.stat_cycles[q];
            ctx->split_stats[3] += tl.stat_cycles[q];
        }
        const SwitchRecord& sw = switched[n + s];
        ctx->split_stats[4] += sw.out < tl.produced;
        ctx->split_stats[5] += sw.out;
    }
    // what is left keeps its longest-first order
    std::vector<uint32_t> left;
    for (uint32_t i : par)
        if (std::find(rest.begin(), rest.end(), i) != rest.end()) left.push_back(i);
    par.swap(left);
    return PNGB200_OK;
}

// Stream checksums (Adler-32, CRC-32 for gzip) of `count` inflated jobs, in chunks laid out from dst_cap (an upper
// bound of `produced`).  `h_base`: count + 1 words of host staging for the chunk bases, uploaded to `d_base`.
int run_checksum(pngb200_ctx* ctx, const StreamJob* h_jobs, const StreamJob* d_jobs, StreamResult* d_results, size_t count,
                 uint32_t* h_base, DevBuf& d_base, DevBuf& d_partial)
{
    uint64_t total = 0;
    for (size_t i = 0; i < count; ++i) {
        h_base[i] = (uint32_t)total;
        total += (h_jobs[i].dst_cap + CK_CHUNK - 1) / CK_CHUNK;
    }
    h_base[count] = (uint32_t)total;
    if (total >= (1ull << 31)) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "batch too large");
    CU(d_base.reserve(sizeof(uint32_t) * (count + 1)));
    CU(d_partial.reserve(sizeof(uint64_t) * 2 * std::max<uint64_t>(total, 1)));
    CU(cudaMemcpyAsync(d_base.p, h_base, sizeof(uint32_t) * (count + 1), cudaMemcpyHostToDevice, ctx->stream));
    ChecksumParams cp;
    cp.jobs = d_jobs;
    cp.results = d_results;
    cp.chunk_base = d_base.as<uint32_t>();
    cp.partial = d_partial.as<uint64_t>();
    cp.count = (uint32_t)count;
    cp.total_chunks = (uint32_t)total;
    cp.crc_tables = nullptr;
    for (size_t i = 0; i < count; ++i)
        if (h_jobs[i].format == PNGB200_FORMAT_GZIP) {
            if (int rc = ensure_crc_tables(ctx)) return rc;
            cp.crc_tables = ctx->d_crctab.as<uint32_t>();
            break;
        }
    if (total) {
        checksum_chunk_kernel<<<(unsigned)total, CK_THREADS, 0, ctx->stream>>>(cp);
        ctx->launches++;
    }
    checksum_fold_kernel<<<(unsigned)count, 32, 0, ctx->stream>>>(cp);
    ctx->launches++;
    CU(cudaGetLastError());
    return PNGB200_OK;
}

// ---- inflate (+ checksum) over a device-resident job table ----
// h_jobs: host copy (for dst_cap based chunk layout); d_jobs/d_results device arrays of `count`.
int run_inflate(pngb200_ctx* ctx, const StreamJob* h_jobs, size_t count)
{
    ctx->last_engine = -1;
    StreamJob*    d_jobs    = ctx->d_jobs.as<StreamJob>();
    StreamResult* d_results = ctx->d_results.as<StreamResult>();
    ctx->seg_streams = ctx->seg_segments = ctx->seg_fallbacks = 0;
    for (uint64_t& v : ctx->split_stats) v = 0;
    CU(cudaMemsetAsync(d_results, 0, sizeof(StreamResult) * count, ctx->stream));
    bool hooked = false;
    auto before_first_launch = [&]() -> int {   // once, in front of the batch's first kernel
        if (hooked) return PNGB200_OK;
        hooked = true;
        int rc = PNGB200_OK;
        if (ctx->bulk_h2d) {
            rc = ctx->bulk_h2d();
            ctx->bulk_h2d = nullptr;
        }
        if (rc == PNGB200_OK) CU(cudaEventRecord(ctx->ev[0], ctx->stream));
        return rc;
    };
    // big streams get a whole CTA each (block-parallel kernel); tiny ones a warp each
    {
        std::vector<uint32_t> par, ser;
        for (size_t i = 0; i < count; ++i) {
            bool big = h_jobs[i].src_len >= ctx->parallel_threshold;
            if (ctx->inflate_mode == 1) big = false;
            if (ctx->inflate_mode == 2) big = true;
            (big ? par : ser).push_back((uint32_t)i);
        }
        // longest first: the persistent CTAs pull streams from a ticket, so this is LPT scheduling
        std::stable_sort(par.begin(), par.end(),
                         [&](uint32_t a, uint32_t b) { return h_jobs[a].src_len > h_jobs[b].src_len; });
        CU(ctx->h_order.reserve(sizeof(uint32_t) * count));
        CU(ctx->d_order.reserve(sizeof(uint32_t) * count));
        uint32_t* ho = ctx->h_order.as<uint32_t>();
        std::copy(par.begin(), par.end(), ho);
        std::copy(ser.begin(), ser.end(), ho + par.size());
        CU(cudaMemcpyAsync(ctx->d_order.p, ho, sizeof(uint32_t) * count, cudaMemcpyHostToDevice, ctx->stream));
        const uint32_t* d_order = ctx->d_order.as<uint32_t>();
        if (ctx->inflate_mode == 0 || ctx->inflate_mode == 5) {
            // few big streams: cut them so that every CTA slot has something to decode
            const size_t before = par.size();
            if (!par.empty() && std::max(par.size(), ctx->peer_streams) * 2 <= plan_slots(ctx)) {
                if (int rc = before_first_launch()) return rc;
                if (int rc = run_segments(ctx, h_jobs, par)) return rc;
            } else if (const double h = split_head_share(ctx, h_jobs, par)) {
                if (int rc = before_first_launch()) return rc;
                if (int rc = run_split(ctx, h_jobs, par, h)) return rc;
            }
            if (par.size() != before) {   // the order table lists what is left for the whole-stream kernels
                std::copy(par.begin(), par.end(), ho);
                std::copy(ser.begin(), ser.end(), ho + par.size());
                CU(cudaMemcpyAsync(ctx->d_order.p, ho, sizeof(uint32_t) * (par.size() + ser.size()), cudaMemcpyHostToDevice, ctx->stream));
            }
        }
        if (!par.empty()) {
            uint64_t max_cap = 0;
            for (uint32_t i : par) max_cap = std::max<uint64_t>(max_cap, h_jobs[i].dst_cap);
            // Three engines for the big streams, same decomposition (8 KiB waves of 256 subsequences):
            //  * inflate_wave_kernel: LZ77 window in a 64 KiB shared-memory ring, Adler-32 folded into the store;
            //    2 CTAs per SM.  Fastest per stream (146 K cycles per wave against 234 K), so it takes every batch
            //    that fits its 2 x SMs CTA slots, and the heads and tails of run_split.
            //  * inflate_parallel_kernel (round 1): 16 KiB output image, window read back from HBM/L2, 4 CTAs per
            //    SM.  Slower per stream, but twice the streams in flight hide its barrier phases once a batch
            //    exceeds the wave kernel's slots.
            //  * inflate_cells_kernel (round 2, second half): the same waves, but the LZ77 half works on 16-bit cells in
            //    shared memory resolved by pointer jumping; no window in shared memory, 3 CTAs per SM.  It decodes the
            //    segments of run_segments; whole streams go to it only in inflate mode 6.
            // The automatic choice goes by how many streams there are to keep the SMs busy.
            const size_t wave_slots = (size_t)ctx->sm_count * WV_CTAS_PER_SM;
            const size_t streams_in_flight = std::max(par.size(), ctx->peer_streams);   // (lanes: the chunks of a host batch run side by side)
            Engine engine = streams_in_flight <= wave_slots ? ENG_WAVE : ENG_PARALLEL;
            if (ctx->inflate_mode == 3) engine = ENG_WAVE;
            if (ctx->inflate_mode == 4) engine = ENG_PARALLEL;
            if (ctx->inflate_mode == 6) engine = ENG_CELLS;
            ctx->last_engine = engine;
            const size_t engine_slots = engine == ENG_CELLS  ? (size_t)ctx->sm_count * CL_CTAS_PER_SM
                                        : engine == ENG_WAVE ? wave_slots
                                                             : (size_t)ctx->sm_count * PAR_CTAS_PER_SM;
            if (int rc = launch_waves(ctx, engine, d_jobs, d_results, d_order, par.size(), (unsigned)std::min(par.size(), engine_slots),
                                      max_cap, nullptr, before_first_launch))
                return rc;
        }
        if (int rc = before_first_launch()) return rc;
        if (!ser.empty()) {
            inflate_serial_kernel<<<(unsigned)ser.size(), 32, 0, ctx->stream>>>(d_jobs, d_results, d_order + par.size(),
                                                                                 (int)ser.size());
            ctx->launches++;
        }
        CU(cudaGetLastError());
    }
    CU(cudaEventRecord(ctx->ev[1], ctx->stream));
    CU(ctx->h_misc.reserve(sizeof(uint32_t) * (count + 1)));
    if (int rc = run_checksum(ctx, h_jobs, d_jobs, d_results, count, ctx->h_misc.as<uint32_t>(), ctx->d_misc, ctx->d_partial))
        return rc;
    CU(cudaEventRecord(ctx->ev[2], ctx->stream));
    return PNGB200_OK;
}

struct Geometry {
    uint64_t filtered;  // total filtered bytes
    uint64_t storage;
    uint32_t pitch;     // non-interlaced pitch
    uint8_t  bpp;
    bool     fast;      // eligible for the wavefront kernel
    bool     passes;    // Adam7 or 1/2/4-bit samples in a PNG layout: eligible for the pass path (see run_unfilter)
};

bool geometry(uint32_t w, uint32_t h, int volume, int depth, int interlaced, Geometry* g)
{
    if (w == 0 || h == 0 || volume <= 0 || volume > 64 || depth <= 0 || depth > 16) return false;
    // Dimensions come from untrusted files: the reference traps when w * h * bpp overflows (PNG.Image.swift:84);
    // here an image whose sizes do not fit is refused before any buffer is sized from a wrapped product.
    {
        if (w > 0x7fffffffu || h > 0x7fffffffu) return false;
        const uint64_t pitch64 = ((uint64_t)w * (uint64_t)volume + 7) >> 3;
        uint64_t prod;
        if (pitch64 > 0xfffffff0ull) return false;
        if (__builtin_mul_overflow((uint64_t)h, pitch64 + 1, &prod) || prod > (1ull << 46)) return false;
        if (__builtin_mul_overflow((uint64_t)w * (uint64_t)h, (uint64_t)((volume + 7) >> 3), &prod) || prod > (1ull << 46)) return false;
    }
    g->filtered = pngb200_filtered_size(w, h, volume, interlaced);
    g->storage  = pngb200_storage_size(w, h, volume);
    g->pitch    = (uint32_t)(((uint64_t)w * volume + 7) >> 3);
    g->bpp      = (uint8_t)((volume + 7) >> 3);
    g->fast     = !interlaced && depth >= 8 &&
              (g->bpp == 1 || g->bpp == 2 || g->bpp == 3 || g->bpp == 4 || g->bpp == 6 || g->bpp == 8);
    // whole bytes per pixel with the wavefront's filter distances, or one 1/2/4-bit sample per pixel
    const bool layout = depth >= 8 ? volume % 8 == 0 && (g->bpp <= 4 || g->bpp == 6 || g->bpp == 8)
                                   : volume == depth && (depth == 1 || depth == 2 || depth == 4);
    g->passes   = !g->fast && layout;
    return true;
}

// a decode or unfilter batch starts: its images are counted from zero on the context and on its lanes
void start_unfilter_stats(pngb200_ctx* ctx)
{
    for (pngb200_ctx* lane : ctx->lanes)
        for (uint64_t& n : lane->unfilter_images) n = 0;
    for (uint64_t& n : ctx->unfilter_images) n = 0;
}

// unfilter stage over device-resident filtered streams
struct UnfilterItem {
    const uint8_t*      filtered;
    uint8_t*            filtered_mut;  // same buffer when the library owns it, else null
    uint8_t*            pixels;
    const StreamResult* inflated;
    uint64_t            filtered_len;
    uint32_t            w, h;
    uint8_t             volume, depth, interlaced;
    Geometry            g;
};

// Images of the pass path (Adam7 or 1/2/4-bit) whose filtered stream is at most this long go to
// unfilter_generic_kernel instead: below it, planning up to seven jobs an image and two launches cost more than one CTA
// per image spends on its rows (DESIGN §4.3, the size sweep of tools/unfilter_passes_bw.py).
constexpr uint64_t UNFILTER_GENERIC_MAX = 65536;

int run_unfilter(pngb200_ctx* ctx, const std::vector<UnfilterItem>& items)
{
    ctx->d_hist = nullptr;

    std::vector<ImageJob>      fast;
    std::vector<GenericJob>    slow;
    std::vector<InterleaveJob> inter;
    std::vector<PassJob>       pass;
    std::vector<uint32_t>      band_base;
    uint64_t                   inter_blocks = 0;
    for (const UnfilterItem& it : items) {
        if (it.g.fast) {
            ImageJob j;
            j.filtered = it.filtered;
            j.pixels = it.pixels;
            j.inflated = it.inflated;
            j.filtered_len = it.filtered_len;
            j.width = it.w;
            j.height = it.h;
            j.pitch = it.g.pitch;
            j.volume = it.volume;
            j.depth = it.depth;
            j.interlaced = 0;
            j.bpp = it.g.bpp;
            fast.push_back(j);
            continue;
        }
        PassImageJob j;
        j.filtered = it.filtered_mut;
        j.pixels = it.pixels;
        j.inflated = it.inflated;
        j.filtered_len = it.filtered_len;
        j.block_base = 0;
        j.width = it.w;
        j.height = it.h;
        j.volume = it.volume;
        j.depth = it.depth;
        j.interlaced = it.interlaced;
        j.bpp = it.g.bpp;
        if (it.g.passes && it.g.filtered > UNFILTER_GENERIC_MAX) plan_passes(j, pass, inter, inter_blocks);
        else slow.push_back(j);
    }
    // the fast and the pass path hand out their bands level by level
    std::vector<uint32_t> level_start, pass_base, pass_levels;
    const uint64_t bands = plan_bands(fast, band_base, level_start);
    const uint64_t pass_bands = plan_bands(pass, pass_base, pass_levels);
    if (bands >= (1ull << 31) || pass_bands >= (1ull << 31)) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "batch too large");
    ctx->unfilter_images[0] += fast.size();
    ctx->unfilter_images[1] += inter.size();
    ctx->unfilter_images[2] += slow.size();
    if (!fast.empty()) {
        Tables t(ctx->h_imgjobs, ctx->d_imgjobs);
        const size_t off_jobs = t.host(fast.data(), sizeof(ImageJob) * fast.size());
        const size_t off_bb = t.host(band_base.data(), sizeof(uint32_t) * band_base.size());
        const size_t off_ls = t.host(level_start.data(), sizeof(uint32_t) * level_start.size());
        t.host(nullptr, 0);   // the copy runs on up to the counters
        // per-band progress and the ticket, padded to 8 bytes, then the filter-type histogram: one zeroed region
        const size_t progress = sizeof(uint32_t) * ((bands + 2) / 2 * 2);
        const size_t off_pr = t.device(progress + 8 * sizeof(unsigned long long), true);
        if (int rc = t.upload(ctx)) return rc;
        WaveParams p;
        p.jobs = t.dev<ImageJob>(off_jobs);
        p.band_base = t.dev<uint32_t>(off_bb);
        p.progress = t.dev<uint32_t>(off_pr);
        p.ticket = p.progress + bands;
        p.hist = t.dev<unsigned long long>(off_pr + progress);
        ctx->d_hist = p.hist;
        p.njobs = (uint32_t)fast.size();
        p.total_bands = (uint32_t)bands;
        p.level_start = t.dev<uint32_t>(off_ls);
        p.levels = level_start.empty() ? 0u : (uint32_t)level_start.size() - 1;
        unsigned grid = (unsigned)std::min<uint64_t>((bands + WAVE_WARPS - 1) / WAVE_WARPS,
                                                     (uint64_t)ctx->sm_count * 8);
        unfilter_wave_kernel<<<grid, WAVE_WARPS * 32, WAVE_SMEM, ctx->stream>>>(p);
        ctx->launches++;
        CU(cudaGetLastError());
    }
    if (pass.empty() && slow.empty()) return PNGB200_OK;
    // the pass path and the generic kernel share one table upload
    Tables t(ctx->h_genjobs, ctx->d_genjobs);
    const size_t off_gen = t.host(slow.data(), sizeof(GenericJob) * slow.size());
    const size_t off_pass = t.host(pass.data(), sizeof(PassJob) * pass.size());
    const size_t off_pb = t.host(pass_base.data(), sizeof(uint32_t) * pass_base.size());
    const size_t off_pl = t.host(pass_levels.data(), sizeof(uint32_t) * pass_levels.size());
    const size_t off_inter = t.host(inter.data(), sizeof(InterleaveJob) * inter.size());
    const size_t off_pr = t.device(sizeof(uint32_t) * (pass_bands + 1), true);   // per-band progress, then the ticket
    if (int rc = t.upload(ctx)) return rc;
    if (!pass.empty()) {
        WaveParams p;
        p.jobs = t.dev<PassJob>(off_pass);
        p.band_base = t.dev<uint32_t>(off_pb);
        p.progress = t.dev<uint32_t>(off_pr);
        p.ticket = p.progress + pass_bands;
        p.hist = nullptr;
        p.njobs = (uint32_t)pass.size();
        p.total_bands = (uint32_t)pass_bands;
        p.level_start = t.dev<uint32_t>(off_pl);
        p.levels = pass_levels.empty() ? 0u : (uint32_t)pass_levels.size() - 1;
        unsigned grid = (unsigned)std::min<uint64_t>((pass_bands + WAVE_WARPS - 1) / WAVE_WARPS,
                                                     (uint64_t)ctx->sm_count * 8);
        unfilter_pass_kernel<<<grid, WAVE_WARPS * 32, WAVE_SMEM, ctx->stream>>>(p);
        ctx->launches++;
        CU(cudaGetLastError());
        grid = (unsigned)std::min<uint64_t>(inter_blocks, (uint64_t)ctx->sm_count * 16);
        unfilter_interleave_kernel<<<grid, INTERLEAVE_THREADS, 0, ctx->stream>>>(t.dev<InterleaveJob>(off_inter),
                                                                                 (uint32_t)inter.size(), inter_blocks);
        ctx->launches++;
        CU(cudaGetLastError());
    }
    if (!slow.empty()) {
        unfilter_generic_kernel<<<(unsigned)slow.size(), 128, 0, ctx->stream>>>(t.dev<GenericJob>(off_gen), (int)slow.size());
        ctx->launches++;
        CU(cudaGetLastError());
    }
    return PNGB200_OK;
}


// Host-memory batches with a lot of bytes to move are cut into chunks that four lanes (helper
// contexts on the same GPU, one host thread each) work through round-robin, so that one chunk's
// H2D / D2H copies overlap another chunk's kernels.  Results are identical: images are
// independent units.  Chunk size is a trade: the inflate kernel runs one CTA per stream, so small
// chunks leave SMs idle, while few chunks leave nothing to overlap.  The rule: about one stream
// per SM in every chunk, chunk count a multiple of the lane count.
// `bytes_of(i)`: bytes item i moves over PCIe; `work(lane, lo, n)`: process items [lo, lo + n) on `lane`.
template <typename BytesOf, typename Work>
int run_over_lanes(pngb200_ctx* ctx, size_t count, int memspace, BytesOf bytes_of, Work work)
{
    for (pngb200_ctx* lane : ctx->lanes) lane->d_hist = nullptr;   // counters describe the batch that starts now
    ctx->d_hist = nullptr;
    start_unfilter_stats(ctx);
    size_t bytes = 0;
    for (size_t i = 0; i < count; ++i) bytes += bytes_of(i);
    // tunable for experiments: PNGB200_LANES, PNGB200_CHUNKS_PER_LANE (0 / unset = the rule above); read once
    static const size_t kLanes = getenv("PNGB200_LANES") ? std::max(1, atoi(getenv("PNGB200_LANES"))) : 4;
    static const size_t kPerLane = getenv("PNGB200_CHUNKS_PER_LANE") ? std::max(0, atoi(getenv("PNGB200_CHUNKS_PER_LANE"))) : 0;
    constexpr size_t kMinChunk = 32;
    if (memspace != PNGB200_MEM_HOST || count < 2 * kMinChunk || bytes < ((size_t)256 << 20)) return work(ctx, 0, count);
    while (ctx->lanes.size() < kLanes) {
        pngb200_ctx* lane = pngb200_ctx_create(ctx->device);
        if (!lane) return set_error(ctx, PNGB200_ERR_CUDA, "cannot create a pipeline lane: %s", g_last_error.c_str());
        ctx->lanes.push_back(lane);
    }
    size_t nchunks;
    if (kPerLane) {
        nchunks = kPerLane * kLanes;
    } else {
        nchunks = std::max<size_t>(1, count / (size_t)ctx->sm_count);
        nchunks = (nchunks + kLanes - 1) / kLanes * kLanes;
    }
    nchunks = std::max<size_t>(1, std::min(nchunks, count / kMinChunk));
    std::vector<size_t> cut(nchunks + 1);  // chunk boundaries balanced by bytes
    {
        size_t acc = 0, k = 1;
        cut[0] = 0;
        for (size_t i = 0; i < count && k < nchunks; ++i) {
            acc += bytes_of(i);
            if (acc * nchunks >= bytes * k) cut[k++] = i + 1;
        }
        while (k <= nchunks) cut[k++] = count;
    }
    std::vector<int> rcs(kLanes, PNGB200_OK);
    std::vector<std::thread> workers;
    for (size_t l = 0; l < kLanes; ++l)
        workers.emplace_back([&, l]() {
            pngb200_ctx* lane = ctx->lanes[l];
            lane->inflate_mode = ctx->inflate_mode;
            lane->parallel_threshold = ctx->parallel_threshold;
            lane->peer_streams = count;
            for (size_t c = l; c < nchunks; c += kLanes) {
                size_t lo = cut[c], n = cut[c + 1] - cut[c];
                if (n == 0) continue;
                int rc = work(lane, lo, n);
                if (rc != PNGB200_OK) { rcs[l] = rc; return; }   // the lane keeps its own error text
            }
        });
    for (std::thread& t : workers) t.join();
    for (size_t l = 0; l < kLanes; ++l)
        if (rcs[l] != PNGB200_OK) {
            ctx->error = ctx->lanes[l]->error;   // after the join: one writer
            return rcs[l];
        }
    return PNGB200_OK;
}
}  // namespace

// ================================ C ABI ================================

extern "C" {

size_t pngb200_filtered_size(uint32_t w, uint32_t h, int volume, int interlaced)
{
    return stream_pass_offset(7, w, h, (size_t)volume, interlaced);
}

size_t pngb200_storage_size(uint32_t w, uint32_t h, int volume)
{
    return (size_t)w * (size_t)h * (size_t)((volume + 7) >> 3);
}

pngb200_ctx* pngb200_ctx_create(int device)
{
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        set_error(nullptr, PNGB200_ERR_CUDA, "no CUDA device: %s (there is no CPU fallback)",
                  e != cudaSuccess ? cudaGetErrorString(e) : "device count is 0");
        return nullptr;
    }
    if (device < 0) cudaGetDevice(&device);
    if (device >= n) {
        set_error(nullptr, PNGB200_ERR_BAD_ARGUMENT, "device %d out of range (%d devices)", device, n);
        return nullptr;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
        set_error(nullptr, PNGB200_ERR_CUDA, "device %d is sm_%d%d; this library is built for sm_90a only",
                  device, prop.major, prop.minor);
        return nullptr;
    }
    pngb200_ctx* ctx = new pngb200_ctx();
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    ctx->device_bytes = prop.totalGlobalMem;
    if (const char* v = getenv("PNGB200_SPLIT")) ctx->split = atoi(v) != 0;   // tuning overrides, read once per context
    if (const char* v = getenv("PNGB200_PLAN_SLOTS")) ctx->plan_slots = (size_t)std::max(0, atoi(v));
    DeviceGuard guard(device);
    // each kernel launched with dynamic shared memory opts in to its size
    const std::pair<const void*, size_t> opt_in[] = {
        {(const void*)deflate_kernel, sizeof(DfShared)},          {(const void*)inflate_parallel_kernel3, sizeof(ParShared)},
        {(const void*)inflate_parallel_kernel, sizeof(ParShared)}, {(const void*)inflate_wave_kernel, sizeof(WvShared)},
        {(const void*)unfilter_wave_kernel, WAVE_SMEM},           {(const void*)inflate_cells_kernel, sizeof(ClShared)},
        {(const void*)unfilter_pass_kernel, WAVE_SMEM},           {(const void*)deflate_resume_kernel, sizeof(DfShared)}};
    for (const auto& [kernel, bytes] : opt_in)
        if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes) != cudaSuccess) {
            set_error(nullptr, PNGB200_ERR_CUDA, "cannot opt in to %zu bytes of shared memory", bytes);
            delete ctx;
            return nullptr;
        }
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess) {
        set_error(nullptr, PNGB200_ERR_CUDA, "cudaStreamCreate failed");
        delete ctx;
        return nullptr;
    }
    for (cudaEvent_t& e : ctx->ev) cudaEventCreate(&e);
    return ctx;
}

void pngb200_ctx_destroy(pngb200_ctx* ctx)
{
    if (!ctx) return;
    for (pngb200_ctx* lane : ctx->lanes) pngb200_ctx_destroy(lane);
    ctx->lanes.clear();
    DeviceGuard guard(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    for (cudaEvent_t e : ctx->ev) if (e) cudaEventDestroy(e);
    cudaStreamDestroy(ctx->stream);
    delete ctx;   // frees the workspaces
}

int pngb200_ctx_trim(pngb200_ctx* ctx)
{
    if (!ctx) return PNGB200_ERR_BAD_ARGUMENT;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    for (pngb200_ctx* lane : ctx->lanes) pngb200_ctx_trim(lane);
    DeviceGuard guard(ctx->device);
    CU(cudaStreamSynchronize(ctx->stream));
    for (DevBuf* b : {&ctx->d_partial, &ctx->d_filtered, &ctx->d_in, &ctx->d_out, &ctx->d_scratch, &ctx->d_dfscratch, &ctx->d_enc, &ctx->d_file, &ctx->d_sgsym, &ctx->d_sgwin,
                      &ctx->d_st, &ctx->d_stbase, &ctx->d_stpartial, &ctx->d_stin})
        b->release();
    for (PinBuf* b : {&ctx->h_st, &ctx->h_stin, &ctx->h_dfout}) b->release();
    ctx->scratch_stride = 0;
    return PNGB200_OK;
}

const char* pngb200_last_error(const pngb200_ctx* ctx) { return ctx ? ctx->error.c_str() : g_last_error.c_str(); }
void*       pngb200_ctx_stream(pngb200_ctx* ctx) { return ctx ? (void*)ctx->stream : nullptr; }
int         pngb200_ctx_device(const pngb200_ctx* ctx) { return ctx ? ctx->device : -1; }
uint64_t    pngb200_ctx_launch_count(const pngb200_ctx* ctx)
{
    if (!ctx) return 0;
    uint64_t n = ctx->launches;
    for (const pngb200_ctx* lane : ctx->lanes) n += lane->launches;
    return n;
}
void        pngb200_ctx_set_inflate_mode(pngb200_ctx* ctx, int mode) { if (ctx) ctx->inflate_mode = mode; }

int pngb200_ctx_inflate_stats(pngb200_ctx* ctx, size_t count, uint64_t out[4])
{
    if (!ctx || !out || ctx->h_results.cap < sizeof(StreamResult) * count) return PNGB200_ERR_BAD_ARGUMENT;
    const StreamResult* r = ctx->h_results.as<StreamResult>();
    out[0] = out[1] = out[2] = out[3] = 0;
    for (size_t i = 0; i < count; ++i) {
        out[0] += r[i].stat_waves;
        out[1] += r[i].stat_sync_rounds;
        out[2] += r[i].stat_resolve_rounds;
        out[3] += r[i].stat_fallback;
    }
    return PNGB200_OK;
}

int pngb200_ctx_inflate_counters(pngb200_ctx* ctx, size_t count, uint64_t out[24])
{
    if (!ctx || !out || ctx->h_results.cap < sizeof(StreamResult) * count) return PNGB200_ERR_BAD_ARGUMENT;
    const StreamResult* r = ctx->h_results.as<StreamResult>();
    for (int k = 0; k < 24; ++k) out[k] = 0;
    for (size_t i = 0; i < count; ++i) {
        out[0] += r[i].stat_waves;
        out[1] += r[i].stat_sync_rounds;
        out[2] += r[i].stat_resolve_rounds;
        out[3] += r[i].stat_fallback;
        out[4] += r[i].stat_tokens;
        out[5] += r[i].stat_matches;
        out[6] += r[i].stat_deferred;
        out[7] += r[i].blocks;
        for (int k = 0; k < 12; ++k) out[8 + k] += r[i].stat_cycles[k];
    }
    return PNGB200_OK;
}

int pngb200_ctx_filter_histogram(pngb200_ctx* ctx, uint64_t out[6])
{
    if (!ctx || !out) return PNGB200_ERR_BAD_ARGUMENT;
    for (int k = 0; k < 6; ++k) out[k] = 0;
    DeviceGuard guard(ctx->device);
    std::vector<pngb200_ctx*> all{ctx};
    all.insert(all.end(), ctx->lanes.begin(), ctx->lanes.end());
    for (pngb200_ctx* c : all) {
        if (!c->d_hist) continue;
        unsigned long long h[6];
        CU(cudaStreamSynchronize(c->stream));
        CU(cudaMemcpy(h, c->d_hist, sizeof h, cudaMemcpyDeviceToHost));
        for (int k = 0; k < 6; ++k) out[k] += h[k];
    }
    return PNGB200_OK;
}

int pngb200_ctx_last_inflate_engine(pngb200_ctx* ctx) { return ctx ? ctx->last_engine : -1; }

int pngb200_ctx_unfilter_stats(pngb200_ctx* ctx, uint64_t out[3])
{
    if (!ctx || !out) return PNGB200_ERR_BAD_ARGUMENT;
    for (int k = 0; k < 3; ++k) {
        out[k] = ctx->unfilter_images[k];
        for (const pngb200_ctx* lane : ctx->lanes) out[k] += lane->unfilter_images[k];
    }
    return PNGB200_OK;
}

int pngb200_ctx_split_stats(pngb200_ctx* ctx, uint64_t out[6])
{
    if (!ctx || !out) return PNGB200_ERR_BAD_ARGUMENT;
    for (int k = 0; k < 6; ++k) out[k] = ctx->split_stats[k];
    return PNGB200_OK;
}

int pngb200_ctx_clone_stats(pngb200_ctx* ctx, uint64_t out[2])
{
    if (!ctx || !out) return PNGB200_ERR_BAD_ARGUMENT;
    out[0] = ctx->clone_bytes[0];
    out[1] = ctx->clone_bytes[1];
    return PNGB200_OK;
}

int pngb200_ctx_segment_stats(pngb200_ctx* ctx, uint64_t out[3])
{
    if (!ctx || !out) return PNGB200_ERR_BAD_ARGUMENT;
    out[0] = ctx->seg_streams;
    out[1] = ctx->seg_segments;
    out[2] = ctx->seg_fallbacks;
    return PNGB200_OK;
}

int pngb200_ctx_stage_ms(pngb200_ctx* ctx, float ms[3])
{
    if (!ctx || !ms) return PNGB200_ERR_BAD_ARGUMENT;
    DeviceGuard guard(ctx->device);
    for (int i = 0; i < 3; ++i)
        if (cudaEventElapsedTime(&ms[i], ctx->ev[i], ctx->ev[i + 1]) != cudaSuccess) {
            cudaGetLastError();
            return set_error(ctx, PNGB200_ERR_CUDA, "stage events not recorded yet");
        }
    return PNGB200_OK;
}

// ---------------- standalone inflate ----------------
int pngb200_inflate_batch(pngb200_ctx* ctx, pngb200_stream_desc* s, size_t count, int memspace)
{
    if (!ctx || (!s && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    if (count == 0) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    CU(ctx->h_jobs.reserve(sizeof(StreamJob) * count));
    CU(ctx->d_jobs.reserve(sizeof(StreamJob) * count));
    CU(ctx->d_results.reserve(sizeof(StreamResult) * count));
    CU(ctx->h_results.reserve(sizeof(StreamResult) * count));
    StreamJob* jobs = ctx->h_jobs.as<StreamJob>();
    std::vector<size_t> in_off(count), out_off(count);
    Slots in{16}, out{16};
    for (size_t i = 0; i < count; ++i) {
        if ((!s[i].src && s[i].src_len) || (!s[i].dst && s[i].dst_cap) || s[i].format < 0 || s[i].format > 2)
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "stream %zu: bad descriptor", i);
        in_off[i] = in.add(s[i].src_len);
        out_off[i] = out.add(s[i].dst_cap);
    }
    if (memspace == PNGB200_MEM_HOST) {
        CU(ctx->d_in.reserve(in.total));
        CU(ctx->d_out.reserve(out.total));
        for (size_t i = 0; i < count; ++i)
            if (s[i].src_len)
                CU(cudaMemcpyAsync(ctx->d_in.as<uint8_t>() + in_off[i], s[i].src, s[i].src_len,
                                   cudaMemcpyHostToDevice, ctx->stream));
    }
    for (size_t i = 0; i < count; ++i) {   // no scratch to borrow: streams are not cut in two
        bool host = memspace == PNGB200_MEM_HOST;
        jobs[i] = whole_stream_job(host ? ctx->d_in.as<uint8_t>() + in_off[i] : s[i].src, s[i].src_len,
                                   host ? ctx->d_out.as<uint8_t>() + out_off[i] : s[i].dst, s[i].dst_cap, s[i].format);
    }
    CU(cudaMemcpyAsync(ctx->d_jobs.p, jobs, sizeof(StreamJob) * count, cudaMemcpyHostToDevice, ctx->stream));
    int rc = run_inflate(ctx, jobs, count);
    if (rc != PNGB200_OK) return rc;
    CU(cudaMemcpyAsync(ctx->h_results.p, ctx->d_results.p, sizeof(StreamResult) * count,
                       cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    const StreamResult* r = ctx->h_results.as<StreamResult>();
    for (size_t i = 0; i < count; ++i) {
        s[i].status = r[i].status;
        s[i].err_a = r[i].err_a;
        s[i].err_b = r[i].err_b;
        s[i].checksum = r[i].checksum;
        s[i].blocks = r[i].blocks;
        s[i].produced = r[i].produced;
        s[i].consumed_bits = r[i].consumed_bits;
        if (memspace == PNGB200_MEM_HOST && r[i].produced)
            CU(cudaMemcpyAsync(s[i].dst, ctx->d_out.as<uint8_t>() + out_off[i], r[i].produced,
                               cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU(cudaStreamSynchronize(ctx->stream));
    return PNGB200_OK;
}

// ---------------- PNG decode: inflate + unfilter ----------------
int pngb200_decode_batch_enqueue(pngb200_ctx* ctx, pngb200_image_desc* im, size_t count, int memspace)
{
    if (!ctx || (!im && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is already pending");
    if (count == 0) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    const bool host = memspace == PNGB200_MEM_HOST;
    std::vector<Geometry> geo(count);
    std::vector<size_t>   f_off(count), in_off(count);
    ctx->expected.assign(count, 0);
    ctx->out_offset.assign(count, 0);
    ctx->out_bytes.assign(count, 0);
    Slots f{64}, in{16}, out{16};
    for (size_t i = 0; i < count; ++i) {
        if (!geometry(im[i].width, im[i].height, im[i].volume, im[i].depth, im[i].interlaced, &geo[i]) ||
            (!im[i].idat && im[i].idat_len) || !im[i].pixels || im[i].format > 1)
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "image %zu: bad descriptor", i);
        if (im[i].pixels_cap < geo[i].storage)
            return set_error(ctx, PNGB200_ERR_OUTPUT_CAPACITY, "image %zu: pixels_cap %zu < %llu", i,
                             im[i].pixels_cap, (unsigned long long)geo[i].storage);
        ctx->expected[i] = geo[i].filtered;
        f_off[i] = f.add(geo[i].filtered);
        in_off[i] = in.add(im[i].idat_len);
        ctx->out_offset[i] = out.add(geo[i].storage);
        ctx->out_bytes[i] = geo[i].storage;
    }
    CU(ctx->d_filtered.reserve(f.total));
    CU(ctx->h_jobs.reserve(sizeof(StreamJob) * count));
    CU(ctx->d_jobs.reserve(sizeof(StreamJob) * count));
    CU(ctx->d_results.reserve(sizeof(StreamResult) * count));
    CU(ctx->h_results.reserve(sizeof(StreamResult) * count));
    if (host) {
        CU(ctx->d_in.reserve(in.total));
        CU(ctx->d_out.reserve(out.total));
        ctx->bulk_h2d = [ctx, im, count, &in_off]() -> int {  // runs inside run_inflate below, after its tables
            for (size_t i = 0; i < count; ++i)
                if (im[i].idat_len)
                    CU(cudaMemcpyAsync(ctx->d_in.as<uint8_t>() + in_off[i], im[i].idat, im[i].idat_len,
                                       cudaMemcpyHostToDevice, ctx->stream));
            return PNGB200_OK;
        };
    }
    StreamJob* jobs = ctx->h_jobs.as<StreamJob>();
    for (size_t i = 0; i < count; ++i) {
        jobs[i] = whole_stream_job(host ? ctx->d_in.as<uint8_t>() + in_off[i] : im[i].idat, im[i].idat_len,
                                   ctx->d_filtered.as<uint8_t>() + f_off[i],
                                   geo[i].filtered + 16,   // room to notice extraneous image data
                                   im[i].format);
        // the pixel buffer is dead until unfilter writes it: a stream cut in two keeps its tail's symbols there
        // (host batches run lanes side by side and are not cut)
        if (!host) {
            jobs[i].scratch = im[i].pixels;
            jobs[i].scratch_cap = im[i].pixels_cap;
        }
    }
    CU(cudaMemcpyAsync(ctx->d_jobs.p, jobs, sizeof(StreamJob) * count, cudaMemcpyHostToDevice, ctx->stream));
    int rc = run_inflate(ctx, jobs, count);
    ctx->bulk_h2d = nullptr;  // captured this frame's locals
    if (rc != PNGB200_OK) return rc;
    std::vector<UnfilterItem> items(count);
    for (size_t i = 0; i < count; ++i) {
        UnfilterItem& it = items[i];
        it.filtered = jobs[i].dst;
        it.filtered_mut = jobs[i].dst;
        it.pixels = host ? ctx->d_out.as<uint8_t>() + ctx->out_offset[i] : im[i].pixels;
        it.inflated = ctx->d_results.as<StreamResult>() + i;
        it.filtered_len = 0;
        it.w = im[i].width;
        it.h = im[i].height;
        it.volume = im[i].volume;
        it.depth = im[i].depth;
        it.interlaced = im[i].interlaced;
        it.g = geo[i];
    }
    rc = run_unfilter(ctx, items);
    if (rc != PNGB200_OK) return rc;
    CU(cudaEventRecord(ctx->ev[3], ctx->stream));
    CU(cudaMemcpyAsync(ctx->h_results.p, ctx->d_results.p, sizeof(StreamResult) * count,
                       cudaMemcpyDeviceToHost, ctx->stream));
    if (host)
        for (size_t i = 0; i < count; ++i)
            CU(cudaMemcpyAsync(im[i].pixels, ctx->d_out.as<uint8_t>() + ctx->out_offset[i], ctx->out_bytes[i],
                               cudaMemcpyDeviceToHost, ctx->stream));
    ctx->pending = true;
    ctx->pending_memspace = memspace;
    return PNGB200_OK;
}

int pngb200_decode_batch_finish(pngb200_ctx* ctx, pngb200_image_desc* im, size_t count)
{
    if (!ctx || (!im && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (count == 0) return PNGB200_OK;
    if (!ctx->pending || ctx->expected.size() != count)
        return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "no matching pending decode batch");
    DeviceGuard guard(ctx->device);
    ctx->pending = false;
    CU(cudaStreamSynchronize(ctx->stream));
    const StreamResult* r = ctx->h_results.as<StreamResult>();
    for (size_t i = 0; i < count; ++i) {
        int st = r[i].status;
        // PNG.Decoder.push / PNG.Context.push(ancillary: IEND) error mapping
        if (st == PNGB200_ERR_OUTPUT_CAPACITY) st = PNGB200_ERR_PNG_EXTRANEOUS_IMAGE_DATA;
        else if (st == PNGB200_NEED_MORE_INPUT) st = PNGB200_ERR_PNG_INCOMPLETE_DATASTREAM;
        else if (st == PNGB200_OK && r[i].produced > ctx->expected[i]) st = PNGB200_ERR_PNG_EXTRANEOUS_IMAGE_DATA;
        im[i].status = st;
        im[i].err_a = r[i].err_a;
        im[i].err_b = r[i].err_b;
        im[i].checksum = r[i].checksum;
        im[i].blocks = r[i].blocks;
        im[i].produced = r[i].produced;
    }
    return PNGB200_OK;
}

int pngb200_decode_batch(pngb200_ctx* ctx, pngb200_image_desc* im, size_t count, int memspace)
{
    if (!ctx || (!im && count)) return PNGB200_ERR_BAD_ARGUMENT;
    return run_over_lanes(ctx, count, memspace,
                          [&](size_t i) { return im[i].idat_len + pngb200_storage_size(im[i].width, im[i].height, im[i].volume); },
                          [&](pngb200_ctx* lane, size_t lo, size_t n) {
                              int rc = pngb200_decode_batch_enqueue(lane, im + lo, n, memspace);
                              return rc != PNGB200_OK ? rc : pngb200_decode_batch_finish(lane, im + lo, n);
                          });
}

int pngb200_unfilter_batch(pngb200_ctx* ctx, pngb200_image_desc* im, size_t count, int memspace)
{
    if (!ctx || (!im && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    if (count == 0) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    start_unfilter_stats(ctx);
    const bool host = memspace == PNGB200_MEM_HOST;
    std::vector<UnfilterItem> items(count);
    std::vector<size_t>       f_off(count), o_off(count);
    Slots f{64}, o{16};
    for (size_t i = 0; i < count; ++i) {
        UnfilterItem& it = items[i];
        if (!geometry(im[i].width, im[i].height, im[i].volume, im[i].depth, im[i].interlaced, &it.g) ||
            !im[i].idat || !im[i].pixels)
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "image %zu: bad descriptor", i);
        if (im[i].pixels_cap < it.g.storage) return set_error(ctx, PNGB200_ERR_OUTPUT_CAPACITY, "image %zu: pixels_cap", i);
        // the generic kernel and the pass path reconstruct in place, so they always work on a private copy
        if (host || !it.g.fast) f_off[i] = f.add(im[i].idat_len);
        o_off[i] = o.add(it.g.storage);
    }
    CU(ctx->d_filtered.reserve(std::max<size_t>(f.total, 256)));
    if (host) CU(ctx->d_out.reserve(o.total));
    for (size_t i = 0; i < count; ++i) {
        UnfilterItem& it = items[i];
        uint8_t* priv = ctx->d_filtered.as<uint8_t>() + f_off[i];
        if (host || !it.g.fast) {
            CU(cudaMemcpyAsync(priv, im[i].idat, im[i].idat_len,
                               host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, ctx->stream));
            it.filtered = priv;
            it.filtered_mut = priv;
        } else {
            it.filtered = im[i].idat;
            it.filtered_mut = nullptr;
        }
        it.pixels = host ? ctx->d_out.as<uint8_t>() + o_off[i] : im[i].pixels;
        it.inflated = nullptr;
        it.filtered_len = im[i].idat_len;
        it.w = im[i].width;
        it.h = im[i].height;
        it.volume = im[i].volume;
        it.depth = im[i].depth;
        it.interlaced = im[i].interlaced;
    }
    int rc = run_unfilter(ctx, items);
    if (rc != PNGB200_OK) return rc;
    if (host)
        for (size_t i = 0; i < count; ++i)
            CU(cudaMemcpyAsync(im[i].pixels, ctx->d_out.as<uint8_t>() + o_off[i], items[i].g.storage,
                               cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < count; ++i) {
        uint64_t expect = items[i].g.filtered;
        im[i].produced = im[i].idat_len;
        im[i].status = im[i].idat_len > expect ? PNGB200_ERR_PNG_EXTRANEOUS_IMAGE_DATA : PNGB200_OK;
    }
    return PNGB200_OK;
}

// ---------------- encode stage 1: filter select + apply ----------------
int pngb200_filter_batch(pngb200_ctx* ctx, pngb200_filter_desc* im, size_t count, int memspace)
{
    if (!ctx || (!im && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    if (count == 0) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    const bool host = memspace == PNGB200_MEM_HOST;
    std::vector<FilterJob> jobs(count);
    std::vector<size_t>    p_off(count), f_off(count);
    Slots p{16}, f{16};
    uint64_t rows = 0;
    std::vector<uint32_t> row_base(count + 1);
    for (size_t i = 0; i < count; ++i) {
        Geometry g;
        if (!geometry(im[i].width, im[i].height, im[i].volume, im[i].depth, im[i].interlaced, &g) ||
            !im[i].pixels || !im[i].filtered)
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "image %zu: bad descriptor", i);
        if (im[i].pixels_len < g.storage || im[i].filtered_cap < g.filtered)
            return set_error(ctx, PNGB200_ERR_OUTPUT_CAPACITY, "image %zu: buffer too small", i);
        p_off[i] = p.add(g.storage);
        f_off[i] = f.add(g.filtered);
        im[i].produced = g.filtered;
        row_base[i] = (uint32_t)rows;
        rows += filter_rows(im[i].width, im[i].height, im[i].interlaced);
    }
    row_base[count] = (uint32_t)rows;
    if (rows >= (1ull << 31)) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "batch too large");
    if (host) {
        CU(ctx->d_in.reserve(p.total));
        CU(ctx->d_out.reserve(f.total));
        for (size_t i = 0; i < count; ++i)
            CU(cudaMemcpyAsync(ctx->d_in.as<uint8_t>() + p_off[i], im[i].pixels,
                               pngb200_storage_size(im[i].width, im[i].height, im[i].volume),
                               cudaMemcpyHostToDevice, ctx->stream));
    }
    for (size_t i = 0; i < count; ++i) {
        jobs[i].pixels = host ? ctx->d_in.as<uint8_t>() + p_off[i] : im[i].pixels;
        jobs[i].filtered = host ? ctx->d_out.as<uint8_t>() + f_off[i] : im[i].filtered;
        jobs[i].width = im[i].width;
        jobs[i].height = im[i].height;
        jobs[i].volume = im[i].volume;
        jobs[i].depth = im[i].depth;
        jobs[i].interlaced = im[i].interlaced;
        jobs[i].bpp = (uint8_t)((im[i].volume + 7) >> 3);
    }
    Tables t(ctx->h_genjobs, ctx->d_genjobs);
    const size_t off_jobs = t.host(jobs.data(), sizeof(FilterJob) * count);
    const size_t off_rb = t.host(row_base.data(), sizeof(uint32_t) * (count + 1));
    if (int rc = t.upload(ctx)) return rc;
    filter_rows_kernel<<<(unsigned)std::max<uint64_t>(1, (rows + FILTER_WARPS - 1) / FILTER_WARPS), FILTER_WARPS * 32, 0, ctx->stream>>>(
        t.dev<FilterJob>(off_jobs), t.dev<uint32_t>(off_rb), (uint32_t)count, (uint32_t)rows);
    ctx->launches++;
    CU(cudaGetLastError());
    if (host)
        for (size_t i = 0; i < count; ++i)
            CU(cudaMemcpyAsync(im[i].filtered, ctx->d_out.as<uint8_t>() + f_off[i], im[i].produced,
                               cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < count; ++i) im[i].status = PNGB200_OK;
    return PNGB200_OK;
}

}  // extern "C"

namespace {

// The call-level checks of the batch pushes: distinct handles of `ctx`, and data for every byte announced
template <typename Desc, typename Handle>
int check_pushes(pngb200_ctx* ctx, const Desc* pushes, size_t count, Handle* Desc::*handle, const char* what)
{
    if (!ctx || (!pushes && count)) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "%s: null argument", what);
    std::vector<const void*> seen(count);
    for (size_t i = 0; i < count; ++i) {
        const Handle* h = pushes[i].*handle;
        if (!h || h->ctx != ctx || (!pushes[i].data && pushes[i].n))
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "%s: item %zu has no handle of this context or no data", what, i);
        seen[i] = h;
    }
    std::sort(seen.begin(), seen.end());
    if (std::adjacent_find(seen.begin(), seen.end()) != seen.end())
        return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "%s: a handle appears twice", what);
    return PNGB200_OK;
}

}  // namespace

// ---------------- streaming LZ77.Deflator handle ----------------
// Two kinds: the buffered handle (pngb200_deflator_create) keeps the input on the host and compresses it in one
// pngb200_deflate_batch call at push(last: true); the online handle (pngb200_deflator_create_online) compresses on the
// device whenever the reference would, through deflate_resume_kernel, and keeps its state there between pushes.
struct pngb200_deflator {
    pngb200_ctx*         ctx = nullptr;
    int                  format = 0, level = 9, exponent = 15;
    size_t               chunk = 65544;
    std::vector<uint8_t> input, output;
    size_t               at = 0;       // next output byte to hand out
    bool                 finished = false;
    // online handles
    bool     online = false;
    int      status = PNGB200_OK;      // sticky: a failed launch leaves the device state unknown
    DevBuf   d_carry, d_dict, d_graph, d_up, d_in, d_out;
    uint64_t total = 0;                // bytes pushed
    uint64_t base = 0;                 // stream position of d_in's byte 0
    int64_t  end_index = -3, count = 0;   // the carry's window end (relative to base) and match-buffer fill
    uint64_t blocks = 0, written = 0;   // blocks and bytes written, the stream header included
    uint64_t held() const { return total - base; }   // bytes of d_in in use
    uint64_t dequeued() const { return std::min<uint64_t>(total, (uint64_t)std::max<int64_t>(0, (int64_t)base + end_index + 3)); }
    size_t   device_bytes() const { return d_carry.cap + d_dict.cap + d_graph.cap + d_up.cap + d_in.cap + d_out.cap; }
};

extern "C" {

pngb200_deflator* pngb200_deflator_create(pngb200_ctx* ctx, int format, int level, int exponent, size_t chunk_bytes)
{
    if (!ctx || format < 0 || format > 2 || level < 0 || level > 13 || exponent < 8 || exponent > 15) {
        set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "deflator_create: bad format / level / exponent");
        return nullptr;
    }
    pngb200_deflator* z = new pngb200_deflator();
    z->ctx = ctx;
    z->format = format;
    z->level = level;
    z->exponent = exponent;
    z->chunk = chunk_bytes ? chunk_bytes : 65544;
    return z;
}

pngb200_deflator* pngb200_deflator_create_online(pngb200_ctx* ctx, int format, int level, int exponent, size_t chunk_bytes)
{
    pngb200_deflator* z = pngb200_deflator_create(ctx, format, level, exponent, chunk_bytes);
    if (!z) return nullptr;
    z->online = true;
    DeviceGuard guard(ctx->device);
    DfCarry init;
    df_carry_init(init);
    if (z->d_carry.reserve(sizeof(DfCarry)) != cudaSuccess || z->d_dict.reserve(sizeof(int32_t) * DF_DICT_WORDS) != cudaSuccess ||
        cudaMemcpy(z->d_carry.p, &init, sizeof init, cudaMemcpyHostToDevice) != cudaSuccess) {
        set_error(ctx, PNGB200_ERR_CUDA, "deflator_create_online: cannot allocate the device state");
        delete z;
        return nullptr;
    }
    // DeflatorBuffers.init writes the stream header (DeflatorBuffers.swift:50-65, Gzip :100-112)
    const int e = format == PNGB200_FORMAT_IOS ? 15 : exponent;
    if (format == PNGB200_FORMAT_ZLIB) {
        const uint32_t unpaired = (uint32_t)(e - 8) << 4 | 8, check = ~(((unpaired << 8) | (unpaired >> 8)) % 31) & 31;
        z->output = {(uint8_t)unpaired, (uint8_t)check};
    } else if (format == PNGB200_FORMAT_GZIP) {
        z->output = {0x1f, 0x8b, 0x08, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0xff};
    }
    z->written = z->output.size();
    return z;
}

void pngb200_deflator_destroy(pngb200_deflator* z)
{
    if (!z) return;
    if (z->online) {
        DeviceGuard guard(z->ctx->device);
        cudaStreamSynchronize(z->ctx->stream);
    }
    delete z;   // frees the device state
}

}  // extern "C"

namespace {

// The deflate side of a push call over online deflators, shared by pngb200_deflator_push_batch and
// pngb200_png_encoder_push_batch.  What a handle needs for a push of n bytes: input from the base on; when it
// compresses, a graph for every vertex the push can add to the unfinished block (full mode) and room for every byte
// the launch can write.
struct DfNeed { bool run; size_t in, graph, up, out; };
constexpr uint64_t kMaxDeflatorPush = 1ull << 30;   // keeps every position of a launch inside int32

DfNeed df_need(const pngb200_deflator* z, uint64_t n_new, bool last)
{
    const uint64_t total = z->total + n_new, n = total - z->base;
    const uint64_t pending = total - z->dequeued();
    DfNeed w;
    w.run = pending > 4096 || last;   // DeflatorBuffers.swift:74, :120
    w.in = n + 16;
    w.graph = w.up = w.out = 0;
    if (w.run) {
        const bool full = z->level >= 8;
        const uint64_t span = (uint64_t)((int64_t)n - z->end_index);
        const uint64_t verts = std::min<uint64_t>(DF_GRAPH_CAP, (uint64_t)z->count + span) + 2;
        if (full) w.graph = 128 * verts, w.up = 4 * (verts + 1);
        w.out = pngb200_deflate_bound((full ? 1 : 8) * (uint64_t)z->count + span) + 4096;
    }
    return w;
}

// the buffers of `z` that `call` grows for `w`
void df_grow(PushCall& call, pngb200_deflator* z, const DfNeed& w)
{
    if (w.in > z->d_in.cap) call.add(z->d_in, w.in, z->held());
    if (w.graph > z->d_graph.cap) call.add(z->d_graph, w.graph, 128 * (size_t)z->count);
    if (w.up > z->d_up.cap) call.add(z->d_up, w.up, 0);
    if (w.out > z->d_out.cap) call.add(z->d_out, w.out, 0);
}

// the job of a handle that compresses, its new input counted in; its bytes and result land in pinned `host_dst` / `res`
DfResumeJob df_job(pngb200_deflator* z, const DfNeed& w, bool last, uint8_t* host_dst, DfResumeResult* res)
{
    DfResumeJob j;
    j.carry = z->d_carry.as<DfCarry>();
    j.in = z->d_in.as<uint8_t>();
    j.n = z->total - z->base;
    j.dict = z->d_dict.as<int32_t>();
    j.graph = z->d_graph.as<uint32_t>();
    j.up = z->d_up.as<uint32_t>();
    j.graph_vertices = z->d_graph.cap / 128;
    j.dst = z->d_out.as<uint8_t>();
    j.cap = w.out;
    j.host_dst = host_dst;   // pinned: the kernel writes it over the bus (unified addressing)
    j.result = res;
    j.format = z->format;
    j.level = z->level;
    j.exponent = z->exponent;
    j.last = last ? 1 : 0;
    return j;
}

// one deflate_resume_kernel launch over `count` jobs already uploaded, then the synchronise
cudaError_t df_launch(pngb200_ctx* ctx, const DfResumeJob* d_jobs, size_t count, const DfEnds* d_ends)
{
    deflate_resume_kernel<<<(unsigned)count, 32, sizeof(DfShared), ctx->stream>>>(d_jobs, (int)count, d_ends);
    ctx->launches++;
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    return e;
}

// takes a launched job's result into its handle (`e`: the launch's CUDA error); returns the item's status
int df_take(pngb200_ctx* ctx, pngb200_deflator* z, const DfResumeJob& j, cudaError_t e)
{
    if (e != cudaSuccess)
        return z->status = set_error(ctx, PNGB200_ERR_CUDA, "deflate_resume_kernel: %s", cudaGetErrorString(e));
    const DfResumeResult& r = *j.result;
    if (r.status != PNGB200_OK) return z->status = set_error(ctx, r.status, "deflate_resume_kernel: status %d", r.status);
    z->output.insert(z->output.end(), j.host_dst, j.host_dst + r.produced);
    z->blocks += r.blocks;
    z->written += r.produced;
    z->base = r.base;
    z->end_index = r.end_index;
    z->count = r.count;
    if (j.last) z->finished = true;
    return PNGB200_OK;
}

// what the reference's pop() handed out is gone from the queue
void df_drop_popped(pngb200_deflator* z)
{
    z->output.erase(z->output.begin(), z->output.begin() + (ptrdiff_t)z->at);
    z->at = 0;
}

// The pushes of one pngb200_deflator_push_batch call, on distinct online handles of `ctx`.  Every buffer the call
// needs is allocated before any device work, so that an allocation failure leaves every handle as it was.
int deflator_pushes(pngb200_ctx* ctx, pngb200_deflator_push_desc* pushes, size_t count)
{
    std::vector<pngb200_deflator_push_desc*> live;
    size_t staged = 0;
    for (size_t i = 0; i < count; ++i) {
        pngb200_deflator_push_desc* d = &pushes[i];
        pngb200_deflator* z = d->deflator;
        if (z->status < 0) d->status = z->status;
        else if (z->finished) d->status = set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "deflator: push after push(last: true)");
        else if (d->n > kMaxDeflatorPush) d->status = set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "deflator: a push is at most 1 GiB");
        else d->status = PNGB200_ERR_CUDA, live.push_back(d), staged += d->n;   // until its push is answered
    }
    std::vector<DfNeed> need(live.size());
    size_t run = 0, host_out = 0;
    for (size_t k = 0; k < live.size(); ++k) {
        need[k] = df_need(live[k]->deflator, live[k]->n, live[k]->last != 0);
        if (need[k].run) host_out += align_up(need[k].out, 256), run++;
    }
    // every allocation, before any device work
    PushCall call(ctx);
    const size_t jobs_bytes = sizeof(DfResumeJob) * std::max<size_t>(run, 1);
    const size_t res_off = align_up(host_out, 256);
    CU(ctx->h_dfout.reserve(res_off + sizeof(DfResumeResult) * std::max<size_t>(run, 1)));
    CU(ctx->h_st.reserve(jobs_bytes));
    CU(ctx->d_st.reserve(jobs_bytes));
    for (size_t k = 0; k < live.size(); ++k) df_grow(call, live[k]->deflator, need[k]);
    if (int rc = call.grow(staged)) return rc;
    // the new input of every handle with one upload, appended to its input
    if (int rc = call.stage(live, &pngb200_deflator_push_desc::deflator,
                            [](pngb200_deflator_push_desc* d) { d->deflator->total += d->n; }))
        return rc;
    std::vector<DfResumeJob> jobs;
    std::vector<size_t>      which;
    size_t out_at = 0;
    for (size_t k = 0; k < live.size(); ++k) {
        pngb200_deflator_push_desc* d = live[k];
        pngb200_deflator* z = d->deflator;
        df_drop_popped(z);
        if (!need[k].run) {
            d->status = PNGB200_OK;
            continue;
        }
        jobs.push_back(df_job(z, need[k], d->last != 0, ctx->h_dfout.as<uint8_t>() + out_at,
                              (DfResumeResult*)(ctx->h_dfout.as<uint8_t>() + res_off) + jobs.size()));
        out_at += align_up(need[k].out, 256);
        which.push_back(k);
    }
    if (!jobs.empty()) {
        memcpy(ctx->h_st.p, jobs.data(), sizeof(DfResumeJob) * jobs.size());
        cudaError_t e = cudaMemcpyAsync(ctx->d_st.p, ctx->h_st.p, sizeof(DfResumeJob) * jobs.size(), cudaMemcpyHostToDevice,
                                        ctx->stream);
        if (e == cudaSuccess) e = df_launch(ctx, ctx->d_st.as<DfResumeJob>(), jobs.size(), nullptr);
        for (size_t t = 0; t < jobs.size(); ++t) live[which[t]]->status = df_take(ctx, live[which[t]]->deflator, jobs[t], e);
        if (e != cudaSuccess) return PNGB200_ERR_CUDA;
    } else if (staged) {
        if (cudaStreamSynchronize(ctx->stream) != cudaSuccess)
            return set_error(ctx, PNGB200_ERR_CUDA, "deflator_push_batch: synchronise failed");
    }
    return call.done();
}

}  // namespace

extern "C" {

int pngb200_deflator_push_batch(pngb200_ctx* ctx, pngb200_deflator_push_desc* pushes, size_t count)
{
    if (int rc = check_pushes(ctx, pushes, count, &pngb200_deflator_push_desc::deflator, "deflator_push_batch")) return rc;
    for (size_t i = 0; i < count; ++i)
        if (!pushes[i].deflator->online)
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "deflator_push_batch: item %zu is a buffered deflator", i);
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    if (!count) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    return deflator_pushes(ctx, pushes, count);
}

int pngb200_deflator_push(pngb200_deflator* z, const uint8_t* data, size_t n, int last)
{
    if (!z || (!data && n)) return PNGB200_ERR_BAD_ARGUMENT;
    if (z->online) {
        pngb200_deflator_push_desc d{z, data, n, last, 0};
        if (int rc = pngb200_deflator_push_batch(z->ctx, &d, 1)) return rc;
        return d.status;
    }
    if (z->finished) return set_error(z->ctx, PNGB200_ERR_BAD_ARGUMENT, "deflator: push after push(last: true)");
    z->input.insert(z->input.end(), data, data + n);
    if (!last) return PNGB200_OK;
    z->output.resize(pngb200_deflate_bound(z->input.size()));
    pngb200_deflate_desc d;
    memset(&d, 0, sizeof d);
    d.src = z->input.data();
    d.src_len = z->input.size();
    d.dst = z->output.data();
    d.dst_cap = z->output.size();
    d.format = z->format;
    d.level = z->level;
    d.exponent = z->exponent;
    int rc = pngb200_deflate_batch(z->ctx, &d, 1, PNGB200_MEM_HOST);
    if (rc != PNGB200_OK) return rc;
    if (d.status != PNGB200_OK) return d.status;
    z->output.resize((size_t)d.produced);
    z->finished = true;
    std::vector<uint8_t>().swap(z->input);
    return PNGB200_OK;
}

int pngb200_deflator_pop(pngb200_deflator* z, const uint8_t** block, size_t* n)
{
    if (!z || !block || !n) return PNGB200_ERR_BAD_ARGUMENT;
    // DeflatorOut queues a block the moment its buffer is full (LZ77.DeflatorOut.swift:109-135): complete blocks only.
    // The buffered handle has none before push(last: true).
    if ((!z->online && !z->finished) || z->output.size() - z->at < z->chunk) return 0;
    *block = z->output.data() + z->at;
    *n = z->chunk;
    z->at += z->chunk;
    return 1;
}

int pngb200_deflator_pull(pngb200_deflator* z, const uint8_t** block, size_t* n)
{
    if (!z || !block || !n) return PNGB200_ERR_BAD_ARGUMENT;
    if (int got = pngb200_deflator_pop(z, block, n)) return got;
    if (!z->finished || z->at >= z->output.size()) return 0;   // pull(): flushed.isEmpty ? nil : flushed
    *block = z->output.data() + z->at;
    *n = z->output.size() - z->at;
    z->at = z->output.size();
    return 1;
}

int pngb200_deflator_stats(const pngb200_deflator* z, uint64_t out[4])
{
    if (!z || !out || !z->online) return PNGB200_ERR_BAD_ARGUMENT;
    out[0] = z->dequeued();
    out[1] = z->written;
    out[2] = z->blocks;
    out[3] = z->device_bytes();
    return PNGB200_OK;
}

}  // extern "C"

// ---------------- colour targets: unpack / pack ----------------
namespace {
int run_color(pngb200_ctx* ctx, pngb200_color_desc* im, size_t count, int target, int alpha_mode, int memspace, bool unpack)
{
    if (!ctx || (!im && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    if (target < PNGB200_TARGET_RGBA8 || target > PNGB200_TARGET_V64 || alpha_mode < PNGB200_ALPHA_ASIS ||
        alpha_mode > PNGB200_ALPHA_STRAIGHTENED_AS32)
        return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "bad colour target / alpha mode");
    // per target: component bits and bytes per pixel
    static const int    kTargetBits[]  = {8, 16, 8, 16, 32, 64, 32, 64, 8, 16, 32, 64};
    static const size_t kTargetBytes[] = {4, 8, 2, 4, 16, 32, 8, 16, 1, 2, 4, 8};
    if (target >= PNGB200_TARGET_V8 && alpha_mode != PNGB200_ALPHA_ASIS)
        return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a scalar target has no alpha to premultiply or straighten");
    if (alpha_mode >= PNGB200_ALPHA_PREMULTIPLIED_AS8) {
        const int u = alpha_mode <= PNGB200_ALPHA_STRAIGHTENED_AS8 ? 8 : alpha_mode <= PNGB200_ALPHA_STRAIGHTENED_AS16 ? 16 : 32;
        if (kTargetBits[target] <= u)
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "premultiplied(as: UInt%d) needs a target wider than %d bits", u, u);
    }
    if (count == 0) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    const bool   host = memspace == PNGB200_MEM_HOST;
    const size_t tpx  = kTargetBytes[target];
    std::vector<ColorJob> jobs(count);
    std::vector<size_t>   s_off(count), p_off(count), s_len(count);
    std::vector<uint32_t> palettes;
    Slots st{16}, px{16};
    uint64_t most = 0;
    for (size_t i = 0; i < count; ++i) {
        const pngb200_pixel_format& f = im[i].format;
        const PixelRule rule = pixel_rule(f.color, f.depth, f.bgr);
        if (!rule.valid || (f.color == 3 && (!f.palette || f.palette_count == 0 || f.palette_count > 256)) ||
            (im[i].count && (!im[i].storage || !im[i].pixels)))
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "image %zu: bad colour descriptor", i);
        s_len[i] = (size_t)im[i].count * rule.channels * (f.depth == 16 ? 2 : 1);
        if (im[i].storage_len < s_len[i] || im[i].pixels_len < im[i].count * tpx)
            return set_error(ctx, PNGB200_ERR_OUTPUT_CAPACITY, "image %zu: buffer too small", i);
        if (!host && (((uintptr_t)im[i].pixels) & (std::min<size_t>(tpx, 16) - 1)))
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "image %zu: pixel array is not aligned to its element size", i);
        s_off[i] = st.add(s_len[i]);
        p_off[i] = px.add(im[i].count * tpx);
        ColorJob& j = jobs[i];
        j.count = im[i].count;
        j.color = f.color, j.depth = f.depth, j.bgr = f.bgr, j.has_key = f.has_key;
        j.key[0] = f.key[0], j.key[1] = f.key[1], j.key[2] = f.key[2];
        j.palette_off = (uint32_t)palettes.size();
        j.palette_count = f.color == 3 ? f.palette_count : 0;
        for (uint32_t k = 0; k < j.palette_count; ++k)
            palettes.push_back(f.palette[4 * k] | f.palette[4 * k + 1] << 8 | f.palette[4 * k + 2] << 16 | (uint32_t)f.palette[4 * k + 3] << 24);
        j.status = PNGB200_OK;
        most = std::max<uint64_t>(most, im[i].count);
    }
    if (host) {
        CU(ctx->d_in.reserve(unpack ? st.total : px.total));
        CU(ctx->d_out.reserve(unpack ? px.total : st.total));
        for (size_t i = 0; i < count; ++i) {
            const size_t n = unpack ? s_len[i] : im[i].count * tpx;
            if (n)
                CU(cudaMemcpyAsync(ctx->d_in.as<uint8_t>() + (unpack ? s_off[i] : p_off[i]), unpack ? im[i].storage : im[i].pixels,
                                   n, cudaMemcpyHostToDevice, ctx->stream));
        }
    }
    for (size_t i = 0; i < count; ++i) {
        uint8_t* dev_s = host ? (unpack ? ctx->d_in : ctx->d_out).as<uint8_t>() + s_off[i] : (uint8_t*)im[i].storage;
        uint8_t* dev_p = host ? (unpack ? ctx->d_out : ctx->d_in).as<uint8_t>() + p_off[i] : (uint8_t*)im[i].pixels;
        jobs[i].storage = dev_s, jobs[i].pixels = dev_p;
    }
    Tables t(ctx->h_genjobs, ctx->d_genjobs);
    const size_t jb = sizeof(ColorJob) * count, off_jobs = t.host(jobs.data(), jb);
    const size_t off_pal = t.host(palettes.empty() ? nullptr : palettes.data(), sizeof(uint32_t) * std::max<size_t>(palettes.size(), 1));
    if (int rc = t.upload(ctx)) return rc;
    ColorParams p;
    p.jobs = t.dev<ColorJob>(off_jobs);
    p.palettes = t.dev<uint32_t>(off_pal);
    p.count = (uint32_t)count;
    p.target = target;
    p.alpha_mode = alpha_mode;
    // x: tiles of the largest image, capped so that x * y stays near 8 CTAs per SM; y: images
    const unsigned gy = (unsigned)std::min<size_t>(count, 65535);
    const uint64_t tiles = std::max<uint64_t>(1, (most + COLOR_TILE - 1) / COLOR_TILE);
    const unsigned gx = (unsigned)std::min<uint64_t>(tiles, std::max<uint64_t>(1, (uint64_t)ctx->sm_count * 8 / gy));
    // the four 8/16-bit targets share one kernel per direction; each wider or scalar target has its own
    using ColorKernel = void (*)(ColorParams);
    static const ColorKernel kUnpack[] = {
        unpack_kernel, unpack_kernel, unpack_kernel, unpack_kernel,
        unpack_wide_kernel<32, COLOR_RGBA>, unpack_wide_kernel<64, COLOR_RGBA>,
        unpack_wide_kernel<32, COLOR_VA>, unpack_wide_kernel<64, COLOR_VA>,
        unpack_wide_kernel<8, COLOR_V>, unpack_wide_kernel<16, COLOR_V>,
        unpack_wide_kernel<32, COLOR_V>, unpack_wide_kernel<64, COLOR_V>};
    static const ColorKernel kPack[] = {
        pack_kernel, pack_kernel, pack_kernel, pack_kernel,
        pack_wide_kernel<32, COLOR_RGBA>, pack_wide_kernel<64, COLOR_RGBA>,
        pack_wide_kernel<32, COLOR_VA>, pack_wide_kernel<64, COLOR_VA>,
        pack_wide_kernel<8, COLOR_V>, pack_wide_kernel<16, COLOR_V>,
        pack_wide_kernel<32, COLOR_V>, pack_wide_kernel<64, COLOR_V>};
    (unpack ? kUnpack : kPack)[target]<<<dim3(gx, gy), COLOR_THREADS, 0, ctx->stream>>>(p);
    ctx->launches++;
    CU(cudaGetLastError());
    if (host)
        for (size_t i = 0; i < count; ++i) {
            const size_t n = unpack ? im[i].count * tpx : s_len[i];
            if (n)
                CU(cudaMemcpyAsync(unpack ? im[i].pixels : im[i].storage, ctx->d_out.as<uint8_t>() + (unpack ? p_off[i] : s_off[i]), n,
                                   cudaMemcpyDeviceToHost, ctx->stream));
        }
    ColorJob* done = t.pin<ColorJob>(off_jobs);   // the jobs come back with their statuses
    CU(cudaMemcpyAsync(done, t.dev<ColorJob>(off_jobs), jb, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < count; ++i) im[i].status = done[i].status;
    return PNGB200_OK;
}
}  // namespace

extern "C" {
int pngb200_unpack_batch(pngb200_ctx* ctx, pngb200_color_desc* im, size_t count, int target, int alpha_mode, int memspace)
{
    return run_color(ctx, im, count, target, alpha_mode, memspace, true);
}
int pngb200_pack_batch(pngb200_ctx* ctx, pngb200_color_desc* im, size_t count, int target, int memspace)
{
    return run_color(ctx, im, count, target, PNGB200_ALPHA_ASIS, memspace, false);
}
}  // extern "C"

// ---------------- encode stage 2: deflate ----------------
namespace {
// device-resident jobs -> compressed streams (results stay in d_dfres / are copied to `hres`)
int run_deflate(pngb200_ctx* ctx, const std::vector<DeflateJob>& jobs, DeflateResult* hres)
{
    size_t count = jobs.size();
    uint64_t verts = 2;
    for (const DeflateJob& j : jobs)
        if (j.level >= 8) verts = std::max<uint64_t>(verts, std::min<uint64_t>(j.n, DF_GRAPH_CAP) + 2);
    uint64_t stride = df_scratch_stride(verts);
    const uint64_t budget = ctx->device_bytes / 4;   // leaves the rest of the device to the caller's images
    size_t slots = std::min<size_t>({count, (size_t)std::max<uint64_t>(1, budget / stride), (size_t)ctx->sm_count * 8});
    CU(ctx->d_dfscratch.reserve(stride * slots + 256));
    CU(ctx->d_dfjobs.reserve(sizeof(DeflateJob) * count));
    CU(ctx->d_dfres.reserve(sizeof(DeflateResult) * count));
    CU(cudaMemcpyAsync(ctx->d_dfjobs.p, jobs.data(), sizeof(DeflateJob) * count, cudaMemcpyHostToDevice, ctx->stream));
    CU(cudaMemsetAsync(ctx->d_dfres.p, 0, sizeof(DeflateResult) * count, ctx->stream));
    DfParams P;
    P.jobs = ctx->d_dfjobs.as<DeflateJob>();
    P.results = ctx->d_dfres.as<DeflateResult>();
    P.scratch = ctx->d_dfscratch.as<uint8_t>();
    P.scratch_stride = stride;
    P.graph_vertices = verts;
    P.ticket = (uint32_t*)(ctx->d_dfscratch.as<uint8_t>() + stride * slots);
    P.count = (int)count;
    CU(cudaMemsetAsync(P.ticket, 0, sizeof(uint32_t), ctx->stream));
    deflate_kernel<<<(unsigned)slots, 32, sizeof(DfShared), ctx->stream>>>(P);
    ctx->launches++;
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(hres, ctx->d_dfres.p, sizeof(DeflateResult) * count, cudaMemcpyDeviceToHost, ctx->stream));
    CU(cudaStreamSynchronize(ctx->stream));
    return PNGB200_OK;
}
}  // namespace

extern "C" size_t pngb200_deflate_bound(size_t n) { return n + n / 2 + 4096; }

extern "C" int pngb200_deflate_batch(pngb200_ctx* ctx, pngb200_deflate_desc* s, size_t count, int memspace)
{
    if (!ctx || (!s && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    if (count == 0) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    const bool host = memspace == PNGB200_MEM_HOST;
    std::vector<DeflateJob> jobs(count);
    std::vector<size_t> in_off(count), out_off(count);
    Slots in{16}, out{16};
    for (size_t i = 0; i < count; ++i) {
        if ((!s[i].src && s[i].src_len) || !s[i].dst || s[i].format < 0 || s[i].format > 2 || s[i].exponent < 8 ||
            s[i].exponent > 15)
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "stream %zu: bad descriptor", i);
        in_off[i] = in.add(s[i].src_len);
        out_off[i] = out.add(s[i].dst_cap);
    }
    if (host) {
        CU(ctx->d_in.reserve(in.total));
        CU(ctx->d_out.reserve(out.total));
        for (size_t i = 0; i < count; ++i)
            if (s[i].src_len)
                CU(cudaMemcpyAsync(ctx->d_in.as<uint8_t>() + in_off[i], s[i].src, s[i].src_len,
                                   cudaMemcpyHostToDevice, ctx->stream));
    }
    for (size_t i = 0; i < count; ++i) {
        jobs[i].src = host ? ctx->d_in.as<uint8_t>() + in_off[i] : s[i].src;
        jobs[i].n = s[i].src_len;
        jobs[i].dst = host ? ctx->d_out.as<uint8_t>() + out_off[i] : s[i].dst;
        jobs[i].cap = s[i].dst_cap;
        jobs[i].format = s[i].format;
        jobs[i].level = s[i].level;
        jobs[i].exponent = s[i].exponent;
        jobs[i].pad = 0;
    }
    std::vector<DeflateResult> res(count);
    int rc = run_deflate(ctx, jobs, res.data());
    if (rc != PNGB200_OK) return rc;
    for (size_t i = 0; i < count; ++i) {
        s[i].status = res[i].status;
        s[i].checksum = res[i].checksum;
        s[i].blocks = res[i].blocks;
        s[i].produced = res[i].produced;
        if (host && res[i].status == PNGB200_OK && res[i].produced)
            CU(cudaMemcpyAsync(s[i].dst, ctx->d_out.as<uint8_t>() + out_off[i], res[i].produced,
                               cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU(cudaStreamSynchronize(ctx->stream));
    return PNGB200_OK;
}

extern "C" int pngb200_encode_batch(pngb200_ctx* ctx, pngb200_encode_desc* im, size_t count, int memspace)
{
    if (!ctx || (!im && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "a decode batch is pending");
    if (count == 0) return PNGB200_OK;
    for (size_t i = 0; i < count; ++i)
        if (!im[i].pixels || !im[i].idat)
            return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "image %zu: bad descriptor", i);
    DeviceGuard guard(ctx->device);
    const bool host = memspace == PNGB200_MEM_HOST;
    // stage 1: filter into a private device workspace (device memspace of the filter entry point)
    std::vector<pngb200_filter_desc> fd(count);
    std::vector<size_t> f_off(count), p_off(count), o_off(count);
    Slots f{16}, p{16}, o{16};
    for (size_t i = 0; i < count; ++i) {
        f_off[i] = f.add(pngb200_filtered_size(im[i].width, im[i].height, im[i].volume, im[i].interlaced));
        p_off[i] = p.add(im[i].pixels_len);
        o_off[i] = o.add(im[i].idat_cap);
    }
    CU(ctx->d_enc.reserve(f.total + (host ? p.total + o.total : 0) + 256));
    uint8_t* d_f = ctx->d_enc.as<uint8_t>();
    uint8_t* d_p = d_f + f.total;
    uint8_t* d_o = d_p + (host ? p.total : 0);
    for (size_t i = 0; i < count; ++i) {
        if (host) CU(cudaMemcpyAsync(d_p + p_off[i], im[i].pixels, im[i].pixels_len, cudaMemcpyHostToDevice, ctx->stream));
        fd[i].pixels = host ? d_p + p_off[i] : im[i].pixels;
        fd[i].pixels_len = im[i].pixels_len;
        fd[i].filtered = d_f + f_off[i];
        fd[i].filtered_cap = pngb200_filtered_size(im[i].width, im[i].height, im[i].volume, im[i].interlaced);
        fd[i].width = im[i].width;
        fd[i].height = im[i].height;
        fd[i].volume = im[i].volume;
        fd[i].depth = im[i].depth;
        fd[i].interlaced = im[i].interlaced;
    }
    int rc = pngb200_filter_batch(ctx, fd.data(), count, PNGB200_MEM_DEVICE);
    if (rc != PNGB200_OK) return rc;
    std::vector<DeflateJob> jobs(count);
    for (size_t i = 0; i < count; ++i) {
        jobs[i].src = fd[i].filtered;
        jobs[i].n = fd[i].filtered_cap;
        jobs[i].dst = host ? d_o + o_off[i] : im[i].idat;
        jobs[i].cap = im[i].idat_cap;
        jobs[i].format = im[i].format;
        jobs[i].level = im[i].level;
        jobs[i].exponent = 15;
        jobs[i].pad = 0;
    }
    std::vector<DeflateResult> res(count);
    rc = run_deflate(ctx, jobs, res.data());
    if (rc != PNGB200_OK) return rc;
    for (size_t i = 0; i < count; ++i) {
        im[i].status = res[i].status;
        im[i].checksum = res[i].checksum;
        im[i].blocks = res[i].blocks;
        im[i].produced = res[i].produced;
        if (host && res[i].status == PNGB200_OK)
            CU(cudaMemcpyAsync(im[i].idat, d_o + o_off[i], res[i].produced, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU(cudaStreamSynchronize(ctx->stream));
    return PNGB200_OK;
}

extern "C" {
// ---------------- streaming inflator handle ----------------
struct pngb200_inflator {
    pngb200_ctx*         ctx;
    int                  format;
    DevBuf               d_in, d_out;     // every byte pushed; the output
    uint64_t             pushed = 0, tail_at = 0;
    std::vector<uint8_t> tail;            // the input from byte tail_at <= resume_bit >> 3 on (stored_in_flight)
    uint64_t             resume_bit = 0, resume_out = 0, produced = 0, current = 0;
    uint32_t             phase = 0;
    ResumePoint          at{};            // the block a phase-3 resume point lies in (uploaded with every launch)
    uint64_t             work[3] = {};    // pngb200_inflator_stats
    bool                 terminal = false;
    int                  status = PNGB200_NEED_MORE_INPUT;
    uint32_t             err_a = 0, err_b = 0;
    uint64_t             held() const { return pushed; }   // bytes of d_in in use
};

pngb200_inflator* pngb200_inflator_create(pngb200_ctx* ctx, int format)
{
    if (!ctx || format < 0 || format > 2) return nullptr;
    pngb200_inflator* z = new pngb200_inflator();
    z->ctx = ctx;
    z->format = format;
    return z;
}

void pngb200_inflator_destroy(pngb200_inflator* z)
{
    if (!z) return;
    DeviceGuard guard(z->ctx->device);
    cudaStreamSynchronize(z->ctx->stream);
    delete z;   // frees the workspaces
}

}  // extern "C"

namespace {

// The pushes of one pngb200_inflator_push_batch call, on distinct handles of `ctx`.  Every item's `status` is
// PNGB200_ERR_CUDA until its push is answered, so that a CUDA failure leaves the items it stopped as a single push that
// failed the same way.
int inflate_pushes(pngb200_ctx* ctx, pngb200_inflator_push_desc* pushes, size_t count)
{
    std::vector<pngb200_inflator_push_desc*> live;
    size_t staged = 0;
    for (size_t i = 0; i < count; ++i) {
        pngb200_inflator_push_desc* d = &pushes[i];
        pngb200_inflator* z = d->inflator;
        if (z->terminal) d->status = PNGB200_OK;   // LZ77.Inflator ignores input after the terminal state
        else if (z->status < 0) d->status = z->status;
        else {
            d->status = PNGB200_ERR_CUDA;
            live.push_back(d);
            staged += d->n;
        }
    }
    if (live.empty()) return PNGB200_OK;
    PushCall call(ctx);
    for (pngb200_inflator_push_desc* d : live) {
        pngb200_inflator* z = d->inflator;
        const uint64_t pushed = z->pushed + d->n;
        if (pushed + 16 > z->d_in.cap)   // 16 bytes of slack behind the input for the decoders' bit reader
            call.add(z->d_in, pushed * 2 + 4096, z->pushed);
        const size_t want = std::max<size_t>(1 << 16, z->produced + 4 * d->n + 1024);
        if (want > z->d_out.cap) call.add(z->d_out, std::max(want, z->d_out.cap * 2), z->produced);
    }
    if (int rc = call.grow(staged)) return rc;
    // the host keeps the input from the resume point's byte on, which is all stored_in_flight reads
    if (int rc = call.stage(live, &pngb200_inflator_push_desc::inflator, [](pngb200_inflator_push_desc* d) {
            pngb200_inflator* z = d->inflator;
            const uint64_t decoded = std::min<uint64_t>((z->resume_bit >> 3) - z->tail_at, z->tail.size());
            z->tail.erase(z->tail.begin(), z->tail.begin() + (ptrdiff_t)decoded);
            z->tail_at += decoded;
            z->tail.insert(z->tail.end(), d->data, d->data + d->n);
            z->pushed += d->n;
        }))
        return rc;
    // Rounds: every live handle decodes once; a handle whose output ran out grows it and goes again in the next round.
    constexpr uint64_t kWave = 64u << 10;
    std::vector<pngb200_inflator_push_desc*> round = live;
    while (!round.empty()) {
        // A push with a lot of undecoded input goes through the intra-stream parallel kernel (one CTA: ~25 x the
        // lock-step warp); short ones, and what is left of the wave the input ends in, through the serial decoder.
        // Both resume where the last push stopped: at a block header, or at the last complete symbol of a Huffman block.
        auto pending = [](const pngb200_inflator* z) { return z->pushed - std::min<uint64_t>(z->pushed, z->resume_bit >> 3); };
        std::stable_partition(round.begin(), round.end(),
                              [&](const pngb200_inflator_push_desc* d) { return pending(d->inflator) >= kWave; });
        const size_t m = round.size();
        size_t big = 0;
        uint64_t max_cap = 0;
        std::vector<StreamJob>    jobs(m);
        std::vector<StreamResult> res(m);
        std::vector<ResumePoint>  at(m);
        for (size_t k = 0; k < m; ++k) {
            pngb200_inflator* z = round[k]->inflator;
            jobs[k] = whole_stream_job(z->d_in.as<uint8_t>(), z->pushed, z->d_out.as<uint8_t>(), z->d_out.cap, z->format);
            jobs[k].start_bit = z->resume_bit;
            jobs[k].start_out = z->resume_out;
            jobs[k].phase = (int32_t)z->phase;
            memset(&res[k], 0, sizeof res[k]);
            at[k] = z->at;
            at[k].bits = at[k].bytes = at[k].serial_bytes = 0;
            if (pending(z) >= kWave) big++, max_cap = std::max<uint64_t>(max_cap, z->d_out.cap);
        }
        Tables t(ctx->h_st, ctx->d_st);
        const size_t off_jobs = t.host(jobs.data(), sizeof(StreamJob) * m);
        const size_t off_res  = t.host(res.data(), sizeof(StreamResult) * m);
        const size_t off_at   = t.host(at.data(), sizeof(ResumePoint) * m);
        CU(ctx->d_st.reserve(t.end));   // now, so that the jobs can point at their resume records
        for (size_t k = 0; k < m; ++k) jobs[k].resume = t.dev<ResumePoint>(off_at) + k;
        if (int rc = t.upload(ctx)) return rc;
        StreamJob*    d_jobs = t.dev<StreamJob>(off_jobs);
        StreamResult* d_res  = t.dev<StreamResult>(off_res);
        if (big) {
            const unsigned grid = (unsigned)std::min<size_t>(big, 2 * (size_t)ctx->sm_count);
            if (int rc = launch_waves(ctx, ENG_WAVE, d_jobs, d_res, nullptr, big, grid, max_cap, nullptr)) return rc;
        }
        if (m > big) {
            inflate_serial_kernel<<<(unsigned)(m - big), 32, 0, ctx->stream>>>(d_jobs + big, d_res + big, nullptr, (int)(m - big));
            ctx->launches++;
        }
        CU(cudaGetLastError());
        // the results and the resume records lie side by side: one readback
        CU(cudaMemcpyAsync(t.pin<char>(off_res), t.dev<char>(off_res), off_at + sizeof(ResumePoint) * m - off_res,
                           cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
        memcpy(res.data(), t.pin<StreamResult>(off_res), sizeof(StreamResult) * m);
        memcpy(at.data(), t.pin<ResumePoint>(off_at), sizeof(ResumePoint) * m);
        // The stream checksum is only due when the trailer has been read: ONE pass over the output at the end of the
        // stream, not one per push, for every stream of the round that ended in it.
        std::vector<size_t> ended;
        for (size_t k = 0; k < m; ++k)
            if (res[k].trailer_seen && !res[k].ck_done) ended.push_back(k);
        if (!ended.empty()) {
            const size_t e = ended.size();
            std::vector<StreamJob>    ck_jobs(e);
            std::vector<StreamResult> ck_res(e);
            for (size_t i = 0; i < e; ++i) ck_jobs[i] = jobs[ended[i]], ck_res[i] = res[ended[i]];
            Tables c(ctx->h_st, ctx->d_st);
            const size_t off_cj = c.host(ck_jobs.data(), sizeof(StreamJob) * e);
            const size_t off_cr = c.host(ck_res.data(), sizeof(StreamResult) * e);
            if (int rc = c.upload(ctx)) return rc;
            std::vector<uint32_t> base(e + 1);
            if (int rc = run_checksum(ctx, ck_jobs.data(), c.dev<StreamJob>(off_cj), c.dev<StreamResult>(off_cr), e, base.data(),
                                      ctx->d_stbase, ctx->d_stpartial))
                return rc;
            CU(cudaMemcpyAsync(c.pin<char>(off_cr), c.dev<char>(off_cr), sizeof(StreamResult) * e, cudaMemcpyDeviceToHost,
                               ctx->stream));
            CU(cudaStreamSynchronize(ctx->stream));
            for (size_t i = 0; i < e; ++i) res[ended[i]] = c.pin<StreamResult>(off_cr)[i];
        }
        std::vector<pngb200_inflator_push_desc*> again;
        for (size_t k = 0; k < m; ++k) {
            pngb200_inflator* z = round[k]->inflator;
            const StreamResult& r = res[k];
            z->at = at[k];
            z->work[0] += at[k].bits;
            z->work[1] += at[k].bytes;
            z->work[2] += at[k].serial_bytes;
            // the next run resumes where this one stopped (after an output capacity error: where it started, or behind a
            // block it completed)
            z->phase = r.phase;
            z->resume_bit = r.resume_bit;
            z->resume_out = r.resume_out;
            if (r.status == PNGB200_ERR_OUTPUT_CAPACITY) {
                z->produced = r.resume_out;
                call.add(z->d_out, z->d_out.cap * 2, z->produced);
                again.push_back(round[k]);
                continue;
            }
            z->produced = r.produced;
            z->status = r.status;
            z->err_a = r.err_a;
            z->err_b = r.err_b;
            if (r.status == PNGB200_OK) z->terminal = true;
            round[k]->status = r.status;
        }
        if (int rc = call.grow(0)) return rc;
        round.swap(again);
    }
    return call.done();
}

}  // namespace

extern "C" {

int pngb200_inflator_push_batch(pngb200_ctx* ctx, pngb200_inflator_push_desc* pushes, size_t count)
{
    if (int rc = check_pushes(ctx, pushes, count, &pngb200_inflator_push_desc::inflator, "inflator_push_batch")) return rc;
    if (!count) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    return inflate_pushes(ctx, pushes, count);
}

int pngb200_inflator_push(pngb200_inflator* z, const uint8_t* data, size_t n)
{
    if (!z || (!data && n)) return PNGB200_ERR_BAD_ARGUMENT;
    pngb200_inflator_push_desc d{z, data, n, 0};
    const int rc = pngb200_inflator_push_batch(z->ctx, &d, 1);
    return rc != PNGB200_OK ? rc : d.status;
}

size_t pngb200_inflator_available(const pngb200_inflator* z) { return z ? (size_t)(z->produced - z->current) : 0; }

int pngb200_inflator_pull(pngb200_inflator* z, uint8_t* dst, size_t count)
{
    if (!z || (!dst && count)) return PNGB200_ERR_BAD_ARGUMENT;
    if (z->produced - z->current < count) return PNGB200_NEED_MORE_INPUT;
    pngb200_ctx* ctx = z->ctx;
    DeviceGuard guard(ctx->device);
    if (count) {
        CU(cudaMemcpyAsync(dst, z->d_out.as<uint8_t>() + z->current, count, cudaMemcpyDeviceToHost, ctx->stream));
        CU(cudaStreamSynchronize(ctx->stream));
    }
    z->current += count;
    return PNGB200_OK;
}

size_t pngb200_inflator_pull_all(pngb200_inflator* z, uint8_t* dst, size_t cap)
{
    if (!z) return 0;
    size_t n = std::min<size_t>(cap, (size_t)(z->produced - z->current));
    if (pngb200_inflator_pull(z, dst, n) != PNGB200_OK) return 0;
    return n;
}

int pngb200_inflator_stats(const pngb200_inflator* z, uint64_t out[3])
{
    if (!z || !out) return PNGB200_ERR_BAD_ARGUMENT;
    for (int k = 0; k < 3; ++k) out[k] = z->work[k];
    return PNGB200_OK;
}

void pngb200_inflator_error(const pngb200_inflator* z, int* status, uint32_t* a, uint32_t* b)
{
    if (!z) return;
    if (status) *status = z->status;
    if (a) *a = z->err_a;
    if (b) *b = z->err_b;
}

// ---------------- online decoding: PNG.Context ----------------
// The inflator handle decodes; each push resumes where the last one stopped, and its output is its window, so
// the rows it makes available are copied into `d_filt`, the context's copy of the filtered stream, and reconstructed
// there.  Storage is written by context_assign_kernel, in `d_img` for host storage (the rows a push wrote are then
// copied back) or straight into the caller's device storage.
struct pngb200_png_context {
    pngb200_ctx*      ctx = nullptr;
    pngb200_inflator* z = nullptr;
    uint32_t          w = 0, h = 0;
    uint32_t          volume = 0, depth = 0;
    bool              interlaced = false;
    int               memspace = 0;
    uint8_t*          pixels = nullptr;   // the caller's storage
    uint64_t          storage = 0;        // its bytes
    uint64_t          fsize = 0;          // filtered bytes of the image
    DevBuf            d_img, d_filt;
    uint64_t          copied = 0;         // bytes of d_filt filled
    uint64_t          drained = 0;        // bytes the decoder has pulled once every row was assigned
    int               pass = 0;           // next pass, 7 once every row is assigned (PNG.Decoder.pass)
    uint64_t          row = 0;            // next row of that pass
    bool              terminal = false;   // the stream is complete (Decoder.continue == nil)
    int               status = PNGB200_OK;
    uint32_t          err_a = 0, err_b = 0;
    uint64_t          band[2] = {0, 0};   // storage rows the last push wrote
};

pngb200_png_context* pngb200_png_context_create(pngb200_ctx* ctx, const pngb200_png_context_desc* d)
{
    if (!ctx || !d) {
        set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_context_create: null argument");
        return nullptr;
    }
    Geometry g;
    const bool whole = d->depth >= 8 && d->volume % 8 == 0;   // g.fast admits volumes that are not whole bytes
    if (!geometry(d->width, d->height, d->volume, d->depth, d->interlaced, &g) || !(g.passes || (g.fast && whole))) {
        set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_context_create: bad geometry %ux%u volume %d depth %d", d->width,
                  d->height, d->volume, d->depth);
        return nullptr;
    }
    if (d->standard > 1 || (d->memspace != PNGB200_MEM_HOST && d->memspace != PNGB200_MEM_DEVICE) || !d->pixels ||
        d->pixels_cap < g.storage) {
        set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_context_create: bad standard, memspace or storage (%zu bytes, need %llu)",
                  d->pixels_cap, (unsigned long long)g.storage);
        return nullptr;
    }
    DeviceGuard guard(ctx->device);
    pngb200_png_context* c = new pngb200_png_context();
    c->ctx = ctx;
    c->w = d->width;
    c->h = d->height;
    c->volume = d->volume;
    c->depth = d->depth;
    c->interlaced = d->interlaced != 0;
    c->memspace = d->memspace;
    c->pixels = (uint8_t*)d->pixels;
    c->storage = g.storage;
    c->fsize = g.filtered;
    c->drained = g.filtered;
    c->z = pngb200_inflator_create(ctx, d->standard ? PNGB200_FORMAT_IOS : PNGB200_FORMAT_ZLIB);
    // PNG.Image(..., uninitialized: false): storage starts out zeroed
    cudaError_t e = c->d_filt.reserve(c->fsize + 16);
    if (e == cudaSuccess && c->memspace == PNGB200_MEM_HOST) {
        memset(c->pixels, 0, c->storage);
        e = c->d_img.reserve(c->storage);
        if (e == cudaSuccess) e = cudaMemsetAsync(c->d_img.p, 0, c->storage, ctx->stream);
    } else if (e == cudaSuccess) {
        e = cudaMemsetAsync(c->pixels, 0, c->storage, ctx->stream);
    }
    if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
    if (e != cudaSuccess) {
        set_error(ctx, PNGB200_ERR_CUDA, "png_context_create: %s", cudaGetErrorString(e));
        pngb200_png_context_destroy(c);
        return nullptr;
    }
    return c;
}

void pngb200_png_context_destroy(pngb200_png_context* c)
{
    if (!c) return;
    pngb200_inflator_destroy(c->z);   // synchronises the stream
    delete c;
}

// Filtered bytes the reference's inflator makes available for the input pushed so far, beyond the inflator handle's
// `produced`: the handle leaves a stored block whose payload has not fully arrived for the next push, while
// LZ77.Inflator releases its payload byte by byte (Stream.readBlock(upTo:), Stream.swift:384-399).  Sets *src to
// where those bytes start in the input.  Reads the block's header from the handle's undecoded tail.
static uint64_t stored_in_flight(const pngb200_inflator* z, uint64_t* src)
{
    if (z->terminal || z->status < 0 || z->phase != 1 || z->produced != z->resume_out) return 0;
    auto in = [z](uint64_t i) { return z->tail[i - z->tail_at]; };
    const uint64_t b = z->resume_bit, bits = 8 * z->pushed;
    if (b + 3 > bits || ((in((b + 1) >> 3) >> ((b + 1) & 7)) & 1) || ((in((b + 2) >> 3) >> ((b + 2) & 7)) & 1)) return 0;
    const uint64_t boundary = (b + 3 + 7) & ~(uint64_t)7;
    if (boundary + 32 > bits) return 0;
    const uint64_t len = in(boundary >> 3) | ((uint64_t)in((boundary >> 3) + 1) << 8);
    *src = (boundary >> 3) + 4;
    return std::min<uint64_t>(len, z->pushed - *src);
}

}  // extern "C"

namespace {

// One push of pngb200_png_context_push_batch: the pass rows it reconstructs and assigns, in pass order
struct ContextRange { int z; uint64_t r0, r1; };

// The pushes of one pngb200_png_context_push_batch call, on distinct contexts of `ctx`: every context inflates in one
// inflate_pushes call, copies its newly available filtered bytes and runs the row state machine; then the rows of
// every context are reconstructed by one unfilter_pass_kernel launch and assigned by at most seven
// context_assign_batch_kernel launches, the k-th over the k-th pass range of every context.  Statuses as in
// inflate_pushes.
int context_pushes(pngb200_ctx* ctx, pngb200_png_push_desc* pushes, size_t count)
{
    std::vector<pngb200_png_push_desc*>      live;
    std::vector<pngb200_inflator_push_desc>  zp;
    for (size_t i = 0; i < count; ++i) {
        pngb200_png_push_desc* d = &pushes[i];
        pngb200_png_context*   c = d->context;
        c->band[0] = c->band[1] = 0;
        if (c->status < 0) d->status = c->status;
        else if (c->terminal) d->status = PNGB200_ERR_PNG_EXTRANEOUS_COMPRESSED_DATA;   // PNG.Decoder.swift:51-55
        else {
            d->status = PNGB200_ERR_CUDA;
            live.push_back(d);
            zp.push_back({c->z, d->data, d->n, 0});
        }
    }
    if (live.empty()) return PNGB200_OK;
    PushCall call(ctx);   // grows nothing: synchronises on the way out of a failed call
    const int irc = inflate_pushes(ctx, zp.data(), zp.size());
    std::vector<pngb200_png_push_desc*>   rowed;    // the pushes whose inflate succeeded
    std::vector<uint64_t>                 avail;    // filtered bytes the reference has released after each of them
    std::vector<std::vector<ContextRange>> ranges;
    std::vector<PassJob>                  jobs;
    for (size_t k = 0; k < live.size(); ++k) {
        pngb200_png_context* c  = live[k]->context;
        const int            rc = zp[k].status;
        if (rc < 0) {   // no row of this push is assigned
            int s;
            pngb200_inflator_error(c->z, &s, &c->err_a, &c->err_b);
            if (s != rc) c->err_a = c->err_b = 0;   // not a stream error (CUDA, capacity): no payload
            live[k]->status = c->status = rc;
        } else if (irc == PNGB200_OK) {
            c->terminal = rc == PNGB200_OK;
            rowed.push_back(live[k]);
        }
    }
    if (irc != PNGB200_OK) return irc;
    for (pngb200_png_push_desc* d : rowed) {
        pngb200_png_context* c = d->context;
        uint64_t src = 0;
        const uint64_t decoded = c->z->produced;
        avail.push_back(decoded + stored_in_flight(c->z, &src));
        const uint64_t fill = std::min(avail.back(), c->fsize);
        uint8_t* filt = c->d_filt.as<uint8_t>();
        if (fill > c->copied) {
            const uint64_t a = std::min(fill, decoded);
            if (a > c->copied)
                CU(cudaMemcpyAsync(filt + c->copied, c->z->d_out.as<uint8_t>() + c->copied, a - c->copied,
                                   cudaMemcpyDeviceToDevice, ctx->stream));
            const uint64_t b = std::max(c->copied, decoded);
            if (fill > b)
                CU(cudaMemcpyAsync(filt + b, c->z->d_in.as<uint8_t>() + src + (b - decoded), fill - b, cudaMemcpyDeviceToDevice,
                                   ctx->stream));
            c->copied = fill;
        }
        // PNG.Decoder.push's row loop (PNG.Decoder.swift:58-140): every complete scanline, in pass order, from where the
        // last push stopped.  The first row a pass resumes at is reconstructed again from the row above it, whose filter
        // byte becomes None: that row already holds its pixels, so it comes out unchanged and serves as the row above.
        ranges.emplace_back();
        const uint32_t bpp = (c->volume + 7) >> 3;
        int z = c->pass;
        for (; z < 7; ++z) {
            const Pass ps = stream_pass(z, c->w, c->h, c->volume, c->interlaced);
            if (ps.height == 0) continue;
            const uint64_t off  = stream_pass_offset(z, c->w, c->h, c->volume, c->interlaced);
            const uint64_t r0   = z == c->pass ? c->row : 0;
            const uint64_t have = c->copied > off ? (c->copied - off) / (ps.pitch + 1) : 0;
            const uint64_t r1   = std::min<uint64_t>(have, ps.height);
            if (r1 > r0) {
                const uint64_t start = r0 ? r0 - 1 : 0;
                uint8_t* first = filt + off + start * (ps.pitch + 1);
                if (r0) CU(cudaMemsetAsync(first, 0, 1, ctx->stream));
                jobs.push_back({first, nullptr, (r1 - start) * (ps.pitch + 1), 0, (uint32_t)(r1 - start), (uint32_t)ps.pitch, bpp});
                ranges.back().push_back({z, r0, r1});
            }
            if (r1 < ps.height) {
                c->pass = z;
                c->row = r1;
                break;
            }
        }
        if (z == 7) {
            c->pass = 7;
            c->row = 0;
        }
        if (!ranges.back().empty()) c->band[0] = c->h;
    }
    // Assign launch k takes the k-th pass range of every context: the passes of one context stay in order (a later pass
    // paints over an earlier one), and different contexts share no storage.
    std::vector<AssignJob> assign[7];
    std::vector<uint32_t>  cta_base[7];
    uint32_t               ctas[7] = {};
    for (size_t k = 0; k < 7; ++k) {
        std::vector<AssignRange> rk;
        std::vector<pngb200_png_context*> owner;
        for (size_t i = 0; i < rowed.size(); ++i) {
            if (ranges[i].size() <= k) continue;
            pngb200_png_context* c = rowed[i]->context;
            const ContextRange&  r = ranges[i][k];
            rk.push_back({r.z, r.r0, r.r1, c->d_filt.as<uint8_t>(), c->memspace == PNGB200_MEM_HOST ? c->d_img.as<uint8_t>() : c->pixels,
                          c->w, c->h, c->volume, c->depth, c->interlaced, rowed[i]->overdraw != 0});
            owner.push_back(c);
        }
        if (rk.empty()) break;
        std::vector<uint64_t> y;
        ctas[k] = plan_assign_batch(rk, (unsigned)ctx->sm_count * 16, assign[k], cta_base[k], y);
        for (size_t i = 0; i < owner.size(); ++i) {
            owner[i]->band[0] = std::min(owner[i]->band[0], y[2 * i]);
            owner[i]->band[1] = std::max(owner[i]->band[1], y[2 * i + 1]);
        }
    }
    if (!jobs.empty()) {
        std::vector<uint32_t> band_base, level_start;
        const uint64_t bands = plan_bands(jobs, band_base, level_start);
        Tables t(ctx->h_st, ctx->d_st);
        const size_t off_jobs = t.host(jobs.data(), sizeof(PassJob) * jobs.size());
        const size_t off_bb = t.host(band_base.data(), sizeof(uint32_t) * band_base.size());
        const size_t off_ls = t.host(level_start.data(), sizeof(uint32_t) * level_start.size());
        size_t off_aj[7], off_cb[7];
        for (size_t k = 0; k < 7 && ctas[k]; ++k) {
            off_aj[k] = t.host(assign[k].data(), sizeof(AssignJob) * assign[k].size());
            off_cb[k] = t.host(cta_base[k].data(), sizeof(uint32_t) * cta_base[k].size());
        }
        const size_t off_pr = t.device(sizeof(uint32_t) * (bands + 1), true);   // per-band progress, then the ticket
        if (int e = t.upload(ctx)) return e;
        WaveParams p;
        p.jobs = t.dev<PassJob>(off_jobs);
        p.band_base = t.dev<uint32_t>(off_bb);
        p.progress = t.dev<uint32_t>(off_pr);
        p.ticket = p.progress + bands;
        p.hist = nullptr;
        p.njobs = (uint32_t)jobs.size();
        p.total_bands = (uint32_t)bands;
        p.level_start = t.dev<uint32_t>(off_ls);
        p.levels = level_start.empty() ? 0u : (uint32_t)level_start.size() - 1;
        const unsigned grid = (unsigned)std::min<uint64_t>((bands + WAVE_WARPS - 1) / WAVE_WARPS, (uint64_t)ctx->sm_count * 8);
        unfilter_pass_kernel<<<grid, WAVE_WARPS * 32, WAVE_SMEM, ctx->stream>>>(p);
        ctx->launches++;
        CU(cudaGetLastError());
        for (size_t k = 0; k < 7 && ctas[k]; ++k) {
            context_assign_batch_kernel<<<ctas[k], ASSIGN_THREADS, 0, ctx->stream>>>(t.dev<AssignJob>(off_aj[k]), t.dev<uint32_t>(off_cb[k]),
                                                                                   (uint32_t)assign[k].size());
            ctx->launches++;
            CU(cudaGetLastError());
        }
    }
    for (pngb200_png_push_desc* d : rowed) {   // host storage: the rows the push wrote
        pngb200_png_context* c = d->context;
        if (c->memspace != PNGB200_MEM_HOST || c->band[1] <= c->band[0]) continue;
        const uint64_t pitch = (uint64_t)c->w * ((c->volume + 7) >> 3);
        CU(cudaMemcpyAsync(c->pixels + c->band[0] * pitch, c->d_img.as<uint8_t>() + c->band[0] * pitch,
                           (c->band[1] - c->band[0]) * pitch, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CU(cudaStreamSynchronize(ctx->stream));
    for (size_t i = 0; i < rowed.size(); ++i) {
        pngb200_png_context* c = rowed[i]->context;
        rowed[i]->status = PNGB200_OK;
        // every row is assigned: any filtered byte beyond them is an error, in this push and in any later one
        // (PNG.Decoder.swift:142-147; the bytes are drained, as inflator.pull() drains them)
        if (c->pass == 7 && avail[i] > c->drained) {
            c->drained = avail[i];
            rowed[i]->status = PNGB200_ERR_PNG_EXTRANEOUS_IMAGE_DATA;
        }
    }
    return call.done();
}

}  // namespace

extern "C" {

int pngb200_png_context_push_batch(pngb200_ctx* ctx, pngb200_png_push_desc* pushes, size_t count)
{
    if (int rc = check_pushes(ctx, pushes, count, &pngb200_png_push_desc::context, "png_context_push_batch")) return rc;
    if (ctx->pending) return set_error(ctx, PNGB200_ERR_BAD_ARGUMENT, "png_context_push: a decode batch is pending");
    if (!count) return PNGB200_OK;
    DeviceGuard guard(ctx->device);
    return context_pushes(ctx, pushes, count);
}

int pngb200_png_context_push(pngb200_png_context* c, const uint8_t* data, size_t n, int overdraw)
{
    if (!c || (!data && n)) return PNGB200_ERR_BAD_ARGUMENT;
    pngb200_png_push_desc d{c, data, n, overdraw, 0};
    const int rc = pngb200_png_context_push_batch(c->ctx, &d, 1);
    return rc != PNGB200_OK ? rc : d.status;
}

int pngb200_png_context_end(pngb200_png_context* c)
{
    if (!c) return PNGB200_ERR_BAD_ARGUMENT;
    return c->terminal ? PNGB200_OK : PNGB200_ERR_PNG_INCOMPLETE_DATASTREAM;   // PNG.Context.swift:134-141
}

int pngb200_png_context_progress(const pngb200_png_context* c, uint64_t out[6])
{
    if (!c || !out) return PNGB200_ERR_BAD_ARGUMENT;
    out[0] = (uint64_t)c->pass;
    out[1] = c->row;
    if (c->pass == 7) {
        out[2] = c->drained;
    } else {
        const Pass ps = stream_pass(c->pass, c->w, c->h, c->volume, c->interlaced);
        out[2] = stream_pass_offset(c->pass, c->w, c->h, c->volume, c->interlaced) + c->row * (ps.pitch + 1);
    }
    out[3] = c->terminal ? 1 : 0;
    out[4] = c->band[0];
    out[5] = c->band[1];
    return PNGB200_OK;
}

void pngb200_png_context_error(const pngb200_png_context* c, int* status, uint32_t* a, uint32_t* b)
{
    if (!c) return;
    if (status) *status = c->status;
    if (a) *a = c->err_a;
    if (b) *b = c->err_b;
}

}  // extern "C"

// ---------------- cloning handles (pngb200_clone_batch) ----------------
// A clone routine fills a new handle from its source: host state by assignment, and for each device buffer a fresh
// allocation plus a CopySegment for the bytes in use, which the call copies for every item with one launch.  The
// carried device state holds positions, not addresses (DfCarry is relative to its base, ResumePoint counts bits and
// bytes, and every launch builds its DfResumeJob / StreamJob pointers anew), so copied bytes are a valid state.  A
// routine that fails leaves what it allocated in the new handle, which the caller destroys.
namespace {

// `dst` takes `size` bytes: as create reserves them (`exact` false: a buffer fixed at create that later pushes write
// without a reserve), or exactly (a buffer pushes grow, given only its bytes in use); `src`'s first `keep` bytes are
// queued for the copy.
cudaError_t clone_buf(std::vector<CopySegment>& segs, DevBuf& dst, const DevBuf& src, size_t size, size_t keep, bool exact)
{
    if (!size) return cudaSuccess;
    cudaError_t e;
    if (exact) {
        e = cudaMalloc(&dst.p, size);
        if (e == cudaSuccess) dst.cap = size;
    } else {
        e = dst.reserve(size);
    }
    if (e == cudaSuccess && keep) segs.push_back({src.as<uint8_t>(), dst.as<uint8_t>(), (uint64_t)keep});
    return e;
}

cudaError_t clone_inflator(const pngb200_inflator* s, pngb200_inflator* z, std::vector<CopySegment>& segs)
{
    z->ctx = s->ctx;
    z->format = s->format;
    z->pushed = s->pushed, z->tail_at = s->tail_at, z->tail = s->tail;
    z->resume_bit = s->resume_bit, z->resume_out = s->resume_out, z->produced = s->produced, z->current = s->current;
    z->phase = s->phase;
    z->at = s->at;
    for (int k = 0; k < 3; ++k) z->work[k] = s->work[k];
    z->terminal = s->terminal;
    z->status = s->status, z->err_a = s->err_a, z->err_b = s->err_b;
    // every byte pushed, with the bit reader's 16 bytes of slack
    cudaError_t e = clone_buf(segs, z->d_in, s->d_in, s->pushed ? s->pushed + 16 : 0, s->pushed, true);
    // Pulls read the output from `current` and a resumed launch reads the window behind `produced`.  The output keeps
    // the source's capacity: a launch that runs out of it stops for another round, which decodes bits again and so
    // shows in stats(), so a smaller buffer would make the clone's stats differ from its source's.
    if (e == cudaSuccess) e = clone_buf(segs, z->d_out, s->d_out, s->d_out.cap, s->produced, true);
    return e;
}

cudaError_t clone_deflator(const pngb200_deflator* s, pngb200_deflator* z, std::vector<CopySegment>& segs)
{
    z->ctx = s->ctx;
    z->format = s->format, z->level = s->level, z->exponent = s->exponent;
    z->chunk = s->chunk;
    z->input = s->input, z->output = s->output, z->at = s->at;
    z->finished = s->finished;
    z->online = s->online;
    z->status = s->status;
    z->total = s->total, z->base = s->base, z->end_index = s->end_index, z->count = s->count;
    z->blocks = s->blocks, z->written = s->written;
    if (!s->online) return cudaSuccess;
    // d_up is scratch of one launch and d_out's bytes reach the host (or the encoder's CRC step) within the call that
    // writes them: neither is carried.  The graph keeps the unfinished block's vertices, as df_grow does.
    cudaError_t e = clone_buf(segs, z->d_carry, s->d_carry, sizeof(DfCarry), sizeof(DfCarry), false);
    if (e == cudaSuccess) e = clone_buf(segs, z->d_dict, s->d_dict, sizeof(int32_t) * DF_DICT_WORDS, sizeof(int32_t) * DF_DICT_WORDS, false);
    const size_t graph = s->d_graph.p ? std::min<size_t>(128 * (size_t)s->count, s->d_graph.cap) : 0;
    if (e == cudaSuccess) e = clone_buf(segs, z->d_graph, s->d_graph, graph, graph, true);
    if (e == cudaSuccess) e = clone_buf(segs, z->d_in, s->d_in, s->held() ? s->held() + 16 : 0, s->held(), true);
    return e;
}

// the context's storage is copied by the caller: device storage in the call's launch, host storage by memcpy after it
cudaError_t clone_context(const pngb200_png_context* s, pngb200_png_context* c, uint8_t* pixels, std::vector<CopySegment>& segs)
{
    c->ctx = s->ctx;
    c->w = s->w, c->h = s->h, c->volume = s->volume, c->depth = s->depth;
    c->interlaced = s->interlaced;
    c->memspace = s->memspace;
    c->pixels = pixels;
    c->storage = s->storage, c->fsize = s->fsize;
    c->copied = s->copied, c->drained = s->drained;
    c->pass = s->pass, c->row = s->row;
    c->terminal = s->terminal;
    c->status = s->status, c->err_a = s->err_a, c->err_b = s->err_b;
    c->band[0] = s->band[0], c->band[1] = s->band[1];
    c->z = new pngb200_inflator();
    cudaError_t e = clone_inflator(s->z, c->z, segs);
    if (e == cudaSuccess) e = clone_buf(segs, c->d_filt, s->d_filt, s->fsize + 16, s->copied, false);
    if (e == cudaSuccess && s->memspace == PNGB200_MEM_HOST) e = clone_buf(segs, c->d_img, s->d_img, s->storage, s->storage, false);
    if (e == cudaSuccess && s->memspace == PNGB200_MEM_DEVICE && s->storage) segs.push_back({s->pixels, pixels, s->storage});
    return e;
}

}  // namespace

#include "png_file.cuh"
