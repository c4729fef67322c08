/*
 * pngb200.h -- C ABI of the H100-native PNG hot path (DEFLATE inflate + scanline unfilter, and
 * the encode-side mirrors), the drop-in boundary for swift-png's `PNG.Decoder` / `PNG.Encoder`
 * / `LZ77.Inflator` / `LZ77.Deflator` call sites.
 *
 * swift-png has no FFI of its own: its hot path sits behind internal Swift value types.  The
 * entry points below are what a Swift `CPNGB200` system-library target would bind (see
 * INTEGRATION.md for the module map and the replacement bodies).  Each one cites the reference
 * interface it replaces (paths relative to the swift-png checkout).
 *
 * Conventions: plain pointers and sizes, no C++/torch types.  Every function returns a
 * pngb200_status; nothing throws or aborts.  Per-item results (status + payload mirroring the
 * Swift error enums' associated values) are written into the descriptor arrays.
 * A pngb200_ctx is bound to one CUDA device and owns one CUDA stream plus grow-only device
 * workspaces; it must be used by one thread at a time (same rule as the Swift structs).
 * There is NO CPU fallback: if CUDA is unavailable pngb200_ctx_create fails.
 */
#ifndef PNGB200_H
#define PNGB200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PNGB200_VERSION 1

/* ---- status codes (negative = error).  The numbering is shared with oracle/oracle.h ---- */
typedef enum pngb200_status {
    PNGB200_OK                                   = 0,  /* stream complete (push returned nil) */
    PNGB200_NEED_MORE_INPUT                      = 1,  /* push returned () : truncated stream */
    /* LZ77.DecompressionError, Sources/LZ77/Inflator/LZ77.DecompressionError.swift:19-60 */
    PNGB200_ERR_STREAM_CHECKSUM                  = -1, /* payload a=declared b=computed */
    PNGB200_ERR_BLOCK_TYPE                       = -2, /* a=code */
    PNGB200_ERR_BLOCK_COUNT_PARITY               = -3, /* a=LEN b=NLEN */
    PNGB200_ERR_RUNLITERAL_SYMBOL_COUNT          = -4, /* a=count */
    PNGB200_ERR_CODELENGTH_HUFFMAN_TABLE         = -5,
    PNGB200_ERR_CODELENGTH_SEQUENCE              = -6,
    PNGB200_ERR_HUFFMAN_TABLE                    = -7,
    PNGB200_ERR_STRING_REFERENCE                 = -8,
    PNGB200_ERR_INVALID_SYMBOL                   = -9, /* stricter than the reference, see DESIGN.md */
    /* LZ77.StreamHeaderError, Sources/LZ77/Inflator/LZ77.StreamHeaderError.swift:5-28 */
    PNGB200_ERR_ZLIB_METHOD                      = -16, /* a=code */
    PNGB200_ERR_ZLIB_WINDOW                      = -17, /* a=exponent */
    PNGB200_ERR_ZLIB_CHECK_BITS                  = -18,
    PNGB200_ERR_ZLIB_DICTIONARY                  = -19,
    /* Gzip.StreamHeaderError, Sources/LZ77/Gzip/Gzip.StreamHeaderError.swift */
    PNGB200_ERR_GZIP_SIGIL                       = -32,
    PNGB200_ERR_GZIP_METHOD                      = -33, /* a=code */
    PNGB200_ERR_GZIP_FLAG_BITS                   = -34, /* a=flags */
    PNGB200_ERR_GZIP_HEADER_CHECKSUM_UNSUPPORTED = -35,
    /* PNG.DecodingError cases raised on this path, Sources/PNG/Decoding/PNG.Decoder.swift:51-55,
     * :142-147 and PNG.Context.swift:134-141 */
    PNGB200_ERR_PNG_EXTRANEOUS_IMAGE_DATA        = -48,
    PNGB200_ERR_PNG_EXTRANEOUS_COMPRESSED_DATA   = -49,
    PNGB200_ERR_PNG_INCOMPLETE_DATASTREAM        = -50,
    PNGB200_ERR_PNG_PALETTE_INDEX                = -51, /* indexed pixel beyond the palette: the reference traps */
    /* PNG.LexingError (Sources/PNG/Lexing/PNG.LexingError.swift), file-level entry points */
    PNGB200_ERR_LEX_TRUNCATED_SIGNATURE          = -80,
    PNGB200_ERR_LEX_INVALID_SIGNATURE            = -81, /* a,b = the eight bytes found */
    PNGB200_ERR_LEX_TRUNCATED_CHUNK_HEADER       = -82,
    PNGB200_ERR_LEX_TRUNCATED_CHUNK_BODY         = -83, /* a = expected bytes */
    PNGB200_ERR_LEX_INVALID_CHUNK_TYPE           = -84, /* a = type code */
    PNGB200_ERR_LEX_INVALID_CHUNK_CHECKSUM       = -85, /* a = declared, b = computed */
    /* PNG.ParsingError (Sources/PNG/Parsing/PNG.ParsingError.swift): what IHDR / PLTE / tRNS can raise */
    PNGB200_ERR_PARSE_HEADER_CHUNK_LENGTH        = -96,  /* a = length */
    PNGB200_ERR_PARSE_HEADER_PIXEL_FORMAT_CODE   = -97,  /* a = depth code, b = colour code */
    PNGB200_ERR_PARSE_HEADER_PIXEL_FORMAT        = -98,  /* not allowed by the ios standard */
    PNGB200_ERR_PARSE_HEADER_COMPRESSION_CODE    = -99,  /* a = code */
    PNGB200_ERR_PARSE_HEADER_FILTER_CODE         = -100, /* a = code */
    PNGB200_ERR_PARSE_HEADER_INTERLACING_CODE    = -101, /* a = code */
    PNGB200_ERR_PARSE_HEADER_SIZE                = -102, /* a = x, b = y */
    PNGB200_ERR_PARSE_UNEXPECTED_PALETTE         = -103,
    PNGB200_ERR_PARSE_PALETTE_CHUNK_LENGTH       = -104, /* a = length */
    PNGB200_ERR_PARSE_PALETTE_COUNT              = -105, /* a = count, b = max */
    PNGB200_ERR_PARSE_UNEXPECTED_TRANSPARENCY    = -106,
    PNGB200_ERR_PARSE_TRANSPARENCY_CHUNK_LENGTH  = -107, /* a = length, b = expected */
    PNGB200_ERR_PARSE_TRANSPARENCY_SAMPLE        = -108, /* a = sample, b = max */
    PNGB200_ERR_PARSE_TRANSPARENCY_COUNT         = -109, /* a = count, b = max */
    /* PNG.DecodingError (Sources/PNG/Decoding/PNG.DecodingError.swift): a = chunk, b = the other chunk */
    PNGB200_ERR_DECODE_REQUIRED_CHUNK            = -112,
    PNGB200_ERR_DECODE_DUPLICATE_CHUNK           = -113,
    PNGB200_ERR_DECODE_UNEXPECTED_CHUNK          = -114,
    /* API-level */
    PNGB200_ERR_OUTPUT_CAPACITY                  = -64,
    PNGB200_ERR_BAD_ARGUMENT                     = -65,
    PNGB200_ERR_CUDA                             = -66, /* see pngb200_last_error */
    PNGB200_ERR_INTERNAL                         = -67
} pngb200_status;

/* LZ77.Format (.zlib, .ios) + Gzip.Format, Sources/LZ77/Wrappers/LZ77.Format.swift:8-12 */
typedef enum pngb200_format { PNGB200_FORMAT_ZLIB = 0, PNGB200_FORMAT_IOS = 1, PNGB200_FORMAT_GZIP = 2 } pngb200_format;

/* where the data pointers of a batch live */
typedef enum pngb200_memspace {
    PNGB200_MEM_HOST   = 0, /* host pointers (pinned or pageable); copies are part of the call */
    PNGB200_MEM_DEVICE = 1  /* device pointers on the context's GPU; nothing is copied */
} pngb200_memspace;

/* ---- context ---- */
typedef struct pngb200_ctx pngb200_ctx;

/* device < 0: the calling thread's current CUDA device.  Returns NULL on failure (no GPU, no
 * sm_90 device, out of memory); pngb200_last_error(NULL) then describes why. */
pngb200_ctx* pngb200_ctx_create(int device);
void         pngb200_ctx_destroy(pngb200_ctx* ctx);
/* Return the context's grow-only device arenas (and its pipeline lanes') to the driver, the streaming
 * handles' push workspaces (tables, checksum partials, staged input and the pinned host buffers behind them)
 * included; the next batch call or push allocates again.  The handles keep their own buffers.  Fails with
 * BAD_ARGUMENT while a decode batch is pending. */
int          pngb200_ctx_trim(pngb200_ctx* ctx);
const char*  pngb200_last_error(const pngb200_ctx* ctx);
/* the cudaStream_t all of this context's work is enqueued on (for event timing / interop) */
void*        pngb200_ctx_stream(pngb200_ctx* ctx);
int          pngb200_ctx_device(const pngb200_ctx* ctx);
/* number of kernels this context has launched since creation (bench.py's gpu_launches) */
uint64_t     pngb200_ctx_launch_count(const pngb200_ctx* ctx);
/* tuning knob: 0 = automatic, 1 = force the one-warp-per-stream inflate kernel,
 * 2 = force the block-parallel inflate kernel */
void         pngb200_ctx_set_inflate_mode(pngb200_ctx* ctx, int mode);
/* device time (CUDA events on the context's stream) of the last completed decode batch's stages:
 * ms[0] inflate kernels, ms[1] checksum kernels, ms[2] unfilter kernels */
int          pngb200_ctx_stage_ms(pngb200_ctx* ctx, float ms[3]);
/* device-side counters of the last finished batch of `count` streams/images, summed:
 * out[0] waves, out[1] sync rounds, out[2] copy-resolve rounds, out[3] streams that fell back to
 * the serial decoder (the analogue of the reference's -DDUMP_LZ77_BLOCKS statistics) */
int          pngb200_ctx_inflate_stats(pngb200_ctx* ctx, size_t count, uint64_t out[4]);
/* the full counter set of the last finished batch, summed over its `count` streams (the reference prints the
 * same kind of numbers under -DDUMP_LZ77_BLOCKS / -DDUMP_LZ77_BLOCKS_STATISTICS,
 * Sources/LZ77/Inflator/LZ77.InflatorBuffers.Stream.swift:11,292-297,364-374,472-486):
 * out[0..3] as pngb200_ctx_inflate_stats (out[1] = tokens decoded by chain walks), out[4] tokens (literals +
 * matches), out[5] matches, out[6] matches whose source was produced in the same 8 KiB wave by another
 * thread (they wait in the deferred-copy list), out[7] DEFLATE blocks, out[8..19] SM cycles per phase of
 * inflate_wave_kernel as seen by thread 0 of each CTA: header+tables, stage, speculate, walk, chain,
 * count+scan, emit, resolve, store, stored blocks, (2 spare); out[20..23] reserved */
int          pngb200_ctx_inflate_counters(pngb200_ctx* ctx, size_t count, uint64_t out[24]);
/* more than one CTA per stream: a batch with fewer big streams than half the CTA slots has its streams cut at
 * DEFLATE block boundaries and decoded segment by segment (csrc/inflate_segments.cuh).  Of the last inflate /
 * decode batch on this context: out[0] streams that were cut, out[1] segments they were cut into, out[2] streams
 * whose segments did not line up and that were decoded whole after all (results are identical either way). */
int          pngb200_ctx_segment_stats(pngb200_ctx* ctx, uint64_t out[3]);
/* streams of the last inflate / decode batch that were cut into a direct head and a symbolic tail and accepted:
 * out[0] heads' bytes, out[1] heads' SM cycles (thread 0 of the CTA, all phases), out[2] tails' bytes, out[3]
 * tails' SM cycles, out[4] tails that left symbolic mode once their last 32 KiB held no marker, out[5] tails'
 * bytes decoded as symbols */
int          pngb200_ctx_split_stats(pngb200_ctx* ctx, uint64_t out[6]);
/* which whole-stream engine the last inflate / decode batch on this context launched: 0 inflate_parallel_kernel
 * (round 1), 1 inflate_wave_kernel (ring window), 2 inflate_cells_kernel, -1 none (tiny streams, segments only) */
int          pngb200_ctx_last_inflate_engine(pngb200_ctx* ctx);
/* scanlines per filter type of the last decode / unfilter batch that went through the wavefront kernel
 * (non-interlaced, >= 8 bits per sample): out[0..4] = None, Sub, Up, Average, Paeth, out[5] = rows with an
 * invalid filter byte (left unchanged, as the reference does).  The device-side form of the reference's
 * -DDUMP_FILTERED_SCANLINES output (Sources/PNG/Decoding/PNG.Decoder.swift:96-98,128).  Rows of Adam7 and
 * 1/2/4-bit images are not counted, whichever kernel reconstructs them. */
int          pngb200_ctx_filter_histogram(pngb200_ctx* ctx, uint64_t out[6]);
/* images of the last decode / unfilter batch by the path that reconstructed their scanlines: out[0] the wavefront
 * kernel (non-interlaced, >= 8 bits per sample), out[1] the pass path (Adam7 or 1/2/4-bit images whose filtered
 * stream is longer than 64 KiB: every pass on the wavefront, then one interleave kernel), out[2] the one-CTA-per-image
 * generic kernel (the other Adam7 and 1/2/4-bit images).  Results are identical whichever path runs.  A batch starts
 * with pngb200_decode_batch, pngb200_unfilter_batch and the PNG file decode calls; a direct
 * pngb200_decode_batch_enqueue adds its images to the batch in progress. */
int          pngb200_ctx_unfilter_stats(pngb200_ctx* ctx, uint64_t out[3]);
/* inflate_mode: 0 automatic; 1 one warp per stream; 2 a whole CTA per stream, never cut; 3 / 4 force the
 * ring-window / the round-1 intra-stream kernel; 5 as 0; 6 force the cell kernel (inflate_cells.cuh) */

/* ---- batched one-shot entry points (the throughput path) ---- */

/* One standalone DEFLATE stream: LZ77.Inflator(format:).push(all); pull()  /  Gzip.extract.
 * Replaces Sources/LZ77/Inflator/LZ77.Inflator.swift:30-61 and Sources/LZ77/Gzip/Gzip.swift:6-11. */
typedef struct pngb200_stream_desc {
    const uint8_t* src;       /* compressed stream */
    size_t         src_len;
    uint8_t*       dst;       /* inflated bytes */
    size_t         dst_cap;
    int32_t        format;    /* pngb200_format */
    /* results */
    int32_t        status;    /* pngb200_status */
    uint32_t       err_a, err_b;
    uint32_t       checksum;  /* Adler-32 (zlib, ios) or CRC-32 (gzip) of the output */
    uint32_t       blocks;    /* DEFLATE blocks decoded */
    uint64_t       produced;  /* bytes written to dst */
    uint64_t       consumed_bits;
} pngb200_stream_desc;

int pngb200_inflate_batch(pngb200_ctx* ctx, pngb200_stream_desc* streams, size_t count, int memspace);

/* One PNG image's IDAT stream: PNG.Decoder.push(data, size:, pixel:, delegate: image.assign)
 * over the concatenated IDAT payload.  Replaces Sources/PNG/Decoding/PNG.Decoder.swift:47-149
 * (+ defilter :152-196, PNG.paeth PNG.swift:124-147) and PNG.Image.assign
 * (Sources/PNG/PNG.Image.swift:186-285).  `pixels` receives PNG.Image.storage exactly:
 * width*height*((volume+7)>>3) bytes, row-major, 16-bit samples big-endian, sub-byte depths
 * expanded to one byte per pixel. */
typedef struct pngb200_image_desc {
    const uint8_t* idat;      /* concatenated IDAT payloads (a zlib stream; raw DEFLATE for .ios) */
    size_t         idat_len;
    uint8_t*       pixels;
    size_t         pixels_cap;
    uint32_t       width, height;
    uint8_t        volume;    /* bits per pixel, PNG.Format.Pixel.volume */
    uint8_t        depth;     /* bits per sample */
    uint8_t        interlaced;
    uint8_t        format;    /* PNGB200_FORMAT_ZLIB (PNG.Standard.common) or _IOS */
    /* results */
    int32_t        status;
    uint32_t       err_a, err_b;
    uint32_t       checksum;  /* Adler-32 of the filtered stream */
    uint32_t       blocks;
    uint64_t       produced;  /* inflated (filtered) bytes */
} pngb200_image_desc;

int pngb200_decode_batch(pngb200_ctx* ctx, pngb200_image_desc* images, size_t count, int memspace);
/* same, split so that device time can be bracketed with events: enqueue returns once all work is
 * queued on pngb200_ctx_stream; finish synchronises and fills in the result fields. */
int pngb200_decode_batch_enqueue(pngb200_ctx* ctx, pngb200_image_desc* images, size_t count, int memspace);
int pngb200_decode_batch_finish(pngb200_ctx* ctx, pngb200_image_desc* images, size_t count);

/* The unfilter stage alone (PNG.Decoder.defilter + PNG.Image.assign over an already inflated
 * stream); `idat`/`idat_len` hold the FILTERED bytes.  Exposed for kernel-level tests/benchmarks. */
int pngb200_unfilter_batch(pngb200_ctx* ctx, pngb200_image_desc* images, size_t count, int memspace);

/* Encode-side stage 1: PNG.Image.collect + PNG.Encoder.filter for every row
 * (Sources/PNG/Encoding/PNG.Encoder.swift:132-204,230-234; PNG.Image.swift:431-544).
 * `pixels` is the INPUT (PNG.Image.storage), `idat`... see pngb200_filter_desc. */
typedef struct pngb200_filter_desc {
    const uint8_t* pixels;    /* PNG.Image.storage */
    size_t         pixels_len;
    uint8_t*       filtered;  /* out: height*(pitch+1) bytes (sum over Adam7 passes if interlaced) */
    size_t         filtered_cap;
    uint32_t       width, height;
    uint8_t        volume, depth, interlaced, reserved;
    int32_t        status;
    uint64_t       produced;
} pngb200_filter_desc;

int pngb200_filter_batch(pngb200_ctx* ctx, pngb200_filter_desc* images, size_t count, int memspace);

/* ---- colour targets (SURVEY.md section 8f row N1) ------------------------------------------------
 * image.unpack(as: PNG.RGBA<T>.self) / PNG.VA<T> and PNG.Image.init(packing:size:layout:) with the
 * default deindexer / indexer, T = UInt8 or UInt16: Sources/PNG/ColorTargets/PNG.RGBA.swift:262-478,
 * PNG.VA.swift, PNG.Color.swift, over the convolve / deconvolve closures of Sources/PNG/PNG.swift:149-1285.
 * The unpack is inside the reference's own timed decode loop (Benchmarks/Decompression/Swift/Main.swift:105-106).
 * For rgba8 -> RGBA<UInt8> and va8 -> VA<UInt8> the unpacked array IS PNG.Image.storage, byte for
 * byte, so pngb200_decode_batch's output needs no second pass.
 *
 * RGBA32 / RGBA64 / VA32 / VA64 are the UInt32 / UInt64 specialisations of the same types
 * (PNG.RGBA.swift:253-257; Swift's UInt is UInt64 on every 64-bit platform): 16 / 32 / 8 / 16 bytes
 * per pixel, chroma key -> alpha 0, bgr samples swapped, VA keeps r, exactly as at 8 and 16 bits.
 * V8 ... V64 are the scalar targets image.unpack(as: T.self) / PNG.Image(packing: [T], ...) with
 * T = UInt8 ... UInt64 (PNG.Image.swift:681-833, 1079-1145), 1 / 2 / 4 / 8 bytes per pixel:
 *   unpack: v of v and va, r of rgb and rgba (c.2 of bgr8 / bgra8), palette[i].r widened from 8 bits;
 *           chroma keys are ignored (the scalar target has no alpha);
 *   pack:   v -> (v), va -> (v, T.max), rgb / bgr -> (v, v, v), rgba / bgra -> (v, v, v, T.max), each
 *           narrowed to the format's depth; indexed formats store the first palette entry equal to
 *           (v8, v8, v8, 255) with v8 = v >> (T.bitWidth - 8), else 0 (the default indexer, :1126-1145).
 * With PNGB200_MEM_DEVICE, `pixels` must be aligned to min(bytes per pixel, 16): RGBA64 needs 16 bytes,
 * V8 needs none. */
typedef enum pngb200_target {
    PNGB200_TARGET_RGBA8 = 0, PNGB200_TARGET_RGBA16 = 1, PNGB200_TARGET_VA8 = 2, PNGB200_TARGET_VA16 = 3,
    PNGB200_TARGET_RGBA32 = 4, PNGB200_TARGET_RGBA64 = 5, PNGB200_TARGET_VA32 = 6, PNGB200_TARGET_VA64 = 7,
    PNGB200_TARGET_V8 = 8, PNGB200_TARGET_V16 = 9, PNGB200_TARGET_V32 = 10, PNGB200_TARGET_V64 = 11
} pngb200_target;
/* applied per pixel after unpacking: .premultiplied / .straightened (PNG.RGBA.swift:115-121, 163-169),
 * or premultiplied(as: U.self) / straightened(as: U.self) with U = UInt8 / UInt16 / UInt32
 * (PNG.RGBA.swift:146-206, PNG.VA.swift:79, 120): shift = T.bitWidth - U.bitWidth,
 * q = T.max / (T.max >> shift), every component including alpha requantised through U.
 * Valid combinations: a scalar target (V8 ... V64) takes only ASIS; _AS{U} needs an RGBA or VA target
 * whose T is wider than U (AS8: 16, 32, 64 bits; AS16: 32, 64; AS32: 64).  Anything else is
 * PNGB200_ERR_BAD_ARGUMENT before any work.  At 64 bits the products are full 128-bit, and
 * straightening saturates at T.max where the reference's dividingFullWidth traps. */
typedef enum pngb200_alpha_mode {
    PNGB200_ALPHA_ASIS = 0, PNGB200_ALPHA_PREMULTIPLIED = 1, PNGB200_ALPHA_STRAIGHTENED = 2,
    PNGB200_ALPHA_PREMULTIPLIED_AS8 = 3, PNGB200_ALPHA_STRAIGHTENED_AS8 = 4,
    PNGB200_ALPHA_PREMULTIPLIED_AS16 = 5, PNGB200_ALPHA_STRAIGHTENED_AS16 = 6,
    PNGB200_ALPHA_PREMULTIPLIED_AS32 = 7, PNGB200_ALPHA_STRAIGHTENED_AS32 = 8
} pngb200_alpha_mode;
/* PNG.Format (Sources/PNG/Formats/PNG.Format.swift:6-43) as these kernels see it */
typedef struct pngb200_pixel_format {
    uint8_t        color;         /* PNG colour type: 0 v, 2 rgb, 3 indexed, 4 va, 6 rgba */
    uint8_t        depth;         /* bits per sample: 1, 2, 4, 8, 16 */
    uint8_t        bgr;           /* 1: .bgr8 / .bgra8 (the ios standard's sample order) */
    uint8_t        has_key;       /* chroma key present (v / rgb / bgr formats) */
    uint16_t       key[3];        /* raw sample values in STORAGE order (Format.recognize, :161-330) */
    uint16_t       palette_count; /* indexed formats: entries in `palette` */
    const uint8_t* palette;       /* palette_count x (r, g, b, a), tRNS merged; always HOST memory */
} pngb200_pixel_format;
typedef struct pngb200_color_desc {
    void*                storage;      /* PNG.Image.storage: unpack reads it, pack writes it */
    size_t               storage_len;  /* bytes (capacity for pack) */
    void*                pixels;       /* [RGBA<T>] / [VA<T>] / [T]: native-endian T components, aligned to min(pixel size, 16) */
    size_t               pixels_len;   /* bytes (capacity for unpack) */
    uint64_t             count;        /* number of pixels */
    pngb200_pixel_format format;
    int32_t              status;       /* out: PNGB200_OK or PNGB200_ERR_PNG_PALETTE_INDEX */
} pngb200_color_desc;
int pngb200_unpack_batch(pngb200_ctx* ctx, pngb200_color_desc* images, size_t count, int target,
                         int alpha_mode, int memspace);
int pngb200_pack_batch(pngb200_ctx* ctx, pngb200_color_desc* images, size_t count, int target, int memspace);

/* Encode-side stage 2: LZ77.Deflator(format:level:exponent:hint:).push(src, last: true) and the
 * concatenation of every pull() -- the reference's compressed bytes, bit for bit (its output does
 * not depend on push granularity or on `hint`).  Replaces Sources/LZ77/Deflator/LZ77.Deflator.swift:8-44,
 * Sources/LZ77/Gzip/Gzip.swift:34-46 (Gzip.archive) and everything behind them.  level 0...13 as in
 * LZ77.DeflatorSearch (0-3 greedy, 4-7 lazy, 8-13 full); exponent 8...15. */
typedef struct pngb200_deflate_desc {
    const uint8_t* src;
    size_t         src_len;
    uint8_t*       dst;
    size_t         dst_cap;   /* pngb200_deflate_bound(src_len) is always enough */
    int32_t        format;    /* pngb200_format */
    int32_t        level;
    int32_t        exponent;
    /* results */
    int32_t        status;
    uint32_t       checksum;  /* Adler-32 / CRC-32 of src as written into the trailer */
    uint32_t       blocks;
    uint64_t       produced;
} pngb200_deflate_desc;

int    pngb200_deflate_batch(pngb200_ctx* ctx, pngb200_deflate_desc* streams, size_t count, int memspace);
size_t pngb200_deflate_bound(size_t src_len);

/* PNG.Encoder.pull over a whole image: collect + filter + deflate (format .zlib / .ios) -> the
 * concatenated IDAT payload.  Replaces Sources/PNG/Encoding/PNG.Encoder.swift:33-129. */
typedef struct pngb200_encode_desc {
    const uint8_t* pixels;    /* PNG.Image.storage */
    size_t         pixels_len;
    uint8_t*       idat;      /* out: concatenated IDAT payload */
    size_t         idat_cap;
    uint32_t       width, height;
    uint8_t        volume, depth, interlaced, format;
    int32_t        level;
    int32_t        status;
    uint32_t       checksum, blocks;
    uint64_t       produced;
} pngb200_encode_desc;

int pngb200_encode_batch(pngb200_ctx* ctx, pngb200_encode_desc* images, size_t count, int memspace);

/* ---- whole PNG files (SURVEY.md section 8f row N2) ------------------------------------------------
 * PNG.Image.decompress(stream:) and PNG.Image.compress(stream:level:hint:) at file level
 * (Sources/PNG/PNG.Image.swift:298-401, 576-670): signature, chunk framing, per-chunk CRC-32
 * (Lexing/PNG.BytestreamSource.swift:17-83, PNG.BytestreamDestination.swift:66-95), IHDR / PLTE / tRNS,
 * the ordering rules that involve them, IDAT concatenation and framing.  The host reads chunk HEADERS
 * only; CRC-32 of every chunk, IDAT gather / scatter and the codec run on the device.  Ancillary chunks
 * other than PLTE / tRNS / bKGD are CRC-checked and otherwise ignored (metadata is not on the hot path).
 * Errors come back in the order the reference's streaming loop meets them. */
typedef struct pngb200_png_desc {
    const uint8_t*       file;          /* in: the PNG file, HOST memory (pngb200_png_*_files: file_memspace) */
    size_t               file_len;
    void*                pixels;        /* out: PNG.Image.storage (memspace of the call) */
    size_t               pixels_cap;    /* >= storage_size (pngb200_png_inspect_batch reports it) */
    /* out: PNG.Header + PNG.Layout.format */
    uint32_t             width, height;
    uint8_t              depth, color, interlaced, standard; /* standard: 0 common, 1 ios (CgBI) */
    pngb200_pixel_format format;        /* ready for pngb200_unpack_batch; palette -> palette_rgba */
    uint8_t              palette_rgba[1024];
    uint64_t             storage_size;  /* width * height * bytes per pixel */
    uint64_t             idat_bytes;    /* concatenated IDAT payload */
    uint32_t             idat_chunks, chunks;
    int32_t              status;        /* pngb200_status */
    uint32_t             err_a, err_b;
    uint32_t             checksum, blocks;
    uint64_t             produced;
} pngb200_png_desc;
/* host only: walk the chunk headers, parse IHDR / PLTE / tRNS, fill the out fields (no CRC check, no
 * GPU) -- what a caller needs to size `pixels`.  pngb200_png_inspect_files(NULL, files, count, PNGB200_MEM_HOST). */
int pngb200_png_inspect_batch(pngb200_png_desc* files, size_t count);
/* `memspace` is where `pixels` live; files are host memory.
 * pngb200_png_decode_files(ctx, files, count, PNGB200_MEM_HOST, memspace). */
int pngb200_png_decode_batch(pngb200_ctx* ctx, pngb200_png_desc* files, size_t count, int memspace);

/* The same calls for files anywhere.  file_memspace: where every `file` points (PNGB200_MEM_DEVICE: the context's
 * GPU, any alignment); memspace: where `pixels` live, as in pngb200_png_decode_batch.  Every out field, every pixel
 * and every error is what the host-file calls give for the same bytes.
 * With device files the chunk walk runs on the GPU (one warp per file; inside an IDAT run the warp checks 32 chunk
 * headers a step) and the host receives a small summary per file and the chunk records; CRC-32 regions point into
 * the files themselves, and the IDAT run is gathered device to device into the context's payload arena, so the
 * decoder never reads a caller pointer.  A device-file batch runs as one piece on the context (there is no host copy
 * to overlap).  pngb200_png_inspect_files needs `ctx` only for device files; it does not check CRCs.
 * A file_memspace other than HOST or DEVICE, or a call while a decode batch is pending: PNGB200_ERR_BAD_ARGUMENT. */
int pngb200_png_inspect_files(pngb200_ctx* ctx, pngb200_png_desc* files, size_t count, int file_memspace);
int pngb200_png_decode_files(pngb200_ctx* ctx, pngb200_png_desc* files, size_t count, int file_memspace, int memspace);

typedef struct pngb200_png_encode_desc {
    const void*          pixels;        /* in: PNG.Image.storage (memspace of the call) */
    size_t               pixels_len;
    uint32_t             width, height;
    pngb200_pixel_format format;        /* bgr = 1 writes the ios standard (CgBI chunk, raw deflate) */
    uint8_t              interlaced;
    int32_t              level;         /* 0...13 */
    uint32_t             idat_chunk;    /* bytes per IDAT chunk; 0 = 65544, what the reference emits for its
                                           default hint (2 x the capacity malloc gives DeflatorOut's buffer) */
    uint8_t*             file;          /* out: the PNG file, HOST memory (pngb200_png_encode_files: file_memspace) */
    size_t               file_cap;      /* >= pngb200_png_encode_bound(...) */
    int32_t              status;
    uint32_t             checksum, blocks;
    uint64_t             produced;      /* file bytes */
} pngb200_png_encode_desc;
size_t pngb200_png_encode_bound(uint32_t width, uint32_t height, const pngb200_pixel_format* format, int interlaced,
                                uint32_t idat_chunk);
int    pngb200_png_encode_batch(pngb200_ctx* ctx, pngb200_png_encode_desc* images, size_t count, int memspace);
/* pngb200_png_encode_batch for files anywhere: with file_memspace PNGB200_MEM_DEVICE, `file` is a device buffer on
 * the context's GPU and the file is written straight into it (head by one small host-to-device copy, IDAT framing and
 * CRC-32 in place, IEND) -- the same bytes pngb200_png_encode_batch writes, with no device-to-host copy.  file_cap and
 * pngb200_png_encode_bound are unchanged.  A file_memspace other than HOST or DEVICE: PNGB200_ERR_BAD_ARGUMENT. */
int    pngb200_png_encode_files(pngb200_ctx* ctx, pngb200_png_encode_desc* images, size_t count, int memspace,
                                int file_memspace);

/* size helpers (host arithmetic only) */
size_t pngb200_filtered_size(uint32_t width, uint32_t height, int volume, int interlaced);
size_t pngb200_storage_size(uint32_t width, uint32_t height, int volume);

/* ---- streaming handles (LZ77.Inflator value-type semantics, layered on the batch path) ----
 * Each push decodes only input no earlier push decoded: it resumes where the last one stopped, at a block header or,
 * inside a fixed or dynamic block, at the last complete symbol (whose block header is parsed again).  A stored block
 * is released once all of it has arrived. */
typedef struct pngb200_inflator pngb200_inflator;
/* LZ77.Inflator.init(format:) / Gzip.Inflator.init(), LZ77.Inflator.swift:18-23 */
pngb200_inflator* pngb200_inflator_create(pngb200_ctx* ctx, int format);
void              pngb200_inflator_destroy(pngb200_inflator* z);
/* push(_:) : copies `data`; returns PNGB200_OK when the stream is complete (Swift: nil),
 * PNGB200_NEED_MORE_INPUT when it wants more (Swift: ()), <0 on error (Swift: throws). */
int    pngb200_inflator_push(pngb200_inflator* z, const uint8_t* data, size_t n);
/* pull(_ count:) : exactly `count` bytes or PNGB200_NEED_MORE_INPUT (Swift: nil) */
int    pngb200_inflator_pull(pngb200_inflator* z, uint8_t* dst, size_t count);
/* pull() : everything available; returns the number of bytes copied (<= cap) */
size_t pngb200_inflator_pull_all(pngb200_inflator* z, uint8_t* dst, size_t cap);
size_t pngb200_inflator_available(const pngb200_inflator* z);
void   pngb200_inflator_error(const pngb200_inflator* z, int* status, uint32_t* a, uint32_t* b);
/* Work the device has done for this handle since it was created: out[0] input bits decoded (a bit decoded twice counts
 * twice), out[1] output bytes written (likewise), out[2] of those written by the one-warp serial decoder. */
int    pngb200_inflator_stats(const pngb200_inflator* z, uint64_t out[3]);

/* Many pushes in one call: the throughput path of the streaming handles, for a caller that holds many streams at once.
 * Each item behaves exactly as the same push made alone through pngb200_inflator_push: its status, error payload,
 * available bytes, pulled bytes and stats are the ones that push would leave, whatever else the call holds.  The handles
 * are distinct, so item order does not matter.  Terminal handles and handles with a sticky error are answered on the
 * host, with no device work.  Items may mix formats.  Usable while a decode batch is pending on the ctx (the pushes
 * have workspaces of their own).
 * Returns PNGB200_OK once every item's status is written, even when some items failed; PNGB200_ERR_BAD_ARGUMENT, before
 * any work and with no item touched, for a null ctx, pushes NULL with count > 0, a null handle, a handle of another ctx,
 * the same handle twice, or data NULL with n > 0 (count == 0 is OK); PNGB200_ERR_CUDA, with every handle unchanged, when
 * the staged input or a buffer a handle grows to take its push in cannot be allocated; PNGB200_ERR_CUDA on any other
 * CUDA failure (a later allocation included), each item not finished then left as a single push failing the same way
 * would leave it (status PNGB200_ERR_CUDA).
 * Fixed cost, whatever `count`: one round of at most 2 kernel launches (the ring inflate kernel over the items with
 * 64 KiB or more of undecoded input, the serial one over the rest) and 1 stream synchronise, then, when streams ended,
 * 2 checksum launches and 1 synchronise.  An item whose output buffer has to grow goes again in a further round, with
 * the other items of that kind only: each such round adds the same costs. */
typedef struct pngb200_inflator_push_desc {
    pngb200_inflator* inflator;
    const uint8_t*    data;      /* host memory, copied, as pngb200_inflator_push */
    size_t            n;
    int32_t           status;    /* out: what pngb200_inflator_push would return for this push */
} pngb200_inflator_push_desc;
int    pngb200_inflator_push_batch(pngb200_ctx* ctx, pngb200_inflator_push_desc* pushes, size_t count);

/* ---- online decoding: PNG.Context (Sources/PNG/Decoding/PNG.Context.swift) ----------------------------------------
 * A caller pushes each IDAT chunk as it arrives; after every push the storage is a valid partial image.  Restates
 * PNG.Context.push(data:overdraw:), the row state machine of PNG.Decoder.push (PNG.Decoder.swift:47-149),
 * PNG.Image.assign and PNG.Image.overdraw (PNG.Image.swift:133-285), and push(ancillary:) with IEND.
 * Inflate runs on the device through a pngb200_inflator; the newly available scanlines are reconstructed by
 * unfilter_pass_kernel and written into storage, pass by pass, by context_assign_batch_kernel.  After each push the rows
 * assigned are exactly the reference's: its inflator releases the payload of a stored block as it arrives, and so
 * does the context (the pngb200_inflator handle itself waits for the whole block). */
typedef struct pngb200_png_context pngb200_png_context;
typedef struct pngb200_png_context_desc {
    void*    pixels;       /* PNG.Image.storage, width*height*((volume+7)>>3) bytes, in `memspace`; any alignment */
    size_t   pixels_cap;
    uint32_t width, height;
    uint8_t  volume, depth, interlaced, standard;   /* standard 0 common (zlib), 1 ios (raw deflate) */
    int32_t  memspace;     /* pngb200_memspace */
} pngb200_png_context_desc;
/* PNG.Context.init(..., uninitialized: false): zero-fills the storage (with `uninitialized: true` the reference leaves
 * unassigned bytes undefined; zero is one of the values they may have).  Bad geometry or pixel format, too small a
 * pixels_cap, an unknown standard or memspace: NULL, and pngb200_last_error says why. */
pngb200_png_context* pngb200_png_context_create(pngb200_ctx* ctx, const pngb200_png_context_desc* desc);
/* push(data:overdraw:) with host `data` (one IDAT payload, any length, empty included).  Returns PNGB200_OK, or:
 *   PNGB200_ERR_PNG_EXTRANEOUS_COMPRESSED_DATA  the stream was already complete (even for an empty push);
 *   an inflate error, with the reference's payload in pngb200_png_context_error: no row of the failing push is
 *     assigned, storage stays as the previous push left it, and every later push returns the same error (the
 *     reference leaves its state after a throw unspecified; this is one consistent choice);
 *   PNGB200_ERR_PNG_EXTRANEOUS_IMAGE_DATA  every row is assigned and filtered bytes remain, in the push that
 *     completes the image or in any later one that brings more; the rows are still assigned;
 *   PNGB200_ERR_BAD_ARGUMENT while a decode batch is pending on the ctx.
 * Otherwise every complete scanline now available is reconstructed and assigned in pass order, resuming mid-pass; with
 * `overdraw` each scanline is overdrawn right after it is assigned (it may differ from one push to the next).  The call
 * returns once the storage holds the new rows, host or device. */
int  pngb200_png_context_push(pngb200_png_context* c, const uint8_t* data, size_t n, int overdraw);

/* Many pushes in one call, one per context: the throughput path for a caller with many images in flight.  Each item
 * behaves exactly as the same push made alone through pngb200_png_context_push: its status, error payload, progress
 * (all six values) and storage are the ones that push would leave.  The contexts are distinct, so item order does not
 * matter; each keeps the stored-block rule (a stored block's payload is released as it arrives).  Terminal contexts
 * and contexts with a sticky error are answered on the host, with no device work.  Items may mix storage memspaces,
 * standards, interlacing, depths, volumes and overdraw.
 * Returns and rejects as pngb200_inflator_push_batch, and also rejects (PNGB200_ERR_BAD_ARGUMENT, no item touched) a
 * call while a decode batch is pending on the ctx.
 * Fixed cost, whatever `count`: the inflator rounds of pngb200_inflator_push_batch, then 1 unfilter_pass_kernel launch
 * over the new rows of every context, at most 7 context_assign_batch_kernel launches (launch k assigns the k-th pass
 * range every context touched in this push) and 1 stream synchronise.  pngb200_png_context_push is this call with
 * one item. */
typedef struct pngb200_png_push_desc {
    pngb200_png_context* context;
    const uint8_t*       data;   /* host memory: one IDAT payload, any length, empty included */
    size_t               n;
    int32_t              overdraw;
    int32_t              status; /* out: what pngb200_png_context_push would return for this push */
} pngb200_png_push_desc;
int  pngb200_png_context_push_batch(pngb200_ctx* ctx, pngb200_png_push_desc* pushes, size_t count);
/* push(ancillary:) with IEND: PNGB200_OK if and only if the DEFLATE stream is complete, else
 * PNGB200_ERR_PNG_INCOMPLETE_DATASTREAM.  A complete stream with too few rows is OK, as in pngb200_decode_batch. */
int  pngb200_png_context_end(pngb200_png_context* c);
/* out[0] next pass (0-6), 7 once every row is assigned (a non-interlaced image reports 0, then 7: PNG.Decoder.pass);
 * out[1] next row of that pass; out[2] filtered bytes consumed; out[3] 1 once the stream is complete; out[4], out[5]
 * the first storage row the last push wrote and one past its last (0, 0 if none): the band a viewer redraws. */
int  pngb200_png_context_progress(const pngb200_png_context* c, uint64_t out[6]);
/* the sticky inflate error (PNGB200_OK if none) and its payload */
void pngb200_png_context_error(const pngb200_png_context* c, int* status, uint32_t* a, uint32_t* b);
void pngb200_png_context_destroy(pngb200_png_context* c);

/* LZ77.Deflator value-type semantics (Sources/LZ77/Deflator/LZ77.Deflator.swift:8-44; the call sites are
 * PNG.Encoder.pull, Sources/PNG/Encoding/PNG.Encoder.swift:68,85,101,117,121,128).
 * init(format:level:exponent:hint:) -- `chunk_bytes` is the size of a complete output block: the reference hands out
 * 2 * capacity bytes, capacity being whatever malloc grants for `hint` UInt16 atoms (LZ77.DeflatorOut.swift:15-27,
 * 109-135); 0 = 65544, the value behind the reference's committed outputs (hint 1 << 15).
 * Two constructors, which differ in *when* blocks become available, not in the bytes:
 *  - pngb200_deflator_create: a buffered handle.  It keeps the input on the host and compresses the whole stream in
 *    one launch at push(last: true), so pop() returns "nil" before that where the reference might already have a
 *    block.
 *  - pngb200_deflator_create_online: an online handle.  Each push does what LZ77.DeflatorBuffers.push(_:last:) does
 *    (DeflatorBuffers.swift:68-137): when more than 4096 bytes are pending, or on `last`, deflate_resume_kernel
 *    compresses on the device while more input than the lookahead (258; 259 for levels 4-7) is pending and writes
 *    every block that fills; the state stays on the device between pushes.  After each push pop() / pull() return
 *    exactly what the reference's would, with one deliberate difference: pull() before `last` returns a complete
 *    block if there is one and otherwise nil, where the reference flushes a byte-padded partial block
 *    (DeflatorOut.swift:96-101) that corrupts the rest of its stream.  The handle holds its dictionary (512 KiB), the
 *    input from min(current block start, window start) on, and in full mode (levels 8-13) the unfinished block's
 *    graph (128 bytes a vertex, at most 2^21 vertices), whatever the stream length.  One push is at most 1 GiB.
 * With either, the sequence of blocks a caller sees -- sizes and bytes -- is the reference's. */
typedef struct pngb200_deflator pngb200_deflator;
pngb200_deflator* pngb200_deflator_create(pngb200_ctx* ctx, int format, int level, int exponent, size_t chunk_bytes);
/* the same arguments and validation; NULL with PNGB200_ERR_CUDA in the last error if the device state cannot be had */
pngb200_deflator* pngb200_deflator_create_online(pngb200_ctx* ctx, int format, int level, int exponent, size_t chunk_bytes);
void              pngb200_deflator_destroy(pngb200_deflator* z);
/* push(_:last:) : copies `data`.  Returns PNGB200_OK, or < 0 when compressing failed.  A push after `last` is
 * PNGB200_ERR_BAD_ARGUMENT.  On an online handle this is pngb200_deflator_push_batch with one item. */
int    pngb200_deflator_push(pngb200_deflator* z, const uint8_t* data, size_t n, int last);
/* push(_:last:) of many online handles in one call.  Each item behaves exactly as the same push made alone; items may
 * mix formats, levels and exponents.  Returns PNGB200_ERR_BAD_ARGUMENT, touching no item, for a null ctx or array, a
 * null handle, a buffered handle, a handle of another ctx, the same handle twice, data NULL with n > 0, or a pending
 * decode batch; PNGB200_ERR_CUDA, with every handle unchanged, when a buffer cannot be allocated.  Otherwise each
 * item's `status` is what pngb200_deflator_push would return.  Costs per call, whatever `count`: one upload of the new
 * input, at most one deflate_resume_kernel launch over the items that compress, and one synchronise; an item that only
 * enqueues costs its copy.  A CUDA error after the launch makes the error of the handles in it sticky. */
typedef struct pngb200_deflator_push_desc {
    pngb200_deflator* deflator;
    const uint8_t*    data;      /* host memory, copied */
    size_t            n;
    int32_t           last;
    int32_t           status;    /* out */
} pngb200_deflator_push_desc;
int    pngb200_deflator_push_batch(pngb200_ctx* ctx, pngb200_deflator_push_desc* pushes, size_t count);
/* online handles: out[0] input bytes the device has dequeued (each byte once), out[1] compressed bytes written (the
 * stream header included), out[2] blocks written, out[3] device bytes the handle holds now.  PNGB200_ERR_BAD_ARGUMENT
 * for a buffered handle. */
int    pngb200_deflator_stats(const pngb200_deflator* z, uint64_t out[4]);
/* pop() : a complete block (exactly chunk_bytes) -> returns 1 and sets *block / *n (valid until the next call on
 * this handle); 0 = nil */
int    pngb200_deflator_pop(pngb200_deflator* z, const uint8_t** block, size_t* n);
/* pull() : a complete block if there is one, else the flushed incomplete block (non-empty); 0 = nil */
int    pngb200_deflator_pull(pngb200_deflator* z, const uint8_t** block, size_t* n);

/* ---- online encoding: PNG.Image.compress(stream:level:hint:) row by row (Sources/PNG/PNG.Image.swift:576-668,
 * PNG.Encoder.pull, Sources/PNG/Encoding/PNG.Encoder.swift:33-129) --------------------------------------------------
 * A caller pushes the rows of PNG.Image.storage as they are produced, top to bottom; the handle collects and filters
 * the scanlines they complete on the device (filter_resume_kernel, one warp a scanline, straight onto the end of an
 * online deflator's input), deflates them (deflate_resume_kernel), CRCs the IDAT payload on the device
 * (crc_regions_kernel) and frames the chunks.  pop() then hands out the file in pieces:
 *   1. the head: signature, [CgBI], IHDR, [PLTE], [tRNS], as pngb200_png_encode_files writes it -- a piece of its own,
 *      so that a caller can splice ancillary chunks in behind it;
 *   2. each IDAT chunk, framed (length, type, payload of idat_chunk bytes, the last one shorter, CRC-32);
 *   3. IEND.
 * For every push schedule the pieces joined are pngb200_png_encode_batch's file for the same image, level and
 * idat_chunk.  After each push the pieces available are exactly the chunks the reference has written by the time
 * PNG.Encoder.pull asks collect for the first scanline the rows pushed so far do not complete: a non-interlaced
 * scanline y needs storage row y; Adam7 pass z's scanline y needs row by + y * sy, in stream order (pass 0 streams
 * while rows arrive, the others follow as the rows they need arrive).  The reference pushes one scanline at a time
 * into its deflator, and each of those pushes compresses when more than 4096 bytes are pending, so the deflate kernel
 * applies that rule at every scanline end inside a push.  The push that brings the last row also does
 * push([], last: true): the rest of the payload and IEND become available.
 * Device memory: the online deflator's (its dictionary, the input from min(block start, window start) on and, at
 * levels 8-13, the unfinished block's graph; see pngb200_deflator_create_online), plus one storage row for a
 * non-interlaced image -- independent of the image's height -- or the whole storage for an Adam7 image, since passes
 * 1 to 6 reread rows pass 0 used.
 * Size limit: one push completes at most 1 GiB of filtered scanlines (the online deflator's limit on one push).  So
 * pngb200_png_encoder_create refuses a non-interlaced image whose filtered scanline (pitch + 1 bytes) is over 1 GiB,
 * and an Adam7 image whose whole filtered stream (pngb200_filtered_size) is over 1 GiB, since its last row completes
 * passes 1 to 6 at once.  pngb200_png_encode_batch encodes such images. */
typedef struct pngb200_png_encoder pngb200_png_encoder;
typedef struct pngb200_png_encoder_desc {
    uint32_t             width, height;
    pngb200_pixel_format format;       /* bgr = 1 writes the ios standard (CgBI chunk, raw deflate) */
    uint8_t              interlaced;
    int32_t              level;        /* 0...13 */
    uint32_t             idat_chunk;   /* bytes per IDAT chunk; 0 = 65544, as pngb200_png_encode_desc */
} pngb200_png_encoder_desc;
/* Validation as pngb200_png_encode_files, plus the size limit above; NULL with the reason in the last error on failure
 * (a bad descriptor or an image over the limit: PNGB200_ERR_BAD_ARGUMENT; no device memory: PNGB200_ERR_CUDA).  The palette is read during the call only. */
pngb200_png_encoder* pngb200_png_encoder_create(pngb200_ctx* ctx, const pngb200_png_encoder_desc* desc);
void                 pngb200_png_encoder_destroy(pngb200_png_encoder* e);
/* `rows`: the next n bytes of storage, a whole number of rows (zero included), in `memspace` (PNGB200_MEM_DEVICE: the
 * context's GPU, read in place).  pngb200_png_encoder_push_batch with one item. */
int  pngb200_png_encoder_push(pngb200_png_encoder* e, const void* rows, size_t n, int memspace);
/* Many pushes in one call, one per encoder.  Each item behaves exactly as the same push made alone: its status,
 * pieces and progress are the ones that push would leave.  Items may mix formats, levels, interlacing, idat_chunk and
 * memspaces.  Returns PNGB200_ERR_BAD_ARGUMENT, touching no item, for a null ctx or array, a null handle, a handle of
 * another ctx, the same handle twice, rows NULL with n > 0, a memspace other than HOST or DEVICE, or a pending decode
 * batch; PNGB200_ERR_CUDA, with every handle unchanged, when a buffer cannot be allocated.  Otherwise each item's
 * status is PNGB200_OK or: PNGB200_ERR_BAD_ARGUMENT for n that is not a whole number of rows, rows past the height,
 * a push after the image is complete, or a push of many non-interlaced rows that completes more than 1 GiB of filtered
 * scanlines (the handle is unchanged: the same rows pushed in smaller bands go through); the handle's sticky error if an earlier push failed on
 * the device; a device error, which then sticks.
 * Cost per call: kernel launches and synchronises are fixed whatever `count` -- at most one filter_resume_kernel, one
 * deflate_resume_kernel and one crc_regions_kernel launch, and at most two stream synchronises.  Copies: one upload of
 * all host rows and one of the launch tables; when new payload bytes were written, one upload of the CRC-32 regions,
 * one clear and one readback of their CRCs; and per item with rows, one device-to-device copy (Adam7: its rows into
 * the handle's storage; otherwise its last row into the carried row, except on the push that completes the image).
 * A device error once the call's buffers are allocated makes every item's handle error sticky. */
typedef struct pngb200_png_encoder_push_desc {
    pngb200_png_encoder* encoder;
    const void*          rows;
    size_t               n;
    int32_t              memspace;    /* pngb200_memspace of `rows` */
    int32_t              status;      /* out */
} pngb200_png_encoder_push_desc;
int  pngb200_png_encoder_push_batch(pngb200_ctx* ctx, pngb200_png_encoder_push_desc* pushes, size_t count);
/* The next piece of the file: returns 1 and sets *bytes / *n (valid until the next call on this handle), or 0 when
 * there is none now (nil). */
int  pngb200_png_encoder_pop(pngb200_png_encoder* e, const uint8_t** bytes, size_t* n);
/* out[0] storage rows received; out[1] scanlines filtered and given to the deflator, in stream order; out[2] filtered
 * bytes the deflator has dequeued; out[3] IDAT chunks handed out by pop(); out[4] 1 once IEND is available; out[5]
 * device bytes the handle holds now. */
int  pngb200_png_encoder_progress(const pngb200_png_encoder* e, uint64_t out[6]);
/* the sticky device error (PNGB200_OK if none); a and b are 0 (kept for the shape of the other handles' calls) */
void pngb200_png_encoder_error(const pngb200_png_encoder* e, int* status, uint32_t* a, uint32_t* b);

/* ---- cloning handles: LZ77.Inflator, LZ77.Deflator, PNG.Context and PNG.Encoder are values ----------------------------
 * In the reference these types are structs whose buffers are copied on write (exclude(), LZ77.InflatorBuffers.swift,
 * LZ77.DeflatorIn.swift, LZ77.DeflatorOut.swift), so after `var b = a` a push into `a` never changes `b`.  A clone is
 * that copy, made eagerly: a new handle of the source's type on the same ctx, with its own device buffers.
 * The contract: take a clone made from source S and any later sequence of calls on it.  Each call returns exactly what
 * the same call on S would have returned at the moment of cloning: statuses and error payloads, available / pull /
 * pull_all, pop and pull blocks, progress (all six values of a context, the band included), storage bytes, encoder
 * pieces and stats() -- except the device bytes a handle holds (pngb200_deflator_stats out[3],
 * pngb200_png_encoder_progress out[5]): a clone holds no launch scratch and only the bytes in use, so right after the
 * clone it holds at most what the source holds, and later pushes grow it from there.  After the clone,
 * no call on either handle changes anything the other returns.  This holds for terminal handles, handles with a sticky
 * error (the clone keeps it), deflators after `last`, and encoders with pieces not yet popped (each handle pops its own
 * copy).  A context clone's storage starts as the bytes of the source's storage; `pixels` must stay valid while the
 * clone lives, as the storage given to pngb200_png_context_create.
 * Rejections, PNGB200_ERR_BAD_ARGUMENT before any work with every `clone` left NULL: a null ctx, or a null array with
 * count > 0; an item whose number of non-null source fields is not exactly one; a source of another ctx; a context
 * item with null `pixels`, a `pixels_cap` below the source's storage bytes, or storage bytes at `pixels` that overlap
 * the source's storage; a call while a decode batch is pending on the ctx.  The same source may appear twice: it gets
 * two clones.
 * All or nothing: if an allocation or a copy fails the call returns PNGB200_ERR_CUDA, every clone it made is destroyed
 * (each `clone` NULL) and every source is unchanged.
 * Fixed cost, whatever `count`: one upload of the copy list, at most one segment_copy_kernel launch (every source's
 * device bytes in use, into freshly allocated buffers) and one stream synchronise.  Host state (queues, tails, a
 * buffered deflator's input, host storage) is copied on the host; a call whose items hold no device bytes (fresh
 * handles, buffered deflators) makes no launch.  A clone's device buffers are those create gives a handle, plus the
 * bytes in use of the buffers pushes grow (an inflator's output keeps the source's capacity, which decides when the
 * decoder stops to grow it); the next push grows them as it would on any handle. */
typedef struct pngb200_clone_desc {
    pngb200_inflator*    inflator;
    pngb200_deflator*    deflator;     /* online or buffered */
    pngb200_png_context* context;
    pngb200_png_encoder* encoder;
    void*                pixels;       /* context only: the clone's storage, in the source's memspace, any alignment */
    size_t               pixels_cap;   /* >= the source's storage bytes */
    void*                clone;        /* out: a handle of the source's type on the same ctx */
} pngb200_clone_desc;
int pngb200_clone_batch(pngb200_ctx* ctx, pngb200_clone_desc* items, size_t count);
/* the bytes the last successful pngb200_clone_batch on `ctx` copied: out[0] device bytes (its one launch), out[1] host
 * bytes (queues, tails, buffered input, host storage); both 0 after a call that failed */
int pngb200_ctx_clone_stats(pngb200_ctx* ctx, uint64_t out[2]);
/* pngb200_clone_batch with one item: the clone, or NULL with the reason in pngb200_last_error */
pngb200_inflator*    pngb200_inflator_clone(const pngb200_inflator* z);
pngb200_deflator*    pngb200_deflator_clone(const pngb200_deflator* z);
pngb200_png_context* pngb200_png_context_clone(const pngb200_png_context* c, void* pixels, size_t pixels_cap);
pngb200_png_encoder* pngb200_png_encoder_clone(const pngb200_png_encoder* e);

#ifdef __cplusplus
}
#endif
#endif /* PNGB200_H */
