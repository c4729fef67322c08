"""swift-png_b200: H100-native PNG hot path (DEFLATE inflate + scanline unfilter, filter-select)
behind swift-png's `PNG.Decoder` / `PNG.Encoder` / `LZ77.Inflator` interface.

This module is the thin host-side binding of the C ABI in include/pngb200.h (ctypes; the
library itself has no Python or torch dependency).  It mirrors the reference's names:

    LZ77.Inflator(format:).push/pull      -> Inflator(ctx, format).push / .pull / .pull_all
    Gzip.extract(from:)                   -> gzip_extract(ctx, data)
    PNG.Decoder.push + PNG.Image.assign   -> decode_batch(ctx, [ImageJob...])
    PNG.Encoder.filter (+ collect)        -> filter_batch(ctx, [...])

There is NO CPU fallback: importing works anywhere (so the symbol table can be checked without a
GPU) but creating a Context raises unless an sm_90 GPU (H100) and the in-tree libpngb200.so exist.
"""
from __future__ import annotations

import ctypes as C
import importlib.util
import os
from dataclasses import dataclass

from . import shard  # noqa: F401  (multi-GPU partitioning helpers)

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PNGB200_LIB") or os.path.join(_HERE, "libpngb200.so")  # override: tuning experiments only
HEADER_PATH = os.path.join(_HERE, "..", "include", "pngb200.h")

# pngb200_status
OK = 0
NEED_MORE_INPUT = 1
ERR_STREAM_CHECKSUM = -1
ERR_BLOCK_TYPE = -2
ERR_BLOCK_COUNT_PARITY = -3
ERR_RUNLITERAL_SYMBOL_COUNT = -4
ERR_CODELENGTH_HUFFMAN_TABLE = -5
ERR_CODELENGTH_SEQUENCE = -6
ERR_HUFFMAN_TABLE = -7
ERR_STRING_REFERENCE = -8
ERR_INVALID_SYMBOL = -9
ERR_ZLIB_METHOD = -16
ERR_ZLIB_WINDOW = -17
ERR_ZLIB_CHECK_BITS = -18
ERR_ZLIB_DICTIONARY = -19
ERR_GZIP_SIGIL = -32
ERR_GZIP_METHOD = -33
ERR_GZIP_FLAG_BITS = -34
ERR_GZIP_HEADER_CHECKSUM_UNSUPPORTED = -35
ERR_PNG_EXTRANEOUS_IMAGE_DATA = -48
ERR_PNG_EXTRANEOUS_COMPRESSED_DATA = -49
ERR_PNG_INCOMPLETE_DATASTREAM = -50
ERR_LEX_TRUNCATED_SIGNATURE, ERR_LEX_INVALID_SIGNATURE, ERR_LEX_TRUNCATED_CHUNK_HEADER = -80, -81, -82
ERR_LEX_TRUNCATED_CHUNK_BODY, ERR_LEX_INVALID_CHUNK_TYPE, ERR_LEX_INVALID_CHUNK_CHECKSUM = -83, -84, -85
ERR_PARSE_HEADER_CHUNK_LENGTH, ERR_PARSE_HEADER_PIXEL_FORMAT_CODE, ERR_PARSE_HEADER_PIXEL_FORMAT = -96, -97, -98
ERR_PARSE_HEADER_COMPRESSION_CODE, ERR_PARSE_HEADER_FILTER_CODE, ERR_PARSE_HEADER_INTERLACING_CODE = -99, -100, -101
ERR_PARSE_HEADER_SIZE, ERR_PARSE_UNEXPECTED_PALETTE, ERR_PARSE_PALETTE_CHUNK_LENGTH = -102, -103, -104
ERR_PARSE_PALETTE_COUNT, ERR_PARSE_UNEXPECTED_TRANSPARENCY, ERR_PARSE_TRANSPARENCY_CHUNK_LENGTH = -105, -106, -107
ERR_PARSE_TRANSPARENCY_SAMPLE, ERR_PARSE_TRANSPARENCY_COUNT = -108, -109
ERR_DECODE_REQUIRED_CHUNK, ERR_DECODE_DUPLICATE_CHUNK, ERR_DECODE_UNEXPECTED_CHUNK = -112, -113, -114
ERR_OUTPUT_CAPACITY = -64
ERR_BAD_ARGUMENT = -65
ERR_CUDA = -66
ERR_INTERNAL = -67

FORMAT_ZLIB, FORMAT_IOS, FORMAT_GZIP = 0, 1, 2
MEM_HOST, MEM_DEVICE = 0, 1


class StreamDesc(C.Structure):
    _fields_ = [
        ("src", C.c_void_p), ("src_len", C.c_size_t),
        ("dst", C.c_void_p), ("dst_cap", C.c_size_t),
        ("format", C.c_int32),
        ("status", C.c_int32), ("err_a", C.c_uint32), ("err_b", C.c_uint32),
        ("checksum", C.c_uint32), ("blocks", C.c_uint32),
        ("produced", C.c_uint64), ("consumed_bits", C.c_uint64),
    ]


class ImageDesc(C.Structure):
    _fields_ = [
        ("idat", C.c_void_p), ("idat_len", C.c_size_t),
        ("pixels", C.c_void_p), ("pixels_cap", C.c_size_t),
        ("width", C.c_uint32), ("height", C.c_uint32),
        ("volume", C.c_uint8), ("depth", C.c_uint8), ("interlaced", C.c_uint8), ("format", C.c_uint8),
        ("status", C.c_int32), ("err_a", C.c_uint32), ("err_b", C.c_uint32),
        ("checksum", C.c_uint32), ("blocks", C.c_uint32),
        ("produced", C.c_uint64),
    ]


class FilterDesc(C.Structure):
    _fields_ = [
        ("pixels", C.c_void_p), ("pixels_len", C.c_size_t),
        ("filtered", C.c_void_p), ("filtered_cap", C.c_size_t),
        ("width", C.c_uint32), ("height", C.c_uint32),
        ("volume", C.c_uint8), ("depth", C.c_uint8), ("interlaced", C.c_uint8), ("reserved", C.c_uint8),
        ("status", C.c_int32), ("produced", C.c_uint64),
    ]


class DeflateDesc(C.Structure):
    _fields_ = [
        ("src", C.c_void_p), ("src_len", C.c_size_t),
        ("dst", C.c_void_p), ("dst_cap", C.c_size_t),
        ("format", C.c_int32), ("level", C.c_int32), ("exponent", C.c_int32),
        ("status", C.c_int32), ("checksum", C.c_uint32), ("blocks", C.c_uint32),
        ("produced", C.c_uint64),
    ]


class EncodeDesc(C.Structure):
    _fields_ = [
        ("pixels", C.c_void_p), ("pixels_len", C.c_size_t),
        ("idat", C.c_void_p), ("idat_cap", C.c_size_t),
        ("width", C.c_uint32), ("height", C.c_uint32),
        ("volume", C.c_uint8), ("depth", C.c_uint8), ("interlaced", C.c_uint8), ("format", C.c_uint8),
        ("level", C.c_int32), ("status", C.c_int32), ("checksum", C.c_uint32), ("blocks", C.c_uint32),
        ("produced", C.c_uint64),
    ]


TARGET_RGBA8, TARGET_RGBA16, TARGET_VA8, TARGET_VA16 = 0, 1, 2, 3
TARGET_RGBA32, TARGET_RGBA64, TARGET_VA32, TARGET_VA64 = 4, 5, 6, 7
TARGET_V8, TARGET_V16, TARGET_V32, TARGET_V64 = 8, 9, 10, 11  # image.unpack(as: UInt8.self) ... UInt64
ALPHA_ASIS, ALPHA_PREMULTIPLIED, ALPHA_STRAIGHTENED, ALPHA_PREMULTIPLIED_AS8, ALPHA_STRAIGHTENED_AS8 = range(5)
ALPHA_PREMULTIPLIED_AS16, ALPHA_STRAIGHTENED_AS16, ALPHA_PREMULTIPLIED_AS32, ALPHA_STRAIGHTENED_AS32 = 5, 6, 7, 8
ERR_PNG_PALETTE_INDEX = -51
_TARGET_BYTES = {TARGET_RGBA8: 4, TARGET_RGBA16: 8, TARGET_VA8: 2, TARGET_VA16: 4,
                 TARGET_RGBA32: 16, TARGET_RGBA64: 32, TARGET_VA32: 8, TARGET_VA64: 16,
                 TARGET_V8: 1, TARGET_V16: 2, TARGET_V32: 4, TARGET_V64: 8}
_CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


class PixelFormat(C.Structure):
    """pngb200_pixel_format: PNG.Format as the colour-target kernels see it."""
    _fields_ = [
        ("color", C.c_uint8), ("depth", C.c_uint8), ("bgr", C.c_uint8), ("has_key", C.c_uint8),
        ("key", C.c_uint16 * 3), ("palette_count", C.c_uint16), ("palette", C.c_void_p),
    ]


class ColorDesc(C.Structure):
    _fields_ = [
        ("storage", C.c_void_p), ("storage_len", C.c_size_t),
        ("pixels", C.c_void_p), ("pixels_len", C.c_size_t),
        ("count", C.c_uint64), ("format", PixelFormat), ("status", C.c_int32),
    ]


class PngDesc(C.Structure):
    """pngb200_png_desc"""
    _fields_ = [
        ("file", C.c_void_p), ("file_len", C.c_size_t), ("pixels", C.c_void_p), ("pixels_cap", C.c_size_t),
        ("width", C.c_uint32), ("height", C.c_uint32),
        ("depth", C.c_uint8), ("color", C.c_uint8), ("interlaced", C.c_uint8), ("standard", C.c_uint8),
        ("format", PixelFormat), ("palette_rgba", C.c_uint8 * 1024),
        ("storage_size", C.c_uint64), ("idat_bytes", C.c_uint64), ("idat_chunks", C.c_uint32), ("chunks", C.c_uint32),
        ("status", C.c_int32), ("err_a", C.c_uint32), ("err_b", C.c_uint32),
        ("checksum", C.c_uint32), ("blocks", C.c_uint32), ("produced", C.c_uint64),
    ]


class PngEncodeDesc(C.Structure):
    """pngb200_png_encode_desc"""
    _fields_ = [
        ("pixels", C.c_void_p), ("pixels_len", C.c_size_t), ("width", C.c_uint32), ("height", C.c_uint32),
        ("format", PixelFormat), ("interlaced", C.c_uint8), ("level", C.c_int32), ("idat_chunk", C.c_uint32),
        ("file", C.c_void_p), ("file_cap", C.c_size_t),
        ("status", C.c_int32), ("checksum", C.c_uint32), ("blocks", C.c_uint32), ("produced", C.c_uint64),
    ]


class PngContextDesc(C.Structure):
    _fields_ = [
        ("pixels", C.c_void_p), ("pixels_cap", C.c_size_t), ("width", C.c_uint32), ("height", C.c_uint32),
        ("volume", C.c_uint8), ("depth", C.c_uint8), ("interlaced", C.c_uint8), ("standard", C.c_uint8),
        ("memspace", C.c_int32),
    ]


class DeflatorPushDesc(C.Structure):
    _fields_ = [("deflator", C.c_void_p), ("data", C.c_void_p), ("n", C.c_size_t), ("last", C.c_int32),
                ("status", C.c_int32)]


class InflatorPushDesc(C.Structure):
    _fields_ = [("inflator", C.c_void_p), ("data", C.c_void_p), ("n", C.c_size_t), ("status", C.c_int32)]


class PngPushDesc(C.Structure):
    _fields_ = [("context", C.c_void_p), ("data", C.c_void_p), ("n", C.c_size_t), ("overdraw", C.c_int32),
                ("status", C.c_int32)]


class PngEncoderDesc(C.Structure):
    _fields_ = [("width", C.c_uint32), ("height", C.c_uint32), ("format", PixelFormat), ("interlaced", C.c_uint8),
                ("level", C.c_int32), ("idat_chunk", C.c_uint32)]


class PngEncoderPushDesc(C.Structure):
    _fields_ = [("encoder", C.c_void_p), ("rows", C.c_void_p), ("n", C.c_size_t), ("memspace", C.c_int32),
                ("status", C.c_int32)]


class CloneDesc(C.Structure):
    _fields_ = [("inflator", C.c_void_p), ("deflator", C.c_void_p), ("context", C.c_void_p), ("encoder", C.c_void_p),
                ("pixels", C.c_void_p), ("pixels_cap", C.c_size_t), ("clone", C.c_void_p)]


class PNGB200Error(RuntimeError):
    def __init__(self, status: int, message: str = ""):
        super().__init__(f"pngb200 status {status}: {message}")
        self.status = status


_lib = None


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile the CUDA library in-tree (nvcc, sm_90a).  Works without a GPU."""
    spec = importlib.util.spec_from_file_location("_pngb200_build", os.path.join(_HERE, "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build(force=force, verbose=verbose)


def lib():
    """Load libpngb200.so (raises if it has not been built: there is no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PNGB200Error(ERR_CUDA, f"{LIB_PATH} is missing: run `python __graft_entry__.py build`; "
                           "there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    L.pngb200_ctx_create.argtypes = [C.c_int]
    L.pngb200_ctx_create.restype = C.c_void_p
    L.pngb200_ctx_destroy.argtypes = [C.c_void_p]
    L.pngb200_ctx_destroy.restype = None
    L.pngb200_unpack_batch.argtypes = [C.c_void_p, C.POINTER(ColorDesc), C.c_size_t, C.c_int, C.c_int, C.c_int]
    L.pngb200_unpack_batch.restype = C.c_int
    L.pngb200_pack_batch.argtypes = [C.c_void_p, C.POINTER(ColorDesc), C.c_size_t, C.c_int, C.c_int]
    L.pngb200_pack_batch.restype = C.c_int
    L.pngb200_png_inspect_batch.argtypes = [C.POINTER(PngDesc), C.c_size_t]
    L.pngb200_png_inspect_batch.restype = C.c_int
    L.pngb200_png_decode_batch.argtypes = [C.c_void_p, C.POINTER(PngDesc), C.c_size_t, C.c_int]
    L.pngb200_png_decode_batch.restype = C.c_int
    L.pngb200_png_encode_bound.argtypes = [C.c_uint32, C.c_uint32, C.POINTER(PixelFormat), C.c_int, C.c_uint32]
    L.pngb200_png_encode_bound.restype = C.c_size_t
    L.pngb200_png_encode_batch.argtypes = [C.c_void_p, C.POINTER(PngEncodeDesc), C.c_size_t, C.c_int]
    L.pngb200_png_encode_batch.restype = C.c_int
    L.pngb200_png_inspect_files.argtypes = [C.c_void_p, C.POINTER(PngDesc), C.c_size_t, C.c_int]
    L.pngb200_png_inspect_files.restype = C.c_int
    L.pngb200_png_decode_files.argtypes = [C.c_void_p, C.POINTER(PngDesc), C.c_size_t, C.c_int, C.c_int]
    L.pngb200_png_decode_files.restype = C.c_int
    L.pngb200_png_encode_files.argtypes = [C.c_void_p, C.POINTER(PngEncodeDesc), C.c_size_t, C.c_int, C.c_int]
    L.pngb200_png_encode_files.restype = C.c_int
    L.pngb200_ctx_trim.argtypes = [C.c_void_p]
    L.pngb200_ctx_trim.restype = C.c_int
    L.pngb200_last_error.argtypes = [C.c_void_p]
    L.pngb200_last_error.restype = C.c_char_p
    L.pngb200_ctx_stream.argtypes = [C.c_void_p]
    L.pngb200_ctx_stream.restype = C.c_void_p
    L.pngb200_ctx_device.argtypes = [C.c_void_p]
    L.pngb200_ctx_device.restype = C.c_int
    L.pngb200_ctx_launch_count.argtypes = [C.c_void_p]
    L.pngb200_ctx_launch_count.restype = C.c_uint64
    L.pngb200_ctx_set_inflate_mode.argtypes = [C.c_void_p, C.c_int]
    L.pngb200_ctx_set_inflate_mode.restype = None
    L.pngb200_ctx_stage_ms.argtypes = [C.c_void_p, C.POINTER(C.c_float)]
    L.pngb200_ctx_stage_ms.restype = C.c_int
    L.pngb200_ctx_inflate_stats.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64)]
    L.pngb200_ctx_inflate_stats.restype = C.c_int
    L.pngb200_deflator_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_size_t]
    L.pngb200_deflator_create.restype = C.c_void_p
    if os.environ.get("PNGB200_LIB") is None or hasattr(L, "pngb200_deflator_create_online"):   # (older builds lack it)
        L.pngb200_deflator_create_online.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_size_t]
        L.pngb200_deflator_create_online.restype = C.c_void_p
        L.pngb200_deflator_push_batch.argtypes = [C.c_void_p, C.POINTER(DeflatorPushDesc), C.c_size_t]
        L.pngb200_deflator_push_batch.restype = C.c_int
        L.pngb200_deflator_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.pngb200_deflator_stats.restype = C.c_int
    L.pngb200_deflator_destroy.argtypes = [C.c_void_p]
    L.pngb200_deflator_destroy.restype = None
    L.pngb200_deflator_push.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int]
    L.pngb200_deflator_push.restype = C.c_int
    for fn in (L.pngb200_deflator_pop, L.pngb200_deflator_pull):
        fn.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)]
        fn.restype = C.c_int
    L.pngb200_ctx_filter_histogram.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    L.pngb200_ctx_filter_histogram.restype = C.c_int
    L.pngb200_ctx_segment_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
    L.pngb200_ctx_segment_stats.restype = C.c_int
    if os.environ.get("PNGB200_LIB") is None or hasattr(L, "pngb200_ctx_unfilter_stats"):   # (older builds lack it)
        L.pngb200_ctx_unfilter_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.pngb200_ctx_unfilter_stats.restype = C.c_int
    if os.environ.get("PNGB200_LIB") is None or hasattr(L, "pngb200_ctx_split_stats"):   # (older tuning builds lack it)
        L.pngb200_ctx_split_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.pngb200_ctx_split_stats.restype = C.c_int
    if os.environ.get("PNGB200_LIB") is None or hasattr(L, "pngb200_ctx_last_inflate_engine"):   # (older tuning builds lack it)
        L.pngb200_ctx_last_inflate_engine.argtypes = [C.c_void_p]
        L.pngb200_ctx_last_inflate_engine.restype = C.c_int
    L.pngb200_ctx_inflate_counters.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64)]
    L.pngb200_ctx_inflate_counters.restype = C.c_int
    L.pngb200_inflate_batch.argtypes = [C.c_void_p, C.POINTER(StreamDesc), C.c_size_t, C.c_int]
    L.pngb200_inflate_batch.restype = C.c_int
    for name in ("pngb200_decode_batch", "pngb200_decode_batch_enqueue", "pngb200_unfilter_batch"):
        getattr(L, name).argtypes = [C.c_void_p, C.POINTER(ImageDesc), C.c_size_t, C.c_int]
        getattr(L, name).restype = C.c_int
    L.pngb200_decode_batch_finish.argtypes = [C.c_void_p, C.POINTER(ImageDesc), C.c_size_t]
    L.pngb200_decode_batch_finish.restype = C.c_int
    L.pngb200_filter_batch.argtypes = [C.c_void_p, C.POINTER(FilterDesc), C.c_size_t, C.c_int]
    L.pngb200_filter_batch.restype = C.c_int
    L.pngb200_deflate_batch.argtypes = [C.c_void_p, C.POINTER(DeflateDesc), C.c_size_t, C.c_int]
    L.pngb200_deflate_batch.restype = C.c_int
    L.pngb200_deflate_bound.argtypes = [C.c_size_t]
    L.pngb200_deflate_bound.restype = C.c_size_t
    L.pngb200_encode_batch.argtypes = [C.c_void_p, C.POINTER(EncodeDesc), C.c_size_t, C.c_int]
    L.pngb200_encode_batch.restype = C.c_int
    L.pngb200_filtered_size.argtypes = [C.c_uint32, C.c_uint32, C.c_int, C.c_int]
    L.pngb200_filtered_size.restype = C.c_size_t
    L.pngb200_storage_size.argtypes = [C.c_uint32, C.c_uint32, C.c_int]
    L.pngb200_storage_size.restype = C.c_size_t
    L.pngb200_inflator_create.argtypes = [C.c_void_p, C.c_int]
    L.pngb200_inflator_create.restype = C.c_void_p
    L.pngb200_inflator_destroy.argtypes = [C.c_void_p]
    L.pngb200_inflator_destroy.restype = None
    L.pngb200_inflator_push.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t]
    L.pngb200_inflator_push.restype = C.c_int
    L.pngb200_inflator_pull.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pngb200_inflator_pull.restype = C.c_int
    L.pngb200_inflator_pull_all.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pngb200_inflator_pull_all.restype = C.c_size_t
    L.pngb200_inflator_available.argtypes = [C.c_void_p]
    L.pngb200_inflator_available.restype = C.c_size_t
    L.pngb200_inflator_error.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_uint32),
                                         C.POINTER(C.c_uint32)]
    L.pngb200_inflator_error.restype = None
    if os.environ.get("PNGB200_LIB") is None or hasattr(L, "pngb200_inflator_stats"):   # (older builds lack it)
        L.pngb200_inflator_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.pngb200_inflator_stats.restype = C.c_int
    if os.environ.get("PNGB200_LIB") is None or hasattr(L, "pngb200_png_context_create"):   # (older builds lack it)
        L.pngb200_png_context_create.argtypes = [C.c_void_p, C.POINTER(PngContextDesc)]
        L.pngb200_png_context_create.restype = C.c_void_p
        L.pngb200_png_context_push.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int]
        L.pngb200_png_context_push.restype = C.c_int
        L.pngb200_png_context_end.argtypes = [C.c_void_p]
        L.pngb200_png_context_end.restype = C.c_int
        L.pngb200_png_context_progress.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.pngb200_png_context_progress.restype = C.c_int
        L.pngb200_png_context_error.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_uint32),
                                                C.POINTER(C.c_uint32)]
        L.pngb200_png_context_error.restype = None
        L.pngb200_png_context_destroy.argtypes = [C.c_void_p]
        L.pngb200_png_context_destroy.restype = None
    if os.environ.get("PNGB200_LIB") is None or hasattr(L, "pngb200_png_context_push_batch"):   # (older builds lack it)
        L.pngb200_inflator_push_batch.argtypes = [C.c_void_p, C.POINTER(InflatorPushDesc), C.c_size_t]
        L.pngb200_inflator_push_batch.restype = C.c_int
        L.pngb200_png_context_push_batch.argtypes = [C.c_void_p, C.POINTER(PngPushDesc), C.c_size_t]
        L.pngb200_png_context_push_batch.restype = C.c_int
    if hasattr(L, "pngb200_png_encoder_create"):
        L.pngb200_png_encoder_create.argtypes = [C.c_void_p, C.POINTER(PngEncoderDesc)]
        L.pngb200_png_encoder_create.restype = C.c_void_p
        L.pngb200_png_encoder_destroy.argtypes = [C.c_void_p]
        L.pngb200_png_encoder_destroy.restype = None
        L.pngb200_png_encoder_push.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int]
        L.pngb200_png_encoder_push.restype = C.c_int
        L.pngb200_png_encoder_push_batch.argtypes = [C.c_void_p, C.POINTER(PngEncoderPushDesc), C.c_size_t]
        L.pngb200_png_encoder_push_batch.restype = C.c_int
        L.pngb200_png_encoder_pop.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(C.c_size_t)]
        L.pngb200_png_encoder_pop.restype = C.c_int
        L.pngb200_png_encoder_progress.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.pngb200_png_encoder_progress.restype = C.c_int
        L.pngb200_png_encoder_error.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_uint32),
                                                C.POINTER(C.c_uint32)]
        L.pngb200_png_encoder_error.restype = None
    if hasattr(L, "pngb200_clone_batch"):
        L.pngb200_clone_batch.argtypes = [C.c_void_p, C.POINTER(CloneDesc), C.c_size_t]
        L.pngb200_clone_batch.restype = C.c_int
        for name in ("inflator", "deflator", "png_encoder"):
            getattr(L, f"pngb200_{name}_clone").argtypes = [C.c_void_p]
            getattr(L, f"pngb200_{name}_clone").restype = C.c_void_p
        L.pngb200_png_context_clone.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
        L.pngb200_png_context_clone.restype = C.c_void_p
        L.pngb200_ctx_clone_stats.argtypes = [C.c_void_p, C.POINTER(C.c_uint64)]
        L.pngb200_ctx_clone_stats.restype = C.c_int
    _lib = L
    return L


def filtered_size(w: int, h: int, volume: int, interlaced: bool = False) -> int:
    return lib().pngb200_filtered_size(w, h, volume, int(interlaced))


def storage_size(w: int, h: int, volume: int) -> int:
    return lib().pngb200_storage_size(w, h, volume)


class Context:
    """One GPU: a CUDA stream plus grow-only workspaces (pngb200_ctx)."""

    def __init__(self, device: int = -1):
        self._lib = lib()
        self.handle = self._lib.pngb200_ctx_create(device)
        if not self.handle:
            raise PNGB200Error(ERR_CUDA, self._lib.pngb200_last_error(None).decode())

    def close(self):
        if getattr(self, "handle", None):
            self._lib.pngb200_ctx_destroy(self.handle)
            self.handle = None

    __del__ = close

    def trim(self):
        """Give the grow-only device arenas back to the driver (pngb200_ctx_trim)."""
        self.check(self._lib.pngb200_ctx_trim(self.handle))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    @property
    def stream(self) -> int:
        return self._lib.pngb200_ctx_stream(self.handle) or 0

    @property
    def device(self) -> int:
        return self._lib.pngb200_ctx_device(self.handle)

    @property
    def launches(self) -> int:
        return self._lib.pngb200_ctx_launch_count(self.handle)

    def stage_ms(self):
        """(inflate, checksum, unfilter) device milliseconds of the last finished decode batch"""
        ms = (C.c_float * 3)()
        self.check(self._lib.pngb200_ctx_stage_ms(self.handle, ms))
        return tuple(ms)

    def inflate_stats(self, count: int):
        """dict of device-side counters summed over the last batch of `count` items"""
        out = (C.c_uint64 * 4)()
        self.check(self._lib.pngb200_ctx_inflate_stats(self.handle, count, out))
        return dict(waves=out[0], sync_rounds=out[1], resolve_rounds=out[2], fallbacks=out[3])

    def inflate_counters(self, count: int):
        """all device-side counters of the last batch (see pngb200_ctx_inflate_counters)"""
        out = (C.c_uint64 * 24)()
        self.check(self._lib.pngb200_ctx_inflate_counters(self.handle, count, out))
        names = ["header_tables", "stage", "speculate", "walk", "chain", "count_scan", "emit", "resolve", "store",
                 "stored_blocks"]
        return dict(waves=out[0], walk_tokens=out[1], resolve_rounds=out[2], fallbacks=out[3], tokens=out[4],
                    matches=out[5], deferred_matches=out[6], blocks=out[7],
                    cycles={n: out[8 + i] for i, n in enumerate(names)})

    def filter_histogram(self):
        """scanlines per filter type (None, Sub, Up, Average, Paeth, invalid) of the last wavefront-unfilter batch"""
        out = (C.c_uint64 * 6)()
        self.check(self._lib.pngb200_ctx_filter_histogram(self.handle, out))
        return list(out)

    def segment_stats(self):
        """(streams cut into segments, segments, streams decoded whole after all) of the last batch"""
        out = (C.c_uint64 * 3)()
        self.check(self._lib.pngb200_ctx_segment_stats(self.handle, out))
        return dict(streams=out[0], segments=out[1], fallbacks=out[2])

    def unfilter_stats(self):
        """images of the last decode / unfilter batch by unfilter path: the wavefront kernel (non-interlaced, >= 8 bits),
        the pass path (Adam7 and 1/2/4-bit images past 64 KiB of filtered stream) and the one-CTA generic kernel"""
        out = (C.c_uint64 * 3)()
        self.check(self._lib.pngb200_ctx_unfilter_stats(self.handle, out))
        return dict(wavefront=out[0], passes=out[1], generic=out[2])

    def clone_stats(self):
        """(device bytes, host bytes) the last clone_batch on this context copied (see pngb200_ctx_clone_stats)"""
        out = (C.c_uint64 * 2)()
        self.check(self._lib.pngb200_ctx_clone_stats(self.handle, out))
        return out[0], out[1]

    def split_stats(self):
        """bytes and SM cycles of the heads and tails of the streams the last batch cut in two, the tails that left
        symbolic mode and the tails' bytes decoded as symbols (see pngb200_ctx_split_stats)"""
        out = (C.c_uint64 * 6)()
        self.check(self._lib.pngb200_ctx_split_stats(self.handle, out))
        return dict(head_bytes=out[0], head_cycles=out[1], tail_bytes=out[2], tail_cycles=out[3], switched=out[4],
                    symbolic_bytes=out[5])

    def last_inflate_engine(self) -> str:
        """kernel name of the whole-stream inflate engine the last batch used ('' when none ran)"""
        if not hasattr(self._lib, "pngb200_ctx_last_inflate_engine"):
            return ""
        return {0: "inflate_parallel_kernel", 1: "inflate_wave_kernel", 2: "inflate_cells_kernel"}.get(
            self._lib.pngb200_ctx_last_inflate_engine(self.handle), "")

    def set_inflate_mode(self, mode: int):
        self._lib.pngb200_ctx_set_inflate_mode(self.handle, mode)

    def check(self, rc: int):
        if rc != OK:
            raise PNGB200Error(rc, self._lib.pngb200_last_error(self.handle).decode())


@dataclass
class DecodedImage:
    status: int
    pixels: bytes
    checksum: int
    produced: int
    blocks: int
    err_a: int = 0
    err_b: int = 0


def _buf_addr(b) -> int:
    return C.addressof(b)


def inflate_batch(ctx: Context, streams, fmt: int = FORMAT_ZLIB, caps=None):
    """LZ77.Inflator one-shot over a batch of host byte strings.
    Returns a list of (status, bytes, StreamDesc)."""
    n = len(streams)
    descs = (StreamDesc * n)()
    keep = []
    for i, s in enumerate(streams):
        cap = caps[i] if caps is not None else max(len(s) * 1100 + 1024, 1024)
        src = C.create_string_buffer(bytes(s), len(s)) if len(s) else C.create_string_buffer(1)
        dst = C.create_string_buffer(max(cap, 1))
        keep.append((src, dst))
        descs[i].src = _buf_addr(src)
        descs[i].src_len = len(s)
        descs[i].dst = _buf_addr(dst)
        descs[i].dst_cap = cap
        descs[i].format = fmt if isinstance(fmt, int) else fmt[i]
    ctx.check(ctx._lib.pngb200_inflate_batch(ctx.handle, descs, n, MEM_HOST))
    return [(descs[i].status, keep[i][1].raw[: descs[i].produced], descs[i]) for i in range(n)]


def gzip_extract(ctx: Context, data: bytes, cap: int | None = None) -> bytes:
    """Gzip.extract(from:)"""
    (st, out, d), = inflate_batch(ctx, [data], FORMAT_GZIP, None if cap is None else [cap])
    if st != OK:
        raise PNGB200Error(st, "gzip_extract")
    return out


def decode_batch(ctx: Context, images, memspace: int = MEM_HOST):
    """PNG.Decoder over a batch.  `images`: iterable of dicts/objects with
    idat (bytes), width, height, volume, depth, interlaced, fmt.  Host memory path."""
    images = list(images)
    n = len(images)
    descs = (ImageDesc * n)()
    keep = []
    for i, im in enumerate(images):
        g = im if isinstance(im, dict) else im.__dict__
        idat = bytes(g["idat"])
        w, h, vol = g["width"], g["height"], g["volume"]
        size = storage_size(w, h, vol)
        src = C.create_string_buffer(idat, len(idat)) if len(idat) else C.create_string_buffer(1)
        dst = C.create_string_buffer(max(size, 1))
        keep.append((src, dst, size))
        descs[i].idat = _buf_addr(src)
        descs[i].idat_len = len(idat)
        descs[i].pixels = _buf_addr(dst)
        descs[i].pixels_cap = size
        descs[i].width, descs[i].height = w, h
        descs[i].volume, descs[i].depth = vol, g["depth"]
        descs[i].interlaced = int(bool(g.get("interlaced", False)))
        descs[i].format = g.get("fmt", FORMAT_ZLIB)
    ctx.check(ctx._lib.pngb200_decode_batch(ctx.handle, descs, n, memspace))
    return [DecodedImage(descs[i].status, keep[i][1].raw[: keep[i][2]], descs[i].checksum,
                         descs[i].produced, descs[i].blocks, descs[i].err_a, descs[i].err_b)
            for i in range(n)]


def unfilter_batch(ctx: Context, images):
    """PNG.Decoder.defilter + PNG.Image.assign over already inflated streams
    (`filtered` bytes per image).  Returns list of (status, pixels)."""
    images = list(images)
    n = len(images)
    descs = (ImageDesc * n)()
    keep = []
    for i, g in enumerate(images):
        f = bytes(g["filtered"])
        w, h, vol = g["width"], g["height"], g["volume"]
        size = storage_size(w, h, vol)
        src = C.create_string_buffer(f, len(f)) if len(f) else C.create_string_buffer(1)
        dst = C.create_string_buffer(max(size, 1))
        keep.append((src, dst, size))
        descs[i].idat = _buf_addr(src)
        descs[i].idat_len = len(f)
        descs[i].pixels = _buf_addr(dst)
        descs[i].pixels_cap = size
        descs[i].width, descs[i].height = w, h
        descs[i].volume, descs[i].depth = vol, g["depth"]
        descs[i].interlaced = int(bool(g.get("interlaced", False)))
    ctx.check(ctx._lib.pngb200_unfilter_batch(ctx.handle, descs, n, MEM_HOST))
    return [(descs[i].status, keep[i][1].raw[: keep[i][2]]) for i in range(n)]


def filter_batch(ctx: Context, images):
    """PNG.Image.collect + PNG.Encoder.filter over a batch of storages.  Returns list of bytes."""
    images = list(images)
    n = len(images)
    descs = (FilterDesc * n)()
    keep = []
    for i, g in enumerate(images):
        px = bytes(g["pixels"])
        w, h, vol = g["width"], g["height"], g["volume"]
        il = bool(g.get("interlaced", False))
        fsz = filtered_size(w, h, vol, il)
        src = C.create_string_buffer(px, len(px))
        dst = C.create_string_buffer(max(fsz, 1))
        keep.append((src, dst, fsz))
        descs[i].pixels = _buf_addr(src)
        descs[i].pixels_len = len(px)
        descs[i].filtered = _buf_addr(dst)
        descs[i].filtered_cap = fsz
        descs[i].width, descs[i].height = w, h
        descs[i].volume, descs[i].depth, descs[i].interlaced = vol, g["depth"], int(il)
    ctx.check(ctx._lib.pngb200_filter_batch(ctx.handle, descs, n, MEM_HOST))
    return [keep[i][1].raw[: keep[i][2]] for i in range(n)]


def _fill_format(f: PixelFormat, keep: list, color, depth, bgr=False, key=None, palette=None):
    f.color, f.depth, f.bgr, f.has_key = color, depth, int(bool(bgr)), int(key is not None)
    for k, v in enumerate(key or ()):
        f.key[k] = v
    if palette is not None:
        pal = C.create_string_buffer(bytes(palette), len(palette))
        keep.append(pal)
        f.palette = _buf_addr(pal)
        f.palette_count = len(palette) // 4


def unpack_batch(ctx: Context, images, target: int = TARGET_RGBA8, alpha_mode: int = ALPHA_ASIS):
    """image.unpack(as: PNG.RGBA<T>.self / PNG.VA<T>.self) [.premultiplied / .straightened] over a
    batch.  images: dicts with storage (bytes) and the PNG.Format fields color, depth[, bgr, key,
    palette (r, g, b, a bytes)].  Returns [(status, bytes of native-endian T components)]."""
    images = list(images)
    n = len(images)
    descs = (ColorDesc * n)()
    keep = []
    for i, g in enumerate(images):
        st = bytes(g["storage"])
        count = len(st) // (_CHANNELS[g["color"]] * (2 if g["depth"] == 16 else 1))
        src = C.create_string_buffer(st, len(st)) if st else C.create_string_buffer(1)
        dst = C.create_string_buffer(max(count * _TARGET_BYTES[target], 1))
        keep.append((src, dst, count))
        descs[i].storage, descs[i].storage_len = _buf_addr(src), len(st)
        descs[i].pixels, descs[i].pixels_len = _buf_addr(dst), count * _TARGET_BYTES[target]
        descs[i].count = count
        _fill_format(descs[i].format, keep, g["color"], g["depth"], g.get("bgr"), g.get("key"), g.get("palette"))
    ctx.check(ctx._lib.pngb200_unpack_batch(ctx.handle, descs, n, target, alpha_mode, MEM_HOST))
    return [(descs[i].status, keep_i[1].raw[: keep_i[2] * _TARGET_BYTES[target]])
            for i, keep_i in enumerate(k for k in keep if isinstance(k, tuple))]


def pack_batch(ctx: Context, images, target: int = TARGET_RGBA8):
    """PNG.Image(packing:size:layout:) storage of [RGBA<T>] / [VA<T>] arrays.  images: dicts with
    pixels (bytes) and the PNG.Format fields.  Returns [bytes] (PNG.Image.storage)."""
    images = list(images)
    n = len(images)
    descs = (ColorDesc * n)()
    keep = []
    for i, g in enumerate(images):
        px = bytes(g["pixels"])
        count = len(px) // _TARGET_BYTES[target]
        size = count * _CHANNELS[g["color"]] * (2 if g["depth"] == 16 else 1)
        src = C.create_string_buffer(px, len(px)) if px else C.create_string_buffer(1)
        dst = C.create_string_buffer(max(size, 1))
        keep.append((src, dst, size))
        descs[i].pixels, descs[i].pixels_len = _buf_addr(src), len(px)
        descs[i].storage, descs[i].storage_len = _buf_addr(dst), size
        descs[i].count = count
        _fill_format(descs[i].format, keep, g["color"], g["depth"], g.get("bgr"), g.get("key"), g.get("palette"))
    ctx.check(ctx._lib.pngb200_pack_batch(ctx.handle, descs, n, target, MEM_HOST))
    return [k[1].raw[: k[2]] for k in keep if isinstance(k, tuple)]


class PngImage:
    """What PNG.Image.decompress(stream:) returns, as far as the hot path goes: status (+ the Swift
    error's associated values), header, PNG.Format fields (`fields`, ready for unpack_batch) and storage."""

    def __init__(self, d: PngDesc, storage):
        self.status, self.err_a, self.err_b = d.status, d.err_a, d.err_b
        self.width, self.height, self.depth, self.color = d.width, d.height, d.depth, d.color
        self.interlaced, self.standard = bool(d.interlaced), d.standard
        self.idat_bytes, self.idat_chunks, self.chunks = d.idat_bytes, d.idat_chunks, d.chunks
        self.checksum, self.blocks, self.produced = d.checksum, d.blocks, d.produced
        f = d.format
        self.fields = dict(color=f.color, depth=f.depth, bgr=bool(f.bgr),
                           key=tuple(f.key[: 1 if f.color == 0 else 3]) if f.has_key else None,
                           palette=bytes(d.palette_rgba[: 4 * f.palette_count]) if f.color == 3 else None)
        self.storage = storage


def _png_descs(files):
    files = [bytes(f) for f in files]
    descs = (PngDesc * max(len(files), 1))()
    keep = []
    for i, f in enumerate(files):
        src = C.create_string_buffer(f, len(f)) if f else C.create_string_buffer(1)
        keep.append(src)
        descs[i].file, descs[i].file_len = _buf_addr(src), len(f)
    return files, descs, keep


def png_inspect(files):
    """pngb200_png_inspect_batch: header walk only (no CRC check, no GPU).  Returns [PngImage]."""
    files, descs, keep = _png_descs(files)
    rc = lib().pngb200_png_inspect_batch(descs, len(files))
    if rc != OK:
        raise PNGB200Error(rc, "png_inspect")
    return [PngImage(descs[i], None) for i in range(len(files))]


def png_decode_batch(ctx: Context, files):
    """PNG.Image.decompress(stream:) over a batch of PNG files (bytes).  Returns [PngImage]."""
    files, descs, keep = _png_descs(files)
    n = len(files)
    rc = ctx._lib.pngb200_png_inspect_batch(descs, n)
    if rc != OK:
        raise PNGB200Error(rc, "png_inspect")
    outs = []
    for i in range(n):
        dst = C.create_string_buffer(max(int(descs[i].storage_size), 1))
        outs.append(dst)
        descs[i].pixels, descs[i].pixels_cap = _buf_addr(dst), int(descs[i].storage_size)
    ctx.check(ctx._lib.pngb200_png_decode_batch(ctx.handle, descs, n, MEM_HOST))
    return [PngImage(descs[i], outs[i].raw[: descs[i].storage_size] if descs[i].status == OK else None) for i in range(n)]


def png_encode_batch(ctx: Context, images, level: int = 9, idat_chunk: int = 0):
    """PNG.Image.compress(stream:level:) over a batch.  images: dicts with storage, width, height,
    [interlaced] and the PNG.Format fields.  Returns [(status, file bytes)]."""
    images = list(images)
    n = len(images)
    descs = (PngEncodeDesc * max(n, 1))()
    keep = []
    for i, g in enumerate(images):
        st = bytes(g["storage"])
        src = C.create_string_buffer(st, len(st))
        _fill_format(descs[i].format, keep, g["color"], g["depth"], g.get("bgr"), g.get("key"), g.get("palette"))
        il = int(bool(g.get("interlaced", False)))
        cap = ctx._lib.pngb200_png_encode_bound(g["width"], g["height"], C.byref(descs[i].format), il, idat_chunk)
        dst = C.create_string_buffer(cap)
        keep.append((src, dst))
        descs[i].pixels, descs[i].pixels_len = _buf_addr(src), len(st)
        descs[i].width, descs[i].height, descs[i].interlaced = g["width"], g["height"], il
        descs[i].level = level if isinstance(level, int) else level[i]
        descs[i].idat_chunk = idat_chunk
        descs[i].file, descs[i].file_cap = _buf_addr(dst), cap
    ctx.check(ctx._lib.pngb200_png_encode_batch(ctx.handle, descs, n, MEM_HOST))
    pairs = [k for k in keep if isinstance(k, tuple)]
    return [(descs[i].status, pairs[i][1].raw[: descs[i].produced]) for i in range(n)]


def _device_png_descs(files):
    """descriptors for PNG files in device memory: `files` are (address, length) pairs"""
    files = [(int(a or 0), int(n)) for a, n in files]
    descs = (PngDesc * max(len(files), 1))()
    for i, (a, n) in enumerate(files):
        descs[i].file, descs[i].file_len = a or None, n
    return descs, len(files)


def png_inspect_files(ctx: Context, files):
    """pngb200_png_inspect_files over device files, (address, length) pairs: the chunk walk on the GPU (no CRC
    check).  Returns [PngImage]."""
    descs, n = _device_png_descs(files)
    ctx.check(ctx._lib.pngb200_png_inspect_files(ctx.handle, descs, n, MEM_DEVICE))
    return [PngImage(descs[i], None) for i in range(n)]


def png_decode_files(ctx: Context, files, pixels=None):
    """PNG.Image.decompress(stream:) over PNG files already in device memory, (address, length) pairs.  pixels=None:
    storage comes back as bytes, as from png_decode_batch; else (address, capacity) device buffers, one per file,
    that receive it (PngImage.storage is then None).  Returns [PngImage]."""
    descs, n = _device_png_descs(files)
    ctx.check(ctx._lib.pngb200_png_inspect_files(ctx.handle, descs, n, MEM_DEVICE))
    outs = []
    for i in range(n):
        if pixels is None:
            dst = C.create_string_buffer(max(int(descs[i].storage_size), 1))
            outs.append(dst)
            descs[i].pixels, descs[i].pixels_cap = _buf_addr(dst), int(descs[i].storage_size)
        else:
            descs[i].pixels, descs[i].pixels_cap = int(pixels[i][0]) or None, int(pixels[i][1])
    memspace = MEM_HOST if pixels is None else MEM_DEVICE
    ctx.check(ctx._lib.pngb200_png_decode_files(ctx.handle, descs, n, MEM_DEVICE, memspace))
    return [PngImage(descs[i], outs[i].raw[: descs[i].storage_size] if pixels is None and descs[i].status == OK else None)
            for i in range(n)]


def png_encode_bound(image, idat_chunk: int = 0) -> int:
    """pngb200_png_encode_bound for one png_encode_batch image dict: the file capacity to provide"""
    f, keep = PixelFormat(), []
    _fill_format(f, keep, image["color"], image["depth"], image.get("bgr"), image.get("key"), image.get("palette"))
    return lib().pngb200_png_encode_bound(image["width"], image["height"], C.byref(f),
                                          int(bool(image.get("interlaced", False))), idat_chunk)


def png_encode_files(ctx: Context, images, files, level: int = 9, idat_chunk: int = 0):
    """PNG.Image.compress(stream:level:) over a batch, each file written straight into a device buffer: images as for
    png_encode_batch, files (address, capacity) pairs of at least png_encode_bound bytes.  Returns [(status, file
    bytes written)]."""
    images = list(images)
    n = len(images)
    descs = (PngEncodeDesc * max(n, 1))()
    keep = []
    for i, g in enumerate(images):
        st = bytes(g["storage"])
        src = C.create_string_buffer(st, len(st))
        keep.append(src)
        _fill_format(descs[i].format, keep, g["color"], g["depth"], g.get("bgr"), g.get("key"), g.get("palette"))
        descs[i].pixels, descs[i].pixels_len = _buf_addr(src), len(st)
        descs[i].width, descs[i].height, descs[i].interlaced = g["width"], g["height"], int(bool(g.get("interlaced", False)))
        descs[i].level = level if isinstance(level, int) else level[i]
        descs[i].idat_chunk = idat_chunk
        descs[i].file, descs[i].file_cap = int(files[i][0]) or None, int(files[i][1])
    ctx.check(ctx._lib.pngb200_png_encode_files(ctx.handle, descs, n, MEM_HOST, MEM_DEVICE))
    return [(descs[i].status, int(descs[i].produced)) for i in range(n)]


def deflate_batch(ctx: Context, streams, level: int = 9, fmt: int = FORMAT_ZLIB, exponent: int = 15):
    """LZ77.Deflator(format:level:exponent:).push(data, last: true) + all pull()s, per stream.
    `level` / `fmt` may be ints or per-stream sequences.  Returns list of (status, bytes)."""
    streams = list(streams)
    n = len(streams)
    descs = (DeflateDesc * n)()
    keep = []
    for i, data in enumerate(streams):
        data = bytes(data)
        cap = ctx._lib.pngb200_deflate_bound(len(data))
        src = C.create_string_buffer(data, len(data)) if len(data) else C.create_string_buffer(1)
        dst = C.create_string_buffer(cap)
        keep.append((src, dst))
        descs[i].src = _buf_addr(src)
        descs[i].src_len = len(data)
        descs[i].dst = _buf_addr(dst)
        descs[i].dst_cap = cap
        descs[i].format = fmt if isinstance(fmt, int) else fmt[i]
        descs[i].level = level if isinstance(level, int) else level[i]
        descs[i].exponent = exponent if isinstance(exponent, int) else exponent[i]
    ctx.check(ctx._lib.pngb200_deflate_batch(ctx.handle, descs, n, MEM_HOST))
    return [(descs[i].status, keep[i][1].raw[: descs[i].produced]) for i in range(n)]


def gzip_archive(ctx: Context, data: bytes, level: int = 7) -> bytes:
    """Gzip.archive(bytes:level:)"""
    (st, out), = deflate_batch(ctx, [data], level, FORMAT_GZIP)
    if st != OK:
        raise PNGB200Error(st, "gzip_archive")
    return out


def encode_batch(ctx: Context, images, level: int = 9):
    """PNG.Encoder over a batch: storage -> concatenated IDAT payload (filter select + deflate).
    `images`: dicts with pixels, width, height, volume, depth, interlaced, fmt."""
    images = list(images)
    n = len(images)
    descs = (EncodeDesc * n)()
    keep = []
    for i, g in enumerate(images):
        px = bytes(g["pixels"])
        w, h, vol = g["width"], g["height"], g["volume"]
        il = bool(g.get("interlaced", False))
        cap = ctx._lib.pngb200_deflate_bound(filtered_size(w, h, vol, il))
        src = C.create_string_buffer(px, len(px))
        dst = C.create_string_buffer(cap)
        keep.append((src, dst))
        descs[i].pixels = _buf_addr(src)
        descs[i].pixels_len = len(px)
        descs[i].idat = _buf_addr(dst)
        descs[i].idat_cap = cap
        descs[i].width, descs[i].height = w, h
        descs[i].volume, descs[i].depth, descs[i].interlaced = vol, g["depth"], int(il)
        descs[i].format = g.get("fmt", FORMAT_ZLIB)
        descs[i].level = g.get("level", level)
    ctx.check(ctx._lib.pngb200_encode_batch(ctx.handle, descs, n, MEM_HOST))
    return [(descs[i].status, keep[i][1].raw[: descs[i].produced]) for i in range(n)]


class Deflator:
    """LZ77.Deflator value semantics (push(_:last:), pop(), pull()) over the GPU encoder.  `online`: compress on the
    device as the pushes arrive, so pop() hands out each block when the reference would (pngb200_deflator_create_online);
    otherwise the whole stream is compressed at push(last: True)."""

    def __init__(self, ctx: Context, fmt: int = FORMAT_ZLIB, level: int = 9, exponent: int = 15, chunk_bytes: int = 0,
                 online: bool = False):
        self.ctx = ctx
        L = ctx._lib
        create = L.pngb200_deflator_create_online if online else L.pngb200_deflator_create
        self.handle = create(ctx.handle, fmt, level, exponent, chunk_bytes)
        if not self.handle:
            raise PNGB200Error(ERR_BAD_ARGUMENT, L.pngb200_last_error(ctx.handle).decode())

    def close(self):
        if getattr(self, "handle", None):
            self.ctx._lib.pngb200_deflator_destroy(self.handle)
            self.handle = None

    __del__ = close

    def push(self, data: bytes, last: bool = False):
        self.ctx.check(self.ctx._lib.pngb200_deflator_push(self.handle, bytes(data), len(data), int(last)))

    def _take(self, fn):
        p, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        got = fn(self.handle, C.byref(p), C.byref(n))
        if got < 0:
            raise PNGB200Error(got, "deflator")
        return C.string_at(p, n.value) if got else None

    def pop(self):
        """a complete block or None (Swift: pop() -> [UInt8]?)"""
        return self._take(self.ctx._lib.pngb200_deflator_pop)

    def pull(self):
        """a complete block, else the flushed rest, else None (Swift: pull() -> [UInt8]?)"""
        return self._take(self.ctx._lib.pngb200_deflator_pull)

    def stats(self) -> tuple:
        """online handles: (input bytes dequeued, compressed bytes written, blocks written, device bytes held)"""
        out = (C.c_uint64 * 4)()
        self.ctx.check(self.ctx._lib.pngb200_deflator_stats(self.handle, out))
        return tuple(out)

    def clone(self) -> "Deflator":
        """a copy that goes on independently (Swift: `var b = a`)"""
        return clone_batch(self.ctx, [self])[0]


class Inflator:
    """LZ77.Inflator / Gzip.Inflator value semantics over the GPU path (streaming push/pull)."""

    def __init__(self, ctx: Context, fmt: int = FORMAT_ZLIB):
        self.ctx = ctx
        self.handle = ctx._lib.pngb200_inflator_create(ctx.handle, fmt)
        if not self.handle:
            raise PNGB200Error(ERR_BAD_ARGUMENT, "inflator_create")

    def close(self):
        if getattr(self, "handle", None):
            self.ctx._lib.pngb200_inflator_destroy(self.handle)
            self.handle = None

    __del__ = close

    def push(self, data: bytes) -> int:
        """Returns OK when the stream is complete (Swift: nil), NEED_MORE_INPUT otherwise;
        raises PNGB200Error on a decompression error (Swift: throws)."""
        st = self.ctx._lib.pngb200_inflator_push(self.handle, bytes(data), len(data))
        if st < 0:
            a, b, s = C.c_uint32(), C.c_uint32(), C.c_int()
            self.ctx._lib.pngb200_inflator_error(self.handle, C.byref(s), C.byref(a), C.byref(b))
            e = PNGB200Error(st, self.ctx._lib.pngb200_last_error(self.ctx.handle).decode())
            e.payload = (a.value, b.value)
            raise e
        return st

    def error(self):
        """(sticky status, payload a, payload b): PNGB200_NEED_MORE_INPUT or OK while there is no error"""
        s, a, b = C.c_int(), C.c_uint32(), C.c_uint32()
        self.ctx._lib.pngb200_inflator_error(self.handle, C.byref(s), C.byref(a), C.byref(b))
        return s.value, a.value, b.value

    def pull(self, count: int):
        """Exactly `count` bytes or None (Swift: pull(_:) -> [UInt8]?)."""
        buf = C.create_string_buffer(max(count, 1))
        st = self.ctx._lib.pngb200_inflator_pull(self.handle, buf, count)
        return buf.raw[:count] if st == OK else None

    def pull_all(self) -> bytes:
        n = self.ctx._lib.pngb200_inflator_available(self.handle)
        buf = C.create_string_buffer(max(n, 1))
        got = self.ctx._lib.pngb200_inflator_pull_all(self.handle, buf, n)
        return buf.raw[:got]

    def stats(self) -> dict:
        """Work the device has done for this handle: input bits decoded and output bytes written (a bit or byte
        decoded twice counts twice), and the bytes of those the one-warp serial decoder wrote."""
        out = (C.c_uint64 * 3)()
        st = self.ctx._lib.pngb200_inflator_stats(self.handle, out)
        if st != OK:
            raise PNGB200Error(st, "inflator_stats")
        return {"bits": out[0], "bytes": out[1], "serial_bytes": out[2]}

    def clone(self) -> "Inflator":
        """a copy that goes on independently (Swift: `var b = a`)"""
        return clone_batch(self.ctx, [self])[0]


class PngContext:
    """PNG.Context (online decoding) on the GPU: push each IDAT payload as it arrives; the storage is a valid partial
    image after every push.  `pixels`: None for host storage owned by this object (storage() returns bytes), or a
    device buffer on the context's GPU as (address, length) (storage() returns the address)."""

    def __init__(self, ctx: Context, width: int, height: int, volume: int, depth: int, interlaced: bool = False,
                 standard: int = 0, pixels=None):
        self.ctx = ctx
        self._size = storage_size(width, height, volume)
        if pixels is None:
            self._host = C.create_string_buffer(max(self._size, 1))
            addr, cap, mem = C.addressof(self._host), self._size, MEM_HOST
        else:
            self._host = None
            (addr, cap), mem = pixels, MEM_DEVICE
        d = PngContextDesc(pixels=addr, pixels_cap=cap, width=width, height=height, volume=volume, depth=depth,
                           interlaced=int(interlaced), standard=standard, memspace=mem)
        self.handle = ctx._lib.pngb200_png_context_create(ctx.handle, C.byref(d))
        if not self.handle:
            raise PNGB200Error(ERR_BAD_ARGUMENT, ctx._lib.pngb200_last_error(ctx.handle).decode())
        self._addr = addr

    def close(self):
        if getattr(self, "handle", None):
            self.ctx._lib.pngb200_png_context_destroy(self.handle)
            self.handle = None

    __del__ = close

    def push(self, data: bytes, overdraw: bool = False) -> None:
        """push(data:overdraw:); raises PNGB200Error (with .payload for inflate errors) as the reference throws"""
        st = self.ctx._lib.pngb200_png_context_push(self.handle, bytes(data), len(data), int(overdraw))
        if st < 0:
            s, a, b = C.c_int(), C.c_uint32(), C.c_uint32()
            self.ctx._lib.pngb200_png_context_error(self.handle, C.byref(s), C.byref(a), C.byref(b))
            e = PNGB200Error(st, self.ctx._lib.pngb200_last_error(self.ctx.handle).decode())
            e.payload = (a.value, b.value) if s.value == st else (0, 0)
            raise e

    def error(self):
        """(sticky inflate status, payload a, payload b): OK while there is no error"""
        s, a, b = C.c_int(), C.c_uint32(), C.c_uint32()
        self.ctx._lib.pngb200_png_context_error(self.handle, C.byref(s), C.byref(a), C.byref(b))
        return s.value, a.value, b.value

    def end(self) -> None:
        """push(ancillary:) with IEND: raises PNGB200Error(ERR_PNG_INCOMPLETE_DATASTREAM) unless the stream is complete"""
        st = self.ctx._lib.pngb200_png_context_end(self.handle)
        if st < 0:
            raise PNGB200Error(st, "incomplete image data stream")

    def progress(self):
        """(next pass or 7, next row, filtered bytes consumed, stream complete, first row, end row the last push wrote)"""
        out = (C.c_uint64 * 6)()
        self.ctx.check(self.ctx._lib.pngb200_png_context_progress(self.handle, out))
        return tuple(out)

    def storage(self):
        """host storage: its bytes; device storage: its address"""
        return C.string_at(self._addr, self._size) if self._host is not None else self._addr

    def clone(self, pixels=None) -> "PngContext":
        """a copy that goes on independently, its storage starting as this one's.  `pixels`: None for new storage in
        this context's memspace (host bytes, or a device buffer the clone owns), or a device buffer (address, length)
        apart from this one's storage for a context with device storage"""
        return clone_batch(self.ctx, [(self, pixels)])[0]


def _push_batch(ctx: Context, kind, entry, items):
    """one batch push of `items` (handle, data[, overdraw]); returns the per-item statuses"""
    descs = (kind * max(len(items), 1))()
    keep = []   # the bytes the descriptors point into
    for d, item in zip(descs, items):
        data = bytes(item[1])
        keep.append(data)
        setattr(d, kind._fields_[0][0], item[0].handle)
        d.data = C.cast(C.c_char_p(data), C.c_void_p)
        d.n = len(data)
        if kind is PngPushDesc:
            d.overdraw = int(item[2])
        elif kind is DeflatorPushDesc:
            d.last = int(item[2])
    ctx.check(entry(ctx.handle, descs, len(items)))
    return [descs[i].status for i in range(len(items))]


def inflator_push_batch(ctx: Context, items) -> list:
    """push(_:) of many Inflators in one call: `items` is [(inflator, data)], distinct inflators of `ctx`.  Returns
    each push's status, as Inflator.push would return or raise it (payloads through the inflator's error()); raises
    PNGB200Error only when the call itself fails."""
    return _push_batch(ctx, InflatorPushDesc, ctx._lib.pngb200_inflator_push_batch, items)


def deflator_push_batch(ctx: Context, items) -> list:
    """push(_:last:) of many online Deflators in one call: `items` is [(deflator, data, last)], distinct online
    deflators of `ctx`.  Returns each push's status, as Deflator.push would raise it; raises PNGB200Error only when the
    call itself fails."""
    return _push_batch(ctx, DeflatorPushDesc, ctx._lib.pngb200_deflator_push_batch, items)


def png_context_push_batch(ctx: Context, items) -> list:
    """push(data:overdraw:) of many PngContexts in one call: `items` is [(png_context, data, overdraw)], distinct
    contexts of `ctx`.  Returns each push's status, as PngContext.push would raise it (payloads through the context's
    error()); raises PNGB200Error only when the call itself fails."""
    return _push_batch(ctx, PngPushDesc, ctx._lib.pngb200_png_context_push_batch, items)


class PngEncoder:
    """PNG.Image.compress(stream:level:) online on the GPU: push the rows of PNG.Image.storage as they are produced, top
    to bottom, and pop() the file in pieces (the head, each IDAT chunk, IEND) as soon as the reference would have
    written them.  The format fields are those of png_encode_batch's image dicts."""

    def __init__(self, ctx: Context, width: int, height: int, color: int, depth: int, bgr: bool = False, key=None,
                 palette=None, interlaced: bool = False, level: int = 9, idat_chunk: int = 0):
        self.ctx = ctx
        d, keep = PngEncoderDesc(width=width, height=height, interlaced=int(bool(interlaced)), level=level,
                                 idat_chunk=idat_chunk), []
        _fill_format(d.format, keep, color, depth, bgr, key, palette)
        self.handle = ctx._lib.pngb200_png_encoder_create(ctx.handle, C.byref(d))
        if not self.handle:
            raise PNGB200Error(ERR_BAD_ARGUMENT, ctx._lib.pngb200_last_error(ctx.handle).decode())

    def close(self):
        if getattr(self, "handle", None):
            self.ctx._lib.pngb200_png_encoder_destroy(self.handle)
            self.handle = None

    __del__ = close

    def push(self, rows, memspace: int = MEM_HOST) -> None:
        """the next whole rows of storage: bytes (MEM_HOST), or (address, length) on the context's GPU (MEM_DEVICE)"""
        (st,) = png_encoder_push_batch(self.ctx, [(self, rows, memspace)])
        if st < 0:
            raise PNGB200Error(st, self.ctx._lib.pngb200_last_error(self.ctx.handle).decode())

    def pop(self):
        """the next piece of the file, or None when there is none now"""
        p, n = C.POINTER(C.c_uint8)(), C.c_size_t()
        got = self.ctx._lib.pngb200_png_encoder_pop(self.handle, C.byref(p), C.byref(n))
        if got < 0:
            raise PNGB200Error(got, "png_encoder_pop")
        return C.string_at(p, n.value) if got else None

    def pop_all(self) -> list:
        out = []
        while (piece := self.pop()) is not None:
            out.append(piece)
        return out

    def progress(self) -> tuple:
        """(rows received, scanlines filtered, filtered bytes dequeued, IDAT chunks popped, IEND available, device
        bytes held)"""
        out = (C.c_uint64 * 6)()
        self.ctx.check(self.ctx._lib.pngb200_png_encoder_progress(self.handle, out))
        return tuple(out)

    def error(self) -> int:
        s, a, b = C.c_int(), C.c_uint32(), C.c_uint32()
        self.ctx._lib.pngb200_png_encoder_error(self.handle, C.byref(s), C.byref(a), C.byref(b))
        return s.value

    def clone(self) -> "PngEncoder":
        """a copy that goes on independently, with its own copy of the pieces not popped yet"""
        return clone_batch(self.ctx, [self])[0]


def png_encoder_push_batch(ctx: Context, items) -> list:
    """pushes of many PngEncoders in one call: `items` is [(encoder, rows[, memspace])], distinct encoders of `ctx`,
    rows as PngEncoder.push takes them.  Returns each push's status; raises PNGB200Error only when the call itself
    fails."""
    descs = (PngEncoderPushDesc * max(len(items), 1))()
    keep = []
    for d, item in zip(descs, items):
        mem = item[2] if len(item) > 2 else MEM_HOST
        d.encoder, d.memspace = item[0].handle, mem
        if mem == MEM_DEVICE:
            d.rows, d.n = int(item[1][0]) or None, int(item[1][1])
        else:
            data = bytes(item[1])
            keep.append(data)
            d.rows, d.n = C.cast(C.c_char_p(data), C.c_void_p), len(data)
    ctx.check(ctx._lib.pngb200_png_encoder_push_batch(ctx.handle, descs, len(items)))
    return [descs[i].status for i in range(len(items))]


def clone_batch(ctx: Context, items) -> list:
    """Clone many handles in one call (pngb200_clone_batch): `items` holds Inflators, Deflators, PngEncoders and
    PngContexts, a context optionally as (png_context, pixels) with `pixels` as PngContext.clone takes it.  Returns the
    clones in order; raises PNGB200Error, with no clone made, when the call fails."""
    descs = (CloneDesc * max(len(items), 1))()
    field = {Inflator: "inflator", Deflator: "deflator", PngContext: "context", PngEncoder: "encoder"}
    storage = []   # per context item: (host buffer, device tensor, address)
    for d, item in zip(descs, items):
        src, pixels = item if isinstance(item, tuple) else (item, None)
        setattr(d, field[type(src)], src.handle)
        if isinstance(src, PngContext):
            host, dev = None, None
            if pixels is not None and src._host is not None:
                raise PNGB200Error(ERR_BAD_ARGUMENT, "clone_batch: a context with host storage takes no pixels")
            if pixels is not None:
                addr, cap = pixels
            elif src._host is not None:
                host = C.create_string_buffer(max(src._size, 1))
                addr, cap = C.addressof(host), src._size
            else:
                import torch
                dev = torch.empty(max(src._size, 1), dtype=torch.uint8, device=f"cuda:{ctx.device}")
                addr, cap = dev.data_ptr(), src._size
            d.pixels, d.pixels_cap = addr, cap
            storage.append((host, dev, addr))
    ctx.check(ctx._lib.pngb200_clone_batch(ctx.handle, descs, len(items)))
    out, k = [], 0
    for d, item in zip(descs, items):
        src = item[0] if isinstance(item, tuple) else item
        c = type(src).__new__(type(src))
        c.ctx, c.handle = src.ctx, d.clone
        if isinstance(src, PngContext):
            c._size, (c._host, c._dev, c._addr) = src._size, storage[k]
            k += 1
        out.append(c)
    return out
