"""Device-resident bandwidth of the colour targets: pngb200_unpack_batch / pngb200_pack_batch for all 12
targets over a batch of 8 x 7680x4320 storages in rgba8, rgb8 and v8.

Bytes moved per call = storage bytes + target bytes (read one, write the other).  Kernel time comes from
torch.profiler (CUDA activities) over repeated calls after a warm-up; call time from CUDA events around
each call on the context's stream (it adds the job-table copies and the host-side preparation).  The
share of peak is bytes / kernel time over the H100 SXM data-sheet 3.35 TB/s.

    python tools/color_bw.py [--reps 5] [--images 8] [--out FILE]

With PNGB200_LIB naming another build of libpngb200.so (for example the parent commit's), both libraries
run in the same process, alternating per target, and each row says which one it came from; targets the
other build does not know are skipped for it.  The card's name and power limit are printed first.
"""
import argparse
import ctypes as C
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM_PEAK = 3.35e12
TARGETS = ["RGBA8", "RGBA16", "VA8", "VA16", "RGBA32", "RGBA64", "VA32", "VA64", "V8", "V16", "V32", "V64"]
TARGET_BYTES = [4, 8, 2, 4, 16, 32, 8, 16, 1, 2, 4, 8]
FORMATS = {"rgba8": (6, 4), "rgb8": (2, 3), "v8": (0, 1)}  # colour type, storage bytes per pixel
MEM_DEVICE = 1


def bind(path: str):
    L = C.CDLL(path)
    L.pngb200_ctx_create.argtypes, L.pngb200_ctx_create.restype = [C.c_int], C.c_void_p
    L.pngb200_ctx_destroy.argtypes, L.pngb200_ctx_destroy.restype = [C.c_void_p], None
    L.pngb200_ctx_stream.argtypes, L.pngb200_ctx_stream.restype = [C.c_void_p], C.c_void_p
    L.pngb200_unpack_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int]
    L.pngb200_pack_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int]
    return L


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.splitlines()[0].split(", ") + ["?", "?", "?"])[:3] if q.returncode == 0 else ["?"] * 3
    return dict(device=torch.cuda.get_device_name(0), name=name, power_limit=power, max_sm_clock=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--width", type=int, default=7680)
    ap.add_argument("--height", type=int, default=4320)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    pkg = importlib.import_module("swift-png_b200")
    libs = [("this", bind(os.path.join(ROOT, "swift-png_b200", "libpngb200.so")))]
    if os.environ.get("PNGB200_LIB"):
        libs.append(("other", bind(os.environ["PNGB200_LIB"])))
    ctxs = {tag: L.pngb200_ctx_create(0) for tag, L in libs}
    rows = []
    head = dict(card(), images=args.images, width=args.width, height=args.height, reps=args.reps)
    print(json.dumps(head), flush=True)
    lines = [json.dumps(head)]

    n = args.width * args.height
    pixels = torch.empty(args.images * n * max(TARGET_BYTES) + 256, dtype=torch.uint8, device="cuda")
    for fname, (color, sbpp) in FORMATS.items():
        gen = torch.Generator(device="cuda").manual_seed(color)
        storage = torch.randint(0, 256, (args.images * n * sbpp,), dtype=torch.uint8, device="cuda", generator=gen)
        for t, tname in enumerate(TARGETS):
            tb = TARGET_BYTES[t]
            descs = (pkg.ColorDesc * args.images)()
            for i in range(args.images):
                d = descs[i]
                d.storage, d.storage_len = storage.data_ptr() + i * n * sbpp, n * sbpp
                d.pixels, d.pixels_len = pixels.data_ptr() + i * n * tb, n * tb
                d.count = n
                d.format.color, d.format.depth = color, 8
            for tag, L in libs:
                ctx = ctxs[tag]
                stream = torch.cuda.ExternalStream(L.pngb200_ctx_stream(ctx))
                for direction in ("unpack", "pack"):
                    def call():
                        if direction == "unpack":
                            return L.pngb200_unpack_batch(ctx, descs, args.images, t, 0, MEM_DEVICE)
                        return L.pngb200_pack_batch(ctx, descs, args.images, t, MEM_DEVICE)
                    torch.cuda.synchronize()
                    if call() != 0:  # a build without this target
                        continue
                    for _ in range(args.warmup - 1):
                        call()
                    ev = []
                    for _ in range(args.reps):
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record(stream)
                        assert call() == 0
                        e1.record(stream)
                        ev.append((e0, e1))
                    torch.cuda.synchronize()
                    call_ms = sorted(a.elapsed_time(b) for a, b in ev)
                    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                        for _ in range(args.reps):
                            call()
                        torch.cuda.synchronize()
                    kern = [e for e in prof.key_averages() if "pack_" in e.key and "kernel" in e.key]
                    total_us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0) for e in kern)
                    count = sum(e.count for e in kern)
                    kernel_ms = total_us / max(count, 1) / 1e3
                    nbytes = args.images * n * (sbpp + tb)
                    row = dict(lib=tag, format=fname, target=tname, dir=direction, bytes=nbytes,
                               kernel_ms=round(kernel_ms, 4), kernels=count, call_ms_median=round(call_ms[len(call_ms) // 2], 4),
                               TBps=round(nbytes / (kernel_ms * 1e-3) / 1e12, 3),
                               peak_frac=round(nbytes / (kernel_ms * 1e-3) / HBM_PEAK, 3),
                               kernel_name=kern[0].key if kern else "")
                    rows.append(row)
                    print(json.dumps(row), flush=True)
                    lines.append(json.dumps(row))
        del storage
    for tag, L in libs:
        L.pngb200_ctx_destroy(ctxs[tag])
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
