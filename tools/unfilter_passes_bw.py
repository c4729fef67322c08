"""Device-resident throughput of the unfilter stage on Adam7 and 1/2/4-bit images: pngb200_unfilter_batch(...,
MEM_DEVICE) over seeded filtered streams (tests/wide_rows.filtered_stream, every filter type) already in device memory.

Batches: 8 x 8K and 64 x 1080p Adam7 RGBA8, 1080p Adam7 RGB16, 8K indexed 4-bit and grey 1-bit, non-interlaced and
interlaced, and a size sweep of Adam7 RGBA8 from 32x32 to 1080p (the sweep that places the generic kernel's threshold,
DESIGN §4.3).  Per batch and library: MPixels/s from CUDA events around each call (the call includes the copy of the
streams into the library's private buffer), and, from torch.profiler in a run of its own, each unfilter kernel's time
and unfilter_interleave_kernel's (read + write) bytes/s: it reads the reconstructed pass rows (the filtered bytes less
one filter byte a row) and writes the storage.

    python tools/unfilter_passes_bw.py [--batches NAME,...] [--seconds 1] [--other NAME=PATH ...] [--out FILE]

With PNGB200_LIB naming another build of libpngb200.so (the parent commit's, tagged "parent"), and any --other builds,
every library runs in the same process: each one's storage is compared byte for byte with this build's before anything
is timed, then the calls alternate between the libraries.  Every shape is warmed up first, and each library gets about
--seconds of timed calls per batch.  The card's name and power limit are printed first.
"""
import argparse
import ctypes as C
import importlib
import json
import math
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
MEM_DEVICE = 1
K8, P1080 = (7680, 4320), (1920, 1080)
# name: [(w, h, volume, depth, interlaced)] * count
BATCHES = {
    "8k-adam7-rgba8": [(*K8, 32, 8, True)] * 8,
    "1080p-adam7-rgba8": [(*P1080, 32, 8, True)] * 64,
    "1080p-adam7-rgb16": [(*P1080, 48, 16, True)] * 8,
    "8k-indexed4": [(*K8, 4, 4, False)] * 4,
    "8k-grey1": [(*K8, 1, 1, False)] * 4,
    "8k-adam7-indexed4": [(*K8, 4, 4, True)] * 4,
    "8k-adam7-grey1": [(*K8, 1, 1, True)] * 4,
}
for s in (32, 48, 64, 96, 128, 256, 512):   # the sweep: about 16 Mpixels a batch
    BATCHES[f"sweep-{s}"] = [(s, s, 32, 8, True)] * min(4096, (1 << 24) // (s * s))
BATCHES["sweep-1080p"] = [(*P1080, 32, 8, True)] * 8


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.splitlines()[0].split(", ") + ["?", "?", "?"])[:3] if q.returncode == 0 else ["?"] * 3
    return dict(device=torch.cuda.get_device_name(0), name=name, power_limit=power, max_sm_clock=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default=",".join(BATCHES))
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--other", action="append", default=[], metavar="NAME=PATH")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    pkg = importlib.import_module("swift-png_b200")
    import wide_rows
    from oracle import oracle

    libs = [("this", pkg.lib())]
    if os.environ.get("PNGB200_LIB"):   # the package itself then loads that build: bind ours by path instead
        libs = [("this", C.CDLL(os.path.join(ROOT, "swift-png_b200", "libpngb200.so"))),
                ("parent", C.CDLL(os.environ["PNGB200_LIB"]))]
    for spec in args.other:
        name, path = spec.split("=", 1)
        libs.append((name, C.CDLL(path)))
    for _, L in libs:
        L.pngb200_ctx_create.argtypes, L.pngb200_ctx_create.restype = [C.c_int], C.c_void_p
        L.pngb200_ctx_destroy.argtypes, L.pngb200_ctx_destroy.restype = [C.c_void_p], None
        L.pngb200_ctx_stream.argtypes, L.pngb200_ctx_stream.restype = [C.c_void_p], C.c_void_p
        L.pngb200_unfilter_batch.argtypes = [C.c_void_p, C.POINTER(pkg.ImageDesc), C.c_size_t, C.c_int]
    ctxs = {tag: L.pngb200_ctx_create(0) for tag, L in libs}
    head = dict(card(), libs=[tag for tag, _ in libs], seconds=args.seconds)
    lines = [json.dumps(head)]
    print(lines[-1], flush=True)

    for name in args.batches.split(","):
        shapes = BATCHES[name]
        distinct = sorted(set(shapes))
        streams = {s: bytes(wide_rows.filtered_stream(s[0], s[1], s[2], s[4], (1, 4, 2, 3, 0, 4, 4, 3), k))
                   for k, s in enumerate(distinct)}
        fsize = [len(streams[s]) for s in shapes]
        psize = [oracle.storage_size(s[0], s[1], s[2]) for s in shapes]
        foff = [0] + [sum(fsize[:i + 1]) for i in range(len(shapes))]
        poff = [0] + [sum(psize[:i + 1]) for i in range(len(shapes))]
        filtered = torch.empty(foff[-1], dtype=torch.uint8, device="cuda")
        for i, s in enumerate(shapes):
            filtered[foff[i]:foff[i + 1]].copy_(torch.frombuffer(bytearray(streams[s]), dtype=torch.uint8))
        del streams
        pixels = torch.empty(poff[-1], dtype=torch.uint8, device="cuda")
        descs = (pkg.ImageDesc * len(shapes))()
        for i, (w, h, v, d, il) in enumerate(shapes):
            g = descs[i]
            g.idat, g.idat_len = filtered.data_ptr() + foff[i], fsize[i]
            g.pixels, g.pixels_cap = pixels.data_ptr() + poff[i], psize[i]
            g.width, g.height, g.volume, g.depth, g.interlaced = w, h, v, d, int(il)
        mpix = sum(w * h for w, h, *_ in shapes) / 1e6
        rows = sum(sum(sh for _, _, sh, _ in wide_rows.adam7_passes(w, h, v)) if il else h for w, h, v, _, il in shapes)
        inter_bytes = (foff[-1] - rows) + poff[-1]

        def call(tag, L):
            return L.pngb200_unfilter_batch(ctxs[tag], descs, len(shapes), MEM_DEVICE)

        # storage first: every build against this one, byte for byte, before anything is timed
        ref, match = None, {}
        for tag, L in libs:
            pixels.fill_(0xA5)
            torch.cuda.synchronize()
            assert call(tag, L) == 0
            torch.cuda.synchronize()
            assert all(descs[i].status == 0 for i in range(len(shapes)))
            if ref is None:
                ref = pixels.clone()
                match[tag] = True
            else:
                match[tag] = bool(torch.equal(pixels, ref))
        del ref
        if "parent" in match and not match["parent"]:
            raise SystemExit(f"{name}: storage differs from the parent build's")

        per_call = {}
        for tag, L in libs:   # warm-up, and the length of one call
            call(tag, L)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            call(tag, L)
            torch.cuda.synchronize()
            per_call[tag] = time.perf_counter() - t0
        reps = {tag: max(3, min(2000, math.ceil(args.seconds / max(per_call[tag], 1e-6)))) for tag, _ in libs}
        ev = {tag: [] for tag, _ in libs}
        for r in range(max(reps.values())):   # alternate the libraries call by call
            for tag, L in libs:
                if r >= reps[tag]:
                    continue
                stream = torch.cuda.ExternalStream(L.pngb200_ctx_stream(ctxs[tag]))
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                assert call(tag, L) == 0
                e1.record(stream)
                stream.synchronize()
                ev[tag].append((e0, e1))
        torch.cuda.synchronize()
        for tag, L in libs:
            ms = sorted(a.elapsed_time(b) for a, b in ev[tag])
            n_prof = max(1, min(reps[tag], 20))
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(n_prof):
                    call(tag, L)
                torch.cuda.synchronize()
            kernels = {}
            for e in prof.key_averages():
                if "unfilter" in e.key:
                    us = getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0)
                    kernels[e.key.split("(")[0].split("::")[-1]] = round(us / n_prof / 1e3, 4)
            inter_ms = kernels.get("unfilter_interleave_kernel")
            med = ms[len(ms) // 2]
            row = dict(lib=tag, batch=name, images=len(shapes), shape=list(shapes[0]), mpixels=round(mpix, 3),
                       storage_matches_this=match[tag], calls=len(ms), call_ms_median=round(med, 4),
                       call_ms_min=round(ms[0], 4), call_ms_max=round(ms[-1], 4),
                       mpixels_per_s=round(mpix / (med * 1e-3), 1), kernel_ms=kernels,
                       interleave_bytes=inter_bytes,
                       interleave_GBps=round(inter_bytes / (inter_ms * 1e-3) / 1e9, 1) if inter_ms else None)
            lines.append(json.dumps(row))
            print(lines[-1], flush=True)
        del filtered, pixels
        torch.cuda.empty_cache()
    for tag, L in libs:
        L.pngb200_ctx_destroy(ctxs[tag])
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
