"""Device-resident bandwidth of the unfilter stage alone: pngb200_unfilter_batch(..., MEM_DEVICE) over the filtered bytes
of bench.py's workloads (8K: 198 x 7680x4320 RGBA8, 1080p: 1056 x 1920x1080 RGBA8), built the way bench.py builds them
(corpus.make + the library's filter kernel, `unique` distinct images repeated over the batch).

Bytes moved per call = filtered bytes F (read once) + pixel bytes P (written once).  Kernel time comes from
torch.profiler (CUDA activities) in a run of its own; call time from CUDA events around each call on the context's
stream (it adds the job-table copies).  The share of peak is (F + P) / kernel time over the H100 SXM data-sheet 3.35 TB/s.

    python tools/unfilter_bw.py [--workload 8k-rgba8,1080p-rgba8] [--reps 10] [--other NAME=PATH ...] [--out FILE]

With PNGB200_LIB naming another build of libpngb200.so (for example the parent commit's, tagged "parent"), and any
--other builds, every library runs in the same process: each one's pixels are compared with this build's before
anything is timed (a parent whose pixels differ is an error; other builds are only reported), then the calls
alternate between the libraries.  The card's name and power limit are printed first.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
HBM_PEAK = 3.35e12
MEM_DEVICE = 1
WORKLOADS = {"8k-rgba8": (7680, 4320, 198, 8), "1080p-rgba8": (1920, 1080, 1056, 64)}   # w, h, batch, unique


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.splitlines()[0].split(", ") + ["?", "?", "?"])[:3] if q.returncode == 0 else ["?"] * 3
    return dict(device=torch.cuda.get_device_name(0), name=name, power_limit=power, max_sm_clock=clock)


def digest(pixels: torch.Tensor, n: int, size: int) -> torch.Tensor:
    """per image: two wrapping int64 sums of its 8-byte words, plain and position-weighted"""
    pos = torch.arange(1, size // 8 + 1, device=pixels.device, dtype=torch.int64)
    out = []
    for i in range(n):   # one image at a time: a batch-sized temporary would not fit next to the batch
        words = pixels[i * size:(i + 1) * size].view(torch.int64)
        out.append(torch.stack([words.sum(), (words * pos).sum()]))
    return torch.stack(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="8k-rgba8,1080p-rgba8")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--other", action="append", default=[], metavar="NAME=PATH")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    pkg = importlib.import_module("swift-png_b200")
    import corpus

    ctx = pkg.Context()
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
    head = dict(card(), libs=[tag for tag, _ in libs], reps=args.reps)
    lines = [json.dumps(head)]
    print(lines[-1], flush=True)

    for wl in args.workload.split(","):
        w, h, batch, unique = WORKLOADS[wl]
        pitch = w * 4
        fsize, psize = h * (pitch + 1), h * pitch
        filtered = torch.empty(batch * fsize, dtype=torch.uint8, device="cuda")
        for u in range(unique):
            st = corpus.make("photo", w, h, u).tobytes()
            f = pkg.filter_batch(ctx, [dict(pixels=st, width=w, height=h, volume=32, depth=8)])[0]
            filtered[u * fsize:(u + 1) * fsize].copy_(torch.frombuffer(bytearray(f), dtype=torch.uint8))
        for i in range(unique, batch):
            filtered[i * fsize:(i + 1) * fsize].copy_(filtered[(i % unique) * fsize:(i % unique + 1) * fsize])
        pixels = torch.empty(batch * psize, dtype=torch.uint8, device="cuda")
        descs = (pkg.ImageDesc * batch)()
        for i in range(batch):
            d = descs[i]
            d.idat, d.idat_len = filtered.data_ptr() + i * fsize, fsize
            d.pixels, d.pixels_cap = pixels.data_ptr() + i * psize, psize
            d.width, d.height, d.volume, d.depth = w, h, 32, 8

        def call(tag, L):
            return L.pngb200_unfilter_batch(ctxs[tag], descs, batch, MEM_DEVICE)

        # pixels first: every build against this one, before anything is timed
        ref = None
        match = {}
        for tag, L in libs:
            pixels.fill_(0xA5)
            torch.cuda.synchronize()
            assert call(tag, L) == 0
            torch.cuda.synchronize()
            assert all(descs[i].status == 0 for i in range(batch))
            got = digest(pixels, batch, psize)
            if ref is None:
                ref = got
            match[tag] = bool(torch.equal(got, ref))
        if "parent" in match and not match["parent"]:
            raise SystemExit(f"{wl}: pixels differ from the parent build's")

        nbytes = batch * (fsize + psize)
        for tag, L in libs:
            for _ in range(args.warmup):
                call(tag, L)
        torch.cuda.synchronize()
        ev = {tag: [] for tag, _ in libs}
        for _ in range(args.reps):   # alternate the libraries call by call
            for tag, L in libs:
                stream = torch.cuda.ExternalStream(L.pngb200_ctx_stream(ctxs[tag]))
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                assert call(tag, L) == 0
                e1.record(stream)
                stream.synchronize()
                ev[tag].append((e0, e1))
        torch.cuda.synchronize()
        for tag, L in libs:
            call_ms = sorted(a.elapsed_time(b) for a, b in ev[tag])
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    call(tag, L)
                torch.cuda.synchronize()
            kern = [e for e in prof.key_averages() if "unfilter_wave_kernel" in e.key]
            total_us = sum(getattr(e, "device_time_total", 0) or getattr(e, "cuda_time_total", 0) for e in kern)
            count = sum(e.count for e in kern)
            kernel_ms = total_us / max(count, 1) / 1e3
            row = dict(lib=tag, workload=wl, images=batch, bytes=nbytes, pixels_match_this=match[tag],
                       kernel_ms=round(kernel_ms, 3), kernels=count,
                       call_ms_median=round(call_ms[len(call_ms) // 2], 3),
                       call_ms_min=round(call_ms[0], 3), call_ms_max=round(call_ms[-1], 3),
                       TBps=round(nbytes / (kernel_ms * 1e-3) / 1e12, 3) if kernel_ms else None,
                       peak_frac=round(nbytes / (kernel_ms * 1e-3) / HBM_PEAK, 3) if kernel_ms else None)
            lines.append(json.dumps(row))
            print(lines[-1], flush=True)
        del filtered, pixels
        torch.cuda.empty_cache()
    for tag, L in libs:
        L.pngb200_ctx_destroy(ctxs[tag])
    ctx.close()
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
