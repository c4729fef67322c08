"""Times pngb200_png_decode_files with the PNG files in device memory against pngb200_png_decode_batch with the same
files in pinned host memory (pixels left on the device both ways), on three batches: the 296 x 1080p RGBA8 batch of
tools/png_file_probe.py (65,544-byte IDATs), and 8K RGBA8 files with 8 KiB and with 65,544-byte IDATs.  A separate
torch.profiler pass over one device-file call gives the device time of the chunk walk (png_walk_kernel, both passes)
and of the device-to-device IDAT gather, and their share of the call.  Prints the card's name and power limit first.

    python tools/png_device_files.py [--reps 5] [--files-8k 4]
"""
import argparse
import importlib
import os
import struct
import subprocess
import sys
import time
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import torch  # noqa: E402

import corpus  # noqa: E402

pkg = importlib.import_module("swift-png_b200")


def chunk(t, body):
    return struct.pack(">I", len(body)) + t + body + struct.pack(">I", zlib.crc32(t + body))


def png(w, h, z, idat):
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 6, 0, 0, 0)) +
            b"".join(chunk(b"IDAT", z[o:o + idat]) for o in range(0, len(z), idat)) + chunk(b"IEND", b""))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


class Batch:
    def __init__(self, ctx, data, n, w, h):
        self.ctx, self.n, self.w, self.h, self.len = ctx, n, w, h, len(data)
        self.host = torch.frombuffer(bytearray(data), dtype=torch.uint8).repeat(n).pin_memory()
        self.dev = self.host.cuda()
        self.out = torch.zeros((n, w * h * 4), dtype=torch.uint8, device="cuda")
        self.descs = (pkg.PngDesc * n)()

    def run(self, device_files):
        base = (self.dev if device_files else self.host).data_ptr()
        for i in range(self.n):
            self.descs[i].file, self.descs[i].file_len = base + i * self.len, self.len
            self.descs[i].pixels, self.descs[i].pixels_cap = self.out[i].data_ptr(), self.w * self.h * 4
        L = self.ctx._lib
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if device_files:
            self.ctx.check(L.pngb200_png_decode_files(self.ctx.handle, self.descs, self.n, pkg.MEM_DEVICE, pkg.MEM_DEVICE))
        else:
            self.ctx.check(L.pngb200_png_decode_batch(self.ctx.handle, self.descs, self.n, pkg.MEM_DEVICE))
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        assert all(self.descs[i].status == 0 for i in range(self.n))
        return dt


def walk_share(batch):
    """device time of the walk kernels and of the device-to-device copies during one device-file call, and the call's
    wall time, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        dt = batch.run(True)
    walk = gather = 0.0
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "png_walk_kernel" in e.name:
            walk += us
        elif "Memcpy DtoD" in e.name or "Memcpy2D DtoD" in e.name or ("Memcpy" in e.name and "Device -> Device" in e.name):
            gather += us
    return walk / 1e3, gather / 1e3, dt * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--files-8k", type=int, default=4)
    args = ap.parse_args()
    name, limit = card()
    print(f"card: {name}, power limit {limit}")
    ctx = pkg.Context(0)
    px = corpus.make("photo", 1920, 1080, 3)
    z = corpus.zlib_png_stream(px, 4, 6)[1]
    batches = [("296 x 1080p RGBA8, 65,544-byte IDATs", Batch(ctx, png(1920, 1080, z, 65544), 296, 1920, 1080))]
    big = corpus.make("photo", 7680, 4320, 5)
    zb = corpus.zlib_png_stream(big, 4, 6)[1]
    for idat in (8192, 65544):
        batches.append((f"{args.files_8k} x 8K RGBA8, {idat:,}-byte IDATs",
                        Batch(ctx, png(7680, 4320, zb, idat), args.files_8k, 7680, 4320)))
    for label, b in batches:
        b.run(True), b.run(False)  # warm-up: arenas, modules
        dev, host = [], []
        for _ in range(args.reps):  # alternated, so drift hits both alike
            dev.append(b.run(True))
            host.append(b.run(False))
        mp = b.n * b.w * b.h / 1e6
        d, h = sorted(dev)[len(dev) // 2], sorted(host)[len(host) // 2]
        walk, gather, call = walk_share(b)
        chunks = b.descs[0].chunks
        print(f"{label} ({chunks} chunks a file): device files {d * 1e3:.2f} ms ({mp / d:.0f} MPixels/s), "
              f"pinned host files {h * 1e3:.2f} ms ({mp / h:.0f} MPixels/s); median of {args.reps}")
        print(f"    profiled device-file call {call:.2f} ms: walk kernels {walk:.3f} ms ({100 * walk / call:.2f} %), "
              f"IDAT gather {gather:.3f} ms ({100 * gather / call:.2f} %)")
        assert bytes(b.out[b.n - 1][:64].cpu().numpy().tobytes()) == (px if b.w == 1920 else big).tobytes()[:64]
    ctx.close()


if __name__ == "__main__":
    main()
