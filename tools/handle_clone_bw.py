"""Times pngb200_clone_batch on the GPU.

Per case: the wall time of one clone call (a host clock around the call, which ends in a stream synchronise; median of
REPEAT calls), the device bytes and host bytes the call copies (pngb200_ctx_clone_stats, summed by the library from the
handles' state), and the launches per call (pngb200_ctx_launch_count).  Cases:
  - a level-8 online deflator halfway through a 6 MB text stream, whose blocks reach 2^21 - 1 vertices;
  - an 8K RGBA8 context halfway through its file, plain and Adam7, with host and with device storage;
  - N = 1, 8 and 64 1080p RGBA8 contexts halfway through their files, cloned in one call against one call per context.
The card's name and power limit come first, read in the same run.

    python3 tools/handle_clone_bw.py [--repeat 5] [--n 1 8 64]
"""
from __future__ import annotations

import argparse
import importlib
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import pngio  # noqa: E402
from png_context_cases import geometry  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def timed(p, ctx, items, repeat):
    """median wall ms of clone_batch(items), launches per call, and the (device, host) bytes one call copies; the
    clones are closed outside the clock"""
    times, launches, copied = [], [], set()
    for _ in range(repeat):
        n0 = ctx.launches
        t0 = time.perf_counter()
        made = p.clone_batch(ctx, items)
        times.append(time.perf_counter() - t0)
        launches.append(ctx.launches - n0)
        copied.add(ctx.clone_stats())
        for m in made:
            m.close()
    times.sort()
    assert len(copied) == 1, copied
    (dev, host), = copied
    return round(1e3 * times[len(times) // 2], 3), max(launches), dict(device_bytes=dev, host_bytes=host)


def half_context(p, ctx, file, device):
    """a context pushed the first half of its file's IDAT chunks (device storage: a buffer it keeps)"""
    import torch
    png = pngio.parse(file)
    g = geometry(png)
    pixels, buf = None, None
    if device:
        size = p.storage_size(g["w"], g["h"], g["volume"])
        buf = torch.empty(size, dtype=torch.uint8, device="cuda")
        pixels = (buf.data_ptr(), size)
    c = p.PngContext(ctx, g["w"], g["h"], g["volume"], g["depth"], g["interlaced"], g["standard"], pixels)
    c._keep = buf
    chunks = pngio.idat_chunks(file)
    for k in chunks[:len(chunks) // 2]:
        c.push(k)
    return c


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=5)
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 64])
    a = ap.parse_args()
    p = importlib.import_module("swift-png_b200")
    from test_gpu_deflator_online import text
    from test_gpu_png_context import big_file
    import deflate_stream as ds
    print(json.dumps(dict(card=card())), flush=True)
    ctx = p.Context(0)
    # a level-8 deflator halfway through 6 MB
    data = text(6 << 20, 77)
    cuts = ds.cuts(len(data), [65544])
    z = p.Deflator(ctx, p.FORMAT_ZLIB, level=8, online=True)
    for lo, hi in cuts[:len(cuts) // 2]:
        z.push(data[lo:hi])
        while z.pop() is not None:
            pass
    held = z.stats()[3]
    ms, launches, copied = timed(p, ctx, [z], a.repeat)
    print(json.dumps(dict(case="deflator level 8, 3 MB of 6 MB", ms=ms, launches=launches, device_bytes_held=held,
                          **copied)), flush=True)
    z.close()
    # 8K contexts halfway
    for il in (False, True):
        file = big_file(7680, 4320, il)[1]
        for device in (False, True):
            c = half_context(p, ctx, file, device)
            ms, launches, copied = timed(p, ctx, [c], a.repeat)
            print(json.dumps(dict(case=f"8K RGBA8 context halfway, {'Adam7' if il else 'plain'}, "
                                       f"{'device' if device else 'host'} storage", ms=ms, launches=launches, **copied)),
                  flush=True)
            c.close()
    # N 1080p contexts: one call against one call each
    file = big_file(1920, 1080, False)[1]
    cs = [half_context(p, ctx, file, False) for _ in range(max(a.n))]
    for n in a.n:
        items = cs[:n]
        one, launches, copied = timed(p, ctx, items, a.repeat)
        t0 = time.perf_counter()
        made = [c.clone() for c in items]
        each = 1e3 * (time.perf_counter() - t0)
        for m in made:
            m.close()
        print(json.dumps(dict(case=f"{n} x 1080p RGBA8 contexts halfway", one_call_ms=one, launches=launches,
                              one_call_per_context_ms=round(each, 3), **copied)), flush=True)
    for c in cs:
        c.close()
    ctx.close()


if __name__ == "__main__":
    main()
