"""Online decoding (pngb200_png_context, PNG.Context) on whole 8K files, against png_decode_batch of the same file.

Files: an 8K RGBA8 photo-like image, non-interlaced and Adam7, each encoded at level 9 into IDAT chunks of 65 544
bytes: the bytes the reference's encoder writes and the library's encoder reproduces.  They are made by the oracle's
restatement of that encoder, both files at once on two host threads, because the library deflates a stream with one
warp and is slower than a CPU core on a single 8K stream (DESIGN §6).  Each file is decoded
  - by pushing its IDAT chunks one by one, overdraw off and on,
  - by one push of the whole IDAT run, overdraw off and on,
  - by png_decode_batch,
into host storage.  Per mode: the whole decode's time, per-push latency (median and p90, host clock around each push:
a push returns once the storage holds its rows) and kernel launches per push.  Every mode's final storage is checked
against png_decode_batch's.  The card's name and power limit are printed first.

    python tools/png_context_bw.py [--repeat 3] [--out FILE] [--modes chunks,...] [--cache DIR]
"""
import argparse
import concurrent.futures
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import corpus  # noqa: E402
import pngio  # noqa: E402
from oracle import oracle  # noqa: E402

W, H = 7680, 4320


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.splitlines()[0].split(", ") + ["?", "?", "?"])[:3] if q.returncode == 0 else ["?"] * 3
    return dict(device=torch.cuda.get_device_name(0), name=name, power_limit=power, max_sm_clock=clock)


def online(pkg, ctx, pieces, interlaced, overdraw, finish=True):
    c = pkg.PngContext(ctx, W, H, 32, 8, interlaced)
    lat, launches = [], []
    t0 = time.perf_counter()
    for p in pieces:
        n0, a = ctx.launches, time.perf_counter()
        c.push(p, overdraw)
        lat.append(time.perf_counter() - a)
        launches.append(ctx.launches - n0)
    if finish:
        c.end()
    total = time.perf_counter() - t0
    out = c.storage()
    c.close()
    return total, lat, launches, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--cache", default=None, help="directory that keeps the two files between runs")
    ap.add_argument("--modes", default="chunks,chunks+overdraw,one push,one push+overdraw",
                    help="comma-separated online modes to time (a slow build may time only some)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    info = card()
    print(json.dumps(info), flush=True)
    pkg = importlib.import_module("swift-png_b200")
    ctx = pkg.Context(0)
    img = corpus.make("photo", W, H, 11).tobytes()
    fmt = oracle.make_format(6, 8)
    cached = [os.path.join(args.cache, f"8k_{n}.png") for n in ("plain", "adam7")] if args.cache else []
    if cached and all(os.path.exists(p) for p in cached):
        files = [open(p, "rb").read() for p in cached]
    else:
        with concurrent.futures.ThreadPoolExecutor(2) as pool:
            files = list(pool.map(lambda il: oracle.png_compress(img, W, H, fmt, il, 9, 65544), (False, True)))
        for p, f in zip(cached, files):
            os.makedirs(args.cache, exist_ok=True)
            open(p, "wb").write(f)
    rows = []
    for interlaced, f in zip((False, True), files):
        chunks = pngio.idat_chunks(f)
        whole = b"".join(chunks)
        (ref,) = pkg.png_decode_batch(ctx, [f])
        assert ref.status == 0 and ref.storage == img
        modes = [("chunks", chunks, False), ("chunks+overdraw", chunks, True),
                 ("one push", [whole], False), ("one push+overdraw", [whole], True)]
        modes = [m for m in modes if m[0] in args.modes.split(",")]
        for name, pieces, od in modes:   # warm-up: every shape the timed runs use
            online(pkg, ctx, pieces[:3], interlaced, od, finish=False)
        pkg.png_decode_batch(ctx, [f])
        for rep in range(args.repeat):
            torch.cuda.synchronize()
            a = time.perf_counter()
            (d,) = pkg.png_decode_batch(ctx, [f])
            dt = time.perf_counter() - a
            assert d.storage == img
            rows.append(dict(file=("adam7" if interlaced else "plain"), mode="png_decode_batch", rep=rep,
                             ms=round(dt * 1e3, 2), idat_bytes=len(whole), chunks=len(chunks)))
            print(json.dumps(rows[-1]), flush=True)
            for name, pieces, od in modes:
                total, lat, launches, out = online(pkg, ctx, pieces, interlaced, od)
                assert out == img, (name, interlaced)
                lat_ms = np.array(lat) * 1e3
                rows.append(dict(file=("adam7" if interlaced else "plain"), mode=name, rep=rep, ms=round(total * 1e3, 2),
                                 pushes=len(pieces), push_ms_median=round(float(np.median(lat_ms)), 3),
                                 push_ms_p90=round(float(np.percentile(lat_ms, 90)), 3),
                                 launches_per_push_mean=round(float(np.mean(launches)), 2),
                                 launches_per_push_max=int(max(launches))))
                print(json.dumps(rows[-1]), flush=True)
    ctx.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
