"""Batch online decoding (pngb200_png_context_push_batch) against the same pushes made one context at a time.

Files: four 1080p RGBA8 photo-like images, two non-interlaced and two Adam7, each encoded once at level 9 into IDAT chunks
of 65 544 bytes by the oracle's restatement of the reference's encoder.  N contexts (N in 1, 8, 64, 256) take the files
in turn, in host storage.  Round r pushes every context's r-th chunk:
  - batch: one png_context_push_batch per round;
  - single: the same pushes, one PngContext.push after another.
The two modes alternate within one process.  Per mode and N: total wall time, MPixels/s, per-round latency (median and
p90, host clock around the round: a push returns once the storage holds its rows) and kernel launches per round.  Every
context's final storage is checked against png_decode_batch's.  The card's name and power limit are printed first.

    python tools/png_context_batch_bw.py [--repeat 2] [--counts 1,8,64,256] [--out FILE] [--cache DIR]
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

W, H = 1920, 1080
FILES = [(seed, interlaced) for seed in (3, 4) for interlaced in (False, True)]


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power, clock = (q.stdout.splitlines()[0].split(", ") + ["?", "?", "?"])[:3] if q.returncode == 0 else ["?"] * 3
    return dict(device=torch.cuda.get_device_name(0), name=name, power_limit=power, max_sm_clock=clock)


def make_files(cache):
    paths = [os.path.join(cache, f"1080p_{s}_{'adam7' if il else 'plain'}.png") for s, il in FILES] if cache else []
    if paths and all(os.path.exists(p) for p in paths):
        return [open(p, "rb").read() for p in paths]
    fmt = oracle.make_format(6, 8)

    def one(spec):
        seed, il = spec
        return oracle.png_compress(corpus.make("photo", W, H, seed).tobytes(), W, H, fmt, il, 9, 65544)

    with concurrent.futures.ThreadPoolExecutor(len(FILES)) as pool:
        files = list(pool.map(one, FILES))
    for p, f in zip(paths, files):
        os.makedirs(cache, exist_ok=True)
        open(p, "wb").write(f)
    return files


def run(pkg, ctx, n, chunks, mode, rounds=None):
    """n contexts over the files in turn; returns (total s, per-round s, launches per round, storages)"""
    cs = [pkg.PngContext(ctx, W, H, 32, 8, FILES[i % len(FILES)][1]) for i in range(n)]
    lat, launches = [], []
    rounds = rounds or max(len(c) for c in chunks)
    t0 = time.perf_counter()
    for r in range(rounds):
        items = [(c, chunks[i % len(chunks)][r]) for i, c in enumerate(cs) if r < len(chunks[i % len(chunks)])]
        n0, a = ctx.launches, time.perf_counter()
        if mode == "batch":
            sts = pkg.png_context_push_batch(ctx, [(c, p, False) for c, p in items])
            assert all(s == 0 for s in sts), sts
        else:
            for c, p in items:
                c.push(p, False)
        lat.append(time.perf_counter() - a)
        launches.append(ctx.launches - n0)
    total = time.perf_counter() - t0
    outs = [c.storage() for c in cs]
    for c in cs:
        c.close()
    return total, lat, launches, outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeat", type=int, default=2)
    ap.add_argument("--counts", default="1,8,64,256")
    ap.add_argument("--out", default=None)
    ap.add_argument("--cache", default=None, help="directory that keeps the four files between runs")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("no CUDA device: nothing to measure")
    info = card()
    print(json.dumps(info), flush=True)
    pkg = importlib.import_module("swift-png_b200")
    ctx = pkg.Context(0)
    files = make_files(args.cache)
    chunks = [pngio.idat_chunks(f) for f in files]
    refs = []
    for f in files:
        (d,) = pkg.png_decode_batch(ctx, [f])
        assert d.status == 0
        refs.append(d.storage)
    for mode in ("batch", "single"):   # warm-up: every shape the timed runs use
        run(pkg, ctx, 8, chunks, mode, rounds=3)
    rows = []
    for n in [int(x) for x in args.counts.split(",")]:
        for rep in range(args.repeat):
            for mode in ("batch", "single"):
                torch.cuda.synchronize()
                total, lat, launches, outs = run(pkg, ctx, n, chunks, mode)
                for i, o in enumerate(outs):
                    assert o == refs[i % len(refs)], (mode, n, i)
                lat_ms = np.array(lat) * 1e3
                rows.append(dict(contexts=n, mode=mode, rep=rep, ms=round(total * 1e3, 1),
                                 mpix_s=round(n * W * H / total / 1e6, 1), rounds=len(lat),
                                 round_ms_median=round(float(np.median(lat_ms)), 3),
                                 round_ms_p90=round(float(np.percentile(lat_ms, 90)), 3),
                                 launches_per_round_mean=round(float(np.mean(launches)), 2),
                                 launches_per_round_max=int(max(launches))))
                print(json.dumps(rows[-1]), flush=True)
    ctx.close()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        json.dump(dict(card=info, rows=rows), open(args.out, "w"), indent=1)


if __name__ == "__main__":
    main()
