"""Measures rho, the cost per output byte of a split stream's tail relative to its head (kSymbolicCost in
pngb200_api.cu), on bench.py's default decode batch: 198 x 7680x4320 RGBA8 photos per GPU (8 distinct images,
reference filter rule, zlib level 6), device-resident.  rho = (tail SM cycles / tail bytes) / (head SM cycles / head
bytes), from the per-CTA phase timers (pngb200_ctx_split_stats).  Needs a GPU.

    python tools/split_cost.py [--batch 198] [--steps 3]"""
import argparse
import importlib
import os
import sys
import zlib
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
import corpus  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=198)
    ap.add_argument("--unique", type=int, default=8)
    ap.add_argument("--steps", type=int, default=3)
    args = ap.parse_args()
    import torch
    pkg = importlib.import_module("swift-png_b200")
    ctx = pkg.Context(0)
    w, h = 7680, 4320
    with ThreadPoolExecutor(max_workers=args.unique) as ex:
        storages = list(ex.map(lambda i: np.ascontiguousarray(corpus.make("photo", w, h, i)).tobytes(), range(args.unique)))
        filtered = [pkg.filter_batch(ctx, [dict(pixels=s, width=w, height=h, volume=32, depth=8)])[0] for s in storages]
        idats = list(ex.map(lambda f: zlib.compress(f, 6), filtered))
    del storages, filtered
    size = 4 * w * h
    d_unique = [torch.frombuffer(bytearray(z), dtype=torch.uint8).cuda() for z in idats]
    d_idat = [d_unique[i % args.unique].clone() for i in range(args.batch)]
    d_pixels = torch.empty((args.batch, size), dtype=torch.uint8, device="cuda")
    descs = (pkg.ImageDesc * args.batch)()
    for i in range(args.batch):
        descs[i].idat, descs[i].idat_len = d_idat[i].data_ptr(), d_idat[i].numel()
        descs[i].pixels, descs[i].pixels_cap = d_pixels[i].data_ptr(), size
        descs[i].width, descs[i].height, descs[i].volume, descs[i].depth = w, h, 32, 8
    torch.cuda.synchronize()
    for step in range(args.steps):
        ctx.check(ctx._lib.pngb200_decode_batch(ctx.handle, descs, args.batch, pkg.MEM_DEVICE))
        assert all(descs[i].status == 0 for i in range(args.batch))
        s = ctx.split_stats()
        seg = ctx.segment_stats()
        head = s["head_cycles"] / max(s["head_bytes"], 1)
        tail = s["tail_cycles"] / max(s["tail_bytes"], 1)
        share = s["head_bytes"] / max(s["head_bytes"] + s["tail_bytes"], 1)
        print(f"step {step}: {seg['streams']} streams cut, {seg['fallbacks']} fallbacks; head share of the bytes {share:.3f}; "
              f"head {head:.2f}, tail {tail:.2f} cycles/byte, rho {tail / head:.3f}; tails switched {s['switched']}, "
              f"symbolic {s['symbolic_bytes'] / max(s['tail_bytes'], 1):.1%} of the tail bytes; "
              f"stage ms {tuple(round(x, 1) for x in ctx.stage_ms())}", flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
