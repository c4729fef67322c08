"""Times the online PNG encoder (pngb200_png_encoder_*) against pngb200_png_encode_batch on the GPU.

One 1920 x ROWS RGBA8 photo at LEVEL is pushed in bands of BAND rows, pop() after each push, and compared with one
png_encode_batch call on the whole image: the time to the first IDAT chunk, the total time, the time per push (median,
p90), the launches per push and the peak device bytes the handle held.  Then N encoders take one band each in one
png_encoder_push_batch call a round, against the same pushes made one encoder at a time.  The joined pieces are checked
against png_encode_batch's file.  The card's name and power limit come first.

    python3 tools/png_encoder_online_bw.py [--rows 270] [--band 16] [--level 9] [--n 1 8 64]
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
import corpus  # noqa: E402

W = 1920


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def stats(times, launches):
    ms = sorted(1e3 * t for t in times)
    return dict(push_ms_median=round(ms[len(ms) // 2], 3), push_ms_p90=round(ms[int(0.9 * (len(ms) - 1))], 3),
                launches_per_push=round(sum(launches) / len(launches), 3), max_launches=max(launches))


def online(p, ctx, images, h, band, level, batched):
    """images pushed band by band, one batch call a round (batched) or one push at a time"""
    encs = [p.PngEncoder(ctx, W, h, color=6, depth=8, level=level) for _ in images]
    out = [[] for _ in images]
    first, times, launches, peak = None, [], [], 0
    row = W * 4
    t0 = time.perf_counter()
    for a in range(0, h, band):
        items = [(e, px[a * row: min(h, a + band) * row]) for e, px in zip(encs, images)]
        l0, r0 = ctx.launches, time.perf_counter()
        if batched:
            assert p.png_encoder_push_batch(ctx, items) == [0] * len(items)
        else:
            for e, rows in items:
                e.push(rows)
        for i, e in enumerate(encs):
            got = e.pop_all()
            out[i] += got
            if first is None and any(g[4:8] == b"IDAT" for g in got):
                first = time.perf_counter() - t0
        times.append(time.perf_counter() - r0)
        launches.append(ctx.launches - l0)
        peak = max([peak] + [e.progress()[5] for e in encs])
    total = time.perf_counter() - t0
    for e in encs:
        e.close()
    return dict(first_idat_s=round(first, 4), total_s=round(total, 3), peak_device_bytes_per_handle=peak,
                pushes=len(times), **stats(times, launches)), [b"".join(o) for o in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=270)
    ap.add_argument("--band", type=int, default=16)
    ap.add_argument("--level", type=int, default=9)
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 64])
    a = ap.parse_args()
    p = importlib.import_module("swift-png_b200")
    ctx = p.Context(0)
    h = a.rows
    print(json.dumps(dict(card=card(), image=f"{W}x{h} RGBA8 photo", level=a.level, band=a.band)), flush=True)
    px = corpus.make("photo", W, h, 0).tobytes()
    t0 = time.perf_counter()
    ((st, whole),) = p.png_encode_batch(ctx, [dict(storage=px, width=W, height=h, color=6, depth=8)], a.level)
    one_shot = time.perf_counter() - t0
    assert st == 0
    res, (got,) = online(p, ctx, [px], h, a.band, a.level, False)
    assert got == whole
    print(json.dumps(dict(one_image=res, png_encode_batch_s=round(one_shot, 3))), flush=True)
    for n in a.n:
        images = [corpus.make("photo", W, h, i % 8).tobytes() for i in range(n)]
        on, got_on = online(p, ctx, images, h, a.band, a.level, True)
        alone, got_alone = online(p, ctx, images, h, a.band, a.level, False)
        assert got_on == got_alone
        print(json.dumps(dict(n=n, push_batch=on, one_at_a_time=alone)), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
