"""Times the online deflator (pngb200_deflator_create_online) against the buffered one on the GPU.

N filtered RGBA8 images (level 9) and one text-like gzip stream (level 7) are pushed in 65 544-byte pieces, one
pngb200_deflator_push_batch call per round, pop() after each round.  The buffered handles take the same pushes and
compress at the last one.  Reports the time to the first chunk, the time per round (median, p90) and in total, the
launches per round, and the peak device bytes per handle, with the card's name and power limit.

    python3 tools/deflator_online_bw.py [--n 1 8 64] [--rows 1080] [--gzip-mb 8]
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

PIECE = 65544


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def run(p, ctx, streams, online):
    """streams: [(data, fmt, level)] -> measurements of one pass"""
    zs = [p.Deflator(ctx, fmt, level, online=online) for _, fmt, level in streams]
    rounds = max((len(d) + PIECE - 1) // PIECE for d, _, _ in streams)
    first, times, launches, peak, out = None, [], [], 0, [[] for _ in zs]
    t0 = time.perf_counter()
    for k in range(rounds + 1):
        items = []
        for i, (d, _, _) in enumerate(streams):
            piece = d[k * PIECE:(k + 1) * PIECE]
            if k * PIECE < len(d) or k == rounds:
                items.append((zs[i], piece, k == rounds))
        l0, r0 = ctx.launches, time.perf_counter()
        if online:
            st = p.deflator_push_batch(ctx, items)
            assert all(s == 0 for s in st), st
        else:
            for z, piece, last in items:
                z.push(piece, last=last)
        for i, z in enumerate(zs):
            while (c := (z.pull() if k == rounds else z.pop())) is not None:
                out[i].append(c)
                if first is None:
                    first = time.perf_counter() - t0
        times.append(time.perf_counter() - r0)
        launches.append(ctx.launches - l0)
        if online:
            peak = max([peak] + [z.stats()[3] for z in zs])
    total = time.perf_counter() - t0
    for z in zs:
        z.close()
    times_ms = sorted(1e3 * t for t in times)
    return dict(first_chunk_s=round(first, 4), round_ms_median=round(times_ms[len(times_ms) // 2], 3),
                round_ms_p90=round(times_ms[int(0.9 * (len(times_ms) - 1))], 3), total_s=round(total, 3),
                launches_per_round=round(sum(launches) / len(launches), 3), max_launches=max(launches),
                peak_device_bytes_per_handle=peak or None, rounds=rounds + 1), [b"".join(o) for o in out]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 64])
    ap.add_argument("--rows", type=int, default=1080)
    ap.add_argument("--gzip-mb", type=float, default=8)
    a = ap.parse_args()
    p = importlib.import_module("swift-png_b200")
    ctx = p.Context(0)
    w, h = 1920, a.rows
    print(json.dumps(dict(card=card(), image=f"{w}x{h} RGBA8 filtered, level 9", piece=PIECE)), flush=True)
    base = [corpus.make("photo", w, h, s).tobytes() for s in range(min(max(a.n), 8))]
    filtered = p.filter_batch(ctx, [dict(pixels=b, width=w, height=h, volume=32, depth=8) for b in base])
    for n in a.n:
        streams = [(filtered[i % len(filtered)], p.FORMAT_ZLIB, 9) for i in range(n)]
        on, got_on = run(p, ctx, streams, True)
        off, got_off = run(p, ctx, streams, False)
        assert got_on == got_off
        print(json.dumps(dict(n=n, online=on, buffered=off)), flush=True)
    text = (b"".join(filtered) * 4)[: int(a.gzip_mb * (1 << 20))]
    on, got_on = run(p, ctx, [(text, p.FORMAT_GZIP, 7)], True)
    off, got_off = run(p, ctx, [(text, p.FORMAT_GZIP, 7)], False)
    assert got_on == got_off
    print(json.dumps(dict(gzip_level7_mb=a.gzip_mb, online=on, buffered=off)), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
