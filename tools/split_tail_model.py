"""How much of a split stream's tail has to stay symbolic (DESIGN.md section 4.2): the benchmark's distinct 8K images
(bench.py's default workload: photo 7680x4320 RGBA8, reference filter rule, zlib level 6) are cut where run_split
cuts them -- the first dynamic block header at or after h of the bits -- and the tail is decoded with the 32 KiB in
front of it unknown (tools/segment_model.c, tail_model).  Once the last 32 KiB a tail has produced hold no marker,
the rest of the tail can be decoded like a head.  Prints, per image and head share h, the tail's length and where
its symbolic prefix ends.

    python tools/split_tail_model.py [--images 8] [--shares 0.805,0.76]"""
import argparse
import ctypes as C
import os
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [HERE, os.path.join(ROOT, "tests")]
import corpus  # noqa: E402
import segment_model  # noqa: E402


def tail_at(L, z: bytes, share: float):
    """(split bit, tail bytes, first clean offset, markers) for the first real dynamic header at or after `share`"""
    hb = C.c_uint64()
    out = (C.c_uint64 * 3)()
    p = int(share * 8 * len(z))
    while p + 17 <= 8 * len(z):
        if L.probe_dynamic_header(z, len(z), p, C.byref(hb)) == 0 and L.tail_model(z, len(z), p, out) == 0:
            return p, out[0], out[1], out[2]
        p += 1
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=8)
    ap.add_argument("--shares", default="0.805,0.76")
    ap.add_argument("--width", type=int, default=7680)
    ap.add_argument("--height", type=int, default=4320)
    args = ap.parse_args()
    shares = [float(s) for s in args.shares.split(",")]
    L = segment_model.lib()
    L.probe_dynamic_header.argtypes = [C.c_char_p, C.c_size_t, C.c_uint64, C.POINTER(C.c_uint64)]
    L.tail_model.argtypes = [C.c_char_p, C.c_size_t, C.c_uint64, C.POINTER(C.c_uint64)]
    row = 4 * args.width + 1

    def one(i):
        _, z = corpus.zlib_png_stream(corpus.make("photo", args.width, args.height, i), 4, 6)
        return [tail_at(L, z, h) for h in shares]

    with ThreadPoolExecutor(max_workers=2) as ex:   # numpy, zlib and the C model release the GIL; ~3 GB per image
        res = list(ex.map(one, range(args.images)))
    for h_i, h in enumerate(shares):
        fr = []
        print(f"h = {h}")
        for i, per in enumerate(res):
            p, n2, clean, markers = per[h_i]
            fr.append(clean / n2)
            print(f"  image {i}: tail {n2} bytes ({n2 / row:.0f} rows), window clean from {clean} ({clean / row:.0f} rows, "
                  f"{clean / n2:.1%} of the tail), {markers} markers")
        print(f"  median symbolic prefix {np.median(fr):.1%} of the tail, worst {max(fr):.1%}")


if __name__ == "__main__":
    main()
