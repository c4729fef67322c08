"""The online encoder's restatement (tests/png_encoder_stream.py) on the CPU: for every push schedule its pieces join
to oracle.png_compress's file, the committed level-9 outputs come back byte for byte when their baselines are pushed a
row at a time, and a file of more than two IDAT chunks hands out its first chunk before its last row."""
from __future__ import annotations

import os

import numpy as np
import pytest

import png_encoder_stream as pes
from oracle import oracle

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "encode")
KEPT = sorted(f[4:] for f in os.listdir(GOLDEN) if f.startswith("out-"))

# the format list of test_gpu_container.py::test_encode_every_format_matches_oracle
FORMATS = ((dict(color=6, depth=8, bgr=True), 5, 4), (dict(color=2, depth=8, bgr=True, key=(3, 2, 1)), 4, 4),
           (dict(color=0, depth=4, key=(9,)), 7, 3), (dict(color=2, depth=16, key=(1, 2, 3)), 3, 3),
           (dict(color=3, depth=2, palette=bytes([1, 2, 3, 255, 4, 5, 6, 7, 8, 9, 10, 255])), 9, 2),
           (dict(color=6, depth=16), 64, 48), (dict(color=4, depth=8), 33, 17))


def image(fields, w, h, seed):
    rng = np.random.default_rng(seed)
    ch = pes.CHANNELS[fields["color"]]
    top = 3 if fields["color"] == 3 else (1 << min(fields["depth"], 8))
    return rng.integers(0, top, w * h * ch * (2 if fields["depth"] == 16 else 1), dtype=np.uint8).tobytes()


def baseline(name):
    info, storage = oracle.png_decompress(open(os.path.join(GOLDEN, "in-" + name), "rb").read())
    assert info.status == 0
    return storage, info.width, info.height, info.fields(), bool(info.interlaced)


@pytest.mark.parametrize("interlaced", [False, True])
@pytest.mark.parametrize("k", range(len(FORMATS)))
def test_every_format_and_schedule_joins_to_the_file(k, interlaced):
    fields, w, h = FORMATS[k]
    storage = image(fields, w, h, 3 + k)
    for level in (0, 6):
        want = oracle.png_compress(storage, w, h, oracle.make_format(**fields), interlaced, level, idat_chunk=16)
        for kind in ("rows", "all", 3, [2, 0, 5]):
            got = pes.pieces(oracle, storage, w, h, fields, interlaced, level, 16, pes.schedule(h, kind))
            assert b"".join(b"".join(p) for p in got) == want, (level, kind)
            assert got[-1][-1][4:8] == b"IEND" and all(p[4:8] == b"IDAT" for ps in got for p in ps[1:-1] if ps)


@pytest.mark.parametrize("name", KEPT)
def test_level9_outputs_row_by_row(name):
    storage, w, h, fields, interlaced = baseline(name)
    got = pes.pieces(oracle, storage, w, h, fields, interlaced, 9, 65544, pes.schedule(h, "rows"))
    assert b"".join(b"".join(p) for p in got) == open(os.path.join(GOLDEN, "out-" + name), "rb").read()
    # more than two chunks of payload: the first IDAT is out before the last row arrives
    first = next(i for i, p in enumerate(got) if any(c[4:8] == b"IDAT" for c in p))
    if sum(c[4:8] == b"IDAT" for p in got for c in p) > 2:
        assert first < h - 1, (name, first)


def test_first_idat_before_last_row_whenever_the_payload_spans_more_than_two_chunks():
    """Adam7 streams pass 0 only while rows arrive: its first IDAT comes early once pass 0 alone passes the 4096-byte
    trigger and fills a block"""
    fields = dict(color=6, depth=8)
    for interlaced, w, h in ((False, 48, 40), (True, 320, 240)):
        storage = image(fields, w, h, 11)
        got = pes.pieces(oracle, storage, w, h, fields, interlaced, 4, 256, pes.schedule(h, 5))
        idat = [i for i, p in enumerate(got) for c in p if c[4:8] == b"IDAT"]
        assert len(idat) > 2 and idat[0] < len(got) - 1, (interlaced, idat[:4])
