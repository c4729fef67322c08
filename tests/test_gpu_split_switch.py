"""Split streams whose tails leave symbolic mode on the GPU: in 8K-wide photos the markers of a tail's first rows die
out within 70-130 rows (tools/split_tail_model.py), so the rest of each tail is decoded as bytes.  Compared with the same batch decoded
with the split off (PNGB200_SPLIT=0): statuses, checksums, byte counts, block counts and pixels."""
from __future__ import annotations

import zlib

import numpy as np
import pytest

import corpus
from test_gpu_split import decode_device, make_ctx

pytestmark = pytest.mark.gpu

SLOTS = 8    # 6 streams on 8 slots: heads take 6, the other 2 CTAs take 3 tails each


@pytest.fixture(scope="module")
def ctxs(pngb200):
    split = make_ctx(pngb200, PNGB200_PLAN_SLOTS=str(SLOTS), PNGB200_SPLIT="1")
    whole = make_ctx(pngb200, PNGB200_PLAN_SLOTS=str(SLOTS), PNGB200_SPLIT="0")
    yield split, whole
    split.close()
    whole.close()


def test_switching_tails_match_whole_stream_decode(pngb200, ctxs):
    split, whole = ctxs
    cases = []
    for k in range(6):
        img = corpus.make("photo", 7680, 720, 70 + k)
        filt, z = corpus.zlib_png_stream(img, 4, 6)
        cases.append((img, filt, dict(idat=z, width=img.shape[1], height=img.shape[0], volume=32, depth=8)))
    jobs = [c[2] for c in cases]
    got = decode_device(pngb200, split, jobs)
    assert split.segment_stats() == dict(streams=6, segments=12, fallbacks=0), split.segment_stats()
    st = split.split_stats()
    assert st["switched"] == 6, st
    assert 0 < st["symbolic_bytes"] < st["tail_bytes"] and st["head_bytes"] + st["tail_bytes"] == sum(len(c[1]) for c in cases)
    ref = decode_device(pngb200, whole, jobs)
    assert whole.segment_stats()["streams"] == 0
    for g, r, (img, filt, _) in zip(got, ref, cases):
        assert g["status"] == r["status"] == 0
        assert g["checksum"] == r["checksum"] == zlib.adler32(filt)
        assert (g["produced"], g["blocks"]) == (r["produced"], r["blocks"]) == (len(filt), r["blocks"])
        assert g["pixels"] == r["pixels"] == np.ascontiguousarray(img).tobytes()
