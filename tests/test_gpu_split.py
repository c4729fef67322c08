"""Streams cut into a direct head and a symbolic tail (csrc/inflate_segments.cuh, run_split in pngb200_api.cu) on the
GPU.  The split engages when a batch holds between N/2 and N big streams for N CTA slots; PNGB200_PLAN_SLOTS lowers
N so that a handful of images takes that path.  Everything is compared with the same batch decoded with the split
off (PNGB200_SPLIT=0): statuses, checksums, byte counts, block counts and pixels."""
from __future__ import annotations

import os
import zlib

import numpy as np
import pytest

import corpus

pytestmark = pytest.mark.gpu

SLOTS = 8    # 6 streams on 8 slots: heads take 6, the other 2 CTAs take 3 tails each


def make_ctx(pngb200, **env):
    saved = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        return pngb200.Context(0)
    finally:
        for k, v in saved.items():
            if v is None:
                os.environ.pop(k)
            else:
                os.environ[k] = v


@pytest.fixture(scope="module")
def ctxs(pngb200):
    split = make_ctx(pngb200, PNGB200_PLAN_SLOTS=str(SLOTS), PNGB200_SPLIT="1")
    whole = make_ctx(pngb200, PNGB200_PLAN_SLOTS=str(SLOTS), PNGB200_SPLIT="0")
    yield split, whole
    split.close()
    whole.close()


def decode_device(pngb200, ctx, jobs):
    """pngb200_decode_batch with device-resident IDAT and pixels (the split borrows the pixel buffers)"""
    import torch
    n = len(jobs)
    descs = (pngb200.ImageDesc * n)()
    keep = []
    for i, j in enumerate(jobs):
        idat = torch.frombuffer(bytearray(j["idat"]), dtype=torch.uint8).cuda()
        size = pngb200.storage_size(j["width"], j["height"], j["volume"])
        pix = torch.full((size,), 0xA5, dtype=torch.uint8, device="cuda")
        keep.append((idat, pix))
        descs[i].idat, descs[i].idat_len = idat.data_ptr(), idat.numel()
        descs[i].pixels, descs[i].pixels_cap = pix.data_ptr(), size
        descs[i].width, descs[i].height = j["width"], j["height"]
        descs[i].volume, descs[i].depth = j["volume"], j["depth"]
        descs[i].interlaced, descs[i].format = 0, 0
    torch.cuda.synchronize()
    ctx.check(ctx._lib.pngb200_decode_batch(ctx.handle, descs, n, pngb200.MEM_DEVICE))
    return [dict(status=descs[i].status, checksum=descs[i].checksum, produced=descs[i].produced, blocks=descs[i].blocks,
                 err=(descs[i].err_a, descs[i].err_b), pixels=keep[i][1].cpu().numpy().tobytes()) for i in range(n)]


def photo_jobs(n, seed):
    out = []
    for k in range(n):
        img = corpus.make("photo", 1024 + 64 * k, 768, seed + k)
        filt, z = corpus.zlib_png_stream(img, 4, 6)
        out.append((img, filt, dict(idat=z, width=img.shape[1], height=img.shape[0], volume=32, depth=8)))
    return out


def test_split_decode_matches_whole_stream_decode(pngb200, ctxs):
    split, whole = ctxs
    cases = photo_jobs(6, 40)
    jobs = [c[2] for c in cases]
    got = decode_device(pngb200, split, jobs)
    assert split.segment_stats() == dict(streams=6, segments=12, fallbacks=0), split.segment_stats()
    ref = decode_device(pngb200, whole, jobs)
    assert whole.segment_stats()["streams"] == 0
    for g, r, (img, filt, _) in zip(got, ref, cases):
        assert g["status"] == r["status"] == 0
        assert g["checksum"] == r["checksum"] == zlib.adler32(filt)
        assert (g["produced"], g["blocks"]) == (r["produced"], r["blocks"]) == (len(filt), r["blocks"])
        assert g["pixels"] == r["pixels"] == np.ascontiguousarray(img).tobytes()


def test_split_streams_that_do_not_line_up_fall_back(pngb200, ctxs):
    """a truncated stream (the tail never reaches the trailer) and a wrong trailer checksum (the combined Adler-32
    differs) among clean ones: those two are decoded whole and report exactly what the unsplit batch reports"""
    split, whole = ctxs
    cases = photo_jobs(6, 50)
    jobs = [dict(c[2]) for c in cases]
    jobs[1]["idat"] = jobs[1]["idat"][: len(jobs[1]["idat"]) - 100]
    bad = bytearray(jobs[4]["idat"])
    bad[-2] ^= 0x40
    jobs[4]["idat"] = bytes(bad)
    got = decode_device(pngb200, split, jobs)
    assert split.segment_stats() == dict(streams=6, segments=12, fallbacks=2), split.segment_stats()
    ref = decode_device(pngb200, whole, jobs)
    for i, (g, r) in enumerate(zip(got, ref)):
        assert (g["status"], g["checksum"], g["produced"], g["blocks"], g["err"]) == \
               (r["status"], r["checksum"], r["produced"], r["blocks"], r["err"]), i
        if r["status"] == 0:
            assert g["pixels"] == r["pixels"] == np.ascontiguousarray(cases[i][0]).tobytes(), i
    assert got[1]["status"] != 0 and got[4]["status"] != 0


def test_split_off_for_host_buffers(pngb200, ctxs):
    """host-memory batches have no device pixel buffer to borrow: decoded whole"""
    split, _ = ctxs
    cases = photo_jobs(6, 60)
    got = pngb200.decode_batch(split, [c[2] for c in cases])
    assert split.segment_stats()["streams"] == 0
    for g, (img, filt, _) in zip(got, cases):
        assert g.status == 0 and g.pixels == np.ascontiguousarray(img).tobytes()
