"""GPU parity for the wide and scalar colour targets: RGBA / VA at 32 and 64 bits and
image.unpack(as: T.self) / PNG.Image(packing: [T]) for T = UInt8 ... UInt64, against the restatement in
colorwide.py (itself pinned to the oracle and the reference's goldens by test_color_wide_ref.py), and
the reference's own scalar decode / encode outputs reproduced entirely on the device."""
import ctypes as C
import os

import numpy as np
import pytest

import colorwide as cw
import pngio
from conftest import GOLDEN

pytestmark = pytest.mark.gpu

PNGSUITE = sorted(f for f in os.listdir(os.path.join(GOLDEN, "pngsuite")) if f.endswith(".png"))
IOS = sorted(f for f in os.listdir(os.path.join(GOLDEN, "ios")) if f.endswith(".png"))
COLOUR = os.path.join(GOLDEN, "colour")


def fields(im):
    return {k: v for k, v in im.items() if k not in ("storage", "pixels")}


def decoded(pngb200, ctx, sub, names):
    pngs = [pngio.parse(open(os.path.join(GOLDEN, sub, n), "rb").read()) for n in names]
    got = pngb200.decode_batch(ctx, [dict(idat=p.idat, width=p.width, height=p.height, volume=p.volume, depth=p.depth,
                                          interlaced=p.interlaced, fmt=p.fmt) for p in pngs])
    assert all(g.status == 0 for g in got)
    return [dict(storage=g.pixels, **pngio.format_fields(p)) for p, g in zip(pngs, got)]


@pytest.mark.parametrize("target", cw.NEW_TARGETS)
def test_goldens_every_alpha_mode_and_pack(pngb200, ctx, target):
    """PngSuite and CgBI inputs decoded on the GPU, then every valid alpha mode, then pack back"""
    for sub, names in (("pngsuite", PNGSUITE), ("ios", IOS)):
        images = decoded(pngb200, ctx, sub, names)
        for mode in cw.modes(target):
            for g, im, name in zip(pngb200.unpack_batch(ctx, images, target, mode), images, names):
                assert g == cw.unpack(im["storage"], target, mode, **fields(im)), (name, mode)
        unpacked = pngb200.unpack_batch(ctx, images, target)
        back = pngb200.pack_batch(ctx, [dict(pixels=px, **fields(im)) for (_, px), im in zip(unpacked, images)], target)
        for b, (_, px), im, name in zip(back, unpacked, images, names):
            assert b == cw.pack(px, target, **fields(im)), name


def random_images(rng, most):
    """every (colour type, depth, bgr, key) the format enum has, random samples, odd pixel counts"""
    images = []
    for color, depths in ((0, (1, 2, 4, 8, 16)), (2, (8, 16)), (3, (1, 2, 4, 8)), (4, (8, 16)), (6, (8, 16))):
        for depth in depths:
            for variant in range(3):
                n = int(rng.integers(1, most)) | 1
                ch = cw.CHANNELS[color]
                if depth < 8 or color == 3:
                    top = min(1 << depth, 200) if color == 3 else 1 << depth
                    st = rng.integers(0, top, n * ch, dtype=np.uint8).tobytes()
                else:
                    st = rng.integers(0, 256, n * ch * (depth // 8), dtype=np.uint8).tobytes()
                im = dict(storage=st, color=color, depth=depth, bgr=False, key=None, palette=None)
                if color == 3:
                    # grey entries too, so scalar pack finds some (v, v, v, 255)
                    pal = rng.integers(0, 256, (200, 4), dtype=np.uint8)
                    pal[::4, 1] = pal[::4, 2] = pal[::4, 0]
                    pal[::4, 3] = 255
                    im["palette"] = pal.tobytes()
                if color in (0, 2) and variant == 1:
                    im["key"] = tuple(int(x) for x in rng.integers(0, min(1 << depth, 4), 3 if color == 2 else 1))
                    if depth >= 8:  # make the key actually occur
                        arr = np.frombuffer(st, dtype=np.uint8).copy().reshape(n, -1)
                        arr[::3] = np.frombuffer(b"".join(int(k).to_bytes(depth // 8, "big") for k in im["key"]), dtype=np.uint8)
                        im["storage"] = arr.tobytes()
                if color in (2, 6) and depth == 8 and variant == 2:
                    im["bgr"] = True
                images.append(im)
    return images


@pytest.mark.parametrize("target", cw.NEW_TARGETS)
def test_random_storages_all_formats(pngb200, ctx, target):
    rng = np.random.default_rng(100 + target)
    images = random_images(rng, 9000)
    for mode in cw.modes(target):
        for g, im in zip(pngb200.unpack_batch(ctx, images, target, mode), images):
            assert g == cw.unpack(im["storage"], target, mode, **fields(im)), (im["color"], im["depth"], mode)
    bits = cw.TARGETS[target][0]
    px = []
    for im in images:
        n = len(im["storage"]) // (cw.CHANNELS[im["color"]] * (2 if im["depth"] == 16 else 1))
        raw = rng.integers(0, 256, n * cw.target_bytes(target), dtype=np.uint8)
        if im["color"] == 3 and cw.TARGETS[target][1] == "v":  # hit the grey palette entries often
            grey = np.frombuffer(im["palette"], np.uint8).reshape(-1, 4)[::4, 0]
            vals = np.frombuffer(raw.tobytes(), cw.DTYPE[bits]).copy()
            vals[::2] = grey[rng.integers(0, len(grey), len(vals[::2]))].astype(cw.DTYPE[bits]) << (bits - 8)
            raw = np.frombuffer(vals.tobytes(), np.uint8)
        px.append(dict(pixels=raw.tobytes(), **fields(im)))
    for b, p in zip(pngb200.pack_batch(ctx, px, target), px):
        assert b == cw.pack(p["pixels"], target, **fields(p)), (p["color"], p["depth"])


def idat_of(data: bytes) -> bytes:
    return pngio.parse(data).idat


def test_reference_scalar_outputs_on_device(pngb200, ctx):
    """png_decode_batch -> unpack(as: UInt8) -> PNG.Image(packing:) -> level-9 png_encode_batch
    reproduces the reference's BasicDecoding.v.png and BasicEncoding-luminance-rgb.png IDATs; the
    first 320 rows of BasicDecoding.png unpack to the first 320 rows of BasicDecoding.v.png"""
    names = ["BasicDecoding-top320.png", "BasicDecoding.v.png", "BasicEncoding-luminance-v.png", "BasicEncoding-luminance-rgb.png"]
    files = [open(os.path.join(COLOUR, n), "rb").read() for n in names]
    rgb, v, lum, lrgb = pngb200.png_decode_batch(ctx, files)
    assert all(x.status == 0 for x in (rgb, v, lum, lrgb))
    assert (rgb.width, rgb.height, v.width, v.height) == (800, 320, 800, 1149)
    ((st, top),) = pngb200.unpack_batch(ctx, [dict(storage=rgb.storage, **rgb.fields)], pngb200.TARGET_V8)
    assert st == 0 and top == v.storage[: 800 * 320]
    ((st, v8),) = pngb200.unpack_batch(ctx, [dict(storage=v.storage, **v.fields)], pngb200.TARGET_V8)
    assert st == 0 and v8 == v.storage
    ((st, l8),) = pngb200.unpack_batch(ctx, [dict(storage=lrgb.storage, **lrgb.fields)], pngb200.TARGET_V8)
    assert st == 0 and l8 == lum.storage
    packed = pngb200.pack_batch(ctx, [dict(pixels=v8, color=0, depth=8), dict(pixels=lum.storage, color=2, depth=8)],
                                pngb200.TARGET_V8)
    assert packed[1] == lrgb.storage
    assert packed[0] == v.storage
    enc = pngb200.png_encode_batch(ctx, [dict(storage=packed[0], width=v.width, height=v.height, color=0, depth=8),
                                         dict(storage=packed[1], width=lum.width, height=lum.height, color=2, depth=8)], level=9)
    assert [s for s, _ in enc] == [0, 0]
    assert idat_of(enc[0][1]) == idat_of(files[1])
    assert idat_of(enc[1][1]) == idat_of(files[3])


def device_call(pngb200, ctx, unpack, target, mode, storage_ptr, s_len, pixels_ptr, p_len, count, f, keep):
    import torch
    d = (pngb200.ColorDesc * 1)()
    d[0].storage, d[0].storage_len = storage_ptr, s_len
    d[0].pixels, d[0].pixels_len = pixels_ptr, p_len
    d[0].count = count
    pngb200._fill_format(d[0].format, keep, f["color"], f["depth"], f.get("bgr"), f.get("key"), f.get("palette"))
    torch.cuda.synchronize()
    if unpack:
        rc = ctx._lib.pngb200_unpack_batch(ctx.handle, d, 1, target, mode, pngb200.MEM_DEVICE)
    else:
        rc = ctx._lib.pngb200_pack_batch(ctx.handle, d, 1, target, pngb200.MEM_DEVICE)
    return rc, d[0].status


GUARD = 0xA5


@pytest.mark.parametrize("target,p_off", [(8, 0), (8, 1), (8, 3), (9, 0), (9, 2), (10, 4), (11, 8), (6, 8), (4, 16), (5, 16), (7, 16)])
def test_device_memspace_offsets_and_guards(pngb200, ctx, target, p_off):
    """DEVICE pointers at unaligned offsets, several tiles per CTA, guard bytes on both sides untouched"""
    import torch
    rng = np.random.default_rng(target * 31 + p_off)
    n = 7680 * 64 + 13
    tb = cw.target_bytes(target)
    for f in (dict(color=6, depth=16), dict(color=0, depth=8), dict(color=3, depth=8, palette=bytes(range(256)) * 4)):
        bpp = cw.CHANNELS[f["color"]] * (2 if f["depth"] == 16 else 1)
        st = rng.integers(0, 256, n * bpp, dtype=np.uint8).tobytes()
        want = cw.unpack(st, target, **f)[1]
        for s_off in (1, 8):
            keep = []
            s_buf = torch.full((n * bpp + 64,), GUARD, dtype=torch.uint8, device="cuda")
            s_buf[s_off:s_off + n * bpp] = torch.frombuffer(bytearray(st), dtype=torch.uint8).cuda()
            p_buf = torch.full((n * tb + 64,), GUARD, dtype=torch.uint8, device="cuda")
            rc, status = device_call(pngb200, ctx, True, target, 0, s_buf.data_ptr() + s_off, n * bpp,
                                     p_buf.data_ptr() + p_off, n * tb, n, f, keep)
            assert rc == 0 and status == 0
            out = p_buf.cpu().numpy()
            assert out[p_off:p_off + n * tb].tobytes() == want, (f, s_off)
            assert (out[:p_off] == GUARD).all() and (out[p_off + n * tb:] == GUARD).all(), (f, s_off)
            # and back: pack from the same pixel buffer into a guarded storage
            s_back = torch.full((n * bpp + 64,), GUARD, dtype=torch.uint8, device="cuda")
            rc, status = device_call(pngb200, ctx, False, target, 0, s_back.data_ptr() + s_off, n * bpp,
                                     p_buf.data_ptr() + p_off, n * tb, n, f, keep)
            assert rc == 0 and status == 0
            got = s_back.cpu().numpy()
            assert got[s_off:s_off + n * bpp].tobytes() == cw.pack(want, target, **f), (f, s_off)
            assert (got[:s_off] == GUARD).all() and (got[s_off + n * bpp:] == GUARD).all(), (f, s_off)


def test_device_rgba64_alignment(pngb200, ctx):
    import torch
    n = 1001
    st = np.random.default_rng(9).integers(0, 256, n * 4, dtype=np.uint8)
    s = torch.from_numpy(st).cuda()
    out = torch.zeros(n * 32 + 16, dtype=torch.uint8, device="cuda")
    keep = []
    f = dict(color=6, depth=8)
    assert out.data_ptr() % 16 == 0
    rc, status = device_call(pngb200, ctx, True, pngb200.TARGET_RGBA64, pngb200.ALPHA_PREMULTIPLIED, s.data_ptr(), n * 4,
                             out.data_ptr(), n * 32, n, f, keep)
    assert rc == 0 and status == 0
    assert out[: n * 32].cpu().numpy().tobytes() == cw.unpack(st.tobytes(), 5, 1, **f)[1]
    rc, _ = device_call(pngb200, ctx, True, pngb200.TARGET_RGBA64, 0, s.data_ptr(), n * 4, out.data_ptr() + 8, n * 32, n, f, keep)
    assert rc == pngb200.ERR_BAD_ARGUMENT
    rc, _ = device_call(pngb200, ctx, False, pngb200.TARGET_RGBA64, 0, s.data_ptr(), n * 4, out.data_ptr() + 8, n * 32, n, f, keep)
    assert rc == pngb200.ERR_BAD_ARGUMENT


def test_palette_index_and_bad_arguments(pngb200, ctx):
    pal = bytes([1, 2, 3, 255, 4, 5, 6, 128])
    for target in cw.NEW_TARGETS:
        got = pngb200.unpack_batch(ctx, [dict(storage=bytes([0, 1, 2]), color=3, depth=8, palette=pal),
                                         dict(storage=bytes([1, 0]), color=3, depth=8, palette=pal)], target)
        assert got[0][0] == pngb200.ERR_PNG_PALETTE_INDEX
        assert got[1] == cw.unpack(bytes([1, 0]), target, color=3, depth=8, palette=pal)
    rgba8 = [dict(storage=b"\0" * 4, color=6, depth=8)]
    for target, mode in ((pngb200.TARGET_V8, pngb200.ALPHA_PREMULTIPLIED), (pngb200.TARGET_V64, pngb200.ALPHA_STRAIGHTENED),
                         (pngb200.TARGET_RGBA16, pngb200.ALPHA_PREMULTIPLIED_AS16),
                         (pngb200.TARGET_VA32, pngb200.ALPHA_PREMULTIPLIED_AS32),
                         (pngb200.TARGET_RGBA32, pngb200.ALPHA_STRAIGHTENED_AS32),
                         (pngb200.TARGET_RGBA8, pngb200.ALPHA_PREMULTIPLIED_AS8), (pngb200.TARGET_RGBA64, 9)):
        with pytest.raises(pngb200.PNGB200Error):
            pngb200.unpack_batch(ctx, rgba8, target, mode)
    # target 12 does not exist, in either direction
    buf = C.create_string_buffer(64)
    d = (pngb200.ColorDesc * 1)()
    d[0].storage, d[0].storage_len, d[0].pixels, d[0].pixels_len, d[0].count = C.addressof(buf), 4, C.addressof(buf) + 32, 32, 1
    d[0].format.color, d[0].format.depth = 6, 8
    assert ctx._lib.pngb200_unpack_batch(ctx.handle, d, 1, 12, 0, pngb200.MEM_HOST) == pngb200.ERR_BAD_ARGUMENT
    assert ctx._lib.pngb200_pack_batch(ctx.handle, d, 1, 12, pngb200.MEM_HOST) == pngb200.ERR_BAD_ARGUMENT
    # the widest valid combinations are accepted
    for target, mode in ((pngb200.TARGET_RGBA64, pngb200.ALPHA_STRAIGHTENED_AS32), (pngb200.TARGET_VA32, pngb200.ALPHA_PREMULTIPLIED_AS16)):
        assert pngb200.unpack_batch(ctx, rgba8, target, mode)[0][0] == 0
