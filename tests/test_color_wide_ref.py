"""Pins the wide and scalar colour targets (RGBA / VA at 32 and 64 bits, image.unpack(as: T.self) /
PNG.Image(packing: [T]) for T = UInt8 ... UInt64) on the CPU: the Python restatement in colorwide.py
against the C oracle where they overlap, against the reference's PngSuite and CgBI goldens through exact
width identities, against the reference's own scalar decode / encode outputs, and against the
Premultiplication suite's identities at 32 and 64 bits."""
import hashlib
import json
import os

import numpy as np
import pytest

import colorwide as cw
import pngio
from conftest import GOLDEN

PNGSUITE = sorted(f for f in os.listdir(os.path.join(GOLDEN, "pngsuite")) if f.endswith(".png"))
IOS = sorted(f for f in os.listdir(os.path.join(GOLDEN, "ios")) if f.endswith(".png"))
DIGESTS = json.load(open(os.path.join(GOLDEN, "pngsuite_rgba.json")))
IOS_DIGESTS = json.load(open(os.path.join(GOLDEN, "ios_rgba.json")))
COLOUR = os.path.join(GOLDEN, "colour")
# 2^d - 1 divides 2^16 - 1 for every PNG depth, so a T-bit component is the 16-bit one times these
SCALE = {32: 0x00010001, 64: 0x0001000100010001}


def load(orc, sub, name):
    png = pngio.parse(open(os.path.join(GOLDEN, sub, name), "rb").read())
    st, storage, _ = orc.png_decode(png.idat, png.width, png.height, png.volume, png.depth,
                                    png.interlaced, fmt=png.fmt)
    assert st == orc.OK
    return png, storage, pngio.format_fields(png)


def decompress(orc, path):
    info, storage = orc.png_decompress(open(path, "rb").read())
    assert storage is not None, path
    return info, storage


def as_rows(px: bytes, target: int) -> np.ndarray:
    bits, shape = cw.TARGETS[target]
    return np.frombuffer(px, cw.DTYPE[bits]).reshape(-1, cw.WIDTH[shape])


def test_restatement_matches_oracle_on_the_shared_targets(orc):
    """colorwide restates the C oracle exactly on RGBA8 / RGBA16 / VA8 / VA16, every alpha mode"""
    for name in PNGSUITE[::3]:
        _, storage, f = load(orc, "pngsuite", name)
        fmt = orc.make_format(**f)
        for target in range(4):
            for mode in cw.modes(target):
                assert cw.unpack(storage, target, mode, **f) == orc.unpack(storage, fmt, target, mode), (name, target, mode)
            px = orc.unpack(storage, fmt, target)[1]
            assert cw.pack(px, target, **f) == orc.pack(px, fmt, target), (name, target)
    rng = np.random.default_rng(3)
    for target in range(4):  # random pixels, including colours missing from a palette
        px = rng.integers(0, 256, 301 * cw.target_bytes(target), dtype=np.uint8).tobytes()
        for f in (dict(color=6, depth=16), dict(color=2, depth=8, bgr=True), dict(color=0, depth=2),
                  dict(color=3, depth=8, palette=bytes(rng.integers(0, 4, 4 * 40, dtype=np.uint8)))):
            assert cw.pack(px, target, **f) == orc.pack(px, orc.make_format(**f), target), (target, f)


@pytest.mark.parametrize("name", PNGSUITE)
def test_wide_targets_scale_the_rgba16_golden(orc, name):
    """RGBA<UInt16> is the reference's golden; every new target follows from it exactly"""
    _, storage, f = load(orc, "pngsuite", name)
    st, rgba16 = orc.unpack(storage, orc.make_format(**f), orc.TARGET_RGBA16)
    assert st == 0 and hashlib.sha256(rgba16).hexdigest() == DIGESTS[name]["sha256"]
    w16 = np.frombuffer(rgba16, "<u2").reshape(-1, 4).astype(np.uint64)
    want = {4: w16 * SCALE[32], 5: w16 * SCALE[64], 6: w16[:, [0, 3]] * SCALE[32], 7: w16[:, [0, 3]] * SCALE[64],
            8: w16[:, :1] >> 8, 9: w16[:, :1], 10: w16[:, :1] * SCALE[32], 11: w16[:, :1] * SCALE[64]}
    for target, rows in want.items():
        st, px = cw.unpack(storage, target, **f)
        assert st == 0 and np.array_equal(as_rows(px, target), rows), target
        # pack inverts unpack: exactly for RGBA, and up to what the target drops for VA / scalar
        if f["color"] != 3 and f["key"] is None:
            back = cw.pack(px, target, **f)
            assert cw.unpack(back, target, **f) == (0, px), target
            if cw.TARGETS[target][1] == "rgba":
                assert back == storage, target


def test_premultiplied_as8_at_32_and_64_bits_matches_ios_goldens(orc):
    """x >> 24 of x16 * 65537 is x16 >> 8, so premultiplied(as: UInt8) at 32 / 64 bits is the CgBI
    golden (Roundtripping.swift:206-211) scaled"""
    checked = 0
    for name in IOS:
        if name not in DIGESTS:
            continue
        _, storage, f = load(orc, "pngsuite", name)
        st, px16 = orc.unpack(storage, orc.make_format(**f), orc.TARGET_RGBA16, orc.ALPHA_PREMULTIPLIED_AS8)
        assert st == 0 and hashlib.sha256(px16).hexdigest() == IOS_DIGESTS[name]["sha256"], name
        w16 = np.frombuffer(px16, "<u2").reshape(-1, 4).astype(np.uint64)
        for target, bits in ((4, 32), (5, 64)):
            st, px = cw.unpack(storage, target, 3, **f)
            assert st == 0 and np.array_equal(as_rows(px, target), w16 * SCALE[bits]), (name, target)
        checked += 1
    assert checked > 20


@pytest.mark.parametrize("bits", [32, 64])
def test_premultiplication_identities_wide(bits):
    """Premultiplication.swift extended to 32 / 64 bits: premultiply is round(c * a / T.max) (no ties:
    T.max is odd), and premultiply . straighten . premultiply == premultiply"""
    m = cw.tmax(bits)
    rng = np.random.default_rng(bits)
    edge = [0, 1, 2, m >> 1, (m >> 1) + 1, m - 1, m]
    pairs = [(c, a) for c in edge for a in edge]
    pairs += [(int.from_bytes(rng.bytes(bits // 8), "little"), int.from_bytes(rng.bytes(bits // 8), "little")) for _ in range(4000)]
    pairs += [(int(rng.integers(0, 1 << 16)), a) for _, a in pairs[-500:]]  # small colours, wide alpha
    for c, a in pairs:
        p = cw.premultiply(c, a, bits)
        assert p == (2 * c * a + m) // (2 * m), (c, a)  # nearest integer to c * a / m
        assert p <= a
        assert cw.premultiply(cw.straighten(p, a, bits), a, bits) == p, (c, a)
    assert cw.straighten(5, 3, bits) == m  # saturates where the reference traps


def test_scalar_edge_cases(orc):
    # the scalar target ignores chroma keys (it has no alpha)
    assert cw.unpack(bytes([7, 9, 7]), 8, color=0, depth=8, key=(7,)) == (0, bytes([7, 9, 7]))
    assert cw.unpack(bytes([1, 2, 3, 4, 5, 6]), 9, color=2, depth=8, bgr=True, key=(1, 2, 3)) == \
        (0, np.array([3 * 257, 6 * 257], "<u2").tobytes())
    # palette[i].r widened; an index past the end is an error (the reference traps)
    pal = bytes([10, 20, 30, 255, 40, 50, 60, 128])
    assert cw.unpack(bytes([1, 0]), 10, color=3, depth=8, palette=pal) == \
        (0, np.array([40 * 0x01010101, 10 * 0x01010101], "<u4").tobytes())
    assert cw.unpack(bytes([0, 2]), 8, color=3, depth=8, palette=pal)[0] == cw.ERR_PALETTE_INDEX
    # indexed pack: v >> (T - 8), then the first (v8, v8, v8, 255) entry, else 0
    gray = bytes([9, 9, 9, 0, 5, 5, 5, 255, 7, 7, 7, 255, 5, 5, 5, 255])
    v16 = np.array([0x05ff, 0x0700, 0x0600, 0x0500], "<u2").tobytes()
    assert cw.pack(v16, 9, color=3, depth=8, palette=gray) == bytes([1, 2, 0, 1])
    assert cw.pack(bytes([5, 9]), 8, color=3, depth=8, palette=gray) == bytes([1, 0])
    # scalar pack: va -> (v, T.max), rgba -> (v, v, v, T.max), 16-bit depth from 8 bits x 257
    assert cw.pack(bytes([3, 200]), 8, color=4, depth=8) == bytes([3, 255, 200, 255])
    assert cw.pack(bytes([3]), 8, color=6, depth=16) == bytes([3, 3] * 3 + [255, 255])
    assert cw.pack(np.array([0xfedcba9876543210], "<u8").tobytes(), 11, color=0, depth=4) == bytes([0xf])
    # valid combinations
    assert [t for t in range(13) if cw.valid(t, 1)] == [0, 1, 2, 3, 4, 5, 6, 7]
    assert [t for t in range(12) if cw.valid(t, 5)] == [4, 5, 6, 7]
    assert [t for t in range(12) if cw.valid(t, 7)] == [5, 7]
    assert [t for t in range(12) if cw.valid(t, 3)] == [1, 3, 4, 5, 6, 7]


def test_reference_scalar_outputs(orc):
    """The reference's own scalar decode and encode outputs (its documentation's images):
    BasicDecoding.v.png is unpack(as: UInt8) of BasicDecoding.png (here its first 320 rows), written
    back at level 9, and BasicEncoding-luminance-rgb.png is PNG.Image(packing: luminance) of
    BasicEncoding-luminance-v.png."""
    info, rgb = decompress(orc, os.path.join(COLOUR, "BasicDecoding-top320.png"))
    assert (info.color, info.depth, info.width, info.height) == (2, 8, 800, 320)
    vinfo, v = decompress(orc, os.path.join(COLOUR, "BasicDecoding.v.png"))
    assert (vinfo.color, vinfo.depth, vinfo.width, vinfo.height) == (0, 8, 800, 1149)
    assert cw.unpack(rgb, 8, color=2, depth=8) == (0, v[: 800 * 320])
    stored = cw.pack(v, 8, color=0, depth=8)
    assert stored == v
    idat = pngio.parse(open(os.path.join(COLOUR, "BasicDecoding.v.png"), "rb").read()).idat
    assert pngio.parse(orc.png_compress(stored, 800, 1149, orc.make_format(0, 8), False, 9)).idat == idat

    linfo, lum = decompress(orc, os.path.join(COLOUR, "BasicEncoding-luminance-v.png"))
    rinfo, lrgb = decompress(orc, os.path.join(COLOUR, "BasicEncoding-luminance-rgb.png"))
    assert (linfo.color, linfo.depth, rinfo.color, rinfo.depth) == (0, 8, 2, 8)
    packed = cw.pack(lum, 8, color=2, depth=8)
    assert packed == lrgb
    idat = pngio.parse(open(os.path.join(COLOUR, "BasicEncoding-luminance-rgb.png"), "rb").read()).idat
    assert pngio.parse(orc.png_compress(packed, rinfo.width, rinfo.height, orc.make_format(2, 8), False, 9)).idat == idat
    assert cw.unpack(lrgb, 8, color=2, depth=8) == (0, lum)
