"""context_assign_batch_kernel (online decoding: the assign launch of many contexts' pushes at once, csrc/unfilter.cuh)
under the host SIMT emulator.  Several images of every depth, volumes from 1 to 64 bits, plain and Adam7, take their
rows in random pushes; launch k of a push assigns the k-th pass range of every image, as the library launches it, with
overdraw on and off per image and on budgets far below the tiles.  After every launch each image's storage equals the
Python overdraw model and the same ranges run one at a time through context_assign_kernel.  Lanes run in order,
reversed and shuffled."""
from __future__ import annotations

import ctypes as C
import os
import random
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "emu"))
import emu  # noqa: E402
from png_context_cases import OverdrawModel, none_stream, random_storage, row_ends  # noqa: E402

ORDERS = (0, 1, 7)
POISON = 0xA5
U64P = C.POINTER(C.c_uint64)


def lib():
    L = emu.load("emu_png_context_batch")
    L.emu_context_assign_batch.argtypes = [C.c_int, C.POINTER(C.c_int), U64P, U64P, C.POINTER(C.c_void_p),
                                           C.POINTER(C.c_void_p), C.POINTER(C.c_uint32), C.POINTER(C.c_int), C.c_uint,
                                           C.c_int, U64P]
    L.emu_context_assign_one.argtypes = [C.c_int, C.c_uint64, C.c_uint64, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32),
                                         C.c_int, C.c_uint, C.c_int, U64P]
    return L


class Image:
    """one context's image: its filtered stream, its storage (batch) and a twin storage (one range at a time), both
    fenced by poison, and the overdraw model"""

    def __init__(self, w, h, volume, depth, interlaced, seed):
        self.w, self.h, self.volume, self.depth, self.interlaced = w, h, volume, depth, interlaced
        final = random_storage(w, h, volume, depth, seed)
        stream = none_stream(final, w, h, volume, depth, interlaced)
        self.src = (C.c_uint8 * (len(stream) + 16)).from_buffer_copy(stream + bytes(16))
        self.size = len(final)
        fenced = bytes([POISON]) * 32 + bytes(self.size) + bytes([POISON]) * 32
        self.buf = (C.c_uint8 * len(fenced)).from_buffer_copy(fenced)
        self.twin = (C.c_uint8 * len(fenced)).from_buffer_copy(fenced)
        self.model = OverdrawModel(w, h, volume, interlaced, final)
        self.ends = row_ends(w, h, volume, interlaced)
        self.next = 0
        self.geometry = (C.c_uint32 * 5)(w, h, volume, depth, int(interlaced))

    def storage(self, buf):
        raw = bytes(buf)
        assert raw[:32] == bytes([POISON]) * 32 and raw[32 + self.size:] == bytes([POISON]) * 32, "written outside"
        return raw[32:32 + self.size]


def push_ranges(img, count):
    """the next `count` rows of the image, as per-pass ranges in pass order"""
    rows = img.ends[img.next:img.next + count]
    img.next += len(rows)
    out = []
    for z, r, _ in rows:
        if out and out[-1][0] == z:
            out[-1][2] = r + 1
        else:
            out.append([z, r, r + 1])
    return out


def run(images, rng, order, max_ctas):
    """pushes until every image is complete; checks after every launch"""
    L = lib()
    while any(img.next < len(img.ends) for img in images):
        plan = []
        for img in images:
            od = rng.random() < 0.5
            ranges = push_ranges(img, rng.choice((0, 1, 2, 5, 17, 64))) if img.next < len(img.ends) else []
            plan.append((img, ranges, od))
        for k in range(7):
            batch = [(img, ranges[k], od) for img, ranges, od in plan if len(ranges) > k]
            if not batch:
                break
            n = len(batch)
            zs = (C.c_int * n)(*[r[0] for _, r, _ in batch])
            r0 = (C.c_uint64 * n)(*[r[1] for _, r, _ in batch])
            r1 = (C.c_uint64 * n)(*[r[2] for _, r, _ in batch])
            src = (C.c_void_p * n)(*[C.addressof(img.src) for img, _, _ in batch])
            dst = (C.c_void_p * n)(*[C.addressof(img.buf) + 32 for img, _, _ in batch])
            geo = (C.c_uint32 * (5 * n))(*[v for img, _, _ in batch for v in img.geometry])
            ods = (C.c_int * n)(*[int(od) for _, _, od in batch])
            y = (C.c_uint64 * (2 * n))()
            L.emu_context_assign_batch(n, zs, r0, r1, src, dst, geo, ods, max_ctas, order, y)
            for i, (img, (z, a, b), od) in enumerate(batch):
                one = (C.c_uint64 * 2)()
                L.emu_context_assign_one(z, a, b, C.addressof(img.src), C.addressof(img.twin) + 32, img.geometry, int(od),
                                         max_ctas, order, one)
                assert (y[2 * i], y[2 * i + 1]) == tuple(one), (z, a, b)
                for r in range(a, b):
                    img.model.row(z, r, od)
                want = img.model.storage()
                assert img.storage(img.buf) == want, (img.w, img.h, img.volume, img.interlaced, z, a, b, od)
                assert img.storage(img.twin) == want


MIXES = [
    # (w, h, volume, depth, interlaced)
    [(9, 11, 1, 1, True), (13, 7, 2, 2, True), (17, 9, 4, 4, False), (21, 19, 8, 8, True), (5, 3, 16, 16, True)],
    [(37, 13, 24, 8, True), (11, 23, 32, 8, False), (19, 17, 48, 16, True), (7, 29, 64, 16, True), (1, 9, 16, 8, True)],
    [(257, 9, 32, 8, True), (263, 5, 1, 1, True), (3, 2, 8, 8, True), (40, 40, 2, 2, False), (33, 8, 4, 4, True)],
]


@pytest.mark.parametrize("mix", range(len(MIXES)))
@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("max_ctas", [3, 16, 2112])
def test_mixed_batches(mix, order, max_ctas):
    """every image of the mix pushed to completion in random row counts, overdraw drawn per image and push"""
    rng = random.Random(100 * mix + 10 * order + max_ctas)
    images = [Image(*g, seed=31 * mix + i) for i, g in enumerate(MIXES[mix])]
    run(images, rng, order, max_ctas)


def test_one_context_equals_the_single_kernel():
    """a batch of one image is the single launch: the same CTA count and the same storage"""
    L = lib()
    img = Image(45, 21, 24, 8, True, seed=5)   # passes 0-2 have 3 rows, pass 6 has 10
    for budget in (1, 4, 2112):
        for a, b, z in ((0, 3, 0), (1, 3, 1), (0, 3, 2), (2, 10, 6)):
            zs, r0, r1 = (C.c_int * 1)(z), (C.c_uint64 * 1)(a), (C.c_uint64 * 1)(b)
            src = (C.c_void_p * 1)(C.addressof(img.src))
            dst = (C.c_void_p * 1)(C.addressof(img.buf) + 32)
            y, one = (C.c_uint64 * 2)(), (C.c_uint64 * 2)()
            ctas = L.emu_context_assign_batch(1, zs, r0, r1, src, dst, img.geometry, (C.c_int * 1)(1), budget, 0, y)
            assert ctas == L.emu_context_assign_one(z, a, b, C.addressof(img.src), C.addressof(img.twin) + 32,
                                                    img.geometry, 1, budget, 0, one)
            assert tuple(y) == tuple(one) and img.storage(img.buf) == img.storage(img.twin)
