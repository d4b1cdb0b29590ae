"""The reconstruct arithmetic of the JPEG kernels (dali_b200/csrc/jpeg_idct_core.h), run on the host through
tools/emul/jpeg_idct_emul.cc:
  - the whole-block IDCT (idct_kernel, idct_color_420, the decode half of fn.jpeg_compression_distortion) against the numpy statement
    of libjpeg-turbo's SIMD islow IDCT (tests/jpeg_idct16.py), on random blocks and at the extremes (DQT up to 65535, coefficients at
    +-32767, blocks whose rows 1..7 are zero);
  - idct_color_420's column-parallel halo path against columns 0 and 7 of the whole block;
  - idct_color_420's colour unit (packed 16-bit upsampling sums, folded constants) against libjpeg's h2v2 fancy upsampling and
    fixed-point YCbCr -> RGB / BGR formulas: every (Y, Cb, Cr) triple, random chroma, and the image's first and last chroma column,
    whose missing neighbour the kernel supplies as a copy of the column."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from jpeg_idct16 import idct16  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tools", "emul", "jpeg_idct_emul.cc")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp_path_factory.mktemp("idct_emul") / "libidctemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-shared", "-fPIC", EMUL, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(out)
    for f in (lib.emul_idct_blocks, lib.emul_idct_halo):
        f.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.emul_color_units.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    return lib


def _blocks(rng, n):
    """random blocks at every range the tests of tests/jpeg_idct16.py use: natural, wide, extreme and mostly-zero"""
    coef = np.zeros((n, 64), np.int64)
    q = np.zeros((n, 64), np.int64)
    k = n // 6
    coef[:k] = rng.integers(-64, 65, (k, 64)); q[:k] = rng.integers(1, 100, (k, 64))
    coef[k:2 * k] = rng.integers(-2048, 2048, (k, 64)); q[k:2 * k] = rng.integers(1, 256, (k, 64))
    coef[2 * k:3 * k] = rng.integers(-32768, 32768, (k, 64)); q[2 * k:3 * k] = rng.integers(0, 65536, (k, 64))
    coef[3 * k:4 * k] = rng.choice([-32768, -32767, 32767, 0, 1, -1], (k, 64)); q[3 * k:4 * k] = rng.choice([1, 255, 65535], (k, 64))
    # rows 1..7 zero (the SIMD kernels' pass-1 skip), row 0 anywhere
    coef[4 * k:5 * k, :8] = rng.integers(-32768, 32768, (k, 8)); q[4 * k:5 * k] = rng.integers(0, 65536, (k, 64))
    # sparse: a few coefficients, rows 1..7 sometimes touched only by one
    m = n - 5 * k
    q[5 * k:] = rng.integers(1, 65536, (m, 64))
    coef[5 * k:, 0] = rng.integers(-32768, 32768, m)
    pos = rng.integers(1, 64, m)
    coef[5 * k + np.arange(m), pos] = rng.integers(-32768, 32768, m)
    return coef, q


def _run_blocks(emul, coef, q):
    c16 = np.ascontiguousarray(coef.astype(np.int16))
    q16 = np.ascontiguousarray(np.broadcast_to(q, coef.shape).astype(np.uint16))
    out = np.zeros((len(coef), 64), np.uint8)
    emul.emul_idct_blocks(c16.ctypes.data, q16.ctypes.data, len(coef), out.ctypes.data)
    halo = np.zeros((len(coef), 16), np.uint8)
    emul.emul_idct_halo(c16.ctypes.data, q16.ctypes.data, len(coef), halo.ctypes.data)
    return out.reshape(-1, 8, 8), halo


def test_pass_sums_fit_32_bits():
    # the largest |t1x +- o_k| of one pass over int16 inputs (jpeg_idct_core.h, idct8) plus pass 2's rounding constant fits 32 bits;
    # with pass 2's + 128 folded in as well (128 << 18) it would not
    t = 32768 * 8192 + 32768 * (10703 + 4433)
    o = 32768 * max(4927 + 7373, 7373 + 4926, 4176 + 20995, 20995 + 4177) + 32768 * max(6436 + 9633, 9633 + 6437)
    assert t + o + (1 << 17) == 2115960832 < 2 ** 31 <= t + o + (1 << 17) + (128 << 18)


def test_blocks_and_halo_equal_idct16(emul):
    rng = np.random.default_rng(7)
    for _ in range(4):
        coef, q = _blocks(rng, 30000)
        got, halo = _run_blocks(emul, coef, q)
        want = idct16(coef, q)
        bad = np.nonzero((got != want).any(axis=(1, 2)))[0]
        assert bad.size == 0, (bad[:5], coef[bad[0]], q[bad[0]])
        assert np.array_equal(halo[:, :8], want[:, :, 0]) and np.array_equal(halo[:, 8:], want[:, :, 7])


def test_blocks_at_the_extremes(emul):
    # every coefficient at one extreme, every table entry at one extreme, the DC alone, one AC alone at every position
    vals = [-32768, -32767, -1, 1, 32767]
    qs = [0, 1, 255, 256, 65535]
    coef, q = [], []
    for v in vals:
        for qq in qs:
            coef.append(np.full(64, v)); q.append(np.full(64, qq))
            dc = np.zeros(64, np.int64); dc[0] = v
            coef.append(dc); q.append(np.full(64, qq))
            for p in range(1, 64):
                one = np.zeros(64, np.int64); one[0] = -v; one[p] = v
                coef.append(one); q.append(np.full(64, qq))
    coef, q = np.array(coef), np.array(q)
    got, halo = _run_blocks(emul, coef, q)
    want = idct16(coef, q)
    assert np.array_equal(got, want)
    assert np.array_equal(halo[:, :8], want[:, :, 0]) and np.array_equal(halo[:, 8:], want[:, :, 7])


def _color_ref(tiles, y, i0, dw, bgr):
    """libjpeg: h2v2 fancy upsampling of the 10 chroma columns i0 - 1 .. i0 + 8 (jdsample.c, edge columns their own neighbours) and
    jdcolor.c's YCbCr -> RGB, clamped; tiles [n, 4, 10] = (s0 near, s0 far, s2 near, s2 far), s0 = Cb for BGR, Cr for RGB"""
    cs = 3 * tiles[:, 0::2].astype(np.int64) + tiles[:, 1::2]          # [n, 2, 10]: cs of channel-0 and channel-2 chroma
    i = i0[:, None] + np.arange(8)[None]                                 # chroma columns of the unit
    cur = cs[:, :, 1:9]
    prev = np.where((i == 0)[:, None], cur, cs[:, :, 0:8])
    nxt = np.where((i >= dw[:, None] - 1)[:, None], cur, cs[:, :, 2:10])
    up = np.empty(cs.shape[:2] + (16,), np.int64)
    up[:, :, 0::2] = (3 * cur + prev + 8) >> 4
    up[:, :, 1::2] = (3 * cur + nxt + 7) >> 4
    cb, cr = (up[:, 0], up[:, 1]) if bgr else (up[:, 1], up[:, 0])
    yy = y.astype(np.int64)
    r = yy + ((91881 * (cr - 128) + 32768) >> 16)
    g = yy + ((-22554 * (cb - 128) + 32768 - 46802 * (cr - 128)) >> 16)
    b = yy + ((116130 * (cb - 128) + 32768) >> 16)
    px = np.stack([b, g, r] if bgr else [r, g, b], -1)
    return np.clip(px, 0, 255).astype(np.uint8).reshape(len(y), 48)


def _color_emul(emul, tiles, y, bgr):
    tiles = np.ascontiguousarray(tiles, np.uint8)
    y = np.ascontiguousarray(y, np.uint8)
    out = np.zeros((len(y), 48), np.uint8)
    emul.emul_color_units(tiles.ctypes.data, y.ctypes.data, len(y), int(bgr), out.ctypes.data)
    return out


def _edge_copy(tiles, i0, dw):
    """idct_color_420: the column left of chroma column 0 and right of column dw - 1 hold a copy of that column"""
    t = tiles.copy()
    left = i0 == 0
    t[left, :, 0] = t[left, :, 1]
    k = dw - 1 - i0                                                     # unit-relative column of dw - 1
    inside = (k >= 0) & (k < 8)
    rows = np.nonzero(inside)[0]
    t[rows, :, k[rows] + 2] = t[rows, :, k[rows] + 1]
    return t


@pytest.mark.parametrize("bgr", [False, True])
def test_color_unit_every_triple(emul, bgr):
    # constant chroma upsamples to itself, so 16 units per (Cb, Cr) pair cover all 256 luma values
    cb, cr = np.meshgrid(np.arange(256), np.arange(256), indexing="ij")
    cb, cr = np.repeat(cb.ravel(), 16), np.repeat(cr.ravel(), 16)
    s0, s2 = (cb, cr) if bgr else (cr, cb)
    n = len(cb)
    tiles = np.empty((n, 4, 10), np.uint8)
    tiles[:, 0:2] = s0[:, None, None]
    tiles[:, 2:4] = s2[:, None, None]
    y = (np.arange(n)[:, None] % 16 * 16 + np.arange(16)[None]).astype(np.uint8)
    i0 = np.full(n, 8); dw = np.full(n, 1000)
    assert np.array_equal(_color_emul(emul, tiles, y, bgr), _color_ref(tiles, y, i0, dw, bgr))


@pytest.mark.parametrize("bgr", [False, True])
def test_color_unit_random_and_edges(emul, bgr):
    rng = np.random.default_rng(11)
    n = 200000
    tiles = rng.integers(0, 256, (n, 4, 10)).astype(np.uint8)
    pick = rng.integers(0, 4, n)                                         # some units of extreme chroma: 0 / 255 patterns
    ext = pick == 0
    tiles[ext] = rng.choice([0, 255], (int(ext.sum()), 4, 10)).astype(np.uint8)
    y = rng.integers(0, 256, (n, 16)).astype(np.uint8)
    y[pick == 1] = rng.choice([0, 255], (int((pick == 1).sum()), 16)).astype(np.uint8)
    # units at the image's first chroma column, at its last one (every position in the unit), and inside
    i0 = 8 * rng.integers(1, 100, n)
    dw = i0 + rng.integers(9, 50, n)
    first = rng.random(n) < 0.25
    i0[first] = 0
    dw[first] = rng.integers(3, 40, int(first.sum()))
    last = rng.random(n) < 0.4
    dw[last] = i0[last] + rng.integers(1, 9, int(last.sum()))
    dw = np.maximum(dw, 3)
    ref = _color_ref(tiles, y, i0, dw, bgr)
    got = _color_emul(emul, _edge_copy(tiles, i0, dw), y, bgr)
    # pixels at or beyond the image's width (x >= 2 dw) are never stored: compare the image's pixels only
    x = 2 * i0[:, None] + np.arange(16)[None]
    keep = np.repeat(x < 2 * dw[:, None], 3, axis=1)
    assert np.array_equal(np.where(keep, got, 0), np.where(keep, ref, 0))
    assert (first & last).any() and first.any() and last.any()
