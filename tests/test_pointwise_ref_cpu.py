"""Pins the numpy references of tests/pointwise_ref.py, which the GPU tests of the decoder's output types and of brightness_contrast
compare with: the u8 YCbCr form equals the oracle's BT.601 conversion over the whole RGB cube, each float32 form agrees with its
float64 statement over every input and an argument grid, and, where the reference's compiled kernels exist, both equal them bit for
bit."""
import itertools

import numpy as np
import pytest

import pointwise_ref as pr
from oracle import pyoracle as po


def _cube_chunks(rows=16):
    """the 2^24 RGB triples, `rows` values of R at a time, as (rows * 256, 256, 3) images"""
    g, b = np.meshgrid(np.arange(256, dtype=np.uint8), np.arange(256, dtype=np.uint8), indexing="ij")
    gb = np.stack([g, b], -1)
    for r0 in range(0, 256, rows):
        r = np.repeat(np.arange(r0, r0 + rows, dtype=np.uint8), 256 * 256).reshape(rows * 256, 256, 1)
        yield np.concatenate([r, np.tile(gb, (rows, 1, 1))], -1)


def test_decoder_ycbcr_over_the_rgb_cube(oracle):
    guarded, worst = 0, 0.0
    for img in _cube_chunks():
        u8 = pr.decoder_convert(img, pr.YCBCR, False)
        assert np.array_equal(u8, oracle.csc(img, oracle.IT_RGB, oracle.IT_YCBCR))
        guarded += pr.assert_u8_matches_f64(u8, pr.decoder_convert_f64(img, pr.YCBCR, False), what="u8 YCbCr")
        f32 = pr.decoder_convert(img, pr.YCBCR, True)
        worst = max(worst, float(np.abs(f32.astype(np.float64) - pr.decoder_convert_f64(img, pr.YCBCR, True)).max()))
    assert guarded <= 1000, guarded                                                  # of 3 * 2^24
    assert worst <= 2e-7, worst


def test_decoder_rgb_bgr_gray_forms():
    v = np.arange(256, dtype=np.uint8)
    img = np.stack([v, v[::-1], (v * 7).astype(np.uint8)], -1).reshape(16, 16, 3)
    for ot in (pr.RGB, pr.BGR):
        assert np.array_equal(pr.decoder_convert(img, ot, False), img if ot == pr.RGB else img[..., ::-1])
        f = pr.decoder_convert(img, ot, True)
        assert f.dtype == np.float32 and np.array_equal(f, (img if ot == pr.RGB else img[..., ::-1]) * np.float32(1 / 255))
        pr.assert_f32_close(f, pr.decoder_convert_f64(img, ot, True), 1.5e-7)
    gray = v.reshape(16, 16, 1)
    assert np.array_equal(pr.decoder_convert(gray, pr.GRAY, False), gray)
    f = pr.decoder_convert(gray, pr.GRAY, True)
    assert f[1, 0, 0] == np.float32(16) * np.float32(1 / 255) and f[15, 15, 0] == np.float32(1.0)
    pr.assert_f32_close(f, pr.decoder_convert_f64(gray, pr.GRAY, True), 1.5e-7)
    # a grayscale stream decoded to YCbCr is the RGB formula with R = G = B: Y is not v itself, Cb / Cr are not exactly 128
    rep = np.repeat(gray, 3, -1)
    y = pr.decoder_convert(rep, pr.YCBCR, False)
    assert y[0, 0].tolist() == [16, 128, 128] and y[15, 15].tolist() == [235, 128, 128]


# arguments whose products rarely land within 1e-4 of a half (0.1 * 255 = 25.4999996 in float64 but 25.5 in float32, for instance)
BC_GRID = list(itertools.product((0.0, 0.5, 1.0, 1.37, 2.1, 3.0), (-1.0, -0.137, 0.0, 0.0731, 1.0), (0.0, 0.31, 0.77, 1.0, 1.5),
                                 (128.0, 100.0, 0.0, 253.7)))


def _bc_tol(b, s, c, ctr, out_float):
    """a few float32 roundings of the largest magnitude that enters the float32 form"""
    b, s, c, ctr = (abs(float(np.float32(x))) for x in (b, s, c, ctr))
    return 4 * 2.0 ** -24 * (255 * b * c + b * (ctr + c * ctr) + s * (1 if out_float else 255) + 1)


def test_brightness_contrast_forms_over_all_inputs_and_an_argument_grid():
    v = np.arange(256, dtype=np.uint8).reshape(16, 16)
    guarded = 0
    for b, s, c, ctr in BC_GRID:
        f32 = pr.brightness_contrast(v, b, s, c, ctr, out_float=True)
        assert f32.dtype == np.float32
        pr.assert_f32_close(f32, pr.brightness_contrast_f64(v, b, s, c, ctr, out_float=True), _bc_tol(b, s, c, ctr, True), (b, s, c, ctr))
        u8 = pr.brightness_contrast(v, b, s, c, ctr)
        guarded += pr.assert_u8_matches_f64(u8, pr.brightness_contrast_f64(v, b, s, c, ctr), what=(b, s, c, ctr))
    assert guarded <= 100, guarded                                                   # of 153 600
    half = pr.brightness_contrast(v, 0.5, 0.0, 1.0)
    assert np.array_equal(half.astype(np.int64), (v.astype(np.int64) + 1) // 2)          # round half AWAY: 1 -> 1, 3 -> 2, 255 -> 128
    assert pr.brightness_contrast_args(1.0, 0.0, 0.9)[1] == np.float32(1.0) * (np.float32(128) - np.float32(0.9) * np.float32(128))


@pytest.mark.skipif(not po.have_ref(), reason="needs oracle/_ref")
def test_forms_equal_the_reference_kernels():
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (64, 256, 3), dtype=np.uint8)
    img[0, :, :] = np.arange(256, dtype=np.uint8)[:, None]
    for it in (po.IT_RGB, po.IT_BGR, po.IT_YCBCR):
        for fl in (False, True):
            want = po.ref_decoder_convert(img, it, fl)
            got = pr.decoder_convert(img, it, fl)
            assert got.dtype == want.dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8)), (it, fl)
    gray = img[..., :1].copy()
    for fl in (False, True):
        assert np.array_equal(pr.decoder_convert(gray, pr.GRAY, fl).view(np.uint8), po.ref_decoder_convert(gray, po.IT_GRAY, fl).view(np.uint8))
    v = np.arange(256, dtype=np.uint8)
    for b, s, c, ctr in BC_GRID:
        for fl in (False, True):
            want = po.ref_brightness_contrast(v, b, s, c, ctr, out_float=fl)
            got = pr.brightness_contrast(v, b, s, c, ctr, out_float=fl)
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (b, s, c, ctr, fl)
