"""The float64 statements of tests/image_f64.py on the CPU: the float32 restatement (oracle/imgproc_oracle.c) meets every bound with at
least 4x margin, so does the reference's output in the committed golden vectors, the known answers hold, and plausible mistakes are
rejected by a wide margin.  Each test prints its worst |error| / bound (for u8 outputs: the part beyond the half-unit rounding)."""
import numpy as np
import pytest

import image_f64 as F

MARGIN = 0.25


def _scaled(b, f):
    return [f * x for x in b] if isinstance(b, list) else f * b


def _roi_pair(roi):
    """pyoracle's ((y0, x0), (y1, x1)) -> per-axis [(y0, y1), (x0, x1)]."""
    if roi is None:
        return None
    return [None if roi[0][d] is None else (roi[0][d], roi[1][d]) for d in range(2)]


def _resize_cases(rng, n):
    for it in range(n):
        H, W = [int(v) for v in rng.integers(1, 120, 2)]
        oh, ow = [int(v) for v in rng.integers(1, 150, 2)]
        C = int(rng.choice([1, 2, 3, 4, 5]))
        ft, aa = int(rng.integers(0, 6)), int(rng.integers(0, 2))
        roi = None
        if it % 3 == 0:
            roi = ((float(rng.uniform(-3, H + 3)), float(rng.uniform(-3, W + 3))), (float(rng.uniform(-3, H + 3)), float(rng.uniform(-3, W + 3))))
        yield (H, W, C), (oh, ow), (ft, aa, 0.0), roi
    # edges: extent 1 in or out, flips on x / y / both, ROI narrower than a pixel, strong down- and up-scaling
    yield (1, 37, 3), (5, 9), (F.F_CUBIC, 1, 0.0), None
    yield (40, 50, 3), (1, 1), (F.F_LINEAR, 1, 0.0), None
    yield (33, 41, 1), (17, 23), (F.F_TRIANGULAR, 1, 0.0), ((0.0, 40.5), (33.0, 0.25))
    yield (33, 41, 1), (17, 23), (F.F_LANCZOS3, 1, 0.0), ((32.0, 1.0), (2.5, 39.0))
    yield (33, 41, 4), (17, 23), (F.F_GAUSSIAN, 1, 0.0), ((30.0, 38.0), (3.0, 2.0))
    yield (20, 20, 3), (9, 11), (F.F_LINEAR, 1, 0.0), ((4.3, 7.1), (4.6, 7.3))
    yield (8, 300, 1), (3, 2), (F.F_TRIANGULAR, 1, 0.0), None
    yield (5, 6, 3), (80, 200), (F.F_CUBIC, 0, 0.0), None
    yield (48, 57, 16), (19, 23), (F.F_GAUSSIAN, 0, 0.0), ((44.0, 3.0), (0.5, 50.0))     # a window the float position may shift


def test_resize_oracle_within_bounds(oracle):
    rng = np.random.default_rng(101)
    worst = {}
    for shape, out_hw, filt, roi in _resize_cases(rng, 80):
        for in_dt in (np.uint8, np.float32):
            img = rng.integers(0, 256, shape).astype(np.uint8) if in_dt == np.uint8 else \
                (rng.normal(0, 1, shape) * rng.choice([1.0, 300.0, 1e5], shape)).astype(np.float32)   # outliers next to small values
            vals, b = F.resize(img, out_hw, _roi_pair(roi), filt, filt)
            what = (shape, out_hw, filt, roi, np.dtype(in_dt).name)
            out = oracle.resample(img, out_hw, filt, filt, np.float32, roi)
            k = ("f32", filt[0])
            worst[k] = max(worst.get(k, 0.0), F.check(out, vals, _scaled(b, MARGIN), what))
            if in_dt == np.uint8:
                out8 = oracle.resample(img, out_hw, filt, filt, np.uint8, roi)
                worst[("u8", filt[0])] = max(worst.get(("u8", filt[0]), 0.0), F.check_u8(out8, vals, _scaled(b, MARGIN), what))
    print("resize worst |err| / bound by filter:", {k: round(v * MARGIN, 4) for k, v in sorted(worst.items())})


def test_resize_exact_filter_form(oracle):
    """The continuous filters (triangle, Gaussian, Keys a = -1/2, Lanczos-3) with the table's interpolation error in the bound.

    This bound is closer to its limit than the others (about 0.3 for the cubic when magnifying): the table's error is not a rounding
    but a systematic deviation of the piecewise-linear interpolant, and h^2 / 8 max|F''| per tap is reached where a tap falls midway
    between two knots near the cubic's peak, whose curvature is the largest.  So the margin asserted here is 2x, not 4x."""
    rng = np.random.default_rng(102)
    img = rng.integers(0, 256, (60, 70, 3)).astype(np.uint8)
    worst = {}
    for ft in (F.F_LINEAR, F.F_TRIANGULAR, F.F_GAUSSIAN, F.F_CUBIC, F.F_LANCZOS3):
        for out_hw in ((23, 31), (97, 130)):
            vals, b = F.resize(img, out_hw, None, (ft, 1, 0.0), (ft, 1, 0.0), exact=True)
            out = oracle.resample(img, out_hw, (ft, 1, 0.0), (ft, 1, 0.0), np.float32)
            worst[ft] = max(worst.get(ft, 0.0), F.check(out, vals, _scaled(b, 0.5), (ft, out_hw)))
    print("resize (continuous filter) worst |err| / bound:", {k: round(v * 0.5, 4) for k, v in worst.items()})


def test_resize3d_oracle_within_bounds(oracle):
    rng = np.random.default_rng(103)
    worst = 0.0
    for shape, out, roi in (((9, 14, 33, 3), (5, 9, 17), None), ((6, 7, 8, 2), (11, 13, 40), None),
                            ((11, 13, 15, 1), (5, 6, 7), ((10.5, 2.0, 1.5), (0.5, 12.0, 14.0))), ((1, 10, 12, 1), (4, 5, 30), None),
                            ((7, 10, 12, 4), (1, 5, 6), None)):
        vol = rng.integers(0, 256, shape).astype(np.uint8)
        for ft in (F.F_NN, F.F_LINEAR, F.F_CUBIC):
            filt = [(ft, 1, 0.0)] * 3
            rois = None if roi is None else [(roi[0][d], roi[1][d]) for d in range(3)]
            vals, b = F.resize(vol, out, rois, filt, filt)
            got = oracle.resample3d(vol, out, filt, filt, np.float32, roi)
            worst = max(worst, F.check(got, vals, _scaled(b, MARGIN), (shape, out, ft, roi)))
            worst = max(worst, F.check_u8(oracle.resample3d(vol, out, filt, filt, np.uint8, roi), vals, _scaled(b, MARGIN), (shape, out, ft, roi)))
    print("resize3d worst |err| / bound:", round(worst * MARGIN, 4))


def test_resize_golden_within_bounds(golden_dir):
    """The committed outputs of the reference's own CPU kernels (tests/golden/resample_ref.npz) meet the bounds."""
    import os
    g = np.load(os.path.join(golden_dir, "resample_ref.npz"))
    n = len([k for k in g.files if k.startswith("in_")])
    worst = 0.0
    for i in range(n):
        oh, ow, tmin, amin, tmag, amag, _ = [int(v) for v in g[f"meta_{i}"]]
        r = g[f"roi_{i}"]
        rois = None if np.isnan(r[0]) else [(float(r[0]), float(r[2])), (float(r[1]), float(r[3]))]
        vals, b = F.resize(g[f"in_{i}"], (oh, ow), rois, (tmin, amin, 0.0), (tmag, amag, 0.0))
        worst = max(worst, F.check(g[f"out_f32_{i}"], vals, _scaled(b, MARGIN), i))
        worst = max(worst, F.check_u8(g[f"out_u8_{i}"], vals, _scaled(b, MARGIN), i))
    print("resize golden worst |err| / bound:", round(worst * MARGIN, 4))


def test_resize_known_answers(oracle):
    rng = np.random.default_rng(104)
    img = rng.integers(0, 256, (37, 53, 3)).astype(np.uint8)
    for ft in (F.F_NN, F.F_LINEAR, F.F_CUBIC):                          # table weights at integer offsets are exactly 0 and 1
        vals, b = F.resize(img, (37, 53), None, (ft, 1, 0.0), (ft, 1, 0.0))
        assert np.array_equal(vals[0], img), ft
        assert np.array_equal(oracle.resample(img, (37, 53), (ft, 1, 0.0), (ft, 1, 0.0), np.uint8), img), ft
    # integer 2x downscale with linear antialias = the [1, 3, 3, 1] / 8 stencil per axis, edge samples clamped
    x = rng.normal(0, 10, (40, 24, 1))
    vals, b = F.resize(x, (20, 12), None, (F.F_LINEAR, 1, 0.0), (F.F_LINEAR, 1, 0.0))

    def stencil(a, axis):
        n = a.shape[axis]
        i = np.arange(n // 2) * 2
        t = lambda k: np.take(a, np.clip(i + k, 0, n - 1), axis=axis)
        return (t(-1) + 3 * t(0) + 3 * t(1) + t(2)) / 8
    want = stencil(stencil(x, 0), 1)
    assert np.abs(vals[0] - want).max() <= 1e-9 * np.abs(x).max()
    assert np.all(np.abs(oracle.resample(x.astype(np.float32), (20, 12), out_dtype=np.float32) - want) <= b[0])


def _warp_cases(rng):
    for it in range(24):
        H, W = [int(v) for v in rng.integers(1, 90, 2)]
        C = (1, 3, 4)[it % 3]
        ang, sc = rng.uniform(-np.pi, np.pi), rng.choice([0.25, 0.7, 1.0, 1.3, 4.0])
        c, s = np.cos(ang) * sc, np.sin(ang) * sc
        M = np.float32([[c, -s, rng.uniform(-20, W + 20)], [s, c, rng.uniform(-20, H + 20)]])
        out = (int(rng.integers(1, 70)), int(rng.integers(1, 600)))
        yield rng.integers(0, 256, (H, W, C)).astype(np.uint8), M, out
    yield np.uint8([[[7, 9, 11]]]), np.float32([[1, 0, 0], [0, 1, 0]]), (3, 4)
    yield np.zeros((5, 5, 3), np.uint8) + 9, np.float32([[1, 0, 500], [0, 1, 500]]), (4, 4)
    y, x = np.meshgrid(np.arange(16.0), np.arange(12000.0), indexing="ij")        # smooth, so the coordinate term stays below a level
    smooth = np.clip(128 + 90 * np.sin(x / 40) * np.cos(y / 30), 0, 255).astype(np.uint8)[..., None].repeat(3, axis=2)
    yield smooth, np.float32([[1.0003, 0.013, 9990.37], [0.0001, 0.97, 0.41]]), (14, 1700)      # coordinates near 10^4, inside the source


def test_warp_oracle_within_bounds(oracle):
    rng = np.random.default_rng(105)
    worst = 0.0
    for img, M, out in _warp_cases(rng):
        for fill in (None, 42.0):
            v, b = F.warp_affine(img, M, out, 1, fill)
            got = oracle.warp_affine(img, M, out, 1, fill, np.float32)
            worst = max(worst, F.check(got, v, MARGIN * b, (img.shape, M.tolist(), out, fill)))
            worst = max(worst, F.check_u8(oracle.warp_affine(img, M, out, 1, fill, np.uint8), v, MARGIN * b, (img.shape, out, fill)))
            F.check_choice(oracle.warp_affine(img, M, out, 0, fill, np.uint8), F.warp_affine(img, M, out, 0, fill), (img.shape, out, fill))
    g = np.load(__import__("os").path.join(__import__("os").path.dirname(__file__), "golden", "warp_color_ref.npz"))
    for fill, name in ((None, "clamp"), (0.0, "fill0")):
        v, b = F.warp_affine(g["in"], g["M"], None, 1, fill)
        worst = max(worst, F.check_u8(g[f"out_1_{name}"], v, MARGIN * b, name))
        F.check_choice(g[f"out_0_{name}"], F.warp_affine(g["in"], g["M"], None, 0, fill), name)
    print("warp worst |err| / bound:", round(worst * MARGIN, 4))


def test_warp_known_answers(oracle):
    rng = np.random.default_rng(106)
    img = rng.integers(0, 256, (30, 40, 3)).astype(np.uint8)
    for interp in (0, 1):
        assert np.array_equal(oracle.warp_affine(img, np.float32([[1, 0, 0], [0, 1, 0]]), None, interp), img)
        shifted = oracle.warp_affine(img, np.float32([[1, 0, 3], [0, 1, -2]]), None, interp)   # src = dst + (3, -2), edges clamped
        want = img[np.clip(np.arange(30) - 2, 0, 29)][:, np.clip(np.arange(40) + 3, 0, 39)]
        assert np.array_equal(shifted, want)
        v = F.warp_affine(img, np.float32([[1, 0, 3], [0, 1, -2]]), None, interp, None)
        assert np.array_equal(v[0] if interp == 1 else v[4], want)


def test_cmn_oracle_within_bounds(oracle):
    rng = np.random.default_rng(107)
    worst = {}
    img = np.stack(np.meshgrid(np.arange(256), np.arange(3), indexing="ij"), -1)[..., 0].astype(np.uint8)
    img = np.repeat(img[:, None, :1], 3, axis=2).reshape(256, 1, 3)      # every byte value in every channel
    cases = [(img, None, None, False, [123.675, 116.28, 103.53], [58.395, 57.12, 57.375], 1.0, 0.0, None, 0.0)]
    for it in range(12):
        H, W = [int(v) for v in rng.integers(1, 60, 2)]
        x = rng.integers(0, 256, (H, W, 3)).astype(np.uint8)
        ch, cw = int(rng.integers(1, H + 4)), int(rng.integers(1, W + 4))
        anchor = (int(rng.integers(-3, H)), int(rng.integers(-3, W)))
        std = rng.uniform(1e-3, 100, 3) if it % 4 else rng.choice([1e-4, 1e4, 3e6], 3)
        cases.append((x, anchor, (ch, cw), bool(it % 2), rng.uniform(0, 255, 3), std, rng.choice([1.0, 64.0]), rng.choice([0.0, 128.0]),
                      4 if it % 3 == 0 else None, 7.5))
    for x, anchor, crop, mirror, mean, std, scale, shift, padc, fill in cases:
        m32, inv32 = oracle.cmn_norm_args(mean, std, scale, shift)
        for layout in ("CHW", "HWC"):
            v, b = F.crop_mirror_normalize(x, anchor or (0, 0), crop, mirror, mean, std, scale, shift, layout, padc, fill)
            got = oracle.cmn(x, anchor, crop, mirror, m32, inv32, np.float32, layout, padc, fill)
            worst["f32"] = max(worst.get("f32", 0.0), F.check(got, v, MARGIN * b, (x.shape, anchor, crop, std)))
            got16 = oracle.cmn(x, anchor, crop, mirror, m32, inv32, np.float16, layout, padc, fill)
            worst["f16"] = max(worst.get("f16", 0.0), F.check_f16(got16, v, MARGIN * b, (x.shape, anchor, crop, std)))
    # mean 0, std 1 returns float(x)
    v, b = F.crop_mirror_normalize(img, layout="HWC")
    assert np.array_equal(v, img.astype(np.float64)) and np.array_equal(oracle.cmn(img, layout="HWC"), img.astype(np.float32))
    print("cmn worst |err| / bound:", {k: round(r * MARGIN, 4) for k, r in worst.items()})


def test_cmn_golden_within_bounds(golden_dir):
    import os
    g = np.load(os.path.join(golden_dir, "cmn_ref.npz"))
    mean, std = [0.485 * 255, 0.456 * 255, 0.406 * 255], [0.229 * 255, 0.224 * 255, 0.225 * 255]
    for i in range(len([k for k in g.files if k.startswith("in_")])):
        ay, ax, ch, cw, mirror, padc = [int(v) for v in g[f"args_{i}"]]
        fill = g[f"fill_{i}"]
        for layout in ("CHW", "HWC"):
            v, b = F.crop_mirror_normalize(g[f"in_{i}"], (ay, ax), (ch, cw), bool(mirror), mean, std, 1.0, 0.0, layout, padc or None,
                                           fill if fill.size else 0.0)
            F.check(g[f"out_f32_{layout}_{i}"], v, MARGIN * b, (i, layout))
            F.check_f16(g[f"out_f16_{layout}_{i}"], v, MARGIN * b, (i, layout))


def _rgb_cube(step=5):
    r = np.arange(0, 256, step)
    return np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 1, 3).astype(np.uint8)


def test_color_twist_oracle_within_bounds(oracle, golden_dir):
    import os
    cube = _rgb_cube(5)
    worst = 0.0
    args = [(0, 1, 1, 1, 1), (180, 1, 1, 1, 1), (-180, 1, 1, 1, 1), (37.5, 0, 1, 1, 1), (-91, 1.7, 0.8, 1, 1), (12, 0.5, 1.3, 1.2, 0.7),
            (0, 1, 1, 0.6, 1.4), (179.9, 2.5, 1.0, 1, 1)]
    for h, s, val, br, co in args:
        v, b = F.twist(cube, h, s, val, br, co)
        Mo, To = oracle.color_twist_matrix(h, s, val, br, co)
        worst = max(worst, F.check(oracle.linear_transform(cube, Mo, To, np.float32), v, MARGIN * b, (h, s, val, br, co)))
        worst = max(worst, F.check_u8(oracle.linear_transform(cube, Mo, To, np.uint8), v, MARGIN * b, (h, s, val, br, co)))
    M, T = F.twist_matrix()
    assert np.abs(M - np.eye(3)).max() < 1e-12 and np.all(T == 0)
    g = np.load(os.path.join(golden_dir, "warp_color_ref.npz"))
    for i, (h, s, val) in enumerate(g["hsv_args"]):
        v, b = F.twist(g["in"], float(h), float(s), float(val))
        worst = max(worst, F.check_u8(g[f"hsv_out_{i}"], v, MARGIN * b, i))
    print("color twist worst |err| / bound:", round(worst * MARGIN, 4))


def test_ycbcr_conversions_within_bounds(oracle, golden_dir):
    import os
    cube = _rgb_cube(3)
    v, b = F.rgb_to_ycbcr(cube)
    F.check_u8(oracle.csc(cube, oracle.IT_RGB, oracle.IT_YCBCR), v, MARGIN * b, "rgb->ycbcr")
    v, b = F.ycbcr_to_rgb(cube)
    F.check_u8(oracle.csc(cube, oracle.IT_YCBCR, oracle.IT_RGB), v, MARGIN * b, "ycbcr->rgb")
    F.check_u8(oracle.csc(cube, oracle.IT_YCBCR, oracle.IT_BGR), v[..., ::-1], MARGIN * b, "ycbcr->bgr")
    v, b = F.ycbcr_to_gray(cube)
    F.check_u8(oracle.csc(cube, oracle.IT_YCBCR, oracle.IT_GRAY), v, MARGIN * b, "ycbcr->gray")
    gray = np.arange(256, dtype=np.uint8).reshape(256, 1, 1)
    v, b = F.gray_to_ycbcr(gray)
    F.check_u8(oracle.csc(gray, oracle.IT_GRAY, oracle.IT_YCBCR), v, MARGIN * b, "gray->ycbcr")
    g = np.load(os.path.join(golden_dir, "warp_color_ref.npz"))
    F.check_u8(g["csc_rgb2ycbcr"], *[MARGIN ** k * a for k, a in enumerate(F.rgb_to_ycbcr(g["csc_in"]))], "golden rgb->ycbcr")
    F.check_u8(g["csc_ycbcr2rgb"], *[MARGIN ** k * a for k, a in enumerate(F.ycbcr_to_rgb(g["csc_in"]))], "golden ycbcr->rgb")
    F.check_u8(g["csc_ycbcr2gray"], *[MARGIN ** k * a for k, a in enumerate(F.ycbcr_to_gray(g["csc_in"]))], "golden ycbcr->gray")


@pytest.mark.parametrize("cfg", [(513, 128, 16000.0, 0.0, 8000.0, False, True), (513, 80, 16000.0, 20.0, 7600.0, True, False),
                                 (1025, 200, 44100.0, 0.0, 0.0, False, True), (257, 13, 22050.0, 100.0, 9000.0, True, True)])
def test_mel_weights_within_bounds(oracle, cfg):
    nbin, nf, sr, fl, fh, htk, norm = cfg
    W, B = F.mel_weights(nbin, nf, sr, fl, fh, htk, norm)
    Wo = oracle.mel_weights(nbin, nf, sr, fl, fh, "htk" if htk else "slaney", norm)
    r = F.check(Wo, W, MARGIN * B, cfg)
    assert (W > 0).sum(axis=1).min() >= 1
    print("mel weights worst |err| / bound:", round(r * MARGIN, 4))


# ------------------------------------------------------------------------------------------------------------------ planted mistakes
def _ratio(wrong, vals, bound):
    """How far a float64 evaluation of a mistaken operation lands outside the statement's bound: max |wrong - value| / bound."""
    vals = vals if isinstance(vals, list) else [vals]
    bound = bound if isinstance(bound, list) else [bound] * len(vals)
    r = np.min([np.abs(np.asarray(wrong, np.float64) - v) / np.maximum(b, 1e-300) for v, b in zip(vals, bound)], axis=0)
    return float(r.max())


def test_planted_mistakes_are_rejected():
    rng = np.random.default_rng(108)
    img = rng.integers(0, 256, (48, 64, 3)).astype(np.uint8)
    lin = (F.F_LINEAR, 1, 0.0)
    res = {}
    vals, b = F.resize(img, (20, 27), None, lin, lin)
    s = (48 / 20, 64 / 27)
    res["pixel centre without 1/2"] = _ratio(F.resize(img, (20, 27), [(-s[0] / 2, 48 - s[0] / 2), (-s[1] / 2, 64 - s[1] / 2)], lin, lin)[0][0], vals, b)
    res["antialias radius not scaled"] = _ratio(F.resize(img, (20, 27), None, (F.F_TRIANGULAR, 1, 1.0), lin)[0][0], vals, b)
    roi = [(2.5, 45.0), (60.25, 3.5)]
    vals_f, b_f = F.resize(img, (20, 27), roi, lin, lin)
    res["flipped x ROI read unflipped"] = _ratio(F.resize(img, (20, 27), [roi[0], (3.5, 60.25)], lin, lin)[0][0], vals_f, b_f)
    nn = (F.F_NN, 0, 0.0)
    vals_n, b_n = F.resize(img, (21, 29), None, nn, nn)
    wrong = F.resize(img, (21, 29), [(0.5, 48.5), (0.5, 64.5)], nn, nn)[0][0]            # floor(c + 1/2) = round(c)
    nn_rejected = int(np.all([np.abs(wrong - v) > b for v, b in zip(vals_n, b_n)], axis=0).sum())     # NN answers are pixels: a count
    cub = (F.F_CUBIC, 0, 0.0)
    vals_c, b_c = F.resize(img, (70, 90), None, cub, cub)
    res["Keys a = -0.75"] = _ratio(F.resize(img, (70, 90), None, cub, cub,
                                            form=lambda t, a: F.keys_cubic(a, -0.75))[0][0], vals_c, b_c)
    lz = (F.F_LANCZOS3, 0, 0.0)
    vals_l, b_l = F.resize(img, (70, 90), None, lz, lz)
    res["Lanczos-2 for Lanczos-3"] = _ratio(F.resize(img, (70, 90), None, lz, lz, form=lambda t, a: F.lanczos(a, 2))[0][0], vals_l, b_l)
    M = np.float32([[0.95, -0.2, 6.0], [0.2, 0.95, -3.0]])
    vw, bw = F.warp_affine(img, M, (40, 60), 1)
    Mw = M.astype(np.float64).copy()
    Mw[:, 2] += 0.5                                                      # corners at floor(p) instead of floor(p - 1/2)
    res["bilinear warp without -1/2"] = _ratio(F.warp_affine(img, Mw, (40, 60), 1)[0], vw, bw)
    cube = _rgb_cube(15)
    vh, bh = F.twist(cube, 25.0, 1.2, 0.9)
    res["hue sign flipped"] = _ratio(F.linear_transform(cube, *F.twist_matrix(-25.0, 1.2, 0.9))[0], vh, bh)
    res["YIQ^-1 taken as the transpose"] = _ratio(F.linear_transform(cube, *F.twist_matrix(25.0, 1.2, 0.9, inverse=np.transpose))[0], vh, bh)
    std = [58.395, 57.12, 57.375]
    vc, bc = F.crop_mirror_normalize(img, mean=[123.675, 116.28, 103.53], std=std)
    res["CMN with std for 1/std"] = _ratio(F.crop_mirror_normalize(img, mean=[123.675, 116.28, 103.53], std=1 / np.asarray(std))[0], vc, bc)
    print("planted mistakes, |error| / bound:", {k: f"{v:.3g}" for k, v in res.items()})
    print(f"planted mistake NN round instead of floor: {nn_rejected} of {wrong.size} outputs match no accepted pixel (a count, not a ratio)")
    assert nn_rejected > wrong.size // 4, nn_rejected
    for k, v in res.items():
        assert v > 100, (k, v)
