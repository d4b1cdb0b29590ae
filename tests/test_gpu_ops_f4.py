"""-m gpu parity tests of the remaining per-pixel / geometry operators (SURVEY 8f rank 4) through the public API:
brightness_contrast, color_twist, flip, crop, slice, rotate, resize_crop_mirror -- each against the reference's own CPU code
(oracle/_ref) or, for pure index arithmetic, numpy.  Bit-exact.  brightness_contrast is always compared with the float32 restatement
of tests/pointwise_ref.py as well.  Where oracle/_ref is absent, color_twist, the rotate warp and resize_crop_mirror are compared with
the oracle's restatements instead (pinned to the reference by tests/golden/*_ref.npz), and the rotate canvas / matrix come from the
library's own host code (pinned to the reference by tests/test_host_cpu.py where _ref exists)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import pointwise_ref as pr  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


def _run(batch, images, build, extra_sources=(), layout="HWC"):
    from dali_b200 import fn, pipeline_def

    @pipeline_def(batch_size=batch, num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: images, device="gpu", layout=layout)
        extras = [fn.external_source(source=(lambda v: (lambda i: v))(v)) for v in extra_sources]
        return build(fn, x, *extras)
    p = pipe()
    p.build()
    return [o.as_cpu() for o in p.run()]


REF = po.have_ref()
_warp = po.ref_warp_affine if REF else po.warp_affine
_resample = po.ref_resample if REF else po.resample


def _rotate_params(angle_deg, in_h, in_w, keep_size=False):
    if REF:
        return po.ref_rotate_params(angle_deg, in_h, in_w, keep_size=keep_size)
    import ctypes as C
    from dali_b200 import backend
    hw, M = (C.c_int * 2)(), np.empty(6, np.float32)
    assert backend.lib().dalihTestRotateParams(C.c_float(angle_deg), in_h, in_w, int(keep_size), None, hw, M.ctypes.data_as(C.c_void_p)) == 0
    return (hw[0], hw[1]), M.reshape(2, 3)


def _imgs(seed=0):
    rng = np.random.default_rng(seed)
    return [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((97, 131), (64, 64), (120, 75), (33, 250))]


def test_brightness_contrast_and_color_twist():
    from dali_b200 import types
    imgs = _imgs(1)
    n = len(imgs)
    br = [np.array(v, np.float32) for v in (1.3, 0.7, 1.0, 2.1)]
    co = [np.array(v, np.float32) for v in (0.8, 1.5, 1.0, 0.3)]
    a, b, c, d = _run(n, imgs, lambda fn, x, brs, cos: (
        fn.brightness_contrast(x, brightness=brs, contrast=cos, brightness_shift=0.1),
        fn.brightness_contrast(x, brightness=1.2, contrast=0.9, contrast_center=100.0, dtype=types.FLOAT),
        fn.color_twist(x, hue=25.0, saturation=1.4, contrast=cos, brightness=brs),
        fn.color_twist(x, hue=-70.0, saturation=0.5, dtype=types.FLOAT)), extra_sources=(br, co))
    for i, im in enumerate(imgs):
        assert np.array_equal(a[i], pr.brightness_contrast(im, float(br[i]), 0.1, float(co[i]))), i
        want = pr.brightness_contrast(im, 1.2, 0.0, 0.9, 100.0, out_float=True)
        assert b[i].dtype == np.float32 and np.array_equal(b[i].view(np.uint32), want.view(np.uint32)), i
        if REF:
            assert np.array_equal(a[i], po.ref_brightness_contrast(im, float(br[i]), 0.1, float(co[i]))), i
            want = po.ref_brightness_contrast(im, 1.2, 0.0, 0.9, 100.0, out_float=True)
            assert np.array_equal(b[i].view(np.uint32), want.view(np.uint32)), i
        M, T = po.color_twist_matrix(25.0, 1.4, 1.0, float(br[i]), float(co[i]), use_ref=REF)
        assert np.array_equal(c[i], po.linear_transform(im, M, T, np.uint8, use_ref=REF)), i
        M, T = po.color_twist_matrix(-70.0, 0.5, use_ref=REF)
        assert np.array_equal(d[i].view(np.uint32), po.linear_transform(im, M, T, np.float32, use_ref=REF).view(np.uint32)), i


def test_flip_crop_slice_are_index_exact():
    imgs = _imgs(2)
    n = len(imgs)
    hz = [np.array(v, np.int32) for v in (1, 0, 1, 0)]
    vt = [np.array(v, np.int32) for v in (0, 1, 1, 0)]
    anchors = [np.array([0.25, 0.1], np.float32)] * n                      # (x, y) normalised
    shapes = [np.array([0.5, 0.7], np.float32)] * n
    a, b, c, d, e = _run(n, imgs, lambda fn, x, h, v, an, sh: (
        fn.flip(x, horizontal=h, vertical=v),
        fn.crop(x, crop=(30, 40), crop_pos_x=0.2, crop_pos_y=0.9),
        fn.crop(x, crop=(140, 300), out_of_bounds_policy="pad", fill_values=[7, 8, 9]),
        fn.slice(x, an, sh),
        fn.slice(x, start=[5, 3], end=[30, 60], axes=[0, 1])), extra_sources=(hz, vt, anchors, shapes))
    for i, im in enumerate(imgs):
        H, W = im.shape[:2]
        want = im[::-1] if vt[i] else im
        want = want[:, ::-1] if hz[i] else want
        assert np.array_equal(a[i], want), i
        y0, x0 = po.crop_anchor(0.9, H, 30), po.crop_anchor(0.2, W, 40)
        assert np.array_equal(b[i], im[y0:y0 + 30, x0:x0 + 40]), i
        y0, x0 = po.crop_anchor(0.5, H, 140), po.crop_anchor(0.5, W, 300)
        want = np.empty((140, 300, 3), np.uint8); want[...] = [7, 8, 9]
        ys, xs = max(0, -y0), max(0, -x0)
        want[ys:ys + H, xs:xs + W] = im
        assert np.array_equal(c[i], want), i
        rnd = lambda v: int(np.floor(v + 0.5))                       # std::llround: half away from zero (slice_attr.h:176-177)
        bx, ex = rnd(np.float32(0.25) * W), rnd((np.float64(np.float32(0.25)) + np.float64(np.float32(0.5))) * W)
        by, ey = rnd(np.float64(np.float32(0.1)) * H), rnd((np.float64(np.float32(0.1)) + np.float64(np.float32(0.7))) * H)
        assert np.array_equal(d[i], im[by:ey, bx:ex]), i
        assert np.array_equal(e[i], im[5:30, 3:60]), i


def test_rotate_and_resize_crop_mirror():
    from dali_b200 import types
    imgs = _imgs(3)
    n = len(imgs)
    angles = [np.array(v, np.float32) for v in (30.0, -45.0, 90.0, 200.0)]
    mir = [np.array(v, np.int32) for v in (1, 0, 3, 2)]
    a, b, c, d = _run(n, imgs, lambda fn, x, ang, m: (
        fn.rotate(x, angle=ang, fill_value=0),
        fn.rotate(x, angle=ang, keep_size=True, interp_type=types.INTERP_NN),
        fn.resize_crop_mirror(x, resize_shorter=50, crop=(40, 44), crop_pos_x=0.3, mirror=m),
        fn.resize_crop_mirror(x, size=[60, 80], crop=(60, 80))), extra_sources=(angles, mir))
    for i, im in enumerate(imgs):
        H, W = im.shape[:2]
        (oh, ow), M = _rotate_params(float(angles[i]), H, W)
        assert a[i].shape[:2] == (oh, ow)
        assert np.array_equal(a[i], _warp(im, M, (oh, ow), 1, 0.0)), i
        (oh, ow), M = _rotate_params(float(angles[i]), H, W, keep_size=True)
        assert np.array_equal(b[i], _warp(im, M, (oh, ow), 0, None)), i
        # resize_shorter=50 -> not_smaller mode; crop on the resized shape; ROI back-projected (resize_crop_mirror.cc:84-108)
        scale = 50.0 / min(H, W)
        rh, rw = max(1, int(np.round(np.float32(H * scale)))), max(1, int(np.round(np.float32(W * scale))))
        y0, x0 = po.crop_anchor(0.5, rh, 40), po.crop_anchor(0.3, rw, 44)
        # subpixel_scale (default): the resize ROI is first adjusted for the rounded size (resize_attr_base.h:97-113) ...
        rlo, rhi = [0.0, 0.0], [float(H), float(W)]
        for dd, (real, frac) in enumerate(((rh, H * scale), (rw, W * scale))):
            if real != np.float32(frac):
                adj = real / float(np.float32(abs(np.float32(frac))))
                cc = 0.5 * rlo[dd] + 0.5 * rhi[dd]
                rlo[dd], rhi[dd] = float(np.float32(cc + (rlo[dd] - cc) * adj)), float(np.float32(cc + (rhi[dd] - cc) * adj))
        # ... then the crop window is projected back through it in double precision
        ry, rx = (rhi[0] - rlo[0]) / rh, (rhi[1] - rlo[1]) / rw
        lo = [np.float32(y0 * ry + rlo[0]), np.float32(x0 * rx + rlo[1])]
        hi = [np.float32((y0 + 40) * ry + rlo[0]), np.float32((x0 + 44) * rx + rlo[1])]
        m = int(mir[i])
        if m & 2:
            lo[0], hi[0] = hi[0], lo[0]
        if m & 1:
            lo[1], hi[1] = hi[1], lo[1]
        want = _resample(im, (40, 44), roi=((float(lo[0]), float(lo[1])), (float(hi[0]), float(hi[1]))))
        assert np.array_equal(c[i], want), i
        assert np.array_equal(d[i], _resample(im, (60, 80))), i
