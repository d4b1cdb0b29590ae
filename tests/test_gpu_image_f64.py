"""-m gpu: resize, warp_affine, crop_mirror_normalize and the colour operators on the GPU against the float64 statements of
tests/image_f64.py, at the edges of every kernel path, and bit for bit against the float32 restatement (oracle/imgproc_oracle.c): the
restatement can only be changed together with the kernels, so both comparisons hold together.  Where a launch reports which kernel ran
(dalib200ResamplePlanGetPath / GetOrder, dalib200WarpPlanGetPath), each path is asserted to have run."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
from oracle import pyoracle as po  # noqa: E402
import image_f64 as F  # noqa: E402


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


WORST = {}


def _note(op, r):
    WORST[op] = max(WORST.get(op, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("largest |GPU - float64| / bound per op:", {k: round(v, 4) for k, v in sorted(WORST.items())})


# ------------------------------------------------------------------------------------------------------------------------ resize
def _resample_dev(din, shapes, out_hws, filt, out_dtype, rois=None):
    """dalib200Resample* on device tensors given as they are (views at any byte offset): (outputs, paths, orders)."""
    import torch
    import gpu_helpers as g
    n = len(din)
    samples = (capi.ResampleSample * n)()
    for i in range(n):
        g.fill_resample_sample(samples[i], shapes[i], out_hws[i], filt, filt, rois[i] if rois else None)
    in_dt = capi.UINT8 if din[0].dtype == torch.uint8 else capi.FLOAT
    out_dt = capi.UINT8 if np.dtype(out_dtype) == np.uint8 else capi.FLOAT
    plan = capi.Plan("Resample", n)
    capi.check(capi.lib().dalib200ResamplePlanSetup(plan.handle, n, samples, in_dt, out_dt))
    outs = [torch.empty((hw[0], hw[1], s[2]), dtype=torch.uint8 if out_dt == capi.UINT8 else torch.float32, device="cuda")
            for hw, s in zip(out_hws, shapes)]
    capi.check(capi.lib().dalib200ResampleLaunch(plan.handle, capi.ptr_array(din), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    paths = [capi.lib().dalib200ResamplePlanGetPath(plan.handle, i) for i in range(n)]
    orders = [capi.lib().dalib200ResamplePlanGetOrder(plan.handle, i) for i in range(n)]
    return [o.cpu().numpy() for o in outs], paths, orders


def _oracle_roi(roi):
    return None if roi is None else ((roi[0][0], roi[1][0]), (roi[0][1], roi[1][1]))


def _check_resize(got, img, out_hw, filt, out_dtype, roi, what):
    vals, b = F.resize(img, out_hw, roi, filt, filt)
    want = po.resample(img, out_hw, filt, filt, out_dtype, _oracle_roi(roi))
    assert np.array_equal(bits(got), bits(want)), ("bit-exact", what)
    if np.dtype(out_dtype) == np.uint8:
        _note("resize u8", F.check_u8(got, vals, b, what))
    else:
        _note(f"resize f32 filter {filt[0]}", F.check(got, vals, b, what))


def _smooth(rng, shape):
    """A u8 image whose values change by at most ~2 levels per pixel, so that the warp bound's coordinate term (the float walk's
    position error times the local sample range) stays well below one level even for coordinates near 10^4."""
    H, W, Cn = shape
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    out = np.empty(shape)
    for c in range(Cn):
        p = rng.uniform(0, 6, 3)
        out[..., c] = 128 + 70 * np.sin(2 * np.pi * x / 260 + p[0]) * np.cos(2 * np.pi * y / 230 + p[1]) + 25 * np.sin(2 * np.pi * (x - y) / 170 + p[2])
    return np.clip(np.round(out), 0, 255).astype(np.uint8)


def _img(rng, shape, dt):
    if dt == np.uint8:
        return rng.integers(0, 256, shape).astype(np.uint8)
    return (rng.normal(0, 1, shape) * rng.choice([1.0, 300.0, 1e5], shape)).astype(np.float32)


def test_resize_paths_orders_and_taps():
    """Tile kernel and streaming kernel in both processing orders; more than 64 vertical taps (1080 -> 8 rows with antialias: 272) and more
    than 64 horizontal taps; 1 -> 4096, 4096 -> 1 and extent-1 axes; magnifications (the row walk with up to 4 slots) and minifications
    whose source rows do not fit the walk."""
    import gpu_helpers as g
    rng = np.random.default_rng(201)
    lin = (F.F_LINEAR, 1, 0.0)
    cases = [((1080, 1920, 3), (224, 224)), ((480, 640, 3), (224, 224)), ((1080, 64, 1), (8, 64)), ((16, 2000, 1), (16, 10)),
             ((1, 3, 1), (4096, 5)), ((4096, 4, 1), (1, 4)), ((7, 1, 3), (9, 1)), ((64, 64, 3), (256, 256)), ((60, 80, 4), (240, 96)),
             ((300, 32, 3), (75, 32)), ((720, 1280, 3), (720, 640)), ((128, 128, 16), (50, 70))]
    seen_paths, seen_orders = set(), set()
    for shape, out_hw in cases:
        for out_dt in (np.uint8, np.float32):
            img = _img(rng, shape, np.uint8)
            got, paths = g.resample([img], [out_hw], lin, lin, out_dt, want_path=True)
            _, orders = g.resample([img], [out_hw], lin, lin, out_dt, want_order=True)
            seen_paths.add(paths[0]); seen_orders.add((orders[0], paths[0]))
            _check_resize(got[0], img, out_hw, lin, out_dt, None, (shape, out_hw, np.dtype(out_dt).name))
    assert {0, 1} <= seen_paths, seen_paths
    assert {(0, 0), (1, 0), (1, 1)} <= seen_orders, seen_orders


def test_resize_filters_channels_types_rois():
    """All six filters as min and mag filter, channels 1, 2, 3, 4, 5, 8, 16, u8 -> u8, u8 -> f32 and f32 -> f32 (negative and large values),
    fractional ROIs flipped on x, on y and on both, partly outside the image, narrower than one pixel."""
    import gpu_helpers as g
    rng = np.random.default_rng(202)
    rois = [None, [(2.5, 40.25), (3.75, 51.5)], [(2.0, 40.0), (60.5, 1.25)], [(44.0, 0.5), (3.0, 50.0)], [(45.5, -3.0), (70.0, -5.5)],
            [(10.3, 10.6), (20.1, 20.4)], [(-6.0, 30.0), (12.0, 12.0 + 1e-3)]]
    for ft in range(6):
        for aa in (0, 1):
            filt = (ft, aa, 0.0)
            for k, roi in enumerate(rois):
                Cn = (1, 2, 3, 4, 5, 8, 16)[(ft + k) % 7]
                for in_dt, out_dt in ((np.uint8, np.uint8), (np.uint8, np.float32), (np.float32, np.float32)):
                    img = _img(rng, (48, 57, Cn), in_dt)
                    out_hw = [(19, 23), (101, 140), (48, 13)][(k + aa) % 3]
                    (got,) = g.resample([img], [out_hw], filt, filt, out_dt, rois=[_oracle_roi(roi)] if roi else None)
                    _check_resize(got, img, out_hw, filt, out_dt, roi, (ft, aa, roi, Cn, np.dtype(in_dt).name, np.dtype(out_dt).name))


def test_resize_unaligned_slices():
    """Inputs that are slices of one allocation at byte offsets 1..15 and rows whose width is not a multiple of 16 bytes: the word loads
    (aligned4) and the streaming kernel are off, the tile kernel's byte path runs."""
    import torch
    rng = np.random.default_rng(203)
    lin = (F.F_LINEAR, 1, 0.0)
    for Cn, (H, W), out_hw in ((3, (97, 131), (40, 50)), (1, (200, 301), (224, 224)), (4, (61, 77), (130, 33))):
        imgs = [_img(rng, (H, W, Cn), np.uint8) for _ in range(15)]
        size = H * W * Cn
        whole = torch.zeros(16 * (size + 16) + 16, dtype=torch.uint8, device="cuda")
        din = []
        for k, im in enumerate(imgs):
            off = k * (size + 16) + 1 + k
            whole[off:off + size] = torch.from_numpy(im.reshape(-1)).cuda()
            din.append(whole[off:off + size].view(H, W, Cn))
        got, paths, _ = _resample_dev(din, [im.shape for im in imgs], [out_hw] * 15, lin, np.uint8)
        assert paths == [0] * 15, paths
        for im, o in zip(imgs, got):
            _check_resize(o, im, out_hw, lin, np.uint8, None, (im.shape, out_hw))


def test_resize_extreme_ratios_and_refusals():
    """20 000 -> 1 crosses the rescale of a support above 8192 taps; a table of 2^26 words or more and a footprint that does not fit the
    on-chip tile are refused at set-up (errors, not outputs)."""
    import gpu_helpers as g
    rng = np.random.default_rng(204)
    tri = (F.F_TRIANGULAR, 1, 0.0)
    img = _img(rng, (20000, 3, 1), np.uint8)
    for out_dt in (np.uint8, np.float32):
        (got,) = g.resample([img], [(1, 3)], tri, tri, out_dt)
        _check_resize(got, img, (1, 3), tri, out_dt, None, ("20000 -> 1", np.dtype(out_dt).name))

    def setup(shape, out_hw):
        s = (capi.ResampleSample * 1)()
        g.fill_resample_sample(s[0], shape, out_hw, tri, tri, None)
        plan = capi.Plan("Resample", 1)
        capi.check(capi.lib().dalib200ResamplePlanSetup(plan.handle, 1, s, capi.UINT8, capi.UINT8))
    with pytest.raises(capi.DaliB200Error, match="256 MB"):
        setup((1, 4096 * 8192, 1), (1, 8192))
    with pytest.raises(capi.DaliB200Error, match="does not fit the on-chip tile"):
        setup((9000, 9000, 16), (1, 1))


def test_resize3d_f64():
    """Volumetric: the same statement on DHWC shapes, including a flipped z ROI and z extent 1."""
    import gpu_helpers as g
    rng = np.random.default_rng(205)
    for shape, out, roi in (((9, 14, 33, 3), (5, 9, 17), None), ((1, 10, 12, 1), (4, 5, 30), None), ((6, 7, 8, 2), (1, 13, 40), None),
                            ((11, 13, 15, 1), (5, 6, 7), ((10.5, 2.0, 1.5), (0.5, 12.0, 14.0)))):
        vol = _img(rng, shape, np.uint8)
        for ft in (F.F_NN, F.F_LINEAR, F.F_CUBIC, F.F_LANCZOS3):
            filt = [(ft, 1, 0.0)] * 3
            rois3 = None if roi is None else [(roi[0][d], roi[1][d]) for d in range(3)]
            vals, b = F.resize(vol, out, rois3, filt, filt)
            for out_dt in (np.uint8, np.float32):
                (got,) = g.resample3d([vol], [out], filt, filt, out_dt, rois=[roi] if roi else None)
                assert np.array_equal(bits(got), bits(po.resample3d(vol, out, filt, filt, out_dt, roi))), (shape, out, ft, roi)
                if out_dt == np.uint8:
                    F.check_u8(got, vals, b, (shape, out, ft, roi))
                else:
                    _note("resize3d f32", F.check(got, vals, b, (shape, out, ft, roi)))


# ------------------------------------------------------------------------------------------------------------------------ warp
def _rot(deg, sc, H, W, oh, ow, t=(0.0, 0.0)):
    M = F.rotation_matrix(deg, (H, W), (oh, ow))
    M[:, :2] *= sc
    M[:, 2] += t
    return M.astype(np.float32)


def _check_warp(got, img, M, out_hw, interp, fill, out_dt, what):
    want = po.warp_affine(img, M, out_hw, interp, fill, out_dt)
    assert np.array_equal(bits(got), bits(want)), ("bit-exact", what)
    if interp == 0:
        F.check_choice(got, F.warp_affine(img, M, out_hw, 0, fill), what)
        return
    v, b = F.warp_affine(img, M, out_hw, 1, fill)
    if np.dtype(out_dt) == np.uint8:
        _note("warp u8", F.check_u8(got, v, b, what))
    else:
        _note("warp f32", F.check(got, v, b, what))


def test_warp_generic_kernel_edges():
    """Outputs wider than 256 and 4096 px (re-anchoring and drift), coordinates near 10^4, angles near 90 and 180 degrees, scales 0.25
    and 4, maps entirely outside the source under fill and clamp, 1 x 1 inputs, C = 1, 3, 4, u8 and f32 outputs."""
    import gpu_helpers as g
    rng = np.random.default_rng(206)
    cases = []
    for Cn in (1, 3, 4):
        H, W = 50, 70
        cases += [((H, W, Cn), _rot(89.9, 1.0, H, W, 3, 5000), (3, 5000)), ((H, W, Cn), _rot(180.05, 0.25, H, W, 40, 300), (40, 300)),
                  ((H, W, Cn), _rot(-90.02, 4.0, H, W, 30, 700), (30, 700)), ((H, W, Cn), np.float32([[1, 0.01, 500], [0, 1, -400]]), (9, 9)),
                  ((1, 1, Cn), _rot(33, 1.0, 1, 1, 5, 6), (5, 6)),
                  ((16, 12000, Cn), np.float32([[1.0003, 0.013, 9990.37], [0.0001, 0.97, 0.41]]), (14, 1700))]   # inside, near 10^4
    for shape, M, out_hw in cases:
        img = _smooth(rng, shape) if shape[0] > 1 else _img(rng, shape, np.uint8)
        for interp in (0, 1):
            for fill in (None, 77.0):
                for out_dt in (np.uint8, np.float32):
                    (got,) = g.warp_affine([img], [M], [out_hw], interp, fill, out_dt)
                    _check_warp(got, img, M, out_hw, interp, fill, out_dt, (shape, M.tolist(), out_hw, interp, fill))


def test_warp_band_kernel_paths(monkeypatch):
    """Path 1: bilinear u8 3-channel frames of one allocation at a 16-byte stride (tensor-map TMA boxes).  Path 2: the band kernel without
    the boxes (rows that are not a multiple of 16 bytes), which the library takes when asked for it.  Path 0: NN or f32 outputs."""
    import gpu_helpers as g
    rng = np.random.default_rng(207)
    seen = set()
    for (H, W), asked in (((200, 448), False), ((120, 301), True)):
        imgs = [_smooth(rng, (H, W, 3)) for _ in range(4)]
        mats = [_rot(d, s, H, W, H, W + 300, t) for d, s, t in ((2.0, 1.0, (0.3, -0.2)), (-12.0, 1.1, (0, 0)), (90.1, 1.0, (1, 2)),
                                                                  (179.0, 0.7, (0, 0)))]
        if asked:
            monkeypatch.setenv("DALIB200_WARP_BAND", "1")
        for fill in (None, 5.0):
            got, path = g.warp_affine(imgs, mats, [(H, W + 300)] * 4, 1, fill, np.uint8, contiguous=True, want_path=True)
            seen.add(path)
            for im, M, o in zip(imgs, mats, got):
                _check_warp(o, im, M, (H, W + 300), 1, fill, np.uint8, ((H, W), M.tolist(), fill, path))
        monkeypatch.delenv("DALIB200_WARP_BAND", raising=False)
        got, path = g.warp_affine(imgs, mats, [(H, W + 300)] * 4, 0, None, np.uint8, contiguous=True, want_path=True)
        seen.add(path)
        for im, M, o in zip(imgs, mats, got):
            _check_warp(o, im, M, (H, W + 300), 0, None, np.uint8, ((H, W), "nn"))
    assert seen == {0, 1, 2}, seen


def test_rotate_matrix_and_warp():
    """fn.rotate: the canvas size and the float32 matrix from the library's host code; that matrix against the float64 rotation about the
    two centres (entries within a few u of their terms), and the operator's output against the warp statement with that matrix."""
    import ctypes as C
    from dali_b200 import backend, fn, pipeline_def
    rng = np.random.default_rng(208)
    imgs = [_img(rng, (37, 61, 3), np.uint8) for _ in range(2)]
    for angle in (0.0, 90.0, 180.0, 270.0, 17.5, -133.0):
        for keep in (False, True):
            @pipeline_def(batch_size=2, num_threads=1, device_id=0)
            def pipe():
                x = fn.external_source(source=lambda i: imgs, device="gpu", layout="HWC")
                return fn.rotate(x, angle=angle, keep_size=keep, fill_value=0.0)
            p = pipe()
            p.build()
            (out,) = p.run()
            out = out.as_cpu()
            for i, im in enumerate(imgs):
                o = np.asarray(out[i])
                hw, Ml = (C.c_int * 2)(), np.empty(6, np.float32)
                assert backend.lib().dalihTestRotateParams(C.c_float(angle), im.shape[0], im.shape[1], int(keep), None, hw,
                                                           Ml.ctypes.data_as(C.c_void_p)) == 0
                assert o.shape[:2] == tuple(hw), (angle, keep, o.shape, tuple(hw))
                M = F.rotation_matrix(angle, im.shape[:2], o.shape[:2])
                # float32 angle, cosf / sinf and two 3 x 3 products: the rotation entries within 8u, the offsets within 8u of their terms
                tol = 8 * F.U * np.array([[1, 1, 1 + abs(M[0, 2]) + o.shape[1] + o.shape[0] + im.shape[1]],
                                          [1, 1, 1 + abs(M[1, 2]) + o.shape[1] + o.shape[0] + im.shape[0]]])
                assert np.all(np.abs(Ml.reshape(2, 3) - M) <= tol), (angle, keep, Ml, M)
                v, b = F.warp_affine(im, Ml, o.shape[:2], 1, 0.0)
                _note("rotate u8", F.check_u8(o, v, b, (angle, keep, i)))
                assert np.array_equal(o, po.warp_affine(im, Ml, o.shape[:2], 1, 0.0)), (angle, keep, i)


# ------------------------------------------------------------------------------------------------------------------------ CMN
def test_cmn_f64():
    """Every byte value in every channel at the C2 shape (224 x 224, mean / std of ImageNet), fp16 and fp32, CHW and HWC, pad and mirror,
    std small enough to clamp at +-65504 and large enough for fp16 subnormals."""
    import gpu_helpers as g
    rng = np.random.default_rng(209)
    byte = np.arange(224 * 224 * 3) % 256
    c2 = np.stack([np.roll(byte, 77 * c)[: 224 * 224] for c in range(3)], -1).reshape(224, 224, 3).astype(np.uint8)
    cases = [(c2, (0, 0), (224, 224), False, [123.675, 116.28, 103.53], [58.395, 57.12, 57.375], None),
             (c2, (-3, 5), (224, 224), True, [123.675, 116.28, 103.53], [58.395, 57.12, 57.375], 4),
             (c2, (0, 0), (224, 224), False, [128.0, 0.0, 255.0], [1e-3, 2e-3, 1e-3], None),
             (c2, (10, 10), (50, 60), True, [0.0, 10.0, 250.0], [3e6, 1e7, 2e8], None)]
    for im in [_img(rng, (17, 23, 3), np.uint8), _img(rng, (1, 1, 3), np.uint8)]:
        cases.append((im, (-2, 3), (21, 19), True, rng.uniform(0, 255, 3), rng.uniform(0.5, 80, 3), 4))
    for img, anchor, crop, mirror, mean, std, padc in cases:
        m32, inv32 = po.cmn_norm_args(mean, std)
        for layout in ("CHW", "HWC"):
            v, b = F.crop_mirror_normalize(img, anchor, crop, mirror, mean, std, 1.0, 0.0, layout, padc, 0.0)
            for dt in (np.float32, np.float16):
                (got,) = g.cmn([img], [anchor], [crop], [mirror], m32, inv32, dt, layout, padc, [0.0] * 4)
                want = po.cmn(img, anchor, crop, mirror, m32, inv32, dt, layout, padc, 0.0)
                assert np.array_equal(bits(got), bits(want)), (img.shape, anchor, crop, std, layout, np.dtype(dt).name)
                if dt == np.float32:
                    _note("cmn f32", F.check(got, v, b, (img.shape, std, layout)))
                else:
                    _note("cmn f16", F.check_f16(got, v, b, (img.shape, std, layout)))


# ------------------------------------------------------------------------------------------------------------------------ colour
def test_color_twist_and_ycbcr_f64():
    """The RGB cube at a stride of 5, hue across +-180 degrees, saturation 0 and above 1, brightness and contrast, with the matrix from the
    library's host code; RGB <-> YCbCr and YCbCr -> GRAY."""
    import gpu_helpers as g
    r = np.arange(0, 256, 5)
    cube = np.stack(np.meshgrid(r, r, r, indexing="ij"), -1).reshape(-1, 1, 3).astype(np.uint8)
    for args in ((0, 1, 1, 1, 1), (-180, 1, 1, 1, 1), (180, 1.3, 1, 1, 1), (91, 0, 1, 1, 1), (-45, 2.2, 0.9, 1, 1), (10, 1, 1, 1.3, 0.6),
                 (0, 1, 1, 0.5, 1.8)):
        M, T = g.color_twist_matrix(*args)
        v, b = F.twist(cube, *args)
        for out_dt in (np.uint8, np.float32):
            (got,) = g.linear_transform([cube], [M], [T], out_dt)
            assert np.array_equal(bits(got), bits(po.linear_transform(cube, M, T, out_dt))), args
            if out_dt == np.uint8:
                _note("color twist u8", F.check_u8(got, v, b, args))
            else:
                _note("color twist f32", F.check(got, v, b, args))
    gray = np.arange(256, dtype=np.uint8).reshape(256, 1, 1)
    for src, a, bt, stmt in ((cube, capi.RGB, capi.YCbCr, F.rgb_to_ycbcr), (cube, capi.YCbCr, capi.RGB, F.ycbcr_to_rgb),
                             (cube, capi.YCbCr, capi.GRAY, F.ycbcr_to_gray), (gray, capi.GRAY, capi.YCbCr, F.gray_to_ycbcr)):
        (got,) = g.csc([src], a, bt)
        _note("ycbcr u8", F.check_u8(got, *stmt(src), (a, bt)))


def test_fn_color_ops_f64():
    """fn.hsv, fn.color_twist and fn.color_space_conversion through the pipeline."""
    from dali_b200 import fn, pipeline_def, types
    rng = np.random.default_rng(210)
    imgs = [_img(rng, (33, 45, 3), np.uint8), _img(rng, (8, 300, 3), np.uint8)]

    @pipeline_def(batch_size=2, num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: imgs, device="gpu", layout="HWC")
        return (fn.hsv(x, hue=-150.0, saturation=1.4, value=0.8), fn.color_twist(x, hue=35.0, saturation=0.0, brightness=1.2, contrast=0.7),
                fn.color_space_conversion(x, image_type=types.RGB, output_type=types.YCbCr))
    p = pipe()
    p.build()
    a, bb, c = [o.as_cpu() for o in p.run()]
    for i, im in enumerate(imgs):
        _note("fn.hsv u8", F.check_u8(np.asarray(a[i]), *F.twist(im, -150.0, 1.4, 0.8), ("hsv", i)))
        _note("fn.color_twist u8", F.check_u8(np.asarray(bb[i]), *F.twist(im, 35.0, 0.0, 1.0, 1.2, 0.7), ("color_twist", i)))
        _note("fn.color_space_conversion u8", F.check_u8(np.asarray(c[i]), *F.rgb_to_ycbcr(im), ("csc", i)))


# ------------------------------------------------------------------------------------------------------------------------ through fn.*
def _pipe(images, build):
    from dali_b200 import fn, pipeline_def

    @pipeline_def(batch_size=len(images), num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: images, device="gpu", layout="HWC")
        return build(fn, x)
    p = pipe()
    p.build()
    return [o.as_cpu() for o in p.run()]


LIN_MIN, LIN_MAG = (F.F_LINEAR, 1, 0.0), (F.F_LINEAR, 0, 0.0)           # fn.resize defaults: antialiased linear shrinking, linear growing


def test_fn_resize_rois():
    """fn.resize with absolute and relative roi_start / roi_end, flipped on x, on y and on both (the host code swaps a flipped ROI, negates
    the requested size and swaps it back): the output is the resize of [r0, r1) on each axis, r1 < r0 flipping it."""
    rng = np.random.default_rng(211)
    imgs = [_img(rng, (61, 83, 3), np.uint8), _img(rng, (40, 100, 3), np.uint8)]
    cases = [([3.5, 10.25], [55.0, 70.5], False), ([55.0, 10.25], [3.5, 70.5], False), ([3.5, 70.5], [55.0, 10.25], False),
             ([0.9, 0.8], [0.1, 0.05], True), ([0.25, 0.0], [0.75, 1.0], True)]
    for rs, re, rel in cases:
        outs = _pipe(imgs, lambda fn, x: (fn.resize(x, resize_x=37, resize_y=29, roi_start=rs, roi_end=re, roi_relative=rel),
                                          fn.resize(x, resize_x=150, resize_y=90, roi_start=rs, roi_end=re, roi_relative=rel)))
        for o, out_hw in zip(outs, ((29, 37), (90, 150))):
            for i, im in enumerate(imgs):
                got = np.asarray(o[i])
                k = [im.shape[0], im.shape[1]] if rel else [1, 1]
                f32 = lambda v: float(np.float32(v))                    # float argument, scaled in double, stored as float
                roi = [(f32(f32(rs[d]) * k[d]), f32(f32(re[d]) * k[d])) for d in range(2)]
                vals, b = F.resize(im, out_hw, roi, [LIN_MIN] * 2, [LIN_MAG] * 2)
                _note("fn.resize u8", F.check_u8(got, vals, b, (rs, re, rel, out_hw, i)))
                want = po.resample(im, out_hw, LIN_MIN, LIN_MAG, np.uint8, ((roi[0][0], roi[1][0]), (roi[0][1], roi[1][1])))
                assert np.array_equal(got, want), (rs, re, rel, out_hw, i)


def test_fn_resize_crop_mirror():
    """fn.resize_crop_mirror with each mirror flag (1 = horizontal, 2 = vertical): the statement resizes the whole image, crops the window
    at round(pos (size - crop)) of the resized image and flips it -- the operator instead resamples the crop window projected back into
    the input, which must come to the same."""
    rng = np.random.default_rng(212)
    imgs = [_img(rng, (97, 131, 3), np.uint8), _img(rng, (50, 64, 3), np.uint8)]
    size, crop, pos = (60, 80), (40, 50), (0.3, 0.8)                    # (y, x)
    outs = _pipe(imgs, lambda fn, x: tuple(fn.resize_crop_mirror(x, size=list(size), crop=crop, crop_pos_y=pos[0], crop_pos_x=pos[1], mirror=m)
                                           for m in range(4)))
    for m, o in enumerate(outs):
        for i, im in enumerate(imgs):
            vals, b = F.resize(im, size, None, [LIN_MIN] * 2, [LIN_MAG] * 2)
            a = [int(np.floor(pos[d] * (size[d] - crop[d]) + 0.5)) for d in range(2)]
            sl = (slice(a[0], a[0] + crop[0]), slice(a[1], a[1] + crop[1]))
            flip = lambda v: v[::-1 if m & 2 else 1, ::-1 if m & 1 else 1]
            _note("fn.resize_crop_mirror u8", F.check_u8(np.asarray(o[i]), [flip(v[sl]) for v in vals], [flip(x[sl]) for x in b], (m, i)))


def test_fn_warp_affine():
    """fn.warp_affine with a destination -> source matrix (inverse_map=True, the default) and with a source -> destination one whose float
    inverse is exact, under clamp and fill, u8 and float outputs."""
    from dali_b200 import types
    rng = np.random.default_rng(213)
    imgs = [_smooth(rng, (90, 140, 3)), _smooth(rng, (64, 64, 3))]
    M = np.float32([[0.93, -0.31, 30.7], [0.29, 0.95, -12.2]])
    A = np.float32([[2.0, 0.0, 4.0], [0.0, 0.5, -3.0]])                   # its inverse [[0.5, 0, -2], [0, 2, 6]] is exact in float32
    Ainv = np.float32([[0.5, 0.0, -2.0], [0.0, 2.0, 6.0]])
    outs = _pipe(imgs, lambda fn, x: (fn.warp_affine(x, matrix=M.reshape(6).tolist(), size=[70, 300]),
                                      fn.warp_affine(x, matrix=M.reshape(6).tolist(), size=[70, 300], fill_value=200.0, dtype=types.FLOAT),
                                      fn.warp_affine(x, matrix=A.reshape(6).tolist(), inverse_map=False, fill_value=9.0)))
    for i, im in enumerate(imgs):
        for o, Mx, hw, fill, dt in ((outs[0], M, (70, 300), None, np.uint8), (outs[1], M, (70, 300), 200.0, np.float32),
                                    (outs[2], Ainv, im.shape[:2], 9.0, np.uint8)):
            got = np.asarray(o[i])
            assert np.array_equal(bits(got), bits(po.warp_affine(im, Mx, hw, 1, fill, dt))), (i, fill)
            v, b = F.warp_affine(im, Mx, hw, 1, fill)
            if dt == np.uint8:
                _note("fn.warp_affine u8", F.check_u8(got, v, b, (i, fill)))
            else:
                _note("fn.warp_affine f32", F.check(got, v, b, (i, fill)))


def test_fn_crop_mirror_normalize():
    """fn.crop_mirror_normalize from the user's mean / std / scale / shift (the library's host code turns them into the kernel's
    arguments), fp16 and fp32, CHW and HWC, channel padding, mirror, a window sticking out of the image under out_of_bounds_policy="pad"."""
    from dali_b200 import types
    rng = np.random.default_rng(214)
    imgs = [_img(rng, (50, 70, 3), np.uint8), _img(rng, (31, 29, 3), np.uint8)]
    mean, std = [123.675, 116.28, 103.53], [58.395, 57.12, 57.375]
    cfgs = [dict(crop=(24, 26), crop_pos_y=0.2, crop_pos_x=0.7, mirror=1, dtype=types.FLOAT, output_layout="CHW", scale=1.0, shift=0.0),
            dict(crop=(24, 26), crop_pos_y=0.9, crop_pos_x=0.1, mirror=0, dtype=types.FLOAT16, output_layout="HWC", scale=64.0, shift=128.0),
            dict(crop=(40, 80), crop_pos_y=0.5, crop_pos_x=0.5, mirror=1, dtype=types.FLOAT16, output_layout="CHW", pad_output=True,
                 out_of_bounds_policy="pad", fill_values=[7.5], scale=1.0, shift=0.0)]
    outs = _pipe(imgs, lambda fn, x: tuple(fn.crop_mirror_normalize(x, mean=mean, std=std, **c) for c in cfgs))
    for c, o in zip(cfgs, outs):
        for i, im in enumerate(imgs):
            H, W = im.shape[:2]
            ch, cw = c["crop"]
            rnd = lambda v: int(np.copysign(np.floor(abs(v) + 0.5), v))
            anchor = (rnd(c["crop_pos_y"] * (H - ch)), rnd(c["crop_pos_x"] * (W - cw)))
            padc = 4 if c.get("pad_output") else None
            fill = c.get("fill_values", [0.0])[0]
            v, b = F.crop_mirror_normalize(im, anchor, (ch, cw), bool(c["mirror"]), mean, std, c["scale"], c["shift"], c["output_layout"],
                                           padc, fill)
            got = np.asarray(o[i])
            dt = np.float32 if c["dtype"] == types.FLOAT else np.float16
            m32, inv32 = po.cmn_norm_args(mean, std, c["scale"], c["shift"])
            want = po.cmn(im, anchor, (ch, cw), bool(c["mirror"]), m32, inv32, dt, c["output_layout"], padc, fill)
            assert np.array_equal(bits(got), bits(want)), (c, i)
            if dt == np.float32:
                _note("fn.crop_mirror_normalize f32", F.check(got, v, b, (c, i)))
            else:
                _note("fn.crop_mirror_normalize f16", F.check_f16(got, v, b, (c, i)))


def test_resize_input_above_2g_bytes():
    """One f32 input of 23200 x 23200 (2.15 GB, more than 2^31 bytes) resized through ROIs in its far corner, so every source row the
    kernel reads sits beyond byte 2^31 and the int64 pitches carry it.  Only the corner block is filled and the statement is evaluated on
    that block with the positions of the whole image (every tap lies inside it)."""
    import torch
    rng = np.random.default_rng(215)
    H = W = 23200
    y0, x0 = 23000, 22900
    block = _img(rng, (H - y0, W - x0, 1), np.float32)
    big = torch.zeros((H, W, 1), dtype=torch.float32, device="cuda")
    big[y0:, x0:] = torch.from_numpy(block).cuda()
    assert big.numel() * 4 > 2 ** 31
    for roi in ([(23010.5, 23180.25), (22950.0, 23190.5)], [(23010.5, 23180.25), (23190.5, 22950.0)]):
        for out_hw in ((40, 60), (300, 500)):
            (got,), _, _ = _resample_dev([big], [(H, W, 1)], [out_hw], LIN_MIN, np.float32, rois=[_oracle_roi(roi)])
            vals, b = F.resize(block, out_hw, roi, [LIN_MIN] * 2, [LIN_MIN] * 2, full_shape=(H, W), origin=(y0, x0))
            _note("resize f32 > 2^31 bytes", F.check(got, vals, b, (roi, out_hw)))
    del big
    torch.cuda.empty_cache()
