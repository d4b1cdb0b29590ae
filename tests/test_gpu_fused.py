"""-m gpu parity tests of decode -> resize without the RGB image (SURVEY 8f rank 1): the resampler reads the decoder's 4:2:0 planes
(dalib200JpegPlanSetPlanesOnly / GetPlanes -> dalib200ResampleLaunchPlanar) and must equal full decode followed by resize -- and, with a
region of interest, crop-then-resize -- bit for bit."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


def _enc(img, q=90, ss=None):
    import cv2
    params = [cv2.IMWRITE_JPEG_QUALITY, q]
    if ss is not None:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, ss]
    ok, enc = cv2.imencode(".jpg", img, params)
    assert ok
    return enc.tobytes()


def _fused(streams, out_hws, rois=None, filt=(capi.FILTER_LINEAR, 1, 0.0), infos=None):
    """decode (planes only where granted) + planar resample with `filt` as min and mag filter; returns (outputs, granted flags).  infos: a
    list that receives dalib200ResamplePlanGetStreamInfo of every sample of the planar plan."""
    import torch
    import gpu_helpers as g
    lib = capi.lib()
    n = len(streams)
    bufs = [np.frombuffer(bytes(s), np.uint8) for s in streams]
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    lens = (C.c_size_t * n)(*[b.size for b in bufs])
    jp, rp, rb = capi.Plan("Jpeg", n), capi.Plan("Resample", n), capi.Plan("Resample", n)
    prm = capi.JpegParams(capi.RGB, 1, capi.UINT8, 1)
    cr = None
    if rois is not None:
        cr = (capi.JpegRoi * n)()
        for i, r in enumerate(rois):
            if r is not None:
                cr[i].use_roi = 1
                cr[i].x0, cr[i].y0, cr[i].x1, cr[i].y1 = r
    capi.check(lib.dalib200JpegPlanSetupEx(jp.handle, n, ptrs, lens, C.byref(prm), cr))
    shapes = []
    for i in range(n):
        hwc = (C.c_int32 * 3)()
        capi.check(lib.dalib200JpegPlanGetOutputShape(jp.handle, i, hwc))
        shapes.append(tuple(hwc))
    rs = (capi.ResampleSample * n)()
    for i in range(n):
        g.fill_resample_sample(rs[i], shapes[i], out_hws[i], filt, filt, None)
    ok = (C.c_uint8 * n)()
    capi.check(lib.dalib200ResamplePlanSetupPlanar(rp.handle, n, rs, ok))
    granted = (C.c_uint8 * n)()
    capi.check(lib.dalib200JpegPlanSetPlanesOnly(jp.handle, ok, granted))
    if list(ok) != list(granted):
        for i in range(n):
            if not granted[i]:
                rs[i].channels = 1
        capi.check(lib.dalib200ResamplePlanSetupPlanar(rp.handle, n, rs, ok))
        for i in range(n):
            rs[i].channels = 3
    if infos is not None:
        infos.extend(capi.resample_stream_info(rp, i) for i in range(n))
    dec = [torch.empty(s, dtype=torch.uint8, device="cuda") for s in shapes]
    outs = [torch.zeros((hw[0], hw[1], 3), dtype=torch.uint8, device="cuda") for hw in out_hws]
    capi.check(lib.dalib200JpegUpload(jp.handle, capi.stream_handle()))
    capi.check(lib.dalib200JpegLaunch(jp.handle, capi.ptr_array(dec), capi.stream_handle()))
    srcs = (capi.PlanarImage * n)()
    for i in range(n):
        if granted[i]:
            capi.check(lib.dalib200JpegPlanGetPlanes(jp.handle, i, C.byref(srcs[i])))
            if rois is not None and rois[i] is not None:
                srcs[i].crop_x, srcs[i].crop_y = rois[i][0], rois[i][1]
    capi.check(lib.dalib200ResampleLaunchPlanar(rp.handle, srcs, capi.ptr_array(outs), capi.stream_handle()))
    rest = [i for i in range(n) if not granted[i]]
    if rest:
        rsb = (capi.ResampleSample * len(rest))(*[rs[i] for i in rest])
        capi.check(lib.dalib200ResamplePlanSetup(rb.handle, len(rest), rsb, capi.UINT8, capi.UINT8))
        capi.check(lib.dalib200ResampleLaunch(rb.handle, capi.ptr_array([dec[i] for i in rest]), capi.ptr_array([outs[i] for i in rest]),
                                              capi.stream_handle()))
    torch.cuda.synchronize()
    st = (C.c_int32 * n)()
    capi.check(lib.dalib200JpegGetStatus(jp.handle, st))
    assert list(st) == [0] * n
    return [o.cpu().numpy() for o in outs], list(granted)


def test_planar_resize_equals_decode_then_resize():
    import cv2
    import gpu_helpers as g
    s420, s444 = cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444
    streams = [_enc(g.synth_image(480, 640, 1), 90, s420), _enc(g.synth_image(1080, 1920, 2), 90, s420), _enc(g.synth_image(333, 517, 3), 80, s420),
               _enc(g.synth_image(301, 299, 4), 95, s420), _enc(g.synth_image(300, 400, 5), 90, s444), _enc(g.synth_image(64, 48, 6), 90, s420),
               _enc(g.synth_image(900, 1203, 7), 60, s420), _enc(g.synth_image(768, 1024, 8)[..., 0], 90)]
    out_hws = [(224, 224), (224, 224), (100, 160), (96, 96), (128, 128), (48, 36), (256, 341), (200, 200)]
    outs, granted = _fused(streams, out_hws)
    assert granted[1] and granted[2] and granted[6], granted       # 4:2:0 down-scales whose vertical pass comes first take the planar path
    assert not granted[4] and not granted[7]                                       # 4:4:4 and grayscale streams do not
    for i, s in enumerate(streams):
        want = po.resample(po.jpeg_decode(s), out_hws[i])
        assert np.array_equal(outs[i], want), (i, granted[i])


def test_planar_resize_with_region_of_interest_equals_crop_then_resize():
    import cv2
    import gpu_helpers as g
    s420 = cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420
    streams = [_enc(g.synth_image(720, 1280, 11), 90, s420), _enc(g.synth_image(1080, 1920, 12), 85, s420), _enc(g.synth_image(600, 800, 13), 90, s420),
               _enc(g.synth_image(513, 771, 14), 90, s420)]
    rng = np.random.default_rng(2)
    for rep in range(4):
        rois, out_hws = [], []
        for s in streams:
            info = po.jpeg_info(s)
            H, W = info["height"], info["width"]
            w, h = int(rng.integers(W // 3, W + 1)), int(rng.integers(H // 3, H + 1))
            x0, y0 = int(rng.integers(0, W - w + 1)), int(rng.integers(0, H - h + 1))
            rois.append((x0, y0, x0 + w, y0 + h))
            out_hws.append((int(rng.integers(32, 160)), int(rng.integers(32, 160))))
        outs, granted = _fused(streams, out_hws, rois)
        for i, s in enumerate(streams):
            x0, y0, x1, y1 = rois[i]
            want = po.resample(np.ascontiguousarray(po.jpeg_decode(s)[y0:y1, x0:x1]), out_hws[i])
            assert np.array_equal(outs[i], want), (rep, i, rois[i], out_hws[i], granted[i])
        assert any(granted)
