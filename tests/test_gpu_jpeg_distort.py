"""-m gpu tests of fn.jpeg_compression_distortion: the CUDA path (forward DCT kernel + the decoder's reconstruct kernels) against
cv2.imdecode(cv2.imencode(".jpg", img, quality)), bit for bit, through the C-ABI and through pipeline_def / fn."""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import jpeg_distort_cases as jc  # noqa: E402


def _samples(shapes_q):
    arr = (capi.JpegDistortSample * max(1, len(shapes_q)))()
    for s, ((h, w), q) in zip(arr, shapes_q):
        s.height, s.width, s.quality = h, w, q
    return arr


def _distort(imgs, qs, plan=None):
    import torch
    plan = plan or capi.Plan("JpegDistort", len(imgs))
    capi.check(capi.lib().dalib200JpegDistortPlanSetup(plan.handle, len(imgs), _samples([(i.shape[:2], q) for i, q in zip(imgs, qs)])))
    src = [torch.from_numpy(np.ascontiguousarray(i)).cuda() for i in imgs]
    dst = [torch.full_like(s, 77) for s in src]
    capi.check(capi.lib().dalib200JpegDistortLaunch(plan.handle, capi.ptr_array(src), capi.ptr_array(dst), capi.stream_handle()))
    torch.cuda.synchronize()
    return [d.cpu().numpy() for d in dst], plan


def test_grid_bit_exact_with_cv2():
    imgs, qs = [], []
    for si, (h, w) in enumerate(jc.SIZES):
        for ki, kind in enumerate(jc.KINDS):
            for q in jc.QUALITIES:
                imgs.append(jc.image(h, w, kind, 1000 * si + 100 * ki + q))
                qs.append(q)
    outs, _ = _distort(imgs, qs)
    for img, q, o in zip(imgs, qs, outs):
        want = jc.reference(img, q)
        assert np.array_equal(o, want), (img.shape, q, int(np.abs(o.astype(int) - want).max()))


def test_mixed_batch_widths_1_to_4_and_1080p():
    """one batch: widths 1..4 (the decoder's box-upsampling path), odd sizes and a 1080p image, each with its own quality"""
    rng = np.random.default_rng(7)
    shapes = [(5, 1), (6, 2), (7, 3), (8, 4), (33, 4), (1, 3), (1080, 1920), (17, 5), (31, 6), (64, 64), (2, 1)]
    imgs = [jc.image(h, w, jc.KINDS[k % 3], k) for k, (h, w) in enumerate(shapes)]
    qs = [int(q) for q in rng.integers(1, 101, len(imgs))]
    outs, _ = _distort(imgs, qs)
    for img, q, o in zip(imgs, qs, outs):
        assert np.array_equal(o, jc.reference(img, q)), (img.shape, q)


def test_debug_coefficients_equal_cv2_stream():
    import torch  # noqa: F401
    imgs = [jc.image(97, 131, "smooth", 1), jc.image(9, 3, "noise", 2), jc.image(224, 224, "saturated", 3)]
    qs = [75, 10, 99]
    _, plan = _distort(imgs, qs)
    for i, (img, q) in enumerate(zip(imgs, qs)):
        want = jc.mcu_coefficients(jc.encode(img, q))
        got = np.zeros(want.size, np.int16)
        capi.check(capi.lib().dalib200JpegDistortDebugGetCoefficients(plan.handle, i, got.ctypes.data_as(C.c_void_p), C.c_size_t(got.size)))
        assert np.array_equal(got, want), i


def test_plan_reuse_with_growing_sizes():
    plan = capi.Plan("JpegDistort", 4)
    for step, (shapes, q) in enumerate([([(16, 16)], 50), ([(3, 2), (120, 200)], 90), ([(480, 640), (1, 1), (250, 3), (301, 517)], 20),
                                        ([(8, 8)], 100)]):
        imgs = [jc.image(h, w, "noise", 10 * step + k) for k, (h, w) in enumerate(shapes)]
        outs, _ = _distort(imgs, [q] * len(imgs), plan)
        for img, o in zip(imgs, outs):
            assert np.array_equal(o, jc.reference(img, q)), (step, img.shape)


def test_sequences_and_per_sample_quality_through_fn():
    """FHWC sequences whose frame sizes differ per sample; every frame takes its sample's quality (a per-sample argument input), and
    the default quality is 50"""
    from dali_b200 import fn, pipeline_def
    seqs = [np.stack([jc.image(37, 53, "smooth", 10 + f) for f in range(3)]), np.stack([jc.image(16, 9, "noise", 20 + f) for f in range(2)]),
            np.stack([jc.image(3, 2, "saturated", 30)])]
    quals = [np.array(q, np.int32) for q in (15, 95, 60)]

    @pipeline_def(batch_size=len(seqs), num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: seqs, device="gpu", layout="FHWC")
        q = fn.external_source(source=lambda i: quals)
        return fn.jpeg_compression_distortion(x, quality=q), fn.jpeg_compression_distortion(x)
    p = pipe()
    p.build()
    a, b = [o.as_cpu() for o in p.run()]
    for i, s in enumerate(seqs):
        ga, gb = np.asarray(a[i]), np.asarray(b[i])
        assert ga.shape == s.shape and gb.shape == s.shape
        for f in range(s.shape[0]):
            assert np.array_equal(ga[f], jc.reference(s[f], int(quals[i]))), (i, f)
            assert np.array_equal(gb[f], jc.reference(s[f], 50)), (i, f)


def test_hwc_images_through_ops_api():
    from dali_b200 import ops, pipeline_def, fn
    imgs = [jc.image(64, 48, "smooth", 1), jc.image(21, 30, "noise", 2)]

    @pipeline_def(batch_size=len(imgs), num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: imgs, device="gpu", layout="HWC")
        return ops.JpegCompressionDistortion(quality=33)(x)
    p = pipe()
    p.build()
    (out,) = p.run()
    out = out.as_cpu()
    for i, img in enumerate(imgs):
        assert np.array_equal(np.asarray(out[i]), jc.reference(img, 33)), i


@pytest.mark.parametrize("case", ["quality0", "quality101", "float", "four_channels", "chw"])
def test_operator_rejects_with_message(case):
    from dali_b200 import fn, pipeline_def
    img = jc.image(8, 8, "noise", 0)
    data = {"float": [img.astype(np.float32)], "four_channels": [np.zeros((8, 8, 4), np.uint8)]}.get(case, [img])
    layout = "CHW" if case == "chw" else "HWC"
    quality = {"quality0": 0, "quality101": 101}.get(case, 50)
    want = {"quality0": "quality must be in [1, 100]", "quality101": "quality must be in [1, 100]", "float": "must be uint8",
            "four_channels": "3 channels", "chw": "HWC and FHWC"}[case]

    @pipeline_def(batch_size=1, num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: data, device="gpu", layout=layout)
        return fn.jpeg_compression_distortion(x, quality=quality)
    p = pipe()
    with pytest.raises(Exception, match=re.escape(want)):
        p.build()
        p.run()


def test_capi_rejects_with_message():
    plan = capi.Plan("JpegDistort", 2)
    lib = capi.lib()
    for shapes_q, want in [([((8, 8), 0)], "quality 0 is outside"), ([((8, 8), 101)], "quality 101 is outside"),
                           ([((65501, 8), 50)], "each side must be in"), ([((8, 0), 50)], "each side must be in"),
                           ([((65500, 65500), 50)], "2^31 or more elements")]:
        rc = lib.dalib200JpegDistortPlanSetup(plan.handle, len(shapes_q), _samples(shapes_q))
        assert rc == 1, want
        assert want in lib.dalib200GetLastError().decode(), want
    assert lib.dalib200JpegDistortPlanSetup(plan.handle, 3, _samples([((8, 8), 50)] * 3)) == 1      # above max_batch
