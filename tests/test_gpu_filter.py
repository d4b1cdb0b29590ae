"""fn.experimental.filter on the H100.  Every output is compared bit for bit with the host build of the kernel bodies
(tools/emul/filter_emul.cc) on the same inputs, and with tests/filter_ref.py: exactly on exact-sum cases, within the gamma_k bound
otherwise.
  * every type x dtype x border x mode x layout, anchors and non-square filters, CPU and GPU filters and fill values;
  * 256 x 1080p x 3 and 256 x 224^2 x 3 batches; a 16-frame 720p FHWC sequence; a 255 x 255 filter, and filters larger than the sample;
  * the sharpness recipe of AutoAugment-style pipelines: a per-sample 3 x 3 kernel built from a magnitude, through pipeline_def,
    DALIGenericIterator and ops.experimental.Filter;
  * inputs and outputs at every byte offset 0-15, 3000 packed tiny samples, a sample alone and inside a mixed batch, outputs in one
    sentinel-filled allocation checked for stray writes;
  * the refusals."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import filter_ref as fr  # noqa: E402
import gpu_helpers as gh  # noqa: E402
from test_filter_cpu import BORDER, MODE, DTYPES, data, exact_kernel, run as host_run, emul  # noqa: E402,F401

pytestmark = pytest.mark.gpu


def capi_filter(xs, fs, layout="", anchors=None, border="reflect_101", mode="same", fills=None, dtype=None, in_offsets=None,
                out_offsets=None, packed=False, on_device=True, plan=None):
    """through the C-ABI: the inputs in one allocation at gh.byte_positions, the outputs in one sentinel-filled allocation; filters and
    fill values in device memory (on_device) or host memory"""
    from dali_b200 import capi
    lib = capi.lib()
    n, nd = len(xs), xs[0].ndim
    it, odt = fr.TYPES[xs[0].dtype], np.dtype(dtype or xs[0].dtype)
    own = plan is None
    if own:
        plan = C.c_void_p()
        capi.check(lib.dalib200FilterPlanCreate(C.byref(plan), max(n, 1)))
    try:
        oshp = (C.c_int64 * max(1, n * nd))()
        fl = [np.ascontiguousarray(f, np.float32) for f in fs]
        fv = [np.ascontiguousarray(np.asarray(v, xs[0].dtype).reshape(-1)) for v in fills] if fills is not None else None
        capi.check(lib.dalib200FilterSetup(plan, it, fr.TYPES[odt], n, nd, (C.c_int64 * max(1, n * nd))(*[e for x in xs for e in x.shape]),
                                           layout.encode(), 9, 2, (C.c_int64 * max(1, 2 * n))(*[e for f in fl for e in f.shape]),
                                           (C.c_int32 * max(1, 2 * n))(*[v for a in (anchors or [(-1, -1)] * n) for v in a]),
                                           BORDER[border], MODE[mode], it if fv is not None else -1,
                                           (C.c_int64 * max(1, n))(*[v.size for v in fv]) if fv is not None else None, oshp))
        oshapes = [tuple(oshp[i * nd:(i + 1) * nd]) for i in range(n)]
        _dev, ip = gh.upload_slices(xs, in_offsets, packed)
        keep = []
        if on_device:
            keep.append(gh.upload_slices(fl)), keep.append(gh.upload_slices(fv) if fv is not None else None)
            fp, vp = keep[0][1], keep[1][1] if fv is not None else None
        else:
            fp, vp = [f.ctypes.data for f in fl], [v.ctypes.data for v in fv] if fv is not None else None
        outs = gh.SentinelSlices([int(np.prod(s)) * odt.itemsize for s in oshapes], odt.itemsize, out_offsets, packed)
        capi.check(lib.dalib200FilterLaunch(plan, (C.c_void_p * n)(*ip), (C.c_void_p * n)(*fp), int(on_device),
                                            (C.c_void_p * n)(*vp) if vp is not None else None, int(on_device), (C.c_void_p * n)(*outs.ptrs),
                                            capi.stream_handle()))
        return [g.view(odt).reshape(s) for g, s in zip(outs.read(layout), oshapes)]
    finally:
        if own:
            lib.dalib200FilterPlanDestroy(plan)


def same_as_host(emul, xs, fs, **kw):
    got = capi_filter(xs, fs, **kw)
    host = host_run(emul, xs, fs, kw.get("layout", ""), kw.get("anchors"), kw.get("border", "reflect_101"), kw.get("mode", "same"),
                    kw.get("fills"), kw.get("dtype"))
    for g, h in zip(got, host):
        assert g.tobytes() == h.tobytes(), kw
    return got


def test_every_type_dtype_border_mode_and_layout(emul):
    rng = np.random.default_rng(1)
    for dt in DTYPES:
        for dtype in (None, np.float32):
            for border in fr.BORDERS:
                for mode in ("same", "valid"):
                    for lay in fr.LAYOUTS:
                        ext = {"F": 2, "H": 23, "W": 37, "C": 3}
                        xs = [data(rng, [ext[a] for a in lay], dt), data(rng, [ext[a] if a in "FC" else ext[a] // 3 + 5 for a in lay], dt)]
                        fs = [rng.standard_normal((3, 5)).astype(np.float32), rng.standard_normal((5, 2)).astype(np.float32)]
                        anchors = [(-1, -1), (4, 0)]
                        fills = [np.asarray(3, dt), np.asarray(100, dt)] if border == "constant" else None
                        got = same_as_host(emul, xs, fs, layout=lay, anchors=anchors, border=border, mode=mode, fills=fills, dtype=dtype,
                                           on_device=bool(rng.integers(2)))
                        for x, f, a, g, v in zip(xs, fs, anchors, got, fills or [None] * 2):
                            assert fr.within(g, x, f, lay, a, border, mode, v, dtype) == 0, (dt, dtype, border, mode, lay)


def test_exact_sums_anchors_and_non_square_filters():
    rng = np.random.default_rng(2)
    x = data(rng, (19, 23, 2), np.uint8)
    for fh, fw in ((1, 1), (1, 7), (7, 1), (3, 3), (4, 6), (7, 7)):
        f = exact_kernel(rng, fh, fw, True)
        anchors = [(r, s) for r in range(fh) for s in range(fw)]
        for border in fr.BORDERS:
            got = capi_filter([x] * len(anchors), [f] * len(anchors), "HWC", anchors, border, dtype=np.float32)
            for a, g in zip(anchors, got):
                assert np.array_equal(g, fr.filter_ref(x, f, "HWC", a, border, dtype=np.float32)), (fh, fw, a, border)


def test_255_filter_and_filters_larger_than_the_sample(emul):
    rng = np.random.default_rng(3)
    big = rng.standard_normal((255, 255)).astype(np.float32) / 255
    x = data(rng, (60, 40, 1), np.uint8)
    (g,) = same_as_host(emul, [x], [big], layout="HWC", dtype=np.float32)
    assert fr.within(g, x, big, "HWC", dtype=np.float32) == 0
    small = [data(rng, s, np.int16) // 64 for s in ((1, 1, 1), (3, 2, 3), (2, 7, 1))]
    for border in fr.BORDERS:
        got = same_as_host(emul, small, [exact_kernel(rng, 15, 9, False)] * 3, layout="HWC", border=border, dtype=np.float32)
        for x, g in zip(small, got):
            assert g.shape == x.shape
    (g,) = same_as_host(emul, [data(rng, (4, 5, 64), np.uint8)], [big], layout="HWC", border="wrap", dtype=np.float32)


def test_256_1080p_and_256_224_batches_and_a_720p_sequence():
    rng = np.random.default_rng(4)
    sharpen = np.array([[0, -1, 0], [-1, 5, -1], [0, -1, 0]], np.float32)
    imgs = [gh.synth_image(1080, 1920, k) for k in range(4)] + [rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8) for _ in range(4)]
    want = [fr.filter_ref(x, sharpen, "HWC") for x in imgs]
    got = capi_filter([imgs[i % 8] for i in range(256)], [sharpen] * 256, "HWC")
    for i in range(256):
        assert np.array_equal(got[i], want[i % 8]), i
    small = [rng.integers(0, 256, (224, 224, 3), dtype=np.uint8) if i % 3 else gh.synth_image(224, 224, i) for i in range(256)]
    blur = exact_kernel(rng, 5, 5, True)
    for x, g in zip(small, capi_filter(small, [blur] * 256, "HWC", border="clamp")):
        assert np.array_equal(g, fr.filter_ref(x, blur, "HWC", border="clamp"))
    seq = np.stack([gh.synth_image(720, 1280, 100 + f) for f in range(16)])
    fills = [np.arange(16, dtype=np.uint8) * 16]
    (g,) = capi_filter([seq], [sharpen], "FHWC", border="constant", fills=fills)
    assert np.array_equal(g, fr.filter_ref(seq, sharpen, "FHWC", border="constant", fill=fills[0]))


def sharpness_kernel(magnitude):
    """the sharpness operation of AutoAugment / RandAugment: the image blended with its smoothed version, factor 1 + magnitude"""
    blur = np.array([[1, 1, 1], [1, 5, 1], [1, 1, 1]], np.float32) / 13
    ident = np.zeros((3, 3), np.float32)
    ident[1, 1] = 1
    factor = np.float32(1 + magnitude)
    return (factor * ident + (1 - factor) * blur).astype(np.float32)


def test_sharpness_recipe_through_the_iterator_and_the_ops_class():
    import cv2
    import nvidia.dali as dali
    from nvidia.dali import fn, ops
    from nvidia.dali.plugin.pytorch import DALIGenericIterator
    streams = [np.frombuffer(cv2.imencode(".jpg", gh.synth_image(375, 500, 40 + k), [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes(), np.uint8)
               for k in range(4)]
    mags = [0.0, 0.3, 0.6, 0.9]
    kernels = [sharpness_kernel(m) for m in mags]
    flt = ops.experimental.Filter(device="gpu", border="clamp")

    @dali.pipeline_def(batch_size=4, num_threads=2, device_id=0)
    def pipe():
        img = fn.decoders.image(fn.external_source(source=lambda: streams), device="mixed")
        k = fn.external_source(source=lambda: kernels)
        return img, fn.experimental.filter(img, k, border="clamp"), flt(img, k)
    it = DALIGenericIterator([pipe()], ["img", "sharp", "sharp_ops"], size=4)
    b = next(iter(it))[0]
    for i in range(4):
        img = b["img"][i].cpu().numpy()
        for key in ("sharp", "sharp_ops"):
            assert fr.within(b[key][i].cpu().numpy(), img, kernels[i], "HWC", border="clamp") == 0, (i, key)
        assert np.array_equal(b["sharp"][i].cpu().numpy(), b["sharp_ops"][i].cpu().numpy())


def test_every_byte_offset_packed_samples_and_batch_independence(emul):
    rng = np.random.default_rng(5)
    f = rng.standard_normal((3, 4)).astype(np.float32)
    xs = [data(rng, (45, 77, 3), np.uint8), data(rng, (1, 5, 3), np.uint8)]
    host = host_run(emul, xs, [f, f], "HWC")
    host_f = host_run(emul, xs, [f, f], "HWC", dtype=np.float32)
    for a in range(16):
        for b in (a, (a + 7) % 16):
            got = capi_filter(xs, [f, f], "HWC", in_offsets=[a, a], out_offsets=[b, (b + 3) % 16])
            assert all(g.tobytes() == h.tobytes() for g, h in zip(got, host)), (a, b)
            got = capi_filter(xs, [f, f], "HWC", in_offsets=[a, a], out_offsets=[b // 4 * 4, (b + 4) % 16 // 4 * 4], dtype=np.float32)
            assert all(g.tobytes() == h.tobytes() for g, h in zip(got, host_f)), (a, b)
    for dt in (np.int16, np.float16, np.float32):
        x = data(rng, (31, 29, 2), dt)
        for a in range(0, 16, np.dtype(dt).itemsize):
            (g,) = capi_filter([x], [f], "HWC", in_offsets=[a], out_offsets=[a])
            (h,) = host_run(emul, [x], [f], "HWC")
            assert g.tobytes() == h.tobytes(), (dt, a)
    tiny = [data(rng, (int(rng.integers(0, 9)), int(rng.integers(1, 9)), 3), np.uint8) for _ in range(3000)]
    fs = [exact_kernel(rng, int(rng.integers(1, 4)), int(rng.integers(1, 4)), True) for _ in range(3000)]
    for x, g, k in zip(tiny, capi_filter(tiny, fs, "HWC", packed=True, dtype=np.float32), fs):
        assert np.array_equal(g, fr.filter_ref(x, k, "HWC", dtype=np.float32))
    one = gh.synth_image(301, 455, 7)
    g7 = rng.standard_normal((7, 7)).astype(np.float32)
    mixed = [tiny[1], one, np.zeros((0, 3, 3), np.uint8), rng.integers(0, 256, (640, 480, 3), dtype=np.uint8), one]
    mf = [fs[1], g7, g7, exact_kernel(rng, 9, 2, False), g7]
    (alone,) = capi_filter([one], [g7], "HWC")
    inmix = capi_filter(mixed, mf, "HWC", out_offsets=[1, 2, 3, 4, 5], on_device=False)
    assert alone.tobytes() == inmix[1].tobytes() == inmix[4].tobytes()


def test_refusals_name_the_problem():
    import nvidia.dali as dali
    from nvidia.dali import fn

    def run(xs, fs, layout=None, **kw):
        @dali.pipeline_def(batch_size=len(xs), num_threads=1, device_id=0, prefetch_queue_depth=1)
        def pipe():
            return fn.experimental.filter(fn.external_source(source=lambda: xs, device="gpu", layout=layout),
                                          fn.external_source(source=lambda: fs), **kw)
        p = pipe()
        p.build()
        return p.run()
    k3 = [np.ones((3, 3), np.float32)] * 2
    with pytest.raises(Exception, match="input 0 must be UINT8, INT8, UINT16, INT16, FLOAT16 or FLOAT, got INT32"):
        run([np.zeros((4, 5, 3), np.int32)] * 2, k3, "HWC")
    with pytest.raises(Exception, match='layout "CHW" of input 0 is channel-first'):
        run([np.zeros((3, 4, 5), np.uint8)] * 2, k3, "CHW")
    with pytest.raises(Exception, match="input 1 \\(the filter\\) must be FLOAT, got FLOAT64"):
        run([np.zeros((4, 5, 3), np.uint8)] * 2, [np.ones((3, 3))] * 2, "HWC")
    with pytest.raises(Exception, match="sample 1 of input 1 \\(the filter\\) has extents \\[3, 256\\]"):
        run([np.zeros((4, 5, 3), np.uint8)] * 2, [np.ones((3, 3), np.float32), np.ones((3, 256), np.float32)], "HWC")
    with pytest.raises(Exception, match='sample 0 of input 0 \\[2, 5, 3\\] is smaller than its 3 x 3 filter in "valid" mode'):
        run([np.zeros((2, 5, 3), np.uint8)] * 2, k3, "HWC", mode="valid")
    with pytest.raises(Exception, match="anchor \\(3, 0\\) is outside its 3 x 3 filter"):
        run([np.zeros((4, 5, 3), np.uint8)] * 2, k3, "HWC", anchor=[3, 0])
    with pytest.raises(Exception, match="sample 0 of input 0 has 65 channels"):
        run([np.zeros((4, 5, 65), np.uint8)] * 2, k3, "HWC")
    (o,) = run([np.full((4, 5, 3), 10, np.uint8)] * 2, k3, "HWC", border="clamp")
    assert np.array_equal(o.as_cpu()[0], np.full((4, 5, 3), 90, np.uint8))
