"""fn.experimental.equalize on the H100, every output compared bit for bit with cv2.equalizeHist applied to each (frame, channel)
plane of the input:
  * the six layouts and the empty layout; 1 to 16 channels, and the refusal of 17;
  * synthetic images encoded to JPEG, decoded and equalized through pipeline_def and DALIGenericIterator, and through
    ops.experimental.Equalize;
  * 256 x 1080p x 3 and 256 x 224^2 x 3 batches; a 16-frame 720p FHWC sequence; flat and two-valued images;
  * a plane of more than 2^24 pixels on which rounding the running sum to float changes a table entry;
  * inputs and outputs at every byte offset 0-15, 3000 packed tiny samples, a sample alone and inside a mixed batch, outputs in one
    sentinel-filled allocation checked for stray writes;
  * the refusals of a non-uint8 input, a bad layout and a CPU input."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import equalize_ref as er  # noqa: E402
import gpu_helpers as gh  # noqa: E402

pytestmark = pytest.mark.gpu
MAX_C = 16


def cv2_equalize(x, layout=""):
    """cv2.equalizeHist on every (frame, channel) plane"""
    import cv2
    if not x.size:
        return x.copy()
    lay = layout or er.BY_RANK[x.ndim]
    hw = [lay.index("H"), lay.index("W")]
    y = np.moveaxis(x, hw, [-2, -1]).copy()
    flat = y.reshape(-1, y.shape[-2], y.shape[-1])
    for k in range(flat.shape[0]):
        if flat[k].size:
            flat[k] = cv2.equalizeHist(np.ascontiguousarray(flat[k]))
    return np.moveaxis(flat.reshape(y.shape), [-2, -1], hw)


def _run(build, batches, layout=None, batch_size=None):
    import nvidia.dali as dali
    from nvidia.dali import fn
    state = {}

    @dali.pipeline_def(batch_size=batch_size or max(len(b) for b in batches), num_threads=1, device_id=0, prefetch_queue_depth=1)
    def pipe():
        return build(fn.external_source(source=lambda: state["b"], device="gpu", layout=layout))
    p = pipe()
    p.build()
    res = []
    for b in batches:
        state["b"] = b
        (o,) = p.run()
        res.append((o.as_cpu(), o.layout()))
    return res


def equalize_fn(xs, layout=None, batch_size=None):
    from nvidia.dali import fn
    ((out, lay),) = _run(lambda x: fn.experimental.equalize(x), [xs], layout, batch_size)
    return [out[i] for i in range(len(xs))], lay


def capi_equalize(xs, layout="", in_offsets=None, out_offsets=None, packed=False, plan=None):
    """through the C-ABI: the inputs in one allocation at gh.byte_positions, the outputs in one sentinel-filled allocation"""
    from dali_b200 import capi
    lib = capi.lib()
    n, nd = len(xs), xs[0].ndim
    own = plan is None
    if own:
        plan = C.c_void_p()
        capi.check(lib.dalib200EqualizePlanCreate(C.byref(plan), max(n, 1)))
    try:
        shp = (C.c_int64 * max(1, n * nd))(*[e for x in xs for e in x.shape])
        capi.check(lib.dalib200EqualizeSetup(plan, 0, n, nd, shp, layout.encode()))
        _dev, ip = gh.upload_slices(xs, in_offsets, packed)
        outs = gh.SentinelSlices([x.nbytes for x in xs], 1, out_offsets, packed)
        capi.check(lib.dalib200EqualizeLaunch(plan, (C.c_void_p * n)(*ip), (C.c_void_p * n)(*outs.ptrs), capi.stream_handle()))
        return [g.reshape(x.shape) for g, x in zip(outs.read(layout), xs)]
    finally:
        if own:
            lib.dalib200EqualizePlanDestroy(plan)


def check(got, xs, layout, what):
    for i, x in enumerate(xs):
        assert np.array_equal(np.asarray(got[i]), cv2_equalize(x, layout)), (what, i, x.shape)


def _images(rng, shape, kinds=(0, 1, 2, 3)):
    out = []
    for k in kinds:
        if k == 0:
            out.append(rng.integers(0, 256, shape, dtype=np.uint8))
        elif k == 1:
            out.append(rng.integers(90, 110, shape, dtype=np.uint8))
        elif k == 2:
            out.append(rng.choice(np.array([3, 200], np.uint8), shape))
        else:
            out.append(np.full(shape, int(rng.integers(0, 256)), np.uint8))
    return out


def test_every_layout_and_the_empty_layout():
    rng = np.random.default_rng(1)
    for lay in er.LAYOUTS + ("",):
        named = lay or "FHWC"
        ext = {"F": 3, "H": 67, "W": 129, "C": 3}
        xs = _images(rng, [ext[a] for a in named]) + [rng.integers(0, 256, [ext[a] * (1 if a in "FC" else 4) for a in named], dtype=np.uint8)]
        got, out_layout = equalize_fn(xs, lay or None)
        assert out_layout == lay
        check(got, xs, lay, ("layout", lay))


def test_channels_1_to_the_limit_and_one_above():
    rng = np.random.default_rng(2)
    for c in range(1, MAX_C + 1):
        for lay, shape in (("HWC", (61, 97, c)), ("CHW", (c, 61, 97))):
            xs = [rng.integers(0, 256, shape, dtype=np.uint8), rng.choice(np.array([9, 77, 250], np.uint8), shape)]
            check(equalize_fn(xs, lay)[0], xs, lay, ("channels", c, lay))
    with pytest.raises(Exception, match=f"sample 1 of input 0 has {MAX_C + 1} channels"):
        equalize_fn([np.zeros((4, 5, 3), np.uint8), np.zeros((4, 5, MAX_C + 1), np.uint8)], "HWC")


def test_jpeg_decode_then_equalize_through_the_iterator_and_the_ops_class():
    import cv2
    import nvidia.dali as dali
    from nvidia.dali import fn, ops
    from nvidia.dali.plugin.pytorch import DALIGenericIterator
    streams = [np.frombuffer(cv2.imencode(".jpg", gh.synth_image(375, 500, 40 + k), [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes(), np.uint8)
               for k in range(4)]
    eq = ops.experimental.Equalize(device="gpu")

    @dali.pipeline_def(batch_size=4, num_threads=2, device_id=0)
    def pipe():
        img = fn.decoders.image(fn.external_source(source=lambda: streams), device="mixed")
        return img, fn.experimental.equalize(img), eq(img)
    it = DALIGenericIterator([pipe()], ["img", "eq", "eq_ops"], size=4)
    b = next(iter(it))[0]
    for i in range(4):
        img = b["img"][i].cpu().numpy()
        want = cv2_equalize(img, "HWC")
        assert np.array_equal(b["eq"][i].cpu().numpy(), want), i
        assert np.array_equal(b["eq_ops"][i].cpu().numpy(), want), i


def test_256_1080p_and_256_224_batches():
    rng = np.random.default_rng(3)
    imgs = [gh.synth_image(1080, 1920, k) for k in range(4)] + _images(rng, (1080, 1920, 3), (0, 2, 3)) + \
        [rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8)]
    batch = [imgs[i % 8] for i in range(256)]
    got, _ = equalize_fn(batch, "HWC")
    want = [cv2_equalize(x, "HWC") for x in imgs]
    for i in range(256):
        assert np.array_equal(np.asarray(got[i]), want[i % 8]), i
    small = [rng.integers(0, 256, (224, 224, 3), dtype=np.uint8) if i % 3 else gh.synth_image(224, 224, i) for i in range(256)]
    check(equalize_fn(small, "HWC")[0], small, "HWC", "224")
    chw = [np.ascontiguousarray(x.transpose(2, 0, 1)) for x in small[:64]]
    check(equalize_fn(chw, "CHW")[0], chw, "CHW", "224 CHW")


def test_16_frame_720p_sequence_flat_and_two_valued():
    rng = np.random.default_rng(4)
    seq = np.stack([gh.synth_image(720, 1280, 100 + f) for f in range(16)])
    seq[3] = 17                                                  # a flat frame
    seq[5, :, :, 1] = rng.choice(np.array([0, 255], np.uint8), (720, 1280))
    check(equalize_fn([seq, seq[:2].copy()], "FHWC")[0], [seq, seq[:2]], "FHWC", "720p sequence")
    flat = [np.full((50, 70, 3), v, np.uint8) for v in (0, 1, 128, 255)] + [np.full((1, 1), 9, np.uint8).reshape(1, 1, 1)]
    two = [rng.choice(np.array([a, b], np.uint8), (50, 70, 3)) for a, b in ((0, 255), (10, 11), (200, 3), (254, 255))]
    check(equalize_fn(flat + two, "HWC")[0], flat + two, "HWC", "flat and two-valued")


def test_plane_above_2_pow_24_where_float_sum_rounding_changes_an_entry():
    x, _d, _s = er.big_plane()
    (got,) = capi_equalize([x], "HW")
    assert got[0, 1] == 164                                      # 163 with the exact sum
    check([got], [x], "HW", "2^24")


def test_every_byte_offset_of_input_and_output():
    rng = np.random.default_rng(5)
    xs = [rng.integers(0, 256, (45, 77, 3), dtype=np.uint8), rng.choice(np.array([5, 6], np.uint8), (3, 45, 77)),
          rng.integers(0, 256, (1, 5, 3), dtype=np.uint8)]
    for a in range(16):
        for b in (a, (a + 7) % 16):
            for lay, ys in (("HWC", [xs[0], xs[2]]), ("CHW", [xs[1], xs[1]])):
                check(capi_equalize(ys, lay, [a] * len(ys), [b, (b + 3) % 16]), ys, lay, ("offset", a, b))


def test_3000_packed_tiny_samples_and_a_sample_alone_and_in_a_mixed_batch():
    rng = np.random.default_rng(6)
    xs = [rng.integers(0, 256, (int(rng.integers(0, 9)), int(rng.integers(1, 9)), 3), dtype=np.uint8) for _ in range(3000)]
    check(capi_equalize(xs, "HWC", packed=True), xs, "HWC", "packed")
    one = gh.synth_image(301, 455, 7)
    mixed = [xs[1], one, np.zeros((0, 3, 3), np.uint8), rng.integers(0, 256, (640, 480, 3), dtype=np.uint8), one]
    (alone,) = capi_equalize([one], "HWC")
    inmix = capi_equalize(mixed, "HWC", out_offsets=[1, 2, 3, 4, 5])
    assert alone.tobytes() == inmix[1].tobytes() == inmix[4].tobytes()
    check(inmix, mixed, "HWC", "mixed")


def test_refusals_name_the_problem():
    import nvidia.dali as dali
    from nvidia.dali import fn
    with pytest.raises(Exception, match="must be UINT8, got FLOAT"):
        equalize_fn([np.zeros((4, 5, 3), np.float32)] * 2, "HWC")
    with pytest.raises(Exception, match='layout "WHC" of input 0 is not supported'):
        equalize_fn([np.zeros((4, 5, 3), np.uint8)] * 2, "WHC")
    with pytest.raises(Exception, match="cannot infer the layout of 5-dimensional input 0"):
        equalize_fn([np.zeros((1, 2, 4, 5, 3), np.uint8)] * 2)

    @dali.pipeline_def(batch_size=2, num_threads=1, device_id=0)
    def cpu_pipe():
        return fn.experimental.equalize(fn.external_source(source=lambda: [np.zeros((4, 5, 3), np.uint8)] * 2, layout="HWC"))
    with pytest.raises(Exception, match="(?i)cpu"):
        p = cpu_pipe()
        p.build()
        p.run()
