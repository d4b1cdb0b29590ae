"""fn.erase on the H100, bit for bit against tests/erase_ref.py (and, where the reference is too slow at full size, against torch's
clone and slice assignment of the same boxes):
  * every type x layout, and every non-empty subset of erased axes at rank 4;
  * 256 x 1080p x 3 uint8 with one region per image; 256 x 3 x 224^2 FLOAT16 CHW after crop_mirror_normalize;
  * a SpecAugment batch through DALIGenericIterator: 64 WAV clips of 10 s -> mel 128 "ft" -> two frequency masks and ten time masks per
    clip, from CPU tensor inputs; the ops.Erase class;
  * 64 regions per sample; 3000 packed tiny samples; one uint8 sample of more than 2^31 elements;
  * inputs and outputs at every byte offset; a sample alone and inside a mixed batch; outputs in one sentinel-filled allocation
    checked for stray writes;
  * the refusals."""
import ctypes as C
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import erase_ref as er  # noqa: E402
import gpu_helpers as gh  # noqa: E402
from test_erase_cpu import DTYPES, LAYOUTS, EXT, data, flat, random_regions  # noqa: E402

pytestmark = pytest.mark.gpu


def capi_erase(xs, axes, anchors, rshapes, fill=(0.0,), layout="", names=None, na=False, ns=False, cen=False, in_offsets=None,
               out_offsets=None, packed=False):
    """through the C-ABI: the inputs in one allocation at gh.byte_positions, the outputs in one sentinel-filled allocation"""
    from dali_b200 import capi
    lib = capi.lib()
    n, nd = len(xs), xs[0].ndim
    plan = C.c_void_p()
    capi.check(lib.dalib200ErasePlanCreate(C.byref(plan), max(n, 1)))
    try:
        av = flat([v for a in anchors for v in flat(a)] or [0])
        sv = flat([v for a in rshapes for v in flat(a)] or [0])
        capi.check(lib.dalib200EraseSetup(plan, er.TYPES[xs[0].dtype], n, nd, (C.c_int64 * (n * nd))(*[e for x in xs for e in x.shape]),
                                          layout.encode(), names.encode() if names is not None else None, (C.c_int32 * len(axes))(*axes),
                                          len(axes), (C.c_float * len(av))(*av), (C.c_int64 * n)(*[len(flat(a)) for a in anchors]),
                                          (C.c_float * len(sv))(*sv), (C.c_int64 * n)(*[len(flat(a)) for a in rshapes]), int(na), int(ns),
                                          int(cen), (C.c_float * len(flat(fill)))(*flat(fill)), len(flat(fill))))
        _dev, ip = gh.upload_slices(xs, in_offsets, packed)
        outs = gh.SentinelSlices([x.nbytes for x in xs], xs[0].itemsize, out_offsets, packed)
        capi.check(lib.dalib200EraseLaunch(plan, (C.c_void_p * n)(*ip), (C.c_void_p * n)(*outs.ptrs), capi.stream_handle()))
        return [g.view(x.dtype).reshape(x.shape) for g, x in zip(outs.read(layout), xs)]
    finally:
        lib.dalib200ErasePlanDestroy(plan)


def check(xs, axes, anchors, rshapes, fill=(0.0,), layout="", names=None, na=False, ns=False, cen=False, **kw):
    got = capi_erase(xs, axes, anchors, rshapes, fill, layout, names, na, ns, cen, **kw)
    for x, g, a, s in zip(xs, got, anchors, rshapes):
        assert g.tobytes() == er.erase_ref(x, axes, a, s, fill, layout, na, ns, cen).tobytes(), (x.dtype, x.shape, layout, axes)
    return got


def test_every_type_layout_and_axis_subset():
    rng = np.random.default_rng(1)
    for lay in LAYOUTS:
        nd = len(lay)
        subsets = [c for r in range(1, nd + 1) for c in itertools.combinations(range(nd), r)] if nd == 4 else \
            [tuple(range(nd)), (nd - 1,), (0,)]
        for sub in subsets:
            for dt in DTYPES:
                axes = list(sub)
                shapes = [[EXT[c] * 3 if c != "C" else 3 for c in lay], [EXT[c] if c == "C" else EXT[c] // 2 + 1 for c in lay]]
                xs = [data(rng, s, dt) for s in shapes]
                regs = [random_regions(rng, s, axes, int(rng.integers(1, 4))) for s in shapes]
                fill = (1.0, 2.0, 3.0) if "C" in lay and lay.index("C") not in axes else (7.0,)
                check(xs, axes, [r[0] for r in regs], [r[1] for r in regs], fill, lay, "".join(lay[a] for a in axes))


def timm_region(rng, h, w, area=(0.02, 1 / 3), ratio=(0.3, 3.3)):
    """timm RandomErasing's rectangle: area fraction and log-uniform aspect, as (y, x), (h, w)"""
    while True:
        a = rng.uniform(*area) * h * w
        r = np.exp(rng.uniform(np.log(ratio[0]), np.log(ratio[1])))
        eh, ew = int(round(np.sqrt(a * r))), int(round(np.sqrt(a / r)))
        if eh < h and ew < w:
            return [float(rng.integers(0, h - eh + 1)), float(rng.integers(0, w - ew + 1))], [float(eh), float(ew)]


def test_256_1080p_uint8_one_region_each():
    rng = np.random.default_rng(2)
    imgs = [gh.synth_image(1080, 1920, k) for k in range(4)] + [rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8) for _ in range(4)]
    regs = [timm_region(rng, 1080, 1920) for _ in range(256)]
    xs = [imgs[i % 8] for i in range(256)]
    got = capi_erase(xs, [0, 1], [r[0] for r in regs], [r[1] for r in regs], (0.0,), "HWC", "HW")
    for i in range(256):
        assert got[i].tobytes() == er.erase_ref(xs[i], [0, 1], regs[i][0], regs[i][1], (0.0,)).tobytes(), i


def test_256_fp16_chw_after_crop_mirror_normalize():
    import nvidia.dali as dali
    from nvidia.dali import fn, types
    rng = np.random.default_rng(3)
    imgs = [rng.integers(0, 256, (256, 256, 3), dtype=np.uint8) for _ in range(8)]
    regs = [timm_region(rng, 224, 224) for _ in range(256)]
    anchors = [np.array(r[0], np.float32) for r in regs]
    shapes = [np.array(r[1], np.float32) for r in regs]
    fill = (0.5, -1.0, 70000.0)

    @dali.pipeline_def(batch_size=256, num_threads=2, device_id=0, prefetch_queue_depth=1)
    def pipe():
        img = fn.external_source(source=lambda: [imgs[i % 8] for i in range(256)], device="gpu", layout="HWC")
        x = fn.crop_mirror_normalize(img, crop=(224, 224), dtype=types.FLOAT16, output_layout="CHW", mean=[120.0, 110.0, 100.0],
                                     std=[60.0, 61.0, 62.0])
        return x, fn.erase(x, anchor=fn.external_source(source=lambda: anchors), shape=fn.external_source(source=lambda: shapes),
                           axis_names="HW", fill_value=list(fill))
    p = pipe()
    p.build()
    x, y = p.run()
    assert y.layout() == "CHW"
    for i in range(256):
        xi, yi = x.as_cpu()[i], y.as_cpu()[i]
        assert yi.dtype == np.float16 and yi.tobytes() == er.erase_ref(xi, [1, 2], anchors[i], shapes[i], fill, "CHW").tobytes(), i


def spec_augment_masks(rng, F, T, nf=2, nt=10, fmax=27, tmax=100):
    fa = [[float(rng.integers(0, F)), 0.0] for _ in range(nf)]
    fs = [[float(rng.integers(0, fmax + 1)), float(2 * T)] for _ in range(nf)]
    ta = [float(rng.integers(0, T)) for _ in range(nt)]
    ts = [float(rng.integers(0, tmax + 1)) for _ in range(nt)]
    return np.array(fa, np.float32).reshape(-1), np.array(fs, np.float32).reshape(-1), np.array(ta, np.float32), np.array(ts, np.float32)


def test_spec_augment_batch_through_the_iterator_and_the_ops_class():
    import nvidia.dali as dali
    from nvidia.dali import fn, ops, types
    from nvidia.dali.plugin.pytorch import DALIGenericIterator
    import audio_streams as aus
    rng = np.random.default_rng(4)
    clips = [aus.wav_pcm(rng.integers(-20000, 20000, (160000, 1)), 16, 16000) for _ in range(64)]
    streams = [np.frombuffer(c, np.uint8) for c in clips]
    T = 1000                                                               # about the frames; masks past the end are clipped
    masks = [spec_augment_masks(rng, 128, T) for _ in range(64)]
    erase_t = ops.Erase(device="gpu", axis_names="t", fill_value=-3.5)

    def column(k):
        return lambda: [m[k] for m in masks]

    @dali.pipeline_def(batch_size=64, num_threads=2, device_id=0)
    def pipe():
        audio, _ = fn.decoders.audio(fn.external_source(source=lambda: streams), downmix=True, dtype=types.FLOAT)
        spec = fn.spectrogram(audio, nfft=512, window_length=400, window_step=160)
        mel = fn.mel_filter_bank(spec, sample_rate=16000.0, nfilter=128)
        fa, fs, ta, ts = (fn.external_source(source=column(k)) for k in range(4))
        f_masked = fn.erase(mel, anchor=fa, shape=fs, axis_names="ft", fill_value=0.0)
        both = erase_t(f_masked, anchor=ta, shape=ts)
        only_t = fn.erase(mel, anchor=ta, shape=ts, axis_names="t", fill_value=-3.5)
        return mel, both, only_t
    it = DALIGenericIterator([pipe()], ["mel", "both", "only_t"], size=64)
    b = next(iter(it))[0]
    for i in range(64):
        mel = b["mel"][i].cpu().numpy()
        fa, fs, ta, ts = masks[i]
        assert mel.shape[0] == 128
        f_masked = er.erase_ref(mel, [0, 1], fa, fs, (0.0,))
        assert b["both"][i].cpu().numpy().tobytes() == er.erase_ref(f_masked, [1], ta, ts, (-3.5,)).tobytes(), i
        assert b["only_t"][i].cpu().numpy().tobytes() == er.erase_ref(mel, [1], ta, ts, (-3.5,)).tobytes(), i


def test_64_regions_per_sample_and_3000_packed_tiny_samples():
    rng = np.random.default_rng(5)
    xs = [rng.integers(0, 256, (540, 960, 3), dtype=np.uint8) for _ in range(8)]
    regs = [random_regions(rng, x.shape, [0, 1], 64) for x in xs]
    check(xs, [0, 1], [r[0] for r in regs], [r[1] for r in regs], (255.0,), "HWC", "HW")
    seqs = [data(rng, (4, 60, 70, 3), np.float32) for _ in range(2)]
    regs = [random_regions(rng, x.shape, [0, 1, 2], 64) for x in seqs]
    check(seqs, [0, 1, 2], [r[0] for r in regs], [r[1] for r in regs], (1.0, 2.0, 3.0), "FHWC", "FHW")
    tiny = [data(rng, (int(rng.integers(0, 9)), int(rng.integers(1, 9)), 3), np.uint8) for _ in range(3000)]
    regs = [random_regions(rng, x.shape, [0, 1], int(rng.integers(0, 3))) for x in tiny]
    check(tiny, [0, 1], [r[0] for r in regs], [r[1] for r in regs], (9.0, 8.0, 7.0), "HWC", "HW", packed=True)


def test_one_uint8_sample_of_more_than_2_31_elements():
    import torch
    from dali_b200 import capi
    if os.environ.get("DALIB200_DRYRUN"):
        pytest.skip("6.5 GB of buffers; the host side of this launch is the other tests'")
    lib = capi.lib()
    h, w = 46400, 46400                                                    # 2 152 960 000 elements
    x = (torch.arange(h * w, dtype=torch.int64, device="cuda") % 251).to(torch.uint8).reshape(h, w)
    out = torch.full_like(x, 0xA5)
    a, s = [100.0, 46000.0, 40000.0, 7.0, 46399.0, 0.0], [300.0, 1000.0, 6400.0, 46393.0, 1.0, 46400.0]
    plan = C.c_void_p()
    capi.check(lib.dalib200ErasePlanCreate(C.byref(plan), 1))
    try:
        capi.check(lib.dalib200EraseSetup(plan, 0, 1, 2, (C.c_int64 * 2)(h, w), b"HW", b"HW", None, 0, (C.c_float * 6)(*a),
                                          (C.c_int64 * 1)(6), (C.c_float * 6)(*s), (C.c_int64 * 1)(6), 0, 0, 0, (C.c_float * 1)(42.0), 1))
        capi.check(lib.dalib200EraseLaunch(plan, (C.c_void_p * 1)(x.data_ptr()), (C.c_void_p * 1)(out.data_ptr()), capi.stream_handle()))
        torch.cuda.synchronize()
    finally:
        lib.dalib200ErasePlanDestroy(plan)
    want = x.clone()
    for (b, e) in er.boxes((h, w), [0, 1], a, s):
        want[b[0]:e[0], b[1]:e[1]] = 42
    assert torch.equal(out, want)


def test_every_byte_offset_and_batch_independence():
    rng = np.random.default_rng(6)
    for dt in (np.uint8, np.int16, np.float32, np.float64):
        x = data(rng, (37, 45, 3), dt)
        a, s = random_regions(rng, x.shape, [0, 1], 3)
        for o in range(0, 16, np.dtype(dt).itemsize):
            for p in (o, (o + 5 * np.dtype(dt).itemsize) % 16):
                check([x, x], [0, 1], [a, a], [s, s], (1.0, 2.0, 3.0), "HWC", "HW", in_offsets=[o, o],
                      out_offsets=[p, (p + 3 * x.itemsize) % 16])
    one = gh.synth_image(301, 455, 7)
    a1, s1 = random_regions(rng, one.shape, [0, 1], 5)
    (alone,) = capi_erase([one], [0, 1], [a1], [s1], (3.0,), "HWC", "HW")
    mixed = [data(rng, (3, 5, 3), np.uint8), one, np.zeros((0, 3, 3), np.uint8), rng.integers(0, 256, (640, 480, 3), dtype=np.uint8), one]
    regs = [random_regions(rng, x.shape, [0, 1], 4) for x in mixed]
    regs[1] = regs[4] = (a1, s1)
    inmix = capi_erase(mixed, [0, 1], [r[0] for r in regs], [r[1] for r in regs], (3.0,), "HWC", "HW", out_offsets=[1, 2, 3, 4, 5])
    assert alone.tobytes() == inmix[1].tobytes() == inmix[4].tobytes()


def test_refusals_name_the_problem():
    import nvidia.dali as dali
    from nvidia.dali import fn

    def run(xs, layout=None, **kw):
        @dali.pipeline_def(batch_size=len(xs), num_threads=1, device_id=0, prefetch_queue_depth=1)
        def pipe():
            return fn.erase(fn.external_source(source=lambda: xs, device="gpu", layout=layout), **kw)
        p = pipe()
        p.build()
        return p.run()
    x = [np.zeros((4, 5, 3), np.uint8)] * 2
    with pytest.raises(Exception, match="'X' is not an axis of the layout \"HWC\""):
        run(x, "HWC", axis_names="HX", anchor=[0, 0], shape=[1, 1])
    with pytest.raises(Exception, match="not a multiple of the 2 erased axes"):
        run(x, "HWC", anchor=[0, 0, 0], shape=[1, 1, 1])
    with pytest.raises(Exception, match="fill_value has 2 values, but the C axis of input 0 has 3 channels"):
        run(x, "HWC", anchor=[0, 0], shape=[1, 1], fill_value=[1, 2])
    with pytest.raises(Exception, match="shape value -1 is a negative extent"):
        run(x, "HWC", anchor=[0, 0], shape=[1, -1])
    (o,) = run([np.full((4, 5, 3), 10, np.uint8)] * 2, "HWC", anchor=[1, 1], shape=[2, 2], fill_value=[300.0])
    want = np.full((4, 5, 3), 10, np.uint8)
    want[1:3, 1:3] = 255
    assert np.array_equal(o.as_cpu()[0], want)
