"""-m gpu edge cases of the per-pixel kernels that the operator tests do not reach, each against a plain reference:
  * multiply_add_kernel (fn.brightness_contrast): sizes around the 8192-element work items and the 4-element quads, a batch whose
    grid loops, unaligned pointers (the scalar branch), exact halves, saturation, the default contrast_center, float output,
    sequences -- against the float32 form of tests/pointwise_ref.py;
  * jpeg_post_kernel (orientation + ROI + output type + dtype): one plan holding every source kind, all EXIF orientations, ROIs
    touching each edge, 1-pixel windows and a 1x1 image, tiny samples between large ones -- against the u8 RGB / GRAY decode of the
    same streams, oriented and cut in numpy, then converted by tests/pointwise_ref.py;
  * cmn_generic_kernel: 1- and 4-channel inputs, padding channels, mirror, out-of-bounds windows, and samples of the fast path,
    the generic path and empty crops interleaved in one batch -- against the oracle (oracle/pyoracle.py cmn);
  * window_copy_kernel (flip / crop / slice): 1- and 4-channel images and sequences, padding with per-channel fill -- against numpy."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
import pointwise_ref as pr  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


# ------------------------------------------------------------------------------------------------------------- multiply-add
def _multiply_add(ins, outs, args, out_float):
    """dalib200MultiplyAddSetup / GenericLaunch over device tensors; args[i] = (brightness, shift, contrast, center) of sample i,
    turned into the kernel's multiplier and addend as BrightnessContrast does"""
    import torch
    n = len(ins)
    ma = [pr.brightness_contrast_args(*a, out_float=out_float) for a in args]
    plan = capi.Plan("Generic", max(n, 1))
    capi.check(capi.lib().dalib200MultiplyAddSetup(plan.handle, n, (C.c_int64 * n)(*[t.numel() for t in ins]),
                                                   (C.c_float * n)(*[float(m) for m, _ in ma]), (C.c_float * n)(*[float(a) for _, a in ma]),
                                                   capi.FLOAT if out_float else capi.UINT8))
    capi.check(capi.lib().dalib200GenericLaunch(plan.handle, capi.ptr_array(ins), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs]


def _assert_bc(got, x, a, out_float, what):
    want = pr.brightness_contrast(x, *a, out_float=out_float)
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, got.dtype)
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (what, a)


VOLUMES = (0, 1, 3, 4, 5, 8191, 8192, 8193, 3 * 8192 + 5, 1080 * 1920 * 3)


def test_multiply_add_sizes_and_alignments():
    """Work-item boundaries and the scalar tail behind the last full quad, first with every sample in an allocation of its own (the
    vector branch), then with inputs at byte offsets 1..3 and outputs at offsets that break the vector alignment (u8: 1..3 bytes,
    float: 4-byte but not 16-byte aligned) inside one allocation each (the scalar branch)."""
    import torch
    rng = np.random.default_rng(1)
    xs = [rng.integers(0, 256, v, dtype=np.uint8) for v in VOLUMES]
    args = [(float(rng.uniform(0.2, 2.5)), float(rng.uniform(-0.3, 0.3)), float(rng.uniform(0.2, 2.0)), float(rng.uniform(0, 255)))
            for _ in VOLUMES]
    for out_float in (False, True):
        tdt = torch.float32 if out_float else torch.uint8
        ins = [torch.from_numpy(x).cuda() for x in xs]
        outs = [torch.empty(x.size, dtype=tdt, device="cuda") for x in xs]
        for k, o in enumerate(_multiply_add(ins, outs, args, out_float)):
            _assert_bc(o, xs[k], args[k], out_float, ("aligned", VOLUMES[k], out_float))
        bases = np.concatenate([[0], np.cumsum([(v + 16 + 15) // 16 * 16 for v in VOLUMES])])      # 16-aligned slots, 16 spare
        shift = [1 + k % 3 for k in range(len(VOLUMES))]
        host = np.zeros(int(bases[-1]), np.uint8)
        for k, x in enumerate(xs):
            host[bases[k] + shift[k]:bases[k] + shift[k] + x.size] = x
        whole_in = torch.from_numpy(host).cuda()
        whole_out = torch.empty(int(bases[-1]), dtype=tdt, device="cuda")
        ins = [whole_in[int(bases[k]) + shift[k]:int(bases[k]) + shift[k] + v] for k, v in enumerate(VOLUMES)]
        outs = [whole_out[int(bases[k]) + shift[k]:int(bases[k]) + shift[k] + v] for k, v in enumerate(VOLUMES)]
        for k, o in enumerate(_multiply_add(ins, outs, args, out_float)):
            _assert_bc(o, xs[k], args[k], out_float, ("unaligned", VOLUMES[k], out_float))


def test_multiply_add_batch_of_many_samples():
    """3000 samples packed back to back (any alignment) with their own arguments: more work items than the grid has CTAs on an H100
    (132 SMs x 16), so the grid loops and every CTA searches the descriptor list more than once."""
    import torch
    rng = np.random.default_rng(2)
    vols = rng.integers(0, 12000, 3000)
    vols[::97] = 0
    assert int(np.sum((vols + 8191) // 8192)) > 132 * 16
    offs = np.concatenate([[0], np.cumsum(vols)])
    host = rng.integers(0, 256, int(offs[-1]), dtype=np.uint8)
    args = [(float(b), float(s), float(c), 128.0) for b, s, c in zip(rng.uniform(0.3, 2.0, vols.size), rng.uniform(-0.2, 0.2, vols.size),
                                                                      rng.uniform(0.3, 1.8, vols.size))]
    whole_in = torch.from_numpy(host).cuda()
    whole_out = torch.empty(host.size, dtype=torch.uint8, device="cuda")
    sl = [(int(offs[k]), int(offs[k + 1])) for k in range(vols.size)]
    got = _multiply_add([whole_in[a:b] for a, b in sl], [whole_out[a:b] for a, b in sl], args, False)
    for k, (a, b) in enumerate(sl):
        _assert_bc(got[k], host[a:b], args[k], False, ("sample", k))


def test_multiply_add_halves_saturation_and_float_range():
    """brightness 0.5, contrast 1: odd inputs land exactly on k + 0.5 and must round AWAY from zero (to k + 1); brightness 3 with
    shift -1 / +1 saturates at 0 and at 255; float output is in * mul + add with shift in units of 1, not rescaled by 1 / 255."""
    import torch
    x = np.arange(256, dtype=np.uint8)
    args = [(0.5, 0.0, 1.0, 128.0), (3.0, -1.0, 1.0, 128.0), (3.0, 1.0, 1.0, 128.0), (1.2, 0.1, 0.9, 100.0)]
    ins = [torch.from_numpy(x).cuda() for _ in args]
    got = _multiply_add(ins, [torch.empty(256, dtype=torch.uint8, device="cuda") for _ in args], args, False)
    for k, a in enumerate(args):
        _assert_bc(got[k], x, a, False, a)
    assert np.array_equal(got[0].astype(np.int64), (x.astype(np.int64) + 1) // 2)
    assert np.array_equal(got[1], np.clip(3 * x.astype(np.int64) - 255, 0, 255))
    assert np.array_equal(got[2], np.clip(3 * x.astype(np.int64) + 255, 0, 255))
    got = _multiply_add(ins, [torch.empty(256, dtype=torch.float32, device="cuda") for _ in args], args, True)
    for k, a in enumerate(args):
        _assert_bc(got[k], x, a, True, a)
        pr.assert_f32_close(got[k], pr.brightness_contrast_f64(x, *a, out_float=True), 2e-4, a)


def test_brightness_contrast_sequences_and_contrast_center():
    """fn.brightness_contrast on FHWC sequences (frames of different sizes per sample), u8 and float, with the default contrast_center
    (128 for u8 input, not 127.5) and an explicit one."""
    from dali_b200 import fn, pipeline_def, types
    rng = np.random.default_rng(4)
    seqs = [rng.integers(0, 256, (3, 37, 53, 3), dtype=np.uint8), rng.integers(0, 256, (5, 16, 9, 3), dtype=np.uint8)]

    @pipeline_def(batch_size=len(seqs), num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: seqs, device="gpu", layout="FHWC")
        return (fn.brightness_contrast(x, brightness=1.0, contrast=0.6),
                fn.brightness_contrast(x, brightness=0.9, contrast=1.4, brightness_shift=-0.05, contrast_center=37.5),
                fn.brightness_contrast(x, brightness=1.1, contrast=0.6, dtype=types.FLOAT))
    p = pipe()
    p.build()
    a, b, c = [o.as_cpu() for o in p.run()]
    for i, s in enumerate(seqs):
        _assert_bc(np.asarray(a[i]), s, (1.0, 0.0, 0.6, 128.0), False, ("default center", i))
        _assert_bc(np.asarray(b[i]), s, (0.9, -0.05, 1.4, 37.5), False, ("center 37.5", i))
        _assert_bc(np.asarray(c[i]), s, (1.1, 0.0, 0.6, 128.0), True, ("float", i))


# ------------------------------------------------------------------------------------------------------------- decoder post pass
def _jpg(img, *params):
    import cv2
    ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90, *params])
    assert ok
    return enc.tobytes()


def _roi(kind, OH, OW):
    """(x0, y0, x1, y1) in displayed coordinates, or None"""
    return {"full": None, "left": (0, 5, OW // 2, OH - 3), "top": (4, 0, OW - 2, OH // 2), "right": (OW // 3, 2, OW, OH - 1),
            "bottom": (1, OH // 3, OW - 5, OH), "col1": (OW // 2, 0, OW // 2 + 1, OH), "row1": (0, OH // 2, OW, OH // 2 + 1),
            "corner": (OW - 1, OH - 1, OW, OH)}[kind]


def _post_samples():
    """[(stream, orientation, roi kind)]: every source kind of the post pass, every orientation, tiny samples between large ones"""
    import cv2
    import gpu_helpers as g
    import png_streams as ps
    import tiff_streams as ts
    import webp_streams as ws
    from jpeg_cmyk_streams import photoshop_ycck
    kinds = ["full", "left", "top", "right", "bottom", "col1", "row1", "corner"]
    j420 = _jpg(g.synth_image(203, 310, 1), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420)
    big = _jpg(g.synth_image(1080, 1920, 2), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420)
    j444 = _jpg(g.synth_image(97, 131, 3), cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444)
    jgray = _jpg(g.synth_image(120, 200, 4)[..., 0])
    jprog = _jpg(g.synth_image(160, 96, 5), cv2.IMWRITE_JPEG_PROGRESSIVE, 1)
    tiny = _jpg(g.synth_image(1, 1, 6))
    ycck = photoshop_ycck(90, 130, 7)
    jo = po.with_exif_orientation
    png = lambda o: ps.encode(ps.samples(50, 61, 4, 16, 8), 4, 16, filters="mixed", exif=o)            # gray + alpha, 16 bits
    tif = lambda o: ts.encode(ts.samples(64, 80, 3, 8, 9), 2, 8, 5, 2, orientation=o)
    webp = lambda o: ws.pil_webp(ws.image(75, 120, 10)[..., ::-1].copy(), quality=70, exif=ws.exif_orientation(o))
    s = [(jo(big, 1), 1, "full"), (jo(tiny, 1), 1, "full")]
    s += [(jo(j420, o), o, kinds[o - 1]) for o in range(1, 9)]
    s += [(jo(tiny, 6), 6, "full"), (jo(j444, 3), 3, "right"), (jo(jgray, 6), 6, "bottom"), (jo(big, 8), 8, "right"),
          (jo(j444, 5), 5, "col1"), (jo(jgray, 2), 2, "left"), (jo(jprog, 8), 8, "top"), (jo(tiny, 3), 3, "corner"),
          (jo(jprog, 7), 7, "full"), (jo(ycck, 4), 4, "row1"), (png(7), 7, "left"), (png(1), 1, "full"), (tif(5), 5, "bottom"),
          (tif(1), 1, "corner"), (webp(6), 6, "right"), (webp(1), 1, "full")]
    return s


def test_post_pass_every_source_orientation_and_window():
    """YCbCr u8 / float, GRAY float and BGR float of one plan holding 4:2:0 (fast colour) / 4:4:4 / grayscale / progressive / YCCK
    JPEG, 16-bit gray + alpha PNG, TIFF and WebP samples with orientations 1..8 and windows touching each edge.  The reference: the u8
    RGB (GRAY) decode of the same streams without orientation and window, oriented and cut in numpy, converted by the float32 form
    (bit-exact) and the float64 form (float: within 1e-6).  A grayscale stream decoded to YCbCr is converted from replicated RGB."""
    import gpu_helpers as g
    samples = _post_samples()
    streams = [s for s, _, _ in samples]
    raw = {}
    for ot in (capi.RGB, capi.GRAY):
        raw[ot], status = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)
        assert status == [0] * len(streams)
    rois, wants = [], {}
    for i, (_, o, kind) in enumerate(samples):
        OH, OW = po.exif_transform(raw[capi.RGB][i], o).shape[:2]
        rois.append(_roi(kind, OH, OW))
    for ot, dt, fl in ((capi.YCbCr, capi.UINT8, False), (capi.YCbCr, capi.FLOAT, True), (capi.GRAY, capi.FLOAT, True),
                       (capi.BGR, capi.FLOAT, True)):
        outs, status = g.jpeg_decode_ex(streams, output_type=ot, dtype=dt, adjust_orientation=True, rois=rois)
        assert status == [0] * len(streams)
        for i, (_, o, kind) in enumerate(samples):
            src = po.exif_transform(raw[capi.GRAY if ot == capi.GRAY else capi.RGB][i], o)
            r = rois[i] or (0, 0, src.shape[1], src.shape[0])
            src = np.ascontiguousarray(src[r[1]:r[3], r[0]:r[2]])
            pr.check_decoder_output(outs[i], src, ot, fl, (i, o, kind, ot, dt))


# ------------------------------------------------------------------------------------------------------------- CMN generic path
def test_cmn_generic_path_any_channel_count():
    """1-, 3- and 4-channel inputs in one batch (padded to 4 output channels) and 1-channel batches without padding, float and fp16,
    CHW and HWC, mirrored and out-of-bounds windows.  In CHW the 3-channel windows inside their image take the fast path, and
    zero-area crops sit between them and the generic samples, so that neighbours share first_unit / first_elem."""
    import gpu_helpers as g
    rng = np.random.default_rng(5)
    mean = np.array([101.5, 17.25, 200.0, 64.0], np.float32)
    inv = np.array([1 / 57.0, 1 / 3.5, 1 / 110.0, 1 / 16.0], np.float32)
    fill = [-1.5, 2.25, 300.0, 0.125]
    im = lambda h, w, c: rng.integers(0, 256, (h, w, c), dtype=np.uint8)
    # (image, anchor, crop, mirror)
    mixed = [(im(40, 50, 3), (3, 4), (30, 40), 0), (im(33, 21, 1), (2, 1), (25, 17), 1), (im(20, 20, 3), (0, 0), (0, 5), 0),
             (im(17, 29, 4), (-3, 5), (22, 30), 1), (im(64, 300, 3), (5, 10), (50, 260), 1), (im(9, 7, 3), (0, 0), (0, 0), 0),
             (im(25, 31, 3), (10, -4), (20, 12), 0), (im(12, 13, 1), (0, 0), (12, 13), 0), (im(8, 8, 4), (0, 0), (0, 3), 0),
             (im(31, 45, 4), (1, 2), (29, 40), 0), (im(16, 130, 3), (0, 0), (16, 130), 0)]
    single = [(im(19, 23, 1), (0, 0), (19, 23), 0), (im(40, 9, 1), (-2, -1), (43, 12), 1), (im(5, 70, 1), (1, 3), (3, 60), 1)]
    for batch, out_channels in ((mixed, 4), (single, 1), (single, 2)):
        imgs = [b[0] for b in batch]
        for dt in (np.float32, np.float16):
            for layout in ("CHW", "HWC"):
                got = g.cmn(imgs, [b[1] for b in batch], [b[2] for b in batch], [b[3] for b in batch], mean, inv, dt, layout,
                            out_channels, fill)
                for k, (img, anchor, crop, mirror) in enumerate(batch):
                    want = po.cmn(img, anchor, crop, bool(mirror), mean, inv, dt, layout, out_channels, fill[:out_channels])
                    assert got[k].shape == want.shape, (k, layout, dt, got[k].shape, want.shape)
                    bits = np.uint32 if dt == np.float32 else np.uint16
                    assert np.array_equal(got[k].view(bits), want.view(bits)), (k, img.shape, layout, np.dtype(dt).name, out_channels)


# ------------------------------------------------------------------------------------------------------------- window copy
def test_flip_crop_slice_other_channel_counts_and_sequences():
    """fn.flip, fn.crop (padded, per-channel fill) and fn.slice (padded) on 1- and 4-channel images and on FHWC sequences, against
    numpy indexing.  Channel k of the fill is fill_values[min(k, 3)]."""
    from dali_b200 import fn, pipeline_def
    rng = np.random.default_rng(6)
    fillv = [7, 8, 9, 10]
    batches = [([rng.integers(0, 256, (31, 45, 1), dtype=np.uint8), rng.integers(0, 256, (17, 9, 1), dtype=np.uint8)], "HWC"),
               ([rng.integers(0, 256, (31, 45, 4), dtype=np.uint8), rng.integers(0, 256, (17, 9, 4), dtype=np.uint8)], "HWC"),
               ([rng.integers(0, 256, (3, 21, 26, 4), dtype=np.uint8), rng.integers(0, 256, (2, 11, 7, 3), dtype=np.uint8)], "FHWC")]
    for data, layout in batches:
        @pipeline_def(batch_size=len(data), num_threads=1, device_id=0)
        def pipe():
            x = fn.external_source(source=lambda i: data, device="gpu", layout=layout)
            return (fn.flip(x, horizontal=1, vertical=1), fn.flip(x, horizontal=0, vertical=1),
                    fn.crop(x, crop=(40, 50), out_of_bounds_policy="pad", fill_values=fillv),
                    fn.slice(x, start=[-2, 3], end=[15, 60], axis_names="HW", out_of_bounds_policy="pad", fill_values=fillv))
        p = pipe()
        p.build()
        a, b, c, d = [o.as_cpu() for o in p.run()]
        for i, x in enumerate(data):
            H, W, Cn = x.shape[-3:]
            fill = np.array([fillv[min(k, 3)] for k in range(Cn)], np.uint8)
            assert np.array_equal(np.asarray(a[i]), x[..., ::-1, ::-1, :]), (layout, i)
            assert np.array_equal(np.asarray(b[i]), x[..., ::-1, :, :]), (layout, i)
            y0, x0 = po.crop_anchor(0.5, H, 40), po.crop_anchor(0.5, W, 50)
            want = np.empty(x.shape[:-3] + (40, 50, Cn), np.uint8)
            want[...] = fill
            want[..., -y0:-y0 + H, -x0:-x0 + W, :] = x
            assert np.array_equal(np.asarray(c[i]), want), (layout, i)
            want = np.empty(x.shape[:-3] + (17, 57, Cn), np.uint8)
            want[...] = fill
            want[..., 2:2 + min(H, 15), :max(0, min(W, 60) - 3), :] = x[..., :min(H, 15), 3:60, :]
            assert np.array_equal(np.asarray(d[i]), want), (layout, i)
