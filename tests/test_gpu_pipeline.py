"""-m gpu tests through the public API (pipeline_def + fn.* + DALIGenericIterator): BASELINE configs C1 / C3 / C4 at test
sizes, compared with the oracle applied stage by stage.  Bit-exact except the STFT (stated tolerance)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import pyoracle as po  # noqa: E402

MEAN = [0.485 * 255, 0.456 * 255, 0.406 * 255]
STD = [0.229 * 255, 0.224 * 255, 0.225 * 255]


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _jpegs(n, h, w, seed0=0):
    import cv2
    import gpu_helpers as g
    out = []
    for i in range(n):
        ok, enc = cv2.imencode(".jpg", g.synth_image(h, w, seed0 + i), [cv2.IMWRITE_JPEG_QUALITY, 90])
        out.append(np.ascontiguousarray(enc.ravel()))
    return out


def test_c1_decode_resize_cmn_fp32():
    """BASELINE configs[0]: decoders.image + resize + crop_mirror_normalize, batch 8, 640x480 JPEG (GPU backends)."""
    from dali_b200 import fn, types, pipeline_def
    streams = _jpegs(8, 480, 640)
    mirror = np.array([0, 1, 0, 1, 1, 0, 0, 1], np.int32)

    @pipeline_def(batch_size=8, num_threads=2, device_id=0)
    def pipe():
        jpegs = fn.external_source(source=lambda i: streams, name="jpegs")
        mir = fn.external_source(source=lambda i: [np.array(m, np.int32) for m in mirror])
        img = fn.decoders.image(jpegs, device="mixed")
        img = fn.resize(img, resize_x=224, resize_y=224)
        return fn.crop_mirror_normalize(img, dtype=types.FLOAT, output_layout="CHW", crop=(224, 224), mean=MEAN, std=STD, mirror=mir)
    p = pipe()
    p.build()
    (out,) = p.run()
    got = out.as_cpu()
    assert out.layout() == "CHW" and out.shape()[0] == (3, 224, 224)
    mean, inv = po.cmn_norm_args(MEAN, STD)
    for i, s in enumerate(streams):
        want = po.cmn(po.resample(po.jpeg_decode(s.tobytes()), (224, 224)), (0, 0), (224, 224), bool(mirror[i]), mean, inv, np.float32, "CHW")
        assert np.array_equal(bits(got[i]), bits(want)), i
    # a second iteration reuses plans and buffers
    (out2,) = p.run()
    assert np.array_equal(bits(out2.as_cpu()[3]), bits(got[3]))


def test_c2_variant_resize_shorter_center_crop_fp16_iterator():
    """The classic ImageNet variant: resize_shorter=256 -> centre crop 224 -> fp16 CHW, through DALIGenericIterator."""
    import torch
    from dali_b200 import fn, types, pipeline_def
    from dali_b200.plugin.pytorch import DALIGenericIterator
    streams = _jpegs(4, 300, 400, 50) + _jpegs(2, 500, 333, 60)

    @pipeline_def(batch_size=6, num_threads=2, device_id=0)
    def pipe():
        jpegs = fn.external_source(source=lambda i: streams)
        img = fn.decoders.image(jpegs, device="mixed", output_type=types.RGB)
        img = fn.resize(img, resize_shorter=256)
        return fn.crop_mirror_normalize(img, dtype=types.FLOAT16, output_layout="CHW", crop=(224, 224), mean=MEAN, std=STD)
    it = DALIGenericIterator([pipe()], ["data"], size=12)
    batches = [next(it), next(it)]
    with pytest.raises(StopIteration):
        next(it)
    data = batches[0][0]["data"]
    assert isinstance(data, torch.Tensor) and data.dtype == torch.float16 and tuple(data.shape) == (6, 3, 224, 224) and data.is_cuda
    mean, inv = po.cmn_norm_args(MEAN, STD)
    got = data.cpu().numpy()
    for i, s in enumerate(streams):
        dec = po.jpeg_decode(s.tobytes())
        H, W = dec.shape[:2]
        sc = 256 / min(H, W)
        oh, ow = (256, int(round(W * sc))) if H < W else (int(round(H * sc)), 256)
        # subpixel_scale: the ROI is adjusted for the rounded size (resize_attr_base.h:97-113)
        fh, fw = H * sc, W * sc
        roi = None
        lo = [0.0, 0.0]; hi = [float(H), float(W)]
        for d, (real, frac, ext) in enumerate(((oh, fh, H), (ow, fw, W))):
            if real != np.float32(frac):
                adj = real / float(np.float32(abs(np.float32(frac))))
                c = 0.5 * lo[d] + 0.5 * hi[d]
                lo[d], hi[d] = float(np.float32(c + (lo[d] - c) * adj)), float(np.float32(c + (hi[d] - c) * adj))
        roi = ((lo[0], lo[1]), (hi[0], hi[1]))
        res = po.resample(dec, (oh, ow), (po.F_TRIANGULAR, 1, 0.0), (po.F_LINEAR, 0, 0.0), roi=roi)
        ay, ax = po.crop_anchor(0.5, oh, 224), po.crop_anchor(0.5, ow, 224)
        want = po.cmn(res, (ay, ax), (224, 224), False, mean, inv, np.float16, "CHW")
        assert np.array_equal(bits(got[i]), bits(want)), (i, H, W, oh, ow)


def test_c3_video_frames_warp_hsv_cmn():
    """BASELINE configs[2] at test size: FHWC sequences, warp_affine + hsv + crop_mirror_normalize(FCHW fp16);
    per-sequence matrix / hue / saturation / value / mirror as tensor arguments."""
    from dali_b200 import fn, types, pipeline_def
    rng = np.random.default_rng(71)
    nseq, F, H, W = 3, 4, 72, 300
    seqs = [rng.integers(0, 256, (F, H, W, 3)).astype(np.uint8) for _ in range(nseq)]
    mats, hues, sats, vals, mirs = [], [], [], [], []
    for _ in range(nseq):
        ang, s = np.deg2rad(rng.uniform(-10, 10)), rng.uniform(0.95, 1.05)
        c, si = np.cos(ang) * s, np.sin(ang) * s
        cx, cy = W / 2, H / 2
        mats.append(np.float32([[c, -si, cx - c * cx + si * cy], [si, c, cy - si * cx - c * cy]]))
        hues.append(np.float32(rng.uniform(-30, 30))); sats.append(np.float32(rng.uniform(0.7, 1.3))); vals.append(np.float32(rng.uniform(0.8, 1.2)))
        mirs.append(np.int32(rng.integers(0, 2)))

    @pipeline_def(batch_size=nseq, num_threads=2, device_id=0)
    def pipe():
        v = fn.external_source(source=lambda i: seqs, device="gpu", layout="FHWC")
        m = fn.external_source(source=lambda i: mats)
        h = fn.external_source(source=lambda i: hues)
        s = fn.external_source(source=lambda i: sats)
        va = fn.external_source(source=lambda i: vals)
        mi = fn.external_source(source=lambda i: mirs)
        x = fn.warp_affine(v, matrix=m, inverse_map=False, fill_value=0, interp_type=types.INTERP_LINEAR)
        x = fn.hsv(x, hue=h, saturation=s, value=va, dtype=types.UINT8)
        return fn.crop_mirror_normalize(x, mirror=mi, mean=MEAN, std=STD, dtype=types.FLOAT16, output_layout="FCHW")
    p = pipe()
    p.build()
    (out,) = p.run()
    assert out.layout() == "FCHW" and out.shape()[0] == (F, 3, H, W)
    got = out.as_cpu()
    mean, inv = po.cmn_norm_args(MEAN, STD)
    for i in range(nseq):
        Minv = po.affine_inv(mats[i])                       # inverse_map=False -> the operator inverts the matrix
        Mh, Th = po.color_twist_matrix(float(hues[i]), float(sats[i]), float(vals[i]))
        for f in range(F):
            w = po.warp_affine(seqs[i][f], Minv, None, 1, 0.0)
            hsv = po.linear_transform(w, Mh, Th)
            want = po.cmn(hsv, (0, 0), (H, W), bool(mirs[i]), mean, inv, np.float16, "CHW")
            assert np.array_equal(bits(got[i][f]), bits(want)), (i, f)


def test_c4_audio_spectrogram_mel():
    """BASELINE configs[3] at test size: spectrogram(nfft=1024) + mel_filter_bank(128) -- STFT by tolerance
    (2e-4 of the maximum), mel bit-exact given the GPU spectrogram."""
    from dali_b200 import fn, pipeline_def
    rng = np.random.default_rng(72)
    clips = []
    for n in (16000, 12345, 160000):
        t = np.arange(n) / 16000.0
        x = sum(rng.uniform(0.05, 0.3) * np.sin(2 * np.pi * rng.uniform(50, 7000) * t) for _ in range(5)) + 0.05 * rng.normal(0, 1, n)
        clips.append(np.clip(x, -1, 1).astype(np.float32))

    @pipeline_def(batch_size=3, num_threads=2, device_id=0)
    def pipe():
        a = fn.external_source(source=lambda i: clips, device="gpu")
        spec = fn.spectrogram(a, nfft=1024, window_length=1024, window_step=256, power=2)
        mel = fn.mel_filter_bank(spec, nfilter=128, sample_rate=16000.0, freq_high=8000.0)
        return spec, mel
    p = pipe()
    p.build()
    spec, mel = p.run()
    assert spec.layout() == "ft" and spec.shape()[2] == (513, 626) and mel.shape()[2] == (128, 626)
    gs, gm = spec.as_cpu(), mel.as_cpu()
    for i, c in enumerate(clips):
        want = po.spectrogram(c, nfft=1024, window_length=1024, window_step=256, power=2)
        assert np.abs(gs[i] - want).max() <= 2e-4 * want.max()
        assert np.array_equal(bits(gm[i]), bits(po.mel_filter_bank(gs[i], 128, 16000.0, 0.0, 8000.0, "slaney", True)))


def test_operator_errors_surface_with_operator_name():
    from dali_b200 import fn, pipeline_def, backend

    @pipeline_def(batch_size=2, num_threads=1, device_id=0)
    def pipe():
        j = fn.external_source(source=lambda i: [np.frombuffer(b"not a jpeg, really", np.uint8)] * 2)
        return fn.decoders.image(j, device="mixed")
    p = pipe()
    p.build()
    with pytest.raises(backend.BackendError, match="decoders__Image"):
        p.run()

    @pipeline_def(batch_size=2, num_threads=1, device_id=0)
    def oob():
        x = fn.external_source(source=lambda i: [np.zeros((10, 10, 3), np.uint8)] * 2, device="gpu", layout="HWC")
        return fn.crop_mirror_normalize(x, crop=(20, 20))
    q = oob()
    q.build()
    with pytest.raises(backend.BackendError, match="out of bounds"):
        q.run()


def test_decoder_crop_family_and_random_resized_crop():
    """fn.decoders.image_crop / image_random_crop / image_slice decode only the blocks under the window and must equal the crop of
    the full decode; the random windows are the library's generator's for the same seed (and the reference's, oracle/_ref, where
    present); fn.random_resized_crop = resize with the window as ROI (random_resized_crop.h:112-120)."""
    import gpu_helpers as g
    from dali_b200 import fn, types, pipeline_def
    streams = _jpegs(3, 300, 400, 70) + _jpegs(2, 333, 251, 80)
    n = len(streams)
    anchors = [np.array([0.1 + 0.05 * i, 0.2], np.float32) for i in range(n)]      # (x, y), normalised ("WH" axes)
    shapes = [np.array([0.5, 0.6 - 0.05 * i], np.float32) for i in range(n)]

    @pipeline_def(batch_size=n, num_threads=2, device_id=0)
    def pipe():
        jpegs = fn.external_source(source=lambda i: streams)
        anc = fn.external_source(source=lambda i: anchors)
        shp = fn.external_source(source=lambda i: shapes)
        a = fn.decoders.image_crop(jpegs, device="mixed", crop=(160, 200), crop_pos_x=0.3, crop_pos_y=0.8)
        b = fn.decoders.image_random_crop(jpegs, device="mixed", seed=1234, random_area=[0.1, 0.9])
        c = fn.decoders.image_slice(jpegs, anc, shp, device="mixed")
        d = fn.decoders.image_slice(jpegs, device="mixed", start=[16, 30], shape=[100, 64], axes=[0, 1])
        e = fn.random_resized_crop(fn.decoders.image(jpegs, device="mixed"), size=[96, 128], seed=77)
        return a, b, c, d, e
    p = pipe()
    p.build()
    for it in range(2):
        a, b, c, d, e = [o.as_cpu() for o in p.run()]
        for i, s in enumerate(streams):
            full = po.jpeg_decode(s.tobytes())
            H, W = full.shape[:2]
            y0, x0 = po.crop_anchor(0.8, H, 160), po.crop_anchor(0.3, W, 200)
            assert np.array_equal(a[i], full[y0:y0 + 160, x0:x0 + 200]), (it, i)
            wy, wx, wh, ww = g.random_crop_window(1234, i, H, W, area=(0.1, 0.9), ncalls=it + 1)
            assert b[i].shape == (wh, ww, 3) and np.array_equal(b[i], full[wy:wy + wh, wx:wx + ww]), (it, i)
            ry, rx, rh, rw = g.random_crop_window(77, i, H, W, ncalls=it + 1)
            roi = ((float(ry), float(rx)), (float(ry + rh), float(rx + rw)))
            assert np.array_equal(e[i], po.resample(full, (96, 128), roi=roi)), (it, i)
            if po.have_ref():
                assert po.ref_random_crop(1234, i, H, W, area=(0.1, 0.9), ncalls=it + 1)[it] == (wy, wx, wh, ww), (it, i)
                assert po.ref_random_crop(77, i, H, W, ncalls=it + 1)[it] == (ry, rx, rh, rw), (it, i)
                assert np.array_equal(e[i], po.ref_resample(full, (96, 128), roi=roi)), (it, i)
            ax, ay = float(anchors[i][0]), float(anchors[i][1])
            sx, sy = float(shapes[i][0]), float(shapes[i][1])
            rnd = lambda v: int(np.floor(v + 0.5))                   # std::llround: half away from zero (slice_attr.h:330-331)
            bx, ex = rnd(ax * W), rnd((ax + sx) * W)
            by, ey = rnd(ay * H), rnd((ay + sy) * H)
            assert np.array_equal(c[i], full[by:ey, bx:ex]), (it, i)
            assert np.array_equal(d[i], full[16:116, 30:94]), (it, i)


def test_decoder_resize_fusion_in_the_executor(monkeypatch):
    """decoders.image* -> resize with no other consumer of the decoded image (opt-in, DALIB200_FUSE_DECODE_RESIZE=1): the executor
    links the two operators, the Resize reads
    the decoder's planes (kernel `resample_planar`) for the samples that qualify and the usual path for the rest (grayscale, 4:4:4);
    results equal decode-then-resize / crop-then-resize on the oracle, and the unfused pipeline (image also returned) bit for bit."""
    import cv2
    import gpu_helpers as g
    from dali_b200 import capi, fn, pipeline_def
    monkeypatch.setenv("DALIB200_FUSE_DECODE_RESIZE", "1")
    streams = _jpegs(3, 480, 640, 90)
    ok, enc = cv2.imencode(".jpg", g.synth_image(300, 400, 95), [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444])
    streams.append(np.ascontiguousarray(enc.ravel()))
    ok, enc = cv2.imencode(".jpg", g.synth_image(300, 400, 96)[..., 0], [cv2.IMWRITE_JPEG_QUALITY, 90])
    streams.append(np.ascontiguousarray(enc.ravel()))
    n = len(streams)

    def build(keep_image):
        @pipeline_def(batch_size=n, num_threads=2, device_id=0)
        def pipe():
            jpegs = fn.external_source(source=lambda i: streams)
            img = fn.decoders.image(jpegs, device="mixed")
            a = fn.resize(img, resize_x=160, resize_y=120)
            crop = fn.decoders.image_random_crop(jpegs, device="mixed", seed=5)
            b = fn.resize(crop, size=[64, 64])
            return (a, b, img) if keep_image else (a, b)
        p = pipe()
        p.build()
        return p
    capi.profiling(True); capi.profiling_collect()
    fused = [o.as_cpu() for o in build(False).run()]
    names = {k for k, _ in capi.profiling_collect()}
    plain = [o.as_cpu() for o in build(True).run()]          # `img` is a pipeline output there: the first pair is not fused
    capi.profiling(False)
    assert "resample_planar" in names
    for i, s in enumerate(streams):
        full = po.jpeg_decode(s.tobytes())
        assert np.array_equal(fused[0][i], po.resample(full, (120, 160))), i
        assert np.array_equal(fused[0][i], plain[0][i]) and np.array_equal(fused[1][i], plain[1][i]), i
        assert np.array_equal(plain[2][i], full), i
        H, W = full.shape[:2]
        wy, wx, wh, ww = g.random_crop_window(5, i, H, W)
        assert np.array_equal(fused[1][i], po.resample(np.ascontiguousarray(full[wy:wy + wh, wx:wx + ww]), (64, 64))), i
        if po.have_ref():
            assert po.ref_random_crop(5, i, H, W)[0] == (wy, wx, wh, ww), i
