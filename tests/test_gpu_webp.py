"""-m gpu tests of lossy WebP streams in the image decoder: the corpus of tests/webp_streams.py in RGB, BGR and GRAY against
cv2.imdecode, YCbCr and float against the post pass of cv2's decode, regions of interest of the C-ABI and the crop operators,
orientations, a batch mixing every JPEG path, PNG, TIFF and WebP samples, each corruption class, the failed sample named by the
pipeline, plan reuse, and fn.readers.file over a directory of .webp files."""
import cv2
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
import png_streams as ps  # noqa: E402
import png_oracle as pngo  # noqa: E402
import tiff_oracle as to  # noqa: E402
import tiff_streams as ts  # noqa: E402
import webp_streams as ws  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

NO = cv2.IMREAD_IGNORE_ORIENTATION


@pytest.fixture(scope="module")
def corpus():
    c = ws.corpus(big=True)
    streams = [s for _, s in c]
    return streams, [ws.decode(s, cv2.IMREAD_COLOR | NO)[..., ::-1] for s in streams], \
        [ws.decode(s, cv2.IMREAD_GRAYSCALE | NO) for s in streams], [n for n, _ in c]


def test_corpus_rgb_bgr_gray(corpus):
    import gpu_helpers as g
    streams, rgbs, grays, names = corpus
    for ot in (capi.RGB, capi.BGR, capi.GRAY):
        outs, status = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)
        assert status == [0] * len(streams)
        for i, o in enumerate(outs):
            w = rgbs[i][..., ::-1] if ot == capi.BGR else grays[i][..., None] if ot == capi.GRAY else rgbs[i]
            assert np.array_equal(o, w), (names[i], ot)


def test_corpus_ycbcr_and_float(corpus):
    """YCbCr and float are the post pass over the RGB (GRAY) decode, as for JPEG, PNG and TIFF"""
    import gpu_helpers as g
    streams, rgbs, grays, names = corpus
    ref = po.have_ref()
    for ot, it in ((capi.RGB, po.IT_RGB), (capi.BGR, po.IT_BGR), (capi.YCbCr, po.IT_YCBCR), (capi.GRAY, po.IT_GRAY)):
        for dt, fl in ((capi.UINT8, False), (capi.FLOAT, True)):
            outs, status = g.jpeg_decode_ex(streams, output_type=ot, dtype=dt, adjust_orientation=False)
            assert status == [0] * len(streams)
            for i, o in enumerate(outs):
                src = grays[i][..., None] if ot == capi.GRAY else rgbs[i]
                if ref:
                    w = po.ref_decoder_convert(src, it, fl)
                elif ot == capi.YCbCr:
                    assert o.shape == src.shape
                    continue
                else:
                    w = np.ascontiguousarray(src[..., ::-1]) if ot == capi.BGR else src
                    if fl:
                        w = w.astype(np.float32) * np.float32(1.0 / 255)
                assert np.array_equal(o, w), (names[i], ot, dt)


def _layouts():
    return [ws.cv2_webp(ws.image(97, 131, 1), 90), ws.cv2_webp(ws.image(64, 80, 2, noise=30.0), 40),
            ws.libwebp_encode(ws.image(75, 120, 3), 70.0, partitions=3, method=2, filter_type=0),
            ws.cv2_webp(ws.image(203, 310, 4), 75)]


def test_roi_windows_equal_crops_of_the_full_decode():
    import gpu_helpers as g
    streams = _layouts()
    rng = np.random.default_rng(8)
    for ot in (capi.RGB, capi.GRAY):
        full = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)[0]
        for i, s in enumerate(streams):
            w = ws.decode(s, cv2.IMREAD_GRAYSCALE)[..., None] if ot == capi.GRAY else ws.decode(s)[..., ::-1]
            assert np.array_equal(full[i], w), (ot, i)
        for rep in range(4):
            rois = []
            for f in full:
                H, W = f.shape[:2]
                x0, y0 = int(rng.integers(0, W - 1)), int(rng.integers(0, H - 1))
                rois.append((x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1))))
            outs, status = g.jpeg_decode_ex(streams, output_type=ot, rois=rois, adjust_orientation=False)
            assert status == [0] * len(streams)
            for i, r in enumerate(rois):
                assert np.array_equal(outs[i], full[i][r[1]:r[3], r[0]:r[2]]), (ot, rep, i, r)


def test_crop_operators_on_webp():
    from dali_b200 import fn, pipeline_def
    streams = [np.frombuffer(s, np.uint8) for s in _layouts()[:3]]
    full = [ws.decode(s.tobytes())[..., ::-1] for s in streams]

    @pipeline_def(batch_size=len(streams), num_threads=1, device_id=0, prefetch_queue_depth=1, seed=5)
    def pipe():
        enc = fn.external_source(source=lambda i: streams)
        a = fn.decoders.image_crop(enc, device="mixed", crop=(40, 50), crop_pos_x=0.3, crop_pos_y=0.6)
        b = fn.decoders.image_random_crop(enc, device="mixed", seed=1234, random_area=[0.1, 0.9])
        d = fn.decoders.image_slice(enc, device="mixed", start=[16, 30], shape=[30, 25], axes=[0, 1])
        e = fn.decoders.image(enc, device="mixed")
        return a, b, d, e
    p = pipe()
    p.build()
    res = [o.as_cpu() for o in p.run()]
    a, b, d, e = [[np.asarray(r[i]) for i in range(len(streams))] for r in res]
    for i, f in enumerate(full):
        H, W = f.shape[:2]
        assert np.array_equal(e[i], f), i
        y0, x0 = po.crop_anchor(0.6, H, 40), po.crop_anchor(0.3, W, 50)
        assert np.array_equal(a[i], f[y0:y0 + 40, x0:x0 + 50]), i
        assert np.array_equal(d[i], f[16:46, 30:55]), i
        h, w = b[i].shape[:2]
        assert any(np.array_equal(f[y:y + h, x:x + w], b[i]) for y in range(H - h + 1) for x in range(W - w + 1)), i


def test_orientations():
    """the EXIF orientation of a VP8X stream is applied, as cv2 applies it"""
    import gpu_helpers as g
    img = ws.image(37, 53, 70)[..., ::-1]
    streams = [ws.pil_webp(img, quality=70, exif=ws.exif_orientation(o)) for o in range(1, 9)]
    outs, status = g.jpeg_decode_ex(streams, adjust_orientation=True)
    assert status == [0] * 8
    for o in range(1, 9):
        assert np.array_equal(outs[o - 1], ws.decode(streams[o - 1])[..., ::-1]), o


def test_mixed_batch():
    """baseline, progressive, YCCK JPEG, PNG, TIFF and WebP samples in one batch: every JPEG sample equals its decode in a JPEG-only
    batch"""
    import gpu_helpers as g
    from jpeg_cmyk_streams import photoshop_ycck
    jpegs = [cv2.imencode(".jpg", g.synth_image(300, 420, 1))[1].tobytes(),
             cv2.imencode(".jpg", g.synth_image(120, 160, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(), photoshop_ycck(97, 131, 3)]
    png = ps.encode(ps.samples(40, 50, 2, 8, 80), 2, 8, filters="mixed")
    tif = cv2.imencode(".tiff", g.synth_image(240, 320, 4))[1].tobytes()
    webps = _layouts()[:3]
    for ot in (capi.RGB, capi.GRAY):
        solo = g.jpeg_decode(jpegs, output_type=ot)[0]
        streams = [webps[0], jpegs[0], png, webps[1], tif, jpegs[1], jpegs[2], webps[2]]
        outs, status = g.jpeg_decode(streams, output_type=ot)
        assert status == [0] * len(streams)
        for o, k in zip([outs[1], outs[5], outs[6]], range(3)):
            assert np.array_equal(o, solo[k]), (ot, k)
        pr = pngo.decode(png)
        assert np.array_equal(outs[2], pr[1][..., None] if ot == capi.GRAY else pr[0])
        tr = to.decode(tif)
        assert np.array_equal(outs[4], tr[1][..., None] if ot == capi.GRAY else tr[0])
        for o, s in zip([outs[0], outs[3], outs[7]], webps):
            w = ws.decode(s, cv2.IMREAD_GRAYSCALE)[..., None] if ot == capi.GRAY else ws.decode(s)[..., ::-1]
            assert np.array_equal(o, w), ot


def test_each_corruption_class():
    """bad data on the device sets the sample's status; a malformed, lossless or animated container fails plan set-up"""
    import gpu_helpers as g
    good = ws.cv2_webp(ws.image(20, 30, 90), 80)
    for name, s in ws.data_corrupt():
        outs, status = g.jpeg_decode([good, s, good])
        assert status == [0, 1, 0], name
        assert np.array_equal(outs[0], ws.decode(good)[..., ::-1]) and np.array_equal(outs[2], outs[0]), name
    for name, s, _ in ws.plan_corrupt():
        with pytest.raises(Exception, match="sample 1"):
            g.jpeg_decode([good, s])
    outs, status = g.jpeg_decode([ws.alph_corrupt()])          # the ALPH deviation: the colour decodes
    assert status == [0]


def test_pipeline_reports_the_failed_sample():
    from dali_b200 import fn, pipeline_def
    good = ws.cv2_webp(ws.image(20, 30, 91), 80)
    bad = dict(ws.data_corrupt())["token_partition_cut"]
    streams = [np.frombuffer(s, np.uint8) for s in (good, bad)]

    @pipeline_def(batch_size=2, num_threads=1, device_id=0, prefetch_queue_depth=1)
    def pipe():
        return fn.decoders.image(fn.external_source(source=lambda i: streams), device="mixed")
    p = pipe()
    p.build()
    try:
        p.run()
        err = ""
    except Exception as e:                    # noqa: BLE001
        err = str(e)
    assert "Failed to decode sample #1" in err, err


def test_plan_reuse_with_growing_webp_sizes():
    import gpu_helpers as g
    plan = capi.Plan("Jpeg", 3)
    for k, (h, w) in enumerate([(8, 8), (120, 160), (17, 400), (480, 640), (33, 47)]):
        streams = [ws.cv2_webp(ws.image(h + j, w, 100 + k), 50 + 20 * j) for j in range(3)]
        outs, status = g.jpeg_decode(streams, plan=plan)
        assert status == [0, 0, 0]
        for s, o in zip(streams, outs):
            assert np.array_equal(o, ws.decode(s)[..., ::-1]), (h, w)


def test_file_reader_over_webp_files(tmp_path):
    """fn.readers.file over a directory of .webp files (and a WebP named .JPEG) through decoders.image"""
    from dali_b200 import fn, types, pipeline_def
    (tmp_path / "a").mkdir()
    streams = [ws.cv2_webp(ws.image(60 + 10 * k, 80, 20 + k), 85) for k in range(3)]
    for n, s in zip(["0.webp", "1.webp", "2.JPEG"], streams):
        (tmp_path / "a" / n).write_bytes(s)

    @pipeline_def(batch_size=3, num_threads=1, device_id=0, seed=11, prefetch_queue_depth=1)
    def pipe():
        data, label = fn.readers.file(file_root=str(tmp_path), random_shuffle=False, name="Reader")
        return fn.decoders.image(data, device="mixed", output_type=types.RGB)
    p = pipe()
    p.build()
    (o,) = p.run()
    c = o.as_cpu()
    got = sorted((np.asarray(c[i]) for i in range(3)), key=lambda a: a.shape[0])
    for a, s in zip(got, streams):
        assert np.array_equal(a, ws.decode(s)[..., ::-1])
