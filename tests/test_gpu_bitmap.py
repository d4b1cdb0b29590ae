"""-m gpu tests of BMP and PNM streams in the image decoder: the corpus of tests/bitmap_streams.py in RGB / BGR / GRAY against
cv2.imdecode, YCbCr and float output against tests/pointwise_ref.py, a batch mixing every JPEG path, PNG, TIFF, WebP, BMP and PNM
samples, the crop operators, each corruption class, the pipeline's error for a corrupt RLE sample, plan reuse, and fn.readers.file over
a directory of .bmp / .ppm / .pgm / .pbm files."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
import bitmap_streams as bs  # noqa: E402
import pointwise_ref as pr  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


def _cv(s, gray=False):
    import cv2
    if gray:
        return cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_GRAYSCALE)
    return cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR)[..., ::-1]


@pytest.fixture(scope="module")
def corpus():
    c = bs.corpus()
    return [s for _, s in c], [(_cv(s), _cv(s, True)) for _, s in c], [n for n, _ in c]


def test_corpus_rgb_bgr_gray(corpus):
    import gpu_helpers as g
    streams, want, names = corpus
    for ot in (capi.RGB, capi.BGR, capi.GRAY):
        outs, status = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)
        assert status == [0] * len(streams)
        for i, o in enumerate(outs):
            rgb, gray = want[i]
            w = rgb[..., ::-1] if ot == capi.BGR else gray[..., None] if ot == capi.GRAY else rgb
            assert np.array_equal(o, w), (names[i], ot)


def test_corpus_ycbcr_and_float(corpus):
    """YCbCr and float are the post pass over the RGB (GRAY) decode, as for the other formats"""
    import gpu_helpers as g
    streams, want, names = corpus
    sel = list(range(0, len(streams), 5))
    for ot in (capi.RGB, capi.BGR, capi.YCbCr, capi.GRAY):
        for dt, fl in ((capi.UINT8, False), (capi.FLOAT, True)):
            outs, status = g.jpeg_decode_ex([streams[i] for i in sel], output_type=ot, dtype=dt, adjust_orientation=False)
            assert status == [0] * len(sel)
            for o, i in zip(outs, sel):
                src = want[i][1][..., None] if ot == capi.GRAY else want[i][0]
                pr.check_decoder_output(o, src, ot, fl, (names[i], ot, dt))


def _layouts():
    return [bs.bmp(131, 97, 24, bs.rows(bs.image(97, 131, 1), 24)), bs.rle_bmp(90, 61, 8, 2), bs.pnm(3, bs.image(50, 61, 3), 255),
            bs.pnm(4, bs.image(64, 203, 4)[..., 0] >> 7), bs.rle_bmp(77, 40, 4, 5)]


def test_roi_windows_equal_crops_of_the_full_decode():
    import gpu_helpers as g
    streams = _layouts()
    rng = np.random.default_rng(8)
    for ot in (capi.RGB, capi.GRAY):
        full = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)[0]
        for i, s in enumerate(streams):
            assert np.array_equal(full[i], _cv(s, True)[..., None] if ot == capi.GRAY else _cv(s)), (ot, i)
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


def test_crop_operators_on_bitmaps():
    from dali_b200 import fn, pipeline_def
    streams = [np.frombuffer(s, np.uint8) for s in _layouts()[:4]]
    full = [_cv(s.tobytes()) for s in streams]

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


def test_mixed_batch():
    """baseline and progressive JPEG, PNG, TIFF, WebP, BMP and PNM samples in one batch: every JPEG sample equals its decode in a
    JPEG-only batch, every other sample equals cv2"""
    import cv2
    import gpu_helpers as g
    import png_streams as ps
    import tiff_streams as ts
    import webp_streams as ws
    jpegs = [cv2.imencode(".jpg", g.synth_image(300, 420, 1))[1].tobytes(),
             cv2.imencode(".jpg", g.synth_image(120, 160, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()]
    others = [ps.encode(ps.samples(40, 50, 2, 8, 80), 2, 8, filters="mixed"), cv2.imencode(".tiff", g.synth_image(240, 320, 4))[1].tobytes(),
              ws.cv2_webp(ws.image(40, 56, 7), 70)] + _layouts()
    for ot in (capi.RGB, capi.GRAY):
        solo = g.jpeg_decode(jpegs, output_type=ot)[0]
        streams = [others[3], jpegs[0], others[0], others[4], jpegs[1], others[1], others[5], others[2], others[6], others[7]]
        outs, status = g.jpeg_decode(streams, output_type=ot)
        assert status == [0] * len(streams)
        assert np.array_equal(outs[1], solo[0]) and np.array_equal(outs[4], solo[1]), ot
        for k in (0, 3, 6, 8, 9):
            s = streams[k]
            assert np.array_equal(outs[k], _cv(s, True)[..., None] if ot == capi.GRAY else _cv(s)), (ot, k)


def test_each_corruption_class():
    """corrupt RLE / ASCII data sets the sample's status; a malformed or unsupported header fails the plan set-up for the batch"""
    import gpu_helpers as g
    good = bs.rle_bmp(30, 20, 8, 90)
    for name, s in bs.data_corrupt():
        outs, status = g.jpeg_decode([good, s, good])
        assert status == [0, 1, 0], name
        assert np.array_equal(outs[0], _cv(good)) and np.array_equal(outs[2], outs[0]), name
    for name, s, _ in bs.plan_corrupt() + bs.refused_here_only():
        with pytest.raises(Exception):
            g.jpeg_decode([good, s])


def test_pipeline_reports_the_failed_sample():
    from dali_b200 import fn, pipeline_def
    good = bs.rle_bmp(30, 20, 8, 91)
    bad = dict(bs.data_corrupt())["rle8_no_eob"]
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


def test_plan_reuse_with_growing_sizes():
    import gpu_helpers as g
    plan = capi.Plan("Jpeg", 4)
    for k, (h, w) in enumerate([(8, 8), (120, 160), (17, 400), (480, 640), (33, 47)]):
        streams = [bs.rle_bmp(w, h, 8, k), bs.bmp(w, -h, 24, bs.rows(bs.image(h, w, k), 24, True)), bs.pnm(2, bs.image(h, w, k)[..., 0], 255),
                   bs.pnm(6, bs.image(h, w, k).astype(np.uint16) * 200, 65535)]
        outs, status = g.jpeg_decode(streams, plan=plan)
        assert status == [0] * 4
        for s, o in zip(streams, outs):
            assert np.array_equal(o, _cv(s)), (h, w)


def test_file_reader_over_bitmap_files(tmp_path):
    """fn.readers.file over a directory of .bmp / .ppm / .pgm / .pbm files (and a BMP named .JPEG) through decoders.image"""
    import cv2
    import gpu_helpers as g
    from dali_b200 import fn, types, pipeline_def
    (tmp_path / "a").mkdir()
    imgs = [g.synth_image(60 + 10 * k, 80, 20 + k) for k in range(5)]
    files = [("0.bmp", ".bmp", imgs[0]), ("1.ppm", ".ppm", imgs[1]), ("2.pgm", ".pgm", imgs[2][..., 1]),
             ("3.pbm", ".pbm", imgs[3][..., 2]), ("4.JPEG", ".bmp", imgs[4])]
    want = []
    for n, ext, img in files:
        s = cv2.imencode(ext, img)[1].tobytes()
        (tmp_path / "a" / n).write_bytes(s)
        want.append(_cv(s))

    @pipeline_def(batch_size=5, num_threads=1, device_id=0, seed=11, prefetch_queue_depth=1)
    def pipe():
        data, label = fn.readers.file(file_root=str(tmp_path), random_shuffle=False, name="Reader")
        return fn.decoders.image(data, device="mixed", output_type=types.RGB)
    p = pipe()
    p.build()
    (o,) = p.run()
    c = o.as_cpu()
    got = sorted((np.asarray(c[i]) for i in range(5)), key=lambda a: a.shape[0])
    for a, w in zip(got, want):
        assert np.array_equal(a, w)
