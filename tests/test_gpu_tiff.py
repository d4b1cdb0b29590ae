"""-m gpu tests of TIFF streams in the image decoder: the corpus of tests/tiff_streams.py in every output type and dtype against the
oracle of tests/tiff_oracle.py (pinned to cv2.imdecode by tests/test_tiff_cpu.py), regions of interest of the C-ABI and the crop
operators, orientations, a batch mixing every JPEG path, PNG and TIFF samples, each corruption class, plan reuse, and fn.readers.file
over a directory of .tif files."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
import png_streams as ps  # noqa: E402
import png_oracle as pngo  # noqa: E402
import tiff_oracle as to  # noqa: E402
import tiff_streams as ts  # noqa: E402
import pointwise_ref as pr  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


@pytest.fixture(scope="module")
def corpus():
    c = ts.corpus()
    return [s for _, s in c], [to.decode(s) for _, s in c], [n for n, _ in c]


def test_corpus_rgb_bgr_gray(corpus):
    import gpu_helpers as g
    streams, want, names = corpus
    for ot in (capi.RGB, capi.BGR, capi.GRAY):
        outs, status = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)
        assert status == [0] * len(streams)
        for i, o in enumerate(outs):
            rgb, gray, _ = want[i]
            w = rgb[..., ::-1] if ot == capi.BGR else gray[..., None] if ot == capi.GRAY else rgb
            assert np.array_equal(o, w), (names[i], ot)


def test_corpus_ycbcr_and_float(corpus):
    """YCbCr and float are the post pass over the RGB (GRAY) decode, as for JPEG and PNG"""
    import gpu_helpers as g
    streams, want, names = corpus
    ref = po.have_ref()
    for ot, it in ((capi.RGB, po.IT_RGB), (capi.BGR, po.IT_BGR), (capi.YCbCr, po.IT_YCBCR), (capi.GRAY, po.IT_GRAY)):
        for dt, fl in ((capi.UINT8, False), (capi.FLOAT, True)):
            outs, status = g.jpeg_decode_ex(streams, output_type=ot, dtype=dt, adjust_orientation=False)
            assert status == [0] * len(streams)
            for i, o in enumerate(outs):
                src = want[i][1][..., None] if ot == capi.GRAY else want[i][0]
                pr.check_decoder_output(o, src, ot, fl, (names[i], ot, dt))
                if ref:
                    assert np.array_equal(o, po.ref_decoder_convert(src, it, fl)), (names[i], ot, dt)


def _layouts():
    return [ts.encode(ts.samples(97, 131, 3, 8, 1), 2, 8, 5, 2, rows_per_strip=1),
            ts.encode(ts.samples(64, 80, 4, 16, 2), 2, 16, 8, 2, planar=2, tile=(32, 16), extra=(2,)),
            ts.encode(ts.samples(50, 61, 1, 4, 3), 3, 4, 32773, colormap=ts.palette(4, 3), rows_per_strip=7, big_endian=True),
            ts.encode(ts.samples(203, 310, 1, 1, 4), 0, 1, 5, tile=(48, 32))]


def test_roi_windows_equal_crops_of_the_full_decode():
    import gpu_helpers as g
    streams = _layouts()
    rng = np.random.default_rng(8)
    for ot in (capi.RGB, capi.GRAY):
        full = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)[0]
        for i, s in enumerate(streams):
            rgb, gray, _ = to.decode(s)
            assert np.array_equal(full[i], gray[..., None] if ot == capi.GRAY else rgb), (ot, i)
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


def test_crop_operators_on_tiff():
    from dali_b200 import fn, pipeline_def
    streams = [np.frombuffer(s, np.uint8) for s in _layouts()[:3]]
    full = [to.decode(s.tobytes())[0] for s in streams]

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
    import cv2
    import gpu_helpers as g
    a = ts.samples(37, 53, 3, 8, 70)
    streams = [ts.encode(a, 2, 8, 5, 2, rows_per_strip=4, orientation=o) for o in range(1, 9)]
    rgb = to.decode(streams[0])[0]
    outs, status = g.jpeg_decode_ex(streams, adjust_orientation=True)
    assert status == [0] * 8
    for o in range(1, 9):
        assert np.array_equal(outs[o - 1], to.orient(rgb, o)), o
        assert np.array_equal(outs[o - 1], cv2.imdecode(np.frombuffer(streams[o - 1], np.uint8), cv2.IMREAD_COLOR)[..., ::-1]), o


def test_mixed_batch():
    """baseline, progressive, YCCK JPEG, PNG and TIFF samples in one batch: every JPEG sample equals its decode in a JPEG-only batch"""
    import cv2
    import gpu_helpers as g
    from jpeg_cmyk_streams import photoshop_ycck
    jpegs = [cv2.imencode(".jpg", g.synth_image(300, 420, 1))[1].tobytes(),
             cv2.imencode(".jpg", g.synth_image(120, 160, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(), photoshop_ycck(97, 131, 3)]
    png = ps.encode(ps.samples(40, 50, 2, 8, 80), 2, 8, filters="mixed")
    tiffs = [cv2.imencode(".tiff", g.synth_image(240, 320, 4))[1].tobytes()] + _layouts()[1:3]
    for ot in (capi.RGB, capi.GRAY):
        solo = g.jpeg_decode(jpegs, output_type=ot)[0]
        streams = [tiffs[0], jpegs[0], png, tiffs[1], jpegs[1], jpegs[2], tiffs[2]]
        outs, status = g.jpeg_decode(streams, output_type=ot)
        assert status == [0] * len(streams)
        for o, k in zip([outs[1], outs[4], outs[5]], range(3)):
            assert np.array_equal(o, solo[k]), (ot, k)
        pr = pngo.decode(png)
        assert np.array_equal(outs[2], pr[1][..., None] if ot == capi.GRAY else pr[0])
        for o, s in zip([outs[0], outs[3], outs[6]], tiffs):
            rgb, gray, _ = to.decode(s)
            assert np.array_equal(o, gray[..., None] if ot == capi.GRAY else rgb), ot


def test_each_corruption_class():
    """a corrupt segment sets the sample's status; a malformed or unsupported IFD fails the plan set-up for the batch"""
    import gpu_helpers as g
    good = ts.encode(ts.samples(20, 30, 3, 8, 90), 2, 8, 5)
    for name, s in ts.data_corrupt():
        outs, status = g.jpeg_decode([good, s, good])
        assert status == [0, 1, 0], name
        assert np.array_equal(outs[0], to.decode(good)[0]) and np.array_equal(outs[2], outs[0]), name
    for name, s in ts.plan_corrupt():
        with pytest.raises(Exception):
            g.jpeg_decode([good, s])


def test_pipeline_reports_the_failed_sample():
    from dali_b200 import fn, pipeline_def
    good = ts.encode(ts.samples(20, 30, 3, 8, 91), 2, 8, 5)
    bad = dict(ts.data_corrupt())["deflate_adler"]
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


def test_plan_reuse_with_growing_tiff_sizes():
    import gpu_helpers as g
    plan = capi.Plan("Jpeg", 4)
    for k, (h, w) in enumerate([(8, 8), (120, 160), (17, 400), (480, 640), (33, 47)]):
        streams = [ts.encode(ts.samples(h + j, w, 3, 8, 100 + k), 2, 8, [5, 8, 32773][j], 2, rows_per_strip=1 + j) for j in range(3)]
        outs, status = g.jpeg_decode(streams, plan=plan)
        assert status == [0, 0, 0]
        for s, o in zip(streams, outs):
            assert np.array_equal(o, to.decode(s)[0]), (h, w)


def test_file_reader_over_tif_files(tmp_path):
    """fn.readers.file over a directory of .tif / .tiff files (and a TIFF named .JPEG) through decoders.image"""
    import cv2
    import gpu_helpers as g
    from dali_b200 import fn, types, pipeline_def
    (tmp_path / "a").mkdir()
    imgs = [g.synth_image(60 + 10 * k, 80, 20 + k) for k in range(3)]
    names = ["0.tif", "1.tiff", "2.JPEG"]
    for n, img in zip(names, imgs):
        (tmp_path / "a" / n).write_bytes(cv2.imencode(".tiff", img)[1].tobytes())

    @pipeline_def(batch_size=3, num_threads=1, device_id=0, seed=11, prefetch_queue_depth=1)
    def pipe():
        data, label = fn.readers.file(file_root=str(tmp_path), random_shuffle=False, name="Reader")
        return fn.decoders.image(data, device="mixed", output_type=types.RGB)
    p = pipe()
    p.build()
    (o,) = p.run()
    c = o.as_cpu()
    got = sorted((np.asarray(c[i]) for i in range(3)), key=lambda a: a.shape[0])
    for a, img in zip(got, imgs):
        assert np.array_equal(a, img[..., ::-1])
