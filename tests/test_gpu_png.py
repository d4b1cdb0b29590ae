"""-m gpu tests of PNG streams in the image decoder: the corpus of tests/png_streams.py in every output type and dtype against the
oracle of tests/png_oracle.py (pinned to cv2.imdecode by tests/test_png_cpu.py), regions of interest of the crop operators, eXIf
orientations, a batch mixing every JPEG path with PNG samples, each corruption class, plan reuse, and fn.readers.file over a directory
where a .JPEG file holds a PNG stream."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
import png_oracle as pngo  # noqa: E402
import png_streams as ps  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


@pytest.fixture(scope="module")
def corpus():
    c = ps.corpus()
    return [s for _, s in c], [pngo.decode(s) for _, s in c], [n for n, _ in c]


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
    """YCbCr and float are the post pass over the RGB (GRAY) decode, as for JPEG: compared with the reference's convert functors where
    present, otherwise float RGB / BGR / GRAY as u8 * (1 / 255) in float32"""
    import gpu_helpers as g
    streams, want, names = corpus
    ref = po.have_ref()
    for ot, it in ((capi.RGB, po.IT_RGB), (capi.BGR, po.IT_BGR), (capi.YCbCr, po.IT_YCBCR), (capi.GRAY, po.IT_GRAY)):
        for dt, fl in ((capi.UINT8, False), (capi.FLOAT, True)):
            outs, status = g.jpeg_decode_ex(streams, output_type=ot, dtype=dt, adjust_orientation=False)
            assert status == [0] * len(streams)
            for i, o in enumerate(outs):
                src = want[i][1][..., None] if ot == capi.GRAY else want[i][0]
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


def test_roi_windows_equal_crops_of_the_full_decode():
    """the C-ABI windows image_crop / image_random_crop / image_slice use; left edges at every phase"""
    import gpu_helpers as g
    streams = [ps.encode(ps.samples(h, w, ct, d, 40 + k), ct, d, filters="mixed", interlace=il,
                         palette=np.random.default_rng(k).integers(0, 256, (256, 3)) if ct == 3 else None, seed=k)
               for k, (h, w, ct, d, il) in enumerate([(97, 131, 2, 8, False), (64, 80, 3, 4, True), (50, 61, 0, 16, True),
                                                       (203, 310, 6, 16, False)])]
    rng = np.random.default_rng(8)
    for ot in (capi.RGB, capi.BGR, capi.GRAY):
        full = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)[0]
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


def test_crop_operators_on_png():
    """fn.decoders.image_crop / image_random_crop / image_slice on PNG samples equal the expected windows of the full decode: the
    crop anchor and slice rounding of the reference (as tests/test_gpu_pipeline.py checks them for JPEG); the random window against
    the reference's generator where its compiled kernels are present, otherwise its shape and placement inside the image"""
    from dali_b200 import fn, pipeline_def
    streams = [np.frombuffer(ps.encode(ps.samples(h, w, 2, 8, 60 + h), 2, 8, filters="mixed", interlace=h % 2 == 1), np.uint8)
               for h, w in ((120, 160), (77, 95), (64, 64))]
    full = [pngo.decode(s.tobytes())[0] for s in streams]
    anchors = [np.array([0.1 + 0.05 * i, 0.2], np.float32) for i in range(len(streams))]
    shapes = [np.array([0.5, 0.6 - 0.05 * i], np.float32) for i in range(len(streams))]

    @pipeline_def(batch_size=len(streams), num_threads=1, device_id=0, prefetch_queue_depth=1, seed=5)
    def pipe():
        enc = fn.external_source(source=lambda i: streams)
        anc = fn.external_source(source=lambda i: anchors)
        shp = fn.external_source(source=lambda i: shapes)
        a = fn.decoders.image_crop(enc, device="mixed", crop=(40, 50), crop_pos_x=0.3, crop_pos_y=0.6)
        b = fn.decoders.image_random_crop(enc, device="mixed", seed=1234, random_area=[0.1, 0.9])
        c = fn.decoders.image_slice(enc, anc, shp, device="mixed")
        d = fn.decoders.image_slice(enc, device="mixed", start=[16, 30], shape=[40, 30], axes=[0, 1])
        e = fn.decoders.image(enc, device="mixed")
        return a, b, c, d, e
    p = pipe()
    p.build()
    res = [o.as_cpu() for o in p.run()]
    a, b, c, d, e = [[np.asarray(r[i]) for i in range(len(streams))] for r in res]
    rnd = lambda v: int(np.floor(v + 0.5))                   # std::llround: half away from zero (slice_attr.h:330-331)
    for i, f in enumerate(full):
        H, W = f.shape[:2]
        assert np.array_equal(e[i], f), i
        y0, x0 = po.crop_anchor(0.6, H, 40), po.crop_anchor(0.3, W, 50)
        assert np.array_equal(a[i], f[y0:y0 + 40, x0:x0 + 50]), i
        ax, ay = float(anchors[i][0]), float(anchors[i][1])
        sx, sy = float(shapes[i][0]), float(shapes[i][1])
        assert np.array_equal(c[i], f[rnd(ay * H):rnd((ay + sy) * H), rnd(ax * W):rnd((ax + sx) * W)]), i
        assert np.array_equal(d[i], f[16:56, 30:60]), i
        if po.have_ref():
            wy, wx, wh, ww = po.ref_random_crop(1234, i, H, W, area=(0.1, 0.9), ncalls=1)[0]
            assert np.array_equal(b[i], f[wy:wy + wh, wx:wx + ww]), i
        else:
            h, w = b[i].shape[:2]
            assert 0.1 * H * W * 0.9 <= h * w <= H * W, (i, b[i].shape)
            assert any(np.array_equal(f[y:y + h, x:x + w], b[i]) for y in range(H - h + 1) for x in range(W - w + 1)), i


def test_exif_orientations():
    import cv2
    import gpu_helpers as g
    a = ps.samples(37, 53, 2, 8, 70)
    streams = [ps.encode(a, 2, 8, filters="mixed", exif=o, exif_after=o % 2 == 0) for o in range(1, 9)]
    rgb = pngo.decode(streams[0])[0]
    outs, status = g.jpeg_decode_ex(streams, adjust_orientation=True)
    assert status == [0] * 8
    for o in range(1, 9):
        assert np.array_equal(outs[o - 1], pngo.orient(rgb, o)), o
        assert np.array_equal(outs[o - 1], cv2.imdecode(np.frombuffer(streams[o - 1], np.uint8), cv2.IMREAD_COLOR)[..., ::-1]), o
    outs, status = g.jpeg_decode_ex(streams, adjust_orientation=False)
    assert status == [0] * 8 and all(np.array_equal(o, rgb) for o in outs)
    gray, status = g.jpeg_decode_ex(streams, output_type=capi.GRAY, adjust_orientation=True, dtype=capi.FLOAT)
    g8 = pngo.decode(streams[0])[1]
    for o in range(1, 9):
        assert np.array_equal(gray[o - 1][..., 0], pngo.orient(g8, o).astype(np.float32) * np.float32(1.0 / 255)), o


def _enc_jpeg(img, **kw):
    import cv2
    p = []
    for k, v in kw.items():
        p += [getattr(cv2, k), v]
    return cv2.imencode(".jpg", img, p)[1].tobytes()


def test_mixed_batch_jpeg_samples_are_bit_identical():
    """baseline 4:2:0, progressive, CMYK / YCCK and PNG samples in one batch: every JPEG sample equals its decode in a JPEG-only batch,
    every PNG sample the oracle"""
    import gpu_helpers as g
    from jpeg_cmyk_streams import photoshop_ycck
    jpegs = [_enc_jpeg(g.synth_image(1080, 1920, 1)), _enc_jpeg(g.synth_image(300, 420, 2), IMWRITE_JPEG_PROGRESSIVE=1),
             photoshop_ycck(97, 131, 3), _enc_jpeg(g.synth_image(123, 77, 4)[..., 0]), photoshop_ycck(61, 77, 5, transform=0)]
    pngs = [ps.encode(ps.samples(h, w, ct, d, 80 + h), ct, d, filters="mixed", interlace=il) for h, w, ct, d, il in
            [(240, 320, 2, 8, False), (17, 9, 0, 1, True), (100, 130, 6, 16, True)]]
    for ot in (capi.RGB, capi.GRAY):
        solo = g.jpeg_decode(jpegs, output_type=ot)[0]
        order = [("p", 0), ("j", 0), ("j", 1), ("p", 1), ("j", 2), ("j", 3), ("p", 2), ("j", 4)]
        streams = [pngs[k] if t == "p" else jpegs[k] for t, k in order]
        outs, status = g.jpeg_decode(streams, output_type=ot)
        assert status == [0] * len(streams)
        for (t, k), o in zip(order, outs):
            if t == "j":
                assert np.array_equal(o, solo[k]), (ot, k)
            else:
                rgb, gray, _ = pngo.decode(pngs[k])
                assert np.array_equal(o, gray[..., None] if ot == capi.GRAY else rgb), (ot, k)


def test_each_corruption_sets_its_status():
    """streams the planner accepts but whose data is bad (CRC, Adler-32, truncation, filter byte, distance, symbol, code lengths, the
    stream's tail) set the sample's status; header-level corruptions (chunk structure, IHDR) are rejected at plan set-up, for the
    batch, as malformed JPEG headers are"""
    import gpu_helpers as g
    good = ps.encode(ps.samples(20, 30, 2, 8, 90), 2, 8)
    data_level = {"idat_crc", "adler", "truncated", "filter5", "distance", "undefined_symbol", "code_lengths"}
    data_level |= {n for n, _, ok in ps.zlib_tails() if not ok}
    for name, s in ps.corrupt():
        if name in data_level:
            outs, status = g.jpeg_decode([good, s, good])
            assert status == [0, 1, 0], name
            assert np.array_equal(outs[0], pngo.decode(good)[0]) and np.array_equal(outs[2], outs[0]), name
        else:
            with pytest.raises(Exception):
                g.jpeg_decode([good, s])


def test_pipeline_reports_the_failed_sample():
    from dali_b200 import fn, pipeline_def
    good = ps.encode(ps.samples(20, 30, 2, 8, 91), 2, 8)
    bad = dict(ps.corrupt())["adler"]
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


def test_plan_reuse_with_growing_png_sizes():
    import gpu_helpers as g
    plan = capi.Plan("Jpeg", 4)
    for k, (h, w) in enumerate([(8, 8), (120, 160), (17, 400), (480, 640), (33, 47)]):
        streams = [ps.encode(ps.samples(h + j, w, 2, 8, 100 + k), 2, 8, filters="mixed", interlace=j == 1) for j in range(3)]
        outs, status = g.jpeg_decode(streams, plan=plan)
        assert status == [0, 0, 0]
        for s, o in zip(streams, outs):
            assert np.array_equal(o, pngo.decode(s)[0]), (h, w)


def test_file_reader_with_a_png_named_jpeg(tmp_path):
    """fn.readers.file over a directory where one .JPEG file holds a PNG stream (as n02105855_2933.JPEG in ILSVRC-2012), through
    decoders.image_random_crop -> resize -> crop_mirror_normalize: every batch runs, and the PNG sample's tensor depends only on its
    pixels (cv2's PNG and one with another filter choice and IDAT split give the same batches)"""
    import cv2
    import gpu_helpers as g
    from dali_b200 import fn, types, pipeline_def
    img = g.synth_image(375, 500, 3)
    (tmp_path / "a").mkdir()
    for k in range(5):
        (tmp_path / "a" / f"{k}.JPEG").write_bytes(_enc_jpeg(g.synth_image(300 + 10 * k, 400, 10 + k)))
    variants = [cv2.imencode(".png", img[..., ::-1])[1].tobytes(), ps.encode(img, 2, 8, filters="mixed", split=777, seed=3)]
    results = []
    for v in variants:
        (tmp_path / "a" / "2933.JPEG").write_bytes(v)

        @pipeline_def(batch_size=3, num_threads=1, device_id=0, seed=11, prefetch_queue_depth=1)
        def pipe():
            data, label = fn.readers.file(file_root=str(tmp_path), random_shuffle=False, name="Reader")
            x = fn.decoders.image_random_crop(data, device="mixed", output_type=types.RGB)
            x = fn.resize(x, resize_x=112, resize_y=112)
            return fn.crop_mirror_normalize(x, dtype=types.FLOAT, output_layout="CHW", crop=(96, 96), mean=[120.0] * 3, std=[60.0] * 3)
        p = pipe()
        p.build()
        outs = []
        for _ in range(2):
            (o,) = p.run()
            c = o.as_cpu()
            outs += [np.asarray(c[i]) for i in range(3)]
        results.append(outs)
    assert len(results[0]) == 6
    for a, b in zip(*results):
        assert a.shape == (3, 96, 96) and np.isfinite(a).all()
        assert np.array_equal(a, b)
