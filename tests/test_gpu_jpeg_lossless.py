"""-m gpu tests of lossless JPEG (SOF3) in the image decoder: the corpus of tests/ljpeg_streams.py in RGB / BGR / GRAY against the encoder's
input and cv2.imdecode, YCbCr and float output against tests/pointwise_ref.py, regions of interest and EXIF orientation, a batch mixing
lossless samples with every other path, each corruption class and each refused stream, mutated entropy data against cv2, plan reuse, and
fn.readers.file over a directory of lossless files."""
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
import ljpeg_streams as ls  # noqa: E402
import pointwise_ref as pr  # noqa: E402


def _gray(a):
    """GRAY of an RGB-coded pixel: libjpeg-turbo's rgb_gray_convert, the rule of the baseline path's RGB JPEG"""
    a = a.astype(np.int64)
    return ((a[..., 0] * 19595 + a[..., 1] * 38470 + a[..., 2] * 7471 + 32768) >> 16).astype(np.uint8)[..., None]


def _want(exp, ot):
    """expected output of the H x W x C samples `exp`: one component is replicated for RGB / BGR (a documented deviation: cv2 refuses
    colour conversion of lossless JPEG), three components go to GRAY by _gray (the other deviation)"""
    if ot == capi.GRAY:
        return exp if exp.shape[2] == 1 else _gray(exp)
    rgb = np.repeat(exp, 3, axis=2) if exp.shape[2] == 1 else exp
    return rgb[..., ::-1] if ot == capi.BGR else rgb


def _cv(s):
    import cv2
    d = cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_UNCHANGED)
    if d is None:
        return None
    return d[..., None] if d.ndim == 2 else d[..., ::-1]


@pytest.fixture(scope="module")
def corpus():
    return ls.corpus(big=True)


def test_corpus_rgb_bgr_gray(corpus):
    import gpu_helpers as g
    streams = [s for _, s, _, _ in corpus]
    for name, s, exp, _ in corpus:
        assert np.array_equal(_cv(s), exp), name          # the encoder's input is what cv2 decodes
    for ot in (capi.RGB, capi.BGR, capi.GRAY):
        outs, status = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)
        assert status == [0] * len(streams)
        for (name, _, exp, _), o in zip(corpus, outs):
            assert np.array_equal(o, _want(exp, ot)), (name, ot)


def test_each_image_alone(corpus):
    """a batch of one sample: the wavefront and the chains of one image alone"""
    import gpu_helpers as g
    for name, s, exp, _ in corpus[::9] + corpus[-3:]:
        outs, status = g.jpeg_decode_ex([s], output_type=capi.RGB, adjust_orientation=False)
        assert status == [0] and np.array_equal(outs[0], _want(exp, capi.RGB)), name


def test_corpus_ycbcr_and_float(corpus):
    """YCbCr and float are the post pass over the RGB (GRAY) decode, as for the other formats"""
    import gpu_helpers as g
    sel = corpus[::4]
    for ot in (capi.RGB, capi.BGR, capi.YCbCr, capi.GRAY):
        for dt, fl in ((capi.UINT8, False), (capi.FLOAT, True)):
            outs, status = g.jpeg_decode_ex([s for _, s, _, _ in sel], output_type=ot, dtype=dt, adjust_orientation=False)
            assert status == [0] * len(sel)
            for o, (name, _, exp, _) in zip(outs, sel):
                src = _want(exp, capi.GRAY) if ot == capi.GRAY else _want(exp, capi.RGB)
                pr.check_decoder_output(o, src, ot, fl, (name, ot, dt))


def _with_exif(s, orientation):
    body = b"Exif\0\0" + b"MM\x00\x2a\x00\x00\x00\x08\x00\x01" + struct.pack(">HHIHH", 0x0112, 3, 1, orientation, 0) + b"\0\0\0\0"
    return s[:2] + b"\xFF\xE1" + struct.pack(">H", len(body) + 2) + body + s[2:]


def _orient(a, o):
    return {1: a, 2: a[:, ::-1], 3: a[::-1, ::-1], 4: a[::-1], 5: a.swapaxes(0, 1), 6: np.rot90(a, -1), 7: a[::-1, ::-1].swapaxes(0, 1),
            8: np.rot90(a, 1)}[o]


def test_roi_and_orientation():
    import gpu_helpers as g
    imgs = [ls.image(37, 53, 3, 8, 60), ls.image(64, 41, 1, 8, 61)]
    streams = [ls.encode(imgs[0], pred=4, restart=53 * 5), ls.encode(imgs[1], pred=7, tables="opt")]
    rng = np.random.default_rng(3)
    for ot in (capi.RGB, capi.GRAY):
        full = [_want(i if i.ndim == 3 else i[..., None], ot) for i in imgs]
        for rep in range(4):
            rois = []
            for f in full:
                H, W = f.shape[:2]
                x0, y0 = int(rng.integers(0, W - 1)), int(rng.integers(0, H - 1))
                rois.append((x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1))))
            outs, status = g.jpeg_decode_ex(streams, output_type=ot, rois=rois, adjust_orientation=False)
            assert status == [0, 0]
            for i, r in enumerate(rois):
                assert np.array_equal(outs[i], full[i][r[1]:r[3], r[0]:r[2]]), (ot, rep, i, r)
        for o in range(1, 9):
            outs, status = g.jpeg_decode_ex([_with_exif(s, o) for s in streams], output_type=ot, adjust_orientation=True)
            assert status == [0, 0]
            for i in range(2):
                assert np.array_equal(outs[i], _orient(full[i], o)), (ot, o, i)


def test_mixed_batch():
    """lossless samples among baseline and progressive JPEG, PNG, TIFF, WebP and BMP samples: every sample equals its decode alone"""
    import cv2
    import gpu_helpers as g
    import bitmap_streams as bs
    import png_streams as ps
    import webp_streams as ws
    lossless = [ls.encode(ls.image(90, 120, 3, 8, 70), pred=5), ls.encode(ls.image(33, 17, 1, 6, 71), P=6, Pt=2, restart=17 * 4),
                ls.encode(ls.image(200, 150, 1, 8, 72), pred=7, tables="deep")]
    others = [cv2.imencode(".jpg", g.synth_image(300, 420, 1))[1].tobytes(),
              cv2.imencode(".jpg", g.synth_image(120, 160, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(),
              ps.encode(ps.samples(40, 50, 2, 8, 80), 2, 8, filters="mixed"), cv2.imencode(".tiff", g.synth_image(240, 320, 4))[1].tobytes(),
              ws.cv2_webp(ws.image(40, 56, 7), 70), bs.bmp(131, 97, 24, bs.rows(bs.image(97, 131, 1), 24))]
    for ot in (capi.RGB, capi.GRAY):
        streams = [others[0], lossless[0], others[1], others[2], lossless[1], others[3], others[4], lossless[2], others[5]]
        solo = [g.jpeg_decode([s], output_type=ot)[0][0] for s in streams]
        outs, status = g.jpeg_decode(streams, output_type=ot)
        assert status == [0] * len(streams)
        for k, (o, w) in enumerate(zip(outs, solo)):
            assert np.array_equal(o, w), (ot, k)
        assert np.array_equal(outs[1], _want(_cv(lossless[0]), ot))


def test_batch_without_lossless_launches_as_before():
    """a batch with no lossless sample launches no ljpeg kernel; a lossless-only batch launches none of the baseline entropy kernels"""
    import cv2
    import gpu_helpers as g
    jpeg = cv2.imencode(".jpg", g.synth_image(64, 80, 3))[1].tobytes()
    capi.profiling(True)
    try:
        for streams, has_l, has_j in (([jpeg], False, True), ([ls.encode(ls.image(30, 40, 3, 8, 73))], True, False)):
            capi.profiling_collect()
            g.jpeg_decode(streams)
            names = [n for n, _ in capi.profiling_collect()]
            assert any(n.startswith("ljpeg_") for n in names) == has_l, names
            assert any(n.startswith(("jpeg_huff_sync", "jpeg_huff_write")) for n in names) == has_j, names
            assert any(n.startswith("jpeg_unstuff") for n in names), names
    finally:
        capi.profiling(False)


def test_each_corruption_class():
    """damaged entropy data sets only its own sample's status; every refused stream fails the plan set-up with its status"""
    import gpu_helpers as g
    good = ls.encode(ls.image(20, 30, 3, 8, 80), restart=30 * 2)
    want = _want(ls.image(20, 30, 3, 8, 80), capi.RGB)
    for name, s, kind in ls.corrupt():
        outs, status = g.jpeg_decode([good, s, good])
        assert status == [0, 1, 0], name
        assert np.array_equal(outs[0], want) and np.array_equal(outs[2], want), name
    for name, s, code, why in ls.refused():
        with pytest.raises(capi.DaliB200Error) as e:
            g.jpeg_decode([good, s])
        assert f"(status {code})" in str(e.value), (name, why, str(e.value))


def test_mutated_entropy_data_against_cv2():
    """bytes of the entropy-coded data replaced at random: wherever the decode reports no error and cv2 decodes, the two agree, which
    pins the reconstruction of out-of-range values (modulo 2^16, then the low 8 bits of the sample << Pt)"""
    import gpu_helpers as g
    rng = np.random.default_rng(5)
    bases = [ls.encode(ls.image(24, 33, 3, 8, 90), pred=p, tables="opt") for p in (1, 4, 5, 6, 7)] + \
            [ls.encode(ls.image(20, 21, 1, 6, 91), P=6, Pt=1, pred=p) for p in (2, 3, 4)]
    streams = []
    for k in range(400):
        b = bytearray(bases[k % len(bases)])
        sos = b.index(b"\xFF\xDA")
        lo = sos + 2 + struct.unpack(">H", bytes(b[sos + 2: sos + 4]))[0]
        for _ in range(int(rng.integers(1, 4))):
            q = int(rng.integers(lo, len(b) - 2))
            v = int(rng.integers(0, 255))                # never a new 0xFF: no new marker, no new stuffing
            if b[q] != 0xFF and (q == 0 or b[q - 1] != 0xFF):
                b[q] = v
        streams.append(bytes(b))
    checked = 0
    for i in range(0, len(streams), 50):
        chunk = streams[i:i + 50]
        outs, status = g.jpeg_decode_ex(chunk, output_type=capi.RGB, adjust_orientation=False)
        for s, o, st in zip(chunk, outs, status):
            c = _cv(s)
            if st == 0 and c is not None:
                assert np.array_equal(o, _want(c, capi.RGB))
                checked += 1
    assert checked > 100, checked


def test_plan_reuse_with_growing_sizes():
    import gpu_helpers as g
    plan = capi.Plan("Jpeg", 3)
    for k, (h, w) in enumerate([(8, 8), (120, 160), (17, 400), (480, 640), (33, 47)]):
        imgs = [ls.image(h, w, 3, 8, k), ls.image(h, w, 1, 8, k + 10), ls.image(h, w, 3, 7, k + 20)]
        streams = [ls.encode(imgs[0], pred=1 + k), ls.encode(imgs[1], restart=w, tables="opt"), ls.encode(imgs[2], P=7, pred=7 - k)]
        outs, status = g.jpeg_decode(streams, plan=plan)
        assert status == [0] * 3
        for o, a in zip(outs, imgs):
            assert np.array_equal(o, _want(a if a.ndim == 3 else a[..., None], capi.RGB)), (h, w)


def test_file_reader_over_lossless_files(tmp_path):
    """fn.readers.file over a directory of lossless JPEG files through decoders.image"""
    from dali_b200 import fn, types, pipeline_def
    (tmp_path / "a").mkdir()
    imgs = [ls.image(60 + 10 * k, 80, 3 if k % 2 else 1, 8, 100 + k) for k in range(4)]
    want = []
    for k, a in enumerate(imgs):
        (tmp_path / "a" / f"{k}.jpg").write_bytes(ls.encode(a, pred=k + 1))
        want.append(_want(a, capi.RGB))

    @pipeline_def(batch_size=4, num_threads=1, device_id=0, seed=11, prefetch_queue_depth=1)
    def pipe():
        data, label = fn.readers.file(file_root=str(tmp_path), random_shuffle=False, name="Reader")
        return fn.decoders.image(data, device="mixed", output_type=types.RGB)
    p = pipe()
    p.build()
    (o,) = p.run()
    c = o.as_cpu()
    got = sorted((np.asarray(c[i]) for i in range(4)), key=lambda a: a.shape[0])
    for a, w in zip(got, want):
        assert np.array_equal(a, w)
