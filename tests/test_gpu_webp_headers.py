"""-m gpu tests of the lossy WebP decode under frame headers and intra modes the encoders never write (ws.rewritten(), partition 0
rewritten by tests/vp8_rewrite.py), and at the two launch edges the corpus never reaches:
  * webp_wave_kernel walks each diagonal x + 2y of macroblocks with one CTA of 128 threads; a 4100 x 2050 image (257 x 129 macroblocks)
    has 129 macroblocks on diagonal 256, so one thread takes a second macroblock there;
  * webp_entropy_kernel packs more than one image into a warp (SerialLaneGeometry) once the batch holds more than 32 x SM-count WebP
    samples.
Everything bit for bit against cv2.imdecode."""
import cv2
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
import conftest  # noqa: E402
import png_oracle as pngo  # noqa: E402
import png_streams as ps  # noqa: E402
import pointwise_ref as pr  # noqa: E402
import tiff_oracle as to  # noqa: E402
import vp8_rewrite as vr  # noqa: E402
import webp_streams as ws  # noqa: E402

NO = cv2.IMREAD_IGNORE_ORIENTATION


def _want(s, ot):
    if ot == capi.GRAY:
        return ws.decode(s, cv2.IMREAD_GRAYSCALE | NO)[..., None]
    bgr = ws.decode(s, cv2.IMREAD_COLOR | NO)
    return bgr if ot == capi.BGR else bgr[..., ::-1]


@pytest.fixture(scope="module")
def rewritten():
    rw = ws.rewritten()
    for name, s, _ in rw:
        assert ws.decode(s) is not None, name
    return [n for n, _, _ in rw], [s for _, s, _ in rw]


def test_rewritten_corpus_in_one_batch(rewritten):
    import gpu_helpers as g
    names, streams = rewritten
    for ot in (capi.RGB, capi.BGR, capi.GRAY):
        outs, status = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)
        assert status == [0] * len(streams)
        for n, s, o in zip(names, streams, outs):
            assert np.array_equal(o, _want(s, ot)), (n, ot)


def test_rewritten_ycbcr_and_float(rewritten):
    import gpu_helpers as g
    names, streams = [v[::9] for v in rewritten]
    for ot in (capi.RGB, capi.YCbCr, capi.GRAY):
        for dt, fl in ((capi.UINT8, False), (capi.FLOAT, True)):
            if ot == capi.RGB and not fl:
                continue
            outs, status = g.jpeg_decode_ex(streams, output_type=ot, dtype=dt, adjust_orientation=False)
            assert status == [0] * len(streams)
            for n, s, o in zip(names, streams, outs):
                src = _want(s, capi.GRAY) if ot == capi.GRAY else _want(s, capi.RGB)
                pr.check_decoder_output(o, src, ot, fl, (n, ot, dt))


def test_rewritten_batches_of_one(rewritten):
    import gpu_helpers as g
    names, streams = rewritten
    plan = capi.Plan("Jpeg", 1)
    for n, s in list(zip(names, streams))[::13]:
        outs, status = g.jpeg_decode_ex([s], adjust_orientation=False, plan=plan)
        assert status == [0] and np.array_equal(outs[0], _want(s, capi.RGB)), n


def _max_diagonal(mb_w, mb_h):
    return max(sum(1 for y in range(mb_h) if 0 <= d - 2 * y < mb_w) for d in range(mb_w + 2 * mb_h - 2))


@pytest.fixture(scope="module")
def wide():
    """a cv2 quality-80 stream of 4100 x 2050, a rewritten variant (random modes, normal filter, filter and segment deltas) and a
    simple-filter variant"""
    s = ws.cv2_webp(ws.image(2050, 4100, 31, noise=12.0), 80)
    f = vr.parse(s)
    assert (f["mb_w"], f["mb_h"]) == (257, 129) and _max_diagonal(257, 129) == 129
    rng = np.random.default_rng(12)
    for m in f["mbs"]:
        m["uvmode"] = int(rng.integers(0, 4))
        if m["i4"]:
            m["bmodes"] = [int(v) for v in rng.integers(0, 10, 16)]
        else:
            m["ymode"] = int(rng.integers(0, 4))
        m["segment"] = int(rng.integers(0, 4))
    h = f["hdr"]
    h.update(use_segment=1, update_map=1, update_data=1, absolute_delta=0, quantizer=[-20, 10, None, 30],
             filter_strength=[-10, 12, 30, None], seg_proba=[120, None, 60], simple=0, level=28, sharpness=3, use_lf_delta=1,
             update_lf_delta=1, ref_lf_delta=[6, -3, None, 9], mode_lf_delta=[-9, None, 4, -5])
    normal = vr.write(f)
    h.update(simple=1, level=40)
    simple = vr.write(f)
    return [s, normal, simple]


def test_wavefront_past_one_cta(wide):
    import gpu_helpers as g
    for ot in (capi.RGB, capi.GRAY):
        outs, status = g.jpeg_decode_ex(wide, output_type=ot, adjust_orientation=False)
        assert status == [0, 0, 0]
        for k, (s, o) in enumerate(zip(wide, outs)):
            assert np.array_equal(o, _want(s, ot)), (k, ot)


def test_wavefront_past_one_cta_roi_windows(wide):
    import gpu_helpers as g
    s = wide[0]
    full = _want(s, capi.RGB)
    # around diagonal 256 (macroblocks (256 - 2y, y)), the corners, and a thin strip across the whole width
    rois = [(4096 - 16 * 40, 16 * 40, 4096 - 16 * 30, 16 * 45), (0, 0, 37, 29), (4100 - 50, 2050 - 33, 4100, 2050),
            (3, 1000, 4099, 1003), (2000, 0, 2100, 2050)]
    outs, status = g.jpeg_decode_ex([s] * len(rois), rois=rois, adjust_orientation=False)
    assert status == [0] * len(rois)
    for r, o in zip(rois, outs):
        assert np.array_equal(o, full[r[1]:r[3], r[0]:r[2]]), r


def test_tall_image_control():
    """2050 x 4100: 129 x 257 macroblocks, never more than 65 on a diagonal"""
    import gpu_helpers as g
    s = ws.cv2_webp(ws.image(4100, 2050, 32, noise=12.0), 80)
    f = vr.parse(s)
    assert (f["mb_w"], f["mb_h"]) == (129, 257) and _max_diagonal(129, 257) == 65
    outs, status = g.jpeg_decode_ex([s], adjust_orientation=False)
    assert status == [0] and np.array_equal(outs[0], _want(s, capi.RGB))


def test_more_than_one_image_per_entropy_warp():
    """32 x SM-count + 300 samples of 1x1 to 24x24, encoder and rewritten streams, with corrupt samples inside the batch: each sets
    only its own status"""
    import gpu_helpers as g
    import torch
    sms = 132 if conftest.DRY_RUN else torch.cuda.get_device_properties(0).multi_processor_count
    n = 32 * sms + 300
    print(f"SM count {sms}: {n} WebP samples in one batch")
    rng = np.random.default_rng(21)
    streams = []
    for k in range(n):
        h, w = int(rng.integers(1, 25)), int(rng.integers(1, 25))
        s = ws.cv2_webp(ws.image(h, w, 1000 + k, noise=float(rng.uniform(2, 40))), int(rng.integers(1, 101)))
        if k % 3 == 0:
            f = vr.parse(s)
            fh = f["hdr"]
            if rng.random() < 0.5:
                fh.update(use_segment=1, update_map=1, update_data=1, absolute_delta=int(rng.integers(0, 2)),
                          quantizer=[int(v) for v in rng.integers(-127, 128, 4)], filter_strength=[int(v) for v in rng.integers(-63, 64, 4)],
                          seg_proba=[int(v) for v in rng.integers(1, 256, 3)])
                for m in f["mbs"]:
                    m["segment"] = int(rng.integers(0, 4))
            fh.update(level=int(rng.integers(0, 64)), simple=int(rng.integers(0, 2)), sharpness=int(rng.integers(0, 8)),
                      base_q0=int(rng.integers(0, 128)), use_lf_delta=1, update_lf_delta=1,
                      ref_lf_delta=[int(rng.integers(-63, 64)), None, None, None], mode_lf_delta=[int(rng.integers(-63, 64)), None, None, None])
            for m in f["mbs"]:
                m["uvmode"] = int(rng.integers(0, 4))
                if m["i4"]:
                    m["bmodes"] = [int(v) for v in rng.integers(0, 10, 16)]
                else:
                    m["ymode"] = int(rng.integers(0, 4))
            s = vr.write(f)
        streams.append(s)
    bad = {n // 2: ws.data_corrupt()[0][1], 33: ws.data_corrupt()[1][1]}
    for k, s in bad.items():
        streams[k] = s
    outs, status = g.jpeg_decode_ex(streams, adjust_orientation=False)
    assert status == [int(k in bad) for k in range(n)]
    for k, (s, o) in enumerate(zip(streams, outs)):
        if k not in bad:
            assert np.array_equal(o, _want(s, capi.RGB)), k


def _q127(rewritten):
    names, streams = rewritten
    return [(n, s) for n, s in zip(names, streams) if n.startswith("q127_")]


def test_q127_streams_alone_and_mixed(rewritten):
    """cv2 quality 90 / 100 streams re-quantised at index 127, where libwebp's full inverse DCT wraps in int16 lanes: alone, and in
    one batch with baseline and progressive JPEG, PNG and TIFF samples"""
    import gpu_helpers as g
    q = _q127(rewritten)
    assert len(q) == 16
    for n, s in q:
        outs, status = g.jpeg_decode_ex([s], output_type=capi.BGR, adjust_orientation=False)
        assert status == [0] and np.array_equal(outs[0], _want(s, capi.BGR)), n
    jpegs = [cv2.imencode(".jpg", g.synth_image(300, 420, 1))[1].tobytes(),
             cv2.imencode(".jpg", g.synth_image(120, 160, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()]
    png = ps.encode(ps.samples(40, 50, 2, 8, 80), 2, 8, filters="mixed")
    tif = cv2.imencode(".tiff", g.synth_image(240, 320, 4))[1].tobytes()
    solo = g.jpeg_decode(jpegs)[0]
    streams = [q[0][1], jpegs[0], png] + [s for _, s in q[1:8]] + [tif, jpegs[1]] + [s for _, s in q[8:]]
    outs, status = g.jpeg_decode(streams)
    assert status == [0] * len(streams)
    assert np.array_equal(outs[1], solo[0]) and np.array_equal(outs[11], solo[1])
    assert np.array_equal(outs[2], pngo.decode(png)[0]) and np.array_equal(outs[10], to.decode(tif)[0])
    for o, (n, s) in zip([outs[0]] + outs[3:10] + outs[12:], q):
        assert np.array_equal(o, _want(s, capi.RGB)), n
