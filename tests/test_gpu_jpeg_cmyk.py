"""-m gpu tests of 4-component (CMYK / YCCK) JPEG in the decoder: bit-exact against cv2.imdecode (the Pillow fixtures of
tests/golden/jpeg_cmyk.npz carry its decodes; the Photoshop-layout YCCK streams of tests/jpeg_cmyk_streams.py are decoded by cv2 here)
and, for box upsampling, against the oracle of tests/jpeg_cmyk_oracle.c, which the CPU tests pin to cv2.  Output types, regions of
interest, EXIF orientations, the multi-scan path, a batch mixed with every other decode path, truncation, and the pipeline operator."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
import pointwise_ref as pr  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


def _fixtures(golden_dir):
    gz = np.load(os.path.join(golden_dir, "jpeg_cmyk.npz"))
    n = len([k for k in gz.files if k.startswith("enc_")])
    return [dict(name=str(gz[f"name_{i}"]), enc=gz[f"enc_{i}"].tobytes(), color=gz[f"color_{i}"], gray=gz[f"gray_{i}"]) for i in range(n)]


def _cv2(s):
    import cv2
    a = np.frombuffer(s, np.uint8)
    return cv2.imdecode(a, cv2.IMREAD_COLOR)[..., ::-1], cv2.imdecode(a, cv2.IMREAD_GRAYSCALE)


def _enc(img, q=90, ss=None):
    import cv2
    p = [cv2.IMWRITE_JPEG_QUALITY, q] + ([cv2.IMWRITE_JPEG_SAMPLING_FACTOR, ss] if ss is not None else [])
    return cv2.imencode(".jpg", img, p)[1].tobytes()


def _check_types(streams, rgb, gray, what):
    import gpu_helpers as g
    for ot in (capi.RGB, capi.BGR, capi.GRAY):
        outs, status = g.jpeg_decode(streams, output_type=ot)
        assert status == [0] * len(streams)
        for i, o in enumerate(outs):
            want = rgb[i][..., ::-1] if ot == capi.BGR else gray[i][..., None] if ot == capi.GRAY else rgb[i]
            assert np.array_equal(o, want), f"{what[i]} type {ot}"


def test_pillow_fixtures_rgb_bgr_gray_and_box(golden_dir):
    """Every fixture -- CMYK, YCCK, no Adobe marker; 4:4:4, h2v1, h2v2; baseline and progressive (the multi-scan path) -- in one batch."""
    import gpu_helpers as g
    import jpeg_cmyk_oracle as cmyk_oracle
    fx = _fixtures(golden_dir)
    streams = [f["enc"] for f in fx]
    _check_types(streams, [f["color"][..., ::-1] for f in fx], [f["gray"] for f in fx], [f["name"] for f in fx])
    base = [f for f in fx if "_base_" in f["name"]]
    outs, status = g.jpeg_decode([f["enc"] for f in base], fancy=False)
    assert status == [0] * len(base)
    for f, o in zip(base, outs):
        assert np.array_equal(o, cmyk_oracle.decode(f["enc"], fancy=False)), f["name"]


def test_photoshop_ycck_layout_with_and_without_restarts():
    from jpeg_cmyk_streams import photoshop_ycck
    cases = [(1080, 1920, 0, 2), (1080, 1920, 7, 2), (1080, 1920, 0, 0), (17, 9, 0, 2), (61, 77, 1, 2), (250, 3, 0, 2), (3, 250, 2, 0),
             (480, 640, 40, 2), (1, 1, 0, 2)]
    streams = [photoshop_ycck(h, w, 10 + k, rst=rst, transform=t) for k, (h, w, rst, t) in enumerate(cases)]
    dec = [_cv2(s) for s in streams]
    _check_types(streams, [d[0] for d in dec], [d[1] for d in dec], cases)


def test_multiscan_four_component_streams(golden_dir):
    """Progressive CMYK / YCCK (Pillow) and sequential frames coded one scan per component, through the multi-scan entropy stage."""
    from jpeg_cmyk_streams import photoshop_ycck
    from jpeg_cmyk_streams import one_scan_per_component
    fx = _fixtures(golden_dir)
    prog = [f["enc"] for f in fx if "_prog_" in f["name"] and f["name"].endswith(("61x77", "250x3"))]
    src = [f["enc"] for f in fx if "_base_" in f["name"] and f["name"].endswith("61x77")] + [photoshop_ycck(120, 200, 3),
                                                                                              photoshop_ycck(240, 320, 4)]
    multi = [one_scan_per_component(s, rst)[0] for s in src for rst in (0, 6)]
    streams = prog + multi
    dec = [_cv2(s) for s in streams]
    _check_types(streams, [d[0] for d in dec], [d[1] for d in dec], list(range(len(streams))))


def test_mixed_batch_equals_solo_decodes():
    """CMYK / YCCK beside 1080p 4:2:0 (idct_color_420), 4:4:4 (color_fast_kernel) and grayscale streams, in two orders: every sample
    equals its decode alone, so the per-path work lists do not interfere."""
    import cv2
    import gpu_helpers as g
    from jpeg_cmyk_streams import photoshop_ycck
    streams = [photoshop_ycck(1080, 1920, 20), _enc(g.synth_image(1080, 1920, 21)), photoshop_ycck(97, 131, 22, rst=3, transform=0),
               _enc(g.synth_image(300, 420, 23), 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444), _enc(g.synth_image(123, 77, 24)[..., 0]),
               photoshop_ycck(480, 640, 25), _enc(g.synth_image(1080, 1920, 26)), photoshop_ycck(33, 47, 27, transform=0)]
    for ot in (capi.RGB, capi.GRAY):
        solo = [g.jpeg_decode([s], output_type=ot)[0][0] for s in streams]
        for order in (list(range(len(streams))), [7, 5, 3, 1, 6, 4, 2, 0]):
            outs, status = g.jpeg_decode([streams[k] for k in order], output_type=ot)
            assert status == [0] * len(streams)
            for k, o in zip(order, outs):
                assert np.array_equal(o, solo[k]), (ot, order, k)
    for k in (0, 2, 5, 7):
        assert np.array_equal(solo[k][..., 0], _cv2(streams[k])[1])


def test_roi_windows_equal_crops_of_the_full_decode(golden_dir):
    import gpu_helpers as g
    from jpeg_cmyk_streams import photoshop_ycck
    fx = _fixtures(golden_dir)
    streams = [f["enc"] for f in fx if f["name"] in ("cmyk_s2_base_61x77", "ycck_s1_base_61x77", "noadobe_s0_prog_61x77")]
    streams += [photoshop_ycck(203, 310, 30, rst=4), photoshop_ycck(1080, 1920, 31, transform=0)]
    full = {ot: g.jpeg_decode(streams, output_type=ot)[0] for ot in (capi.RGB, capi.BGR, capi.GRAY)}
    assert np.array_equal(full[capi.RGB][3], _cv2(streams[3])[0])
    rng = np.random.default_rng(6)
    for rep in range(5):
        rois = []
        for f in full[capi.RGB]:
            H, W = f.shape[:2]
            x0 = int(rng.integers(1, min(W - 1, 60)))                    # left edge inside an MCU (never a multiple of 16 below)
            x0 += x0 % 16 == 0
            y0 = int(rng.integers(0, H - 1))
            rois.append((x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1))))
        for ot in (capi.RGB, capi.BGR, capi.GRAY):
            outs, status = g.jpeg_decode_ex(streams, output_type=ot, rois=rois)
            assert status == [0] * len(streams)
            for i, r in enumerate(rois):
                assert np.array_equal(outs[i], full[ot][i][r[1]:r[3], r[0]:r[2]]), (rep, ot, i, r)


def test_exif_orientations(golden_dir):
    import cv2
    import gpu_helpers as g
    from jpeg_cmyk_streams import photoshop_ycck
    for base in (photoshop_ycck(123, 200, 40), next(f["enc"] for f in _fixtures(golden_dir) if f["name"] == "cmyk_s2_base_61x77")):
        dec = _cv2(base)[0]
        streams = [po.with_exif_orientation(base, o) for o in range(1, 9)]
        outs, status = g.jpeg_decode_ex(streams, adjust_orientation=True)
        assert status == [0] * 8
        for o in range(1, 9):
            assert np.array_equal(outs[o - 1], po.exif_transform(dec, o)), f"orientation {o}"
            cv = cv2.imdecode(np.frombuffer(streams[o - 1], np.uint8), cv2.IMREAD_COLOR)[..., ::-1]      # cv2 applies the EXIF tag
            assert np.array_equal(outs[o - 1], cv), f"orientation {o} vs cv2"
        gray, _ = g.jpeg_decode_ex(streams, output_type=capi.GRAY, adjust_orientation=True)
        for o in range(1, 9):
            cv = cv2.imdecode(np.frombuffer(streams[o - 1], np.uint8), cv2.IMREAD_GRAYSCALE)
            assert np.array_equal(gray[o - 1][..., 0], cv), f"gray orientation {o} vs cv2"


def test_ycbcr_and_float_outputs(golden_dir):
    """As for 3-component streams: the post pass converts the RGB (GRAY) decode.  Compared with the float32 and float64 forms of the
    convert functors (tests/pointwise_ref.py) and, where present, the reference's own functors (oracle/_ref)."""
    import gpu_helpers as g
    from jpeg_cmyk_streams import photoshop_ycck
    fx = _fixtures(golden_dir)
    streams = [f["enc"] for f in fx if f["name"] in ("cmyk_s0_base_61x77", "ycck_s2_prog_61x77")] + [photoshop_ycck(97, 131, 50, rst=2)]
    full = [g.jpeg_decode([s])[0][0] for s in streams]
    gray = [g.jpeg_decode([s], output_type=capi.GRAY)[0][0] for s in streams]
    for i, s in enumerate(streams):
        assert np.array_equal(full[i], _cv2(s)[0]) and np.array_equal(gray[i][..., 0], _cv2(s)[1])
    ref = po.have_ref()
    for ot, it in ((capi.RGB, po.IT_RGB), (capi.BGR, po.IT_BGR), (capi.YCbCr, po.IT_YCBCR), (capi.GRAY, po.IT_GRAY)):
        for dt, fl in ((capi.UINT8, False), (capi.FLOAT, True)):
            outs, status = g.jpeg_decode_ex(streams, output_type=ot, dtype=dt)
            assert status == [0] * len(streams)
            for i in range(len(streams)):
                src = gray[i] if ot == capi.GRAY else full[i]
                pr.check_decoder_output(outs[i], src, ot, fl, f"type {ot} dtype {dt} sample {i}")
                if ref:
                    assert np.array_equal(outs[i], po.ref_decoder_convert(src, it, fl)), f"type {ot} dtype {dt} sample {i}"


def test_truncated_cmyk_stream_sets_its_status():
    import gpu_helpers as g
    from jpeg_cmyk_streams import photoshop_ycck
    good = photoshop_ycck(240, 320, 60)
    cut = good[: len(good) * 6 // 10]
    outs, status = g.jpeg_decode([cut, good])
    assert status == [1, 0]
    full = _cv2(good)[0]
    assert np.array_equal(outs[1], full)
    assert np.array_equal(outs[0][:96], full[:96])                        # 60 % of the bytes cover more than 40 % of the rows


def test_pipeline_decodes_a_batch_with_cmyk_files(golden_dir):
    """fn.decoders.image on a batch that mixes CMYK / YCCK files with ordinary ones: the same output as the per-sample decode."""
    import gpu_helpers as g
    from dali_b200 import fn, pipeline_def
    from jpeg_cmyk_streams import photoshop_ycck
    fx = _fixtures(golden_dir)
    raw = [_enc(g.synth_image(120, 160, 70)), next(f["enc"] for f in fx if f["name"] == "cmyk_s2_base_61x77"),
           photoshop_ycck(90, 130, 71), next(f["enc"] for f in fx if f["name"] == "ycck_s1_prog_17x9")]
    streams = [np.frombuffer(s, np.uint8) for s in raw]

    @pipeline_def(batch_size=len(streams), num_threads=1, device_id=0, prefetch_queue_depth=1)
    def pipe():
        return fn.decoders.image(fn.external_source(source=lambda i: streams), device="mixed")
    p = pipe()
    p.build()
    (out,) = p.run()
    got = out.as_cpu()
    for i, s in enumerate(raw):
        assert np.array_equal(got[i], g.jpeg_decode([s])[0][0]), i
        assert np.array_equal(got[i], _cv2(s)[0]), i
