"""-m gpu parity tests for the JPEG decoder: CUDA path (through the C-ABI) vs the oracle / libjpeg-turbo.
Bit-exact on every byte (integer pipeline)."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


def _enc(img, q=90, ss=None, rst=0):
    import cv2
    params = [cv2.IMWRITE_JPEG_QUALITY, q]
    if ss is not None:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, ss]
    if rst:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    ok, enc = cv2.imencode(".jpg", img, params)
    assert ok
    return enc.tobytes()


def test_golden_libjpeg_turbo(golden_dir):
    import gpu_helpers as g
    gz = np.load(os.path.join(golden_dir, "jpeg_cv2.npz"))
    n = len([k for k in gz.files if k.startswith("enc_")])
    streams = [gz[f"enc_{i}"].tobytes() for i in range(n)]
    outs, status = g.jpeg_decode(streams)
    assert status == [0] * n
    for i in range(n):
        assert np.array_equal(outs[i], gz[f"dec_{i}"]), f"golden case {i}"


def test_huffman_stage_coefficients_match_oracle():
    import gpu_helpers as g
    import cv2
    streams = [_enc(g.synth_image(136, 200, 3), 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420),
               _enc(g.synth_image(97, 61, 4), 50, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444),
               _enc(g.synth_image(480, 640, 5), 95, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420)]
    outs, status, plan = g.jpeg_decode(streams, want_coefs=True)
    assert status == [0, 0, 0]
    for si, s in enumerate(streams):
        comps = po.jpeg_coeffs(s)
        info = po.jpeg_info(s)
        hs, vs, mcux, mcuy = info["hs"], info["vs"], info["mcux"], info["mcuy"]
        # oracle layout: per component [bh][bw][64] -> MCU order
        blocks = []
        for my in range(mcuy):
            for mx in range(mcux):
                for c in range(info["ncomp"]):
                    for v in range(vs[c]):
                        for h in range(hs[c]):
                            blocks.append(comps[c][my * vs[c] + v, mx * hs[c] + h])
        want = np.stack(blocks).reshape(-1)
        got = g.jpeg_coefs(plan, si, want.size)
        assert np.array_equal(got, want), f"coefficients of stream {si}"


def test_all_samplings_qualities_sizes_vs_oracle():
    import gpu_helpers as g
    import cv2
    ss = [cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
          cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411]
    streams = []
    for hw in [(480, 640), (33, 47), (17, 16), (8, 8), (1, 1), (250, 3), (3, 250), (100, 101), (9, 5), (2, 2), (260, 517)]:
        for s in ss:
            for q in (30, 90, 100):
                streams.append(_enc(g.synth_image(hw[0], hw[1], hw[0] * 7 + hw[1] + q), q, s))
    outs, status = g.jpeg_decode(streams)
    assert all(s == 0 for s in status)
    for s, o in zip(streams, outs):
        assert np.array_equal(o, po.jpeg_decode(s)), po.jpeg_info(s)


def test_restart_intervals_and_gray():
    import gpu_helpers as g
    import cv2
    streams = []
    for rst in (1, 3, 7, 40):
        for s in (cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444):
            streams.append(_enc(g.synth_image(150, 210, rst), 85, s, rst))
    streams.append(_enc(g.synth_image(123, 77, 9)[..., 0], 85))          # grayscale JPEG -> RGB
    streams.append(_enc(g.synth_image(64, 64, 10)[..., 0], 70, rst=2))
    outs, status = g.jpeg_decode(streams)
    assert all(s == 0 for s in status)
    for s, o in zip(streams, outs):
        assert np.array_equal(o, po.jpeg_decode(s)), po.jpeg_info(s)


def test_output_types_and_box_upsampling():
    import gpu_helpers as g
    import cv2
    s = _enc(g.synth_image(90, 130, 11), 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420)
    rgb = po.jpeg_decode(s)
    (bgr,), _ = g.jpeg_decode([s], capi.BGR)
    assert np.array_equal(bgr, rgb[..., ::-1])
    (gray,), _ = g.jpeg_decode([s], capi.GRAY)
    assert np.array_equal(gray[..., 0], cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_GRAYSCALE))
    (box,), _ = g.jpeg_decode([s], capi.RGB, fancy=False)
    assert np.array_equal(box, po.jpeg_decode(s, fancy=False))


def test_1080p_batch_and_plan_reuse():
    """C2-sized images, batch of 6, plan reused for a second (different) batch."""
    import gpu_helpers as g
    plan = capi.Plan("Jpeg", 8)
    for base in (0, 100):
        streams = [_enc(g.synth_image(1080, 1920, base + i), 90) for i in range(6)]
        outs, status = g.jpeg_decode(streams, plan=plan)
        assert status == [0] * 6
        for s, o in zip(streams, outs):
            assert np.array_equal(o, po.jpeg_decode(s))


def test_truncated_stream_is_flagged_not_crashing():
    import gpu_helpers as g
    s = _enc(g.synth_image(200, 300, 12), 90)
    cut = s[: len(s) // 2]
    outs, status = g.jpeg_decode([cut, s])
    assert status[0] == 1 and status[1] == 0
    assert np.array_equal(outs[1], po.jpeg_decode(s))


def test_unsupported_streams_fail_loudly():
    import gpu_helpers as g
    import cv2
    img = g.synth_image(64, 64, 13)
    ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])
    arith = bytearray(enc.tobytes())
    arith[arith.find(b"\xff\xc0") + 1] = 0xC9           # SOF9: arithmetic coding (progressive streams are decoded: test_zzy_c_gpu_jpeg_multiscan.py)
    with pytest.raises(capi.DaliB200Error, match="not supported"):
        g.jpeg_decode([bytes(arith)])
    with pytest.raises(capi.DaliB200Error):
        g.jpeg_decode([b"\xff\xd8\xff\xd9"])


def test_mixed_huffman_tables_and_extreme_content():
    """One batch mixing the standard tables with per-image OPTIMISED tables (several table sets: the grid-wide
    synchronisation rounds keep only one set in shared memory), flat images (one byte per block: thousands of blocks per
    subsequence), noise at q100 (long codes, blocks longer than a subsequence), tiny and restart-interval streams."""
    import cv2
    import gpu_helpers as g
    rng = np.random.default_rng(21)
    imgs = [g.synth_image(300, 420, 30), g.synth_image(211, 333, 31),
            np.full((256, 384, 3), 128, np.uint8), np.zeros((64, 1024, 3), np.uint8),
            rng.integers(0, 256, (120, 200, 3)).astype(np.uint8), rng.integers(0, 256, (64, 64, 3)).astype(np.uint8),
            g.synth_image(17, 9, 32), g.synth_image(640, 640, 33)]
    streams = []
    for i, im in enumerate(imgs):
        params = [cv2.IMWRITE_JPEG_QUALITY, [90, 75, 90, 50, 100, 98, 90, 85][i]]
        if i % 2 == 1:
            params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
        if i == 7:
            params += [cv2.IMWRITE_JPEG_RST_INTERVAL, 3]
        if i == 4:
            params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]
        ok, enc = cv2.imencode(".jpg", im, params)
        assert ok
        streams.append(enc.tobytes())
    for order in (list(range(8)), [7, 5, 3, 1, 6, 4, 2, 0]):
        outs, status = g.jpeg_decode([streams[k] for k in order])
        assert status == [0] * 8
        for k, o in zip(order, outs):
            assert np.array_equal(o, po.jpeg_decode(streams[k])), f"image {k}"


def test_decode_is_deterministic_over_repeated_batches():
    """The self-synchronisation uses atomics for its work lists; the RESULT must not depend on their order."""
    import gpu_helpers as g
    streams = [_enc(g.synth_image(540, 960, 50 + i), 90) for i in range(24)]
    want = [po.jpeg_decode(s) for s in streams]
    plan = capi.Plan("Jpeg", 24)
    for rep in range(5):
        outs, status = g.jpeg_decode(streams, plan=plan)
        assert status == [0] * 24
        for i, (o, w) in enumerate(zip(outs, want)):
            assert np.array_equal(o, w), (rep, i)


# ------------------------------------------------------------------------------------------------------------------
# decoder variants (SURVEY 8 a2 / f1): region of interest, EXIF orientation, output_type / dtype conversion
def _variant_streams():
    import cv2
    import gpu_helpers as g
    return [_enc(g.synth_image(203, 310, 11), 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420),
            _enc(g.synth_image(97, 131, 12), 75, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444),
            _enc(g.synth_image(160, 96, 13), 85, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422),
            _enc(g.synth_image(480, 640, 14), 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, rst=8),
            _enc(g.synth_image(120, 200, 15)[..., 0], 90)]                                        # grayscale JPEG


def test_roi_decode_equals_crop_of_full_decode():
    import gpu_helpers as g
    streams = _variant_streams()
    full = [po.jpeg_decode(s) for s in streams]
    rng = np.random.default_rng(5)
    for rep in range(6):
        rois = []
        for f in full:
            H, W = f.shape[:2]
            if rep == 0:
                rois.append((0, 0, W, H))                                 # whole image through the ROI path
            elif rep == 1:
                rois.append((8, 3, min(W, 8 + 64), min(H, 3 + 40)))       # 8-aligned left edge: direct window
            else:
                x0, y0 = int(rng.integers(0, W - 1)), int(rng.integers(0, H - 1))
                rois.append((x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1))))
        for ot in (capi.RGB, capi.BGR, capi.GRAY):
            outs, status = g.jpeg_decode_ex(streams, output_type=ot, rois=rois)
            assert status == [0] * len(streams)
            for i, (f, r) in enumerate(zip(full, rois)):
                want = f[r[1]:r[3], r[0]:r[2]]
                if ot == capi.BGR:
                    want = want[..., ::-1]
                elif ot == capi.GRAY:
                    want = g.jpeg_decode([streams[i]], output_type=capi.GRAY)[0][0][r[1]:r[3], r[0]:r[2]]
                assert np.array_equal(outs[i], want), f"rep {rep} type {ot} sample {i} roi {r}"


def test_exif_orientation_matches_libjpeg_consumers():
    import cv2
    import gpu_helpers as g
    base = _enc(g.synth_image(123, 200, 21), 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420)
    dec = po.jpeg_decode(base)
    streams = [po.with_exif_orientation(base, o) for o in range(1, 9)]
    outs, status = g.jpeg_decode_ex(streams, adjust_orientation=True)
    assert status == [0] * 8
    for o in range(1, 9):
        want = po.exif_transform(dec, o)
        assert np.array_equal(outs[o - 1], want), f"orientation {o}"
        cv = cv2.imdecode(np.frombuffer(streams[o - 1], np.uint8), cv2.IMREAD_COLOR)[..., ::-1]      # cv2 applies the EXIF tag
        assert np.array_equal(outs[o - 1], cv), f"orientation {o} vs cv2"
    raw, _ = g.jpeg_decode_ex(streams, adjust_orientation=False)
    for o in range(8):
        assert np.array_equal(raw[o], dec)
    # region of interest in oriented coordinates
    rois = []
    for o in range(1, 9):
        OH, OW = (200, 123) if o >= 5 else (123, 200)
        rois.append((5, 7, OW - 11, OH - 3))
    outs, _ = g.jpeg_decode_ex(streams, adjust_orientation=True, rois=rois)
    for o in range(1, 9):
        r = rois[o - 1]
        assert np.array_equal(outs[o - 1], po.exif_transform(dec, o)[r[1]:r[3], r[0]:r[2]]), f"orientation {o} + roi"


def test_output_type_and_dtype_conversion_match_reference_convert():
    """Every output type and dtype against the float32 and float64 forms of the convert functors (tests/pointwise_ref.py) and, where
    present, the reference's own functors (oracle/_ref)."""
    import gpu_helpers as g
    import pointwise_ref as pr
    ref = po.have_ref()
    streams = _variant_streams()
    full = [po.jpeg_decode(s) for s in streams]
    gray = [g.jpeg_decode([s], output_type=capi.GRAY)[0][0] for s in streams]
    for ot, it in ((capi.RGB, po.IT_RGB), (capi.BGR, po.IT_BGR), (capi.YCbCr, po.IT_YCBCR), (capi.GRAY, po.IT_GRAY)):
        for dt, fl in ((capi.UINT8, False), (capi.FLOAT, True)):
            outs, status = g.jpeg_decode_ex(streams, output_type=ot, dtype=dt)
            assert status == [0] * len(streams)
            for i in range(len(streams)):
                src = gray[i] if ot == capi.GRAY else full[i]           # GRAY is decoded as the Y plane (image_decoder.h:537-540)
                pr.check_decoder_output(outs[i], src, ot, fl, f"type {ot} dtype {dt} sample {i}")
                if ref:
                    assert np.array_equal(outs[i], po.ref_decoder_convert(src, it, fl)), f"type {ot} dtype {dt} sample {i}"
    # everything at once: orientation + ROI + YCbCr float
    s6 = po.with_exif_orientation(streams[0], 6)
    win = np.ascontiguousarray(po.exif_transform(full[0], 6)[9:260, 3:150])
    out, status = g.jpeg_decode_ex([s6], output_type=capi.YCbCr, dtype=capi.FLOAT, rois=[(3, 9, 150, 260)])
    assert status == [0]
    pr.check_decoder_output(out[0], win, capi.YCbCr, True, "orientation 6 + roi")
    if ref:
        assert np.array_equal(out[0], po.ref_decoder_convert(win, po.IT_YCBCR, True))


def test_truncated_stream_status_gray_tail_and_pipeline_error():
    """A stream cut in the middle of the scan: status 1, everything decoded before the damage is intact, the MCU rows well behind it
    are mid-gray (libjpeg leaves all-zero blocks there: jdhuff.c insufficient_data), and a pipeline raises at run() -- the status
    words travel with the outputs (no extra synchronisation)."""
    import cv2
    import gpu_helpers as g
    from dali_b200 import fn, pipeline_def
    good = _enc(g.synth_image(240, 320, 31), 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420)
    full = po.jpeg_decode(good)
    cut = good[: len(good) * 6 // 10]
    outs, status = g.jpeg_decode([cut, good])
    assert status == [1, 0]
    assert np.array_equal(outs[1], full)
    assert np.array_equal(outs[0][:96], full[:96])                        # 60 % of the bytes cover more than 40 % of the rows
    assert (outs[0][-48:] == 128).all()                                   # zero coefficients, DC 0 -> Y = Cb = Cr = 128 -> RGB gray
    streams = [np.frombuffer(cut, np.uint8), np.frombuffer(good, np.uint8)]

    @pipeline_def(batch_size=2, num_threads=1, device_id=0, prefetch_queue_depth=1)
    def pipe():
        return fn.decoders.image(fn.external_source(source=lambda i: streams), device="mixed")
    p = pipe()
    p.build()
    with pytest.raises(RuntimeError, match="Failed to decode sample #0"):
        p.run()


def test_direct_upload_from_page_locked_sources():
    """Streams in page-locked memory that the caller declares stable are copied by DMA straight from the caller's buffers (one
    batched submission, or one copy per sample when the driver lacks the batch call); pageable or undeclared sources go through
    the pinned staging buffer.  All three routes decode to the same bytes."""
    import cv2
    import gpu_helpers as g
    streams = []
    for i, (h, w) in enumerate(((300, 420), (64, 64), (481, 641), (200, 333))):
        ok, enc = cv2.imencode(".jpg", g.synth_image(h, w, 70 + i), [cv2.IMWRITE_JPEG_QUALITY, 85])
        streams.append(np.ascontiguousarray(enc.ravel()))
    a, sa, pa = g.jpeg_decode_ex(streams, want_upload_path=True)
    b, sb, pb = g.jpeg_decode_ex(streams, pinned=True, want_upload_path=True)
    assert pa == 0 and pb in (1, 2) and sa == sb == [0] * len(streams)
    for x, y, s in zip(a, b, streams):
        assert np.array_equal(x, y) and np.array_equal(x, po.jpeg_decode(s.tobytes()))
