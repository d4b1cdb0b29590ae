"""-m gpu: the entropy decode at every subsequence size.

The planner picks the subsequence size from the batch's entropy-coded bytes (>= ~200 k subsequences per batch), so small test
batches always run at 32 bytes; DALIB200_JPEG_SUBSEQ_BYTES pins the size.  The same streams are decoded at 32, 64 and 128 bytes
and compared with the oracle: quantised coefficients and pixels, bit-exact."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import pyoracle as po  # noqa: E402


def _enc(img, q, ss=None, rst=0, optimize=False):
    import cv2
    params = [cv2.IMWRITE_JPEG_QUALITY, q]
    if ss is not None:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, ss]
    if rst:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if optimize:
        params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
    ok, enc = cv2.imencode(".jpg", img, params)
    assert ok
    return enc.tobytes()


def _streams():
    import cv2
    import gpu_helpers as g
    s420, s444 = cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444
    noise = np.random.default_rng(7).integers(0, 256, (96, 128, 3), dtype=np.uint8)
    return [
        _enc(noise, 100, s444),                                         # blocks longer than a 128-byte subsequence
        _enc(noise, 100, s420, optimize=True),
        _enc(g.synth_image(1080, 1920, 31), 90, s420),                   # the benchmark's shape
        _enc(g.synth_image(240, 320, 32), 90, s420, optimize=True),      # optimised tables next to standard ones: several table sets
        _enc(g.synth_image(200, 150, 33), 75, s444, optimize=True),
        _enc(g.synth_image(150, 210, 34), 85, s420, rst=3),              # restart intervals: many short units
        _enc(g.synth_image(150, 210, 35), 95, s444, rst=1),
        _enc(g.synth_image(16, 16, 36), 90, s420),                       # one MCU
        _enc(g.synth_image(8, 8, 37), 50, s444),
        _enc(g.synth_image(123, 77, 38)[..., 0], 85),                    # grayscale
    ]


def _mcu_order_coefs(s):
    comps = po.jpeg_coeffs(s)
    info = po.jpeg_info(s)
    hs, vs, mcux, mcuy = info["hs"], info["vs"], info["mcux"], info["mcuy"]
    blocks = []
    for my in range(mcuy):
        for mx in range(mcux):
            for c in range(info["ncomp"]):
                for v in range(vs[c]):
                    for h in range(hs[c]):
                        blocks.append(comps[c][my * vs[c] + v, mx * hs[c] + h])
    return np.stack(blocks).reshape(-1)


@pytest.mark.parametrize("sub_bytes", [32, 64, 128])
def test_every_subsequence_size_matches_oracle(sub_bytes, monkeypatch):
    import gpu_helpers as g
    streams = _streams()
    monkeypatch.setenv("DALIB200_JPEG_SUBSEQ_BYTES", str(sub_bytes))
    outs, status, plan = g.jpeg_decode(streams, want_coefs=True)
    assert status == [0] * len(streams)
    for si, s in enumerate(streams):
        want = _mcu_order_coefs(s)
        assert np.array_equal(g.jpeg_coefs(plan, si, want.size), want), f"coefficients of stream {si} at {sub_bytes} B"
        assert np.array_equal(outs[si], po.jpeg_decode(s)), f"pixels of stream {si} at {sub_bytes} B"
