"""-m gpu: WebP streams whose VP8 data runs past the VP8 chunk (into chunks or bytes behind it) and the EXIF orientation rules of
tests/webp_streams.py, decoded by the library against cv2.imdecode."""
import cv2
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import webp_streams as ws  # noqa: E402


def test_edge_streams_and_orientations():
    import gpu_helpers as g
    edge = [s for _, s in ws.edge_decodable()]
    outs, status = g.jpeg_decode_ex(edge, adjust_orientation=False)
    assert status == [0] * len(edge)
    for o, s in zip(outs, edge):
        assert np.array_equal(o, ws.decode(s, cv2.IMREAD_COLOR | cv2.IMREAD_IGNORE_ORIENTATION)[..., ::-1])
    cases = ws.orientation_cases()
    outs, status = g.jpeg_decode_ex([s for _, s in cases], adjust_orientation=True)
    assert status == [0] * len(cases)
    for o, (name, s) in zip(outs, cases):
        assert np.array_equal(o, ws.decode(s)[..., ::-1]), name
