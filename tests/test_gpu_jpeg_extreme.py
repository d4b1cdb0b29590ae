"""-m gpu tests of the JPEG decoder on streams whose IDCT values leave the range natural streams reach, and on damaged entropy data, against
cv2.imdecode directly (libjpeg-turbo with its x86 SIMD islow IDCT, whose 16-bit dataflow tests/jpeg_idct16.py states):
  - the extreme corpus of tests/jpeg_extreme_streams.py in RGB, BGR and GRAY through every reconstruction path -- the fused 4:2:0
    IDCT + colour kernel, IDCT + colour_fast (4:4:4, 4:2:2), the generic colour kernel (gray, 4:4:0, CMYK / YCCK), regions of interest,
    and the multi-scan stage (one scan per component, progressive); each batch holds blocks on which the 16-bit and the C arithmetic
    differ and launches its path's kernel;
  - damaged baseline, restart-interval and progressive streams: wherever the decoder reports status 0 and cv2 decodes, the bytes are
    equal (invalid Huffman codes take 17 bits, runs past coefficient 63 land on 63)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
import jpeg_cmyk_streams as cs  # noqa: E402
import jpeg_extreme_streams as xs  # noqa: E402
from jpeg_idct16 import idct16, idct_c  # noqa: E402


def _cv(s, ot):
    import cv2
    b = np.frombuffer(s, np.uint8)
    if ot == capi.GRAY:
        d = cv2.imdecode(b, cv2.IMREAD_GRAYSCALE)
        return None if d is None else d[..., None]
    d = cv2.imdecode(b, cv2.IMREAD_COLOR)
    return None if d is None else (d if ot == capi.BGR else d[..., ::-1])


def _differing_blocks(planes, qtabs):
    """blocks of the batch on which the two statements of the IDCT differ"""
    return sum(int((idct16(p.reshape(-1, 64), q) != idct_c(p.reshape(-1, 64), q)).any(axis=(1, 2)).sum()) for p, q in zip(planes, qtabs))


def _decode_profiled(streams, ot, rois=None):
    import gpu_helpers as g
    capi.profiling(True)
    try:
        capi.profiling_collect()
        outs, status = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False, rois=rois)
        names = [n for n, _ in capi.profiling_collect()]
    finally:
        capi.profiling(False)
    return outs, status, names


# path: (kernel that must run, [(layout, h, w)]); sizes are whole MCUs so that the progressive twins code every block
PATHS = {
    "idct_color_420": ("jpeg_idct_color", [("420", 272, 352), ("420", 48, 64), ("420", 32, 48)]),
    "idct_color_fast": ("jpeg_upsample_color", [("444", 64, 72), ("422", 56, 96)]),
    "color_generic": ("jpeg_upsample_color_generic", [("gray", 64, 80), ("440", 64, 56), ("cmyk", 40, 48), ("ycck", 48, 64)]),
}
VARIANTS = [(False, False, 0), (False, True, 3), (True, True, 0), (True, False, 7)]     # (16-bit DQT, wide tables, restart interval)


def _corpus(path, seed0=0):
    out = []
    for i, (layout, h, w) in enumerate(PATHS[path][1]):
        for j, (dqt16, wide, rst) in enumerate(VARIANTS):
            s, planes, q = xs.extreme_stream(seed0 + 100 * i + j, h, w, layout, dqt16, wide, rst)
            out.append((f"{layout}-{h}x{w}-dqt16={dqt16}-wide={wide}-rst={rst}", s, planes, q, (layout, h, w, dqt16, wide, rst)))
    return out


@pytest.mark.parametrize("path", list(PATHS))
def test_extreme_corpus_against_cv2(path):
    corpus = _corpus(path)
    assert _differing_blocks([p for c in corpus for p in c[2]], [q for c in corpus for q in c[3]]) > 100
    streams = [c[1] for c in corpus]
    for ot in (capi.RGB, capi.BGR, capi.GRAY):
        outs, status, names = _decode_profiled(streams, ot)
        assert status == [0] * len(streams)
        if ot != capi.GRAY or path == "color_generic":
            assert PATHS[path][0] in names, (path, ot, names)
        for (name, s, *_), o in zip(corpus, outs):
            assert np.array_equal(o, _cv(s, ot)), (path, ot, name)


def test_extreme_regions_of_interest_equal_crops():
    corpus = _corpus("idct_color_420", 7) + _corpus("idct_color_fast", 7) + _corpus("color_generic", 7)
    streams = [c[1] for c in corpus]
    rng = np.random.default_rng(4)
    for ot in (capi.RGB, capi.GRAY):
        full = [_cv(s, ot) for s in streams]
        rois = []
        for f in full:
            H, W = f.shape[:2]
            x0, y0 = int(rng.integers(0, W - 1)), int(rng.integers(0, H - 1))
            rois.append((x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1))))
        outs, status, names = _decode_profiled(streams, ot, rois)
        assert status == [0] * len(streams)
        if ot == capi.RGB:
            assert "jpeg_idct_color" in names, names
        for (name, *_), o, f, r in zip(corpus, outs, full, rois):
            assert np.array_equal(o, f[r[1]:r[3], r[0]:r[2]]), (ot, name, r)


def test_extreme_multiscan_against_cv2():
    """the same content as one scan per component (sequential frame) and as a progressive script: the multi-scan stage"""
    streams, planes, qtabs = [], [], []
    for i, (layout, h, w) in enumerate([("420", 48, 64), ("444", 32, 40), ("422", 32, 48), ("440", 48, 40), ("gray", 40, 56),
                                        ("cmyk", 32, 32), ("ycck", 32, 48)]):
        for j, (dqt16, wide, rst) in enumerate(VARIANTS):
            rng = np.random.default_rng(500 + 10 * i + j)
            sampling = xs.SAMPLINGS[layout]
            amax, dmax = (32767, 16383) if wide else (1023, 1023)
            p = xs.planes_for(rng, h, w, sampling, amax, dmax)
            q = [xs.extreme_qtab(rng, dqt16) for _ in sampling]
            adobe = {"cmyk": 0, "ycck": 2}.get(layout)
            streams.append(xs.progressive(h, w, sampling, p, q, dqt16, wide, rst, adobe))
            streams.append(cs.one_scan_per_component(xs.baseline(h, w, sampling, p, q, dqt16, wide, 0, adobe), rst)[0])
            planes += p
            qtabs += q
    assert _differing_blocks(planes, qtabs) > 100
    for ot in (capi.RGB, capi.BGR, capi.GRAY):
        outs, status, names = _decode_profiled(streams, ot)
        assert status == [0] * len(streams)
        assert "jpeg_prog_scan" in names, names
        for k, (s, o) in enumerate(zip(streams, outs)):
            assert np.array_equal(o, _cv(s, ot)), (ot, k)


@pytest.mark.parametrize("kind", ["gray", "color", "progressive"])
def test_damaged_streams_against_cv2(kind):
    import gpu_helpers as g
    if kind == "progressive":
        streams = xs.mutated(21, 500, progressive=True) + xs.mutated(22, 500, color=True, progressive=True)
    else:
        streams = xs.mutated(23 if kind == "gray" else 24, 900, color=kind == "color")
    checked = 0
    for ot in (capi.RGB, capi.GRAY):
        for i in range(0, len(streams), 100):
            chunk = streams[i:i + 100]
            outs, status = g.jpeg_decode_ex(chunk, output_type=ot, adjust_orientation=False)
            for k, (s, o, st) in enumerate(zip(chunk, outs, status)):
                want = _cv(s, ot)
                if st == 0 and want is not None:
                    assert np.array_equal(o, want), (kind, ot, i + k)
                    checked += ot == capi.RGB
    assert checked > 500, checked
