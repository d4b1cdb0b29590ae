"""CPU tests of progressive JPEG under the scan scripts real encoders write (libjpeg, mozjpeg, jpegtran -scans, Photoshop): the test
encoder of jpeg_extreme_streams codes the coefficients of a baseline twin (cv2 at quality 30 / 90 / 100, 4-component Adobe streams,
random extreme planes) under each script of its catalogue.  libjpeg-turbo must decode every complete stream to the twin's picture (the
encoder is sound), and the product's planner and scan decoder, built for the host by tools/emul/jpeg_prog_emul.cc, must leave exactly
the coefficients expected() states after EVERY prefix of every script, with the wave count waves() states and the incomplete status
exactly where the progression is unfinished.  No GPU runs here."""
import numpy as np
import pytest

import jpeg_cmyk_oracle as cmyk_oracle
import jpeg_cmyk_streams as cs
import jpeg_extreme_streams as xs
from oracle import pyoracle as po
from test_jpeg_prog_cpu import decode, emul, multiscan_expected, synth  # noqa: F401  (emul: the fixture)

LAYOUTS = ["gray", "444", "422", "440", "420", "411", "ycck", "cmyk"]
# (h, w): 1x1, 1xN, Nx1, odd sizes, and widths at which luma's block row is shorter than mcux * hs (4:2:0 at 17, 4:1:1 at 40 / 97)
SIZES = [(1, 1), (1, 37), (29, 1), (17, 23), (33, 47), (97, 61), (24, 17), (16, 40)]
QUALITIES = [30, 90, 100]
SCRIPTS = {"spectral": xs.spectral, "simple": xs.simple, "deep3": xs.deep, "deep10": lambda n: xs.deep(n, 10),
           "per_component_dc": xs.per_component_dc, "subset_dc": xs.subset_dc, "single_coefficient": xs.single_coefficient,
           "reordered": xs.reordered, "restarts": xs.restarts, "table_slots": xs.table_slots,
           "repeated_dc_refinement": xs.repeated_dc_refinement}
NEEDS_CHROMA = {"subset_dc"}


def _qtables(stream):
    """the quantisation tables of a stream's DQT segments, {id: 64 values, natural order}"""
    out = {}
    for seg in cs._segments(stream)[0xDB]:
        o = 0
        while o < len(seg):
            pq, t = seg[o] >> 4, seg[o] & 15
            n = 128 if pq else 64
            zz = [(seg[o + 1 + 2 * k] << 8) | seg[o + 2 + 2 * k] if pq else seg[o + 1 + k] for k in range(64)]
            q = np.zeros(64, np.int64)
            q[cs._ZZ] = zz
            out[t] = q
            o += 1 + n
    return out


def source(layout, h, w, quality, seed):
    """A baseline stream and what the scripts code: dict(base, planes, qtabs, sampling, adobe, dqt16).  cv2 twins for the YCbCr / gray
    layouts, Photoshop's YCCK layout from jpeg_cmyk_streams, random extreme planes with (at quality 100) 16-bit DQT for CMYK."""
    import cv2
    if layout == "ycck":
        base = cs.photoshop_ycck(h, w, seed, quality)
        tq = _qtables(base)
        return dict(base=base, planes=cmyk_oracle.coeffs(base), qtabs=[tq[0], tq[1], tq[1], tq[2]], sampling=xs.SAMPLINGS["ycck"],
                    adobe=2, dqt16=False)
    if layout == "cmyk":
        rng = np.random.default_rng(seed)
        dqt16 = quality == 100
        sampling = xs.SAMPLINGS["cmyk"]
        planes = xs.planes_for(rng, h, w, sampling)
        qtabs = [xs.extreme_qtab(rng, dqt16) for _ in sampling]
        return dict(base=xs.baseline(h, w, sampling, planes, qtabs, dqt16, adobe=0), planes=planes, qtabs=qtabs, sampling=sampling,
                    adobe=0, dqt16=dqt16)
    img = synth(h, w, seed)
    p = [cv2.IMWRITE_JPEG_QUALITY, quality]
    if layout == "gray":
        img = img[..., 0]
    else:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR_" + layout)]
    base = cv2.imencode(".jpg", img, p)[1].tobytes()
    info = po.jpeg_info(base)
    n = info["ncomp"]
    tq = _qtables(base)
    return dict(base=base, planes=po.jpeg_coeffs(base)[:n], qtabs=[tq[min(c, 1)] for c in range(n)],
                sampling=[(info["hs"][c], info["vs"][c]) for c in range(n)], adobe=None, dqt16=False)


def encode(src, h, w, script, wide=False, rst=0, **kw):
    return xs.progressive(h, w, src["sampling"], src["planes"], src["qtabs"], src["dqt16"], wide, rst, src["adobe"], script, **kw)


def cases():
    """every script meets every layout: (name, layout, h, w, quality, wide) -- a seeded walk over sizes and qualities"""
    out = []
    for i, name in enumerate(SCRIPTS):
        for j, layout in enumerate(LAYOUTS):
            if name in NEEDS_CHROMA and layout == "gray":
                continue
            h, w = SIZES[(3 * i + j) % len(SIZES)]
            out.append((name, layout, h, w, QUALITIES[(i + 2 * j) % 3], name == "table_slots" and j % 2 == 1))
    return out


def imdecode(s):
    import cv2
    return cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_UNCHANGED)


def check_prefixes(lib, stream, src, h, w, script):
    """the host build after every prefix of the script: coefficients, wave count, incomplete status"""
    ncomp = len(src["sampling"])
    for k in range(1, len(script) + 1):
        cut = xs.prefix(stream, k)
        rc, got, info = decode(lib, cut)
        assert rc == 0, (k, rc)
        assert info["nscans"] == k and info["nwaves"] == xs.waves(script[:k]), (k, info)
        assert info["truncated"] == (not xs.complete(script, ncomp, k)), (k, info)
        want = xs.expected(h, w, src["sampling"], src["planes"], script, k)
        assert np.array_equal(got, want), (k, np.argwhere(got != want)[:4])


@pytest.mark.parametrize("name,layout,h,w,quality,wide", cases())
def test_script_against_libjpeg_and_the_statement(emul, name, layout, h, w, quality, wide):
    seed = 1000 + 37 * list(SCRIPTS).index(name) + LAYOUTS.index(layout)
    src = source(layout, h, w, quality, seed)
    script = SCRIPTS[name](len(src["sampling"]))
    stream = encode(src, h, w, script, wide)
    assert np.array_equal(imdecode(stream), imdecode(src["base"])), "the test encoder disagrees with libjpeg-turbo"
    check_prefixes(emul, stream, src, h, w, script)


def test_eob_runs_end_at_restart_markers(emul):
    """runs sent longer than their restart interval: the decoder drops what is left of a run at the marker, as libjpeg does"""
    for k, (layout, h, w) in enumerate([("420", 33, 47), ("gray", 97, 61), ("422", 17, 23), ("ycck", 24, 17)]):
        src = source(layout, h, w, 90, 90 + k)
        script = xs.restarts(len(src["sampling"]))
        stream = encode(src, h, w, script, overlong_runs=True)
        assert stream != encode(src, h, w, script)
        assert np.array_equal(imdecode(stream), imdecode(src["base"])), layout
        check_prefixes(emul, stream, src, h, w, script)


def test_long_codes_are_long():
    """the skewed tables put the rare symbols on codes longer than the decoder's 8-bit lookup, up to the 16-bit limit"""
    src = source("420", 97, 61, 90, 5)
    s = encode(src, 97, 61, xs.table_slots(3), wide=True)
    longest = [max(l for l in range(1, 17) if seg[l]) for _, m, seg in xs.segments(s) if m == 0xC4]
    assert max(longest) == 16 and sum(l > 8 for l in longest) >= 6, longest


def test_sequential_subset_scans(emul):
    """a SEQUENTIAL frame coded as Y + Cb in one scan and Cr (and K) in another: was refused, must decode to the twin"""
    for k, (layout, h, w) in enumerate([("420", 33, 47), ("444", 17, 23), ("422", 97, 61), ("411", 16, 40), ("ycck", 24, 17),
                                        ("cmyk", 29, 1)]):
        src = source(layout, h, w, 90, 70 + k)
        script = xs.sequential_subset(len(src["sampling"]))
        stream = encode(src, h, w, script, sof=0xC1 if src["dqt16"] else 0xC0)
        assert np.array_equal(imdecode(stream), imdecode(src["base"])), layout
        check_prefixes(emul, stream, src, h, w, script)
    # one scan per component: the statement agrees with multiscan_expected of test_jpeg_prog_cpu
    src = source("420", 33, 47, 90, 3)
    per = [xs.Scan((c,), 0, 63, 0, 0) for c in range(3)]
    stream = encode(src, 33, 47, per, sof=0xC0)
    _, _, blk = xs._geometry(33, 47, src["sampling"])
    want = multiscan_expected(src["base"], [b[0] for b in blk], [b[1] for b in blk])
    assert np.array_equal(xs.expected(33, 47, src["sampling"], src["planes"], per), want)
    assert np.array_equal(decode(emul, stream)[1], want)


def test_maximum_eob_runs(emul):
    """a flat 2048 x 2048 gray image: every AC scan is EOB runs of 32767, 32767 and 2 blocks, refinements included"""
    import cv2
    img = np.full((2048, 2048), 77, np.uint8)
    base = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
    src = dict(base=base, planes=po.jpeg_coeffs(base)[:1], qtabs=[_qtables(base)[0]], sampling=[(1, 1)], adobe=None, dqt16=False)
    script = xs.simple(1)
    stream = encode(src, 2048, 2048, script)
    assert np.array_equal(imdecode(stream), imdecode(base))
    rc, got, info = decode(emul, stream)
    assert rc == 0 and info["truncated"] == 0 and np.array_equal(got, xs.expected(2048, 2048, [(1, 1)], src["planes"], script))


def late_dqt(layout="420", h=33, w=47, seed=8):
    """per_component_dc() with the tables of components 1 and 2 in a DQT after the first scan: table 1 is defined there for the first
    time, table 2 (already in the frame header, with wrong values) redefined; then table 0, already latched by component 0, redefined
    with wrong values in front of the last scan.  libjpeg latches each component's table when its first scan starts."""
    src = source(layout, h, w, 90, seed)
    n = len(src["sampling"])
    bogus = np.arange(64) % 7 + 40
    script = xs.per_component_dc(n)
    script[1] = script[1]._replace(dqt={c: src["qtabs"][c] for c in range(1, n)})
    script[-1] = script[-1]._replace(dqt={0: bogus})
    qhead = {0: src["qtabs"][0], 2: bogus}
    return src, encode(src, h, w, script, qhead=qhead), script


def test_late_dqt_latches_like_libjpeg(emul):
    import ctypes as C
    for layout in ("420", "ycck"):
        src, stream, script = late_dqt(layout)
        assert np.array_equal(imdecode(stream), imdecode(src["base"])), layout
        b = np.frombuffer(stream, np.uint8)
        qt = np.zeros((4, 64), np.uint16)
        assert emul.emul_jpeg_prog_quant(b.ctypes.data_as(C.c_void_p), C.c_size_t(b.size), qt.ctypes.data_as(C.c_void_p)) == 0
        for c, q in enumerate(src["qtabs"]):
            assert np.array_equal(qt[c], q), (layout, c)
    # a table that no DQT defines before its component's first scan is refused as bad data
    src = source("420", 17, 23, 90, 9)
    stream = encode(src, 17, 23, xs.per_component_dc(3), qhead={0: src["qtabs"][0], 1: src["qtabs"][1]})
    assert decode(emul, stream)[0] == 4


def test_scan_limit(emul):
    src = source("444", 17, 23, 90, 12)
    ok = xs.scan_limit(1024)
    assert len(ok) == 1024
    s = encode(src, 17, 23, ok)
    assert np.array_equal(imdecode(s), imdecode(src["base"]))
    rc, got, info = decode(emul, s)
    assert rc == 0 and info["nscans"] == 1024 and info["truncated"] == 0 and info["nwaves"] == xs.waves(ok)
    assert np.array_equal(got, xs.expected(17, 23, src["sampling"], src["planes"], ok))
    over = xs.scan_limit(1025)
    assert len(over) == 1025 and decode(emul, encode(src, 17, 23, over))[0] == 2          # DALIB200_ERROR_UNSUPPORTED


def test_malformed_successive_approximation_is_bad_data(emul):
    src = source("420", 17, 23, 90, 13)
    for ah, al in ((2, 0), (3, 1), (1, 1)):
        script = xs.deep(3, 2)
        script[5] = script[5]._replace(ah=ah, al=al)
        assert decode(emul, encode(src, 17, 23, script))[0] == 4, (ah, al)
