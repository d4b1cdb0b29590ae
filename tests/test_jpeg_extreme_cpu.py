"""JPEG reconstruction outside the range natural streams reach, and damaged entropy data, against cv2.imdecode (libjpeg-turbo with its
x86 SIMD islow IDCT), on the CPU:
  - the numpy 16-bit statement of that IDCT (tests/jpeg_idct16.py) equals cv2 on >= 10^5 random extreme blocks and on targeted blocks
    for each wrap, saturation and shortcut of the SIMD dataflow, and equals the C statement on every block of the natural corpora;
  - the oracle (oracle/jpeg_oracle.c) equals cv2 on the extreme corpus and on damaged baseline streams wherever its bit reader stayed
    inside the data, and the progressive scan decoder of the product (jpeg_prog_core.h, built for the host) does on damaged progressive
    streams;
  - each planted mistake -- the C IDCT, a 16-bit invalid code, a run past coefficient 63 that stops the block -- fails those comparisons."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import jpeg_cmyk_oracle as cmyk_oracle
import jpeg_cmyk_streams as cs
import jpeg_distort_cases as dc
import jpeg_extreme_streams as xs
from jpeg_idct16 import _pass16, idct16, idct_c, w16
from oracle import pyoracle as po

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def imdecode(s, flag):
    return cv2.imdecode(np.frombuffer(s, np.uint8), flag)


def to_image(blocks, bh, bw):
    """[bh * bw, 8, 8] blocks in raster order -> [8 bh, 8 bw] samples"""
    return blocks.reshape(bh, bw, 8, 8).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def block_diff(a, b):
    """per 8x8 block: any sample differs"""
    return (a != b).reshape(a.shape[0] // 8, 8, a.shape[1] // 8, 8).any(axis=(1, 3))


def gray_blocks(stream, plane, q):
    """(statement, C statement, cv2) of a grayscale extreme stream whose size is a whole number of blocks"""
    bh, bw = plane.shape[:2]
    flat = plane.reshape(-1, 64)
    return to_image(idct16(flat, q), bh, bw), to_image(idct_c(flat, q), bh, bw), imdecode(stream, cv2.IMREAD_GRAYSCALE)


# ---- the statement ---------------------------------------------------------------------------------------------------------------
def test_statement_equals_cv2_on_random_extreme_blocks():
    n = differ_c = 0
    for seed in range(100):
        wide, dqt16 = [(False, False), (True, False), (True, True), (False, True)][seed % 4]
        s, planes, q = xs.extreme_stream(seed, 256, 256, "gray", dqt16=dqt16, wide=wide, rst=[0, 1, 7][seed % 3])
        got16, gotc, want = gray_blocks(s, planes[0], q[0])
        assert np.array_equal(got16, want), (seed, block_diff(got16, want).sum())
        n += planes[0].shape[0] * planes[0].shape[1]
        differ_c += block_diff(gotc, want).sum()
    assert n >= 100_000
    assert differ_c > n // 2, differ_c          # the corpus is extreme: the C arithmetic misses most of its blocks


def _block(entries, q):
    b = np.zeros(64, np.int64)
    for (y, x), v in entries.items():
        b[y * 8 + x] = v
    return b, np.broadcast_to(np.asarray(q, np.int64), (64,)).copy()


def _per_column_shortcut(coef, q):
    """planted: the pass-1 shortcut decided per column instead of per block"""
    d = w16(coef * q).reshape(8, 8)
    ws = _pass16(d.T, 11).T
    skip = ~coef.reshape(8, 8)[1:].any(axis=0)
    ws[:, skip] = w16(d[0, skip] << 2)
    return (np.clip(_pass16(ws, 18), -128, 127) + 128).astype(np.uint8)


def _no_wrap_dequant(coef, q):
    """planted: 32-bit dequantisation, the rest of the 16-bit dataflow kept"""
    d = coef * q
    return idct16(np.clip(d, -32768, 32767), np.ones(64, np.int64)) if (np.abs(d) > 32767).any() else idct16(coef, q)


TARGETED = {
    # name: (block, quantisation, planted variant that must differ from cv2 on it)
    "coef*q wraps": (_block({(0, 0): 10, (0, 1): 300, (1, 0): -200}, 200), _no_wrap_dequant),
    "i0 + i4 wraps": (_block({(0, 0): 200, (4, 0): 200, (1, 1): 1}, 90), None),
    "i7 + i3 and i5 + i1 wrap": (_block({(0, 0): 5, (7, 0): 300, (3, 0): 300, (0, 5): 300, (0, 1): 300}, 60), None),
    "pass 1 saturates": (_block({(0, 0): 250, (1, 0): 250, (2, 0): 250}, 120), None),
    "pass 2 saturates": (_block({(0, 0): 90, (0, 1): 90, (0, 2): 90, (1, 0): 3}, 90), None),
    "shortcut wraps (DC only)": (_block({(0, 0): 1000}, 16), None),
    "shortcut wraps (row 0 AC)": (_block({(0, 0): 400, (0, 3): -350}, 60), None),
    "coef*q = 0 mod 2^16 keeps pass 1": (_block({(0, 0): 100, (1, 0): 512}, 128), lambda c, q: idct16(w16(c * q), np.ones(64, np.int64))),
    "per-block shortcut": (_block({(0, 0): 120, (0, 3): 120, (1, 0): 1}, 100), _per_column_shortcut),
    "issue example": (_block({(0, 0): 60, (0, 1): -40, (1, 0): 35, (1, 1): 20}, 50), None),
}


@pytest.mark.parametrize("name", list(TARGETED))
def test_statement_equals_cv2_on_targeted_blocks(name):
    (coef, q), planted = TARGETED[name]
    s = xs.baseline(8, 8, [(1, 1)], [coef.reshape(1, 1, 64)], [q], dqt16=bool(q.max() > 255), wide=True)
    want = imdecode(s, cv2.IMREAD_GRAYSCALE)
    assert np.array_equal(idct16(coef, q), want)
    if name != "issue example" and not name.startswith("shortcut wraps (DC"):
        assert not np.array_equal(idct_c(coef, q), want), "the block must reach past the C arithmetic"
    if planted is not None:
        assert not np.array_equal(planted(coef, q), want)


def _natural_streams():
    g = np.load(os.path.join(ROOT, "tests", "golden", "jpeg_cv2.npz"))
    out = [g[k].tobytes() for k in g.files if k.startswith("enc_")]
    for i, (h, w) in enumerate(dc.SIZES):
        for j, q in enumerate(dc.QUALITIES):
            for k, kind in enumerate(dc.KINDS):
                out.append(dc.encode(dc.image(h, w, kind, 1000 * i + 10 * j + k), q))
    return out


def test_statement_equals_c_statement_on_natural_corpora():
    nblk = 0
    for s in _natural_streams():
        segs = cs._segments(s)
        sof = (segs.get(0xC0) or segs[0xC1])[0]
        tq = [sof[8 + 3 * c] for c in range(sof[5])]
        tabs = dc.dqt_tables(s)
        for c, plane in enumerate(po.jpeg_coeffs(s)):
            flat = plane.reshape(-1, 64)
            assert np.array_equal(idct16(flat, tabs[tq[c]]), idct_c(flat, tabs[tq[c]]))
            nblk += flat.shape[0]
    assert nblk > 10_000


# ---- the oracle ------------------------------------------------------------------------------------------------------------------
def extreme_corpus_baseline():
    """(name, stream) of interleaved baseline extreme streams: every layout, 8- and 16-bit DQT, standard and wide tables, restarts"""
    out = []
    for i, layout in enumerate(xs.SAMPLINGS):
        for j, (dqt16, wide, rst) in enumerate([(False, False, 0), (False, True, 2), (True, True, 0), (True, False, 5)]):
            out.append((f"{layout}-{dqt16}-{wide}-{rst}", xs.extreme_stream(100 + 10 * i + j, 48, 64, layout, dqt16, wide, rst)[0]))
    return out


def test_oracle_equals_cv2_on_extreme_corpus():
    for name, s in extreme_corpus_baseline():
        assert np.array_equal(cmyk_oracle.decode(s), imdecode(s, cv2.IMREAD_COLOR)[..., ::-1]), name
        assert np.array_equal(cmyk_oracle.decode_gray(s), imdecode(s, cv2.IMREAD_GRAYSCALE)), name
        assert not cmyk_oracle.overrun(), name


def _compare_damaged(streams, defines=()):
    """(compared, equal): streams the oracle variant decodes without overrun and cv2 decodes, and how many of them equal cv2"""
    n = eq = 0
    for s in streams:
        want = imdecode(s, cv2.IMREAD_COLOR)
        if want is None:
            continue
        try:
            got = cmyk_oracle.decode(s, defines=defines)
        except ValueError:
            continue
        if cmyk_oracle.overrun(defines):
            continue
        n += 1
        eq += np.array_equal(got, want[..., ::-1])
    return n, eq


@pytest.fixture(scope="module")
def damaged():
    return xs.mutated(7, 800) + xs.mutated(8, 800, color=True)


def test_oracle_equals_cv2_on_damaged_streams(damaged):
    n, eq = _compare_damaged(damaged)
    assert n >= 1000 and eq == n, (n, eq)


@pytest.mark.parametrize("defines", [("JO_BAD_CODE_BITS=16",), ("JO_RUN_PAST_63_BREAKS",)])
def test_planted_entropy_mistakes_fail(damaged, defines):
    n, eq = _compare_damaged(damaged, defines)
    assert n >= 1000 and eq < n, (defines, n, eq)


def test_planted_c_idct_fails_on_extreme_corpus():
    s, planes, q = xs.extreme_stream(3, 64, 64, "gray")
    _, gotc, want = gray_blocks(s, planes[0], q[0])
    assert not np.array_equal(gotc, want)


# ---- the product's progressive scan decoder on damaged streams --------------------------------------------------------------------
@pytest.fixture(scope="module")
def prog_emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emul") / "libjpegprog.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-I/usr/local/cuda/include",
                        os.path.join(ROOT, "tools", "emul", "jpeg_prog_emul.cc"), "-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(out)


def _prog_luma(lib, stream):
    """the Y (or gray) samples the product reconstructs from its progressive decode, through the statement; None when a scan ran out
    of data (status 1 on the GPU)"""
    b = np.frombuffer(stream, np.uint8)
    info = (C.c_int * 8)()
    if lib.emul_jpeg_progressive(b.ctypes.data_as(C.c_void_p), C.c_size_t(b.size), None, info):
        return None
    ncomp, mcux, mcuy, bpm = info[0], info[1], info[2], info[3]
    coef = np.zeros((mcux * mcuy * bpm, 64), np.int16)
    lib.emul_jpeg_progressive(b.ctypes.data_as(C.c_void_p), C.c_size_t(b.size), coef.ctypes.data_as(C.c_void_p), info)
    if info[6]:
        return None
    pi = po.jpeg_info(stream)
    hs, vs = pi["hs"][0], pi["vs"][0]
    segs = cs._segments(stream)
    sof = segs[0xC2][0]
    q = dc.dqt_tables(stream)[sof[8]]
    y = coef.reshape(mcuy, mcux, bpm, 64)[:, :, :hs * vs].reshape(mcuy, mcux, vs, hs, 64).transpose(0, 2, 1, 3, 4)
    img = to_image(idct16(y.reshape(-1, 64), q), mcuy * vs, mcux * hs)
    return img[:pi["height"], :pi["width"]]


def test_progressive_scan_decoder_equals_cv2_on_damaged_streams(prog_emul):
    n = 0
    for s in xs.mutated(11, 300, progressive=True) + xs.mutated(12, 300, color=True, progressive=True):
        want = imdecode(s, cv2.IMREAD_GRAYSCALE)
        got = _prog_luma(prog_emul, s)
        if want is None or got is None:
            continue
        n += 1
        assert np.array_equal(got, want), n
    assert n >= 300, n
