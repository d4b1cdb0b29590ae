"""Lossless JPEG corpus checks without a GPU: the hand encoder of tests/ljpeg_streams.py against cv2.imdecode (libjpeg-turbo), the
corpus's coverage read back from the parsed headers of its streams, and what cv2 does with every stream the decoder refuses or flags, so
that each refusal and each documented deviation (DESIGN section 2) is pinned against the reference."""
import ctypes as C
import os
import shutil
import struct
import subprocess
import sys

import numpy as np
import pytest

import ljpeg_streams as ls

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tools", "emul", "ljpeg_emul.cc")
RGB, BGR, GRAY = 0, 1, 2


def _build(tmp, flags):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp / "libljpegemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-shared", "-fPIC", "-Wall", "-ffp-contract=off", "-I/usr/local/cuda/include"] + flags + [EMUL, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    lib = C.CDLL(_build(tmp_path_factory.mktemp("ljpeg_emul"), ["-O2"]))
    lib.emul_ljpeg_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def emul_decode(lib, s, out_type):
    """(status, output): the planner's status, or 0 / -1 (the sample's status) with the H x W x C output"""
    info = (C.c_int * 4)()
    rc = lib.emul_ljpeg_decode(s, len(s), out_type, None, info)
    if rc:
        return rc, None
    ch = 1 if out_type == GRAY else 3
    out = np.zeros((info[1], info[0], ch), np.uint8)
    return lib.emul_ljpeg_decode(s, len(s), out_type, out.ctypes.data, info), out


def _want(exp, ot):
    """the decoder's output for the samples `exp`: one component replicated for RGB / BGR, three to GRAY by the RGB-JPEG rule"""
    if ot == GRAY:
        if exp.shape[2] == 1:
            return exp
        a = exp.astype(np.int64)
        return ((a[..., 0] * 19595 + a[..., 1] * 38470 + a[..., 2] * 7471 + 32768) >> 16).astype(np.uint8)[..., None]
    rgb = np.repeat(exp, 3, axis=2) if exp.shape[2] == 1 else exp
    return rgb[..., ::-1] if ot == BGR else rgb


def test_emulated_decode_of_the_corpus(emul):
    """the planner and the kernel bodies compiled for the host (chains in reverse order) against the encoder's samples, which cv2
    decodes too (test below), in RGB, BGR and GRAY"""
    for name, s, exp, _ in ls.corpus():
        for ot in (RGB, BGR, GRAY):
            st, out = emul_decode(emul, s, ot)
            assert st == 0 and np.array_equal(out, _want(exp, ot)), (name, ot, st)


def test_emulated_refusals_and_corruption(emul):
    for name, s, code, why in ls.refused():
        assert emul_decode(emul, s, RGB)[0] == code, (name, why)
    for name, s, kind in ls.corrupt():
        assert emul_decode(emul, s, RGB)[0] == -1, name


def test_emulated_decode_agrees_with_cv2_on_mutated_entropy_data(emul):
    """damaged entropy data: wherever the decode reports no error and cv2 decodes, the two agree (out-of-range reconstruction)"""
    rng = np.random.default_rng(5)
    bases = [ls.encode(ls.image(24, 33, 3, 8, 90), pred=p, tables="opt") for p in (1, 4, 5, 6, 7)] + \
            [ls.encode(ls.image(20, 21, 1, 6, 91), P=6, Pt=1, pred=p) for p in (2, 3, 4)]
    checked = 0
    for k in range(400):
        b = bytearray(bases[k % len(bases)])
        sos = b.index(b"\xFF\xDA")
        lo = sos + 2 + struct.unpack(">H", bytes(b[sos + 2: sos + 4]))[0]
        for _ in range(int(rng.integers(1, 4))):
            q = int(rng.integers(lo, len(b) - 2))
            if b[q] != 0xFF and b[q - 1] != 0xFF:
                b[q] = int(rng.integers(0, 255))
        st, out = emul_decode(emul, bytes(b), RGB)
        c = _cv(bytes(b))
        if st == 0 and c is not None:
            c = c[..., None] if c.ndim == 2 else c[..., ::-1]
            assert np.array_equal(out, _want(c, RGB)), k
            checked += 1
    assert checked > 100, checked


MUTATE = r"""
import ctypes as C, sys
import numpy as np
sys.path.insert(0, %(tests)r)
import ljpeg_streams as ls
lib = C.CDLL(%(lib)r)
lib.emul_ljpeg_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
rng = np.random.default_rng(13)
seeds = [s for _, s, _, _ in ls.corpus()][::3] + [s for _, s, _, _ in ls.refused()] + [s for _, s, _ in ls.corrupt()]
n = 0
for it in range(%(n)d):
    s = bytearray(seeds[it %% len(seeds)])
    hdr = s.index(b"\xFF\xDA") + 2 if b"\xFF\xDA" in s else len(s)
    for _ in range(int(rng.integers(1, 6))):
        k = int(rng.integers(0, 4))
        # half of the edits land in the headers (DHT counts and values, SOF, SOS, DRI), half anywhere
        i = int(rng.integers(0, hdr + 1)) if rng.integers(0, 2) else int(rng.integers(0, len(s) + 1))
        if k == 0 and i < len(s): s[i] ^= 1 << int(rng.integers(0, 8))
        elif k == 1 and i < len(s): s[i] = int(rng.integers(0, 256))
        elif k == 2: del s[i:i + int(rng.integers(1, 16))]
        else: s[i:i] = bytes(rng.integers(0, 256, int(rng.integers(1, 8))).astype(np.uint8))
    info = (C.c_int * 4)()
    b = bytes(s)
    if lib.emul_ljpeg_decode(b, len(b), 0, None, info) == 0 and info[0] * info[1] <= 1 << 20:
        out = np.zeros(info[0] * info[1] * 3 + 1, np.uint8)
        lib.emul_ljpeg_decode(b, len(b), int(rng.integers(0, 3)), out.ctypes.data, info)
        n += 1
print("mutated-ok", n)
"""


def test_mutated_streams_under_asan_and_ubsan(tmp_path):
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    if not os.path.isabs(asan) or not os.path.exists(asan):
        pytest.skip("needs the sanitizer runtimes")
    lib = _build(tmp_path, ["-O1", "-g", "-fsanitize=address,undefined", "-fno-omit-frame-pointer", "-fno-sanitize-recover=undefined"])
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    code = MUTATE % dict(tests=os.path.dirname(os.path.abspath(__file__)), lib=lib, n=1500)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=900, env=env)
    assert r.returncode == 0 and "mutated-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])


def _cv(s, flag=None):
    return cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_UNCHANGED if flag is None else flag)


def _headers(s):
    """(P, H, W, Nc, sampling, predictor, Pt, restart interval, DHT tables, longest code, markers)"""
    pos, out = 2, dict(tables=[], maxlen=0, jfif=False, adobe=None, ri=0)
    while True:
        m, L = s[pos + 1], struct.unpack(">H", s[pos + 2: pos + 4])[0]
        body = s[pos + 4: pos + 2 + L]
        if m == 0xC3:
            out.update(P=body[0], H=struct.unpack(">H", body[1:3])[0], W=struct.unpack(">H", body[3:5])[0], C=body[5],
                       samp={body[7 + 3 * c] for c in range(body[5])})
        elif m == 0xC4:
            bits = list(body[1:17])
            out["tables"].append(bytes(body))
            out["maxlen"] = max(out["maxlen"], max(n + 1 for n in range(16) if bits[n]))
        elif m == 0xDD:
            out["ri"] = struct.unpack(">H", body[:2])[0]
        elif m == 0xE0:
            out["jfif"] = True
        elif m == 0xEE:
            out["adobe"] = body[11]
        elif m == 0xDA:
            n = body[0]
            out.update(pred=body[1 + 2 * n], Pt=body[3 + 2 * n] & 15, td={body[2 + 2 * c] >> 4 for c in range(n)})
            out["data"] = s[pos + 2 + L:]
            return out
        pos += 2 + L


def test_corpus_decodes_in_cv2_to_the_encoder_input():
    for name, s, exp, _ in ls.corpus():
        d = _cv(s)
        assert d is not None, name
        d = d[..., None] if d.ndim == 2 else d[..., ::-1]       # 3 components come back unconverted, in B, G, R order
        assert np.array_equal(d, exp), name


def test_corpus_covers_what_it_claims():
    hs = [(_headers(s), exp) for _, s, exp, _ in ls.corpus()]
    assert {h["P"] for h, _ in hs} == set(range(2, 9))
    assert {h["pred"] for h, _ in hs} == set(range(1, 8))
    assert {(h["P"], h["Pt"]) for h, _ in hs} >= {(8, 7), (8, 4), (2, 1), (6, 5), (6, 3), (4, 0)}
    assert {h["C"] for h, _ in hs} == {1, 3} and all(h["samp"] == {0x11} for h, _ in hs)
    assert max(h["maxlen"] for h, _ in hs) == 16
    assert any(len(h["td"]) == 3 for h, _ in hs)                          # a distinct table per component
    assert any(h["ri"] and h["ri"] == h["W"] for h, _ in hs) and any(h["ri"] > h["W"] for h, _ in hs)
    assert any(h["ri"] == 1 and h["W"] == 1 for h, _ in hs)               # one-sample units
    assert any(h["H"] * h["W"] == 1 for h, _ in hs)
    assert any(h["data"].count(b"\xFF\x00") > 100 for h, _ in hs)        # stuffing everywhere
    assert any(len(h["data"]) < 128 for h, _ in hs)                       # a unit shorter than a subsequence
    big = [_headers(s) for _, s, _, _ in ls.corpus(big=True)]
    assert {(h["W"], h["H"]) for h in big} >= {(1920, 1080), (3840, 2160)}


def test_refused_streams_in_cv2():
    """cv2 refuses every stream the plan refuses, except three it decodes, which the decoder refuses on purpose (DESIGN section 2):
    4 components and sampling factors other than 1x1"""
    decoded_by_cv2 = {"four_components", "sampling_2x1"}                # the other refusals: cv2 refuses them too
    for name, s, code, why in ls.refused():
        assert code in (ls.UNSUPPORTED, ls.BAD_DATA)
        assert (_cv(s) is not None) == (name in decoded_by_cv2), (name, why)


def test_corrupt_streams_in_cv2():
    """cv2 returns None for truncated data and decodes through the other damage with a warning; the decoder sets the sample's status
    for all of them (DESIGN section 2)"""
    for name, s, kind in ls.corrupt():
        assert (_cv(s) is None) == (kind == "truncated"), name


def test_cv2_refuses_colour_conversion_of_lossless():
    """the two deviations: cv2 decodes one component only to GRAY and three components only to colour"""
    g = ls.encode(ls.image(10, 12, 1, 8, 1))
    c = ls.encode(ls.image(10, 12, 3, 8, 2))
    assert _cv(g, cv2.IMREAD_GRAYSCALE) is not None and _cv(g, cv2.IMREAD_COLOR) is None
    assert _cv(c, cv2.IMREAD_COLOR) is not None and _cv(c, cv2.IMREAD_GRAYSCALE) is None
