"""CPU tests of the lossy WebP decode: the PRODUCT's planner and decode bodies (dali_b200/csrc/webp_plan.h + webp_core.h -- the body of
the webp.cu kernels) compiled for the host by tools/emul/webp_emul.cc, bit for bit against cv2.imdecode on the corpus of
tests/webp_streams.py in RGB, BGR and GRAY; the parity rules pinned against cv2; every corrupt stream rejected as listed; mutated
streams run under ASan + UBSan."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import webp_streams as ws  # noqa: E402

cv2 = pytest.importorskip("cv2")
EMUL = os.path.join(ROOT, "tools", "emul", "webp_emul.cc")
RGB, BGR, GRAY = 0, 1, 2
NOORIENT = cv2.IMREAD_IGNORE_ORIENTATION


def _build(tmp, flags):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp / "libwebpemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-shared", "-fPIC", "-I/usr/local/cuda/include", *flags, EMUL, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    lib = C.CDLL(_build(tmp_path_factory.mktemp("webp_emul"), ["-O2"]))
    lib.emul_webp_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    lib.emul_webp_header.argtypes = [C.c_char_p, C.c_size_t, C.c_void_p]
    return lib


def _decode(lib, s, out_type):
    info = np.zeros(4, np.int32)
    rc = lib.emul_webp_decode(s, len(s), out_type, None, info.ctypes.data)
    if rc:
        return rc, None, info
    out = np.zeros((info[1], info[0], 1 if out_type == GRAY else 3), np.uint8)
    rc = lib.emul_webp_decode(s, len(s), out_type, out.ctypes.data, info.ctypes.data)
    return rc, out, info


@pytest.fixture(scope="module")
def corpus():
    return ws.corpus(big=True)


def test_corpus_bit_exact_with_cv2(emul, corpus):
    for name, s in corpus:
        bgr = ws.decode(s, cv2.IMREAD_COLOR | NOORIENT)
        gray = ws.decode(s, cv2.IMREAD_GRAYSCALE | NOORIENT)
        for ot, want in ((RGB, bgr[..., ::-1]), (BGR, bgr), (GRAY, gray[..., None])):
            rc, out, _ = _decode(emul, s, ot)
            assert rc == 0, (name, ot, rc)
            assert np.array_equal(out, want), (name, ot, int(np.abs(out.astype(int) - want).max()))


def test_corpus_covers_what_it_claims(emul, corpus):
    """read from the parsed frame headers and the entropy decode, not from the encoder settings"""
    h = {}
    for name, s in corpus:
        v = np.zeros(7, np.int32)
        assert emul.emul_webp_header(s, len(s), v.ctypes.data) == 0, name
        h[name] = v.tolist()
    vals = list(h.values())
    assert {v[0] for v in vals} == {1, 2, 4, 8}                      # token partitions
    assert {v[1] for v in vals} == {0, 1, 2}                         # no filter, simple, normal
    assert {v[6] for v in vals} >= {1, 2, 3, 4}                      # segments in use
    assert any(v[3] == 0 for v in vals) and any(v[3] == 1 for v in vals)   # with and without a segment map
    assert any(v[4] == 0 for v in vals) and any(v[4] == 1 for v in vals)   # skip probability off and on
    assert any(v[5] > 0 for v in vals) and any(v[5] == 0 for v in vals)    # 4x4 and 16x16 macroblocks
    assert len({h[f"enc_filter_sharpness{k}_filter_strength60"][2] for k in range(8)}) >= 3  # sharpness limits the inner level
    assert h["enc_filter_type0_filter_strength100"][1] == 1 and h["enc_filter_type1_filter_strength100"][1] == 2
    for p in range(4):
        assert h[f"enc_partitions{p}_method2"][0] == 1 << p


def test_info_and_orientation(emul, corpus):
    """components 3, or 4 when VP8X flags alpha; the EXIF orientation is read, and cv2 applies it"""
    d = dict(corpus)
    for name, s in corpus:
        rc, _, info = _decode(emul, s, RGB)
        assert info[2] == (4 if name == "pil_alpha" else 3), name
        assert info[3] == (int(name[8:]) if name.startswith("pil_exif") else 1), name
    s = d["pil_exif6"]
    assert np.array_equal(ws.decode(s), np.ascontiguousarray(np.rot90(ws.decode(s, cv2.IMREAD_COLOR | NOORIENT), -1)))


def test_parity_rules_pinned_against_cv2(corpus):
    d = dict(corpus)
    # GRAY is cv2's BGR2GRAY of the colour decode, (9798 R + 19235 G + 3735 B + 16384) >> 15
    for name in ("cv2_128x200_q90", "pil_method3", "enc_use_sharp_yuv1"):
        s = d[name]
        bgr = ws.decode(s, cv2.IMREAD_COLOR | NOORIENT).astype(np.int64)
        rule = (9798 * bgr[..., 2] + 19235 * bgr[..., 1] + 3735 * bgr[..., 0] + 16384) >> 15
        assert np.array_equal(ws.decode(s, cv2.IMREAD_GRAYSCALE | NOORIENT), rule.astype(np.uint8)), name
    rng = np.random.default_rng(0)
    px = rng.integers(0, 256, (1 << 20, 1, 3), dtype=np.uint8)
    p = px.astype(np.int64)
    assert np.array_equal(cv2.cvtColor(px, cv2.COLOR_BGR2GRAY)[:, 0],
                          ((9798 * p[..., 2] + 19235 * p[..., 1] + 3735 * p[..., 0] + 16384) >> 15)[:, 0])
    # alpha: COLOR is UNCHANGED[..., :3], unpremultiplied, and equals the decode of the stream without its ALPH chunk
    s = d["pil_alpha"]
    un = ws.decode(s, cv2.IMREAD_UNCHANGED)
    assert un.shape[2] == 4 and np.array_equal(ws.decode(s), un[..., :3])
    i = s.index(b"ALPH")
    n = int.from_bytes(s[i + 4:i + 8], "little")
    body = s[12:i] + s[i + 8 + n + (n & 1):]
    body = body[:8] + bytes([body[8] & ~0x10]) + body[9:]      # VP8X: clear the alpha flag
    stripped = b"RIFF" + (len(body) + 4).to_bytes(4, "little") + b"WEBP" + body
    assert np.array_equal(ws.decode(stripped), ws.decode(s))


def test_corrupt_streams_are_rejected(emul):
    for name, s, status in ws.plan_corrupt():
        rc, _, _ = _decode(emul, s, RGB)
        assert rc == status, (name, rc)
        if name != "vp8l":                                          # cv2 decodes lossless streams: not supported here
            assert ws.decode(s) is None, name
    for name, s in ws.data_corrupt():
        rc, _, _ = _decode(emul, s, RGB)
        assert rc == -1, (name, rc)
        assert ws.decode(s) is None, name


def test_alph_deviation(emul):
    """cv2 refuses a stream whose ALPH data is corrupt, even in COLOR mode (it decodes the alpha plane); the colour decode here does not
    read ALPH, so the stream decodes to the colour of the intact stream (DESIGN.md section 2)"""
    s = ws.alph_corrupt()
    assert ws.decode(s) is None
    rc, out, _ = _decode(emul, s, BGR)
    assert rc == 0
    i = s.index(b"ALPH")
    n = int.from_bytes(s[i + 4:i + 8], "little")
    body = s[12:i] + s[i + 8 + n + (n & 1):]
    body = body[:8] + bytes([body[8] & ~0x10]) + body[9:]
    intact = b"RIFF" + (len(body) + 4).to_bytes(4, "little") + b"WEBP" + body
    assert np.array_equal(out, ws.decode(intact))


MUTATE = r"""
import ctypes as C, sys
import numpy as np
sys.path.insert(0, %(tests)r)
import webp_streams as ws
lib = C.CDLL(%(lib)r)
lib.emul_webp_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
rng = np.random.default_rng(7)
seeds = [s for _, s in ws.corpus()[::6]] + [s for _, s, _ in ws.plan_corrupt()] + [s for _, s in ws.data_corrupt()]
info = np.zeros(4, np.int32)
n = 0
for it in range(1500):
    b = bytearray(seeds[it %% len(seeds)])
    k = int(rng.integers(0, 4))
    if k == 0:
        for _ in range(int(rng.integers(1, 8))):
            b[int(rng.integers(0, len(b)))] = int(rng.integers(0, 256))
    elif k == 1:
        b = b[:int(rng.integers(12, len(b) + 1))]
    elif k == 2:
        i = int(rng.integers(20, len(b)))
        b[i:i + 4] = rng.integers(0, 256, 4, dtype=np.uint8).tobytes()
    else:
        i = int(rng.integers(12, len(b)))
        b[i] ^= 1 << int(rng.integers(0, 8))
    b = bytes(b)
    if lib.emul_webp_decode(b, len(b), 0, None, info.ctypes.data) == 0 and info[0] * info[1] <= 1 << 20:
        out = np.zeros(int(info[0]) * int(info[1]) * 3, np.uint8)
        lib.emul_webp_decode(b, len(b), int(rng.integers(0, 3)), out.ctypes.data, info.ctypes.data)
        n += 1
print("mutated-ok", n)
"""


def test_mutated_streams_under_sanitizers(tmp_path):
    lib = _build(tmp_path, ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-fno-omit-frame-pointer"])
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    ubsan = subprocess.run(["g++", "-print-file-name=libubsan.so"], capture_output=True, text=True).stdout.strip()
    env = dict(os.environ, LD_PRELOAD=f"{asan} {ubsan}", ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([sys.executable, "-c", MUTATE % dict(tests=os.path.join(ROOT, "tests"), lib=lib)], capture_output=True,
                       text=True, env=env, timeout=1500)
    assert r.returncode == 0 and "mutated-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
