"""CPU tests of the PNG decode: the numpy oracle (tests/png_oracle.py) pinned against cv2.imdecode, and the PRODUCT's planner and
decode core (dali_b200/csrc/png_plan.h + png_core.h -- the body of the png.cu kernels) compiled for the host by tools/emul/png_emul.cc,
bit for bit against the oracle, with every corrupt stream rejected and mutated streams run under ASan + UBSan."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import png_oracle as po  # noqa: E402
import png_streams as ps  # noqa: E402

cv2 = pytest.importorskip("cv2")
EMUL = os.path.join(ROOT, "tools", "emul", "png_emul.cc")


def _cv2(s, flag):
    return cv2.imdecode(np.frombuffer(s, np.uint8), flag | cv2.IMREAD_IGNORE_ORIENTATION)


@pytest.fixture(scope="module")
def corpus():
    return ps.corpus()


def test_oracle_matches_cv2_on_the_corpus(corpus):
    for name, s in corpus:
        got = po.decode(s)
        assert got is not None, name
        rgb, gray, _ = got
        col = _cv2(s, cv2.IMREAD_COLOR)
        assert col is not None and np.array_equal(rgb, col[..., ::-1]), name
        assert np.array_equal(gray, _cv2(s, cv2.IMREAD_GRAYSCALE)), name


def test_oracle_and_cv2_reject_the_corrupt_streams():
    for name, s in ps.corrupt():
        assert _cv2(s, cv2.IMREAD_COLOR) is None, name
        assert po.decode(s) is None, name


def test_exif_orientation_is_what_cv2_applies():
    a = ps.samples(5, 9, 2, 8, 3)
    for o in range(1, 9):
        for after in (False, True):
            s = ps.encode(a, 2, 8, exif=o, exif_after=after)
            rgb, _, got = po.decode(s)
            assert got == o
            assert np.array_equal(po.orient(rgb, o), cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR)[..., ::-1]), (o, after)
    # an eXIf chunk with a bad CRC is discarded
    s = ps.encode(a, 2, 8, exif=6)
    i = s.index(b"eXIf")
    n = int.from_bytes(s[i - 4:i], "big")
    s = s[:i + 4 + n] + bytes([s[i + 4 + n] ^ 1]) + s[i + 5 + n:]
    assert po.decode(s)[2] == 1 and cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR).shape == (5, 9, 3)


def test_gray_rule_on_every_8bit_colour():
    """(9797 R + 19234 G + 3737 B) >> 15 equals cv2's IMREAD_GRAYSCALE on all 2^24 colours (one 4096 x 4096 PNG)"""
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    ok, b = cv2.imencode(".png", img[..., ::-1], [cv2.IMWRITE_PNG_COMPRESSION, 1])
    assert ok
    g = cv2.imdecode(b, cv2.IMREAD_GRAYSCALE).astype(np.int64)
    r_, g_, b_ = (img[..., k].astype(np.int64) for k in range(3))
    assert np.array_equal(g, (po.GRAY8[0] * r_ + po.GRAY8[1] * g_ + po.GRAY8[2] * b_) >> 15)


def _build(tmp, flags):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp / "libpngemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-shared", "-fPIC", "-I/usr/local/cuda/include"] + flags + [EMUL, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    lib = C.CDLL(_build(tmp_path_factory.mktemp("png_emul"), ["-O2"]))
    lib.emul_png_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def emul_decode(lib, s, out_type):
    info = (C.c_int * 4)()
    rc = lib.emul_png_decode(s, len(s), out_type, None, info)
    if rc:
        return rc, None, None
    ch = 1 if out_type == 2 else 3
    out = np.zeros((info[1], info[0], ch), np.uint8)
    rc = lib.emul_png_decode(s, len(s), out_type, out.ctypes.data, info)
    return rc, out, list(info)


def test_emulated_core_matches_the_oracle(emul, corpus):
    for name, s in corpus:
        rgb, gray, orientation = po.decode(s)
        rc, out, info = emul_decode(emul, s, 0)
        assert rc == 0 and np.array_equal(out, rgb), name
        assert info[3] == orientation
        rc, out, _ = emul_decode(emul, s, 1)
        assert rc == 0 and np.array_equal(out, rgb[..., ::-1]), name
        rc, out, _ = emul_decode(emul, s, 2)
        assert rc == 0 and np.array_equal(out[..., 0], gray), name


def test_emulated_core_rejects_every_corrupt_stream(emul):
    for name, s in ps.corrupt():
        rc, _, _ = emul_decode(emul, s, 0)
        assert rc != 0, name


MUTATE = r"""
import ctypes as C, sys
import numpy as np
sys.path.insert(0, %(tests)r)
import png_streams as ps
lib = C.CDLL(%(lib)r)
lib.emul_png_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
rng = np.random.default_rng(7)
seeds = [s for _, s in ps.corpus()[::3]] + [s for _, s in ps.corrupt()]
n = 0
for it in range(%(n)d):
    s = bytearray(seeds[it %% len(seeds)])
    for _ in range(int(rng.integers(1, 6))):
        k = int(rng.integers(0, 4))
        i = int(rng.integers(0, len(s)))
        if k == 0: s[i] ^= 1 << int(rng.integers(0, 8))
        elif k == 1: s[i] = int(rng.integers(0, 256))
        elif k == 2: del s[i:i + int(rng.integers(1, 16))]
        else: s[i:i] = bytes(rng.integers(0, 256, int(rng.integers(1, 8))).astype(np.uint8))
    info = (C.c_int * 4)()
    b = bytes(s)
    if lib.emul_png_decode(b, len(b), 0, None, info) == 0 and info[0] * info[1] <= 1 << 22:
        out = np.zeros(info[0] * info[1] * 3 + 1, np.uint8)
        lib.emul_png_decode(b, len(b), int(rng.integers(0, 3)), out.ctypes.data, info)
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
