"""CPU tests of the TIFF decode: the numpy oracle (tests/tiff_oracle.py) pinned against cv2.imdecode, and the PRODUCT's planner and
decode core (dali_b200/csrc/tiff_plan.h + tiff_core.h -- the body of the tiff.cu kernels) compiled for the host by
tools/emul/tiff_emul.cc, bit for bit against the oracle, with every corrupt or unsupported stream rejected and mutated streams run
under ASan + UBSan."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import tiff_oracle as to  # noqa: E402
import tiff_streams as ts  # noqa: E402

cv2 = pytest.importorskip("cv2")
EMUL = os.path.join(ROOT, "tools", "emul", "tiff_emul.cc")
UNSUPPORTED, BAD_DATA = 2, 4


def _cv2(s, flag):
    return cv2.imdecode(np.frombuffer(s, np.uint8), flag | cv2.IMREAD_IGNORE_ORIENTATION)


@pytest.fixture(scope="module")
def corpus():
    return ts.corpus()


def test_oracle_matches_cv2_on_the_corpus(corpus):
    for name, s in corpus:
        got = to.decode(s)
        assert got is not None, name
        rgb, gray, _ = got
        col = _cv2(s, cv2.IMREAD_COLOR)
        assert col is not None and np.array_equal(rgb, col[..., ::-1]), name
        assert np.array_equal(gray, _cv2(s, cv2.IMREAD_GRAYSCALE)), name


def test_rules_pinned_against_cv2():
    """the rules of tiff_oracle.py one by one, on crafted streams"""
    a = ts.samples(9, 13, 4, 8, 1)
    # unassociated alpha premultiplies, associated alpha is dropped
    for extra, want in (((2,), (a[..., :3] * a[..., 3:] + 127) // 255), ((1,), a[..., :3])):
        s = ts.encode(a, 2, 8, 5, extra=extra)
        assert np.array_equal(_cv2(s, cv2.IMREAD_COLOR)[..., ::-1], want.astype(np.uint8)), extra
    # 16-bit RGB -> round(v / 257); 16-bit gray -> high byte
    a16 = ts.samples(9, 13, 3, 16, 2)
    assert np.array_equal(_cv2(ts.encode(a16, 2, 16, 8), cv2.IMREAD_COLOR)[..., ::-1], ((a16 + 128) // 257).astype(np.uint8))
    assert np.array_equal(_cv2(ts.encode(a16[..., :1], 1, 16, 8), cv2.IMREAD_GRAYSCALE), (a16[..., 0] >> 8).astype(np.uint8))
    # GRAY of a colour pixel, MinIsWhite, 1-bit gray
    rgb = a[..., :3].astype(np.int64)
    g = (1868 * rgb[..., 2] + 9617 * rgb[..., 1] + 4899 * rgb[..., 0] + 8192) >> 14
    assert np.array_equal(_cv2(ts.encode(a[..., :3], 2, 8, 5), cv2.IMREAD_GRAYSCALE), g.astype(np.uint8))
    assert np.array_equal(_cv2(ts.encode(a[..., :1], 0, 8, 5), cv2.IMREAD_GRAYSCALE), 255 - a[..., 0].astype(np.uint8))
    b = ts.samples(9, 13, 1, 1, 3)
    assert set(np.unique(_cv2(ts.encode(b, 1, 1, 5), cv2.IMREAD_GRAYSCALE))) <= {0, 255}
    # a ColorMap whose entries all lie below 256 is used as it is; otherwise its high bytes
    p = ts.samples(9, 13, 1, 8, 4)
    for wide in (True, False):
        m = ts.palette(8, 5, wide)
        want = (m >> 8 if wide else m)[p[..., 0]]
        assert np.array_equal(_cv2(ts.encode(p, 3, 8, 5, colormap=m), cv2.IMREAD_COLOR)[..., ::-1], want.astype(np.uint8)), wide
    # Predictor is ignored without LZW / Deflate
    s = ts.encode(a[..., :3], 2, 8, 1, extra_tags=[(317, (3, [2]))])
    assert np.array_equal(_cv2(s, cv2.IMREAD_COLOR)[..., ::-1], a[..., :3].astype(np.uint8))
    # orientation 6 transposes the shape
    s = ts.encode(a[..., :3], 2, 8, 5, orientation=6)
    assert cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR).shape == (13, 9, 3)
    assert to.decode(s)[2] == 6


def test_corrupt_segments_fail_here_and_decode_partially_in_cv2():
    """documented deviation (DESIGN 2): cv2 returns an image for a corrupt segment; the oracle (and the decoder) fail it"""
    for name, s in ts.data_corrupt():
        assert _cv2(s, cv2.IMREAD_COLOR) is not None, name
        assert to.decode(s) is None, name


def test_malformed_and_unsupported_streams():
    """the oracle refuses every stream the plan set-up refuses; cv2 refuses those of CV2_REJECTS too (2- and 4-bit gray, 2-bit palette,
    uncompressed tiles, the size limits, ...) and decodes the others (FillOrder 2, CMYK, YCbCr, 16-bit gray tiles, old-style LZW)"""
    for name, s in ts.plan_corrupt():
        assert to.decode(s) is None, name
        try:
            got = cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR)
        except cv2.error:
            got = None
        assert (got is None) == (name in ts.CV2_REJECTS), name


def _build(tmp, flags):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp / "libtiffemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-shared", "-fPIC", "-I/usr/local/cuda/include"] + flags + [EMUL, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    lib = C.CDLL(_build(tmp_path_factory.mktemp("tiff_emul"), ["-O2"]))
    lib.emul_tiff_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def emul_decode(lib, s, out_type):
    info = (C.c_int * 4)()
    rc = lib.emul_tiff_decode(s, len(s), out_type, None, info)
    if rc:
        return rc, None, None
    ch = 1 if out_type == 2 else 3
    out = np.zeros((info[1], info[0], ch), np.uint8)
    rc = lib.emul_tiff_decode(s, len(s), out_type, out.ctypes.data, info)
    return rc, out, list(info)


def test_emulated_core_matches_the_oracle(emul, corpus):
    for name, s in corpus:
        rgb, gray, orientation = to.decode(s)
        rc, out, info = emul_decode(emul, s, 0)
        assert rc == 0 and np.array_equal(out, rgb), name
        assert info[3] == orientation
        rc, out, _ = emul_decode(emul, s, 1)
        assert rc == 0 and np.array_equal(out, rgb[..., ::-1]), name
        rc, out, _ = emul_decode(emul, s, 2)
        assert rc == 0 and np.array_equal(out[..., 0], gray), name


def test_emulated_core_rejects_every_corrupt_stream(emul):
    for name, s in ts.data_corrupt():
        assert emul_decode(emul, s, 0)[0] == -1, name
    unsupported = {"bigtiff", "jpeg_compression", "fill_order_2", "float_samples", "predictor_3", "cmyk", "ycbcr", "too_wide",
                   "too_many_pixels", "oversized_tile", "gray2", "gray4", "palette2", "raw_tiles", "gray16_tiles", "old_lzw"}
    for name, s in ts.plan_corrupt():
        assert emul_decode(emul, s, 0)[0] == (UNSUPPORTED if name in unsupported else BAD_DATA), name


MUTATE = r"""
import ctypes as C, sys
import numpy as np
sys.path.insert(0, %(tests)r)
import tiff_streams as ts
lib = C.CDLL(%(lib)r)
lib.emul_tiff_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
rng = np.random.default_rng(7)
seeds = [s for _, s in ts.corpus()[::3]] + [s for _, s in ts.data_corrupt() + ts.plan_corrupt()]
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
    if lib.emul_tiff_decode(b, len(b), 0, None, info) == 0 and info[0] * info[1] <= 1 << 22:
        out = np.zeros(info[0] * info[1] * 3 + 1, np.uint8)
        lib.emul_tiff_decode(b, len(b), int(rng.integers(0, 3)), out.ctypes.data, info)
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
