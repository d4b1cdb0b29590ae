"""CPU tests of the BMP / PNM decode: the PRODUCT's planner and decode core (dali_b200/csrc/bitmap_plan.h + bitmap_core.h -- the body of
the bitmap.cu kernels) compiled for the host by tools/emul/bitmap_emul.cc, bit for bit against cv2.imdecode on the corpus of
tests/bitmap_streams.py, each parity rule pinned against cv2 itself, every corrupt or unsupported stream rejected (and refused by cv2
too), and mutated streams run under ASan + UBSan."""
import ctypes as C
import os
import shutil
import struct
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bitmap_streams as bs  # noqa: E402

cv2 = pytest.importorskip("cv2")
EMUL = os.path.join(ROOT, "tools", "emul", "bitmap_emul.cc")
RGB, BGR, GRAY = 0, 1, 2


def _cv2(s, flag):
    try:
        return cv2.imdecode(np.frombuffer(s, np.uint8), flag)
    except cv2.error:
        return None


def _build(tmp, flags):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp / "libbitmapemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-shared", "-fPIC", "-Wall", "-ffp-contract=off", "-I/usr/local/cuda/include"] + flags + [EMUL, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    lib = C.CDLL(_build(tmp_path_factory.mktemp("bitmap_emul"), ["-O2"]))
    lib.emul_bitmap_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def corpus():
    return bs.corpus()


def emul_decode(lib, s, out_type, shift=0):
    """(status, output, info); `shift` moves the output off 16-byte alignment (the byte-store path)."""
    info = (C.c_int * 12)()
    rc = lib.emul_bitmap_decode(s, len(s), out_type, None, info)
    if rc:
        return rc, None, None
    ch = 1 if out_type == GRAY else 3
    buf = np.zeros(info[1] * info[0] * ch + 32, np.uint8)
    base = (-buf.ctypes.data) % 16 + shift
    rc = lib.emul_bitmap_decode(s, len(s), out_type, buf.ctypes.data + base, info)
    return rc, buf[base:base + info[1] * info[0] * ch].reshape(info[1], info[0], ch), list(info)


def decode_all(lib, s, shift=0):
    """RGB and GRAY of the emulated decode, BGR checked against RGB on the way"""
    rc, rgb, info = emul_decode(lib, s, RGB, shift)
    assert rc == 0, rc
    rc, bgr, _ = emul_decode(lib, s, BGR, shift)
    assert rc == 0 and np.array_equal(bgr, rgb[..., ::-1])
    rc, gray, _ = emul_decode(lib, s, GRAY, shift)
    assert rc == 0
    return rgb, gray[..., 0], info


def test_emulated_core_matches_cv2_on_the_corpus(emul, corpus):
    for k, (name, s) in enumerate(corpus):
        col, gray = _cv2(s, cv2.IMREAD_COLOR), _cv2(s, cv2.IMREAD_GRAYSCALE)
        assert col is not None and gray is not None, name
        got_rgb, got_gray, info = decode_all(emul, s, shift=k % 3)
        assert np.array_equal(got_rgb, col[..., ::-1]), name
        assert np.array_equal(got_gray, gray), name
        assert info[3] == 1


def _one(lib, s, out_type=RGB):
    rc, out, _ = emul_decode(lib, s, out_type)
    assert rc == 0
    return out if out_type != GRAY else out[..., 0]


def test_rules_pinned_against_cv2(emul):
    """the parity rules of DESIGN section 2, each on a crafted stream, against cv2 and against the emulated decode"""
    def both(s, want, flag=cv2.IMREAD_COLOR):
        got_cv2 = _cv2(s, flag)
        want = np.asarray(want, np.uint8)
        if flag == cv2.IMREAD_COLOR:
            assert np.array_equal(got_cv2[..., ::-1], want), (got_cv2, want)
            assert np.array_equal(_one(emul, s), want)
        else:
            assert np.array_equal(got_cv2, want), (got_cv2, want)
            assert np.array_equal(_one(emul, s, GRAY), want)

    gray_rule = lambda r, g, b: (1868 * b + 9617 * g + 4899 * r + 8192) >> 14  # noqa: E731
    # GRAY of a colour pixel (24-bit BMP, P6, palette, 16-bit P6 after >> 8), the CMYK / TIFF rule
    px = bytes([10, 200, 30, 250, 5, 99, 0, 0])                               # B, G, R of two pixels, row padding
    both(bs.bmp(2, 1, 24, px), [[gray_rule(30, 200, 10), gray_rule(99, 5, 250)]], cv2.IMREAD_GRAYSCALE)
    both(b"P6 1 1 255\n" + bytes([30, 200, 10]), [[gray_rule(30, 200, 10)]], cv2.IMREAD_GRAYSCALE)
    pal = bytes([200, 100, 50, 0, 0, 255, 0, 0])
    both(bs.bmp(2, 1, 8, bytes([0, 1, 0, 0]), palette=pal, clrused=2), [[gray_rule(50, 100, 200), gray_rule(0, 255, 0)]],
         cv2.IMREAD_GRAYSCALE)
    both(b"P6\n1 1\n65535\n" + bytes([0x12, 0x34, 0xAB, 0xCD, 0x56, 0x78]), [[gray_rule(0x12, 0xAB, 0x56)]], cv2.IMREAD_GRAYSCALE)
    # 5-6-5 and 5-5-5 expand by shifting, without bit replication
    m565, m555 = struct.pack("<III", 0xF800, 0x7E0, 0x1F), struct.pack("<III", 0x7C00, 0x3E0, 0x1F)
    both(bs.bmp(2, 1, 16, struct.pack("<HH", 0xF800, 0x07E0), comp=3, masks=m565), [[[248, 0, 0], [0, 252, 0]]])
    both(bs.bmp(1, 1, 16, struct.pack("<HH", 0x7FFF, 0)), [[[248, 248, 248]]])
    both(bs.bmp(1, 1, 16, struct.pack("<HH", 0x7FFF, 0), comp=3, masks=m555), [[[248, 248, 248]]])
    # 32-bit BITFIELDS: the masks are ignored, the bytes are B, G, R, alpha
    for masks in ((0xFF0000, 0xFF00, 0xFF), (0xFF, 0xFF00, 0xFF0000), (0xFF000000, 0xFF0000, 0xFF00)):
        both(bs.bmp(1, 1, 32, bytes([10, 20, 30, 40]), comp=3, masks=struct.pack("<III", *masks)), [[[30, 20, 10]]])
    # 32-bit BITFIELDS in a V3 - V5 header with all three colour masks set: cv2's mask path, whose GRAY is the float32 sum
    # (0.299 R + 0.587 G) + 0.114 B, truncated (equal to cv2 on the whole RGB cube); COLOR is still B, G, R bytes, alpha dropped.  With a
    # colour mask empty, or in a 52-byte header, the integer rule holds
    def float_gray(r, g, b):
        f = np.float32
        return int((f(0.299) * f(r) + f(0.587) * f(g)) + f(0.114) * f(b))
    rng = np.random.default_rng(4)
    px = rng.integers(0, 256, (16, 16, 4)).astype(np.uint8)
    v = np.arange(1 << 24, dtype=np.int64)[rng.integers(0, 1 << 24, 256)]
    px[..., 0], px[..., 1], px[..., 2] = (v & 255).reshape(16, 16), ((v >> 8) & 255).reshape(16, 16), (v >> 16).reshape(16, 16)
    rows = bs.rows(px, 32, True)
    fg = [[float_gray(*p[2::-1]) for p in r] for r in px.astype(np.int64)]
    ig = [[gray_rule(*p[2::-1]) for p in r] for r in px.astype(np.int64)]
    assert fg != ig
    for hdr, hm in ((56, (0xFF0000, 0xFF00, 0xFF, 0xFF000000)), (108, (0xFF0000, 0xFF00, 0xFF, 0)), (124, (0xFF0000, 0xFF00, 0xFF, 0xFF))):
        s = bs.bmp(16, -16, 32, rows, comp=3, header=hdr, header_masks=hm)
        both(s, fg, cv2.IMREAD_GRAYSCALE)
        both(s, px[..., 2::-1])
    for hdr, hm in ((52, (0xFF0000, 0xFF00, 0xFF, 0)), (108, (0xFF0000, 0xFF00, 0, 0xFF000000)), (108, (0, 0, 0, 0))):
        both(bs.bmp(16, -16, 32, rows, comp=3, header=hdr, header_masks=hm), ig, cv2.IMREAD_GRAYSCALE)
    both(bs.bmp(16, -16, 32, rows, comp=0, header=108), ig, cv2.IMREAD_GRAYSCALE)
    # palette indices past clrused are black
    both(bs.bmp(3, 1, 8, bytes([0, 1, 2, 0]), palette=bytes([1, 2, 3, 0]), clrused=1), [[[3, 2, 1], [0, 0, 0], [0, 0, 0]]])
    # RLE8: skipped pixels take palette entry 0; a delta skips dx + dy * width pixels
    p = bytes([9, 9, 9, 0, 1, 1, 1, 0, 2, 2, 2, 0]) + bytes(1012)
    both(bs.bmp(4, 2, 8, bytes([1, 1, 0, 2, 2, 0, 1, 2, 0, 1]), comp=1, palette=p), [[[9] * 3] * 4, [[1] * 3, [9] * 3, [9] * 3, [2] * 3]])
    # RLE4: the delta's dy byte is ignored, end-of-bitmap before the last row acts as end-of-line
    p16 = bytes([0, 0, 0, 0] + [k * 16 for k in range(1, 16) for _ in range(4)])
    both(bs.bmp(4, 2, 4, bytes([1, 0x11, 0, 2, 1, 1, 1, 0x22, 0, 1, 4, 0x33, 0, 1]), comp=2, palette=p16),
         [[[48] * 3] * 4, [[16] * 3, [0] * 3, [32] * 3, [0] * 3]])
    # negative height is top-down, positive bottom-up
    rows2 = bytes([1, 2, 3, 0, 4, 5, 6, 0])
    both(bs.bmp(1, 2, 24, rows2), [[[6, 5, 4]], [[3, 2, 1]]])
    both(bs.bmp(1, -2, 24, rows2), [[[3, 2, 1]], [[6, 5, 4]]])
    # binary P5 with maxval 100 copies its samples; ASCII scales and saturates
    both(b"P5 2 1 100\n" + bytes([50, 200]), [[50, 200]], cv2.IMREAD_GRAYSCALE)
    both(b"P2 2 1 100\n50 200\n", [[127, 255]], cv2.IMREAD_GRAYSCALE)
    both(b"P3 1 1 255\n400 10 20\n", [[[255, 10, 20]]])
    # maxval above 255: v >> 8 whatever the maxval, binary and ASCII
    both(b"P2 3 1 1000\n255 256 1000\n", [[0, 1, 3]], cv2.IMREAD_GRAYSCALE)
    both(b"P5 3 1 1000\n" + struct.pack(">HHH", 255, 256, 1000), [[0, 1, 3]], cv2.IMREAD_GRAYSCALE)
    both(b"P5 2 1 65535\n" + struct.pack(">HH", 0xFFFF, 0x1234), [[255, 0x12]], cv2.IMREAD_GRAYSCALE)
    # P1 / P4: 1 is black, 0 white; P1 digits need no separator
    both(b"P1 3 1\n101", [[0, 255, 0]], cv2.IMREAD_GRAYSCALE)
    both(b"P4 3 1\n" + bytes([0b10100000]), [[0, 255, 0]], cv2.IMREAD_GRAYSCALE)
    # comments inside the header and the ASCII raster; any whitespace separates; one byte ends the header
    both(b"P5 #c\n2 #d\n1 255\n" + bytes([7, 8]), [[7, 8]], cv2.IMREAD_GRAYSCALE)
    both(b"P2 4 1 255\t1\x0b2 # x\r3\x0c4,", [[1, 2, 3, 4]], cv2.IMREAD_GRAYSCALE)
    both(b"P5 2 1 255  " + bytes([7]), [[32, 7]], cv2.IMREAD_GRAYSCALE)
    # a 32-bit BI_RGB BMP written by Pillow from RGBA: alpha dropped, not premultiplied
    if bs.Image is not None:
        rgba = np.array([[[200, 100, 50, 0], [10, 20, 30, 128]]], np.uint8)
        s = bs._pil(rgba, "RGBA", "BMP")
        assert struct.unpack_from("<H", s, 28)[0] == 32 and struct.unpack_from("<I", s, 30)[0] in (0, 3)
        both(s, rgba[..., :3])


REQUIRED = {"hdr40", "hdr52", "hdr56", "hdr64", "hdr108", "hdr124", "os2", "bmp1_c0", "bmp4_c0", "bmp8_c0", "bmp4_c2", "bmp8_c1",
            "bmp16_c0", "bmp16_c3", "bmp24_c0", "bmp32_c0", "bmp32_c3", "bf555", "bf565", "clrused", "top_down", "bottom_up", "rle_eol",
            "rle_delta", "rle_odd_absolute", "P1", "P2", "P3", "P4", "P5", "P6", "pnm_comment", "bf32_header_masks",
            "bf32_header_partial_masks"}


def test_corpus_covers_every_variant(emul, corpus):
    tags, layouts, maxvals, sizes = set(), set(), set(), set()
    for name, s in corpus:
        tags |= bs.kinds(s)
        rc, _, info = emul_decode(emul, s, RGB)
        assert rc == 0, name
        layouts.add((info[4], info[5], info[6], info[9], info[10]))
        if s[:1] == b"P" and s[1:2] not in (b"1", b"4"):
            maxvals.add("lt255" if info[11] and info[11] < 255 else "mid" if info[11] and 255 < info[11] < 65535 else
                        "65535" if info[11] == 65535 else "255" if info[11] == 255 else None)
        sizes.add((info[0], info[1]))
    assert REQUIRED <= tags, REQUIRED - tags
    # every (unpack, layout) the planner produces: direct palettes of 1 / 4 / 8 bits, 5-5-5, 5-6-5, 24 / 32-bit and PNM 8 / 16-bit
    # samples of 1 and 3 channels, RLE and P1 index planes, ASCII sample planes
    want = {(0, 0, 1, 0, 0), (0, 0, 4, 0, 0), (0, 0, 8, 0, 0), (0, 1, 0, 0, 0), (0, 2, 0, 0, 0), (0, 3, 0, 3, 3), (0, 3, 0, 4, 3),
            (0, 3, 0, 1, 1), (0, 3, 0, 2, 1), (0, 3, 0, 3, 3), (0, 3, 0, 6, 3), (1, 0, 8, 0, 0), (2, 0, 8, 0, 0), (3, 0, 8, 0, 0),
            (3, 3, 0, 1, 1), (3, 3, 0, 3, 3)}
    assert want <= layouts, want - layouts
    assert {"lt255", "255", "mid"} <= maxvals, maxvals                  # binary 65535 is checked in the rules; ASCII ranges here
    assert (1, 1) in sizes and (1920, 1080) in sizes


def test_emulated_core_rejects_every_corrupt_stream(emul):
    for name, s, status in bs.plan_corrupt():
        assert emul_decode(emul, s, RGB)[0] == status, name
        assert _cv2(s, cv2.IMREAD_COLOR) is None, name
    for name, s in bs.data_corrupt():
        assert emul_decode(emul, s, RGB)[0] == -1, name
        assert _cv2(s, cv2.IMREAD_COLOR) is None and _cv2(s, cv2.IMREAD_GRAYSCALE) is None, name


def test_streams_refused_here_that_cv2_decodes(emul):
    """documented deviation (DESIGN section 2): non-standard colour masks of a 32-bit V3 - V5 BITFIELDS header are refused"""
    for name, s, status in bs.refused_here_only():
        assert emul_decode(emul, s, RGB)[0] == status, name
        assert _cv2(s, cv2.IMREAD_COLOR) is not None, name


def test_formats_that_stay_out_are_not_bitmap_streams(emul):
    """P7 (PAM), PFM and JPEG 2000 are not taken by the BMP / PNM planner (cv2 decodes P7 and PFM; decoders.image refuses them)"""
    for s in (b"P7\nWIDTH 1\nHEIGHT 1\nDEPTH 1\nMAXVAL 255\nTUPLTYPE GRAYSCALE\nENDHDR\n\x07", b"Pf\n1 1\n-1.0\n\0\0\x80\x3f",
              b"\0\0\0\x0cjP  \r\n\x87\n", b"P8 1 1 255\n\x00", b"P5x1 1 255\n\x00"):
        assert emul_decode(emul, s, RGB)[0] == bs.BAD_DATA


MUTATE = r"""
import ctypes as C, sys
import numpy as np
sys.path.insert(0, %(tests)r)
import bitmap_streams as bs
lib = C.CDLL(%(lib)r)
lib.emul_bitmap_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
rng = np.random.default_rng(11)
seeds = [s for n, s in bs.corpus() if len(s) < 200000][::2] + [s for _, s, _ in bs.plan_corrupt() + bs.refused_here_only()]
seeds += [s for _, s in bs.data_corrupt()]
n = 0
for it in range(%(n)d):
    s = bytearray(seeds[it %% len(seeds)])
    for _ in range(int(rng.integers(1, 6))):
        k = int(rng.integers(0, 4))
        i = int(rng.integers(0, len(s) + 1))
        if k == 0 and i < len(s): s[i] ^= 1 << int(rng.integers(0, 8))
        elif k == 1 and i < len(s): s[i] = int(rng.integers(0, 256))
        elif k == 2: del s[i:i + int(rng.integers(1, 16))]
        else: s[i:i] = bytes(rng.integers(0, 256, int(rng.integers(1, 8))).astype(np.uint8))
    info = (C.c_int * 12)()
    b = bytes(s)
    if lib.emul_bitmap_decode(b, len(b), 0, None, info) == 0 and info[0] * info[1] <= 1 << 22:
        out = np.zeros(info[0] * info[1] * 3 + 1, np.uint8)
        lib.emul_bitmap_decode(b, len(b), int(rng.integers(0, 3)), out.ctypes.data + int(rng.integers(0, 2)), info)
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
