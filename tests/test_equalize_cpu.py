"""fn.experimental.equalize without a GPU:
  * tests/equalize_ref.py pinned to cv2.equalizeHist on random, narrow, bimodal and flat planes, the half-to-even tie, and a plane of
    more than 2^24 pixels on which rounding the running sum to float changes a table entry;
  * the type, layout and shape rules through the operator's plan set-up (dalihTestEqualize), every refusal included;
  * the planner and the kernel bodies compiled for the host (tools/emul/equalize_emul.cc), every work item and thread run in reverse
    order, against equalize_ref: every layout and the empty layout, 1 to 16 channels, zero-size samples and frames, frames over several
    work items, inputs and outputs at every byte offset;
  * random cases under ASan + UBSan."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from dali_b200 import backend

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import equalize_ref as er  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tools", "emul", "equalize_emul.cc")
P64 = C.POINTER(C.c_int64)
MAX_C = 16


def test_reference_is_cv2_equalize_hist():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    for t in range(200):
        h, w = (int(v) for v in rng.integers(1, 300, 2))
        kind = t % 5
        if kind == 0:
            x = rng.integers(0, 256, (h, w), dtype=np.uint8)
        elif kind == 1:
            x = rng.integers(50, 60, (h, w), dtype=np.uint8)
        elif kind == 2:
            x = np.clip(rng.normal(128, 3, (h, w)), 0, 255).astype(np.uint8)
        elif kind == 3:
            x = rng.choice(np.array([3, 200], np.uint8), (h, w))
        else:
            x = np.full((h, w), int(rng.integers(0, 256)), np.uint8)
        assert np.array_equal(er.equalize_plane(x), cv2.equalizeHist(x)), t
    # ties round half to even: 10 pixels of 0, one of 1 (0.5 -> 0), two of 2 (1.5 -> 2), 507 of 255
    x = np.array([0] * 10 + [1] + [2] * 2 + [255] * 507, np.uint8).reshape(1, -1)
    e = er.equalize_plane(x)
    assert np.array_equal(e, cv2.equalizeHist(x)) and (e[0, 10], e[0, 11]) == (0, 2)


def test_float_sum_rounding_on_a_plane_above_2_pow_24():
    cv2 = pytest.importorskip("cv2")
    x, d, s = er.big_plane()
    scale = np.float32(255) / np.float32(d)
    assert np.rint(np.float64(s) * np.float64(scale)) == 163
    lut = er.plane_lut(x)
    assert lut[1] == 164
    assert np.array_equal(cv2.equalizeHist(x), lut[x])


# ---- type, layout and shape rules (the operator's plan set-up)
def rule(shapes, layout="", in_type=0):
    s = np.ascontiguousarray(shapes, np.int64).reshape(len(shapes), -1)
    buf = C.create_string_buffer(16)
    rc = backend.lib().dalihTestEqualize(in_type, s.shape[0], s.shape[1], s.ctypes.data_as(P64), layout.encode(), buf, 16)
    return backend.lib().dalihLastError().decode() if rc else buf.value.decode()


def test_layouts_and_empty_layout_by_rank():
    for lay in er.LAYOUTS:
        shape = [{"F": 2, "H": 3, "W": 4, "C": 3}[a] for a in lay]
        assert rule([shape], lay) == lay
    assert rule([[3, 4]]) == "HW" and rule([[3, 4, 3]]) == "HWC" and rule([[2, 3, 4, 3]]) == "FHWC"
    assert rule([[0, 4, 3], [3, 0, 3], [3, 4, 0]], "HWC") == "HWC"          # empty samples are accepted
    assert rule([[0, 3, 4, 3]], "FHWC") == "FHWC"
    assert rule([[3, 4, MAX_C]], "HWC") == "HWC" and rule([[MAX_C, 3, 4]], "CHW") == "CHW"


def test_refusals_name_the_problem():
    for t, name in ((1, "UINT16"), (4, "INT8"), (9, "FLOAT"), (11, "BOOL")):
        assert f"must be UINT8, got {name}" in rule([[3, 4]], "HW", t)
    assert "cannot infer the layout of 5-dimensional input 0" in rule([[1, 2, 3, 4, 3]])
    assert "cannot infer the layout of 1-dimensional input 0" in rule([[3]])
    assert 'layout "NHWC" of input 0 is not supported' in rule([[1, 3, 4, 3]], "NHWC")
    assert 'layout "HWC" but 2 dimensions' in rule([[3, 4]], "HWC")
    assert f"sample 1 of input 0 has {MAX_C + 1} channels" in rule([[3, 4, 3], [3, 4, MAX_C + 1]], "HWC")
    assert f"sample 0 of input 0 has {MAX_C + 1} channels" in rule([[MAX_C + 1, 3, 4]], "CHW")
    assert "sample 1 of input 0 has a plane of 46341 x 46341 pixels" in rule([[2, 2], [46341, 46341]], "HW")
    assert rule([[46340, 46341]], "HW") == "HW"                             # 2 147 441 940 pixels: one plane below 2^31
    assert "negative extent" in rule([[3, -4]], "HW")


# ---- the host build
@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    so = str(tmp_path_factory.mktemp("eq") / "equalize_emul.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", SRC, "-o", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


def placed(x, off, keep, fill=0):
    buf = np.full(x.nbytes + 64, fill, np.uint8)
    base = (-buf.ctypes.data) % 16 + 16 + off
    buf[base:base + x.nbytes] = x.reshape(-1)
    keep.append((buf, base, x.nbytes))
    return buf.ctypes.data + base


def run(lib, xs, layout="", offs=(0, 0)):
    """outputs of the host build, sample i's input (offs[0] + i) % 16 and output (offs[1] + 3 i) % 16 bytes past a 16-byte boundary;
    also the planner's (items per frame, channels, stride, items) of each sample"""
    n, nd = len(xs), xs[0].ndim
    shp = (C.c_int64 * (n * nd))(*[e for x in xs for e in x.shape])
    geom = (C.c_int64 * (4 * n))()
    err = C.create_string_buffer(512)
    ins, outs = [], []
    ip = (C.c_void_p * n)(*[placed(x, (offs[0] + i) % 16, ins) for i, x in enumerate(xs)])
    op = (C.c_void_p * n)(*[placed(np.zeros(x.shape, np.uint8), (offs[1] + 3 * i) % 16, outs, 0xA5) for i, x in enumerate(xs)])
    assert lib.emul_equalize(0, n, nd, shp, layout.encode(), ip, op, geom, err, 512) == 0, err.value
    res = []
    for (buf, base, nb), x in zip(outs, xs):
        assert np.all(buf[:base] == 0xA5) and np.all(buf[base + nb:] == 0xA5), "a write outside the output"
        res.append(buf[base:base + nb].reshape(x.shape))
    return res, [tuple(geom[4 * i:4 * i + 4]) for i in range(n)]


def sample(rng, shape, kind=None):
    kind = int(rng.integers(0, 4)) if kind is None else kind
    if kind == 0:
        return rng.integers(0, 256, shape, dtype=np.uint8)
    if kind == 1:
        return rng.integers(100, 110, shape, dtype=np.uint8)
    if kind == 2:
        return rng.choice(np.array([7, 240], np.uint8), shape)
    return np.full(shape, int(rng.integers(0, 256)), np.uint8)


def test_every_layout_and_the_empty_layout(emul):
    rng = np.random.default_rng(1)
    for lay in er.LAYOUTS + ("",):
        named = lay or "FHWC"
        for c in (1, 3, 4):
            ext = {"F": 3, "H": 37, "W": 61, "C": c}
            xs = [sample(rng, [ext[a] for a in named]), sample(rng, [max(1, ext[a] // 2) for a in named], 3),
                  sample(rng, [ext[a] if a in "CF" else ext[a] * 5 for a in named])]
            got, geom = run(emul, xs, lay, (int(rng.integers(0, 16)), int(rng.integers(0, 16))))
            for i, x in enumerate(xs):
                assert np.array_equal(got[i], er.equalize(x, lay)), (lay, c, i)
                stride = 1 if "C" not in named or named.index("C") > named.index("H") else x.shape[named.index("H")] * x.shape[named.index("W")]
                assert geom[i][1:3] == ((x.shape[named.index("C")] if "C" in named else 1), stride), (lay, geom[i])


def test_channels_1_to_the_limit_and_frames_over_several_items(emul):
    rng = np.random.default_rng(2)
    for c in range(1, MAX_C + 1):
        for lay in ("HWC", "CHW"):
            shape = (c, 97, 131) if lay == "CHW" else (97, 131, c)
            xs = [sample(rng, shape, 0), sample(rng, shape, 2)]
            got, geom = run(emul, xs, lay, (c, 2 * c))
            for x, g in zip(xs, got):
                assert np.array_equal(g, er.equalize(x, lay)), (c, lay)
            assert geom[0][0] == -(-x.size // 32768)                       # items per frame: 32 KiB each
    x = sample(rng, (2, 300, 301, 3), 0)                                  # 271 KiB frames: 9 items each
    got, geom = run(emul, [x], "FHWC", (5, 11))
    assert geom[0][0] == 9 and geom[0][3] == 18 and np.array_equal(got[0], er.equalize(x, "FHWC"))


def test_zero_size_samples_and_frames(emul):
    rng = np.random.default_rng(3)
    xs = [np.zeros((0, 5, 3), np.uint8), sample(rng, (4, 5, 3)), np.zeros((4, 0, 3), np.uint8), np.zeros((4, 5, 0), np.uint8),
          sample(rng, (1, 1, 3))]
    got, geom = run(emul, xs, "HWC")
    for x, g, gm in zip(xs, got, geom):
        assert np.array_equal(g, er.equalize(x, "HWC"))
        assert (gm[3] == 0) == (x.size == 0)
    fs = [np.zeros((0, 4, 5), np.uint8), sample(rng, (3, 4, 5)), np.zeros((2, 0, 5), np.uint8)]
    got, geom = run(emul, fs, "FHW")
    assert [g[3] for g in geom] == [0, 3, 0] and np.array_equal(got[1], er.equalize(fs[1], "FHW"))


def test_every_byte_offset(emul):
    rng = np.random.default_rng(4)
    xs = [sample(rng, (45, 29, 3), 0), sample(rng, (3, 45, 29), 0)]
    for a in range(16):
        for b in (a, (a + 5) % 16):
            for lay, x in (("HWC", xs[0]), ("CHW", xs[1])):
                got, _ = run(emul, [x, x], lay, (a, b))
                want = er.equalize(x, lay)
                assert np.array_equal(got[0], want) and np.array_equal(got[1], want), (lay, a, b)


def test_random_cases_under_sanitizers(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path / "eq_fuzz")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-DEQUALIZE_EMUL_MAIN", SRC, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    for seed in (1, 2, 3):
        r = subprocess.run([exe, "250", str(seed)], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0 and r.stdout.strip() == "ok 250", (r.stdout[-2000:], r.stderr[-3000:])
