"""CPU tests of the encode half of fn.jpeg_compression_distortion: the PRODUCT's planner and forward-DCT bodies
(dali_b200/csrc/jpeg_distort_plan.h + jpeg_distort_core.h -- the body of the jpeg_distort_fdct kernel) compiled for the host by
tools/emul/jpeg_distort_emul.cc.  Every block of all three components, dummy blocks included, must equal the coefficients cv2.imencode
writes (read back by the oracle), and the quantisation tables must equal the stream's DQT."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import jpeg_distort_cases as jc  # noqa: E402

cv2 = pytest.importorskip("cv2")
EMUL = os.path.join(ROOT, "tools", "emul", "jpeg_distort_emul.cc")


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp_path_factory.mktemp("jd_emul") / "libjdemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-I/usr/local/cuda/include", EMUL, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(out)
    lib.emul_jd_coefficients.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _coefs(lib, rgb, q):
    h, w = rgb.shape[:2]
    out = np.zeros(((w + 15) // 16) * ((h + 15) // 16) * 6 * 64, np.int16)
    qt = np.zeros(128, np.uint16)
    rgb = np.ascontiguousarray(rgb)
    assert lib.emul_jd_coefficients(rgb.ctypes.data, h, w, q, out.ctypes.data, qt.ctypes.data) == 0
    return out, qt


def test_coefficients_equal_cv2_imencode(emul):
    n = 0
    for si, (h, w) in enumerate(jc.SIZES):
        for ki, kind in enumerate(jc.KINDS):
            for q in jc.QUALITIES:
                rgb = jc.image(h, w, kind, 1000 * si + 100 * ki + q)
                got, _ = _coefs(emul, rgb, q)
                want = jc.mcu_coefficients(jc.encode(rgb, q))
                assert np.array_equal(got, want), (h, w, kind, q, int(np.flatnonzero(got != want)[0]))
                n += 1
    assert n == len(jc.SIZES) * len(jc.KINDS) * len(jc.QUALITIES)


@pytest.mark.parametrize("q", [50, 95])
def test_coefficients_1080p(emul, q):
    rgb = jc.image(1080, 1920, "smooth", q)
    got, _ = _coefs(emul, rgb, q)
    assert np.array_equal(got, jc.mcu_coefficients(jc.encode(rgb, q)))


def test_quant_tables_equal_stream_dqt(emul):
    rgb = jc.image(16, 16, "noise", 0)
    for q in range(1, 101):
        _, qt = _coefs(emul, rgb, q)
        dqt = jc.dqt_tables(jc.encode(rgb, q))
        assert np.array_equal(qt[:64], dqt[0]) and np.array_equal(qt[64:], dqt[1]), q


def test_rejected_arguments(emul):
    px = np.zeros(3, np.uint8)
    for h, w, q in [(1, 1, 0), (1, 1, 101), (1, 1, -5), (0, 5, 50), (5, 0, 50), (65501, 1, 50), (1, 65501, 50), (65500, 65500, 50)]:
        assert emul.emul_jd_coefficients(px.ctypes.data, h, w, q, None, None) == 1, (h, w, q)    # DALIB200_ERROR_INVALID_ARGUMENT
    assert emul.emul_jd_coefficients(px.ctypes.data, 65500, 1, 50, None, None) == 0
