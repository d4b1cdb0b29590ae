"""CPU tests of the boundary: the C-ABI library loads, exports every symbol include/dali_b200.h declares, and
its host-only entry points (header parse, matrix helpers, argument validation) behave -- no kernel is launched."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from dali_b200 import capi
from oracle import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    hdr = open(os.path.join(ROOT, "include", "dali_b200.h")).read()
    declared = set(re.findall(r"\b(dalib200[A-Za-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 40
    lib = capi.lib()
    missing = [s for s in sorted(declared) if not hasattr(lib, s)]
    assert not missing, missing
    assert set(capi.EXPORTS) <= declared
    assert lib.dalib200GetVersion() >= 100


def test_jpeg_get_info_matches_oracle_parser(golden_dir):
    g = np.load(os.path.join(golden_dir, "jpeg_cv2.npz"))
    n = len([k for k in g.files if k.startswith("enc_")])
    for i in range(n):
        enc = g[f"enc_{i}"]
        info = capi.JpegInfo()
        capi.check(capi.lib().dalib200JpegGetInfo(enc.ctypes.data_as(C.c_void_p), C.c_size_t(enc.size), C.byref(info)))
        oi = po.jpeg_info(enc.tobytes())
        assert (info.width, info.height, info.components) == (oi["width"], oi["height"], oi["ncomp"])
        assert info.height == g[f"dec_{i}"].shape[0] and info.width == g[f"dec_{i}"].shape[1]
        assert info.restart_interval == oi["restart_interval"]


def test_jpeg_get_info_rejects_garbage():
    bad = np.frombuffer(b"definitely not a jpeg", np.uint8)
    info = capi.JpegInfo()
    rc = capi.lib().dalib200JpegGetInfo(bad.ctypes.data_as(C.c_void_p), C.c_size_t(bad.size), C.byref(info))
    assert rc != 0 and b"SOI" in capi.lib().dalib200GetLastError()


def test_resample_stream_info_rejects_bad_arguments():
    info = (C.c_int32 * 4)()
    assert capi.lib().dalib200ResamplePlanGetStreamInfo(None, 0, info) == 1
    assert b"GetStreamInfo" in capi.lib().dalib200GetLastError()


def test_color_twist_matrix_matches_reference_composition():
    rng = np.random.default_rng(5)
    for _ in range(300):
        h, s, v, b, c = rng.uniform(-180, 180), rng.uniform(0, 2), rng.uniform(0, 2), rng.uniform(0.5, 1.5), rng.uniform(0.5, 1.5)
        M, T = np.empty(9, np.float32), np.empty(3, np.float32)
        capi.lib().dalib200ColorTwistMatrix(C.c_float(h), C.c_float(s), C.c_float(v), C.c_float(b), C.c_float(c), C.c_float(128.0),
                                           M.ctypes.data_as(C.c_void_p), T.ctypes.data_as(C.c_void_p))
        Mo, To = po.color_twist_matrix(h, s, v, b, c, 128.0)
        assert np.array_equal(M.reshape(3, 3), Mo) and np.array_equal(T, To)


def test_affine_inverse_matches_reference():
    rng = np.random.default_rng(6)
    for _ in range(300):
        M = rng.normal(0, 1, 6).astype(np.float32)
        out = np.empty(6, np.float32)
        capi.lib().dalib200AffineInverse(M.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p))
        assert np.array_equal(out.reshape(2, 3), po.affine_inv(M))


def test_hann_window_matches_reference():
    for n in (400, 512, 1024):
        w = np.empty(n, np.float32)
        capi.lib().dalib200HannWindow(w.ctypes.data_as(C.c_void_p), n)
        assert np.array_equal(w, po.hann_window(n))


def test_missing_library_is_an_error_not_a_fallback(monkeypatch):
    monkeypatch.setattr(capi, "_lib", None)
    monkeypatch.setattr(capi, "LIB_PATH", "/nonexistent/libdali_b200.so")
    with pytest.raises(capi.DaliB200Error):
        capi.lib()
