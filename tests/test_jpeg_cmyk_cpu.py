"""CPU tests of 4-component (CMYK / YCCK) JPEG: the oracle's decode (tests/jpeg_cmyk_oracle.c) against cv2.imdecode, COLOR and
GRAYSCALE, on the Pillow fixtures (tests/golden/jpeg_cmyk.npz) and on Photoshop-layout YCCK streams (tests/jpeg_cmyk_streams.py); and
the product's multi-scan planner and scan decoder (compiled for the host by tools/emul/jpeg_prog_emul.cc) on progressive and
one-scan-per-component 4-component streams."""
import os

import numpy as np
import pytest

from oracle import pyoracle as po

import jpeg_cmyk_oracle as cmyk_oracle
from jpeg_cmyk_streams import multiscan_expected, one_scan_per_component, photoshop_ycck
from test_jpeg_prog_cpu import decode
from test_jpeg_prog_cpu import emul  # noqa: F401  (fixture)


@pytest.fixture(scope="module")
def cmyk(golden_dir):
    gz = np.load(os.path.join(golden_dir, "jpeg_cmyk.npz"))
    n = len([k for k in gz.files if k.startswith("enc_")])
    return [dict(name=str(gz[f"name_{i}"]), enc=gz[f"enc_{i}"].tobytes(), color=gz[f"color_{i}"], gray=gz[f"gray_{i}"]) for i in range(n)]


def test_fixture_layouts(cmyk):
    assert len(cmyk) == 72
    for f in cmyk:
        info = po.jpeg_info(f["enc"])
        sub = int(f["name"].split("_")[1][1])
        assert info["ncomp"] == 4 and info["progressive"] == ("_prog_" in f["name"]), f["name"]
        assert (info["hs"], info["vs"]) == ([1, 1, 1, 1], [1, 1, 1, 1]) if sub == 0 else \
               (info["hs"], info["vs"]) == ([2, 1, 1, 1], [1 if sub == 1 else 2, 1, 1, 1]), (f["name"], info)
        assert (b"Adobe" in f["enc"]) == (not f["name"].startswith("noadobe"))


def test_oracle_equals_cv2_on_pillow_streams(cmyk):
    n = 0
    for f in cmyk:
        if "_prog_" in f["name"]:
            continue                                           # the oracle decodes baseline streams; the twins' coefficients are compared below
        assert np.array_equal(cmyk_oracle.decode(f["enc"]), f["color"][..., ::-1]), f["name"]
        assert np.array_equal(cmyk_oracle.decode_gray(f["enc"]), f["gray"]), f["name"]
        n += 1
    assert n == 36


def test_oracle_equals_cv2_on_photoshop_ycck_layout():
    import cv2
    for (h, w, rst, transform) in [(1, 1, 0, 2), (17, 9, 0, 2), (61, 77, 3, 2), (250, 3, 0, 0), (33, 250, 1, 2), (1080, 1920, 0, 2),
                                   (1080, 1920, 17, 2)]:
        s = photoshop_ycck(h, w, h + w + rst, rst=rst, transform=transform)
        info = po.jpeg_info(s)
        assert info["ncomp"] == 4 and info["hs"] == [2, 1, 1, 2] and info["vs"] == [2, 1, 1, 2] and info["restart_interval"] == rst
        a = np.frombuffer(s, np.uint8)
        assert np.array_equal(cmyk_oracle.decode(s), cv2.imdecode(a, cv2.IMREAD_COLOR)[..., ::-1]), (h, w, rst, transform)
        assert np.array_equal(cmyk_oracle.decode_gray(s), cv2.imdecode(a, cv2.IMREAD_GRAYSCALE)), (h, w, rst, transform)


def test_progressive_cmyk_coefficients_equal_the_baseline_twin(emul, cmyk):  # noqa: F811
    base = {f["name"]: f["enc"] for f in cmyk if "_base_" in f["name"]}
    n = 0
    for f in cmyk:
        if "_prog_" not in f["name"]:
            continue
        rc, got, info = decode(emul, f["enc"])
        assert rc == 0 and info["ncomp"] == 4 and info["truncated"] == 0, (f["name"], rc, info)
        assert np.array_equal(got, cmyk_oracle.mcu_order(base[f["name"].replace("_prog_", "_base_")])), f["name"]
        n += 1
    assert n == 36


def test_one_scan_per_component_cmyk(emul, cmyk):  # noqa: F811
    import cv2
    streams = [f["enc"] for f in cmyk if "_base_" in f["name"] and f["name"].endswith(("61x77", "17x9"))]
    streams += [photoshop_ycck(40, 56, 7), photoshop_ycck(17, 33, 8, transform=0)]
    for s in streams:
        for rst in (0, 5):
            multi, hblk, wblk = one_scan_per_component(s, rst)
            a, b = np.frombuffer(multi, np.uint8), np.frombuffer(s, np.uint8)
            assert np.array_equal(cv2.imdecode(a, cv2.IMREAD_COLOR), cv2.imdecode(b, cv2.IMREAD_COLOR))
            rc, got, info = decode(emul, multi)
            assert rc == 0 and info["nscans"] == 4 and info["nwaves"] == 1 and info["truncated"] == 0, (rc, info)
            assert np.array_equal(got, multiscan_expected(s, hblk, wblk))


def test_scan_interleaving_a_subset_of_four_components_is_rejected(emul, cmyk):  # noqa: F811
    prog = bytearray(next(f["enc"] for f in cmyk if f["name"] == "cmyk_s0_prog_61x77"))
    i = prog.find(b"\xff\xda")
    assert prog[i + 4] == 4                                   # the first (DC) scan interleaves all four components
    three = prog[:i + 2] + bytes([0, 12, 3]) + prog[i + 5:i + 11] + prog[i + 13:]
    assert decode(emul, bytes(three))[0] == 2                 # DALIB200_ERROR_UNSUPPORTED
