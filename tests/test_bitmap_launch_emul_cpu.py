"""The launch path of the BMP / PNM stage, executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc is preloaded in place of the CUDA
runtime, and the launches of bitmap_unpack_kernel / bitmap_color_kernel run on the host through the same host/device functions the
device code consists of (dali_b200/csrc/bitmap_core.h); every other kernel is a no-op.  Everything around the launches is the library's
real code -- plan set-up of BMP / PNM samples beside JPEG, PNG, TIFF and WebP ones, staging of the pixel arrays and rasters, the
descriptor arena with the unpack list, the forked stream, the plane scratch, the serial-lane geometry, the window pointers and the group
prefix -- so the outputs are compared with cv2 for real:
  * a BMP / PNM-only batch has no JPEG units: no JPEG kernel may be launched with an empty grid (the stub reports that as the runtime's
    sticky error, which the launch returns), and bitmap_unpack runs only when an RLE or ASCII image is in the batch;
  * samples mixed with baseline and progressive JPEG, PNG, TIFF and WebP samples, more serial images than resident warps, plan reuse
    with growing sizes, ROI windows;
  * a corrupt RLE or ASCII sample sets its own status word only."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul_env(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    stub = str(tmp_path_factory.mktemp("emul") / "cuda_emul_stub.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include",
                        os.path.join(ROOT, "tools", "emul", "cuda_emul_stub.cc"), "-o", stub, "-ldl"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return dict(os.environ, DALIB200_DRYRUN="emul", LD_PRELOAD=stub, EMUL_STUB=stub)


SCRIPT = r"""
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests"))
import conftest                      # DALIB200_DRYRUN=emul: "device" tensors are host memory
import cv2
import gpu_helpers as g
from dali_b200 import capi
import bitmap_streams as bs
import png_oracle as pngo
import png_streams as ps
import tiff_oracle as to
import tiff_streams as ts
import webp_streams as ws

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
counts = lambda: [stub.emul_launch_count(k) for k in range(14)]
def cv(s, ot):
    if ot == capi.GRAY:
        return cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_GRAYSCALE)[..., None]
    bgr = cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR)
    return bgr if ot == capi.BGR else bgr[..., ::-1]
def check(outs, streams, ot=capi.RGB):
    for k, (o, s) in enumerate(zip(outs, streams)):
        assert np.array_equal(o, cv(s, ot)), (k, ot)

corpus = [s for n, s in bs.corpus() if "1080p" not in n]
direct = [s for s in corpus if s[:2] in (b"P4", b"P5", b"P6") or (s[:2] == b"BM" and s[30:31] not in (b"\1", b"\2"))]
# BMP / PNM only: no progressive JPEG, PNG, TIFF, WebP or 3-D resize kernel, and no bitmap_unpack without an RLE or ASCII image
for ot in (capi.RGB, capi.BGR, capi.GRAY):
    c0 = counts()
    outs, status = g.jpeg_decode(corpus, output_type=ot)
    assert status == [0] * len(corpus)
    check(outs, corpus, ot)
    assert [b - a for a, b in zip(c0, counts())] == [0] * 12 + [1, 1], (c0, counts())
c0 = counts()
outs, status = g.jpeg_decode(direct[:40])
assert status == [0] * 40
check(outs, direct[:40])
assert [b - a for a, b in zip(c0, counts())] == [0] * 13 + [1], (c0, counts())
# more serial images than resident warps (132 SMs x 32 = 4224): several lanes per warp, grid-stride over the unpack list
many = [bs.rle_bmp(3 + j %% 5, 2, 8, j) if j %% 2 else bs.pnm(2, bs.image(2, 3, j)[..., 0], 255) for j in range(4500)]
outs, status = g.jpeg_decode(many)
assert status == [0] * len(many)
check(outs[::97], many[::97])
# mixed with baseline and progressive JPEG, PNG, TIFF and WebP samples (JPEG kernels are no-ops here: the others are compared)
jpg = cv2.imencode(".jpg", g.synth_image(96, 128, 1))[1].tobytes()
prog = cv2.imencode(".jpg", g.synth_image(64, 80, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
png = ps.encode(ps.samples(30, 41, 2, 8, 5), 2, 8, filters="mixed")
tif = ts.encode(ts.samples(20, 30, 3, 8, 6), 2, 8, 5, 2, rows_per_strip=3)
webp = ws.cv2_webp(ws.image(40, 56, 7), 70)
bm = [corpus[3], corpus[40], corpus[77], corpus[120], corpus[200]]
streams = [jpg, bm[0], png, prog, bm[1], tif, bm[2], webp, bm[3], jpg, bm[4]]
outs, status = g.jpeg_decode(streams)
assert status == [0] * len(streams)
check([outs[k] for k in (1, 4, 6, 8, 10)], bm)
assert np.array_equal(outs[2], pngo.decode(png)[0]) and np.array_equal(outs[5], to.decode(tif)[0])
# plan reuse with growing sizes, and corrupt RLE / ASCII samples beside good ones
plan = capi.Plan("Jpeg", 4)
for k, (h, w) in enumerate([(8, 8), (60, 90), (17, 200), (120, 160)]):
    ss = [bs.rle_bmp(w, h, 8, k), bs.bmp(w, -h, 24, bs.rows(bs.image(h, w, k), 24, True)), bs.pnm(3, bs.image(h, w, k), 255),
          bs.rle_bmp(w + 1, h, 4, k)]
    outs, status = g.jpeg_decode(ss, plan=plan)
    assert status == [0] * 4
    check(outs, ss)
bad = dict(bs.data_corrupt())
ss = [corpus[5], bad["rle8_no_eob"], corpus[6], bad["p2_bad_char"], jpg, bad["rle4_run_past_row"]]
outs, status = g.jpeg_decode(ss, plan=capi.Plan("Jpeg", 6))
assert status == [0, 1, 0, 1, 0, 1], status
check([outs[0], outs[2]], [corpus[5], corpus[6]])
# ROI windows at any edge, written directly (orientation 1, u8, RGB) and through the post pass (float)
rng = np.random.default_rng(3)
sel = [s for s in corpus if min(cv(s, capi.RGB).shape[:2]) > 4][::9][:16]
rois = []
for s in sel:
    H, W = cv(s, capi.RGB).shape[:2]
    x0, y0 = int(rng.integers(0, W - 1)), int(rng.integers(0, H - 1))
    rois.append((x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1))))
for ot in (capi.RGB, capi.GRAY):
    outs, status = g.jpeg_decode_ex(sel, rois=rois, output_type=ot, adjust_orientation=False)
    assert status == [0] * len(sel)
    for o, s, r in zip(outs, sel, rois):
        assert np.array_equal(o, cv(s, ot)[r[1]:r[3], r[0]:r[2]]), r
print("bitmap-emul-ok")
"""


def test_bitmap_launch_path_decodes_bitmap_only_and_mixed_batches(emul_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=1500, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "bitmap-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
