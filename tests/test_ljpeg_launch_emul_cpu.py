"""The launch path of the lossless JPEG stage, executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc is preloaded in place of the CUDA
runtime, "device" memory is host memory, and U2 / U3 and the kernels of ljpeg.cu run on the host through the same bodies the device runs
(ljpeg_core.h), the chains of ljpeg_sync in reverse order.  Lossless-only batches (no baseline entropy kernel), batches mixed with PNG, TIFF,
WebP and BMP samples, plan reuse with growing sizes, ROI windows, corrupt samples and JpegGetInfo on lossless streams."""
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
import ljpeg_streams as ls
import png_streams as ps
import webp_streams as ws

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
counts = lambda: [stub.emul_launch_count(k) for k in range(21)]
def want(exp, ot):
    if ot == capi.GRAY:
        if exp.shape[2] == 1:
            return exp
        a = exp.astype(np.int64)
        return ((a[..., 0] * 19595 + a[..., 1] * 38470 + a[..., 2] * 7471 + 32768) >> 16).astype(np.uint8)[..., None]
    rgb = np.repeat(exp, 3, axis=2) if exp.shape[2] == 1 else exp
    return rgb[..., ::-1] if ot == capi.BGR else rgb

corpus = ls.corpus()
streams = [s for _, s, _, _ in corpus]
# lossless-only batches: every output type; no baseline entropy kernel runs, U2 / U3 and all five ljpeg kernels do
for ot in (capi.RGB, capi.BGR, capi.GRAY):
    c0 = counts()
    outs, status = g.jpeg_decode_ex(streams, output_type=ot, adjust_orientation=False)
    c1 = counts()
    assert status == [0] * len(streams)
    for (name, _, exp, _), o in zip(corpus, outs):
        assert np.array_equal(o, want(exp, ot)), (name, ot)
    assert all(c1[k] > c0[k] for k in range(14, 20)), (c0, c1)
    assert c1[:14] == c0[:14], (c0, c1)
# JpegGetInfo: components 1 or 3, subsampling 0x11
for name, s, exp, _ in corpus[:20]:
    info = capi.JpegInfo()
    b = np.frombuffer(s, np.uint8)
    capi.check(capi.lib().dalib200JpegGetInfo(b.ctypes.data_as(C.POINTER(C.c_uint8)), b.size, C.byref(info)))
    assert (info.height, info.width, info.components, info.subsampling) == (exp.shape[0], exp.shape[1], exp.shape[2], 0x11), name
# mixed with PNG, WebP and BMP samples
lossless = [ls.encode(ls.image(50, 61, 3, 8, 70), pred=5), ls.encode(ls.image(33, 17, 1, 6, 71), P=6, Pt=2, restart=17 * 4)]
others = [ps.encode(ps.samples(40, 50, 2, 8, 80), 2, 8, filters="mixed"), ws.cv2_webp(ws.image(40, 56, 7), 70),
          bs.bmp(31, 17, 24, bs.rows(bs.image(17, 31, 1), 24))]
mixed = [others[0], lossless[0], others[1], lossless[1], others[2]]
solo = [g.jpeg_decode([s])[0][0] for s in mixed]
outs, status = g.jpeg_decode(mixed)
assert status == [0] * 5
for k, (o, w) in enumerate(zip(outs, solo)):
    assert np.array_equal(o, w), k
assert np.array_equal(outs[1], ls.image(50, 61, 3, 8, 70))
# plan reuse with growing sizes
plan = capi.Plan("Jpeg", 3)
for k, (h, w) in enumerate([(8, 8), (40, 60), (17, 130), (90, 70)]):
    imgs = [ls.image(h, w, 3, 8, k), ls.image(h, w, 1, 8, k + 10), ls.image(h, w, 3, 7, k + 20)]
    ss = [ls.encode(imgs[0], pred=1 + k), ls.encode(imgs[1], restart=w, tables="opt"), ls.encode(imgs[2], P=7, pred=7 - k)]
    outs, status = g.jpeg_decode(ss, plan=plan)
    assert status == [0] * 3
    for o, a in zip(outs, imgs):
        assert np.array_equal(o, want(a, capi.RGB)), (h, w)
# ROI windows
img = ls.image(37, 53, 3, 8, 60)
s = ls.encode(img, pred=4, restart=53 * 5)
for r in [(0, 0, 53, 37), (5, 7, 20, 30), (52, 36, 53, 37)]:
    outs, status = g.jpeg_decode_ex([s], rois=[r], adjust_orientation=False)
    assert status == [0] and np.array_equal(outs[0], img[r[1]:r[3], r[0]:r[2]]), r
# corrupt samples set only their own status
good = ls.encode(ls.image(20, 30, 3, 8, 80), restart=30 * 2)
for name, bad, kind in ls.corrupt():
    outs, status = g.jpeg_decode([good, bad, good])
    assert status == [0, 1, 0], name
    assert np.array_equal(outs[0], ls.image(20, 30, 3, 8, 80)) and np.array_equal(outs[2], outs[0]), name
print("ljpeg-emul-ok")
"""


def test_ljpeg_launch_path(emul_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=1500, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "ljpeg-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
