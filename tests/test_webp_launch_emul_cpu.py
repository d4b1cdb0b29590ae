"""The launch path of the WebP stage, executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc is preloaded in place of the CUDA runtime,
and the launches of webp_entropy / webp_recon / webp_filter / webp_color run on the host through the same host/device functions the
device code consists of (dali_b200/csrc/webp_core.h); the macroblocks of each wavefront diagonal run in reverse thread order.  Every
other kernel is a no-op.  Everything around the launches is the library's real code -- plan set-up of WebP samples beside JPEG, PNG and
TIFF ones, staging of the VP8 payloads, the descriptor arena, the forked stream, the scratch layout, the window pointers and pixel
prefix -- so the WebP outputs are compared with cv2.imdecode for real:
  * a WebP-only batch has no JPEG units: no JPEG kernel may be launched with an empty grid;
  * WebP samples mixed with baseline and progressive JPEG, PNG and TIFF samples, plan reuse with growing sizes, ROI windows;
  * a corrupt WebP sets its own status word only."""
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
import png_oracle as pngo
import png_streams as ps
import tiff_oracle as to
import tiff_streams as ts
import webp_streams as ws

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
counts = lambda: [stub.emul_launch_count(k) for k in (3, 4, 5, 6, 7, 8, 9, 10, 11)]
corpus = [s for _, s in ws.corpus()]
NO = cv2.IMREAD_IGNORE_ORIENTATION
want = [ws.decode(s, cv2.IMREAD_COLOR | NO)[..., ::-1] for s in corpus]
gray = [ws.decode(s, cv2.IMREAD_GRAYSCALE | NO)[..., None] for s in corpus]

def check(outs, idx, ot):
    for o, k in zip(outs, idx):
        w = want[k][..., ::-1] if ot == capi.BGR else gray[k] if ot == capi.GRAY else want[k]
        assert np.array_equal(o, w), (k, ot)

# WebP only: no other stage has work, and no JPEG kernel may be launched with an empty grid
for ot in (capi.RGB, capi.BGR, capi.GRAY):
    c0 = counts()
    outs, status = g.jpeg_decode_ex(corpus, output_type=ot, adjust_orientation=False)
    assert status == [0] * len(corpus)
    check(outs, range(len(corpus)), ot)
    assert [b - a for a, b in zip(c0, counts())] == [0, 0, 0, 0, 0, 1, 1, 1, 1], (c0, counts())
# mixed with baseline and progressive JPEG, PNG and TIFF samples (JPEG kernels are no-ops here: only WebP, PNG and TIFF are compared)
jpg = cv2.imencode(".jpg", g.synth_image(96, 128, 1))[1].tobytes()
prog = cv2.imencode(".jpg", g.synth_image(64, 80, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
png = ps.encode(ps.samples(30, 41, 2, 8, 5), 2, 8, filters="mixed")
tif = ts.encode(ts.samples(20, 30, 3, 8, 6), 2, 8, 5, 2, rows_per_strip=3)
idx = [3, 40, 7, 60]
streams = [jpg, corpus[3], png, prog, corpus[40], tif, corpus[7], jpg, corpus[60]]
outs, status = g.jpeg_decode_ex(streams, adjust_orientation=False)
assert status == [0] * len(streams)
check([outs[1], outs[4], outs[6], outs[8]], idx, capi.RGB)
assert np.array_equal(outs[2], pngo.decode(png)[0])
assert np.array_equal(outs[5], to.decode(tif)[0])
# plan reuse with growing WebP sizes, and corrupt WebPs beside good ones
plan = capi.Plan("Jpeg", 3)
for k, (h, w) in enumerate([(8, 8), (60, 90), (17, 200), (120, 160)]):
    ss = [ws.cv2_webp(ws.image(h + j, w, 10 + k), 60 + 10 * j) for j in range(3)]
    outs, status = g.jpeg_decode(ss, plan=plan)
    assert status == [0, 0, 0]
    for s, o in zip(ss, outs):
        assert np.array_equal(o, ws.decode(s)[..., ::-1]), (h, w)
bad = dict(ws.data_corrupt())
outs, status = g.jpeg_decode([corpus[5], bad["token_partition_cut"], corpus[6], bad["partition0_cut"], jpg],
                             plan=capi.Plan("Jpeg", 5))
assert status == [0, 1, 0, 1, 0], status
check([outs[0], outs[2]], [5, 6], capi.RGB)
# ROI windows at any edge (written directly: orientation 1, u8, RGB)
rng = np.random.default_rng(3)
sel = [k for k in range(len(corpus)) if min(want[k].shape[:2]) > 4][:12]
rois = []
for k in sel:
    H, W = want[k].shape[:2]
    x0, y0 = int(rng.integers(0, W - 1)), int(rng.integers(0, H - 1))
    rois.append((x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1))))
outs, status = g.jpeg_decode_ex([corpus[k] for k in sel], rois=rois, adjust_orientation=False)
assert status == [0] * len(sel)
for o, k, r in zip(outs, sel, rois):
    assert np.array_equal(o, want[k][r[1]:r[3], r[0]:r[2]]), (k, r)
print("webp-emul-ok")
"""


def test_webp_launch_path_decodes_webp_only_and_mixed_batches(emul_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=1500, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "webp-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
