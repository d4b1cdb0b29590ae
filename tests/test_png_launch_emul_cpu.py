"""The launch path of the PNG stage, executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc is preloaded in place of the CUDA runtime, and
the launches of png_crc_kernel / png_inflate_kernel / png_color_kernel run on the host through the same host/device functions the
device code consists of (dali_b200/csrc/png_core.h); every other kernel is a no-op.  Everything around the launches is the library's
real code -- plan set-up of PNG samples beside JPEG ones, staging of the IDAT runs, the descriptor arena, the forked stream, the
scanline scratch, the window pointers -- so the PNG outputs are compared with the oracle for real:
  * a PNG-only batch has no JPEG units: no JPEG kernel may be launched with an empty grid (the stub reports that as the runtime's
    sticky error, which the launch returns);
  * PNG samples mixed with baseline and progressive JPEG samples, plan reuse with growing sizes, ROI windows;
  * a corrupt PNG sets its own status word only."""
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

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
counts = lambda: [stub.emul_launch_count(k) for k in (3, 4, 5)]
corpus = [s for _, s in ps.corpus()]
want = [pngo.decode(s) for s in corpus]

def check(outs, idx, ot):
    for o, k in zip(outs, idx):
        rgb, gray, _ = want[k]
        w = rgb[..., ::-1] if ot == capi.BGR else gray[..., None] if ot == capi.GRAY else rgb
        assert np.array_equal(o, w), (k, ot)

# PNG only: the JPEG entropy kernels have no work and must not be launched
for ot in (capi.RGB, capi.BGR, capi.GRAY):
    c0 = counts()
    outs, status = g.jpeg_decode(corpus, output_type=ot)
    assert status == [0] * len(corpus)
    check(outs, range(len(corpus)), ot)
    assert [b - a for a, b in zip(c0, counts())] == [1, 1, 1], (c0, counts())
# mixed with baseline and progressive JPEG samples (their kernels are no-ops here: only the PNG outputs are compared)
jpg = cv2.imencode(".jpg", g.synth_image(96, 128, 1))[1].tobytes()
prog = cv2.imencode(".jpg", g.synth_image(64, 80, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
idx = [3, 40, 7, 70]
streams = [jpg, corpus[3], prog, corpus[40], corpus[7], jpg, corpus[70]]
outs, status = g.jpeg_decode(streams)
assert status == [0] * len(streams)
check([outs[1], outs[3], outs[4], outs[6]], idx, capi.RGB)
# plan reuse with growing PNG sizes, and a corrupt PNG beside good ones
plan = capi.Plan("Jpeg", 4)
for k, (h, w) in enumerate([(8, 8), (60, 90), (17, 200), (120, 160)]):
    ss = [ps.encode(ps.samples(h + j, w, 2, 8, 10 + k), 2, 8, filters="mixed", interlace=j == 1) for j in range(3)]
    outs, status = g.jpeg_decode(ss, plan=plan)
    assert status == [0, 0, 0]
    for s, o in zip(ss, outs):
        assert np.array_equal(o, pngo.decode(s)[0]), (h, w)
bad = dict(ps.corrupt())
outs, status = g.jpeg_decode([corpus[5], bad["adler"], corpus[6], bad["idat_crc"], jpg], plan=capi.Plan("Jpeg", 5))
assert status == [0, 1, 0, 1, 0], status
check([outs[0], outs[2]], [5, 6], capi.RGB)
# ROI windows at any left edge (written directly: orientation 1, u8, RGB)
rng = np.random.default_rng(3)
sel = [k for k in range(len(corpus)) if min(want[k][0].shape[:2]) > 4][:12]
rois = []
for k in sel:
    H, W = want[k][0].shape[:2]
    x0, y0 = int(rng.integers(0, W - 1)), int(rng.integers(0, H - 1))
    rois.append((x0, y0, int(rng.integers(x0 + 1, W + 1)), int(rng.integers(y0 + 1, H + 1))))
outs, status = g.jpeg_decode_ex([corpus[k] for k in sel], rois=rois, adjust_orientation=False)
assert status == [0] * len(sel)
for o, k, r in zip(outs, sel, rois):
    assert np.array_equal(o, want[k][0][r[1]:r[3], r[0]:r[2]]), (k, r)
print("png-emul-ok")
"""


def test_png_launch_path_decodes_png_only_and_mixed_batches(emul_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=1500, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "png-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
