"""The launch path of the TIFF stage, executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc is preloaded in place of the CUDA runtime,
and the launches of tiff_segment_kernel / tiff_color_kernel run on the host through the same host/device functions the device code
consists of (dali_b200/csrc/tiff_core.h); every other kernel is a no-op.  Everything around the launches is the library's real code --
plan set-up of TIFF samples beside JPEG and PNG ones, staging of the segment spans, the descriptor arena, the forked stream, the
decoded-segment scratch, the working slots and the launch geometry (one lane per warp for few segments, up to 32 for many), the
window pointers and pixel prefix -- so the TIFF outputs are compared with the oracle for real:
  * a TIFF-only batch has no JPEG units: no JPEG kernel may be launched with an empty grid (the stub reports that as the runtime's
    sticky error, which the launch returns);
  * TIFF samples mixed with baseline and progressive JPEG and PNG samples, plan reuse with growing sizes, ROI windows;
  * a corrupt TIFF sets its own status word only."""
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

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
counts = lambda: [stub.emul_launch_count(k) for k in (3, 4, 5, 6, 7)]
corpus = [s for _, s in ts.corpus()]
want = [to.decode(s) for s in corpus]

def check(outs, idx, ot, ws=None):
    for o, k in zip(outs, idx):
        rgb, gray, _ = (ws or want)[k]
        w = rgb[..., ::-1] if ot == capi.BGR else gray[..., None] if ot == capi.GRAY else rgb
        assert np.array_equal(o, w), (k, ot)

# TIFF only: neither the JPEG kernels nor the PNG stage have work, and no JPEG kernel may be launched with an empty grid
for ot in (capi.RGB, capi.BGR, capi.GRAY):
    c0 = counts()
    outs, status = g.jpeg_decode(corpus, output_type=ot)
    assert status == [0] * len(corpus)
    check(outs, range(len(corpus)), ot)
    assert [b - a for a, b in zip(c0, counts())] == [0, 0, 0, 1, 1], (c0, counts())
# more segments than resident warps: several working lanes per warp, grid-stride over the segments
many = [ts.encode(ts.samples(4400 + 7 * j, 3, 3, 8, 30 + j), 2, 8, [5, 32773][j], 2, rows_per_strip=1) for j in range(2)]
outs, status = g.jpeg_decode(many)
assert status == [0, 0]
check(outs, range(2), capi.RGB, [to.decode(s) for s in many])
# mixed with baseline and progressive JPEG and PNG samples (JPEG kernels are no-ops here: only the TIFF and PNG outputs are compared)
jpg = cv2.imencode(".jpg", g.synth_image(96, 128, 1))[1].tobytes()
prog = cv2.imencode(".jpg", g.synth_image(64, 80, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
png = ps.encode(ps.samples(30, 41, 2, 8, 5), 2, 8, filters="mixed")
idx = [3, 40, 7, 70]
streams = [jpg, corpus[3], png, prog, corpus[40], corpus[7], jpg, corpus[70]]
outs, status = g.jpeg_decode(streams)
assert status == [0] * len(streams)
check([outs[1], outs[4], outs[5], outs[7]], idx, capi.RGB)
assert np.array_equal(outs[2], pngo.decode(png)[0])
# plan reuse with growing TIFF sizes, and corrupt TIFFs beside good ones
plan = capi.Plan("Jpeg", 4)
for k, (h, w) in enumerate([(8, 8), (60, 90), (17, 200), (120, 160)]):
    ss = [ts.encode(ts.samples(h + j, w, 3, 8, 10 + k), 2, 8, [5, 8, 32773][j], 2, rows_per_strip=1 + 2 * j,
                    tile=(32, 16) if j == 1 else None) for j in range(3)]
    outs, status = g.jpeg_decode(ss, plan=plan)
    assert status == [0, 0, 0]
    for s, o in zip(ss, outs):
        assert np.array_equal(o, to.decode(s)[0]), (h, w)
bad = dict(ts.data_corrupt())
outs, status = g.jpeg_decode([corpus[5], bad["lzw_bad_code"], corpus[6], bad["deflate_adler"], jpg, bad["packbits_truncated"]],
                             plan=capi.Plan("Jpeg", 6))
assert status == [0, 1, 0, 1, 0, 1], status
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
print("tiff-emul-ok")
"""


def test_tiff_launch_path_decodes_tiff_only_and_mixed_batches(emul_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=1500, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "tiff-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
