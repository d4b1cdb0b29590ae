"""The launch path of fn.experimental.equalize, executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc is preloaded in place of the CUDA
runtime and equalize_hist_kernel / equalize_apply_kernel run on the host through the host/device bodies of
dali_b200/csrc/equalize_core.h.  Everything around the launches is the library's real code -- the operator, the planner, the
descriptor arena, the histogram scratch and its zeroing, the executor -- and the outputs are compared with cv2.equalizeHist per plane:
  * PNG images decoded by decoders.image, then equalized; the equalized image feeding an arithmetic expression;
  * one plan reused across batches whose shapes, layouts and histogram sizes change;
  * two launches per batch, whatever its size."""
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
    pytest.importorskip("cv2")
    stub = str(tmp_path_factory.mktemp("emul") / "cuda_emul_stub.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include",
                        os.path.join(ROOT, "tools", "emul", "cuda_emul_stub.cc"), "-o", stub, "-ldl"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return dict(os.environ, DALIB200_DRYRUN="emul", LD_PRELOAD=stub, EMUL_STUB=stub)


SCRIPT = r"""
import ctypes as C, os, sys
import numpy as np
import cv2
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests"))
import conftest                      # DALIB200_DRYRUN=emul: "device" tensors are host memory
import gpu_helpers as gh
from test_gpu_equalize import cv2_equalize
import nvidia.dali as dali
from nvidia.dali import fn

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
launches = lambda: (stub.emul_launch_count(30), stub.emul_launch_count(31))
rng = np.random.default_rng(9)

imgs = [gh.synth_image(61, 97, 1), rng.integers(0, 256, (40, 33, 3), dtype=np.uint8), np.full((17, 300, 3), 90, np.uint8),
        rng.choice(np.array([4, 250], np.uint8), (130, 70, 3))]
streams = [np.frombuffer(cv2.imencode(".png", im)[1].tobytes(), np.uint8) for im in imgs]

@dali.pipeline_def(batch_size=4, num_threads=1, device_id=0, prefetch_queue_depth=1)
def decode():
    img = fn.decoders.image(fn.external_source(source=lambda: streams), device="mixed")
    e = fn.experimental.equalize(img)
    return img, e, e // 2 + 1
p = decode()
p.build()
h0, a0 = launches()
img, e, half = p.run()
assert launches() == (h0 + 1, a0 + 1), launches()
for k, im in enumerate(imgs):
    dec = img.as_cpu()[k]
    assert np.array_equal(dec, im[:, :, ::-1]), k                 # PNG decodes to RGB
    want = cv2_equalize(dec, "HWC")
    assert np.array_equal(e.as_cpu()[k], want), k
    assert np.array_equal(half.as_cpu()[k], want // 2 + 1), k

state = {}
@dali.pipeline_def(batch_size=3, num_threads=1, device_id=0, prefetch_queue_depth=1)
def seq():
    return fn.experimental.equalize(fn.external_source(source=lambda: state["b"], device="gpu", layout="FCHW"))
q = seq()
q.build()
for it, shapes in enumerate([[(2, 3, 40, 50), (1, 1, 7, 7), (3, 16, 9, 13)], [(4, 3, 200, 190), (0, 3, 5, 5), (1, 2, 1, 1)],
                             [(1, 1, 1, 1), (2, 4, 30, 31), (5, 3, 64, 64)]]):
    state["b"] = [rng.integers(0, 256, s, dtype=np.uint8) if k != 1 else np.full(s, 3, np.uint8) for k, s in enumerate(shapes)]
    h0, a0 = launches()
    (o,) = q.run()
    assert launches() == (h0 + 1, a0 + 1), (it, launches())
    assert o.layout() == "FCHW"
    for k, x in enumerate(state["b"]):
        assert np.array_equal(o.as_cpu()[k], cv2_equalize(x, "FCHW")), (it, k)
print("equalize-emul-ok")
"""


def test_equalize_launch_path_after_decode_into_arithmetic_with_plan_reuse(emul_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=900, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "equalize-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
