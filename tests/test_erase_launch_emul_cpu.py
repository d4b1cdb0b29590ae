"""The launch path of fn.erase, executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc is preloaded in place of the CUDA runtime and
erase_kernel runs on the host through the host/device bodies of dali_b200/csrc/erase_core.h.  Everything around the launch is the
library's real code -- the operator, the argument resolution, the planner, the descriptor arena with the bands, intervals and fill
table, the executor -- and the outputs are compared with tests/erase_ref.py:
  * decode -> erase (normalised anchors from fn.random.uniform(shape=(2,))) -> crop_mirror_normalize (whose kernel the stub does not
    run: its output is checked for shape only);
  * spectrogram -> mel -> erase on "f" and on "t", per-sample masks from CPU tensor inputs, one clip without a mask;
  * one plan reused through the C-ABI across batches whose shapes, axes and region counts change;
  * exactly one `erase` launch per batch: the launch counter, the stub's trace and the profile records agree."""
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
    d = tmp_path_factory.mktemp("emul")
    stub = str(d / "cuda_emul_stub.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include",
                        os.path.join(ROOT, "tools", "emul", "cuda_emul_stub.cc"), "-o", stub, "-ldl"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return dict(os.environ, DALIB200_DRYRUN="emul", LD_PRELOAD=stub, EMUL_STUB=stub, DALIB200_EMUL_TRACE=str(d / "trace.txt"))


SCRIPT = r"""
import ctypes as C, os, sys
import numpy as np
import cv2
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests"))
import conftest                      # DALIB200_DRYRUN=emul: "device" tensors are host memory
import gpu_helpers as gh
import erase_ref as er
import nvidia.dali as dali
from nvidia.dali import fn, types
from dali_b200 import capi

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
lib = capi.lib()
rng = np.random.default_rng(12)

def trace_launches():
    if not os.path.exists(os.environ["DALIB200_EMUL_TRACE"]):
        return 0
    with open(os.environ["DALIB200_EMUL_TRACE"]) as f:
        return sum(line.startswith("launch dalib200::erase_kernel") for line in f)

# decode -> erase (random normalised anchor, fixed normalised shape) -> crop_mirror_normalize
imgs = [gh.synth_image(61, 97, 1), rng.integers(0, 256, (40, 33, 3), dtype=np.uint8), gh.synth_image(17, 300, 2)]
streams = [np.frombuffer(cv2.imencode(".png", im)[1].tobytes(), np.uint8) for im in imgs]

@dali.pipeline_def(batch_size=3, num_threads=1, device_id=0, prefetch_queue_depth=1, seed=7)
def image():
    img = fn.decoders.image(fn.external_source(source=lambda: streams), device="mixed")
    anchor = fn.random.uniform(range=(0.0, 0.7), shape=(2,))
    x = fn.erase(img, anchor=anchor, shape=[0.3, 0.25], normalized=True, fill_value=[0, 128, 255])
    return img, anchor, x, fn.crop_mirror_normalize(x, dtype=types.FLOAT, output_layout="CHW", mean=[0.0] * 3, std=[1.0] * 3)
p = image()
p.build()
k0, t0 = stub.emul_launch_count(33), trace_launches()
img, anchor, x, cmn = p.run()
assert stub.emul_launch_count(33) - k0 == 1 and trace_launches() - t0 == 1
assert x.layout() == "HWC"
for k in range(3):
    dec, a = img.as_cpu()[k], np.asarray(anchor[k])
    want = er.erase_ref(dec, [0, 1], a, [0.3, 0.25], (0, 128, 255), "HWC", True, True)
    assert x.as_cpu()[k].tobytes() == want.tobytes(), k
    assert cmn.as_cpu()[k].shape == (3,) + dec.shape[:2], k          # the stub does not run crop_mirror_normalize's kernel

# spectrogram -> mel -> erase on f and on t, masks from CPU tensor inputs; the second clip has no time mask
sigs = [rng.standard_normal(4000).astype(np.float32), rng.standard_normal(2500).astype(np.float32)]
fa = [np.array([3.0, 40.0], np.float32), np.array([0.0], np.float32)]
fs = [np.array([5.0, 4.0], np.float32), np.array([2.5], np.float32)]
ta = [np.array([2.0, 9.5, 30.0], np.float32), np.zeros(0, np.float32)]
ts = [np.array([4.0, 2.0, 99.0], np.float32), np.zeros(0, np.float32)]

@dali.pipeline_def(batch_size=2, num_threads=1, device_id=0, prefetch_queue_depth=1)
def audio():
    a = fn.external_source(source=lambda: sigs, device="gpu")
    mel = fn.mel_filter_bank(fn.spectrogram(a, nfft=256, window_length=256, window_step=128), sample_rate=16000.0, nfilter=64)
    src = lambda v: fn.external_source(source=lambda: v)
    f = fn.erase(mel, anchor=src(fa), shape=src(fs), axis_names="f", fill_value=-1.0)
    t = fn.erase(f, anchor=src(ta), shape=src(ts), axis_names="t", fill_value=-2.0)
    return mel, f, t
p = audio()
p.build()
mel, f, t = p.run()
assert t.layout() == "ft"
for k in range(2):
    m = mel.as_cpu()[k]
    wf = er.erase_ref(m, [0], fa[k], fs[k], (-1.0,))
    assert f.as_cpu()[k].tobytes() == wf.tobytes(), k
    assert t.as_cpu()[k].tobytes() == er.erase_ref(wf, [1], ta[k], ts[k], (-2.0,)).tobytes(), k

# one plan through the C-ABI: batches of changing shapes, axes and region counts; "device" memory is host memory here
plan = C.c_void_p()
capi.check(lib.dalib200ErasePlanCreate(C.byref(plan), 4))
P64 = C.c_int64
batches = [([(30, 40, 3), (7, 9, 3)], "HWC", [0, 1], [1, 64]),
           ([(2, 50, 20, 1), (1, 6, 6, 1), (3, 9, 70, 1)], "FHWC", [0, 2], [0, 3, 2]),
           ([(300, 17)], "ft", [1], [5])]
for it, (shapes, lay, axes, counts) in enumerate(batches):
    xs = [rng.integers(0, 2 ** 16, s, dtype=np.uint16) for s in shapes]
    n, nd = len(xs), len(shapes[0])
    anchors = [[float(rng.integers(-2, s[a] + 2)) for _ in range(k) for a in axes] for s, k in zip(shapes, counts)]
    rshapes = [[float(rng.integers(0, s[a] + 1)) for _ in range(k) for a in axes] for s, k in zip(shapes, counts)]
    av = [v for a in anchors for v in a] or [0.0]
    sv = [v for a in rshapes for v in a] or [0.0]
    cnt = (P64 * n)(*[len(a) for a in anchors])
    capi.check(lib.dalib200EraseSetup(plan, 1, n, nd, (P64 * (n * nd))(*[e for s in shapes for e in s]), lay.encode(), None,
                                      (C.c_int32 * len(axes))(*axes), len(axes), (C.c_float * len(av))(*av), cnt,
                                      (C.c_float * len(sv))(*sv), cnt, 0, 0, 0, (C.c_float * 1)(77.0), 1))
    outs = [np.zeros_like(x) for x in xs]
    k0, n0, t0 = stub.emul_launch_count(33), capi.launch_count(), trace_launches()
    capi.profiling(True)
    capi.check(lib.dalib200EraseLaunch(plan, (C.c_void_p * n)(*[x.ctypes.data for x in xs]), (C.c_void_p * n)(*[o.ctypes.data for o in outs]),
                                       None))
    assert stub.emul_launch_count(33) - k0 == 1 and capi.launch_count() - n0 == 1 and trace_launches() - t0 == 1, it
    assert [name for name, _ in capi.profiling_collect()] == ["erase"], it
    capi.profiling(False)
    for x, o, a, s in zip(xs, outs, anchors, rshapes):
        assert o.tobytes() == er.erase_ref(x, axes, a, s, (77.0,)).tobytes(), it
# a batch without elements: no launch
capi.check(lib.dalib200EraseSetup(plan, 0, 2, 2, (P64 * 4)(0, 5, 3, 0), b"HW", b"HW", None, 0, (C.c_float * 1)(0.0), (P64 * 2)(0, 0),
                                  (C.c_float * 1)(0.0), (P64 * 2)(0, 0), 0, 0, 0, (C.c_float * 1)(0.0), 1))
n0 = capi.launch_count()
capi.check(lib.dalib200EraseLaunch(plan, (C.c_void_p * 2)(None, None), (C.c_void_p * 2)(None, None), None))
assert capi.launch_count() == n0
lib.dalib200ErasePlanDestroy(plan)
print("erase-emul-ok")
"""


def test_erase_launch_path_after_decode_and_mel_and_plan_reuse(emul_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=900, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "erase-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
