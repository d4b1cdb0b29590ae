"""The launch path of fn.experimental.filter, executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc is preloaded in place of the CUDA
runtime and filter_kernel runs on the host through the host/device bodies of dali_b200/csrc/filter_core.h.  Everything around the launch
is the library's real code -- the operator, the planner, the descriptor arena with the uploaded filters and fill values, the executor --
and the outputs are compared with tests/filter_ref.py:
  * JPEG and PNG images decoded by decoders.image, filtered, then cast;
  * CPU and GPU filter inputs, CPU and GPU fill values, and an argument-input anchor;
  * one plan reused through the C-ABI across batches whose shapes, filters, borders and modes change;
  * exactly one `filter` launch per batch, named in the profile."""
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
import filter_ref as fr
import nvidia.dali as dali
from nvidia.dali import fn, types
from dali_b200 import capi

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
lib = capi.lib()
rng = np.random.default_rng(11)

imgs = [gh.synth_image(61, 97, 1), rng.integers(0, 256, (40, 33, 3), dtype=np.uint8), gh.synth_image(17, 300, 2)]
streams = [np.frombuffer(cv2.imencode(".png", imgs[0])[1].tobytes(), np.uint8),
           np.frombuffer(cv2.imencode(".png", imgs[1])[1].tobytes(), np.uint8),
           np.frombuffer(cv2.imencode(".jpg", imgs[2], [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes(), np.uint8)]
sharpen = np.array([[0, -1, 0], [-1, 5, -1], [0, -1, 0]], np.float32)
filters = [sharpen, np.full((5, 3), 1 / 16, np.float32), np.array([[1, 2, 1]], np.float32) / 4]     # exact sums on bytes
anchors = [np.array([0, 0], np.int32), np.array([-1, -1], np.int32), np.array([0, 2], np.int32)]
fills = [np.array(v, np.uint8) for v in (0, 128, 255)]

@dali.pipeline_def(batch_size=3, num_threads=1, device_id=0, prefetch_queue_depth=1)
def decode():
    img = fn.decoders.image(fn.external_source(source=lambda: streams), device="mixed")
    cpu_f = fn.external_source(source=lambda: filters)
    gpu_f = fn.external_source(source=lambda: filters, device="gpu")
    a = fn.external_source(source=lambda: anchors)
    fill = fn.external_source(source=lambda: fills, device="gpu")
    f1 = fn.experimental.filter(img, cpu_f, anchor=a)
    f2 = fn.experimental.filter(img, gpu_f, fill, border="constant", dtype=types.FLOAT)
    f3 = fn.experimental.filter(img, cpu_f, fn.external_source(source=lambda: fills), border="wrap", mode="valid")
    return img, f1, fn.cast(f2, dtype=types.INT16), f3
p = decode()
p.build()
k0 = stub.emul_launch_count(32)
img, f1, f2, f3 = p.run()
assert stub.emul_launch_count(32) - k0 == 3, stub.emul_launch_count(32) - k0      # one launch for each filter operator's batch
for k in range(3):
    dec = img.as_cpu()[k]
    assert np.array_equal(f1.as_cpu()[k], fr.filter_ref(dec, filters[k], "HWC", tuple(anchors[k]))), k
    f32 = fr.filter_ref(dec, filters[k], "HWC", border="constant", fill=fills[k], dtype=np.float32)   # exact: dyadic taps, bytes
    assert np.array_equal(f2.as_cpu()[k], fr.ar.convert_sat(f32, fr.ar.F32, fr.ar.I16)), k
    assert np.array_equal(f3.as_cpu()[k], fr.filter_ref(dec, filters[k], "HWC", border="wrap", mode="valid")), k
    assert f1.layout() == "HWC" and f3.as_cpu()[k].shape == (dec.shape[0] - filters[k].shape[0] + 1, dec.shape[1] - filters[k].shape[1] + 1, 3)

# one plan through the C-ABI: batches of changing shapes, filters, borders and modes; "device" memory is host memory here
plan = C.c_void_p()
capi.check(lib.dalib200FilterPlanCreate(C.byref(plan), 4))
P64 = C.c_int64
for it, (shapes, fshapes, border, mode) in enumerate([([(30, 40, 3), (7, 9, 3)], [(3, 3), (7, 1)], 0, 0),
                                                     ([(2, 50, 20, 1), (1, 6, 6, 1), (3, 9, 70, 1)], [(5, 5), (2, 6), (1, 9)], 2, 1),
                                                     ([(300, 17, 4)], [(15, 15)], 4, 0)]):
    nd = len(shapes[0])
    lay = {2: "HW", 3: "HWC", 4: "FHWC"}[nd]
    xs = [rng.integers(0, 256, s, dtype=np.uint8) for s in shapes]
    fs = [(rng.integers(-4, 5, s) / 8).astype(np.float32) for s in fshapes]
    n = len(xs)
    oshp = (P64 * (n * nd))()
    capi.check(lib.dalib200FilterSetup(plan, 0, 9, n, nd, (P64 * (n * nd))(*[e for s in shapes for e in s]), lay.encode(), 9, 2,
                                       (P64 * (2 * n))(*[e for s in fshapes for e in s]), None, border, mode, -1, None, oshp))
    outs = [np.zeros(tuple(oshp[i * nd:(i + 1) * nd]), np.float32) for i in range(n)]
    k0, n0 = stub.emul_launch_count(32), capi.launch_count()
    capi.profiling(True)
    capi.check(lib.dalib200FilterLaunch(plan, (C.c_void_p * n)(*[x.ctypes.data for x in xs]), (C.c_void_p * n)(*[f.ctypes.data for f in fs]), 0,
                                        None, 0, (C.c_void_p * n)(*[o.ctypes.data for o in outs]), None))
    assert stub.emul_launch_count(32) - k0 == 1 and capi.launch_count() - n0 == 1, it
    assert [name for name, _ in capi.profiling_collect()] == ["filter"], it
    capi.profiling(False)
    for x, f, o in zip(xs, fs, outs):
        bname = fr.BORDERS[border]
        assert np.array_equal(o, fr.filter_ref(x, f, lay, border=bname, mode=("same", "valid")[mode], dtype=np.float32)), it
lib.dalib200FilterPlanDestroy(plan)
print("filter-emul-ok")
"""


def test_filter_launch_path_after_decode_with_cpu_and_gpu_inputs_and_plan_reuse(emul_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=900, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "filter-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
