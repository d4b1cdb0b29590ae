"""The launch path of fn.multi_paste and fn.paste, executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc is preloaded in place of the
CUDA runtime and paste_kernel runs on the host through the host/device bodies of dali_b200/csrc/paste_core.h.  Everything around the
launch is the library's real code -- the operators, the argument reading, the planner, the descriptor arena with the input pointers,
fill table, bands and segments, the executor -- and the outputs are compared with tests/paste_ref.py:
  * decode -> resize(640) -> multi_paste (a 4-tile mosaic, in_ids and the region arguments from external_source) ->
    crop_mirror_normalize (the stub runs neither resize's nor crop_mirror_normalize's kernel: the mosaic is checked against the tiles
    as they are, the normalised output for shape only);
  * decode -> paste -> resize;
  * one plan reused through the C-ABI across batches whose region counts and sizes change;
  * exactly one `paste` launch per batch: the launch counter, the stub's trace and the profile records agree."""
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
import paste_ref as pr
import nvidia.dali as dali
from nvidia.dali import fn, types
from dali_b200 import capi

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
lib = capi.lib()
rng = np.random.default_rng(13)

def trace_launches():
    if not os.path.exists(os.environ["DALIB200_EMUL_TRACE"]):
        return 0
    with open(os.environ["DALIB200_EMUL_TRACE"]) as f:
        return sum(line.startswith("launch dalib200::paste_kernel") for line in f)

# decode -> resize(640) -> 4-tile mosaic -> crop_mirror_normalize
imgs = [gh.synth_image(61, 97, 1), rng.integers(0, 256, (40, 33, 3), dtype=np.uint8), gh.synth_image(170, 300, 2), gh.synth_image(90, 90, 3)]
streams = [np.frombuffer(cv2.imencode(".png", im)[1].tobytes(), np.uint8) for im in imgs]
n = len(imgs)
ids, ia, sh, oa = [], [], [], []
for i in range(n):
    yc, xc = int(rng.integers(320, 960)), int(rng.integers(320, 960))
    q = [[min(yc, 640), min(xc, 640)], [min(yc, 640), min(1280 - xc, 640)], [min(1280 - yc, 640), min(xc, 640)], [min(1280 - yc, 640), min(1280 - xc, 640)]]
    ids.append(np.array(rng.integers(0, n, 4), np.int32))
    sh.append(np.array(q, np.int32))
    oa.append(np.array([[yc - q[0][0], xc - q[0][1]], [yc - q[1][0], xc], [yc, xc - q[2][1]], [yc, xc]], np.int32))
    ia.append(np.array([[640 - q[0][0], 640 - q[0][1]], [640 - q[1][0], 0], [0, 640 - q[2][1]], [0, 0]], np.int32))

@dali.pipeline_def(batch_size=n, num_threads=1, device_id=0, prefetch_queue_depth=1)
def mosaic():
    img = fn.decoders.image(fn.external_source(source=lambda: streams), device="mixed")
    tiles = fn.resize(img, resize_x=640, resize_y=640)
    src = lambda v: fn.external_source(source=lambda: v)
    m = fn.multi_paste(tiles, in_ids=src(ids), in_anchors=src(ia), shapes=src(sh), out_anchors=src(oa), output_size=[1280, 1280])
    return tiles, m, fn.crop_mirror_normalize(m, dtype=types.FLOAT, output_layout="CHW", mean=[0.0] * 3, std=[1.0] * 3)
p = mosaic()
p.build()
k0, t0 = stub.emul_launch_count(34), trace_launches()
tiles, m, cmn = p.run()
assert stub.emul_launch_count(34) - k0 == 1 and trace_launches() - t0 == 1
assert m.layout() == "HWC"
tl = [tiles.as_cpu()[k] for k in range(n)]
for i in range(n):
    want = pr.multi_paste_ref([tl[j] for j in ids[i]], (1280, 1280), dict(in_anchors=ia[i], shapes=sh[i], out_anchors=oa[i]), np.uint8, 3)
    assert m.as_cpu()[i].tobytes() == want.tobytes(), i
    assert cmn.as_cpu()[i].shape == (3, 1280, 1280), i

# decode -> paste -> resize
ratio = [1.0, 2.5, 3.75, 1.5]
@dali.pipeline_def(batch_size=n, num_threads=1, device_id=0, prefetch_queue_depth=1)
def zoom():
    img = fn.decoders.image(fn.external_source(source=lambda: streams), device="mixed")
    z = fn.paste(img, ratio=fn.external_source(source=lambda: [np.array(r, np.float32) for r in ratio]), paste_x=0.25, paste_y=1.0,
                 fill_value=[123, 117, 104], min_canvas_size=100.0)
    return img, z, fn.resize(z, resize_x=300, resize_y=300)
p = zoom()
p.build()
k0 = stub.emul_launch_count(34)
img, z, r = p.run()
assert stub.emul_launch_count(34) - k0 == 1
for i in range(n):
    want = pr.paste_ref(img.as_cpu()[i], ratio[i], 0.25, 1.0, 100.0, (123, 117, 104))
    assert z.as_cpu()[i].tobytes() == want.tobytes(), i
    assert r.as_cpu()[i].shape == (300, 300, 3), i

# one plan through the C-ABI: batches whose region counts and sizes change; "device" memory is host memory here
plan = C.c_void_p()
capi.check(lib.dalib200PastePlanCreate(C.byref(plan), 4))
P64 = C.POINTER(C.c_int64)
for it, (shapes, k, out_hw) in enumerate([([(30, 40, 3), (7, 9, 3)], 1, (33, 41)), ([(50, 20, 3), (6, 6, 3), (9, 70, 3)], 64, (60, 80)),
                                          ([(300, 17, 3)], 0, (5, 5)), ([(12, 12, 3)] * 4, 4, (24, 24))]):
    xs = [rng.integers(0, 2 ** 16, s, dtype=np.uint16) for s in shapes]
    nb = len(xs)
    rid = [[int(v) for v in rng.integers(0, nb, k)] for _ in xs]
    args = {"in_anchors": [], "shapes": [], "out_anchors": []}
    for row in rid:
        a, s, o = [], [], []
        for j in row:
            hs, ws, _ = shapes[j]
            h, w = int(rng.integers(0, min(hs, out_hw[0]) + 1)), int(rng.integers(0, min(ws, out_hw[1]) + 1))
            a.append([int(rng.integers(0, hs - h + 1)), int(rng.integers(0, ws - w + 1))])
            s.append([h, w])
            o.append([int(rng.integers(0, out_hw[0] - h + 1)), int(rng.integers(0, out_hw[1] - w + 1))])
        args["in_anchors"].append(a), args["shapes"].append(s), args["out_anchors"].append(o)
    av, ac, keep = (C.POINTER(C.c_double) * 6)(), (P64 * 6)(), []
    for a, name in enumerate(pr.ARGS):
        if name in args:
            vals = np.array([v for row in args[name] for pair in row for v in pair] + [0.0], np.float64)
            cnt = np.array([2 * len(row) for row in args[name]], np.int64)
            keep += [vals, cnt]
            av[a], ac[a] = vals.ctypes.data_as(C.POINTER(C.c_double)), cnt.ctypes.data_as(P64)
    flat = [j for row in rid for j in row] or [0]
    oshapes = (C.c_int64 * (3 * nb))()
    capi.check(lib.dalib200PasteSetup(plan, 1, -1, 1, nb, (C.c_int * 1)(3), None, (C.c_int64 * (3 * nb))(*[e for s in shapes for e in s]),
                                      (C.c_int32 * len(flat))(*flat), (C.c_int64 * nb)(*[len(r) for r in rid]), av, ac,
                                      (C.c_int64 * (2 * nb))(*(list(out_hw) * nb)), (C.c_float * 1)(0.0), 1, oshapes))
    outs = [np.zeros(out_hw + (3,), np.uint16) for _ in xs]
    k0, n0, t0 = stub.emul_launch_count(34), capi.launch_count(), trace_launches()
    capi.profiling(True)
    capi.check(lib.dalib200PasteLaunch(plan, (C.c_void_p * nb)(*[x.ctypes.data for x in xs]), (C.c_void_p * nb)(*[o.ctypes.data for o in outs]), None))
    assert stub.emul_launch_count(34) - k0 == 1 and capi.launch_count() - n0 == 1 and trace_launches() - t0 == 1, it
    assert [name for name, _ in capi.profiling_collect()] == ["paste"], it
    capi.profiling(False)
    for i, o in enumerate(outs):
        want = pr.multi_paste_ref([xs[j] for j in rid[i]], out_hw, {kk: v[i] for kk, v in args.items()}, np.uint16, 3)
        assert o.tobytes() == want.tobytes(), (it, i)
# a batch without elements: no launch
oshapes = (C.c_int64 * 6)()
capi.check(lib.dalib200PasteSetup(plan, 0, -1, 1, 2, (C.c_int * 1)(3), None, (C.c_int64 * 6)(4, 5, 3, 4, 5, 3), (C.c_int32 * 1)(0), (C.c_int64 * 2)(0, 0),
                                  (C.POINTER(C.c_double) * 6)(), (P64 * 6)(), (C.c_int64 * 4)(0, 5, 3, 0), (C.c_float * 1)(0.0), 1, oshapes))
n0 = capi.launch_count()
capi.check(lib.dalib200PasteLaunch(plan, (C.c_void_p * 2)(None, None), (C.c_void_p * 2)(None, None), None))
assert capi.launch_count() == n0
lib.dalib200PastePlanDestroy(plan)
print("paste-emul-ok")
"""


def test_paste_launch_path_after_decode_and_resize_and_plan_reuse(emul_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=900, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "paste-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
