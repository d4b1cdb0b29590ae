"""Stream ordering of the image decoder's side stages, checked WITHOUT a GPU.  Progressive JPEG, PNG, TIFF, WebP, BMP / PNM and lossless
JPEG samples are decoded on side streams of their own, forked from the caller's stream and joined back into it; a missing fork, join or
upload wait is a race that a GPU shows only as an intermittent wrong image, and the emulated launches (which run synchronously) never
show.  So this test reads the call trace of tools/emul/cuda_emul_stub.cc (DALIB200_EMUL_TRACE) of a batch holding every sample kind,
launched twice on one plan with float output, then a JPEG-only batch on the same plan, and a WebP-only batch with YCbCr output on a plan
of its own (float and YCbCr output make the post pass run):
  1. every side-stage kernel runs on its stage's stream, one stream per stage, none of them the caller's;
  2. before a stage's first upload, memset or launch, its stream waits on an event the caller's stream recorded behind the status clear;
     the lossless stage's event is recorded behind unstuff_scatter, whose clean streams it reads;
  3. the caller's stream waits on the progressive stage's join in front of dc_scan, on the other stages' joins in front of jpeg_post;
  4. on the second launch, each stage's upload event is synchronised before its descriptor arena is uploaded again;
  5. a batch without a side stage makes no stream or event call for it."""
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def stub(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    so = str(tmp_path_factory.mktemp("emul") / "cuda_emul_stub.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include",
                        os.path.join(ROOT, "tools", "emul", "cuda_emul_stub.cc"), "-o", so, "-ldl"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return so


# Decodes through the C-ABI with host buffers ("device" memory is host memory under the stub); writes a "# <section>" line in front of
# each set-up + upload + launch and in front of the plan's destruction.
SCRIPT = r"""
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests"))
import cv2
import gpu_helpers as g
from dali_b200 import capi
import png_streams as ps
import tiff_streams as ts
import webp_streams as ws
import bitmap_streams as bs
import ljpeg_streams as ls

lib = capi.lib()
stub = C.CDLL(os.environ["EMUL_STUB"])
mark = lambda s: stub.emul_trace_mark(s.encode())

def decode(plan, streams, output_type, dtype):
    n = len(streams)
    bufs = [np.frombuffer(bytes(s), np.uint8) for s in streams]
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    lens = (C.c_size_t * n)(*[b.size for b in bufs])
    prm = capi.JpegParams(output_type, 1, dtype, 0)
    capi.check(lib.dalib200JpegPlanSetupEx(plan.handle, n, ptrs, lens, C.byref(prm), None))
    outs = []
    for i in range(n):
        hwc = (C.c_int32 * 3)()
        capi.check(lib.dalib200JpegPlanGetOutputShape(plan.handle, i, hwc))
        outs.append(np.zeros(tuple(hwc), np.float32 if dtype == capi.FLOAT else np.uint8))
    capi.check(lib.dalib200JpegUpload(plan.handle, None))
    capi.check(lib.dalib200JpegLaunch(plan.handle, (C.c_void_p * n)(*[o.ctypes.data for o in outs]), None))
    status = (C.c_int32 * n)()
    capi.check(lib.dalib200JpegGetStatus(plan.handle, status))
    assert list(status) == [0] * n, list(status)

jpg = cv2.imencode(".jpg", g.synth_image(96, 128, 1))[1].tobytes()
prog = cv2.imencode(".jpg", g.synth_image(64, 80, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
png = ps.encode(ps.samples(30, 41, 2, 8, 5), 2, 8, filters="mixed")
tif = ts.encode(ts.samples(20, 30, 3, 8, 6), 2, 8, 5, 2, rows_per_strip=3)
webp = ws.cv2_webp(ws.image(40, 56, 7), 70)
bmp = bs.bmp(31, 17, 24, bs.rows(bs.image(17, 31, 1), 24))
ljp = ls.encode(ls.image(33, 17, 1, 6, 71), P=6, Pt=2, restart=17 * 4)
mixed = [jpg, prog, png, tif, webp, bmp, ljp]
plan = capi.Plan("Jpeg", 7)
for k in range(2):
    mark("mixed %%d" %% k)
    decode(plan, mixed, capi.RGB, capi.FLOAT)
mark("jpeg-only 3")
decode(plan, [jpg, jpg, jpg], capi.RGB, capi.FLOAT)
mark("destroy")
del plan
plan = capi.Plan("Jpeg", 2)
mark("webp-only 2")
decode(plan, [webp, webp], capi.YCbCr, capi.UINT8)
mark("destroy")
del plan
print("trace-ok")
"""

STAGES = ("prog", "png", "tiff", "webp", "bitmap", "ljpeg")


def run_trace(stub, trace):
    env = dict(os.environ, LD_PRELOAD=stub, EMUL_STUB=stub, DALIB200_EMUL_TRACE=trace)
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "trace-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
    sections = []
    with open(trace) as f:
        for line in f:
            w = line.split()
            if w[0] == "#":
                sections.append((w[1:], []))
            elif sections:
                sections[-1][1].append(w)
    return sections


def stream_of(op):
    """The stream an operation is enqueued on, or None."""
    return op[2] if op[0] in ("launch", "record") else op[1] if op[0] in ("wait", "memset", "h2d") else None


def stage_of(op):
    if op[0] != "launch":
        return None
    kernel = op[1].split("::")[-1]
    return next((s for s in STAGES if kernel.startswith(s + "_")), None)


def check_launch(ops, n, want_stages):
    """Rules 1-3 on one set-up + upload + launch of n samples; returns {stage: (stream, upload event, first arena upload index)}."""
    memsets = [i for i, o in enumerate(ops) if o[0] == "memset"]
    status = memsets[0]
    assert ops[status][2] == str(4 * n), ops[status]                    # the status clear is the launch's first memset
    main = ops[status][1]
    streams = {}
    for o in ops:
        if stage_of(o):
            streams.setdefault(stage_of(o), set()).add(o[2])
    assert set(streams) == set(want_stages), streams
    out = {}
    for stage, ss in streams.items():
        # 1. one stream per stage, not the caller's
        assert len(ss) == 1 and main not in ss, (stage, ss, main)
        s = next(iter(ss))
        on_s = [i for i, o in enumerate(ops) if stream_of(o) == s and o[0] != "wait" and o[0] != "record"]
        launches = [i for i in on_s if ops[i][0] == "launch"]
        assert all(stage_of(ops[i]) == stage for i in launches), [ops[i] for i in launches]
        # 2. forked behind the status clear
        first = on_s[0]
        forks = [ops[i][2] for i in range(first) if ops[i][0] == "wait" and ops[i][1] == s]
        recorded = {ops[i][1]: i for i in range(status + 1, first) if ops[i][0] == "record" and ops[i][2] == main}
        assert any(e in recorded for e in forks), (stage, forks, recorded)
        if stage == "ljpeg":
            scatter = next(i for i, o in enumerate(ops) if o[0] == "launch" and o[1] == "dalib200::unstuff_scatter_kernel")
            assert any(recorded[e] > scatter for e in forks if e in recorded), (stage, forks, recorded, scatter)
        # 3. joined in front of the kernel that reads the stage's result
        last = launches[-1]
        joins = [ops[i][1] for i in range(last + 1, len(ops)) if ops[i][0] == "record" and ops[i][2] == s]
        assert joins, stage
        reader = "dalib200::dc_scan_kernel" if stage == "prog" else "dalib200::jpeg_post_kernel"
        r = next(i for i, o in enumerate(ops) if o[0] == "launch" and o[1].startswith(reader))
        assert any(ops[i][0] == "wait" and ops[i][1] == main and ops[i][2] == joins[0] for i in range(last + 1, r)), (stage, reader)
        h2d = next(i for i in on_s if ops[i][0] == "h2d")
        upload = next(ops[i][1] for i in range(h2d + 1, len(ops)) if ops[i][0] == "record" and ops[i][2] == s)
        out[stage] = (s, upload, h2d)
    return out


def test_side_stages_fork_join_and_reuse_their_arenas_in_order(stub, tmp_path):
    sections = run_trace(stub, str(tmp_path / "trace.txt"))
    names = [" ".join(t) for t, _ in sections]
    assert names == ["mixed 0", "mixed 1", "jpeg-only 3", "destroy", "webp-only 2", "destroy"], names
    first = check_launch(sections[0][1], 7, STAGES)
    second = check_launch(sections[1][1], 7, STAGES)
    ops = sections[1][1]
    assert not any(o[0] == "stream_create" for o in ops), "a stage stream was created twice"
    for stage, (s, upload, h2d) in second.items():
        assert first[stage][:2] == (s, upload), stage                     # the stage's stream and events persist across launches
        # 4. the previous upload of the pinned arena has finished before it is overwritten
        assert any(o[0] == "event_sync" and o[1] == upload for o in ops[:h2d]), stage
    # 5. no side-stage stream or event in a JPEG-only batch, even on a plan whose stages have run before
    side_streams = {s for s, _, _ in first.values()}
    side_events = {o[1] for _, sec in sections[:2] for o in sec if o[0] == "record" and o[2] in side_streams}
    side_events |= {o[2] for _, sec in sections[:2] for o in sec if o[0] == "wait" and o[1] in side_streams}
    for o in sections[2][1]:
        assert o[0] not in ("wait", "stream_create"), o
        assert stream_of(o) not in side_streams and not (o[0] in ("record", "event_sync") and o[1] in side_events), o
    check_launch(sections[2][1], 3, ())
    check_launch(sections[4][1], 2, ("webp",))
    assert sum(o[0] == "stream_create" for o in sections[4][1]) == 1
