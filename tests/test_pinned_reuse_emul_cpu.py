"""Reuse of the page-locked staging buffers, checked WITHOUT a GPU.  Every plan stages its per-batch descriptors (and the decoder its
scan bytes) in pinned host memory and copies them to the device with asynchronous H2D copies; rewriting such a buffer while the
previous copy may still read it is a race that a GPU shows only as an intermittent wrong result, and the emulated copies (which run
synchronously) never show.  So this test reads the call trace of tools/emul/cuda_emul_stub.cc (DALIB200_EMUL_TRACE), in which each H2D
copy names the cudaMallocHost allocation it reads, while one plan of every kind is set up and launched twice (with shapes that change,
so that tables are uploaded again too).  For every pinned buffer the second run copies out of, the event recorded on the stream of the
first run's last copy out of it must be synchronised before the second run's first copy out of it."""
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


# Each case sets up and launches one plan twice, through the C-ABI with host buffers ("device" memory is host memory under the stub),
# writing a "# <case> <run>" line in front of each run.
SCRIPT = r"""
import ctypes as C, os, sys
import numpy as np
root = sys.argv[1]
sys.path.insert(0, root); sys.path.insert(0, os.path.join(root, "tests"))
from dali_b200 import capi
import gpu_helpers as g

lib = capi.lib()
stub = C.CDLL(os.environ["EMUL_STUB"])
chk = capi.check
keep = []

def ptrs(sizes):
    out = []
    for s in sizes:
        a = np.zeros(max(int(s), 64), np.uint8)
        keep.append(a)
        out.append(a.ctypes.data)
    return (C.c_void_p * len(out))(*out)

def i64(v): return (C.c_int64 * len(v))(*v)
def f32(v): return (C.c_float * len(v))(*v)

class WindowSample(C.Structure):
    _fields_ = [("in_h", C.c_int32), ("in_w", C.c_int32), ("channels", C.c_int32), ("anchor_y", C.c_int32), ("anchor_x", C.c_int32),
                ("out_h", C.c_int32), ("out_w", C.c_int32), ("flip_x", C.c_int32), ("flip_y", C.c_int32), ("fill", C.c_uint8 * 4)]

class AudioResampleSample(C.Structure):
    _fields_ = [("in_rate", C.c_double), ("out_rate", C.c_double), ("in_length", C.c_int64), ("out_length", C.c_int64), ("channels", C.c_int32)]

class NonsilentSample(C.Structure):
    _fields_ = [("cutoff_db", C.c_float), ("reference_power", C.c_float), ("use_reference_power", C.c_int32)]

N = 3
IMG = [48 * 64 * 3] * N

def warp(h, k):
    s = (capi.WarpSample * N)()
    for x in s:
        x.in_h, x.in_w, x.channels, x.out_h, x.out_w = 48, 64, 3, 40 + k, 56
        x.matrix[:] = [1.0, 0.0, 0.5, 0.0, 1.0, 0.25]
    chk(lib.dalib200WarpPlanSetup(h, N, s, 1, 0, C.c_float(0.0), capi.UINT8))
    chk(lib.dalib200WarpLaunch(h, ptrs(IMG), ptrs(IMG), None))

def cmn(h, k):
    s = (capi.CmnSample * N)()
    for x in s:
        x.in_h, x.in_w, x.channels, x.anchor_y, x.anchor_x, x.crop_h, x.crop_w = 48, 64, 3, 2, 3, 32 + k, 40
        x.inv_std[:] = [1.0] * 4
    chk(lib.dalib200CmnPlanSetup(h, N, s, capi.FLOAT, capi.LAYOUT_CHW, 3))
    chk(lib.dalib200CmnLaunch(h, ptrs(IMG), ptrs([4 * 48 * 64 * 3] * N), None))

def linear(h, k):
    s = (capi.ColorSample * N)()
    for x in s:
        x.num_pixels = 48 * 64 - k
        x.matrix[:] = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
    chk(lib.dalib200LinearTransformSetup(h, N, s, capi.UINT8))
    chk(lib.dalib200PointwiseLaunch(h, ptrs(IMG), ptrs(IMG), None))

def csc(h, k):
    chk(lib.dalib200ColorSpaceSetup(h, N, i64([48 * 64 - k] * N), capi.RGB, capi.GRAY))
    chk(lib.dalib200PointwiseLaunch(h, ptrs(IMG), ptrs(IMG), None))

def multiply_add(h, k):
    chk(lib.dalib200MultiplyAddSetup(h, N, i64([4000 + k] * N), f32([1.5] * N), f32([2.0] * N), capi.UINT8))
    chk(lib.dalib200GenericLaunch(h, ptrs([4001] * N), ptrs([4001] * N), None))

def window_copy(h, k):
    s = (WindowSample * N)()
    for x in s:
        x.in_h, x.in_w, x.channels, x.anchor_y, x.anchor_x, x.out_h, x.out_w = 48, 64, 3, -2, 5, 30 + k, 40
    chk(lib.dalib200WindowCopySetup(h, N, s))
    chk(lib.dalib200GenericLaunch(h, ptrs(IMG), ptrs(IMG), None))

def pad(h, k):
    fill = C.c_uint8(7)
    chk(lib.dalib200PadSetup(h, N, 2, 1, i64([10, 20] * N), i64([12 + k, 24] * N), C.byref(fill)))
    chk(lib.dalib200GenericLaunch(h, ptrs([200] * N), ptrs([300] * N), None))

def resample(h, k):
    s = (capi.ResampleSample * N)()
    for x in s:
        g.fill_resample_sample(x, (64, 64, 3), (30 + k, 32), capi.FILTER_LINEAR, capi.FILTER_LINEAR, None)
    chk(lib.dalib200ResamplePlanSetup(h, N, s, capi.UINT8, capi.UINT8))
    chk(lib.dalib200ResampleLaunch(h, ptrs([64 * 64 * 3] * N), ptrs([64 * 64 * 3] * N), None))

def resample3d(h, k):
    s = (capi.Resample3DSample * N)()
    for x in s:
        for d in range(3):
            x.in_shape[d], x.out_shape[d] = 6 + d, 4 + d + k
            x.min_filter[d] = x.mag_filter[d] = capi.FilterDesc(capi.FILTER_LINEAR, 1, 0.0)
        x.channels = 2
    chk(lib.dalib200Resample3DPlanSetup(h, N, s, capi.UINT8, capi.UINT8))
    chk(lib.dalib200Resample3DLaunch(h, ptrs([6 * 7 * 8 * 2] * N), ptrs([(4 + k) * (5 + k) * (6 + k) * 2] * N), None))

def jpeg_distort(h, k):
    s = (capi.JpegDistortSample * N)(*[capi.JpegDistortSample(40 + k, 48, 50 + 10 * i) for i in range(N)])
    chk(lib.dalib200JpegDistortPlanSetup(h, N, s))
    chk(lib.dalib200JpegDistortLaunch(h, ptrs([41 * 48 * 3] * N), ptrs([41 * 48 * 3] * N), None))

def signal(setup):
    def step(h, k):
        setup(h, k)
        chk(lib.dalib200SignalLaunch(h, ptrs([4 * 4096] * N), ptrs([4 * 4096] * N), None))
    return step

def todb(h, k):
    a = capi.ToDecibelsArgs(10.0, 1.0, -80.0, 0)
    chk(lib.dalib200ToDecibelsSetup(h, C.byref(a), N, i64([1000 + k] * N)))

def mfcc(h, k):
    a = capi.MfccArgs(8 + k, 2, 0, 0.0)
    chk(lib.dalib200MfccSetup(h, C.byref(a), N, i64([16, 20] * N)))

def normalize(h, k):
    a = capi.NormalizeArgs(1, 0, 1.0, 0.0, 0.0)
    chk(lib.dalib200NormalizeSetup(h, C.byref(a), N, i64([8, 20 + k] * N)))

def audio_resample(h, k):
    s = (AudioResampleSample * N)(*[AudioResampleSample(16000.0, 8000.0, 1000, 500, 1) for _ in range(N)])
    chk(lib.dalib200AudioResampleSetup(h, N, s, C.c_float(50.0 + 10 * k)))

def preemphasis(h, k):
    chk(lib.dalib200PreemphasisSetup(h, N, i64([1000 + k] * N), f32([0.97] * N), capi.BORDER_CLAMP, capi.FLOAT))

def nonsilent(h, k):
    s = (NonsilentSample * N)(*[NonsilentSample(-60.0, 0.0, 0) for _ in range(N)])
    chk(lib.dalib200NonsilentSetup(h, N, i64([1000 + k] * N), s, 8, -1))
    chk(lib.dalib200NonsilentLaunch(h, ptrs([4 * 1001] * N), ptrs([4] * N), ptrs([4] * N), None))

def spectrogram_args(nfft):
    return capi.SpectrogramArgs(nfft, nfft, nfft // 2, 2, 1, 1, 1)

def spectrogram(h, k):
    a = spectrogram_args(256)
    chk(lib.dalib200SpectrogramPlanSetup(h, C.byref(a), None, N, i64([2000 + k] * N)))
    chk(lib.dalib200SpectrogramLaunch(h, ptrs([4 * 2001] * N), ptrs([4 * 129 * 20] * N), None))

def mel(tensor_cores):
    def step(h, k):
        a = capi.MelArgs(16 + k, 16000.0, 0.0, 0.0, 0, 1)
        chk(lib.dalib200MelPlanSetTensorCores(h, tensor_cores))
        chk(lib.dalib200MelPlanSetup(h, C.byref(a), 129, N, i64([20] * N)))
        chk(lib.dalib200MelLaunch(h, ptrs([4 * 129 * 20] * N), ptrs([4 * 17 * 20] * N), None))
    return step

mel_for_fused = []
def spectrogram_mel(h, k):
    if not mel_for_fused:
        mel_for_fused.append(capi.Plan("Mel", N))
    m = mel_for_fused[0].handle
    a = spectrogram_args(1024)
    chk(lib.dalib200SpectrogramPlanSetup(h, C.byref(a), None, N, i64([8000 + k] * N)))
    nwin = [lib.dalib200SpectrogramNumWindows(h, i) for i in range(N)]
    ma = capi.MelArgs(32 + k, 16000.0, 0.0, 0.0, 0, 1)
    chk(lib.dalib200MelPlanSetup(m, C.byref(ma), 513, N, i64(nwin)))
    chk(lib.dalib200SpectrogramMelLaunch(h, m, ptrs([4 * 8001] * N), None, ptrs([4 * 33 * 20] * N), None))

def jpeg(h, k):
    import cv2
    import png_streams as ps
    import tiff_streams as ts
    import webp_streams as ws
    streams = [cv2.imencode(".jpg", g.synth_image(96, 128, 1))[1].tobytes(),
               cv2.imencode(".jpg", g.synth_image(64, 80, 2), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes(),
               ps.encode(ps.samples(30, 41, 2, 8, 5), 2, 8, filters="mixed"),
               ts.encode(ts.samples(20, 30, 3, 8, 6), 2, 8, 5, 2, rows_per_strip=3),
               ws.cv2_webp(ws.image(40, 56, 7), 70)]
    n = len(streams)
    bufs = [np.frombuffer(bytes(s), np.uint8) for s in streams]
    prm = capi.JpegParams(capi.RGB, 1, capi.FLOAT, 0)
    chk(lib.dalib200JpegPlanSetupEx(h, n, (C.c_void_p * n)(*[b.ctypes.data for b in bufs]), (C.c_size_t * n)(*[b.size for b in bufs]),
                                    C.byref(prm), None))
    chk(lib.dalib200JpegUpload(h, None))
    chk(lib.dalib200JpegLaunch(h, ptrs([4 * 96 * 144 * 3] * n), None))

CASES = [("warp", "Warp", warp), ("cmn", "Cmn", cmn), ("linear_transform", "Pointwise", linear), ("color_space", "Pointwise", csc),
         ("multiply_add", "Generic", multiply_add), ("window_copy", "Generic", window_copy), ("pad", "Generic", pad),
         ("resample", "Resample", resample), ("resample3d", "Resample3D", resample3d), ("jpeg_distort", "JpegDistort", jpeg_distort),
         ("to_decibels", "Signal", signal(todb)), ("mfcc", "Signal", signal(mfcc)), ("normalize", "Signal", signal(normalize)),
         ("audio_resample", "Signal", signal(audio_resample)), ("preemphasis", "Signal", signal(preemphasis)),
         ("nonsilent", "Signal", nonsilent), ("spectrogram", "Spectrogram", spectrogram), ("mel", "Mel", mel(0)),
         ("mel_tensor_cores", "Mel", mel(1)), ("spectrogram_mel", "Spectrogram", spectrogram_mel), ("jpeg", "Jpeg", jpeg)]
for name, kind, step in CASES:
    plan = capi.Plan(kind, 6)
    for k in range(2):
        stub.emul_trace_mark(("%s %d" % (name, k)).encode())
        step(plan.handle, k)
    del plan
print("trace-ok")
"""

# pinned buffers each case must copy out of in both runs, at least (descriptor arenas, tables, the decoder's staging buffers and side
# stage arenas)
MIN_BUFFERS = {"warp": 1, "cmn": 1, "linear_transform": 1, "color_space": 1, "multiply_add": 1, "window_copy": 1, "pad": 1,
               "resample": 3, "resample3d": 2, "jpeg_distort": 1, "to_decibels": 1, "mfcc": 1, "normalize": 1, "audio_resample": 1,
               "preemphasis": 1, "nonsilent": 1, "spectrogram": 1, "mel": 2, "mel_tensor_cores": 3, "spectrogram_mel": 3, "jpeg": 6}


def run_trace(stub, trace):
    env = dict(os.environ, LD_PRELOAD=stub, EMUL_STUB=stub, DALIB200_EMUL_TRACE=trace)
    r = subprocess.run([sys.executable, "-c", SCRIPT, ROOT], capture_output=True, text=True, timeout=600, env=env, cwd=ROOT)
    assert r.returncode == 0 and "trace-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
    sections = {}
    ops = None
    with open(trace) as f:
        for line in f:
            w = line.split()
            if w[0] == "#":
                ops = sections.setdefault(" ".join(w[1:]), [])
            elif ops is not None:
                ops.append(w)
    return sections


def test_every_plan_waits_for_the_last_copy_out_of_a_pinned_buffer_before_reusing_it(stub, tmp_path):
    sections = run_trace(stub, str(tmp_path / "trace.txt"))
    assert sorted(sections) == sorted("%s %d" % (c, k) for c in MIN_BUFFERS for k in range(2)), sorted(sections)
    for case, want in MIN_BUFFERS.items():
        first, second = sections[case + " 0"], sections[case + " 1"]
        ops = first + second
        last = {o[3]: i for i, o in enumerate(first) if o[0] == "h2d" and o[3] != "-"}
        reused = {}
        for i, o in enumerate(second):
            if o[0] == "h2d" and o[3] in last:
                reused.setdefault(o[3], len(first) + i)
        for buf, again in reused.items():
            stream = ops[last[buf]][1]
            rec = next((i for i in range(last[buf] + 1, len(ops)) if ops[i][0] == "record" and ops[i][2] == stream), None)
            assert rec is not None and rec < again, (case, buf, "no event recorded behind the copy")
            assert any(o[0] == "event_sync" and o[1] == ops[rec][1] for o in ops[rec + 1:again]), (case, buf, "copied again without a wait")
        assert len(reused) >= want, (case, sorted(reused))
