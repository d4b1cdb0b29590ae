"""Launch accounting, checked WITHOUT a GPU.  Every kernel launch of the library adds one to dalib200GetLaunchCount (bench.py's
gpu_launches) and, with profiling on, one named record to dalib200ProfilingCollect (the per-kernel breakdown bench.py's roofline is
keyed on).  This test runs one batch of every plan family with tools/emul/cuda_emul_stub.cc preloaded, which writes every
cudaLaunchKernel call to its trace (DALIB200_EMUL_TRACE), and checks for each batch that the three agree: the change of the counter,
the number of launches the trace gained and the number of profile records, each of which must carry a name."""
import json
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
    pytest.importorskip("cv2")
    so = str(tmp_path_factory.mktemp("emul") / "cuda_emul_stub.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I/usr/local/cuda/include",
                        os.path.join(ROOT, "tools", "emul", "cuda_emul_stub.cc"), "-o", so, "-ldl"], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return so


# Runs each workload through the C-ABI (host buffers: "device" memory is host memory under the stub) and prints one JSON line per
# workload: the counter's change, the launch lines the trace gained and the profile records' names.
SCRIPT = r"""
import ctypes as C, json, os, sys
import numpy as np
root = sys.argv[1]
sys.path.insert(0, root); sys.path.insert(0, os.path.join(root, "tests"))
import conftest                      # DALIB200_DRYRUN=emul: "device" tensors are host memory
import cv2
import gpu_helpers as g
from dali_b200 import capi
from dali_b200.hotpath import ImagePipelineC2
import audio_streams as aus
import bitmap_streams as bs
import ljpeg_streams as ls
import png_streams as ps
import tiff_streams as ts
import webp_streams as ws

lib = capi.lib()
chk = capi.check
keep = []

def buf(nbytes):
    a = np.zeros(max(int(nbytes), 64), np.uint8)
    keep.append(a)
    return a.ctypes.data

def ptrs(sizes):
    return (C.c_void_p * len(sizes))(*[buf(s) for s in sizes])

def i64(v): return (C.c_int64 * len(v))(*v)
def f32(v): return (C.c_float * len(v))(*v)

def trace_launches():
    if not os.path.exists(os.environ["DALIB200_EMUL_TRACE"]):    # the stub opens it at its first traced call
        return 0
    with open(os.environ["DALIB200_EMUL_TRACE"]) as f:
        return sum(line.startswith("launch ") for line in f)

def jpg(h, w, seed, *flags):
    return cv2.imencode(".jpg", g.synth_image(h, w, seed), [cv2.IMWRITE_JPEG_QUALITY, 90, *flags])[1].tobytes()

N = 3
IMG = [48 * 64 * 3] * N

def c2(fused):
    def run():
        streams = [np.frombuffer(jpg(h, w, i), np.uint8) for i, (h, w) in enumerate([(480, 640), (360, 500), (1080, 1920), (97, 131)])]
        pipe = ImagePipelineC2(len(streams), fused=fused)
        pipe.run(streams, [0, 1, 0, 1])
        assert pipe.status() == [0] * len(streams)
        if fused:
            assert any(pipe.planar)
    return run

def progressive():
    streams = [jpg(64, 80, 2, cv2.IMWRITE_JPEG_PROGRESSIVE, 1), jpg(97, 61, 3, cv2.IMWRITE_JPEG_PROGRESSIVE, 1)]
    _, status = g.jpeg_decode(streams)
    assert status == [0, 0], status

def mixed():
    streams = [jpg(96, 128, 1), jpg(64, 80, 2, cv2.IMWRITE_JPEG_PROGRESSIVE, 1), ps.encode(ps.samples(30, 41, 2, 8, 5), 2, 8, filters="mixed"),
               ts.encode(ts.samples(20, 30, 3, 8, 6), 2, 8, 5, 2, rows_per_strip=3), ws.cv2_webp(ws.image(40, 56, 7), 70),
               bs.bmp(31, 17, 24, bs.rows(bs.image(17, 31, 1), 24)), ls.encode(ls.image(33, 17, 1, 6, 71), P=6, Pt=2, restart=17 * 4)]
    n = len(streams)
    bufs = [np.frombuffer(s, np.uint8) for s in streams]
    plan = capi.Plan("Jpeg", n)
    prm = capi.JpegParams(capi.RGB, 1, capi.FLOAT, 0)
    chk(lib.dalib200JpegPlanSetupEx(plan.handle, n, (C.c_void_p * n)(*[b.ctypes.data for b in bufs]), (C.c_size_t * n)(*[b.size for b in bufs]),
                                    C.byref(prm), None))
    outs = []
    for i in range(n):
        hwc = (C.c_int32 * 3)()
        chk(lib.dalib200JpegPlanGetOutputShape(plan.handle, i, hwc))
        outs.append(4 * hwc[0] * hwc[1] * hwc[2])
    chk(lib.dalib200JpegUpload(plan.handle, None))
    chk(lib.dalib200JpegLaunch(plan.handle, ptrs(outs), None))
    status = (C.c_int32 * n)()
    chk(lib.dalib200JpegGetStatus(plan.handle, status))
    assert list(status) == [0] * n, list(status)

def launch(kind, setup, run):
    def step():
        plan = capi.Plan(kind, 8)
        setup(plan.handle)
        run(plan.handle)
    return step

def jpeg_distort(h):                 # a sample 4 pixels wide takes the IDCT kernel and a colour kernel instead of the fused 4:2:0 one
    s = (capi.JpegDistortSample * N)(capi.JpegDistortSample(40, 48, 50), capi.JpegDistortSample(40, 48, 60), capi.JpegDistortSample(8, 4, 70))
    chk(lib.dalib200JpegDistortPlanSetup(h, N, s))

def resample(h):                     # 16-byte rows take the streaming kernel, the others the tile kernel
    s = (capi.ResampleSample * N)()
    for x, w in zip(s, (64, 50, 64)):
        g.fill_resample_sample(x, (64, w, 3), (30, 32), capi.FILTER_LINEAR, capi.FILTER_LINEAR, None)
    chk(lib.dalib200ResamplePlanSetup(h, N, s, capi.UINT8, capi.UINT8))

def resample3d(h):
    s = (capi.Resample3DSample * N)()
    for x in s:
        for d in range(3):
            x.in_shape[d], x.out_shape[d] = 6 + d, 4 + d
            x.min_filter[d] = x.mag_filter[d] = capi.FilterDesc(capi.FILTER_LINEAR, 1, 0.0)
        x.channels = 2
    chk(lib.dalib200Resample3DPlanSetup(h, N, s, capi.UINT8, capi.UINT8))

def warp(h):
    s = (capi.WarpSample * N)()
    for x in s:
        x.in_h, x.in_w, x.channels, x.out_h, x.out_w = 48, 64, 3, 40, 56
        x.matrix[:] = [1.0, 0.0, 0.5, 0.0, 1.0, 0.25]
    chk(lib.dalib200WarpPlanSetup(h, N, s, 1, 0, C.c_float(0.0), capi.UINT8))

def cmn(layout):
    def setup(h):
        s = (capi.CmnSample * N)()
        for x in s:
            x.in_h, x.in_w, x.channels, x.anchor_y, x.anchor_x, x.crop_h, x.crop_w = 48, 64, 3, 2, 3, 32, 40
            x.inv_std[:] = [1.0] * 4
        chk(lib.dalib200CmnPlanSetup(h, N, s, capi.FLOAT16, layout, 3))
    return setup

def linear(h):
    s = (capi.ColorSample * N)()
    for x in s:
        x.num_pixels = 48 * 64
        x.matrix[:] = [1.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0]
    chk(lib.dalib200LinearTransformSetup(h, N, s, capi.FLOAT))

class WindowSample(C.Structure):
    _fields_ = [("in_h", C.c_int32), ("in_w", C.c_int32), ("channels", C.c_int32), ("anchor_y", C.c_int32), ("anchor_x", C.c_int32),
                ("out_h", C.c_int32), ("out_w", C.c_int32), ("flip_x", C.c_int32), ("flip_y", C.c_int32), ("fill", C.c_uint8 * 4)]

def window_copy(h):
    s = (WindowSample * N)()
    for x in s:
        x.in_h, x.in_w, x.channels, x.anchor_y, x.anchor_x, x.out_h, x.out_w = 48, 64, 3, -2, 5, 30, 40
    chk(lib.dalib200WindowCopySetup(h, N, s))

def pad(h):
    fill = C.c_uint8(7)
    chk(lib.dalib200PadSetup(h, N, 2, 1, i64([10, 20] * N), i64([12, 24] * N), C.byref(fill)))

def spectrogram(nfft):
    def setup(h):
        a = capi.SpectrogramArgs(nfft, nfft, nfft // 2, 2, 1, 1, 1)
        chk(lib.dalib200SpectrogramPlanSetup(h, C.byref(a), None, N, i64([2000] * N)))
    return setup

def mel(tensor_cores):
    def setup(h):
        a = capi.MelArgs(16, 16000.0, 0.0, 0.0, 0, 1)
        chk(lib.dalib200MelPlanSetTensorCores(h, tensor_cores))
        chk(lib.dalib200MelPlanSetup(h, C.byref(a), 129, N, i64([20] * N)))
    return setup

def spectrogram_mel():
    sp, mp = capi.Plan("Spectrogram", N), capi.Plan("Mel", N)
    a = capi.SpectrogramArgs(1024, 1024, 512, 2, 1, 1, 1)
    chk(lib.dalib200SpectrogramPlanSetup(sp.handle, C.byref(a), None, N, i64([8000] * N)))
    nwin = [lib.dalib200SpectrogramNumWindows(sp.handle, i) for i in range(N)]
    ma = capi.MelArgs(32, 16000.0, 0.0, 0.0, 0, 1)
    chk(lib.dalib200MelPlanSetup(mp.handle, C.byref(ma), 513, N, i64(nwin)))
    chk(lib.dalib200SpectrogramMelLaunch(sp.handle, mp.handle, ptrs([4 * 8001] * N), None, ptrs([4 * 33 * 20] * N), None))

def todb(h):
    a = capi.ToDecibelsArgs(10.0, 1.0, -80.0, 1)
    chk(lib.dalib200ToDecibelsSetup(h, C.byref(a), N, i64([1000] * N)))

def mfcc(h):
    a = capi.MfccArgs(8, 2, 0, 0.0)
    chk(lib.dalib200MfccSetup(h, C.byref(a), N, i64([16, 20] * N)))

def normalize(h):
    a = capi.NormalizeArgs(1, 0, 1.0, 0.0, 0.0)
    chk(lib.dalib200NormalizeSetup(h, C.byref(a), N, i64([8, 20] * N)))

class AudioResampleSample(C.Structure):
    _fields_ = [("in_rate", C.c_double), ("out_rate", C.c_double), ("in_length", C.c_int64), ("out_length", C.c_int64), ("channels", C.c_int32)]

def audio_resample(h):
    s = (AudioResampleSample * N)(*[AudioResampleSample(16000.0, 8000.0, 1000, 500, 1) for _ in range(N)])
    chk(lib.dalib200AudioResampleSetup(h, N, s, C.c_float(50.0)))

def preemphasis(h):
    chk(lib.dalib200PreemphasisSetup(h, N, i64([1000] * N), f32([0.97] * N), capi.BORDER_CLAMP, capi.FLOAT))

class NonsilentSample(C.Structure):
    _fields_ = [("cutoff_db", C.c_float), ("reference_power", C.c_float), ("use_reference_power", C.c_int32)]

def nonsilent(h):
    s = (NonsilentSample * N)(*[NonsilentSample(-60.0, 0.0, 0) for _ in range(N)])
    chk(lib.dalib200NonsilentSetup(h, N, i64([1000] * N), s, 8, -1))

def audio_decode():
    rng = np.random.default_rng(3)
    x = aus.signal(1252, 2, 16, rng)
    streams = [aus.wav_pcm(x, 16, 16000), aus.flac(x, 16, 16000, [576, 576, 100])]
    n = len(streams)
    bufs = [np.frombuffer(s, np.uint8) for s in streams]
    plan = capi.Plan("Audio", n)
    prm = (capi.AudioParams * n)(*[capi.AudioParams(0, 0.0, 50.0, capi.FLOAT)] * n)
    chk(lib.dalib200AudioPlanSetup(plan.handle, n, (C.c_void_p * n)(*[b.ctypes.data for b in bufs]), (C.c_size_t * n)(*[b.size for b in bufs]), prm))
    chk(lib.dalib200AudioLaunch(plan.handle, ptrs([4 * x.size] * n), ptrs([4] * n), None))
    chk(lib.dalib200AudioStatusAsync(plan.handle, None))
    st = (C.c_int32 * n)()
    chk(lib.dalib200AudioStatusFetch(plan.handle, st, n))
    assert list(st) == [0] * n, list(st)

def arith():
    plan = capi.Plan("Arith", N)
    ot = C.c_int32()
    chk(lib.dalib200ArithCompile(plan.handle, b"add(&0 &1)", 2, (C.c_int32 * 2)(capi.FLOAT, capi.FLOAT), (C.c_uint8 * 2)(0, 0), None, 0,
                                 None, 0, C.byref(ot)))
    shp = (C.c_int64 * (N * 2 * 6))(*([16, 24, 3, 0, 0, 0] * 2 * N))
    osh, ond = (C.c_int64 * (6 * N))(), C.c_int32()
    chk(lib.dalib200ArithSetup(plan.handle, N, (C.c_int32 * 2)(3, 3), shp, None, osh, C.byref(ond)))
    chk(lib.dalib200ArithLaunch(plan.handle, ptrs([4 * 16 * 24 * 3] * 2 * N), ptrs([4 * 16 * 24 * 3] * N), None))

def permute():
    plan = capi.Plan("Permute", N)
    osh = (C.c_int64 * (3 * N))()
    chk(lib.dalib200TransposeSetup(plan.handle, N, 3, 1, i64([48, 64, 3] * N), (C.c_int32 * 3)(2, 0, 1), osh))
    chk(lib.dalib200PermuteLaunch(plan.handle, ptrs(IMG), ptrs(IMG), None))

def reduce_split():                  # a sum over 2^20 elements is cut into chunks: a pass and a combine launch
    plan = capi.Plan("Reduce", 2)
    ot, osh = C.c_int32(-1), (C.c_int64 * 2)()
    chk(lib.dalib200ReduceSetup(plan.handle, 2, capi.FLOAT, C.byref(ot), 2, 1, i64([1 << 20, 1000]), C.c_uint32(1), 0, 0, osh))
    chk(lib.dalib200ReduceLaunch(plan.handle, ptrs([4 << 20, 4000]), None, ptrs([8, 8]), None))

def equalize():
    plan = capi.Plan("Equalize", N)
    chk(lib.dalib200EqualizeSetup(plan.handle, capi.UINT8, N, 3, i64([48, 64, 3] * N), b"HWC"))
    chk(lib.dalib200EqualizeLaunch(plan.handle, ptrs(IMG), ptrs(IMG), None))

def signal(setup):
    return launch("Signal", setup, lambda h: chk(lib.dalib200SignalLaunch(h, ptrs([4 * 4096] * N), ptrs([4 * 4096] * N), None)))

WORKLOADS = [
    ("c2", c2(False)), ("c2_fused", c2(True)), ("progressive", progressive), ("mixed", mixed),
    ("jpeg_distort", launch("JpegDistort", jpeg_distort, lambda h: chk(lib.dalib200JpegDistortLaunch(h, ptrs([40 * 48 * 3] * N), ptrs([40 * 48 * 3] * N), None)))),
    ("resample", launch("Resample", resample, lambda h: chk(lib.dalib200ResampleLaunch(h, ptrs([64 * 64 * 3] * N), ptrs([30 * 32 * 3] * N), None)))),
    ("resample3d", launch("Resample3D", resample3d, lambda h: chk(lib.dalib200Resample3DLaunch(h, ptrs([6 * 7 * 8 * 2] * N), ptrs([4 * 5 * 6 * 2] * N), None)))),
    ("warp", launch("Warp", warp, lambda h: chk(lib.dalib200WarpLaunch(h, ptrs(IMG), ptrs(IMG), None)))),
    ("cmn_chw", launch("Cmn", cmn(capi.LAYOUT_CHW), lambda h: chk(lib.dalib200CmnLaunch(h, ptrs(IMG), ptrs([2 * 48 * 64 * 3] * N), None)))),
    ("cmn_hwc", launch("Cmn", cmn(capi.LAYOUT_HWC), lambda h: chk(lib.dalib200CmnLaunch(h, ptrs(IMG), ptrs([2 * 48 * 64 * 3] * N), None)))),
    ("linear_transform", launch("Pointwise", linear, lambda h: chk(lib.dalib200PointwiseLaunch(h, ptrs(IMG), ptrs([4 * 48 * 64 * 3] * N), None)))),
    ("color_space", launch("Pointwise", lambda h: chk(lib.dalib200ColorSpaceSetup(h, N, i64([48 * 64] * N), capi.RGB, capi.GRAY)),
                           lambda h: chk(lib.dalib200PointwiseLaunch(h, ptrs(IMG), ptrs(IMG), None)))),
    ("multiply_add", launch("Generic", lambda h: chk(lib.dalib200MultiplyAddSetup(h, N, i64([4000] * N), f32([1.5] * N), f32([2.0] * N), capi.FLOAT)),
                            lambda h: chk(lib.dalib200GenericLaunch(h, ptrs([4000] * N), ptrs([4 * 4000] * N), None)))),
    ("window_copy", launch("Generic", window_copy, lambda h: chk(lib.dalib200GenericLaunch(h, ptrs(IMG), ptrs(IMG), None)))),
    ("pad", launch("Generic", pad, lambda h: chk(lib.dalib200GenericLaunch(h, ptrs([200] * N), ptrs([300] * N), None)))),
    ("spectrogram_mel_two_kernels", lambda: [
        launch("Spectrogram", spectrogram(256), lambda h: chk(lib.dalib200SpectrogramLaunch(h, ptrs([4 * 2000] * N), ptrs([4 * 129 * 20] * N), None)))(),
        launch("Mel", mel(0), lambda h: chk(lib.dalib200MelLaunch(h, ptrs([4 * 129 * 20] * N), ptrs([4 * 16 * 20] * N), None)))()]),
    ("spectrogram_dft", launch("Spectrogram", spectrogram(200), lambda h: chk(lib.dalib200SpectrogramLaunch(h, ptrs([4 * 2000] * N), ptrs([4 * 101 * 21] * N), None)))),
    ("spectrogram_mel_fused", spectrogram_mel),
    ("mel_tensor_cores", launch("Mel", mel(1), lambda h: chk(lib.dalib200MelLaunch(h, ptrs([4 * 129 * 20] * N), ptrs([4 * 16 * 20] * N), None)))),
    ("to_decibels_max", signal(todb)), ("mfcc", signal(mfcc)), ("normalize", signal(normalize)),
    ("audio_resample", signal(audio_resample)), ("preemphasis", signal(preemphasis)),
    ("nonsilent", launch("Signal", nonsilent, lambda h: chk(lib.dalib200NonsilentLaunch(h, ptrs([4 * 1000] * N), ptrs([4] * N), ptrs([4] * N), None)))),
    ("audio_decode", audio_decode), ("arith", arith), ("permute", permute), ("reduce_split", reduce_split), ("equalize", equalize),
]

only = sys.argv[2].split(",") if len(sys.argv) > 2 else None
capi.profiling(True)
for name, run in WORKLOADS:
    if only and name not in only:
        continue
    capi.profiling_collect()
    count, traced = capi.launch_count(), trace_launches()
    run()
    records = capi.profiling_collect()
    print(json.dumps({"workload": name, "count": capi.launch_count() - count, "traced": trace_launches() - traced,
                      "records": [r for r, _ in records]}))
capi.profiling(False)
print("accounting-ok")
"""

# profile names each workload must reach, so that it covers the launches it is meant to
WANT = {
    "c2": {"jpeg_unstuff_scatter", "jpeg_huff_sync_intra", "jpeg_huff_sync_walk3", "jpeg_huff_write", "jpeg_idct_color", "resample_stream",
           "cmn_hwc2chw"},
    "c2_fused": {"jpeg_idct", "resample_planar", "cmn_hwc2chw"},
    "progressive": {"jpeg_prog_scan", "jpeg_prog_dc", "jpeg_dc_scan"},
    "mixed": {"jpeg_prog_scan", "png_inflate", "tiff_segment", "webp_filter", "bitmap_color", "ljpeg_write", "jpeg_post"},
    "jpeg_distort": {"jpeg_distort_fdct", "jpeg_idct_color", "jpeg_idct"},
    "resample": {"resample_stream", "resample_fused"},
    "resample3d": {"resample3d_pass"},
    "warp": {"warp_affine"},
    "cmn_chw": {"cmn_hwc2chw"},
    "cmn_hwc": {"cmn_generic"},
    "linear_transform": {"linear_transform"},
    "color_space": {"color_space_conversion"},
    "multiply_add": {"multiply_add"},
    "window_copy": {"window_copy"},
    "pad": {"pad"},
    "spectrogram_mel_two_kernels": {"spectrogram_stft_radix2", "mel_filter_bank"},
    "spectrogram_dft": {"spectrogram_dft"},
    "spectrogram_mel_fused": {"spectrogram_mel_fused"},
    "mel_tensor_cores": {"mel_filter_bank_mma"},
    "to_decibels_max": {"to_decibels_max", "to_decibels"},
    "mfcc": {"mfcc_dct"},
    "normalize": {"normalize"},
    "audio_resample": {"audio_resample"},
    "preemphasis": {"preemphasis_filter"},
    "nonsilent": {"nonsilent_mms", "nonsilent_region"},
    "audio_decode": {"flac_sync", "flac_frame", "flac_chain", "flac_decode", "audio_convert"},
    "arith": {"arith"},
    "permute": {"permute_tiled", "permute_rows", "permute_small", "permute_mixed"},
    "reduce_split": {"reduce_combine"},
    "equalize": {"equalize_hist", "equalize_apply"},
}
ANY_OF = {"permute"}                   # the path name depends on the planner's choice


def test_launch_count_trace_and_profile_records_agree(stub, tmp_path):
    trace = str(tmp_path / "trace.txt")
    env = dict(os.environ, DALIB200_DRYRUN="emul", LD_PRELOAD=stub, EMUL_STUB=stub, DALIB200_EMUL_TRACE=trace)
    r = subprocess.run([sys.executable, "-c", SCRIPT, ROOT], capture_output=True, text=True, timeout=1500, env=env, cwd=ROOT)
    assert r.returncode == 0 and "accounting-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
    results = {d["workload"]: d for d in map(json.loads, (line for line in r.stdout.splitlines() if line.startswith("{")))}
    assert sorted(results) == sorted(WANT), sorted(results)
    for name, d in results.items():
        names = d["records"]
        assert d["count"] == d["traced"] == len(names) > 0, (name, d["count"], d["traced"], len(names), names)
        assert all(names), (name, names)
        want = WANT[name]
        assert (want & set(names)) if name in ANY_OF else want <= set(names), (name, sorted(want - set(names)))
