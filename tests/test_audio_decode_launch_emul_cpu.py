"""The launch path of decoders.audio, executed WITHOUT a GPU: tools/emul/cuda_emul_stub.cc is preloaded in place of the CUDA runtime,
"device" memory is host memory, and the kernels of audio_decode.cu run on the host through the same bodies the device runs
(audio_decode_core.h), every pass in reverse thread order.  Through the library's own C-ABI: mixed WAV / FLAC batches (the batch-wide
index searches, the scratch layout, the descriptor upload), plan reuse with growing lengths, corrupt samples among good ones, a failed
set-up, and downmix + resampling (the resampler's launch is recorded by the stub: its inputs, lengths and channels are checked)."""
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
import ctypes as C, math, os, sys
import numpy as np
sys.path.insert(0, %(root)r); sys.path.insert(0, os.path.join(%(root)r, "tests"))
import conftest                      # DALIB200_DRYRUN=emul
from dali_b200 import capi
import audio_streams as aus
from test_audio_decode_cpu import FLOAT, INT16, INT32, expected

stub = C.CDLL(os.environ["EMUL_STUB"]); stub.emul_launch_count.restype = C.c_long
stub.emul_resample_sample.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
counts = lambda: [stub.emul_launch_count(k) for k in range(27)]
lib = capi.lib()
NP = {FLOAT: np.float32, INT16: np.int16, INT32: np.int32}

def decode(plan, streams, downmix=False, rate=0.0, dtype=FLOAT):
    n = len(streams)
    bufs = [np.frombuffer(s, np.uint8) for s in streams]
    ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    lens = (C.c_size_t * n)(*[b.size for b in bufs])
    prm = (capi.AudioParams * n)(*[capi.AudioParams(int(downmix), rate, 50.0, dtype)] * n)
    capi.check(lib.dalib200AudioPlanSetup(plan.handle, n, ptrs, lens, prm))
    outs, rates = [], []
    for i in range(n):
        sh, nd, r = (C.c_int64 * 2)(), C.c_int32(), C.c_float()
        capi.check(lib.dalib200AudioPlanGetOutputShape(plan.handle, i, sh, C.byref(nd), C.byref(r)))
        outs.append(np.full((sh[0], sh[1]) if nd.value == 2 else (sh[0],), 7, NP[dtype]))
        rates.append(np.zeros(1, np.float32))
    capi.check(lib.dalib200AudioLaunch(plan.handle, capi.ptr_array([o.ctypes.data for o in outs]),
                                       capi.ptr_array([r.ctypes.data for r in rates]), None))
    capi.check(lib.dalib200AudioStatusAsync(plan.handle, None))
    st = (C.c_int32 * n)()
    capi.check(lib.dalib200AudioStatusFetch(plan.handle, st, n))
    return outs, [float(r[0]) for r in rates], list(st)

corpus = [c for c in aus.corpus() if len(c[1]) < 40000]
# mixed WAV / FLAC batches, several samples per batch, in FLOAT / INT16 / INT32 and downmixed
plan = capi.Plan("Audio", 8)
for dtype in (FLOAT, INT16, INT32):
    items = [c for c in corpus if not (dtype != FLOAT and c[2].dtype == np.float32)]
    for b in range(0, len(items), 7):
        batch = items[b:b + 7]
        c0 = counts()
        outs, rates, st = decode(plan, [s for _, s, _, _ in batch], dtype=dtype)
        c1 = counts()
        assert st == [0] * len(batch), (dtype, b, st)
        for (name, s, x, bits), o in zip(batch, outs):
            w = expected(x, bits, dtype)
            assert o.dtype == w.dtype and np.array_equal(o.view(np.uint8), w.view(np.uint8)), (name, dtype)
        has_flac = any(n.startswith("flac") for n, _, _, _ in batch)
        assert (c1[21] > c0[21]) == has_flac and (c1[24] > c0[24]) == has_flac and c1[25] == c0[25] + 1, (c0, c1)
outs, rates, st = decode(plan, [s for _, s, _, _ in corpus[:8]], downmix=True)
assert st == [0] * 8
for (name, s, x, bits), o in zip(corpus[:8], outs):
    assert np.array_equal(o.view(np.uint32), expected(x, bits, FLOAT, downmix=True)[:, 0].view(np.uint32)), name
# plan reuse with growing lengths (the scratch, the staging arena and the descriptors grow; the old batch's sizes must not leak)
plan = capi.Plan("Audio", 3)
rng = np.random.default_rng(4)
for T in (300, 2500, 17000, 60001):
    xs = [aus.signal(T, 2, 16, rng), aus.signal(T, 1, 24, rng), aus.signal(T + 5, 3, 16, rng)]
    ss = [aus.flac(xs[0], 16, 44100, [4096] * (T // 4096) + ([T %% 4096] if T %% 4096 else []), assign=lambda k: 10),
          aus.wav_pcm(xs[1], 24, 16000),
          aus.flac(xs[2], 16, 8000, [1152] * ((T + 5) // 1152) + ([(T + 5) %% 1152] if (T + 5) %% 1152 else []))]
    outs, rates, st = decode(plan, ss, dtype=INT32)
    assert st == [0, 0, 0] and rates == [44100.0, 16000.0, 8000.0], (T, st, rates)
    for x, bits, o in zip(xs, (16, 24, 16), outs):
        assert np.array_equal(o, expected(x, bits, INT32)), T
# corrupt samples set only their own status
good = corpus[0]
for name, bad in aus.corrupt():
    outs, rates, st = decode(plan, [good[1], bad, good[1]])
    assert st == [0, 1, 0], (name, st)
    assert np.array_equal(outs[0], expected(good[2], good[3])) and np.array_equal(outs[2], outs[0]), name
# a set-up that fails leaves nothing to launch behind it
bufs = [np.frombuffer(good[1], np.uint8), np.frombuffer(aus.refused()[0][1], np.uint8)]
ptrs = (C.c_void_p * 2)(*[b.ctypes.data for b in bufs]); lens = (C.c_size_t * 2)(*[b.size for b in bufs])
prm = (capi.AudioParams * 2)(*[capi.AudioParams(0, 0.0, 50.0, FLOAT)] * 2)
assert lib.dalib200AudioPlanSetup(plan.handle, 2, ptrs, lens, prm) == aus.UNSUPPORTED
assert b"sample 1" in lib.dalib200GetLastError()
c0 = counts()
capi.check(lib.dalib200AudioLaunch(plan.handle, None, None, None))
assert counts() == c0
# downmix + resampling: the resampler gets the downmixed signal of each sample whose rate differs, at the AudioResample lengths
xs = [(aus.signal(5000, 2, 16, rng), 44100), (aus.signal(3000, 1, 16, rng), 16000), (aus.signal(4410, 3, 8, rng), 22050),
      (aus.signal(2000, 2, 24, rng), 8000)]
ss = [aus.flac(x, 16, r, [1000] * 5, assign=lambda k: 9) if k == 0 else aus.wav_pcm(x, 16, r) if k == 1 else
      aus.flac(x, 8, r, [576] * 7 + [4410 - 7 * 576]) if k == 2 else aus.wav_pcm(x, 24, r) for k, (x, r) in enumerate(xs)]
plan = capi.Plan("Audio", 4)
c0 = counts()
outs, rates, st = decode(plan, ss, downmix=True, rate=16000.0)
c1 = counts()
assert st == [0] * 4 and rates == [16000.0] * 4 and c1[26] == c0[26] + 1
assert stub.emul_resample_count() == 3
k = 0
for i, ((x, r), bits) in enumerate(zip(xs, (16, 16, 8, 24))):
    want = expected(x, bits, FLOAT, downmix=True)[:, 0]
    n_out = math.ceil(len(x) * 16000.0 / r)
    assert outs[i].shape == (n_out,), (i, outs[i].shape)
    if r == 16000:
        assert np.array_equal(outs[i].view(np.uint32), want.view(np.uint32))
        continue
    info = (C.c_int64 * 3)()
    got = np.zeros(len(x), np.float32)
    stub.emul_resample_sample(k, info, got.ctypes.data)
    assert tuple(info) == (len(x), n_out, 1) and np.array_equal(got.view(np.uint32), want.view(np.uint32)), (i, tuple(info))
    k += 1
print("audio-emul-ok")
"""


def test_audio_decode_launch_path(emul_env):
    r = subprocess.run([sys.executable, "-c", SCRIPT % dict(root=ROOT)], capture_output=True, text=True, timeout=1500, env=emul_env, cwd=ROOT)
    assert r.returncode == 0 and "audio-emul-ok" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
