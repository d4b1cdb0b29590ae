"""Timing of decoders.audio on the GPU (C-ABI, plan reused across steps):
    python tools/audio_decode_bench.py [--batch 64] [--steps 20] [--warmup 3] [--out DIR]
Batches of 10 s 16 kHz mono clips (8 distinct seeded clips, cycled), as FLAC (the encoder of tests/audio_streams.py: LPC order 8 and
FIXED order 2 subframes, Rice partitions of order 2, 4096-sample blocks) and as 16-bit WAV.  For each: ms per batch for
dalib200AudioLaunch (staging copy, upload and all kernels; CUDA events, the plan set up once), per-kernel ms from the library's own
per-launch events (a separate run), the decode plus the Jasper front-end (preemphasis -> spectrogram -> mel -> to_decibels -> normalize
-> pad) through a pipeline, end to end per batch, and the host-compiled kernel bodies (tools/emul/audio_decode_emul.cc, one CPU thread)
on the same batch as a reference point.  Prints the card's name and power limit with the numbers; the first step's outputs are checked
against the encoder's samples."""
import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

T = 160000


def clips(kind):
    import audio_streams as aus
    rng = np.random.default_rng(42)
    out = []
    for j in range(8):
        x = aus.signal(T, 1, 16, rng)
        if kind == "wav":
            out.append((aus.wav_pcm(x, 16, 16000), x))
            continue
        blocks = [4096] * (T // 4096) + [T % 4096]
        s = aus.flac(x, 16, 16000, blocks, spec=lambda k, c, b: {"kind": "lpc", "order": 8, "precision": 12, "porder": 2} if k % 2 else
                     {"kind": "fixed", "order": 2, "porder": 2})
        out.append((s, x))
    return out


def false_sync_flood(nbytes):
    """The costliest input for the frame search found so far: a mono 16-bit stream whose STREAMINFO allows 65535-sample blocks and whose
    audio region is nothing but 9-byte units of a valid frame header (65535 samples, CRC-8 right) and a VERBATIM subframe byte, so that
    every unit is a candidate and each candidate's parse reads 65535 samples (131 KB) of the units behind it before its CRC-16 fails."""
    import audio_streams as aus
    units = []
    for k in range(nbytes // 9):
        h = bytearray([0xFF, 0xF8, (7 << 4) | 5, 4 << 1]) + aus.utf8_number(k % 128) + (65534).to_bytes(2, "big")
        h.append(aus.crc8(h))
        units.append(bytes(h) + b"\x02")
    return b"fLaC" + aus.meta_block(0, aus.streaminfo(16, 65535, 16000, 1, 16, 1 << 24), True) + b"".join(units)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from dali_b200 import capi, fn, pipeline_def
    assert torch.cuda.is_available(), "needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    lib = capi.lib()
    res = {"card": card, "batch": a.batch, "clip": "10 s, 16 kHz, mono, 16-bit", "kinds": {}}
    print("card:", card)
    with tempfile.TemporaryDirectory() as tmp:
        emul_so = os.path.join(tmp, "emul.so")
        subprocess.check_call(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-ffp-contract=off", "-I/usr/local/cuda/include",
                               os.path.join(ROOT, "tools", "emul", "audio_decode_emul.cc"), "-o", emul_so])
        emul = C.CDLL(emul_so)
        emul.emul_audio_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        for kind in ("flac", "wav"):
            distinct = clips(kind)
            streams = [distinct[j % 8][0] for j in range(a.batch)]
            bufs = [np.frombuffer(s, np.uint8) for s in streams]
            n = a.batch
            ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
            lens = (C.c_size_t * n)(*[b.size for b in bufs])
            plan = capi.Plan("Audio", n)
            prm = (capi.AudioParams * n)(*[capi.AudioParams(0, 0.0, 50.0, capi.FLOAT)] * n)
            capi.check(lib.dalib200AudioPlanSetup(plan.handle, n, ptrs, lens, prm))
            outs = [torch.empty((T, 1), dtype=torch.float32, device="cuda") for _ in range(n)]
            rates = [torch.empty((), dtype=torch.float32, device="cuda") for _ in range(n)]
            st = capi.stream_handle()
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]

            def step():
                capi.check(lib.dalib200AudioLaunch(plan.handle, capi.ptr_array(outs), capi.ptr_array(rates), st))
            for k in range(a.warmup):
                step()
                torch.cuda.synchronize()
                if k == 0:
                    capi.check(lib.dalib200AudioStatusAsync(plan.handle, st))
                    torch.cuda.synchronize()
                    status = (C.c_int32 * n)()
                    capi.check(lib.dalib200AudioStatusFetch(plan.handle, status, n))
                    assert list(status) == [0] * n
                    for i in range(8):
                        want = distinct[i][1].astype(np.float32) * np.float32(2.0 ** -15)
                        assert np.array_equal(outs[i].cpu().numpy(), want), (kind, i)
            t = []
            for _ in range(a.steps):
                ev[0].record()
                step()
                ev[1].record()
                torch.cuda.synchronize()
                t.append(ev[0].elapsed_time(ev[1]))
            capi.profiling(True)
            capi.profiling_collect()
            for _ in range(a.steps):
                step()
            recs = capi.profiling_collect()
            capi.profiling(False)
            prof = {}
            for name, ms in recs:
                prof.setdefault(name, []).append(ms)
            prof = {k: float(np.median(v)) for k, v in prof.items()}
            # host-compiled kernel bodies, one thread, the same batch
            out = np.zeros((T, 1), np.float32)
            info = (C.c_int64 * 5)()
            t0 = time.perf_counter()
            for s in streams[:8]:
                emul.emul_audio_decode(s, len(s), 0, 9, out.ctypes.data, info)
            cpu_ms = (time.perf_counter() - t0) * 1e3 * n / 8

            # decode + Jasper chain through a pipeline, end to end
            @pipeline_def(batch_size=n, num_threads=1, device_id=0)
            def jasper():
                x, _ = fn.decoders.audio(fn.external_source(source=lambda i: bufs), downmix=True, sample_rate=16000)
                x = fn.preemphasis_filter(x)
                x = fn.spectrogram(x, nfft=512, window_length=320, window_step=160)
                x = fn.mel_filter_bank(x, sample_rate=16000.0, nfilter=64)
                x = fn.to_decibels(x, multiplier=math.log(10), reference=1.0, cutoff_db=math.log(1e-20))
                x = fn.normalize(x, axes=[1])
                return fn.pad(x, axes=[1], fill_value=0.0, align=16)
            p = jasper()
            p.build()
            for _ in range(a.warmup):
                p.run()
            torch.cuda.synchronize()
            tj = []
            for _ in range(a.steps):
                t0 = time.perf_counter()
                p.run()
                torch.cuda.synchronize()
                tj.append((time.perf_counter() - t0) * 1e3)
            r = {"ms_per_batch_launch": float(np.median(t)), "encoded_bytes": sum(len(s) for s in streams), "kernels_ms": prof,
                 "jasper_end_to_end_ms_per_batch": float(np.median(tj)), "host_compiled_core_one_thread_ms_per_batch": cpu_ms,
                 "samples_per_s_launch": n * T / (float(np.median(t)) * 1e-3)}
            res["kinds"][kind] = r
            print(kind, json.dumps(r))
        # the frame search's worst case: one crafted 256 KiB stream (the sample fails; the time is what it costs to find that out)
        flood = np.frombuffer(false_sync_flood(1 << 18), np.uint8)
        plan = capi.Plan("Audio", 1)
        ptrs = (C.c_void_p * 1)(flood.ctypes.data)
        lens = (C.c_size_t * 1)(flood.size)
        prm = (capi.AudioParams * 1)(capi.AudioParams(0, 0.0, 50.0, capi.FLOAT))
        capi.check(lib.dalib200AudioPlanSetup(plan.handle, 1, ptrs, lens, prm))
        out = torch.empty((1 << 24, 1), dtype=torch.float32, device="cuda")
        rate = torch.empty((), dtype=torch.float32, device="cuda")
        st = capi.stream_handle()
        tf = []
        for k in range(1 + min(a.steps, 3)):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            capi.check(lib.dalib200AudioLaunch(plan.handle, capi.ptr_array([out]), capi.ptr_array([rate]), st))
            ev[1].record()
            torch.cuda.synchronize()
            if k:
                tf.append(ev[0].elapsed_time(ev[1]))
        capi.check(lib.dalib200AudioStatusAsync(plan.handle, st))
        torch.cuda.synchronize()
        status = (C.c_int32 * 1)()
        capi.check(lib.dalib200AudioStatusFetch(plan.handle, status, 1))
        assert status[0] == 1
        res["false_sync_flood_256KiB"] = {"candidates": len(flood) // 9, "ms_per_launch": float(np.median(tf)), "status": int(status[0])}
        print("false-sync flood", json.dumps(res["false_sync_flood_256KiB"]))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "audio_decode_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
