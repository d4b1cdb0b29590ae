"""Lossless JPEG decode on the GPU: batches of 256 1080p lossless images (grey and RGB; predictors 1 and 7; no restarts and a restart
every 8 lines) and each as a single image alone.  Prints per-kernel times (dalib200ProfilingEnable, a run of its own), upload + launch per
batch with the profiler off, algorithmic bytes per second (encoded bytes + 2 B per sample of differences written and read + output), and
cv2.imdecode over the host's cores on the same streams.  Needs a GPU; the streams are generated from a seed (tests/ljpeg_streams.py).

  python tools/ljpeg_bench.py [--batch 256] [--iters 5]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


_keep = []


def ctypes_addr(b):
    a = np.frombuffer(b, np.uint8)
    _keep.append(a)
    return a.ctypes.data


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    import cv2
    import torch
    from dali_b200 import capi
    import ljpeg_streams as ls
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    results = []
    for c in (1, 3):
        base = ls.image(1080, 1920, c, 8, 7, "smooth")
        for pred in (1, 7):
            for rst in (0, 8):
                s = ls.encode(base, pred=pred, restart=1920 * rst, tables="opt")
                for n in (a.batch, 1):
                    streams = [s] * n
                    plan = capi.Plan("Jpeg", n)
                    outs = [torch.empty((1080, 1920, 3), dtype=torch.uint8, device="cuda") for _ in range(n)]
                    ptrs = (C.c_void_p * n)(*[ctypes_addr(s) for s in streams])
                    lens = (C.c_size_t * n)(*[len(s) for s in streams])
                    optrs = capi.ptr_array(outs)

                    def run():
                        capi.check(capi.lib().dalib200JpegPlanSetup(plan.handle, n, ptrs, lens, capi.RGB, 1))
                        capi.check(capi.lib().dalib200JpegUpload(plan.handle, capi.stream_handle()))
                        capi.check(capi.lib().dalib200JpegLaunch(plan.handle, optrs, capi.stream_handle()))
                    run()
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    for _ in range(a.iters):
                        run()
                    torch.cuda.synchronize()
                    ms = (time.perf_counter() - t0) * 1e3 / a.iters
                    capi.profiling(True)
                    capi.profiling_collect()
                    run()
                    torch.cuda.synchronize()
                    prof = {}
                    for k, v in capi.profiling_collect():
                        prof[k] = prof.get(k, 0.0) + v
                    capi.profiling(False)
                    assert np.array_equal(outs[0].cpu().numpy(), np.repeat(base, 3, 2) if c == 1 else base)
                    nbytes = n * (len(s) + 4 * 1080 * 1920 * c + 1080 * 1920 * 3)
                    with ThreadPoolExecutor(os.cpu_count()) as ex:
                        t0 = time.perf_counter()
                        list(ex.map(lambda b: cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_UNCHANGED), streams))
                        cv_ms = (time.perf_counter() - t0) * 1e3
                    r = dict(comp=c, pred=pred, restart_lines=rst, batch=n, stream_bytes=len(s), ms_per_batch=round(ms, 3),
                             algo_GBps=round(nbytes / ms / 1e6, 2), kernels_ms={k: round(v, 3) for k, v in prof.items() if k.startswith("ljpeg") or k.startswith("jpeg_unstuff")},
                             cv2_ms=round(cv_ms, 2), cv2_threads=os.cpu_count())
                    results.append(r)
                    print(json.dumps(r), flush=True)
    print(json.dumps(dict(card=card, results=len(results))))


if __name__ == "__main__":
    main()
