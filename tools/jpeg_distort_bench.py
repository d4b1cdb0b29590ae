"""Timing of fn.jpeg_compression_distortion on the GPU (C-ABI, inputs already in device memory):
    python tools/jpeg_distort_bench.py [--steps 20] [--warmup 3] [--out DIR]
Two batches: 256 x 224x224 and 64 x 1080p (seeded smooth images with noise, quality 75).  For each: device-resident ms per batch (CUDA
events around the launch, L2 flushed between steps outside the events), per-kernel ms from the library's own per-launch events
(dalib200ProfilingEnable, a separate run), the forward kernel's achieved bytes/s over its algorithmic bytes (3 B/px RGB read + int16
coefficients and DC written), and the CPU path it replaces -- cv2.imencode + cv2.imdecode -- over all usable cores.  Prints the card's name
and power limit with the numbers; a few outputs are checked against cv2 bit for bit."""
import argparse
import json
import multiprocessing as mp
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

QUALITY = 75


def _image(h, w, seed):
    import cv2
    rng = np.random.default_rng(seed)
    lo = rng.uniform(0, 255, (max(2, h // 32), max(2, w // 32), 3)).astype(np.float32)
    return np.clip(cv2.resize(lo, (w, h), interpolation=cv2.INTER_CUBIC) + rng.normal(0, 5, (h, w, 3)), 0, 255).astype(np.uint8)


def _cv2_roundtrip(img):
    import cv2
    ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, QUALITY])
    return cv2.imdecode(enc, cv2.IMREAD_COLOR)


def _cpu_worker(args):
    h, w, seeds = args
    import cv2
    cv2.setNumThreads(1)
    imgs = [_image(h, w, s) for s in seeds]
    t0 = time.perf_counter()
    for im in imgs:
        _cv2_roundtrip(im)
    return time.perf_counter() - t0


def usable_cores():
    try:
        n = len(os.sched_getaffinity(0))
    except AttributeError:
        n = os.cpu_count() or 1
    try:   # cgroup v2 quota
        q, p = open("/sys/fs/cgroup/cpu.max").read().split()
        if q != "max":
            n = min(n, max(1, int(int(q) / int(p))))
    except (OSError, ValueError):
        pass
    return n


def cpu_ms_per_batch(h, w, n):
    """the batch's encode + decode spread over the usable cores: the slowest worker's time over its share of the images"""
    cores = min(usable_cores(), n)
    chunks = [list(range(k, n, cores)) for k in range(cores)]
    with mp.get_context("spawn").Pool(cores) as pool:
        pool.map(_cpu_worker, [(h, w, c[:1]) for c in chunks])           # warm the workers
        return max(pool.map(_cpu_worker, [(h, w, c) for c in chunks])) * 1e3, cores


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    batches = [(256, 224, 224), (64, 1080, 1920)]
    cpu = {} if a.no_cpu else {b: cpu_ms_per_batch(b[1], b[2], b[0]) for b in batches}     # before this process touches the GPU
    print("cpu:", {f"{n} x {h}x{w}": v for (n, h, w), v in cpu.items()}, flush=True)
    import torch
    from dali_b200 import capi
    assert torch.cuda.is_available(), "needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card, "| torch:", torch.cuda.get_device_name(0), flush=True)
    lib = capi.lib()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    results = {"card": card, "quality": QUALITY, "batches": []}
    for n, h, w in batches:
        imgs = [_image(h, w, s) for s in range(n)]
        src = [torch.from_numpy(im).cuda() for im in imgs]
        dst = [torch.empty_like(s) for s in src]
        plan = capi.Plan("JpegDistort", n)
        ss = (capi.JpegDistortSample * n)()
        for s in ss:
            s.height, s.width, s.quality = h, w, QUALITY
        capi.check(lib.dalib200JpegDistortPlanSetup(plan.handle, n, ss))
        ip, op = capi.ptr_array(src), capi.ptr_array(dst)
        stream = capi.stream_handle()
        launch = lambda: capi.check(lib.dalib200JpegDistortLaunch(plan.handle, ip, op, stream))   # noqa: E731
        for _ in range(a.warmup):
            launch()
        torch.cuda.synchronize()
        for k in (0, n // 2, n - 1):      # parity of a few outputs (the tests cover the rest)
            assert np.array_equal(dst[k].cpu().numpy(), _cv2_roundtrip(np.ascontiguousarray(imgs[k][..., ::-1]))[..., ::-1]), k
        ms = []
        for _ in range(a.steps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            launch()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        capi.profiling(True)
        prof = {}
        for _ in range(a.steps):
            flush.zero_()
            torch.cuda.synchronize()
            launch()
            torch.cuda.synchronize()
            for name, t in capi.profiling_collect():
                prof.setdefault(name, []).append(t)
        capi.profiling(False)
        kern = {k: float(np.mean(v)) for k, v in prof.items()}
        mcux, mcuy = (w + 15) // 16, (h + 15) // 16
        blocks = mcux * mcuy * 6
        fdct_bytes = n * (h * w * 3 + blocks * 64 * 2 + blocks * 2)
        fdct_ms = kern.get("jpeg_distort_fdct", float("nan"))
        r = {"batch": f"{n} x {h}x{w}", "ms_per_batch_mean": float(np.mean(ms)), "ms_per_batch_median": float(np.median(ms)),
             "kernels_ms": kern, "fdct_algorithmic_bytes": fdct_bytes, "fdct_achieved_GBps": fdct_bytes / fdct_ms / 1e6}
        if (n, h, w) in cpu:
            r["cpu_cv2_ms_per_batch"], r["cpu_cores"] = cpu[(n, h, w)]
        print(json.dumps(r), flush=True)
        results["batches"].append(r)
        del src, dst, plan
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "jpeg_distort_bench.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
