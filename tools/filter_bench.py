"""Kernel times of fn.experimental.filter (csrc/filter.cu) on the GPU, driven through the C-ABI with torch device buffers, against
torch.nn.functional.conv2d on the same work and cv2.filter2D on 16 host threads.

Workloads (name: batch x sample shape, layout, type, filter):
  hwc_1080p_3x3 / 5x5 / 7x7 / 15x15   256 x 1080 x 1920 x 3, HWC, uint8
  hwc_224_3x3                         256 x 224 x 224 x 3, HWC, uint8
  fhwc_720p_3x3                       8 x 16 x 720 x 1280 x 3, FHWC, uint8 (8 sequences of 16 frames)
  f32_1080p_7x7                       64 x 1080 x 1920 x 3, HWC, float32

Each is launched `--iters` times after `--warmup` launches, the L2 cache flushed (a 256 MB buffer written) before every launch; the
kernel is timed with CUDA events around it (dalib200ProfilingEnable).  Algorithmic bytes: the input read once plus the output written
once; FMAs: one per tap and output element.  The bound reported is the larger of bytes / 3.35 TB/s and FMAs / 33.5 T/s (the H100 SXM
data sheet's 67 TFLOP/s FP32), and the kernel's share of it.  torch: conv2d in float32, grouped (one group per channel), the uint8 ->
float32 conversion, the reflect_101 padding, the rounding and the layout changes included, checked equal to the kernel's float32 output
within twice the gamma_k bound on one sample.  cv2: cv2.filter2D per image on 16 host threads (BORDER_REFLECT_101).  The card name and
power limit are read in the same run.  Prints one JSON object.

    python tools/filter_bench.py [--iters 20] [--warmup 3] [--only NAME,...] [--no-cv2]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12
FMA_PER_S = 67e12 / 2
WORKLOADS = {
    "hwc_1080p_3x3": (256, (1080, 1920, 3), "HWC", "uint8", 3),
    "hwc_1080p_5x5": (256, (1080, 1920, 3), "HWC", "uint8", 5),
    "hwc_1080p_7x7": (256, (1080, 1920, 3), "HWC", "uint8", 7),
    "hwc_1080p_15x15": (256, (1080, 1920, 3), "HWC", "uint8", 15),
    "hwc_224_3x3": (256, (224, 224, 3), "HWC", "uint8", 3),
    "fhwc_720p_3x3": (8, (16, 720, 1280, 3), "FHWC", "uint8", 3),
    "f32_1080p_7x7": (64, (1080, 1920, 3), "HWC", "float32", 7),
}
TYPE_CODE = {"uint8": 0, "float32": 9}


def torch_filter(x, w, layout, out_float=False):
    """x: (N, *sample) on the GPU, channel-last -> the same correlated with w (k x k) by a grouped float32 conv2d, reflect_101 borders"""
    import torch
    import torch.nn.functional as F
    c = x.shape[-1]
    k = w.shape[0]
    y = x.reshape((-1,) + tuple(x.shape[-3:])).permute(0, 3, 1, 2).to(torch.float32)
    y = F.pad(y, (k // 2, k - 1 - k // 2, k // 2, k - 1 - k // 2), mode="reflect")
    y = F.conv2d(y, w.expand(c, 1, k, k), groups=c)                 # conv2d is a correlation: the filter is not flipped
    if x.dtype == torch.uint8 and not out_float:
        y = torch.clamp(torch.floor(y + 0.5), 0, 255).to(torch.uint8)   # half away from zero for the non-negative range kept
    return y.permute(0, 2, 3, 1).reshape(x.shape).contiguous()


def cv2_batch(host, w, threads=16):
    import cv2
    from concurrent.futures import ThreadPoolExecutor
    cv2.setNumThreads(1)

    def one(img):
        return cv2.filter2D(img, -1, w, borderType=cv2.BORDER_REFLECT_101)
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(one, host[:threads]))                                # warm-up
        t0 = time.perf_counter()
        list(ex.map(one, host))
        return (time.perf_counter() - t0) * 1e3


def time_events(fn, iters, flush):
    import torch
    t = 0.0
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        t += a.elapsed_time(b) / iters
    return t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default="")
    ap.add_argument("--no-cv2", action="store_true")
    args = ap.parse_args()
    import torch
    import filter_ref as fr
    from dali_b200 import capi
    assert torch.cuda.is_available(), "filter_bench measures on the GPU; no GPU was found"
    lib = capi.lib()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {"device": smi.stdout.strip(), "iters": args.iters, "warmup": args.warmup, "workloads": {}}
    only = [s for s in args.only.split(",") if s]
    g = torch.Generator(device="cuda").manual_seed(0)
    rng = np.random.default_rng(0)
    stream = capi.stream_handle()
    for name, (n, shape, layout, dt, k) in WORKLOADS.items():
        if only and name not in only:
            continue
        if dt == "uint8":
            x = torch.randint(0, 256, (n,) + shape, dtype=torch.uint8, device="cuda", generator=g)
        else:
            x = torch.randn((n,) + shape, dtype=torch.float32, device="cuda", generator=g) * 100
        w = torch.from_numpy(rng.random((k, k)).astype(np.float32) / (k * k)).cuda()
        wh = w.cpu().numpy()
        out = torch.empty_like(x)
        out_f = torch.empty(x.shape, dtype=torch.float32, device="cuda")
        plan = C.c_void_p()
        capi.check(lib.dalib200FilterPlanCreate(C.byref(plan), n))
        nd = len(shape)
        shp = (C.c_int64 * (n * nd))(*(list(shape) * n))
        fshp = (C.c_int64 * (2 * n))(*([k, k] * n))
        oshp = (C.c_int64 * (n * nd))()
        ip = (C.c_void_p * n)(*[x[i].data_ptr() for i in range(n)])
        fp = (C.c_void_p * n)(*([w.data_ptr()] * n))

        def setup(out_type):
            capi.check(lib.dalib200FilterSetup(plan, TYPE_CODE[dt], out_type, n, nd, shp, layout.encode(), 9, 2, fshp, None, 0, 0, -1, None, oshp))

        def launch(o):
            capi.check(lib.dalib200FilterLaunch(plan, ip, fp, 1, None, 0, (C.c_void_p * n)(*[o[i].data_ptr() for i in range(n)]), stream))
        # the float32 output of sample 0 against the statement and against torch's float32 result, within the bound
        setup(9)
        launch(out_f)
        tf = torch_filter(x[:1], w, layout, out_float=True)
        torch.cuda.synchronize()
        x0 = x[0].cpu().numpy()
        lay0 = layout[1:] if layout[0] == "F" else layout
        fr0 = x0[0] if layout[0] == "F" else x0
        got0 = out_f[0].cpu().numpy()
        got0 = got0[0] if layout[0] == "F" else got0
        b = fr.bound(fr0, wh, lay0)[0]
        v = fr.correlate64(fr0, wh, lay0)[0]
        t0 = tf[0].cpu().numpy()
        t0 = t0[0] if layout[0] == "F" else t0
        assert np.all(np.abs(got0 - v) <= b), f"{name}: the kernel is outside the bound"
        assert np.all(np.abs(t0 - got0) <= 2 * b + 1e-30), f"{name}: torch and the kernel differ by more than twice the bound"
        setup(-1)
        for _ in range(args.warmup):
            launch(out)
        torch.cuda.synchronize()
        capi.profiling(True)
        capi.profiling_collect()
        for _ in range(args.iters):
            flush.zero_()
            launch(out)
        torch.cuda.synchronize()
        prof = capi.profiling_collect()
        capi.profiling(False)
        assert [p[0] for p in prof] == ["filter"] * args.iters, prof[:4]
        t_kernel = sum(ms for _, ms in prof) / args.iters
        for _ in range(args.warmup):
            torch_filter(x, w, layout)
        torch.cuda.synchronize()
        t_torch = time_events(lambda: torch_filter(x, w, layout), args.iters, flush)
        elems = x.numel()
        nbytes = 2 * elems * x.element_size()
        fmas = elems * k * k
        t_bytes, t_fma = nbytes / HBM_BYTES_PER_S * 1e3, fmas / FMA_PER_S * 1e3
        bound = "HBM" if t_bytes >= t_fma else "FP32 FMA"
        wres = {"algorithmic_bytes": nbytes, "fmas": fmas, "kernel_ms": round(t_kernel, 4), "GB_per_s": round(nbytes / t_kernel / 1e6, 1),
                "TFMA_per_s": round(fmas / t_kernel / 1e9, 2), "bound": bound, "bound_ms": round(max(t_bytes, t_fma), 4),
                "share_of_bound": round(max(t_bytes, t_fma) / t_kernel, 3), "torch_ms": round(t_torch, 4)}
        if not args.no_cv2 and dt == "uint8" and layout == "HWC":
            host = list(x.cpu().numpy())
            wres["cv2_16_threads_ms"] = round(cv2_batch(host, wh), 2)
        res["workloads"][name] = wres
        print(name, wres, file=sys.stderr, flush=True)
        lib.dalib200FilterPlanDestroy(plan)
        del x, out, out_f, tf
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
