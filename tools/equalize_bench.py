"""Kernel times of fn.experimental.equalize (csrc/equalize.cu) on the GPU, driven through the C-ABI with torch device buffers, against
torch on the same batch and cv2 on 16 host threads.

Workloads (name: batch x sample shape, layout):
  hwc_1080p     256 x 1080 x 1920 x 3, HWC, uniform random bytes
  hwc_224       256 x 224 x 224 x 3, HWC (where augmentation runs, after crop / resize)
  chw_224       256 x 3 x 224 x 224, CHW
  fhwc_720p     8 x 16 x 720 x 1280 x 3, FHWC
  hw_4k         32 x 2160 x 3840, HW
  flat_1080p    256 x 1080 x 1920 x 3, HWC, every image one value (every lane of the histogram hits the same bin)
  tiny_3000     3000 x 8 x 8 x 3, HWC

Each is launched `--iters` times after `--warmup` launches, the L2 cache flushed (a 256 MB buffer written) before every launch; each
kernel is timed with CUDA events around it (dalib200ProfilingEnable).  Algorithmic bytes: the input read twice (the histogram must be
complete before the first output byte) plus the output written once.  Share: those bytes at the H100 SXM data sheet's 3.35 TB/s over
the time of both kernels.  torch: a batched bincount over plane * 256 + value, cumsum, the formula and a gather, checked equal to
the kernels' output.  cv2: cv2.equalizeHist per channel on 16 host threads (hwc_1080p and hwc_224 only).  The card name and power
limit are read in the same run.  Prints one JSON object.

    python tools/equalize_bench.py [--iters 20] [--warmup 3] [--only NAME,...]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
WORKLOADS = {
    "hwc_1080p": (256, (1080, 1920, 3), "HWC"),
    "hwc_224": (256, (224, 224, 3), "HWC"),
    "chw_224": (256, (3, 224, 224), "CHW"),
    "fhwc_720p": (8, (16, 720, 1280, 3), "FHWC"),
    "hw_4k": (32, (2160, 3840), "HW"),
    "flat_1080p": (256, (1080, 1920, 3), "HWC"),
    "tiny_3000": (3000, (8, 8, 3), "HWC"),
}
CV2_WORKLOADS = ("hwc_1080p", "hwc_224")


def torch_equalize(x, layout):
    """x: (N, *sample) uint8 on the GPU -> the same equalized, by bincount / cumsum / formula / gather"""
    import torch
    lay = "N" + layout
    hw = [lay.index("H"), lay.index("W")]
    xp = torch.movedim(x, hw, [-2, -1])
    shp = xp.shape
    P, npx = xp.numel() // (shp[-2] * shp[-1]), shp[-2] * shp[-1]
    key = (torch.arange(P, device=x.device, dtype=torch.int64)[:, None] * 256 + xp.reshape(P, npx).to(torch.int64))
    h = torch.bincount(key.reshape(-1), minlength=P * 256).view(P, 256)
    first = torch.argmax((h > 0).to(torch.uint8), dim=1, keepdim=True)
    hfirst = torch.gather(h, 1, first)
    scale = torch.tensor(255.0, device=x.device) / (npx - hfirst).to(torch.float32)
    s = (torch.cumsum(h, 1) - hfirst).to(torch.float32)
    lut = torch.clamp(torch.round(s * scale), 0, 255).to(torch.uint8)
    k = torch.arange(256, device=x.device)[None, :]
    lut = torch.where(k <= first, torch.zeros_like(lut), lut)
    lut = torch.where(hfirst == npx, k.to(torch.uint8).expand(P, 256), lut)
    y = torch.take(lut.reshape(-1), key.reshape(-1)).view(shp)
    return torch.movedim(y, [-2, -1], hw).contiguous()


def cv2_batch(host, threads=16):
    import cv2
    from concurrent.futures import ThreadPoolExecutor
    cv2.setNumThreads(1)

    def one(img):
        return cv2.merge([cv2.equalizeHist(c) for c in cv2.split(img)])
    with ThreadPoolExecutor(threads) as ex:
        list(ex.map(one, host[:threads]))                                # warm-up
        t0 = time.perf_counter()
        list(ex.map(one, host))
        return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    import torch
    from dali_b200 import capi
    assert torch.cuda.is_available(), "equalize_bench measures on the GPU; no GPU was found"
    lib = capi.lib()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {"device": smi.stdout.strip(), "iters": args.iters, "warmup": args.warmup, "workloads": {}}
    only = [s for s in args.only.split(",") if s]
    g = torch.Generator(device="cuda").manual_seed(0)
    stream = capi.stream_handle()
    for name, (n, shape, layout) in WORKLOADS.items():
        if only and name not in only:
            continue
        if name.startswith("flat"):
            x = torch.randint(0, 256, (n,) + (1,) * len(shape), dtype=torch.uint8, device="cuda", generator=g).expand((n,) + shape).contiguous()
        else:
            x = torch.randint(0, 256, (n,) + shape, dtype=torch.uint8, device="cuda", generator=g)
        out = torch.empty_like(x)
        plan = C.c_void_p()
        capi.check(lib.dalib200EqualizePlanCreate(C.byref(plan), n))
        shp = (C.c_int64 * (n * len(shape)))(*(list(shape) * n))
        capi.check(lib.dalib200EqualizeSetup(plan, 0, n, len(shape), shp, layout.encode()))
        ip = (C.c_void_p * n)(*[x[i].data_ptr() for i in range(n)])
        op = (C.c_void_p * n)(*[out[i].data_ptr() for i in range(n)])
        launch = lambda: capi.check(lib.dalib200EqualizeLaunch(plan, ip, op, stream))
        launch()
        want = torch_equalize(x, layout)
        torch.cuda.synchronize()
        assert torch.equal(out, want), f"{name}: the kernels' output differs from torch's"
        for _ in range(args.warmup):
            launch()
        torch.cuda.synchronize()
        capi.profiling(True)
        capi.profiling_collect()
        for _ in range(args.iters):
            flush.zero_()
            launch()
        torch.cuda.synchronize()
        prof = capi.profiling_collect()
        capi.profiling(False)
        kern = {}
        for k, ms in prof:
            kern[k] = kern.get(k, 0.0) + ms / args.iters
        for _ in range(args.warmup):
            torch_equalize(x, layout)
        torch.cuda.synchronize()
        t_torch = 0.0
        for _ in range(args.iters):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            torch_equalize(x, layout)
            b.record()
            b.synchronize()
            t_torch += a.elapsed_time(b) / args.iters
        nbytes = 3 * x.numel()
        total = sum(kern.values())
        w = {"algorithmic_bytes": nbytes, "kernel_ms": {k: round(v, 4) for k, v in kern.items()}, "total_ms": round(total, 4),
             "GB_per_s": round(nbytes / total / 1e6, 1), "share_of_3.35TBps": round(nbytes / (total * 1e-3) / HBM_BYTES_PER_S, 3),
             "torch_ms": round(t_torch, 4)}
        if name in CV2_WORKLOADS:
            host = list(x.cpu().numpy())
            w["cv2_16_threads_ms"] = round(cv2_batch(host), 2)
        res["workloads"][name] = w
        lib.dalib200EqualizePlanDestroy(plan)
        del x, out, want
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
