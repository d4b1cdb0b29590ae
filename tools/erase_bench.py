"""Kernel times of fn.erase (csrc/erase.cu) on the GPU, driven through the C-ABI with torch device buffers, against torch's clone() plus
one slice assignment per region on the same work.

Workloads (name: batch x sample shape, layout, type, regions):
  hwc_1080p_u8          256 x 1080 x 1920 x 3, HWC, uint8, one region per image (timm RandomErasing: area 0.02-1/3, aspect 0.3-3.3)
  chw_224_f16           256 x 3 x 224 x 224, CHW, float16, one region per image (same distribution)
  specaugment_mel       64 x 128 x 1001, ft, float32, two frequency and ten time masks per clip (F <= 27, T <= 100)
  hwc_1080p_u8_64       workload 1 with 64 regions per image (each of the timm distribution)
  tiny_3000             3000 x (1-8) x (1-8) x 3, HWC, uint8, one region each

Each is launched `--iters` times after `--warmup` launches, the L2 cache flushed (a 256 MB buffer written) before every launch; the
kernel is timed with CUDA events around it (dalib200ProfilingEnable).  Algorithmic bytes: the input bytes outside the erased union
(counted from the planner's boxes) plus every output byte.  Reported beside them: GB/s, the share of 3.35 TB/s (the H100 SXM data
sheet's HBM3 bandwidth), torch's time (clone + slice assignments, every launch in the timed window) and the outputs checked equal.
The card name and power limit are read in the same run.  Prints one JSON object.

    python tools/erase_bench.py [--iters 50] [--warmup 5] [--only NAME,...]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12
TYPE_CODE = {"uint8": 0, "float16": 8, "float32": 9}


def timm(rng, h, w):
    while True:
        a = rng.uniform(0.02, 1 / 3) * h * w
        r = np.exp(rng.uniform(np.log(0.3), np.log(3.3)))
        eh, ew = int(round(np.sqrt(a * r))), int(round(np.sqrt(a / r)))
        if eh < h and ew < w:
            return [int(rng.integers(0, h - eh + 1)), int(rng.integers(0, w - ew + 1))], [eh, ew]


def workload(name, rng):
    """(batch shapes, layout, dtype, erased axes, per-sample anchors, per-sample shapes) with integer regions"""
    if name in ("hwc_1080p_u8", "hwc_1080p_u8_64"):
        k = 64 if name.endswith("64") else 1
        shapes = [(1080, 1920, 3)] * 256
        regs = [[timm(rng, 1080, 1920) for _ in range(k)] for _ in shapes]
        return shapes, "HWC", "uint8", [0, 1], regs
    if name == "chw_224_f16":
        shapes = [(3, 224, 224)] * 256
        return shapes, "CHW", "float16", [1, 2], [[timm(rng, 224, 224)] for _ in shapes]
    if name == "specaugment_mel":
        shapes = [(128, 1001)] * 64
        regs = []
        for _ in shapes:
            r = [([int(rng.integers(0, 128)), 0], [int(rng.integers(0, 28)), 1001]) for _ in range(2)]
            r += [([0, int(rng.integers(0, 1001))], [128, int(rng.integers(0, 101))]) for _ in range(10)]
            regs.append(r)
        return shapes, "ft", "float32", [0, 1], regs
    if name == "tiny_3000":
        shapes = [(int(rng.integers(1, 9)), int(rng.integers(1, 9)), 3) for _ in range(3000)]
        regs = [[([int(rng.integers(0, s[0])), int(rng.integers(0, s[1]))], [int(rng.integers(1, 4)), int(rng.integers(1, 4))])]
                for s in shapes]
        return shapes, "HWC", "uint8", [0, 1], regs
    raise KeyError(name)


def erased_elements(shape, axes, regs):
    """elements inside the union of the clipped boxes of one sample"""
    mask = np.zeros(tuple(shape[a] for a in axes), bool)
    for a, s in regs:
        mask[tuple(slice(max(lo, 0), min(lo + n, shape[ax])) for lo, n, ax in zip(a, s, axes))] = True
    rest = int(np.prod(shape)) // mask.size
    return int(mask.sum()) * rest


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    import torch
    from dali_b200 import capi
    assert torch.cuda.is_available(), "erase_bench measures on the GPU; no GPU was found"
    lib = capi.lib()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {"device": smi.stdout.strip(), "iters": args.iters, "warmup": args.warmup, "workloads": {}}
    only = [s for s in args.only.split(",") if s]
    stream = capi.stream_handle()
    names = ("hwc_1080p_u8", "chw_224_f16", "specaugment_mel", "hwc_1080p_u8_64", "tiny_3000")
    for name in names:
        if only and name not in only:
            continue
        rng = np.random.default_rng(0)
        shapes, layout, dt, axes, regs = workload(name, rng)
        n, nd = len(shapes), len(shapes[0])
        tdt = getattr(torch, dt)
        xs = [(torch.rand(s, device="cuda") * 200).to(tdt) for s in shapes]
        outs = [torch.empty_like(x) for x in xs]
        plan = C.c_void_p()
        capi.check(lib.dalib200ErasePlanCreate(C.byref(plan), n))
        av = [float(v) for r in regs for a, _ in r for v in a]
        sv = [float(v) for r in regs for _, s in r for v in s]
        cnt = (C.c_int64 * n)(*[len(r) * len(axes) for r in regs])
        capi.check(lib.dalib200EraseSetup(plan, TYPE_CODE[dt], n, nd, (C.c_int64 * (n * nd))(*[e for s in shapes for e in s]),
                                          layout.encode(), None, (C.c_int32 * len(axes))(*axes), len(axes), (C.c_float * len(av))(*av), cnt,
                                          (C.c_float * len(sv))(*sv), cnt, 0, 0, 0, (C.c_float * 1)(0.0), 1))
        ip = (C.c_void_p * n)(*[x.data_ptr() for x in xs])
        op = (C.c_void_p * n)(*[o.data_ptr() for o in outs])

        def launch():
            capi.check(lib.dalib200EraseLaunch(plan, ip, op, stream))

        def torch_erase():
            ys = []
            for x, r in zip(xs, regs):
                y = x.clone()
                for a, s in r:
                    idx = [slice(None)] * nd
                    for lo, k, ax in zip(a, s, axes):
                        idx[ax] = slice(max(lo, 0), lo + k)
                    y[tuple(idx)] = 0
                ys.append(y)
            return ys
        for _ in range(args.warmup):
            launch()
        ref = torch_erase()
        torch.cuda.synchronize()
        assert all(torch.equal(o, r) for o, r in zip(outs, ref)), f"{name}: the kernel and torch differ"
        capi.profiling(True)
        capi.profiling_collect()
        for _ in range(args.iters):
            flush.zero_()
            launch()
        torch.cuda.synchronize()
        prof = capi.profiling_collect()
        capi.profiling(False)
        assert [p[0] for p in prof] == ["erase"] * args.iters, prof[:4]
        t_kernel = sum(ms for _, ms in prof) / args.iters
        t_torch = 0.0
        for _ in range(args.iters):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            torch_erase()
            b.record()
            b.synchronize()
            t_torch += a.elapsed_time(b) / args.iters
        esz = xs[0].element_size()
        total = sum(int(np.prod(s)) for s in shapes)
        erased = sum(erased_elements(s, axes, r) for s, r in zip(shapes, regs))
        nbytes = (total - erased + total) * esz
        wres = {"samples": n, "algorithmic_bytes": nbytes, "erased_fraction": round(erased / total, 4), "kernel_ms": round(t_kernel, 4),
                "GB_per_s": round(nbytes / t_kernel / 1e6, 1), "share_of_3.35TB_s": round(nbytes / HBM_BYTES_PER_S * 1e3 / t_kernel, 3),
                "torch_ms": round(t_torch, 4), "speedup_vs_torch": round(t_torch / t_kernel, 2)}
        res["workloads"][name] = wres
        print(name, wres, file=sys.stderr, flush=True)
        lib.dalib200ErasePlanDestroy(plan)
        del xs, outs, ref
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
