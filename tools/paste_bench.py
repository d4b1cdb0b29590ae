"""Kernel times of fn.multi_paste and fn.paste (csrc/paste.cu) on the GPU, driven through the C-ABI with torch device buffers, against
torch's zeros (or full, for paste's canvas) plus one slice assignment per region on the same work.

Workloads (name: batch x output, regions):
  mosaic_u8          256 x 1280 x 1280 x 3 uint8 YOLO mosaics from 640^2 tiles: a random centre in [320, 960), four clipped tiles
  mosaic_u8_to_f16   the same, output FLOAT16 (a converting paste)
  copy_paste_32      256 x 640 x 640 x 3 uint8, 32 regions per output from random samples (the first the whole own image, then 31
                     rectangles of 32-256 pixels a side)
  zoom_out_ssd       paste of 256 x 300 x 300 x 3 uint8 at ratio 1-4, random placement, fill (123, 117, 104)
  tiny_3000          3000 x 8 x 8 x 3 uint8 outputs, two regions each from 1-8 x 1-8 inputs

Each is launched `--iters` times after `--warmup` launches, the L2 cache flushed (a 256 MB buffer written) before every launch; the
kernel is timed with CUDA events around it (dalib200ProfilingEnable).  Algorithmic bytes: the visible source bytes read (each output
pixel some region covers, once) plus every output byte.  Reported beside them: GB/s, the share of 3.35 TB/s (the H100 SXM data sheet's
HBM3 bandwidth), torch's time (every launch in the timed window) and whether the outputs are equal.  The card name and power limit
are read in the same run.  Prints one JSON object.

    python tools/paste_bench.py [--iters 50] [--warmup 5] [--only NAME,...]
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

HBM_BYTES_PER_S = 3.35e12
P64 = C.POINTER(C.c_int64)


def mosaic(rng, n, tile=640):
    regs = []
    for _ in range(n):
        yc, xc = int(rng.integers(tile // 2, 3 * tile // 2)), int(rng.integers(tile // 2, 3 * tile // 2))
        ids = [int(v) for v in rng.integers(0, n, 4)]
        s = 2 * tile
        q = [(min(yc, tile), min(xc, tile)), (min(yc, tile), min(s - xc, tile)), (min(s - yc, tile), min(xc, tile)),
             (min(s - yc, tile), min(s - xc, tile))]
        oa = [(yc - q[0][0], xc - q[0][1]), (yc - q[1][0], xc), (yc, xc - q[2][1]), (yc, xc)]
        ia = [(tile - q[0][0], tile - q[0][1]), (tile - q[1][0], 0), (0, tile - q[2][1]), (0, 0)]
        regs.append([(j, a, h, o) for j, a, h, o in zip(ids, ia, q, oa)])
    return regs


def copy_paste(rng, n, size=640, k=32):
    regs = []
    for i in range(n):
        r = [(i, (0, 0), (size, size), (0, 0))]
        for _ in range(k - 1):
            h, w = int(rng.integers(32, 257)), int(rng.integers(32, 257))
            r.append((int(rng.integers(0, n)), (int(rng.integers(0, size - h + 1)), int(rng.integers(0, size - w + 1))), (h, w),
                      (int(rng.integers(0, size - h + 1)), int(rng.integers(0, size - w + 1)))))
        regs.append(r)
    return regs


def workload(name, rng):
    """(source shapes, output (H, W), per-output regions (src, in anchor, shape, out anchor), output dtype)"""
    if name in ("mosaic_u8", "mosaic_u8_to_f16"):
        return [(640, 640, 3)] * 256, [(1280, 1280)] * 256, mosaic(rng, 256), "uint8" if name == "mosaic_u8" else "float16"
    if name == "copy_paste_32":
        return [(640, 640, 3)] * 256, [(640, 640)] * 256, copy_paste(rng, 256), "uint8"
    if name == "tiny_3000":
        shapes = [(int(rng.integers(1, 9)), int(rng.integers(1, 9)), 3) for _ in range(3000)]
        regs = []
        for _ in shapes:
            r = []
            for _ in range(2):
                j = int(rng.integers(0, 3000))
                h, w = int(rng.integers(1, shapes[j][0] + 1)), int(rng.integers(1, shapes[j][1] + 1))
                r.append((j, (int(rng.integers(0, shapes[j][0] - h + 1)), int(rng.integers(0, shapes[j][1] - w + 1))), (h, w),
                          (int(rng.integers(0, 8 - h + 1)), int(rng.integers(0, 8 - w + 1)))))
            regs.append(r)
        return shapes, [(8, 8)] * 3000, regs, "uint8"
    raise KeyError(name)


def covered(out_hw, regs):
    m = np.zeros(out_hw, bool)
    for _, _, (h, w), (oy, ox) in regs:
        m[oy:oy + h, ox:ox + w] = True
    return int(m.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--only", default="")
    args = ap.parse_args()
    import torch
    from dali_b200 import capi
    assert torch.cuda.is_available(), "paste_bench measures on the GPU; no GPU was found"
    lib = capi.lib()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    res = {"device": smi.stdout.strip(), "iters": args.iters, "warmup": args.warmup, "workloads": {}}
    only = [s for s in args.only.split(",") if s]
    stream = capi.stream_handle()
    for name in ("mosaic_u8", "mosaic_u8_to_f16", "copy_paste_32", "zoom_out_ssd", "tiny_3000"):
        if only and name not in only:
            continue
        rng = np.random.default_rng(0)
        plan = C.c_void_p()
        if name == "zoom_out_ssd":
            n = 256
            shapes = [(300, 300, 3)] * n
            xs = [torch.randint(0, 256, s, dtype=torch.uint8, device="cuda") for s in shapes]
            ratio = rng.uniform(1.0, 4.0, n).astype(np.float32)
            px, py = rng.uniform(0, 1, n).astype(np.float32), rng.uniform(0, 1, n).astype(np.float32)
            fill = (123.0, 117.0, 104.0)
            capi.check(lib.dalib200PastePlanCreate(C.byref(plan), n))
            oshapes = (C.c_int64 * (3 * n))()
            f = lambda v: (C.c_float * n)(*[float(x) for x in v])  # noqa: E731
            capi.check(lib.dalib200PasteCanvasSetup(plan, 0, n, 3, b"HWC", (C.c_int64 * (3 * n))(*[e for s in shapes for e in s]), 3, f(ratio),
                                                    f(px), f(py), f([0.0] * n), (C.c_float * 3)(*fill), 3, oshapes))
            outs_hw = [(oshapes[3 * i], oshapes[3 * i + 1]) for i in range(n)]
            regs = []
            for i in range(n):
                ho, wo = outs_hw[i]
                regs.append([(i, (0, 0), (300, 300), (int(np.float32(py[i]) * np.float32(ho - 300)), int(np.float32(px[i]) * np.float32(wo - 300))))])
            odt = torch.uint8
            fillt = torch.tensor(fill, device="cuda").to(torch.uint8)
        else:
            shapes, outs_hw, regs, odt_name = workload(name, rng)
            n = len(outs_hw)
            xs = [torch.randint(0, 256, s, dtype=torch.uint8, device="cuda") for s in shapes]
            odt = getattr(torch, odt_name)
            fillt = None
            capi.check(lib.dalib200PastePlanCreate(C.byref(plan), n))
            ids = [r[0] for rr in regs for r in rr]
            vals = {a: np.array([v for rr in regs for r in rr for v in r[k]] + [0], np.float64)
                    for a, k in (("in_anchors", 1), ("shapes", 2), ("out_anchors", 3))}
            cnt = np.array([2 * len(rr) for rr in regs], np.int64)
            av, ac = (C.POINTER(C.c_double) * 6)(), (P64 * 6)()
            for a, k in (("in_anchors", 0), ("shapes", 2), ("out_anchors", 4)):
                av[k], ac[k] = vals[a].ctypes.data_as(C.POINTER(C.c_double)), cnt.ctypes.data_as(P64)
            oshapes = (C.c_int64 * (3 * n))()
            capi.check(lib.dalib200PasteSetup(plan, 0, 0 if odt == torch.uint8 else 8, 1, n, (C.c_int * 1)(3), None,
                                              (C.c_int64 * (3 * n))(*[e for s in shapes for e in s]), (C.c_int32 * len(ids))(*ids),
                                              (C.c_int64 * n)(*[len(rr) for rr in regs]), av, ac,
                                              (C.c_int64 * (2 * n))(*[v for hw in outs_hw for v in hw]), (C.c_float * 1)(0.0), 1, oshapes))
        outs = [torch.empty(hw + (3,), dtype=odt, device="cuda") for hw in outs_hw]
        ip = (C.c_void_p * len(xs))(*[x.data_ptr() for x in xs])
        op = (C.c_void_p * n)(*[o.data_ptr() for o in outs])

        def launch():
            capi.check(lib.dalib200PasteLaunch(plan, ip, op, stream))

        def torch_paste():
            ys = []
            for hw, rr in zip(outs_hw, regs):
                y = torch.zeros(hw + (3,), dtype=odt, device="cuda") if fillt is None else fillt.expand(hw + (3,)).contiguous()
                for j, (iy, ix), (h, w), (oy, ox) in rr:
                    y[oy:oy + h, ox:ox + w] = xs[j][iy:iy + h, ix:ix + w]
                ys.append(y)
            return ys
        for _ in range(args.warmup):
            launch()
        ref = torch_paste()
        torch.cuda.synchronize()
        equal = all(torch.equal(o, r) for o, r in zip(outs, ref))
        capi.profiling(True)
        capi.profiling_collect()
        for _ in range(args.iters):
            flush.zero_()
            launch()
        torch.cuda.synchronize()
        prof = capi.profiling_collect()
        capi.profiling(False)
        assert [p[0] for p in prof] == ["paste"] * args.iters, prof[:4]
        t_kernel = sum(ms for _, ms in prof) / args.iters
        t_torch = 0.0
        for _ in range(args.iters):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            torch_paste()
            b.record()
            b.synchronize()
            t_torch += a.elapsed_time(b) / args.iters
        osz = outs[0].element_size()
        out_bytes = sum(hw[0] * hw[1] * 3 for hw in outs_hw) * osz
        read_bytes = sum(covered(hw, rr) for hw, rr in zip(outs_hw, regs)) * 3
        nbytes = out_bytes + read_bytes
        wres = {"outputs": n, "algorithmic_bytes": nbytes, "kernel_ms": round(t_kernel, 4), "GB_per_s": round(nbytes / t_kernel / 1e6, 1),
                "share_of_3.35TB_s": round(nbytes / HBM_BYTES_PER_S * 1e3 / t_kernel, 3), "torch_ms": round(t_torch, 4),
                "speedup_vs_torch": round(t_torch / t_kernel, 2), "equal": bool(equal)}
        res["workloads"][name] = wres
        print(name, wres, file=sys.stderr, flush=True)
        lib.dalib200PastePlanDestroy(plan)
        del xs, outs, ref
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
