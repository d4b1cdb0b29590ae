"""Timing of BMP / PNM decoding in decoders.image on the GPU (C-ABI, plan reused across steps):
    python tools/bitmap_bench.py [--batch 256] [--steps 10] [--warmup 2] [--out DIR]
Four batches of 1080p images made from bench.py's synth_image (8 distinct images, cycled): 24-bit BMP and P6 PPM (cv2-written), 8-bit
palette BMP (the green channel as palette indices) and RLE8 BMP (the image quantised to 16 levels, encoded as runs of each row).  For
each: ms per batch for upload + launch (CUDA events, the plan set up once), the upload alone and the launch alone, with the streams in
pageable memory (the upload packs them into the plan's pinned staging on the host, then copies it) and again in page-locked memory
declared stable (dalib200JpegPlanSetSourceStable: the upload is then the host-to-device DMA of each sample's pixel data alone, with
no host pack); per-kernel ms from the library's own per-launch events (dalib200ProfilingEnable, a separate run); bitmap_color's algorithmic bytes (raster or plane read plus
the RGB window written) over its time, also as a share of the H100 SXM data-sheet 3.35 TB/s; and for RLE8 the serial bitmap_unpack
lane alone, for the batch and for one image.  Prints the card's name and power limit with the numbers; every output of the first step
is checked against cv2 bit for bit."""
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

H, W = 1080, 1920
PEAK = 3.35e12


def rle8_rows(idx):
    """RLE8 data of an index image (top row last: BMP rows are bottom-up), runs split at 255, end-of-line per row, end-of-bitmap."""
    out = bytearray()
    for r in idx[::-1]:
        edges = np.flatnonzero(np.diff(r)) + 1
        starts = np.concatenate([[0], edges]); ends = np.concatenate([edges, [len(r)]])
        for s, e in zip(starts.tolist(), ends.tolist()):
            while e - s > 0:
                n = min(255, e - s)
                out += bytes([n, int(r[s])])
                s += n
        out += b"\0\0"
    return bytes(out[:-2]) + b"\0\1"


def make(kind, seed):
    import cv2
    import bench
    import bitmap_streams as bs
    img = bench.synth_image(H, W, seed)
    if kind == "bmp24":
        return cv2.imencode(".bmp", img)[1].tobytes()
    if kind == "ppm":
        return cv2.imencode(".ppm", img)[1].tobytes()
    pal = b"".join(bytes([v, 255 - v, v // 2, 0]) for v in range(256))
    if kind == "bmp8":
        return bs.bmp(W, H, 8, bs.rows(img[..., 1], 8), palette=pal)
    return bs.bmp(W, H, 8, rle8_rows(img[..., 1] >> 4), comp=1, palette=pal)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import cv2
    import torch
    from dali_b200 import capi
    assert torch.cuda.is_available(), "needs a GPU"
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    lib = capi.lib()
    res = {"card": card, "batch": a.batch, "size": f"{W}x{H}", "kinds": {}}
    print("card:", card)

    def run(streams, steps, check=False, profile=False, pinned=False):
        n = len(streams)
        bufs = [np.frombuffer(s, np.uint8) for s in streams]
        if pinned:
            arena = capi.pinned_empty(sum((b.size + 63) & ~63 for b in bufs) + 64)
            off, pb = 0, []
            for b in bufs:
                v = arena[off:off + b.size]
                v[:] = b
                pb.append(v)
                off += (b.size + 63) & ~63
            bufs = pb
        ptrs = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
        lens = (C.c_size_t * n)(*[b.size for b in bufs])
        plan = capi.Plan("Jpeg", n)
        prm = capi.JpegParams(capi.RGB, 1, capi.UINT8, 0)
        capi.check(lib.dalib200JpegPlanSetSourceStable(plan.handle, int(pinned)))
        capi.check(lib.dalib200JpegPlanSetupEx(plan.handle, n, ptrs, lens, C.byref(prm), None))
        outs = [torch.empty((H, W, 3), dtype=torch.uint8, device="cuda") for _ in range(n)]
        st = capi.stream_handle()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        t_all, t_up, t_launch = [], [], []
        direct = 0
        if profile:
            capi.profiling(True)
            capi.profiling_collect()
        for k in range(steps):
            ev[0].record()
            capi.check(lib.dalib200JpegUpload(plan.handle, st))
            ev[1].record()
            direct = int(lib.dalib200JpegPlanLastUploadDirect(plan.handle))
            capi.check(lib.dalib200JpegLaunch(plan.handle, capi.ptr_array(outs), st))
            ev[2].record()
            torch.cuda.synchronize()
            t_up.append(ev[0].elapsed_time(ev[1])); t_launch.append(ev[1].elapsed_time(ev[2])); t_all.append(ev[0].elapsed_time(ev[2]))
            if check and k == 0:
                status = (C.c_int32 * n)()
                capi.check(lib.dalib200JpegGetStatus(plan.handle, status))
                assert list(status) == [0] * n
                for i in range(min(n, 8)):
                    assert np.array_equal(outs[i].cpu().numpy(), cv2.imdecode(bufs[i], cv2.IMREAD_COLOR)[..., ::-1]), i
        prof = {}
        if profile:
            recs = capi.profiling_collect()
            capi.profiling(False)
            for name, ms in recs:
                prof.setdefault(name, []).append(ms)
            prof = {k: float(np.median(v)) for k, v in prof.items()}
        return float(np.median(t_all)), float(np.median(t_up)), float(np.median(t_launch)), prof, direct

    for kind in ("bmp24", "ppm", "bmp8", "rle8"):
        distinct = [make(kind, 100 + j) for j in range(8)]
        streams = [distinct[j % 8] for j in range(a.batch)]
        run(streams, a.warmup, check=True)
        t_all, t_up, t_launch = run(streams, a.steps)[:3]
        run(streams, a.warmup, check=True, pinned=True)
        p_all, p_up, p_launch, _, p_direct = run(streams, a.steps, pinned=True)
        prof = run(streams, a.warmup + a.steps, profile=True)[3]
        encoded = sum(len(s) for s in streams)
        read = a.batch * H * W * (1 if kind in ("bmp8", "rle8") else 3)        # raster (or RLE plane) bytes bitmap_color reads
        written = a.batch * H * W * 3
        r = {"ms_per_batch": t_all, "ms_upload_pack_and_h2d": t_up, "ms_launch": t_launch,
             "pinned_ms_per_batch": p_all, "pinned_ms_upload_h2d_only": p_up, "pinned_ms_launch": p_launch,
             "pinned_upload_path": p_direct,
             "encoded_bytes": encoded, "kernels_ms": prof}
        if "bitmap_color" in prof:
            bw = (read + written) / (prof["bitmap_color"] * 1e-3)
            r["bitmap_color_GBps"] = bw / 1e9
            r["bitmap_color_share_of_datasheet_3.35TBps"] = bw / PEAK
        if kind == "rle8":
            r["one_image_ms_unpack"] = run([distinct[0]], a.warmup + a.steps, profile=True)[3].get("bitmap_unpack")
        res["kinds"][kind] = r
        print(kind, json.dumps(r))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bitmap_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
