"""Times dalib200ResampleLaunch alone on the shapes the streaming resize serves, so that a change tuned on the C2 shape is
checked on the others too.  One JSON line per case: mean launch time over --iters launches (CUDA events, L2 flushed before
each), algorithmic bytes (input + output) over that time, how many samples took the streaming kernel, and a checksum of the
outputs (equal checksums across two builds: same outputs).
  python tools/resample_stream_bench.py [--iters 30]          (DALIB200_LIB selects another build of the library)"""
import argparse
import hashlib
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from dali_b200 import capi  # noqa: E402

TRI = (capi.FILTER_LINEAR, 1, 0.0)   # linear with antialias = triangular on down-scales (the C2 default)
MAG = (capi.FILTER_LINEAR, 0, 0.0)
# name, batch, (H, W, C) in, (h, w) out, output dtype.  Every case must take the streaming kernel (vertical pass first, rows a
# multiple of 16 bytes): a 16:9 source shrunk to a square runs horizontal-first and a 500-pixel RGB row is not 16-byte aligned, so
# the non-C2 cases keep the source's aspect ratio and the ImageNet-sized one is 512 pixels wide.
CASES = [
    ("1080p->224", 256, (1080, 1920, 3), (224, 224), torch.uint8),
    ("720p->224x398", 256, (720, 1280, 3), (224, 398), torch.uint8),
    ("2160p->512x910", 64, (2160, 3840, 3), (512, 910), torch.uint8),
    ("512x384->224x168", 512, (384, 512, 3), (168, 224), torch.uint8),
    ("1080p->224 gray", 256, (1080, 1920, 1), (224, 224), torch.uint8),
    ("1080p->224 f32 out", 256, (1080, 1920, 3), (224, 224), torch.float32),
]


def run_case(name, n, shape, hw, odt, iters, flush):
    L = capi.lib()
    samples = (capi.ResampleSample * n)()
    for s in samples:
        s.in_h, s.in_w, s.channels = shape
        s.out_h, s.out_w = hw
        for d in range(2):
            s.use_roi[d] = 0
            s.min_filter[d] = capi.FilterDesc(*TRI)
            s.mag_filter[d] = capi.FilterDesc(*MAG)
    plan = capi.Plan("Resample", n)
    out_code = capi.UINT8 if odt == torch.uint8 else capi.FLOAT
    capi.check(L.dalib200ResamplePlanSetup(plan.handle, n, samples, capi.UINT8, out_code))
    g = torch.Generator(device="cuda").manual_seed(5)
    ins = [torch.randint(0, 256, shape, dtype=torch.uint8, device="cuda", generator=g) for _ in range(n)]
    outs = [torch.empty(hw + (shape[2],), dtype=odt, device="cuda") for _ in range(n)]
    pin, pout = capi.ptr_array(ins), capi.ptr_array(outs)
    stream = capi.stream_handle()
    for _ in range(3):
        capi.check(L.dalib200ResampleLaunch(plan.handle, pin, pout, stream))
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        flush.fill_(1)
        a.record()
        capi.check(L.dalib200ResampleLaunch(plan.handle, pin, pout, stream))
        b.record()
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]
    streamed = sum(L.dalib200ResamplePlanGetPath(plan.handle, i) for i in range(n))
    if streamed != n:
        raise SystemExit(f"{name}: {streamed} of {n} samples took the streaming kernel; this bench times that kernel only")
    nbytes = n * (shape[0] * shape[1] * shape[2] + hw[0] * hw[1] * shape[2] * (1 if odt == torch.uint8 else 4))
    h = hashlib.sha1()
    for o in outs:
        h.update(o.cpu().numpy().tobytes())
    mean = sum(ms) / len(ms)
    return {"case": name, "batch": n, "ms": round(mean, 4), "ms_min": round(min(ms), 4), "ms_max": round(max(ms), 4),
            "GB_per_s": round(nbytes / mean / 1e6, 1), "streamed": streamed, "sha1": h.hexdigest()[:16]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    args = ap.parse_args()
    assert args.iters >= 20, "average at least 20 launches"
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")   # larger than the 50 MB L2
    print(json.dumps({"gpu": torch.cuda.get_device_name(), "lib": os.environ.get("DALIB200_LIB", "in-tree")}))
    for c in CASES:
        print(json.dumps(run_case(*c, args.iters, flush)), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
