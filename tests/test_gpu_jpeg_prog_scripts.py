"""GPU tests of progressive JPEG under the scan scripts of the catalogue in jpeg_extreme_streams (the CPU side of the same cases is
tests/test_jpeg_prog_scripts_cpu.py): mixed batches through the C ABI -- with baseline samples, incomplete prefixes, a reused plan and
outputs at unaligned byte offsets -- must leave in the coefficient arena exactly what expected() states, decode complete streams to
cv2.imdecode's pixels (RGB, GRAY, a region of interest), report status 1 exactly for the incomplete ones, and launch jpeg_prog_scan once
per wave of the batch."""
import ctypes as C

import numpy as np
import pytest

import gpu_helpers as gh
import jpeg_extreme_streams as xs
from dali_b200 import capi
from oracle import pyoracle as po
from test_jpeg_prog_scripts_cpu import LAYOUTS, SCRIPTS, _qtables, cases, encode, late_dqt, source

pytestmark = pytest.mark.gpu


def reference(s, ot):
    import cv2
    b = np.frombuffer(s, np.uint8)
    if ot == capi.GRAY:
        return cv2.imdecode(b, cv2.IMREAD_GRAYSCALE)[..., None]
    return cv2.imdecode(b, cv2.IMREAD_COLOR)[..., ::-1]


def decode(streams, ot, plan, rois=None, offsets=None):
    """(outputs, status, number of jpeg_prog_scan launches); the outputs in one sentinel-guarded allocation at `offsets` bytes"""
    lib, n = capi.lib(), len(streams)
    bufs = [np.frombuffer(s, np.uint8) for s in streams]
    prm = capi.JpegParams(ot, 1, capi.UINT8, 0)
    cr = None
    if rois is not None:
        cr = (capi.JpegRoi * n)()
        for i, r in enumerate(rois):
            if r is not None:
                cr[i].use_roi = 1
                cr[i].x0, cr[i].y0, cr[i].x1, cr[i].y1 = r
    capi.check(lib.dalib200JpegPlanSetupEx(plan.handle, n, (C.c_void_p * n)(*[b.ctypes.data for b in bufs]),
                                           (C.c_size_t * n)(*[b.size for b in bufs]), C.byref(prm), cr))
    shapes = []
    for i in range(n):
        hwc = (C.c_int32 * 3)()
        capi.check(lib.dalib200JpegPlanGetOutputShape(plan.handle, i, hwc))
        shapes.append(tuple(hwc))
    outs = gh.SentinelSlices([int(np.prod(s)) for s in shapes], 1, offsets)
    capi.profiling(True)
    try:
        capi.profiling_collect()
        capi.check(lib.dalib200JpegUpload(plan.handle, capi.stream_handle()))
        capi.check(lib.dalib200JpegLaunch(plan.handle, (C.c_void_p * n)(*outs.ptrs), capi.stream_handle()))
        got = outs.read()
        launches = sum(nm == "jpeg_prog_scan" for nm, _ in capi.profiling_collect())
    finally:
        capi.profiling(False)
    status = (C.c_int32 * n)()
    capi.check(lib.dalib200JpegGetStatus(plan.handle, status))
    return [g.reshape(s) for g, s in zip(got, shapes)], list(status), launches


def catalogue():
    """(stream, statement arena, waves, complete) of every case of the CPU catalogue, plus an incomplete prefix of every third"""
    out = []
    for k, (name, layout, h, w, quality, wide) in enumerate(cases()):
        src = source(layout, h, w, quality, 1000 + 37 * list(SCRIPTS).index(name) + LAYOUTS.index(layout))
        script = SCRIPTS[name](len(src["sampling"]))
        s = encode(src, h, w, script, wide)
        out.append((s, xs.expected(h, w, src["sampling"], src["planes"], script), xs.waves(script), True))
        if k % 3 == 0:
            cut = len(script) // 2 + 1
            out.append((xs.prefix(s, cut), xs.expected(h, w, src["sampling"], src["planes"], script, cut), xs.waves(script[:cut]),
                        xs.complete(script, len(src["sampling"]), cut)))
    return out


def run_batch(items, baseline, ot, plan, offsets=None, rois=None):
    """items: (stream, arena, waves, complete); baseline: plain baseline streams put between them"""
    streams, want = [], []
    for k, it in enumerate(items):
        streams.append(it[0])
        want.append(it)
        if k % 5 == 0 and baseline:
            streams.append(baseline[(k // 5) % len(baseline)])
            want.append(None)
    outs, status, launches = decode(streams, ot, plan, rois=rois, offsets=offsets)
    assert launches == max(it[2] for it in items), (launches, max(it[2] for it in items))
    for i, (s, o, st, it) in enumerate(zip(streams, outs, status, want)):
        complete = it is None or it[3]
        assert st == (0 if complete else 1), (i, st)
        if it is not None:
            got = gh.jpeg_coefs(plan, i, it[1].size).reshape(it[1].shape)
            assert np.array_equal(got, it[1]), ("coefficients", i, np.argwhere(got != it[1])[:4])
        if complete:
            ref = reference(s, ot)
            r = rois[i] if rois is not None else None
            if r is not None:
                ref = ref[r[1]:r[3], r[0]:r[2]]
            assert np.array_equal(o, ref), ("pixels", i, ot)
    return streams


@pytest.fixture(scope="module")
def items():
    return catalogue()


@pytest.fixture(scope="module")
def baseline():
    return [source(layout, h, w, 90, 77)["base"] for layout, h, w in [("420", 33, 47), ("444", 17, 23), ("gray", 24, 17)]]


@pytest.mark.parametrize("ot", [capi.RGB, capi.GRAY])
def test_catalogue_in_mixed_batches(items, baseline, ot):
    plan = capi.Plan("Jpeg", len(items) + len(items) // 5 + 2)
    run_batch(items, baseline, ot, plan, offsets=[(5 * k) % 16 for k in range(len(items) + len(items) // 5 + 2)])
    run_batch(items[::-1][:20], baseline, ot, plan)                                 # the plan again, a smaller batch


def test_region_of_interest(items):
    full = [it for it in items if it[3]][:24]
    rois = []
    for s, *_ in full:
        H, W = reference(s, capi.RGB).shape[:2]
        rois.append((W // 3, H // 4, max(W // 3 + 1, W - W // 5), max(H // 4 + 1, H - 1)))
    run_batch(full, [], capi.RGB, capi.Plan("Jpeg", len(full)), rois=rois)


def test_late_dqt_and_sequential_subset():
    items = []
    for layout in ("420", "ycck"):
        src, s, script = late_dqt(layout)
        items.append((s, xs.expected(33, 47, src["sampling"], src["planes"], script), xs.waves(script), True))
    for layout, h, w in [("420", 33, 47), ("cmyk", 29, 1)]:
        src = source(layout, h, w, 90, 5)
        script = xs.sequential_subset(len(src["sampling"]))
        s = encode(src, h, w, script, sof=0xC1 if src["dqt16"] else 0xC0)
        items.append((s, xs.expected(h, w, src["sampling"], src["planes"], script), xs.waves(script), True))
    for ot in (capi.RGB, capi.GRAY):
        run_batch(items, [], ot, capi.Plan("Jpeg", len(items)))


def test_large_images():
    """1080p 4:2:0 under three scripts other than libjpeg's, and the flat 2048 x 2048 image (EOB runs at their 32767 maximum)"""
    import cv2
    src = source("420", 1080, 1920, 75, 5)
    items = []
    for script in (xs.per_component_dc(3), xs.reordered(3), xs.restarts(3)):
        items.append((encode(src, 1080, 1920, script), xs.expected(1080, 1920, src["sampling"], src["planes"], script), xs.waves(script),
                      True))
    flat = cv2.imencode(".jpg", np.full((2048, 2048), 77, np.uint8), [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
    planes, script = po.jpeg_coeffs(flat)[:1], xs.simple(1)
    s = xs.progressive(2048, 2048, [(1, 1)], planes, [_qtables(flat)[0]], script=script)
    items.append((s, xs.expected(2048, 2048, [(1, 1)], planes, script), xs.waves(script), True))
    run_batch(items, [src["base"]], capi.RGB, capi.Plan("Jpeg", 6))
