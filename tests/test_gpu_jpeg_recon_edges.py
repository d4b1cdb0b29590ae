"""The JPEG reconstruct kernels on the H100 at the edges of their own geometry, against cv2.imdecode (libjpeg-turbo: islow IDCT, fancy
upsampling), bit for bit, and with every output in one sentinel-filled allocation so that a write outside a sample is seen:
  * idct_color_420 (4:2:0 fancy -> RGB / BGR): every width residue mod 16 and so every column of the copied last chroma column,
    the (width + 1) / 2 > 2 threshold, strips of one MCU and strips whose right halo is the last MCU column, heights 1-33, the
    segment splits of 24-band segments (checked against a copy of fused_geo), windows whose top, bottom, left and right edges sit on
    segment, carry-row, MCU and strip boundaries, with and without the post pass, and restart intervals;
  * color_fast_kernel (4:4:4, 4:2:2 and the other layouts it takes): rows of one, two and three 1024-pixel items, windows that start
    around the first item boundary, and a batch in which 4:2:0 images (which own no items) sit between its images;
  * color_kernel (4:1:1, gray): widths of every residue mod 4 around 1024 with odd heights;
  * output placement: one mixed batch (every path, progressive, window, EXIF orientation, YCbCr and float output) at every byte
    offset and packed, each sample equal to its own decode into an aligned buffer;
  * fn.jpeg_compression_distortion, which reuses these kernels, over the same widths.
Each case names the kernel it is written for and asserts that the kernel ran."""
import ctypes as C
import functools
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gpu_helpers as gh  # noqa: E402
import jpeg_distort_cases as jc  # noqa: E402
from dali_b200 import capi  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUSED, FAST, GENERIC, POST = "jpeg_idct_color", "jpeg_upsample_color", "jpeg_upsample_color_generic", "jpeg_post"
OT = {capi.RGB: "RGB", capi.BGR: "BGR", capi.GRAY: "GRAY", capi.YCbCr: "YCbCr"}


def _constant(path, name):
    with open(os.path.join(ROOT, "dali_b200", "csrc", path)) as f:
        return int(re.search(rf"constexpr int {name} = (\d+);", f.read()).group(1))


# read from the sources, so that the geometry below follows a change of the constants and the asserted splits notice it
FUSED_MCUS, FUSED_MAX_BANDS = _constant("jpeg_recon.h", "kFusedMcus"), _constant("jpeg_recon.h", "kFusedMaxBands")
COLOR_SEG = _constant("jpeg.cu", "kColorSeg")


# ------------------------------------------------------------------------------------------------------------------
# geometry: the decode window of PlanGeometry (jpeg.cu) and fused_geo (jpeg_recon.h)
def window(W, H, roi=None):
    """(win_x0, win_w, win_y0, win_h, direct) of a 3-component sample without orientation, u8 RGB / BGR: the window is widened to
    whole 8-pixel columns, and unless that is the region itself the kernels write plan scratch and the post pass crops it"""
    x0, y0, x1, y1 = roi or (0, 0, W, H)
    wx0 = x0 & ~7
    ww = min(W, (x1 + 7) & ~7) - wx0
    return wx0, ww, y0, y1 - y0, wx0 == x0 and wx0 + ww == x1


def fused_geo(W, H, roi=None):
    """fused_geo of a 4:2:0 image's window: MCU columns [mx0, mx_end), strips, and the segments [b_lo, b_hi) of bands it walks"""
    wx0, ww, wy0, wh, _ = window(W, H, roi)
    last = -(-H // 16) - 1
    mx0, mx_end = wx0 >> 4, ((wx0 + ww - 1) >> 4) + 1
    m0 = min((wy0 + 1) >> 4, last)
    nbands = min((wy0 + wh) >> 4, last) - m0 + 1
    nseg = -(-nbands // FUSED_MAX_BANDS)
    seg_len = -(-nbands // nseg)
    segs = [(b, min(m0 + nbands, b + seg_len)) for b in range(m0, m0 + nbands, seg_len)]
    strips = [(mx, min(mx_end, mx + FUSED_MCUS)) for mx in range(mx0, mx_end, FUSED_MCUS)]
    return {"mcux": -(-W // 16), "segs": segs, "strips": strips}


def chroma_edge(W):
    """column of the image's last chroma column inside the last MCU column's chroma block (`edge` of idct_color_420)"""
    return (W + 1) // 2 - 1 - 8 * (-(-W // 16) - 1)


def test_geometry_copy_reaches_the_cases_below():
    """the sizes of the cases below reach what they are written for; runs without a GPU as well"""
    assert sorted(chroma_edge(w) for w in range(5, 37)) == sorted(list(range(8)) * 4)
    assert sorted(w % 16 for w in range(5, 37)) == sorted(list(range(16)) * 2)
    for w in (257, 513):                                               # a last strip of one MCU column
        s = fused_geo(w, 24)["strips"]
        assert s[-1][1] - s[-1][0] == 1, w
    g = fused_geo(264, 24)                                             # the right halo of a full strip is the last MCU column
    assert g["strips"][0][1] == g["mcux"] - 1
    splits = {h: [b - a for a, b in fused_geo(264, h)["segs"]] for h in (384, 385, 401, 768, 769, 1153)}
    assert splits == {384: [24], 385: [13, 12], 401: [13, 13], 768: [24, 24], 769: [17, 17, 15], 1153: [19, 19, 19, 16]}, splits
    assert [len(fused_geo(40, h)["segs"]) for h in (1, 16, 17, 33)] == [1, 1, 1, 1]
    assert fused_geo(40, 16)["segs"] == [(0, 1)]                       # mcuy = 1: the only band is also the last
    # windows of the 1153 x 1300 image: a window's own walk starts a segment on band 19, 38 or 57 and first transforms the band above
    for m in (19, 38, 57):
        g = fused_geo(1300, 1153, (256, 16 * m - 1, 768, 16 * m + 39))
        assert g["segs"][0][0] == m, m
    assert len(fused_geo(1300, 1153, (0, 303, 1300, 1153))["segs"]) == 3
    assert window(1300, 1153, (8, 0, 24, 5))[4] and not window(1300, 1153, (8, 0, 255, 5))[4] and not window(1300, 1153, (3, 0, 24, 5))[4]


# ------------------------------------------------------------------------------------------------------------------
# streams and references (cached: cv2 on the CPU is most of this file's time)
def _image(h, w, seed):
    """gh.synth_image plus independent noise per channel, so that the chroma changes at every column and row"""
    rng = np.random.default_rng(seed + 7919)
    img = gh.synth_image(h, w, seed).astype(np.int16) + rng.integers(-40, 41, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


@functools.lru_cache(maxsize=None)
def stream(h, w, layout="420", rst=0, progressive=False, q=90):
    import cv2
    img = _image(h, w, 1000 * h + w + 17 * rst)
    params = [cv2.IMWRITE_JPEG_QUALITY, q]
    if layout == "gray":
        img = img[..., 0]
    else:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, getattr(cv2, f"IMWRITE_JPEG_SAMPLING_FACTOR_{layout}")]
    if rst:
        params += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    if progressive:
        params += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
    ok, enc = cv2.imencode(".jpg", img, params)
    assert ok
    return enc.tobytes()


@functools.lru_cache(maxsize=None)
def reference(s, ot=capi.RGB, fancy=True):
    """cv2's decode of the stream (box upsampling: the oracle's, which cv2 cannot do)"""
    import cv2
    if not fancy:
        out = po.jpeg_decode(s, fancy=False)
        return out[..., ::-1] if ot == capi.BGR else out
    if ot == capi.GRAY:
        return cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_GRAYSCALE)[..., None]
    out = cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR)
    return out if ot == capi.BGR else out[..., ::-1]


def decode(streams, ot=capi.RGB, fancy=True, dtype=capi.UINT8, orient=False, rois=None, offsets=None, packed=False, what=""):
    """the streams through dalib200JpegPlanSetupEx / JpegLaunch, the outputs in one gh.SentinelSlices allocation (at `offsets` bytes
    past 256-byte boundaries, or packed), the launch profiled: (outputs, names of the kernels that ran)"""
    lib = capi.lib()
    n = len(streams)
    bufs = [np.frombuffer(s, np.uint8) for s in streams]
    plan = capi.Plan("Jpeg", n)
    prm = capi.JpegParams(ot, int(fancy), dtype, int(orient))
    cr = None
    if rois is not None:
        cr = (capi.JpegRoi * n)()
        for i, r in enumerate(rois):
            if r is not None:
                cr[i].use_roi = 1
                cr[i].x0, cr[i].y0, cr[i].x1, cr[i].y1 = [int(v) for v in r]
    capi.check(lib.dalib200JpegPlanSetupEx(plan.handle, n, (C.c_void_p * n)(*[b.ctypes.data for b in bufs]),
                                           (C.c_size_t * n)(*[b.size for b in bufs]), C.byref(prm), cr))
    shapes = []
    for i in range(n):
        hwc = (C.c_int32 * 3)()
        capi.check(lib.dalib200JpegPlanGetOutputShape(plan.handle, i, hwc))
        shapes.append(tuple(hwc))
    item, dt = (1, np.uint8) if dtype == capi.UINT8 else (4, np.float32)
    outs = gh.SentinelSlices([int(np.prod(s)) * item for s in shapes], item, offsets, packed)
    capi.profiling(True)
    try:
        capi.profiling_collect()
        capi.check(lib.dalib200JpegUpload(plan.handle, capi.stream_handle()))
        capi.check(lib.dalib200JpegLaunch(plan.handle, (C.c_void_p * n)(*outs.ptrs), capi.stream_handle()))
        got = outs.read(what)
        names = {nm for nm, _ in capi.profiling_collect()}
    finally:
        capi.profiling(False)
    status = (C.c_int32 * n)()
    capi.check(lib.dalib200JpegGetStatus(plan.handle, status))
    assert list(status) == [0] * n, what
    return [g.view(dt).reshape(s) for g, s in zip(got, shapes)], names


def check_against_cv2(streams, kernel, ot=capi.RGB, rois=None, fancy=True, offsets=None, what="", absent=()):
    """decodes the streams in one batch, each output equal to cv2's decode (or its crop), the target kernel among those that ran"""
    want = [reference(s, ot, fancy) for s in streams]
    if rois is not None:
        want = [w[r[1]:r[3], r[0]:r[2]] if r else w for w, r in zip(want, rois)]
    if offsets is None:
        offsets = [(3 * k) % 16 for k in range(len(streams))]     # every output alignment, so every store width of the kernels
    outs, names = decode(streams, ot, fancy, rois=rois, offsets=offsets, what=what)
    for k, (o, w) in enumerate(zip(outs, want)):
        assert np.array_equal(o, w), (what, k, o.shape, rois[k] if rois else None)
    assert kernel in names, (what, kernel, names)
    for a in absent:
        assert a not in names, (what, a, names)
    return names


# ------------------------------------------------------------------------------------------------------------------
# 1. idct_color_420
STRIP_WIDTHS = (255, 256, 257, 264, 511, 512, 513)


@pytest.mark.parametrize("ot", [capi.RGB, capi.BGR], ids=["rgb", "bgr"])
def test_420_width_sweep(ot):
    """h = 24 (two bands): widths 5-36 (every residue mod 16 twice, every value of the last chroma column's `edge` four times) and the
    strip edges; width 4 is below the fused kernel's threshold and takes color_fast_kernel, width 5 is above it"""
    widths = list(range(5, 37)) + list(STRIP_WIDTHS)
    check_against_cv2([stream(24, w) for w in widths], FUSED, ot, what=f"widths {OT[ot]}")
    check_against_cv2([stream(24, 4)], FAST, ot, what="width 4", absent=(FUSED,))
    check_against_cv2([stream(24, 5)], FUSED, ot, what="width 5", absent=(FAST,))


@pytest.mark.parametrize("ot", [capi.RGB, capi.BGR], ids=["rgb", "bgr"])
def test_420_height_sweep_and_segment_splits(ot):
    """w = 40: heights 1-33 (one band that is also the last, one- and two-row chroma planes, the last band's extra row at 16 and 32);
    w = 264: 24-band segments split as fused_geo splits them"""
    check_against_cv2([stream(h, 40) for h in range(1, 34)], FUSED, ot, what=f"heights {OT[ot]}")
    check_against_cv2([stream(h, 264) for h in (384, 385, 401, 768, 769, 1153)], FUSED, ot, what=f"segments {OT[ot]}")


def _windows_1153x1300():
    W, H = 1300, 1153
    bands = [a for a, _ in fused_geo(W, H)["segs"]][1:]               # 19, 38, 57: first band of each later segment
    xs = [(256, 768), (8, 264), (1032, 1300), (0, W)]
    wins = []
    for i, m in enumerate(bands):
        for dy in (-1, 0, 1):                                          # top edge at, above and below a segment's first emitted row
            x0, x1 = xs[(3 * i + dy + 1) % len(xs)]
            wins.append((x0, 16 * m - 1 + dy, x1, min(H, 16 * m + 40 + dy)))
        x0, x1 = xs[i]
        wins.append((x0, 16 * m - 30, x1, 16 * m))                     # bottom edge on a carry row (row 16m - 1, emitted by band m)
    wins.append((0, 303, W, H))                                        # three segments of the window's own walk
    for x0 in (8, 24, 136, 520, 1032, 1288):                           # x = 8 (mod 16): mid-MCU, no post pass
        wins.append((x0, 100, min(W, x0 + 48), 140))
    for k in (1, 2, 3, 4):                                             # around the strip boundaries 256k
        for x0 in (256 * k - 8, 256 * k, 256 * k + 8):
            wins.append((x0, 290, min(W, x0 + 264), 320))
        for x1 in (256 * k - 1, 256 * k + 1):
            wins.append((x1 - 200, 590, x1, 630))
    for x in (0, 255, 256, 263, 1291, 1299):                           # one pixel wide
        wins.append((x, 280, x + 1, 340))
    for y in (0, 302, 303, 304, 1151, 1152):                           # one pixel tall
        wins.append((248, y, 776, y + 1))
    wins.append((1296, 0, W, H))                                       # the last MCU column alone
    wins += [(x0 + 3, y0, x1, y1) for x0, y0, x1, y1 in list(wins) if x0 + 3 < x1]    # the same through the post pass
    return wins


@pytest.mark.parametrize("ot", [capi.RGB, capi.BGR], ids=["rgb", "bgr"])
def test_420_windows_on_segment_strip_and_mcu_edges(ot):
    s = stream(1153, 1300)
    check_against_cv2([s], FUSED, ot, what="full 1153 x 1300")
    wins = _windows_1153x1300()
    direct = [r for r in wins if window(1300, 1153, r)[4]]
    post = [r for r in wins if not window(1300, 1153, r)[4]]
    assert len(direct) > 30 and len(post) > 30
    check_against_cv2([s] * len(direct), FUSED, ot, direct, what=f"direct windows {OT[ot]}", absent=(POST,))
    names = check_against_cv2([s] * len(post), FUSED, ot, post, what=f"windows through the post pass {OT[ot]}")
    assert POST in names, names


def test_420_restart_intervals():
    streams = [stream(h, w, rst=rst) for rst in (1, 3) for h, w in ((24, 5), (24, 21), (24, 36), (17, 40), (24, 257), (385, 264))]
    for ot in (capi.RGB, capi.BGR):
        check_against_cv2(streams, FUSED, ot, what=f"restarts {OT[ot]}")


# ------------------------------------------------------------------------------------------------------------------
# 2. color_fast_kernel
WIDE = (1019, 1021, 1023, 1024, 1025, 1027, 1029, 2043, 2045, 2047, 2048, 2049, 2051, 2053)


@pytest.mark.parametrize("layout", ["444", "422"])
def test_fast_rows_of_one_two_and_three_items(layout):
    """rows of one, two and three kColorSeg-pixel items; 2041-2048 px rows are where a misplaced second item leaves pixels unwritten"""
    assert {-(-w // COLOR_SEG) for w in WIDE} == {1, 2, 3}
    streams = [stream(3 + 2 * (k % 3), w, layout) for k, w in enumerate(WIDE)]
    for ot in (capi.RGB, capi.BGR):
        check_against_cv2(streams, FAST, ot, what=f"{layout} {OT[ot]}", absent=(FUSED, GENERIC))
    s = stream(7, 2049, layout)
    rois = [(1016, 0, 2049, 7), (1024, 1, 2049, 6), (1032, 2, 2048, 5), (1016, 0, 2040, 1), (1024, 3, 2041, 7), (1032, 0, 1043, 7)]
    check_against_cv2([s] * len(rois), FAST, capi.RGB, rois, what=f"{layout} windows")


def _sms():
    import torch
    import conftest
    return 132 if conftest.DRY_RUN else torch.cuda.get_device_properties(0).multi_processor_count


# 4:4:4 / 4:2:2 images with 4:2:0 images, which own no color_fast_kernel items, between them; every fast image is followed by others
INTERLEAVED = [(9, 1000, "444"), (24, 300, "420"), (33, 1000, "420"), (1153, 1300, "444"), (17, 257, "420"), (1153, 1300, "422"),
               (24, 40, "420"), (24, 5, "420"), (1153, 1300, "444"), (40, 264, "420"), (1151, 1299, "422"), (24, 36, "420")]


def test_fast_items_step_over_420_images():
    """more color_fast_kernel items than its grid of NumSMs x 64 CTAs, so that a CTA owns several consecutive items: ranges that start
    in one image and end in the next fast image walk over the 4:2:0 images between them after the CTA's one search"""
    items = [-(-w // COLOR_SEG) * h if lay != "420" else 0 for h, w, lay in INTERLEAVED]
    first, total = np.cumsum([0] + items[:-1]), sum(items)
    grid = min(total, _sms() * 64)                                     # LaunchReconstruct's grid of color_fast_kernel
    assert total > grid, (total, grid)
    per_cta = -(-total // grid)
    image_of = lambda it: int(np.searchsorted(first, it, "right")) - 1     # noqa: E731
    crossings = {(image_of(it0), image_of(min(total, it0 + per_cta) - 1)) for it0 in range(0, total, per_cta)}
    crossings = {(a, b) for a, b in crossings if b > a + 1}           # a range that steps over at least one zero-item image
    assert crossings == {(0, 3), (3, 5), (5, 8), (8, 10)}, crossings
    streams = [stream(h, w, lay) for h, w, lay in INTERLEAVED]
    names = check_against_cv2(streams, FAST, what="interleaved")
    assert FUSED in names, names


# ------------------------------------------------------------------------------------------------------------------
# 3. color_kernel, and the layouts that take color_fast_kernel although they are not 4:4:4 / 4:2:2
# (layout, fancy, kernel): ReconAddImage sends 3-component YCbCr with a horizontal factor of 1 or 2 to color_fast_kernel
LAYOUT_PATHS = [("411", True, GENERIC), ("gray", True, GENERIC), ("440", True, FAST), ("420", False, FAST)]


@pytest.mark.parametrize("layout,fancy,kernel", LAYOUT_PATHS, ids=[f"{a}-{'fancy' if b else 'box'}" for a, b, _ in LAYOUT_PATHS])
def test_layouts_widths_around_1024_odd_heights(layout, fancy, kernel):
    streams = [stream(2 * (k % 4) + 3, w, layout) for k, w in enumerate(range(1018, 1030))]
    for ot in (capi.RGB, capi.BGR):
        others = tuple(k for k in (FUSED, FAST, GENERIC) if k != kernel)
        check_against_cv2(streams, kernel, ot, fancy=fancy, what=f"{layout} {OT[ot]}", absent=others)
    if layout == "gray":
        check_against_cv2(streams, GENERIC, capi.GRAY, what="gray -> gray")


# ------------------------------------------------------------------------------------------------------------------
# 4. output placement
def _mixed():
    """(stream, region of interest): every reconstruct path, the multi-scan stage, a window, EXIF orientation 6"""
    return [(stream(97, 203), None), (stream(61, 131, "444"), None), (stream(45, 77, "411"), None), (stream(33, 70, "gray"), None),
            (stream(50, 90, progressive=True), None), (stream(120, 260), (13, 5, 203, 77)),
            (po.with_exif_orientation(stream(71, 150), 6), None), (stream(31, 1037, "422"), None), (stream(16, 37), (8, 0, 32, 16)),
            (stream(3, 5), None)]


@pytest.mark.parametrize("ot,dtype", [(capi.RGB, capi.UINT8), (capi.YCbCr, capi.UINT8), (capi.RGB, capi.FLOAT)],
                         ids=["rgb-u8", "ycbcr-u8", "rgb-float"])
def test_mixed_batch_at_every_offset_equals_solo_decodes(ot, dtype):
    mixed = _mixed()
    solo = []
    for k, (s, r) in enumerate(mixed):
        (out,), status = gh.jpeg_decode_ex([s], output_type=ot, dtype=dtype, rois=[r])
        assert status == [0], (OT[ot], dtype, "solo decode", k)
        solo.append(out)
    streams, rois = [s for s, _ in mixed], [r for _, r in mixed]
    step = 1 if dtype == capi.UINT8 else 4
    layouts = [dict(offsets=[(a + step * k) % 16 for k in range(len(mixed))]) for a in range(0, 16, step)] + [dict(packed=True)]
    for lay in layouts:
        outs, names = decode(streams, ot, dtype=dtype, orient=True, rois=rois, what=f"{OT[ot]} {dtype} {lay}", **lay)
        for k, (o, w) in enumerate(zip(outs, solo)):
            assert o.shape == w.shape and np.array_equal(o, w), (OT[ot], dtype, lay, k)
        for kernel in (FUSED, FAST, GENERIC, POST):
            assert kernel in names, (OT[ot], dtype, kernel, names)


# ------------------------------------------------------------------------------------------------------------------
# 5. fn.jpeg_compression_distortion through the same kernels
def distort(imgs, qs, offsets):
    lib = capi.lib()
    n = len(imgs)
    plan = capi.Plan("JpegDistort", n)
    samples = (capi.JpegDistortSample * n)()
    for s, im, q in zip(samples, imgs, qs):
        s.height, s.width, s.quality = im.shape[0], im.shape[1], q
    capi.check(lib.dalib200JpegDistortPlanSetup(plan.handle, n, samples))
    _src, ip = gh.upload_slices(imgs, [(o + 5) % 16 for o in offsets])
    outs = gh.SentinelSlices([im.nbytes for im in imgs], 1, offsets)
    capi.profiling(True)
    try:
        capi.profiling_collect()
        capi.check(lib.dalib200JpegDistortLaunch(plan.handle, (C.c_void_p * n)(*ip), (C.c_void_p * n)(*outs.ptrs), capi.stream_handle()))
        got = outs.read("distortion")
        names = {nm for nm, _ in capi.profiling_collect()}
    finally:
        capi.profiling(False)
    return [g.reshape(im.shape) for g, im in zip(got, imgs)], names


def test_distortion_width_sweep_and_wide_rows():
    shapes = [(24, w) for w in list(range(5, 37)) + list(STRIP_WIDTHS)] + [(3 + 2 * (k % 3), w) for k, w in enumerate(WIDE)]
    imgs = [_image(h, w, 31 * h + w) for h, w in shapes]
    qs = [(37 * k) % 100 + 1 for k in range(len(imgs))]
    want = [jc.reference(im, q) for im, q in zip(imgs, qs)]
    outs, names = distort(imgs, qs, [(3 * k) % 16 for k in range(len(imgs))])
    for o, w, im, q in zip(outs, want, imgs, qs):
        assert np.array_equal(o, w), (im.shape, q)
    assert FUSED in names, names
