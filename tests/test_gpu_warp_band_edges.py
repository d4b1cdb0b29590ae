"""-m gpu: warp_affine at the parts of its three kernels (csrc/warp.cu) that small batches never reach.  Each case asserts the path it targets
(dalib200WarpPlanGetPath: 0 the generic kernel, 1 the band kernel with tensor-map source boxes, 2 the band kernel without them):

  1. at least three work items per CTA on every path, so that CTAs walk on from their first item into later items and later frames (the
     sample walk, the mbarrier phases carried from item to item, the tensor map's frame coordinate);
  2. band-path outputs wider than one 2048-column band (the anchor replay of the second band, several 128-column tiles, partial runs and
     partial tiles);
  3. the tensor map's eligibility rules: 432- against 480-byte rows, frames at a stride of frame + 16 and frame + 4096 bytes, one frame, a
     base 16-byte but not 128-byte aligned, strides and bases that are not 16-byte multiples;
  4. the plan's cached tensor map across launches on another base, another frame count, another shape, a non-uniform batch and back;
  5. outputs at byte offsets 0, 1, 4 and 16 (the band kernel's three store forms, the generic kernel's packed 4-pixel store);
  6. the generic kernel's 8-channel instance at C = 2, 5, 6, 7, 8, and the 3-channel funnel-shift path next to the last row pair;
  7. the C3 benchmark's frames: 3 x 16 frames of 720p (about four band items per CTA) through hotpath.VideoPipelineC3, and one FHWC sample
     of 16 such frames through fn.warp_affine;
  8. the band kernel and the nfft = 1024 spectrogram on a second device in the same process (skipped with fewer than two devices).

Every output is compared bit for bit with oracle.pyoracle.warp_affine and held to the float64 statement of tests/image_f64.py; the float64
statement is applied to a fixed subset where a test's docstring says so (the generic kernel's many-tile batches and the 720p frames).
Inputs are frames of one device allocation at a chosen stride and base offset; outputs are views at chosen byte offsets inside an
allocation filled with gpu_helpers.SENTINEL, and every byte outside the views is checked unchanged.

Run time on an H100 80GB HBM3 (700 W power limit): about 80 s, most of it the host oracle and the float64 statement."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
from oracle import pyoracle as po  # noqa: E402
import image_f64 as F  # noqa: E402

GENERIC, TMA, BAND = 0, 1, 2
# warp.cu: the band kernel's work item is a band of 32 rows x 2048 columns, on a grid of 2 CTAs per SM; the generic kernel's is a tile of
# 16 rows x 256 columns, on a grid of 16 CTAs per SM
BAND_ITEM, BAND_CTAS_PER_SM = (32, 2048), 2
TILE, GENERIC_CTAS_PER_SM = (16, 256), 16

ITEMS_PER_CTA = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("work items per CTA (largest launch per case):", {k: round(v, 2) for k, v in sorted(ITEMS_PER_CTA.items())})


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _sms():
    import torch
    import conftest
    return 132 if conftest.DRY_RUN else torch.cuda.get_device_properties(0).multi_processor_count


def work(out_hws, path, case):
    """(work items of a launch on `path`, the kernel's grid); notes items per CTA for the report."""
    (h, w), per_sm = (TILE, GENERIC_CTAS_PER_SM) if path == GENERIC else (BAND_ITEM, BAND_CTAS_PER_SM)
    items, grid = sum(-(-oh // h) * -(-ow // w) for oh, ow in out_hws), per_sm * _sms()
    ITEMS_PER_CTA[case] = max(ITEMS_PER_CTA.get(case, 0.0), items / grid)
    return items, grid


def _smooth(rng, shape):
    """A u8 image whose values change by a few levels per pixel, so that the float64 bound's coordinate term stays below a level."""
    H, W, Cn = shape
    y, x = np.meshgrid(np.arange(H, dtype=np.float64), np.arange(W, dtype=np.float64), indexing="ij")
    out = np.empty(shape)
    for c in range(Cn):
        p = rng.uniform(0, 6, 3)
        out[..., c] = 128 + 70 * np.sin(2 * np.pi * x / 260 + p[0]) * np.cos(2 * np.pi * y / 230 + p[1]) + 25 * np.sin(2 * np.pi * (x - y) / 170 + p[2])
    return np.clip(np.round(out), 0, 255).astype(np.uint8)


def frames(rng, n, H, W, Cn=3):
    """n different smooth frames: crops of one larger smooth image at random offsets."""
    field = _smooth(rng, (H + 128, W + 128, Cn))
    return [np.ascontiguousarray(field[y:y + H, x:x + W]) for y, x in rng.integers(0, 129, (n, 2))]


def noise(rng, shapes):
    return [rng.integers(0, 256, s).astype(np.uint8) for s in shapes]


def mat(kind, in_hw, out_hw, rng):
    """dst -> src matrix about the two centres, of a kind the band kernel treats differently: 0 a small rotation (the tile's footprint
    inside the loaded box), 1 +-12 degrees (the box's limit), 2 a scale of 2.2 (the footprint larger than the box), 3 a map partly outside
    the source, 4 one wholly outside it, 5 a rotated magnification that fits the output onto the source."""
    (H, W), (oh, ow) = in_hw, out_hw
    t = (0.0, 0.0)
    if kind == 0:
        deg, sc, t = rng.uniform(-3, 3), 1.0, rng.uniform(-2, 2, 2)
    elif kind == 1:
        deg, sc, t = rng.choice([-12.0, 12.0]), 1.0, rng.uniform(-1, 1, 2)
    elif kind == 2:
        deg, sc = rng.uniform(-5, 5), 2.2
    elif kind == 3:
        deg, sc, t = rng.uniform(-6, 6), 1.0, (0.45 * W, -0.4 * H)
    elif kind == 4:
        deg, sc, t = 0.0, 1.0, (3.0 * W + 50.0, 0.0)
    else:
        deg, sc = rng.uniform(-4, 4), 0.95 * min(W / ow, H / oh)
    a = np.deg2rad(deg)
    c, s = np.cos(a) * sc, np.sin(a) * sc
    return np.float32([[c, -s, W / 2 - c * ow / 2 + s * oh / 2 + t[0]], [s, c, H / 2 - s * ow / 2 - c * oh / 2 + t[1]]])


class WarpPlan:
    """One dalib200WarpPlan, set up and launched again for every batch."""

    def __init__(self, max_batch):
        self.plan = capi.Plan("Warp", max_batch)

    def run(self, imgs, mats, out_hws, interp=1, fill=None, out_dtype=np.uint8, stride=None, base=0, buf=None, out_offsets=None):
        """Input i at byte base + i * stride of `buf` (a uint8 CUDA tensor; default a new one) counted from its first 256-byte boundary;
        stride None: each input's bytes rounded up to 256, back to back.  Output i at out_offsets[i] bytes past a 256-byte boundary of one
        SENTINEL-filled allocation (gpu_helpers.SentinelSlices: a byte changed outside the outputs fails).  Returns (outputs, path)."""
        import torch
        import gpu_helpers as g
        n = len(imgs)
        samples = (capi.WarpSample * n)()
        for s, im, M, hw in zip(samples, imgs, mats, out_hws):
            s.in_h, s.in_w, s.channels = im.shape
            s.out_h, s.out_w = hw
            s.matrix[:] = [float(v) for v in np.asarray(M, np.float32).reshape(6)]
        odt = capi.UINT8 if np.dtype(out_dtype) == np.uint8 else capi.FLOAT
        capi.check(capi.lib().dalib200WarpPlanSetup(self.plan.handle, n, samples, int(interp), int(fill is not None), C.c_float(fill or 0.0), odt))
        if stride is None:
            pos = np.cumsum([0] + [-(-im.nbytes // 256) * 256 for im in imgs])[:n]
        else:
            pos = np.arange(n) * stride
        pos = [base + int(p) for p in pos]
        end = max(p + im.nbytes for p, im in zip(pos, imgs))
        host = np.zeros(end, np.uint8)
        for p, im in zip(pos, imgs):
            host[p:p + im.nbytes] = np.ascontiguousarray(im).reshape(-1)
        if buf is None:
            buf = torch.empty(end + 256, dtype=torch.uint8, device="cuda")
        a = -buf.data_ptr() % 256
        assert buf.numel() >= a + end
        buf[a:a + end].copy_(torch.from_numpy(host))
        isz = np.dtype(out_dtype).itemsize
        outs = g.SentinelSlices([oh * ow * im.shape[2] * isz for (oh, ow), im in zip(out_hws, imgs)], isz, out_offsets)
        capi.check(capi.lib().dalib200WarpLaunch(self.plan.handle, capi.ptr_array([buf.data_ptr() + a + p for p in pos]),
                                                 capi.ptr_array(outs.ptrs), capi.stream_handle()))
        got = outs.read(("output offsets", out_offsets))
        path = capi.lib().dalib200WarpPlanGetPath(self.plan.handle)
        return [o.view(out_dtype).reshape(tuple(hw) + (im.shape[2],)) for o, hw, im in zip(got, out_hws, imgs)], path


def check(got, img, M, out_hw, interp, fill, out_dt, what, f64=True):
    """Bit for bit against the oracle, then (f64) within the float64 statement's bound, as test_gpu_image_f64._check_warp does."""
    want = po.warp_affine(img, M, out_hw, interp, fill, out_dt)
    bad = bits(got) != bits(want)
    assert not bad.any(), ("bit-exact", what, f"{int(bad.sum())} of {bad.size} bytes differ")
    if not f64:
        return
    if interp == 0:
        F.check_choice(got, F.warp_affine(img, M, out_hw, 0, fill), what)
        return
    v, b = F.warp_affine(img, M, out_hw, 1, fill)
    if np.dtype(out_dt) == np.uint8:
        F.check_u8(got, v, b, what)
    else:
        F.check(got, v, b, what)


def check_batch(got, imgs, mats, out_hws, interp, fill, out_dt, what, f64_every=1):
    for i, (o, im, M, hw) in enumerate(zip(got, imgs, mats, out_hws)):
        check(o, im, M, hw, interp, fill, out_dt, (what, i, im.shape, hw, M.tolist()), f64=i % f64_every == 0)


# ------------------------------------------------------------------------------------------------------------ 1. many items per CTA
def test_band_paths_many_items_per_cta(monkeypatch):
    """Path 1: 600 frames of 64 x 160 (two band items each) under clamp, then 300 frames of 72 x 160 (three items each, so that CTA ranges
    start and end inside frames) under fill.  Path 2 (DALIB200_WARP_BAND=1): the same at 150 columns, whose 450-byte rows a tensor map
    cannot describe.  The six matrix kinds of mat() alternate from frame to frame."""
    rng = np.random.default_rng(901)
    wp = WarpPlan(600)
    for path, W in ((TMA, 160), (BAND, 150)):
        if path == BAND:
            monkeypatch.setenv("DALIB200_WARP_BAND", "1")
        for H, n, fill in ((64, 600, None), (72, 300, 33.0)):
            imgs, hws = frames(rng, n, H, W), [(H, W)] * n
            mats = [mat(k % 6, (H, W), (H, W), rng) for k in range(n)]
            items, grid = work(hws, path, "1 band")
            assert items >= 3 * grid, (items, grid)
            got, p = wp.run(imgs, mats, hws, 1, fill, stride=H * W * 3)
            assert p == path, (p, path, (H, W))
            check_batch(got, imgs, mats, hws, 1, fill, np.uint8, ("many items", path, (H, W), fill))


def test_generic_kernel_many_tiles_per_cta():
    """Path 0: one batch of mixed sizes (1 to 48 rows, 1 to 700 columns out; C = 1, 3, 4) with at least three 16 x 256 tiles per CTA of
    the generic kernel's grid, bilinear u8, nearest-neighbour u8 and bilinear float, clamp and fill.  Every sample is compared bit for bit;
    the float64 statement is applied to every fourth sample (it would take about a minute for the whole batch)."""
    rng = np.random.default_rng(902)
    shapes, hws, tiles = [], [], 0
    while tiles < 3 * GENERIC_CTAS_PER_SM * _sms() + 64:
        shapes.append((int(rng.integers(8, 97)), int(rng.integers(8, 261)), int(rng.choice([1, 3, 4]))))
        hws.append((int(rng.integers(1, 49)), int(rng.integers(1, 701))))
        tiles += -(-hws[-1][0] // TILE[0]) * -(-hws[-1][1] // TILE[1])
    items, grid = work(hws, GENERIC, "1 generic")
    assert items >= 3 * grid, (items, grid)
    n = len(shapes)
    imgs = noise(rng, shapes)
    mats = [mat(k % 6, s[:2], hw, rng) for k, (s, hw) in enumerate(zip(shapes, hws))]
    wp = WarpPlan(n)
    for interp, fill, odt in ((1, None, np.uint8), (0, 9.0, np.uint8), (1, 200.0, np.float32)):
        got, p = wp.run(imgs, mats, hws, interp, fill, odt)
        assert p == GENERIC, p
        check_batch(got, imgs, mats, hws, interp, fill, odt, ("many tiles", interp, fill, np.dtype(odt).name), f64_every=4)


# ------------------------------------------------------------------------------------------------------------ 2. wider than one band
def test_band_outputs_wider_than_one_band(monkeypatch):
    """Out widths 2047, 2048, 2049, 2184, 3840, 4096 + 17 and 4113 (one to three bands of 2048 columns; runs of 16 and tiles of 128
    columns cut short), out heights 31, 32, 33, 63, 64, 65 and 95, from 96 x 640 frames (path 1) and 96 x 630 frames (path 2), clamp and
    fill: mostly magnifications that keep the footprint inside the source, plus a rotation, the 12-degree limit and a partial map."""
    rng = np.random.default_rng(903)
    hws = [(31, 2047), (32, 2048), (33, 2049), (64, 2184), (63, 3840), (65, 4096 + 17), (95, 4113), (32, 2049), (33, 4096)]
    kinds = [5, 5, 5, 0, 5, 5, 1, 3, 5]
    wp = WarpPlan(len(hws))
    for path, W in ((TMA, 640), (BAND, 630)):
        if path == BAND:
            monkeypatch.setenv("DALIB200_WARP_BAND", "1")
        H = 96
        imgs = frames(rng, len(hws), H, W)
        mats = [mat(k, (H, W), hw, rng) for k, hw in zip(kinds, hws)]
        work(hws, path, "2 wide")
        for fill in (None, 77.0):
            got, p = wp.run(imgs, mats, hws, 1, fill, stride=H * W * 3)
            assert p == path, (p, path)
            check_batch(got, imgs, mats, hws, 1, fill, np.uint8, ("wide", path, fill))


# ------------------------------------------------------------------------------------------------------------ 3. eligibility
def test_tensor_map_eligibility(monkeypatch):
    """Which batches get a tensor map (path 1), and that those which do not stay exact on the generic kernel (path 0) or, when asked
    for it, on the band kernel without boxes (path 2)."""
    rng = np.random.default_rng(904)
    H = 40
    fb = lambda W: H * W * 3
    # (what, in_w, frames, stride, base, path, path with DALIB200_WARP_BAND=1)
    cases = [("432-byte rows", 144, 4, fb(144), 0, GENERIC, BAND),
             ("480-byte rows", 160, 4, fb(160), 0, TMA, TMA),
             ("stride frame + 16", 160, 4, fb(160) + 16, 0, TMA, TMA),
             ("stride frame + 4096", 160, 4, fb(160) + 4096, 0, TMA, TMA),
             ("one frame", 160, 1, None, 0, TMA, TMA),
             ("base 16-byte, not 128-byte aligned", 160, 4, fb(160), 48, TMA, TMA),
             ("stride frame + 4", 160, 4, fb(160) + 4, 0, GENERIC, BAND),
             ("stride frame + 1", 160, 4, fb(160) + 1, 0, GENERIC, BAND),
             ("stride frame + 24", 160, 4, fb(160) + 24, 0, GENERIC, BAND),
             ("base 8", 160, 4, fb(160), 8, GENERIC, BAND)]
    wp = WarpPlan(4)
    for k, (what, W, n, stride, base, path, asked) in enumerate(cases):
        imgs = frames(rng, n, H, W)
        hws = [(H + 9, W + 40)] * n
        mats = [mat((k + i) % 6, (H, W), hws[i], rng) for i in range(n)]
        fill = None if k % 2 else 5.0
        for env, want in ((False, path), (True, asked)):
            if env:
                monkeypatch.setenv("DALIB200_WARP_BAND", "1")
            else:
                monkeypatch.delenv("DALIB200_WARP_BAND", raising=False)
            got, p = wp.run(imgs, mats, hws, 1, fill, stride=stride, base=base)
            assert p == want, (what, env, p, want)
            check_batch(got, imgs, mats, hws, 1, fill, np.uint8, (what, env))


# ------------------------------------------------------------------------------------------------------------ 4. tensor-map cache
def test_tensor_map_cache_across_launches():
    """One plan, the map cached per (base, stride, height, width, frames): base A, base B (A still holds other frames), six frames at B
    (a map for four would read zeros), another shape at B, a non-uniform batch, A again with new frames, and A once more unchanged."""
    import torch
    rng = np.random.default_rng(905)
    H, W = 48, 160
    room = 6 * H * W * 3 + 4096
    A = torch.empty(room, dtype=torch.uint8, device="cuda")
    B = torch.empty(room, dtype=torch.uint8, device="cuda")
    steps = [("base A", A, 4, (H, W), TMA), ("base B", B, 4, (H, W), TMA), ("six frames at B", B, 6, (H, W), TMA),
             ("40 x 176 at B", B, 4, (40, 176), TMA), ("non-uniform", None, 4, None, GENERIC), ("base A again", A, 4, (H, W), TMA),
             ("base A, same key", A, 4, (H, W), TMA)]
    wp = WarpPlan(6)
    imgs = None
    for k, (what, buf, n, hw, path) in enumerate(steps):
        if hw is None:
            imgs = [frames(rng, 1, H + 8 * i, W)[0] for i in range(n)]
        elif what != "base A, same key":
            imgs = frames(rng, n, *hw)
        hws = [im.shape[:2] for im in imgs]
        mats = [mat((k + i) % 6, im.shape[:2], im.shape[:2], rng) for i, im in enumerate(imgs)]
        fill = 0.0 if k % 2 else None
        got, p = wp.run(imgs, mats, hws, 1, fill, stride=None if hw is None else hw[0] * hw[1] * 3, buf=buf)
        assert p == path, (what, p, path)
        check_batch(got, imgs, mats, hws, 1, fill, np.uint8, what)


# ------------------------------------------------------------------------------------------------------------ 5. output offsets
def test_output_byte_offsets(monkeypatch):
    """Outputs at byte offsets 0, 1, 4 and 16 from a 256-byte boundary, with the sentinel checked around each: the band kernel's 16-byte,
    4-byte and byte stores (out widths that are multiples of 16 and ones that are not) on paths 1 and 2, the generic kernel's packed
    4-pixel store (u8, C = 3, NN and bilinear) and its float stores at offsets 0, 4, 8 and 16."""
    rng = np.random.default_rng(906)
    offs = [0, 1, 4, 16] * 2
    hws = [(40, 320), (40, 320), (40, 320), (40, 320), (33, 336), (33, 327), (17, 2064), (41, 400)]
    wp = WarpPlan(len(hws))
    H = 40
    for path, W in ((TMA, 320), (BAND, 318), (GENERIC, 318)):
        if path == BAND:
            monkeypatch.setenv("DALIB200_WARP_BAND", "1")
        else:
            monkeypatch.delenv("DALIB200_WARP_BAND", raising=False)
        imgs = frames(rng, len(hws), H, W)
        mats = [mat(k % 6, (H, W), hw, rng) for k, hw in enumerate(hws)]
        runs = [(1, None, np.uint8, offs), (1, 3.0, np.uint8, offs)]
        if path == GENERIC:
            runs += [(0, None, np.uint8, offs), (1, None, np.float32, [0, 4, 8, 16] * 2)]
        for interp, fill, odt, o in runs:
            got, p = wp.run(imgs, mats, hws, interp, fill, odt, stride=H * W * 3, out_offsets=o)
            assert p == (path if interp == 1 and odt == np.uint8 else GENERIC), (path, p, interp)
            check_batch(got, imgs, mats, hws, interp, fill, odt, ("offsets", path, interp, np.dtype(odt).name))


# ------------------------------------------------------------------------------------------------------------ 6. channels
def test_generic_kernel_channels():
    """C = 2, 5, 6, 7 and 8 (every channel a different random plane) with C = 3 samples in one batch, NN and bilinear, u8 and float, clamp
    and fill; outputs wider than 256 columns.  The C = 3 samples under a shift of (0.25, 0.5) sample the last row pair as interior
    pixels, where the 3-channel funnel-shift loads (warp_pixel, CMAX = 3) must give way to the byte loads."""
    rng = np.random.default_rng(907)
    shapes = [(37, 53, 2), (37, 53, 5), (29, 61, 6), (37, 53, 7), (41, 47, 8), (23, 41, 3), (30, 64, 3), (1, 9, 8), (37, 53, 8)]
    hws = [(45, 300), (45, 300), (30, 520), (45, 300), (41, 47), (23, 44), (30, 64), (5, 260), (60, 90)]
    imgs = noise(rng, shapes)
    mats = [mat(k % 6, s[:2], hw, rng) for k, (s, hw) in enumerate(zip(shapes, hws))]
    mats[5] = mats[6] = np.float32([[1, 0, 0.25], [0, 1, 0.5]])
    wp = WarpPlan(len(shapes))
    for interp in (0, 1):
        for fill in (None, 21.0):
            for odt in (np.uint8, np.float32):
                got, p = wp.run(imgs, mats, hws, interp, fill, odt)
                assert p == GENERIC, p
                check_batch(got, imgs, mats, hws, interp, fill, odt, ("channels", interp, fill, np.dtype(odt).name))


# ------------------------------------------------------------------------------------------------------------ 7. C3 frames
def _c3_params(nseq, flen, fh, fw):
    """bench.py's C3 recipe: per sequence a src -> dst rotation by up to 10 degrees and a scale of 0.95 to 1.05 about the centre (the
    kernel gets its inverse), hue / saturation / value and a mirror flag; frames of a sequence share them."""
    rng = np.random.default_rng(3)
    inv, hsvp, mir = [], [], []
    for _ in range(nseq):
        ang, sc = np.deg2rad(rng.uniform(-10, 10)), rng.uniform(0.95, 1.05)
        cx, cy = fw / 2, fh / 2
        a, b = sc * np.cos(ang), sc * np.sin(ang)
        fwd = np.array([[a, -b, cx - a * cx + b * cy], [b, a, cy - b * cx - a * cy]], np.float32)
        hp = (rng.uniform(-30, 30), rng.uniform(0.7, 1.3), rng.uniform(0.8, 1.2))
        inv += [po.affine_inv(fwd)] * flen
        hsvp += [hp] * flen
        mir += [int(rng.integers(0, 2))] * flen
    return inv, hsvp, mir


def _profiled(fn):
    """fn() with the library's launch timing on: (fn's result, names of the kernels it launched)."""
    import torch
    capi.profiling(True)
    try:
        capi.profiling_collect()
        r = fn()
        torch.cuda.synchronize()
        names = [name for name, _ in capi.profiling_collect()]
    finally:
        capi.profiling(False)
    return r, names


def test_c3_benchmark_frames():
    """hotpath.VideoPipelineC3 on 3 x 16 random frames of 720p with bench.py's parameters: 23 band items per frame, about four per CTA.
    Every frame's warp, hsv and crop_mirror_normalize outputs equal the oracle's, stage by stage; the float64 statement is applied to the
    warp of frames 5, 30 and 47 (about 2 s each on the host)."""
    import torch
    from dali_b200.hotpath import VideoPipelineC3, IMAGENET_MEAN, IMAGENET_STD
    nseq, flen, fh, fw = 3, 16, 720, 1280
    nfr = nseq * flen
    inv, hsvp, mir = _c3_params(nseq, flen, fh, fw)
    items, grid = work([(fh, fw)] * nfr, TMA, "7 C3")
    assert items >= 3 * grid, (items, grid)
    host = np.random.default_rng(908).integers(0, 256, (nfr, fh, fw, 3), dtype=np.uint8)
    dev = torch.from_numpy(host).cuda()
    v = VideoPipelineC3(nfr, (fh, fw))
    v.setup(inv, hsvp, mir)
    _, names = _profiled(lambda: v.launch(dev))
    assert "warp_affine_tma" in names, names
    assert capi.lib().dalib200WarpPlanGetPath(v.warp.handle) == TMA
    warped, twisted, out = v.warped.cpu().numpy(), v.twisted.cpu().numpy(), v.output.cpu().numpy()
    mean, istd = po.cmn_norm_args(IMAGENET_MEAN, IMAGENET_STD)
    for i in range(nfr):
        w = po.warp_affine(host[i], inv[i], None, 1, 0.0)
        assert np.array_equal(warped[i], w), ("warp", i, int((warped[i] != w).sum()))
        t = po.hsv(w, *hsvp[i])
        assert np.array_equal(twisted[i], t), ("hsv", i)
        c = po.cmn(t, (0, 0), (fh, fw), bool(mir[i]), mean, istd, np.float16, "CHW")
        assert np.array_equal(bits(out[i]), bits(c)), ("cmn", i)
        if i in (5, 30, 47):
            F.check_u8(warped[i], *F.warp_affine(host[i], inv[i], None, 1, 0.0), ("C3 warp", i))


def test_fn_warp_affine_fhwc_720p():
    """fn.warp_affine (u8, bilinear, fill 0) on one FHWC sample of 16 random 720p frames: the operator hands the frames to the band kernel
    with a tensor map; every frame equals the oracle, and frames 0 and 15 are held to the float64 statement."""
    from dali_b200 import fn, pipeline_def, types
    F_, fh, fw = 16, 720, 1280
    seq = np.random.default_rng(909).integers(0, 256, (F_, fh, fw, 3), dtype=np.uint8)
    M = _c3_params(1, 1, fh, fw)[0][0]

    @pipeline_def(batch_size=1, num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: [seq], device="gpu", layout="FHWC")
        return fn.warp_affine(x, matrix=M.reshape(6).tolist(), fill_value=0.0, interp_type=types.INTERP_LINEAR)
    p = pipe()
    p.build()
    (out,), names = _profiled(lambda: p.run())
    assert "warp_affine_tma" in names, names
    got = np.asarray(out.as_cpu()[0])
    assert got.shape == seq.shape, got.shape
    for f in range(F_):
        want = po.warp_affine(seq[f], M, None, 1, 0.0)
        assert np.array_equal(got[f], want), ("fn.warp_affine frame", f, int((got[f] != want).sum()))
        if f in (0, F_ - 1):
            F.check_u8(got[f], *F.warp_affine(seq[f], M, None, 1, 0.0), ("fn.warp_affine", f))


# ------------------------------------------------------------------------------------------------------------ 8. second device
def test_second_device_band_kernel_and_spectrogram():
    """The band kernel (90 KB of dynamic shared memory) and the nfft = 1024 spectrogram kernel need their shared-memory attribute set on
    each device they run on: the same batches on cuda:0 and then cuda:1 in one process give equal, exact outputs."""
    import torch
    import gpu_helpers as g
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    rng = np.random.default_rng(910)
    H, W, n = 96, 640, 6
    imgs = frames(rng, n, H, W)
    hws = [(H, W)] * 4 + [(33, 2100)] * 2
    mats = [mat(k % 6, (H, W), hw, rng) for k, hw in enumerate(hws)]
    t = np.arange(40000) / 16000.0
    sigs = [(0.3 * np.sin(2 * np.pi * f * t[:m]) + 0.01 * rng.normal(0, 1, m)).astype(np.float32) for f, m in ((440.0, 40000), (3000.0, 17001))]
    res = []
    for d in (0, 1):
        with torch.cuda.device(d):
            got, p = WarpPlan(n).run(imgs, mats, hws, 1, None, stride=H * W * 3)
            assert p == TMA, (d, p)
            spec = g.spectrogram(sigs, nfft=1024, window_length=1024, window_step=256)
        res.append((got, spec))
    for a, b in zip(res[0][0], res[1][0]):
        assert np.array_equal(a, b)
    check_batch(res[1][0], imgs, mats, hws, 1, None, np.uint8, "cuda:1")
    for s, a, b in zip(sigs, res[0][1], res[1][1]):
        assert np.array_equal(bits(a), bits(b))
        want = po.spectrogram(s, nfft=1024, window_length=1024, window_step=256)
        assert np.abs(b - want).max() <= 2e-4 * want.max()
