"""-m gpu: the streaming resize (resample_stream_kernel) at the boundaries of its own structure, each case built to reach one of them and
asserted to have reached it (dalib200ResamplePlanGetPath and dalib200ResamplePlanGetStreamInfo), so that a case that drifts away fails
instead of quietly testing the tile kernel:
  * chunks of 8 output rows and work items of 56 (out_h at every residue mod 8, around 56, 112 and at 224);
  * the walk limit of 96 source rows per chunk (J = 94, 95, 96 stream, 97 does not) and chunks whose J is not a multiple of the 4-row ring
    slot;
  * every walk width W = 1..4 alone and W = 1, 2 next to a W = 4 sample, so that every WMAX instance runs, with closed slots in the 4-slot one;
  * channel counts 1, 2, 3, 4, 8, 16, a strip of exactly 2048 bytes (one ring row) and one of 2064 (two strips), strips whose start is not
    16-byte aligned, a 1-pixel-wide output;
  * regions of interest on 16-byte-aligned rows: horizontal and vertical offsets, a flipped horizontal ROI (streams), a flipped vertical
    one (tile kernel), rows clamped above and below the image;
  * more than four work items per CTA in one launch, and one plan set up again with growing, shrinking and returning walk records.
Every input row is a multiple of 16 bytes (the kernel's condition at launch).  Every output is compared bit for bit with the oracle and, but
for the large mixed batch, with the float64 statement of tests/image_f64.py within its bound.  The planar variant (resample_planar_kernel,
the same walk records) runs a reduced set on 4:2:0 JPEGs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
from oracle import pyoracle as po  # noqa: E402
import image_f64 as F  # noqa: E402

LIN = (F.F_LINEAR, 1, 0.0)          # fn.resize's default: triangular (antialiased linear) on a down-scale
LNA = (F.F_LINEAR, 0, 0.0)          # linear without antialias: 2 taps whatever the scale
L3 = (F.F_LANCZOS3, 0, 0.0)
L3AA = (F.F_LANCZOS3, 1, 0.0)
CUBAA = (F.F_CUBIC, 1, 0.0)
WALK_MAX, SEG, CHUNK = 96, 56, 8

COVER = {"W, WMAX": set(), "largest streamed J": 0, "channels": set(), "items per CTA": 0.0, "|GPU - float64| / bound": 0.0}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("streaming resize coverage:", {k: sorted(v) if isinstance(v, set) else round(v, 4) if isinstance(v, float) else v
                                         for k, v in COVER.items()})


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _content(rng, shape, kind):
    """0: random bytes; 1: a 0 / 255 checkerboard; 2: 0 / 255 rows (the worst case of the vertical pass); 3: 0 / 255 columns."""
    H, W, Cn = shape
    if kind == 0:
        return rng.integers(0, 256, shape).astype(np.uint8)
    y, x = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    v = ((y + x) if kind == 1 else y if kind == 2 else x) % 2
    return np.repeat((255 * v)[..., None], Cn, axis=2).astype(np.uint8)


class Case:
    """One sample: input, output size, filters, region of interest ((y0, x0), (y1, x1)) with None for an axis without one, and what the
    planner must have made of it: path (1 = streamed) and any of info = (eligible, W, J, items) (None = not asserted)."""

    def __init__(self, img, out_hw, minf=LIN, magf=LNA, roi=None, path=1, info=(None, None, None, None), f64=True):
        self.img, self.out_hw, self.minf, self.magf, self.roi, self.path, self.info, self.f64 = img, out_hw, minf, magf, roi, path, info, f64

    def f64_roi(self):
        return None if self.roi is None else [None if self.roi[0][d] is None else (self.roi[0][d], self.roi[1][d]) for d in range(2)]


def _grid():
    import torch
    import conftest
    sms = 132 if conftest.DRY_RUN else torch.cuda.get_device_properties(0).multi_processor_count
    return 2 * sms                  # the streaming kernel's grid: two CTAs per SM


def setup_plan(cases, out_dtype, plan=None):
    import gpu_helpers as g
    n = len(cases)
    samples = (capi.ResampleSample * n)()
    for s, c in zip(samples, cases):
        g.fill_resample_sample(s, c.img.shape, c.out_hw, c.minf, c.magf, c.roi)
    plan = plan or capi.Plan("Resample", n)
    capi.check(capi.lib().dalib200ResamplePlanSetup(plan.handle, n, samples, capi.UINT8,
                                                    capi.UINT8 if np.dtype(out_dtype) == np.uint8 else capi.FLOAT))
    return plan, [capi.resample_stream_info(plan, i) for i in range(n)]


def run(cases, out_dtype, plan=None, what=""):
    """Sets up and launches one batch, asserts each case's path and stream info, then checks its output."""
    import torch
    import gpu_helpers as g
    plan, infos = setup_plan(cases, out_dtype, plan)
    din = g.to_dev([c.img for c in cases])
    tdt = torch.uint8 if np.dtype(out_dtype) == np.uint8 else torch.float32
    outs = [torch.empty((c.out_hw[0], c.out_hw[1], c.img.shape[2]), dtype=tdt, device="cuda") for c in cases]
    capi.check(capi.lib().dalib200ResampleLaunch(plan.handle, capi.ptr_array(din), capi.ptr_array(outs), capi.stream_handle()))
    torch.cuda.synchronize()
    paths = [capi.lib().dalib200ResamplePlanGetPath(plan.handle, i) for i in range(len(cases))]
    for i, (c, info, path) in enumerate(zip(cases, infos, paths)):
        tag = (what, i, c.img.shape, c.out_hw, c.minf, c.roi, np.dtype(out_dtype).name, info)
        assert path == c.path, ("path", tag, path)
        for k, want in enumerate(c.info):
            assert want is None or info[k] == want, ("stream info", k, tag)
    streamed = [info for info, p in zip(infos, paths) if p == 1]
    if streamed:
        wmax = max(2, max(info[1] for info in streamed))          # the kernel instance the launch picks
        COVER["W, WMAX"] |= {(info[1], wmax) for info in streamed}
        COVER["largest streamed J"] = max(COVER["largest streamed J"], max(info[2] for info in streamed))
        COVER["channels"] |= {c.img.shape[2] for c, p in zip(cases, paths) if p == 1}
        COVER["items per CTA"] = max(COVER["items per CTA"], sum(info[3] for info in streamed) / min(sum(info[3] for info in infos), _grid()))
    for i, (c, o) in enumerate(zip(cases, outs)):
        got = o.cpu().numpy()
        tag = (what, i, c.img.shape, c.out_hw, c.minf, c.roi, np.dtype(out_dtype).name)
        want = po.resample(c.img, c.out_hw, c.minf, c.magf, out_dtype, c.roi)
        assert np.array_equal(bits(got), bits(want)), ("bit-exact", tag, int((got != want).sum()))
        if c.f64:
            vals, b = F.resize(c.img, c.out_hw, c.f64_roi(), c.minf, c.magf)
            r = F.check_u8(got, vals, b, tag) if np.dtype(out_dtype) == np.uint8 else F.check(got, vals, b, tag)
            COVER["|GPU - float64| / bound"] = max(COVER["|GPU - float64| / bound"], r)
    return infos, paths


def items(out_h, strips=1):
    return -(-out_h // SEG) * strips


# ------------------------------------------------------------------------------------------------------------------------ cases
def test_chunk_and_segment_edges():
    """out_h = 49..57 (every residue mod 8), 111..113 and 224 from about 4 times as many rows: a last chunk of 1..8 rows, a last work item of
    one chunk or of one row."""
    rng = np.random.default_rng(301)
    for k, out_dt in enumerate((np.uint8, np.float32)):
        cases = [Case(_content(rng, (4 * oh + 7, 64, 3), (j + k) % 4), (oh, 40), info=(1, 3, None, items(oh)))
                 for j, oh in enumerate(list(range(49, 58)) + [111, 112, 113, 224])]
        run(cases, out_dt, what="chunk edges")


def _exact_linear_rows(in_h, out_h):
    """Source row of each output of linear resampling without antialias when in_h / out_h is a multiple of 1/8: the filter's anchor is 1 and
    its scale 1, so idx[t] = ceil(t s + s / 2 - 3 / 2) is exact in float32, as the planner computes it."""
    s = in_h / out_h
    return [int(np.ceil(t * s + s / 2 - 1.5)) for t in range(out_h)]


def _chunk_steps(iy, Sy):
    """J of every chunk of every work item (the chunking of the walk records)."""
    Js = []
    for o in range(0, len(iy), SEG):
        o1 = min(o + SEG, len(iy))
        for c0 in range(o, o1, CHUNK):
            cs = iy[o] if c0 == o else iy[c0 - 1] + Sy
            Js.append(iy[min(c0 + CHUNK, o1) - 1] + Sy - cs)
    return Js


def test_partial_ring_slots():
    """Scales 49/8, 50/8, 51/8 (linear, 2 taps): every chunk after the first of a work item walks 49, 50 or 51 rows, so consecutive chunks
    end with a ring slot of 1, 2 or 3 rows.  The same shapes with the triangular filter (W = 3) vary J from chunk to chunk."""
    rng = np.random.default_rng(302)
    cases = []
    for a in (49, 50, 51):
        Js = _chunk_steps(_exact_linear_rows(a * 15, 120), 2)
        assert {J % 4 for J in Js[1:7]} == {a % 4}, Js
        cases.append(Case(_content(rng, (a * 15, 64, 1), a % 4), (120, 64), LNA, LNA, info=(1, 1, max(Js), items(120))))
        cases.append(Case(_content(rng, (a * 15, 32, 3), a % 3), (120, 40), LIN, info=(1, 3, None, items(120))))
    for out_dt in (np.uint8, np.float32):
        run(cases, out_dt, what="partial slots")


def _find_J(filt, target, C=1, w=64):
    """(in_h, out_h) of a one-sample plan (vertical pass first, walkable) whose largest chunk walks exactly `target` source rows."""
    plan = capi.Plan("Resample", 1)
    for in_h in (1237, 1000, 1111, 853, 400):
        for out_h in range(in_h // 16, in_h // 4):
            _, (info,) = setup_plan([Case(np.zeros((in_h, w, C), np.uint8), (out_h, w // 2), filt, filt)], np.uint8, plan)
            if info[2] == target and info[1] > 0 and capi.lib().dalib200ResamplePlanGetOrder(plan.handle, 0) == 1:
                return in_h, out_h
    raise AssertionError(("no shape walks", target, "rows", filt))


def test_walk_limit():
    """Linear (2 taps, W = 1), triangular (W = 3) and Lanczos3 (6 taps, W = 1) with J = 96, 95 and 94 stream; J = 97 goes to the tile
    kernel in the same launch.  Lanczos3 with antialias spans more than 4 output rows per source row on every down-scale (W = 0): it never
    streams, which the last case asserts."""
    rng = np.random.default_rng(303)
    for filt in (LNA, LIN, L3):
        cases = []
        for k, J in enumerate((96, 95, 94, 97)):
            in_h, out_h = _find_J(filt, J)
            cases.append(Case(_content(rng, (in_h, 64, 1), k), (out_h, 32), filt, filt, path=int(J <= WALK_MAX),
                              info=(int(J <= WALK_MAX), None, J, items(out_h) if J <= WALK_MAX else 0)))
        run(cases, np.uint8 if filt != LIN else np.float32, what=("walk limit", filt))
    in_h, out_h = _find_J(L3, 96)
    run([Case(_content(rng, (in_h, 64, 1), 1), (out_h, 32), L3AA, L3AA, path=0, info=(0, 0, None, 0))], np.uint8, what="lanczos3 aa")


W_CASES = {1: ((735, 96, 1), (120, 64), LNA), 2: ((150, 96, 1), (100, 64), LNA), 3: ((700, 96, 3), (224, 48), LIN),
           4: ((150, 64, 3), (96, 48), L3)}


def test_every_walk_width():
    """W = 1, 2, 3, 4 alone (kernel instances WMAX = 2, 2, 3, 4), then W = 1 and W = 2 next to a W = 4 sample in one WMAX = 4 launch,
    where their unused slots stay closed; a cubic antialiased sample is the second W = 4 filter.  u8 and f32 outputs."""
    rng = np.random.default_rng(304)
    for out_dt in (np.uint8, np.float32):
        for W, (shape, hw, filt) in W_CASES.items():
            run([Case(_content(rng, shape, W % 4), hw, filt, filt, info=(1, W, None, None))], out_dt, what=("W alone", W))
        mix = [Case(_content(rng, W_CASES[W][0], k), W_CASES[W][1], W_CASES[W][2], W_CASES[W][2], info=(1, W, None, None))
               for k, W in enumerate((1, 4, 2, 1))]
        mix.append(Case(_content(rng, (300, 64, 3), 2), (60, 48), CUBAA, CUBAA, info=(1, 4, None, None)))
        run(mix, out_dt, what="W mixed")


def test_strip_geometry():
    """Channels 1, 2, 3, 4, 8 and 16; rows of exactly 2048 bytes (one strip per work item) and of 2064 (two strips); strips that start
    inside a 16-byte granule (3 channels, several strips); outputs 1 pixel wide."""
    rng = np.random.default_rng(305)
    cases = [Case(_content(rng, (500, w, Cn), Cn % 4), (90, w // 3), info=(1, 3, None, None)) for Cn, w in ((1, 640), (2, 320), (3, 640),
                                                                                                        (4, 160), (8, 80), (16, 40))]
    cases += [Case(_content(rng, (600, 2048, 1), 1), (100, 300), info=(1, 2, None, items(100, 1))),          # 2048 bytes
              Case(_content(rng, (600, 128, 16), 2), (100, 40), info=(1, 2, None, items(100, 1))),
              Case(_content(rng, (600, 1024, 2), 0), (100, 300), info=(1, 2, None, items(100, 1))),
              Case(_content(rng, (600, 688, 3), 3), (100, 300), info=(1, 2, None, items(100, 2))),          # 2064 bytes: two strips
              Case(_content(rng, (560, 1920, 3), 0), (112, 500), info=(1, None, None, None)),
              Case(_content(rng, (600, 1, 16), 1), (100, 1), info=(1, None, None, items(100, 1))),
              Case(_content(rng, (600, 16, 1), 0), (100, 1), info=(1, None, None, items(100, 1)))]
    for out_dt in (np.uint8, np.float32):
        run(cases, out_dt, what="strips")


def test_regions_of_interest_on_aligned_rows():
    """ROIs on a 700 x 1024 x 3 image (3072-byte rows): horizontal offset (the strips start inside the row), vertical offset, both, a flipped
    horizontal ROI (decreasing columns inside a strip: streams), a flipped vertical one (decreasing rows: the tile kernel), and ROIs reaching
    above and below the image, whose clamped border rows are walked once per tap."""
    rng = np.random.default_rng(306)
    rois = [(((None, 100.5), (None, 900.25)), 1), (((50.25, None), (600.5, None)), 1), (((50.25, 100.5), (600.5, 900.25)), 1),
            (((None, 900.25), (None, 100.5)), 1), (((600.5, None), (50.25, None)), 0), (((-20.5, None), (730.25, None)), 1),
            (((-40.0, 3.0), (600.0, 1021.5)), 1), (((300.0, 999.0), (710.5, 517.0)), 1)]
    cases = [Case(_content(rng, (700, 1024, 3), k % 4), (150, 200), roi=roi, path=p, info=(p, None, None, None))
             for k, (roi, p) in enumerate(rois)]
    for out_dt in (np.uint8, np.float32):
        run(cases, out_dt, what="rois")


def test_many_items_per_cta():
    """One launch with more than four work items per CTA: C2 images (1080 x 1920 -> 224 x 224) shuffled among the shapes above, so a CTA
    carries its ring and record-buffer phases from item to item across samples of every W and strip geometry.  Everything against the
    oracle, a subset against float64."""
    rng = np.random.default_rng(307)
    cases = [Case(_content(rng, (1080, 1920, 3), 0), (224, 224), f64=False) for _ in range(92)]
    for W, (shape, hw, filt) in W_CASES.items():
        cases.append(Case(_content(rng, shape, W % 4), hw, filt, filt, f64=False))
    cases += [Case(_content(rng, (600, 688, 3), 1), (100, 300), f64=False), Case(_content(rng, (500, 40, 16), 2), (90, 13), f64=False),
              Case(_content(rng, (700, 1024, 3), 3), (150, 200), roi=((-20.5, 900.25), (730.25, 100.5)), f64=False)]
    for c in rng.choice(len(cases), 6, replace=False):
        cases[c].f64 = True
    cases = [cases[i] for i in rng.permutation(len(cases))]
    infos, _ = run(cases, np.uint8, what="many items")
    total = sum(info[3] for info in infos)
    assert total > 4 * _grid(), (total, _grid())


def test_plan_reuse_with_changing_walk_records():
    """One plan set up in turn with batches whose walk records grow (J near 96, W = 4), shrink (one short output) and come back; two samples
    share a vertical axis (the same walk records) with different widths."""
    rng = np.random.default_rng(308)
    plan = capi.Plan("Resample", 4)
    shared = [Case(_content(rng, (600, 96, 1), 0), (100, 64)), Case(_content(rng, (600, 512, 3), 1), (100, 200))]
    in_h, out_h = _find_J(LNA, 96)
    grown = [Case(_content(rng, (in_h, 64, 1), 2), (out_h, 32), LNA, LNA, info=(1, 1, 96, None)),
             Case(_content(rng, (150, 64, 3), 3), (96, 48), L3, L3, info=(1, 4, None, None)), shared[1]]
    small = [Case(_content(rng, (64, 32, 1), 1), (9, 16))]
    for k, batch in enumerate((shared, grown, small, shared, grown)):
        run(batch, np.uint8, plan, what=("reuse", k))


# ------------------------------------------------------------------------------------------------------------------------ planar
def test_planar_walk_records():
    """resample_planar_kernel reads the same walk records: out_h at every residue mod 8, J = 96, W = 1..4 and odd image sizes, decoded from
    4:2:0 JPEGs straight into the resize; each output equals decode-then-resize bit for bit."""
    import cv2
    import gpu_helpers as g
    from test_gpu_fused import _enc, _fused
    s420 = cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420
    in_h96, out_h96 = _find_J(LNA, 96, C=3, w=96)
    groups = [(LIN, [((333, 517), (49 + k, 100)) for k in range(8)], 3),
              (LNA, [((735, 97), (120, 48)), ((151, 99), (100, 90)), ((in_h96, 96), (out_h96, 48))], None),
              (L3, [((151, 65), (96, 48)), ((150, 64), (96, 60))], 4)]
    for filt, shapes, W in groups:
        streams = [_enc(g.synth_image(h, w, 40 + k), 90, s420) for k, ((h, w), _) in enumerate(shapes)]
        hws = [hw for _, hw in shapes]
        infos = []
        outs, granted = _fused(streams, hws, filt=filt, infos=infos)
        assert all(granted), (filt, granted)
        for i, s in enumerate(streams):
            assert infos[i][0] == 1 and (W is None or infos[i][1] == W), (filt, i, infos[i])
            assert np.array_equal(outs[i], po.resample(po.jpeg_decode(s), hws[i], filt, filt)), (filt, shapes[i])
        if filt == LNA:
            assert sorted(info[1] for info in infos) == [1, 1, 2] and infos[2][2] == WALK_MAX, infos
