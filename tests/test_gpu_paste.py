"""fn.multi_paste and fn.paste on the H100, bit for bit against tests/paste_ref.py (and, where the reference is too slow at full size,
against torch slice assignments of the same rectangles, with a subset also checked against paste_ref):
  * 256 YOLO-style 4-tile mosaics of 1280 x 1280 x 3 from 640^2 uint8 inputs, centres drawn at random, and the same to FLOAT16;
  * 32 overlapping regions per sample over several type pairs; 3000 packed tiny samples; one output of more than 2^31 elements;
  * inputs and outputs at every byte offset; an output alone and inside a mixed batch; outputs in one sentinel-filled allocation checked
    for stray writes;
  * decode -> resize(640) -> multi_paste (in_ids from external_source) -> crop_mirror_normalize through DALIGenericIterator and through
    ops.MultiPaste; decode -> paste -> resize;
  * the refusals."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gpu_helpers as gh  # noqa: E402
import paste_ref as pr  # noqa: E402
from erase_ref import TYPES  # noqa: E402
from test_erase_cpu import data  # noqa: E402
from test_paste_cpu import ids_case  # noqa: E402

pytestmark = pytest.mark.gpu
P64 = C.POINTER(C.c_int64)


def region_arrays(args, n):
    av, ac, keep = (C.POINTER(C.c_double) * 6)(), (P64 * 6)(), []
    for a, name in enumerate(pr.ARGS):
        if name in args:
            rows = [np.asarray(v, np.float64).reshape(-1) for v in args[name]]
            vals, cnt = np.concatenate(rows + [np.zeros(1)]), np.array([len(r) for r in rows], np.int64)
            keep += [vals, cnt]
            av[a], ac[a] = vals.ctypes.data_as(C.POINTER(C.c_double)), cnt.ctypes.data_as(P64)
    return av, ac, keep


def setup(lib, plan, inputs_shapes, it, n, ninputs, args, in_ids, out_sizes, dtype):
    av, ac, _keep = region_arrays(args, n)
    shp = [e for s in inputs_shapes for e in s]
    ids = idc = None
    if in_ids is not None:
        flat = [int(v) for r in in_ids for v in r] or [0]
        ids, idc = (C.c_int32 * len(flat))(*flat), (C.c_int64 * n)(*[len(r) for r in in_ids])
    osz = (C.c_int64 * (2 * n))(*[v for s in out_sizes for v in s]) if out_sizes is not None else None
    oshapes = (C.c_int64 * (3 * n))()
    from dali_b200 import capi
    capi.check(lib.dalib200PasteSetup(plan, it, -1 if dtype is None else TYPES[np.dtype(dtype)], ninputs, n, (C.c_int * ninputs)(*[3] * ninputs),
                                      None, (C.c_int64 * len(shp))(*shp), ids, idc, av, ac, osz, (C.c_float * 1)(0.0), 1, oshapes))
    return [tuple(oshapes[3 * i:3 * i + 3]) for i in range(n)]


def capi_mp(inputs, args=None, in_ids=None, out_sizes=None, dtype=None, in_offsets=None, out_offsets=None, packed=False):
    """through the C-ABI: the inputs in one allocation at gh.byte_positions, the outputs in one sentinel-filled allocation"""
    from dali_b200 import capi
    lib = capi.lib()
    n, ninputs = len(inputs[0]), len(inputs)
    flat = [x for inp in inputs for x in inp]
    plan = C.c_void_p()
    capi.check(lib.dalib200PastePlanCreate(C.byref(plan), max(n, 1)))
    try:
        oshapes = setup(lib, plan, [x.shape for x in flat], TYPES[flat[0].dtype], n, ninputs, args or {}, in_ids, out_sizes, dtype)
        odt = np.dtype(dtype or flat[0].dtype)
        _dev, ip = gh.upload_slices(flat, in_offsets, packed)
        outs = gh.SentinelSlices([int(np.prod(s)) * odt.itemsize for s in oshapes], odt.itemsize, out_offsets, packed)
        capi.check(lib.dalib200PasteLaunch(plan, (C.c_void_p * len(ip))(*ip), (C.c_void_p * n)(*outs.ptrs), capi.stream_handle()))
        return [g.view(odt).reshape(s) for g, s in zip(outs.read("multi_paste"), oshapes)]
    finally:
        lib.dalib200PastePlanDestroy(plan)


def check(inputs, args=None, in_ids=None, out_sizes=None, dtype=None, **kw):
    args = args or {}
    got = capi_mp(inputs, args, in_ids, out_sizes, dtype, **kw)
    for i in range(len(inputs[0])):
        srcs = [inputs[0][j] for j in in_ids[i]] if in_ids is not None else [inp[i] for inp in inputs]
        hw = tuple(out_sizes[i]) if out_sizes is not None else inputs[0][0].shape[:2]
        want = pr.multi_paste_ref(srcs, hw, {k: v[i] for k, v in args.items()}, dtype or inputs[0][0].dtype, inputs[0][0].shape[2])
        assert got[i].tobytes() == want.tobytes(), (i, inputs[0][0].dtype, dtype)
    return got


def mosaic_args(rng, n, tile=640):
    """YOLO mosaic: a centre (yc, xc) in [tile / 2, 3 tile / 2); each of the four tiles fills its quadrant of the 2 tile canvas,
    clipped to the tile"""
    ids, ia, sh, oa = [], [], [], []
    s = 2 * tile
    for _ in range(n):
        yc, xc = int(rng.integers(tile // 2, 3 * tile // 2)), int(rng.integers(tile // 2, 3 * tile // 2))
        ids.append([int(v) for v in rng.integers(0, n, 4)])
        q_sh = [[min(yc, tile), min(xc, tile)], [min(yc, tile), min(s - xc, tile)], [min(s - yc, tile), min(xc, tile)],
                [min(s - yc, tile), min(s - xc, tile)]]
        q_oa = [[yc - q_sh[0][0], xc - q_sh[0][1]], [yc - q_sh[1][0], xc], [yc, xc - q_sh[2][1]], [yc, xc]]
        q_ia = [[tile - q_sh[0][0], tile - q_sh[0][1]], [tile - q_sh[1][0], 0], [0, tile - q_sh[2][1]], [0, 0]]
        sh.append(q_sh), oa.append(q_oa), ia.append(q_ia)
    return ids, {"in_anchors": ia, "shapes": sh, "out_anchors": oa}


def torch_mp(srcs, ids, args, out_hw, dtype):
    import torch
    outs = []
    for i, row in enumerate(ids):
        o = torch.zeros(out_hw + (srcs[0].shape[2],), dtype=dtype, device="cuda")
        for k, j in enumerate(row):
            (iy, ix), (h, w), (oy, ox) = (args[a][i][k] for a in ("in_anchors", "shapes", "out_anchors"))
            o[oy:oy + h, ox:ox + w] = srcs[j][iy:iy + h, ix:ix + w].to(dtype)
        outs.append(o)
    return outs


@pytest.mark.parametrize("dtype", ["uint8", "float16"])
def test_256_mosaics_of_1280_from_640_tiles(dtype):
    import torch
    from dali_b200 import capi
    if os.environ.get("DALIB200_DRYRUN"):
        pytest.skip("torch device buffers of 1.3 GB; the host side of this launch is the other tests'")
    lib = capi.lib()
    rng = np.random.default_rng(1)
    n = 256
    srcs = [(torch.arange(640 * 640 * 3, device="cuda", dtype=torch.int64).reshape(640, 640, 3) * (2 * i + 1) % 251).to(torch.uint8)
            for i in range(n)]
    ids, args = mosaic_args(rng, n)
    tdt = getattr(torch, dtype)
    esz = torch.empty(0, dtype=tdt).element_size()
    per = 1280 * 1280 * 3 * esz
    stride = per + 256                                                      # a sentinel gap behind every output
    buf = torch.full((n * stride,), 0xA5, dtype=torch.uint8, device="cuda")
    plan = C.c_void_p()
    capi.check(lib.dalib200PastePlanCreate(C.byref(plan), n))
    try:
        setup(lib, plan, [(640, 640, 3)] * n, 0, n, 1, args, ids, [(1280, 1280)] * n, None if dtype == "uint8" else np.float16)
        capi.check(lib.dalib200PasteLaunch(plan, (C.c_void_p * n)(*[s.data_ptr() for s in srcs]),
                                           (C.c_void_p * n)(*[buf.data_ptr() + i * stride for i in range(n)]), capi.stream_handle()))
        torch.cuda.synchronize()
    finally:
        lib.dalib200PastePlanDestroy(plan)
    view = buf.view(n, stride)
    assert bool((view[:, per:] == 0xA5).all()), "a write outside the outputs"
    got = [view[i, :per].view(tdt).view(1280, 1280, 3) for i in range(n)]
    want = torch_mp(srcs, ids, args, (1280, 1280), tdt)
    for i in range(n):
        assert torch.equal(got[i], want[i]), i
    for i in (0, 77, 255):                                                 # against the numpy statement
        ref = pr.multi_paste_ref([srcs[j].cpu().numpy() for j in ids[i]], (1280, 1280), {k: v[i] for k, v in args.items()}, np.dtype(dtype), 3)
        assert got[i].cpu().numpy().tobytes() == ref.tobytes(), i


def test_32_overlapping_regions_per_sample_and_type_pairs():
    rng = np.random.default_rng(2)
    for it, ot in ((np.uint8, None), (np.uint8, np.float16), (np.float32, None), (np.float32, np.uint8), (np.int16, np.float64),
                   (np.float64, np.int32), (np.bool_, np.float32)):
        batch = [data(rng, (int(rng.integers(100, 240)), int(rng.integers(100, 240)), 3), it) for _ in range(12)]
        ids, args = ids_case(rng, batch, 32, (300, 320))
        check([batch], args, ids, [(300, 320)] * 12, ot)


def test_3000_packed_tiny_samples_and_the_multi_input_form():
    rng = np.random.default_rng(3)
    tiny = [data(rng, (int(rng.integers(1, 9)), int(rng.integers(1, 9)), 3), np.uint8) for _ in range(3000)]
    ids, args = ids_case(rng, tiny, 2, (6, 7))
    check([tiny], args, ids, [(6, 7)] * 3000, packed=True)
    inputs = [[data(rng, (33, 47, 4), np.float32) for _ in range(5)] for _ in range(4)]
    check(inputs, out_offsets=[1 * 4, 2 * 4, 0, 3 * 4, 4])


def test_one_output_of_more_than_2_31_elements():
    import torch
    from dali_b200 import capi
    if os.environ.get("DALIB200_DRYRUN"):
        pytest.skip("3 GB of buffers; the host side of this launch is the other tests'")
    lib = capi.lib()
    src = (torch.arange(30000 * 30000, dtype=torch.int64, device="cuda") % 251).to(torch.uint8).reshape(30000, 30000, 1)
    out = torch.full((46400, 46400, 1), 0xA5, dtype=torch.uint8, device="cuda")   # 2 152 960 000 elements
    ids = [[0, 0, 0]]
    args = {"in_anchors": [[[0, 0], [100, 7], [29999, 0]]], "shapes": [[[30000, 30000], [29000, 29990], [1, 30000]]],
            "out_anchors": [[[0, 0], [17400, 16407], [46399, 16400]]]}
    plan = C.c_void_p()
    capi.check(lib.dalib200PastePlanCreate(C.byref(plan), 1))
    try:
        setup(lib, plan, [(30000, 30000, 1)], 0, 1, 1, args, ids, [(46400, 46400)], None)
        capi.check(lib.dalib200PasteLaunch(plan, (C.c_void_p * 1)(src.data_ptr()), (C.c_void_p * 1)(out.data_ptr()), capi.stream_handle()))
        torch.cuda.synchronize()
    finally:
        lib.dalib200PastePlanDestroy(plan)
    (want,) = torch_mp([src], ids, args, (46400, 46400), torch.uint8)
    assert torch.equal(out, want)


def test_every_byte_offset_and_batch_independence():
    rng = np.random.default_rng(4)
    for dt in (np.uint8, np.int16, np.float32, np.float64):
        batch = [data(rng, (37, 45, 3), dt) for _ in range(2)]
        ids, args = ids_case(rng, batch, 3, (40, 50))
        sz = np.dtype(dt).itemsize
        for o in range(0, 16, sz):
            for p in (o, (o + 5 * sz) % 16):
                check([batch], args, ids, [(40, 50)] * 2, in_offsets=[o, (o + sz) % 16], out_offsets=[p, (p + 3 * sz) % 16])
    one = [gh.synth_image(301, 455, 7), gh.synth_image(200, 300, 8)]
    ids1, args1 = ids_case(rng, one, 6, (350, 400))
    (alone, _) = capi_mp([one], args1, ids1, [(350, 400)] * 2)
    mixed = [data(rng, (3, 5, 3), np.uint8), one[0], np.zeros((0, 3, 3), np.uint8), rng.integers(0, 256, (640, 480, 3), dtype=np.uint8),
             one[1]]
    idsm, argsm = ids_case(rng, mixed, 4, (350, 400))
    idsm[1] = [1 if j == 0 else 4 for j in ids1[0]]
    for k in argsm:
        argsm[k][1] = args1[k][0]
    inmix = check([mixed], argsm, idsm, [(350, 400)] * 5, out_offsets=[1, 2, 3, 4, 5])
    assert alone.tobytes() == inmix[1].tobytes()


def test_mosaic_pipeline_through_the_iterator_and_the_ops_class():
    import cv2
    import nvidia.dali as dali
    from nvidia.dali import fn, ops, types
    from nvidia.dali.plugin.pytorch import DALIGenericIterator
    rng = np.random.default_rng(5)
    n = 8
    imgs = [gh.synth_image(int(rng.integers(300, 900)), int(rng.integers(300, 900)), k) for k in range(n)]
    streams = [np.frombuffer(cv2.imencode(".jpg", im)[1].tobytes(), np.uint8) for im in imgs]
    ids, args = mosaic_args(rng, n)
    col = lambda a: [np.array(v, np.int32) for v in a]  # noqa: E731
    paste_op = ops.MultiPaste(device="gpu", output_size=[1280, 1280])

    @dali.pipeline_def(batch_size=n, num_threads=2, device_id=0, prefetch_queue_depth=1)
    def pipe():
        img = fn.decoders.image(fn.external_source(source=lambda: streams), device="mixed")
        tiles = fn.resize(img, resize_x=640, resize_y=640)
        src = lambda v: fn.external_source(source=lambda: v)  # noqa: E731
        kw = dict(in_ids=src(col(ids)), in_anchors=src(col(args["in_anchors"])), shapes=src(col(args["shapes"])),
                  out_anchors=src(col(args["out_anchors"])))
        m = fn.multi_paste(tiles, output_size=[1280, 1280], **kw)
        m2 = paste_op(tiles, **kw)
        norm = fn.crop_mirror_normalize(m, dtype=types.FLOAT, output_layout="CHW", mean=[0.0] * 3, std=[255.0] * 3)
        return tiles, m, m2, norm
    it = DALIGenericIterator([pipe()], ["tiles", "m", "m2", "norm"], size=n)
    b = next(iter(it))[0]
    tiles = [b["tiles"][i].cpu().numpy() for i in range(n)]
    for i in range(n):
        want = pr.multi_paste_ref([tiles[j] for j in ids[i]], (1280, 1280), {k: v[i] for k, v in args.items()}, np.uint8, 3)
        assert b["m"][i].cpu().numpy().tobytes() == want.tobytes(), i
        assert b["m2"][i].cpu().numpy().tobytes() == want.tobytes(), i
        assert tuple(b["norm"][i].shape) == (3, 1280, 1280)


def test_paste_pipeline_decode_paste_resize():
    import cv2
    import nvidia.dali as dali
    from nvidia.dali import fn
    rng = np.random.default_rng(6)
    imgs = [gh.synth_image(300, 300, k) for k in range(6)] + [gh.synth_image(171, 233, 9)]
    streams = [np.frombuffer(cv2.imencode(".png", im)[1].tobytes(), np.uint8) for im in imgs]
    ratio = [np.float32(v) for v in rng.uniform(1.0, 4.0, len(imgs))]
    px = [np.float32(v) for v in rng.uniform(0, 1, len(imgs))]
    py = [np.float32(v) for v in rng.uniform(0, 1, len(imgs))]
    px[0], py[0], ratio[1], px[2], py[2] = 0.0, 1.0, 1.0, 1.0, 0.0

    @dali.pipeline_def(batch_size=len(imgs), num_threads=2, device_id=0, prefetch_queue_depth=1)
    def pipe():
        img = fn.decoders.image(fn.external_source(source=lambda: streams), device="mixed")
        src = lambda v: fn.external_source(source=lambda: [np.array(x, np.float32) for x in v])  # noqa: E731
        z = fn.paste(img, ratio=src(ratio), paste_x=src(px), paste_y=src(py), fill_value=[123, 117, 104], min_canvas_size=350.0)
        return img, z, fn.resize(z, resize_x=300, resize_y=300)
    p = pipe()
    p.build()
    img, z, r = p.run()
    assert z.layout() == "HWC"
    for i in range(len(imgs)):
        want = pr.paste_ref(img.as_cpu()[i], ratio[i], px[i], py[i], 350.0, (123, 117, 104))
        assert z.as_cpu()[i].tobytes() == want.tobytes(), i
        assert r.as_cpu()[i].shape == (300, 300, 3)


def test_refusals_name_the_problem():
    import nvidia.dali as dali
    from nvidia.dali import fn

    def run(xs, op="multi_paste", layout=None, **kw):
        @dali.pipeline_def(batch_size=len(xs), num_threads=1, device_id=0, prefetch_queue_depth=1)
        def pipe():
            return getattr(fn, op)(fn.external_source(source=lambda: xs, device="gpu", layout=layout), **kw)
        p = pipe()
        p.build()
        return p.run()
    x = [np.zeros((4, 5, 3), np.uint8)] * 2
    with pytest.raises(Exception, match='input 0 has layout "CHW"'):
        run(x, layout="CHW")
    with pytest.raises(Exception, match="in_ids 5 is not a sample of the batch of 2"):
        run(x, layout="HWC", in_ids=[0, 5])
    with pytest.raises(Exception, match="both out_anchors and out_anchors_rel are given"):
        run(x, layout="HWC", in_ids=[0], out_anchors=[0, 0], out_anchors_rel=[0.0, 0.0])
    with pytest.raises(Exception, match="leave the output"):
        run(x, layout="HWC", in_ids=[0], out_anchors=[1, 0])
    with pytest.raises(Exception, match="sample 0: ratio 0.5 is less than 1"):
        run(x, "paste", "HWC", ratio=0.5)
    (o,) = run([np.full((4, 5, 3), 10, np.uint8)] * 2, "multi_paste", "HWC", in_ids=[1, 0], out_anchors=[0, 0, 2, 3],
               shapes=[2, 2, 2, 2], output_size=[6, 7])
    want = np.zeros((6, 7, 3), np.uint8)
    want[0:2, 0:2] = 10
    want[2:4, 3:5] = 10
    assert np.array_equal(o.as_cpu()[0], want)
