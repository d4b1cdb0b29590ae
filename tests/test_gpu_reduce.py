"""fn.reductions.* on the H100, through pipeline_def / fn.* / ops.* and through the C-ABI, against tests/reduce_ref.py (the float
bound takes the depth of each sample's accumulation tree from dalib200ReducePlanGetPaths):
  * every operator and type; ranks 0-6 with axis subsets, negative axes, axis_names and keep_dims; unit and zero extents; shapes that
    differ per sample; each path on both sides of its threshold;
  * 256 x 1080p x 3 uint8 per-channel mean; 3000 tiny samples; one uint8 sample of more than 2^31 elements;
  * a sample alone and inside a mixed batch, and a repeated run: bit-identical, and within the bound of the reference;
  * per-image standardisation (x - mean) / std_dev through pipeline_def against float64; 0-d outputs through DALIGenericIterator;
  * outputs written into one sentinel-filled allocation, checked for stray writes."""
import ctypes as C
import itertools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import reduce_ref as rr  # noqa: E402

pytestmark = pytest.mark.gpu
FN = ["min", "max", "sum", "mean", "mean_square", "rms", "std_dev", "variance"]


_data = rr.random_data


def depths(op, xs, axes, keep_dims=False, dtype=None):
    """the planner's depth for each sample (host-side plan set-up only)"""
    from dali_b200 import capi
    lib = capi.lib()
    n, nd = len(xs), xs[0].ndim
    mask = sum(1 << a for a in (rr._axes(xs[0], axes) if nd else ()))
    plan = C.c_void_p()
    capi.check(lib.dalib200ReducePlanCreate(C.byref(plan), max(n, 1)))
    try:
        shp = (C.c_int64 * max(1, n * nd))(*[e for x in xs for e in x.shape])
        osh = (C.c_int64 * max(1, n * nd))()
        ot = C.c_int32(-1 if dtype is None else dtype)
        capi.check(lib.dalib200ReduceSetup(plan, op, rr.CODE[xs[0].dtype], C.byref(ot), n, nd, shp, C.c_uint32(mask), int(keep_dims), 0, osh))
        kinds, dep = (C.c_int32 * (3 * n))(), (C.c_int32 * n)()
        capi.check(lib.dalib200ReducePlanGetPaths(plan, kinds, dep, n))
        return list(dep), [list(kinds[3 * i:3 * i + 3]) for i in range(n)]
    finally:
        lib.dalib200ReducePlanDestroy(plan)


def _run(build, batches, layout=None, batch_size=None):
    import nvidia.dali as dali
    from nvidia.dali import fn
    state = {}

    @dali.pipeline_def(batch_size=batch_size or max(len(b) for b in batches), num_threads=1, device_id=0, prefetch_queue_depth=1)
    def pipe():
        return build(fn.external_source(source=lambda: state["b"], device="gpu", layout=layout))
    p = pipe()
    p.build()
    res = []
    for b in batches:
        state["b"] = b
        outs = p.run()
        outs = outs if isinstance(outs, (tuple, list)) else (outs,)
        res.append([(o.as_cpu(), o.layout()) for o in outs])
    return res


def _means(xs, axes, keep_dims):
    out = []
    for x in xs:
        ax = rr._axes(x, axes) if x.ndim else ()
        out.append(np.mean(x.astype(np.float64), axis=ax, keepdims=keep_dims).astype(np.float32))
    return out


def check_fn(op, xs, axes=None, keep_dims=False, dtype=None, layout=None, what=""):
    from nvidia.dali import fn
    kw = {} if axes is None else {"axes": list(axes)}
    if dtype is not None:
        kw["dtype"] = dtype
    f = getattr(fn.reductions, FN[op])
    dep, kinds = depths(op, xs, axes, keep_dims, dtype)
    if op in (rr.STD_DEV, rr.VARIANCE):
        import nvidia.dali as dali
        means = _means(xs, axes, keep_dims)
        state = {"m": means}

        def build(x):
            m = fn.external_source(source=lambda: state["m"], device="gpu")
            return f(x, m, keep_dims=keep_dims, **kw)
    else:
        means = None

        def build(x):
            return f(x, keep_dims=keep_dims, **kw)
    ((outs,),) = _run(build, [xs], layout)
    got, lay = outs
    for i, x in enumerate(xs):
        want, tol = rr.reference(op, x, (rr._axes(x, axes) if x.ndim else None), keep_dims, dtype, 0,
                                 None if means is None else means[i], dep[i])
        rr.check(got[i], np.asarray(want), tol, (what, FN[op], x.dtype, x.shape, axes))
    return lay, kinds


def test_every_operator_and_type():
    rng = np.random.default_rng(1)
    for op in range(8):
        for t in rr.TYPES:
            xs = [_data((7, 9, 3), t, rng), _data((1, 300, 3), t, rng), _data((50, 1, 2), t, rng)]
            for axes in (None, (0, 1), (-1,)):
                check_fn(op, xs, axes, keep_dims=bool(rng.integers(0, 2)), what="types")


def test_ranks_axes_names_keep_dims_and_extents():
    rng = np.random.default_rng(2)
    for rank in range(7):
        big = {0: 1, 1: 5000, 2: 90, 3: 20, 4: 8}.get(rank, 5)
        subsets = [c for k in range(rank + 1) for c in itertools.combinations(range(rank), k)]
        subsets = subsets[::max(1, len(subsets) // 8)] + [tuple(range(rank))]
        for j, sub in enumerate(subsets):
            shapes = [tuple(int(v) for v in rng.integers(1, big + 1, rank)) for _ in range(2)]
            shapes.append(tuple(1 if a % 2 else int(rng.integers(1, big + 1)) for a in range(rank)))
            op = [rr.SUM, rr.MEAN, rr.MAX, rr.STD_DEV, rr.RMS][j % 5]
            t = [np.int16, np.float32, np.uint8, np.float32, np.int32][j % 5]
            check_fn(op, [_data(s, t, rng) for s in shapes], sub if rank else None, keep_dims=bool(j % 2), what=("rank", rank))
    from nvidia.dali import fn
    xs = [_data((4, 5, 3), np.uint8, rng), _data((6, 2, 3), np.uint8, rng)]
    ((a, b, c),) = _run(lambda x: (fn.reductions.mean(x, axis_names="HW"), fn.reductions.sum(x, axes=[-1], keep_dims=True),
                                  fn.reductions.max(x, axis_names="C")), [xs], layout="HWC")
    assert (a[1], b[1], c[1]) == ("C", "HWC", "HW")
    for i, x in enumerate(xs):
        assert np.array_equal(a[0][i], (x.astype(np.int64).sum((0, 1)) / (x.shape[0] * x.shape[1])).astype(np.float32))
        assert np.array_equal(b[0][i], x.astype(np.uint64).sum(2, keepdims=True))
        assert np.array_equal(c[0][i], x.max(2))
    zs = [np.zeros((4, 0, 3), np.float32), _data((4, 5, 3), np.float32, rng), np.zeros((0, 5, 3), np.float32)]
    for op in (rr.SUM, rr.MEAN, rr.RMS):
        check_fn(op, zs, (1,), keep_dims=True, what="zero extents")


def test_paths_on_both_sides_of_each_threshold():
    rng = np.random.default_rng(3)
    cases = [((40, 32), (0,), 0), ((200, 31), (0,), 1), ((66, 31), (0,), 0), ((2048,), None, 1), ((256, 40), (0,), 0),
             ((257, 40), (0,), 2), ((32768,), None, 1), ((32769,), None, 2), ((10923, 3), (0,), 2), ((10922, 3), (0,), 1)]
    for shape, axes, kind in cases:
        for t in (np.uint8, np.float32, np.int64):
            for op in (rr.SUM, rr.MEAN, rr.MIN, rr.STD_DEV):
                _, kinds = check_fn(op, [_data(shape, t, rng)], axes, what=("path", shape))
                assert kinds[0][0] == kind, (shape, kinds)


def test_dtypes_and_nan():
    rng = np.random.default_rng(4)
    xs = [_data((40, 50), np.uint8, rng), _data((3, 700), np.uint8, rng)]
    for d in range(11):
        check_fn(rr.SUM, xs, (1,), dtype=d, what="sum dtype")
    for op in (rr.MEAN, rr.MEAN_SQUARE, rr.RMS):
        for d in (rr.F16, rr.F32, rr.F64):
            check_fn(op, [_data((40, 50), np.int16, rng)], (0,), dtype=d, what="mean dtype")
    x = np.arange(5000, dtype=np.float32).reshape(50, 100)
    x[17, 33] = np.nan
    for op in (rr.MIN, rr.MAX):
        for axes in (None, (0,), (1,)):
            check_fn(op, [x, x[:, :7].copy()], axes, what="nan")


def test_per_channel_mean_of_256_1080p_images_and_determinism():
    from nvidia.dali import fn
    rng = np.random.default_rng(5)
    imgs = [rng.integers(0, 256, (1080, 1920, 3), dtype=np.uint8) for _ in range(8)]
    batch = [imgs[i % 8] for i in range(256)]
    ((m,),) = _run(lambda x: fn.reductions.mean(x, axes=[0, 1]), [batch], layout="HWC")
    for i in range(8):
        want = (imgs[i].astype(np.int64).sum((0, 1)) / (1080 * 1920)).astype(np.float32)
        assert np.array_equal(m[0][i], want) and np.array_equal(m[0][i + 8], want)
    # a float sample alone, inside a mixed batch and run twice: bit-identical
    f = [(rng.standard_normal((1080, 1920, 3)) * 50).astype(np.float32), (rng.standard_normal((300, 17, 3))).astype(np.float32)]
    mixed = [f[1], f[0], _data((5, 5, 3), np.float32, rng), f[0]]
    def build(x):
        m = fn.reductions.mean(x, axes=[0, 1], keep_dims=True)
        return fn.reductions.sum(x), fn.reductions.std_dev(x, m, axes=[0, 1]), m
    alone, again = _run(build, [[f[0]], [f[0]]], batch_size=4)
    (inmix,) = _run(build, [mixed])
    for k in range(3):
        a = alone[k][0][0]
        assert a.tobytes() == again[k][0][0].tobytes() == inmix[k][0][1].tobytes() == inmix[k][0][3].tobytes()
    # and each of them within the bound of its accumulation tree (tests/test_gpu_reduce_exact.py pins them bit for bit)
    s, sd, m = (alone[k][0][0] for k in range(3))
    for op, got, axes, keep, mean in ((rr.SUM, s, None, False, None), (rr.MEAN, m, (0, 1), True, None), (rr.STD_DEV, sd, (0, 1), False, m)):
        dep, _ = depths(op, [f[0]], axes, keep)
        want, tol = rr.reference(op, f[0], axes, keep, mean=mean, depth=dep[0])
        rr.check(got, np.asarray(want), tol, ("1080p", rr.NAMES[op]))


def test_3000_tiny_samples():
    from nvidia.dali import fn
    rng = np.random.default_rng(6)
    xs = [_data((int(rng.integers(0, 4)), int(rng.integers(1, 5)), 3), np.float32, rng) for _ in range(3000)]
    ((s, m),) = _run(lambda x: (fn.reductions.sum(x, axes=[0, 1]), fn.reductions.max(x, axes=[2])), [xs])
    dep, _ = depths(rr.SUM, xs, (0, 1))
    for i, x in enumerate(xs):
        want, tol = rr.reference(rr.SUM, x, (0, 1), depth=dep[i])
        rr.check(s[0][i], want, tol, i)
        assert np.array_equal(m[0][i], x.max(2))


def test_per_image_standardisation_and_0d_outputs_through_the_iterator():
    import nvidia.dali as dali
    from nvidia.dali import fn, types
    from nvidia.dali.plugin.pytorch import DALIGenericIterator
    rng = np.random.default_rng(7)
    data = [rng.integers(0, 256, (64, 48, 3), dtype=np.uint8) for _ in range(4)]

    @dali.pipeline_def(batch_size=4, num_threads=1, device_id=0)
    def pipe():
        x = fn.cast(fn.external_source(source=lambda: data, device="gpu", layout="HWC"), dtype=types.FLOAT)
        m = fn.reductions.mean(x, axes=(0, 1), keep_dims=True)
        s = fn.reductions.std_dev(x, m, axes=(0, 1), keep_dims=True)
        return (x - m) / s, fn.reductions.sum(x), fn.reductions.max(x)
    it = DALIGenericIterator([pipe()], ["y", "total", "peak"], size=4)
    b = next(iter(it))[0]
    assert tuple(b["total"].shape) == (4,) and tuple(b["peak"].shape) == (4,)
    y = b["y"].cpu().numpy()
    for i, x in enumerate(data):
        x64 = x.astype(np.float64)
        mu = x64.mean((0, 1), keepdims=True)
        sd = np.sqrt(((x64 - mu) ** 2).mean((0, 1), keepdims=True))
        assert np.allclose(y[i], (x64 - mu) / sd, rtol=0, atol=1e-4), i
        assert float(b["total"][i]) == float(x64.sum()) and float(b["peak"][i]) == float(x.max())


def test_legacy_ops_class():
    import nvidia.dali as dali
    from nvidia.dali import fn, ops
    x = [np.arange(24, dtype=np.int32).reshape(2, 3, 4)] * 2
    red = ops.reductions.Sum(device="gpu", axes=[1])

    @dali.pipeline_def(batch_size=2, num_threads=1, device_id=0)
    def pipe():
        return red(fn.external_source(source=lambda: x, device="gpu"))
    p = pipe()
    p.build()
    (o,) = p.run()
    assert np.array_equal(o.as_cpu()[1], x[1].astype(np.int64).sum(1))


def test_c_abi_sentinel_fill_and_sample_larger_than_2_pow_31():
    import torch
    from dali_b200 import capi
    lib = capi.lib()
    rng = np.random.default_rng(8)
    plan = C.c_void_p()
    capi.check(lib.dalib200ReducePlanCreate(C.byref(plan), 4))
    try:
        # four samples packed into one sentinel-filled allocation, outputs into another
        shapes = [(33, 17, 3), (2, 4000), (1, 1, 1), (70, 2, 9)]
        xs = [_data(s, np.float32, rng) for s in shapes]
        src = torch.from_numpy(np.concatenate([x.ravel() for x in xs])).cuda()
        offs = np.cumsum([0] + [x.size for x in xs])
        dst = torch.tensor(np.full(4096, -7.0, np.float32), device="cuda")
        mask = 0b1                                                   # axis 0 of each sample, viewed as 2-D
        xs3 = [x.reshape(x.shape[0], -1) for x in xs]
        shp = (C.c_int64 * 8)(*[e for x in xs3 for e in x.shape])
        osh = (C.c_int64 * 4)()
        ot = C.c_int32(-1)
        capi.check(lib.dalib200ReduceSetup(plan, rr.MEAN, 9, C.byref(ot), 4, 2, shp, C.c_uint32(mask), 0, 0, osh))
        oofs = np.cumsum([0] + [x.shape[1] + 5 for x in xs3])
        ip = (C.c_void_p * 4)(*[src.data_ptr() + 4 * int(o) for o in offs[:4]])
        op = (C.c_void_p * 4)(*[dst.data_ptr() + 4 * int(o) for o in oofs[:4]])
        capi.check(lib.dalib200ReduceLaunch(plan, ip, None, op, capi.stream_handle()))
        torch.cuda.synchronize()
        got = dst.cpu().numpy()
        dep, _ = depths(rr.MEAN, xs3, (0,))
        for i, x in enumerate(xs3):
            want, tol = rr.reference(rr.MEAN, x, (0,), depth=dep[i])
            rr.check(got[oofs[i]:oofs[i] + x.shape[1]], want, tol, i)
            assert np.all(got[oofs[i] + x.shape[1]:oofs[i + 1]] == -7.0), "a write outside the output"
        assert np.all(got[oofs[4]:] == -7.0)
        if os.environ.get("DALIB200_DRYRUN"):
            return
        # one uint8 sample of 2^31 + 2^20 + 3 elements: per-channel sum and max, and the sum of all
        n = (1 << 31) + (1 << 20) + 3
        big = torch.empty(n, dtype=torch.uint8, device="cuda")
        big.copy_(torch.arange(251, dtype=torch.uint8, device="cuda").repeat(n // 251 + 1)[:n])
        out = torch.zeros(2, dtype=torch.int64, device="cuda")
        shp1 = (C.c_int64 * 1)(n)
        o1 = (C.c_int64 * 1)()
        for k, op_ in enumerate((rr.SUM, rr.MAX)):
            ot = C.c_int32(7 if op_ == rr.SUM else -1)
            capi.check(lib.dalib200ReduceSetup(plan, op_, 0, C.byref(ot), 1, 1, shp1, C.c_uint32(1), 0, 0, o1))
            capi.check(lib.dalib200ReduceLaunch(plan, (C.c_void_p * 1)(big.data_ptr()), None,
                                                (C.c_void_p * 1)(out.data_ptr() + 8 * k), capi.stream_handle()))
        torch.cuda.synchronize()
        full, rem = divmod(n, 251)
        want = full * (250 * 251 // 2) + rem * (rem - 1) // 2
        s, mx = out.cpu().tolist()
        del big
        torch.cuda.empty_cache()
        assert s == want and (mx & 0xFF) == 250, (s, want, mx)
    finally:
        lib.dalib200ReducePlanDestroy(plan)


def test_refusals_name_the_problem():
    from nvidia.dali import fn
    x = [np.zeros((2, 3, 4), np.uint8)] * 2
    with pytest.raises(Exception, match=r"axis 3 is out of range \[-3, 2\]"):
        _run(lambda a: fn.reductions.sum(a, axes=[3]), [x])
    with pytest.raises(Exception, match="mutually exclusive"):
        _run(lambda a: fn.reductions.sum(a, axes=[0], axis_names="H"), [x], layout="HWC")
    with pytest.raises(Exception, match="BOOL input is not supported"):
        _run(lambda a: fn.reductions.sum(a), [[np.zeros((2, 3), np.bool_)] * 2])
    with pytest.raises(Exception, match="the reduced axes are empty"):
        _run(lambda a: fn.reductions.min(a, axes=[1]), [[np.zeros((2, 0), np.uint8)] * 2])
    with pytest.raises(Exception, match=r"sample 0 of input 1 \(the mean\) has shape"):
        _run(lambda a: fn.reductions.std_dev(a, fn.reductions.mean(a, axes=[0]), axes=[1]), [[np.zeros((2, 3), np.float32)] * 2])
