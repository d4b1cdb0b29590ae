"""fn.reductions.* on the H100, bit for bit, through the C-ABI:
  * exact-sum inputs (tests/reduce_ref.py exact_data: every partial sum exact in any order) against exact_reference, byte for byte:
    every operator, type and dtype, std_dev / variance with ddof 0 and 1 fed integer channel centres as their mean;
  * the device against the host build of the same planner and bodies (tools/emul/reduce_emul.cc through tests/reduce_host.py) on
    random data, byte for byte: the device adds in the order the planner states, as the host build does;
  * inputs, means and outputs as slices of single allocations at every element offset of 1-, 2-, 4- and 8-byte types, for narrow
    channel counts and the columns / inner / split shapes, with the bytes around every output checked against a sentinel fill;
  * 3000 packed samples of every path kind with empty ones among them; a plan reused across split and unsplit batches and a batch
    that grows its scratch; per-channel mean / std_dev of 1080p x 3, std_dev over HW of 224^2 x 3, max / mean over t of 513 x 626."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gpu_helpers as gh  # noqa: E402
import reduce_host as rh  # noqa: E402
import reduce_ref as rr  # noqa: E402

pytestmark = pytest.mark.gpu
COLUMNS, INNER, SPLIT = 0, 1, 2
NARROW = [(max(2048 // i + 5, 70), i) for i in (1, 3, 4, 5, 7, 16, 31)]     # inner path, one channel slot per i
EVERY_SIZE = [np.uint8, np.int8, np.uint16, np.int16, np.float16, np.uint32, np.int32, np.float32, np.uint64, np.int64, np.float64]


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    lib = rh.build(tmp_path_factory.mktemp("reduce"))
    if lib is None:
        pytest.skip("needs g++")
    return lib


class Plan:
    def __init__(self, n):
        from dali_b200 import capi
        self.lib, self.capi = capi.lib(), capi
        self.h = C.c_void_p()
        capi.check(self.lib.dalib200ReducePlanCreate(C.byref(self.h), max(n, 1)))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.lib.dalib200ReducePlanDestroy(self.h)
        return False


def _offsets(arrays, off, step):
    return [((off + step * i) % (16 // a.itemsize)) * a.itemsize for i, a in enumerate(arrays)]


def run_dev(plan, op, xs, axes=None, keep_dims=False, dtype=None, ddof=0, means=None, off=0, moff=0, ooff=0, packed=False):
    """one batch on the device with the same placement as reduce_host.run (or packed back to back): (outputs, kinds, depths)"""
    lib, capi = plan.lib, plan.capi
    n, nd = len(xs), xs[0].ndim
    mask = sum(1 << a for a in (rr._axes(xs[0], axes) if nd else ()))
    ond = nd if keep_dims else nd - bin(mask).count("1")
    shp = (C.c_int64 * max(1, n * nd))(*[e for x in xs for e in x.shape])
    osh = (C.c_int64 * max(1, n * ond))()
    ot = C.c_int32(-1 if dtype is None else dtype)
    capi.check(lib.dalib200ReduceSetup(plan.h, op, rr.CODE[xs[0].dtype], C.byref(ot), n, nd, shp, C.c_uint32(mask), int(keep_dims), ddof, osh))
    ots = np.dtype(rr.TYPES[ot.value])
    oshapes = [tuple(osh[i * ond + a] for a in range(ond)) for i in range(n)]
    _keep_in, ip = gh.upload_slices(xs, None if packed else _offsets(xs, off, 3), packed)
    mp, _keep_m = None, None
    if means is not None:
        ms = [np.asarray(m, np.float32) for m in means]
        _keep_m, mps = gh.upload_slices(ms, None if packed else [((moff + i) % 4) * 4 for i in range(n)], packed)
        mp = (C.c_void_p * n)(*mps)
    sizes = [int(np.prod(s, dtype=np.int64)) * ots.itemsize for s in oshapes]
    outs = gh.SentinelSlices(sizes, ots.itemsize, None if packed else [((ooff + i) % (16 // ots.itemsize)) * ots.itemsize for i in range(n)],
                             packed)
    capi.check(lib.dalib200ReduceLaunch(plan.h, (C.c_void_p * n)(*ip), mp, (C.c_void_p * n)(*outs.ptrs), capi.stream_handle()))
    got = [b.view(ots).reshape(s) for b, s in zip(outs.read((rr.NAMES[op], n)), oshapes)]
    kinds, dep = (C.c_int32 * (3 * n))(), (C.c_int32 * n)()
    capi.check(lib.dalib200ReducePlanGetPaths(plan.h, kinds, dep, n))
    return got, [list(kinds[3 * i:3 * i + 3]) for i in range(n)], list(dep)


def check_exact(plan, op, xs, cs, axes, keep_dims=False, off=0, packed=False, what="", **kw):
    """a batch of exact_data against exact_reference, byte for byte; returns the kinds"""
    means = [rr.exact_mean(c, x, axes, keep_dims) for x, c in zip(xs, cs)] if op in (rr.STD_DEV, rr.VARIANCE) else None
    got, kinds, _ = run_dev(plan, op, xs, axes, keep_dims, means=means, off=off, moff=off, ooff=off, packed=packed, **kw)
    for i, x in enumerate(xs):
        want = rr.exact_reference(op, x, axes, keep_dims, mean=None if means is None else means[i], **kw)
        rr.same_bytes(got[i], want, (what, rr.NAMES[op], kw, x.dtype, x.shape, axes, off, i))
    return kinds


# ---- A: exact-sum inputs
def test_exact_sums_bit_for_bit():
    rng = np.random.default_rng(11)
    with Plan(16) as plan:
        for what, types, ops, shapes, ch, axes, keep in rr.exact_cases(rng):
            for t in types:
                xs, cs = rr.exact_batch(rng, t, shapes, ch, axes)
                for op in ops:
                    for kw in rr.VARIANTS.get(op, [{}]):
                        check_exact(plan, op, xs, cs, axes, keep, off=int(rng.integers(0, 16)), what=what, **kw)


# ---- B: the device against the host build
_data = rr.random_data


def _same_as_host(host, plan, op, xs, axes, keep_dims=False, off=0, what="", **kw):
    means = None
    if op in (rr.STD_DEV, rr.VARIANCE):
        means = [np.mean(x.astype(np.float64), axis=rr._axes(x, axes), keepdims=keep_dims).astype(np.float32) for x in xs]
    want, hkinds, _ = rh.run(host, op, xs, axes, keep_dims, means=means, off=off, moff=off, ooff=off, **kw)
    assert want is not None, (what, hkinds)
    got, kinds, _ = run_dev(plan, op, xs, axes, keep_dims, means=means, off=off, moff=off, ooff=off, **kw)
    assert kinds == hkinds, (what, kinds, hkinds)
    for i, x in enumerate(xs):
        rr.same_bytes(got[i], want[i], (what, rr.NAMES[op], kw, x.dtype, x.shape, axes, off, i))
    return kinds


def test_device_adds_in_the_order_of_the_host_build(host):
    rng = np.random.default_rng(12)
    with Plan(16) as plan:
        seen = set()
        for t in rr.TYPES:
            xs = [_data(s, t, rng) for s in rr.PATH_SHAPES]                 # columns, inner and split, I = 1 among them
            for op in range(8):
                for kw in rr.VARIANTS.get(op, [{}]):
                    kinds = _same_as_host(host, plan, op, xs, (0,), off=int(rng.integers(1, 16)), what="paths", **kw)
                    seen.update(k[0] for k in kinds)
        assert seen == {COLUMNS, INNER, SPLIT}, seen
        # three passes, the first of them split; a split inner pass reduced again; per-channel HWC
        for shapes, axes, ts in (([(3, 2, 5, 4, 600, 2), (2, 3, 2, 1, 3000, 3)], (0, 2, 4), (np.float32, np.float16, np.uint8)),
                                 ([(3, 40000, 2)], (0, 1), (np.float32, np.float64)),
                                 ([(300, 200, 3), (37, 41, 3)], (0, 1), (np.float32, np.int16))):
            for t in ts:
                xs = [_data(s, t, rng) for s in shapes]
                for op in range(8):
                    kinds = _same_as_host(host, plan, op, xs, axes, keep_dims=bool(op % 2), off=int(rng.integers(1, 16)), what=shapes)
                    if len(shapes[0]) == 6:
                        assert kinds[0] == [SPLIT, COLUMNS, COLUMNS], kinds


# ---- C: alignment, packing and batch edges
def test_every_element_offset_of_inputs_means_and_outputs():
    rng = np.random.default_rng(13)
    shapes = NARROW + rr.PATH_SHAPES
    with Plan(len(shapes)) as plan:
        for t in EVERY_SIZE:
            xs, cs = rr.exact_batch(rng, t, shapes, 1, (0,))
            for off in range(16 // np.dtype(t).itemsize):
                for op in range(8):
                    check_exact(plan, op, xs, cs, (0,), off=off, what=("offset", off))


def test_3000_packed_samples_of_every_path():
    rng = np.random.default_rng(14)
    shapes = []
    for k in range(3000):
        if k in (0, 2999) or k % 97 == 0:
            shapes.append((0, 3) if k % 2 else (5, 0))                      # an empty reduction, an empty output
        elif k % 53 == 0:
            shapes.append((300, 40) if k % 2 else (33000 // 3 + 7, 3))      # split columns, split inner
        elif k % 3 == 0:
            i = int(rng.integers(1, 32))
            shapes.append((2048 // i + int(rng.integers(0, 64)), i))         # inner
        else:
            shapes.append((int(rng.integers(1, 40)), int(rng.integers(1, 70))))   # columns
    with Plan(3000) as plan:
        for t in (np.float32, np.uint8):
            xs, cs = rr.exact_batch(rng, t, shapes, 1, (0,))
            for op in (rr.SUM, rr.MEAN, rr.MEAN_SQUARE, rr.STD_DEV):
                kinds = check_exact(plan, op, xs, cs, (0,), packed=True, what="packed")
                assert {k[0] for k in kinds} == {-1, COLUMNS, INNER, SPLIT}, sorted({k[0] for k in kinds})


def test_plan_reused_across_split_unsplit_and_growing_batches():
    rng = np.random.default_rng(15)
    batches = [([(32769, 1), (257, 40), (1000, 3)], [SPLIT, SPLIT, INNER]),
               ([(32768, 1), (256, 40), (1000, 3)], [INNER, COLUMNS, INNER]),    # unsplit: no partial of the last batch may leak in
               ([(32769, 1), (257, 40), (1000, 3)], [SPLIT, SPLIT, INNER]),
               ([(5 * 32768 + 1, 1), (2000, 40), (40000, 3)], [SPLIT, SPLIT, SPLIT])]   # more partials: the scratch grows
    with Plan(3) as plan:
        for op in (rr.SUM, rr.STD_DEV, rr.MAX):
            for b, (shapes, want) in enumerate(batches):
                xs, cs = rr.exact_batch(rng, np.float32, shapes, 1, (0,))
                kinds = check_exact(plan, op, xs, cs, (0,), off=b, what=("reuse", b))
                assert [k[0] for k in kinds] == want, (b, kinds)


def test_large_exact_cases():
    rng = np.random.default_rng(16)
    with Plan(8) as plan:
        # per-channel mean and std_dev of 1080p x 3 (inner + split)
        for t in (np.uint8, np.float32):
            xs, cs = zip(*[rr.exact_data((1080, 1920, 3), t, 2, rng, count=1080 * 1920, terms=("x", "dev")) for _ in range(2)])
            for op in (rr.MEAN, rr.STD_DEV, rr.VARIANCE):
                kinds = check_exact(plan, op, list(xs), list(cs), (0, 1), off=1, what=("1080p", t))
                assert kinds[0][0] == SPLIT, kinds
        # std_dev over HW of 224^2 x 3
        xs, cs = zip(*[rr.exact_data((224, 224, 3), np.float32, 2, rng, count=224 * 224, terms=("dev",)) for _ in range(8)])
        for op in (rr.STD_DEV, rr.VARIANCE):
            check_exact(plan, op, list(xs), list(cs), (0, 1), keep_dims=True, what="224^2")
        # max and mean over t of 513 x 626 (columns, split)
        xs, cs = zip(*[rr.exact_data((513, 626), np.float32, 1, rng, count=513, terms=("x",)) for _ in range(4)])
        for op in (rr.MAX, rr.MEAN, rr.SUM):
            kinds = check_exact(plan, op, list(xs), list(cs), (0,), what="513 x 626")
            assert kinds[0][0] == SPLIT, kinds
