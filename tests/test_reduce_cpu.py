"""fn.reductions.* without a GPU:
  * the argument, type and shape rules through the operators' own host code (dalihTestReduce: the argument resolution and mean check
    of host/operators.cc followed by the plan set-up of csrc/reduce_plan.h);
  * the planner and the kernel bodies compiled for the host (tools/emul/reduce_emul.cc), every work item and every thread run in
    reverse order, against tests/reduce_ref.py: every operator and type, ranks 0-6 with every subset of axes at ranks 4 and 6,
    negative axes, both keep_dims, unit and zero extents, shapes that differ per sample, unaligned inputs and both sides of every path
    threshold and of the chunk sizes (the path of each pass is read back); and on exact-sum inputs (reduce_ref.exact_data) byte for
    byte against reduce_ref.exact_reference;
  * random cases under ASan + UBSan."""
import ctypes as C
import itertools
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from dali_b200 import backend

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import reduce_host as rh  # noqa: E402
import reduce_ref as rr  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tools", "emul", "reduce_emul.cc")
COLUMNS, INNER, SPLIT = 0, 1, 2
P64 = C.POINTER(C.c_int64)


# ---- argument, type and shape rules (the operators' host code)
def rule(op, shapes, layout="", axes=None, axis_names=None, keep_dims=False, dtype=-1, in_code=0, mean=None, ddof=0):
    """(out_shapes, out_type, out_layout) or the error message"""
    s = np.ascontiguousarray(shapes, np.int64).reshape(len(shapes), -1)
    n, nd = len(shapes), len(shapes[0])
    ax = np.asarray(axes if axes is not None else [], np.int64)
    out = np.zeros(n * max(nd, 1), np.int64)
    ond, ot, lay = C.c_int(), C.c_int(), C.create_string_buffer(64)
    ms = None if mean is None else np.ascontiguousarray(mean, np.int64).reshape(n, -1)
    rc = backend.lib().dalihTestReduce(op, in_code, n, nd, s.ctypes.data_as(P64), layout.encode(), ax.ctypes.data_as(P64),
                                       -1 if axes is None else ax.size, None if axis_names is None else axis_names.encode(), int(keep_dims),
                                       dtype, ddof, None if ms is None else ms.ctypes.data_as(P64), 0 if ms is None else ms.shape[1],
                                       out.ctypes.data_as(P64), C.byref(ond), C.byref(ot), lay, 64)
    if rc:
        return backend.lib().dalihLastError().decode()
    return out[:n * ond.value].reshape(n, ond.value).tolist(), ot.value, lay.value.decode()


def test_axes_layouts_and_keep_dims():
    hwc = [[4, 5, 3], [2, 7, 3]]
    assert rule(rr.MEAN, hwc, "HWC", axes=[0, 1]) == ([[3], [3]], 9, "C")
    assert rule(rr.MEAN, hwc, "HWC", axis_names="HW", keep_dims=True) == ([[1, 1, 3], [1, 1, 3]], 9, "HWC")
    assert rule(rr.MEAN, hwc, "HWC", axes=[-1]) == ([[4, 5], [2, 7]], 9, "HW")
    assert rule(rr.SUM, hwc, "HWC") == ([[], []], 3, "")                     # default: all axes, 0-d outputs
    assert rule(rr.SUM, hwc, "HWC", axes=[]) == (hwc, 3, "HWC")              # no axes: every element is its own output
    assert rule(rr.MAX, [[]], "") == ([[]], 0, "")                           # a 0-d input
    assert rule(rr.MAX, [[2, 0, 3]], "", axes=[0], keep_dims=True)[0] == [[1, 0, 3]]


def test_refusals_name_the_problem():
    hwc = [[4, 5, 3]]
    e = rule(rr.SUM, hwc, "HWC", axes=[3])
    assert "axis 3 is out of range [-3, 2]" in e, e
    e = rule(rr.SUM, hwc, "HWC", axes=[-4])
    assert "axis -4 is out of range [-3, 2]" in e, e
    e = rule(rr.SUM, hwc, "HWC", axes=[1, -2])
    assert "axis 1 of input 0 is given more than once" in e, e
    e = rule(rr.SUM, hwc, "HWC", axes=[0], axis_names="H")
    assert "`axes` and `axis_names` are mutually exclusive" in e, e
    e = rule(rr.SUM, hwc, "HWC", axis_names="F")
    assert "axis name 'F' is not in the layout \"HWC\"" in e, e
    e = rule(rr.SUM, hwc, "HWC", in_code=11)
    assert "BOOL input is not supported" in e, e
    e = rule(rr.SUM, hwc, "HWC", in_code=9, dtype=0)
    assert "an integer dtype needs an integer input" in e, e
    for op in (rr.MEAN, rr.MEAN_SQUARE, rr.RMS):
        e = rule(op, hwc, "HWC", dtype=5)
        assert "dtype must be FLOAT16, FLOAT or FLOAT64" in e, e
    e = rule(rr.SUM, hwc, "HWC", dtype=11)
    assert "invalid dtype 11" in e, e
    e = rule(rr.SUM, hwc, "HWC", in_code=42)
    assert "unsupported input type 42" in e, e
    e = rule(rr.MIN, [[4, 5, 3], [2, 0, 3]], "HWC", axes=[1])
    assert "sample 1 of input 0 has shape [2, 0, 3]: the reduced axes are empty" in e, e
    assert rule(rr.MIN, [[2, 0, 3]], "", axes=[0])[0] == [[0, 3]]           # an empty output needs no identity
    e = rule(rr.STD_DEV, [[4, 5, 3], [2, 2, 3]], "HWC", axes=[0, 1], mean=[[3], [4]])
    assert "sample 1 of input 1 (the mean) has shape [4]; expected [3] or [1, 1, 3]" in e, e
    assert rule(rr.STD_DEV, [[4, 5, 3]], "HWC", axes=[0, 1], mean=[[1, 1, 3]])[1] == 9
    e = rule(rr.SUM, [[3, -1]], "")
    assert "sample 0 of input 0 has a negative extent [3, -1]" in e, e
    e = rule(rr.SUM, [[1 << 31, 1 << 31, 1 << 31]], "")
    assert "too many elements" in e, e
    e = rule(rr.SUM, [[1] * 7], "")
    assert "at most 6 dimensions" in e, e


# ---- the host build of the planner and the kernel bodies (tests/reduce_host.py)
@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    lib = rh.build(tmp_path_factory.mktemp("reduce"))
    if lib is None:
        pytest.skip("needs g++")
    return lib


run = rh.run


_data = rr.random_data


def check_all(lib, op, xs, axes=None, keep_dims=False, dtype=None, ddof=0, off=0, moff=0, what=""):
    means = None
    if op in (rr.STD_DEV, rr.VARIANCE):
        ax = rr._axes(xs[0], axes) if xs[0].ndim else ()
        means = [np.mean(x.astype(np.float64), axis=ax, keepdims=keep_dims).astype(np.float32) if x.size else
                 np.zeros([1 if a in ax else e for a, e in enumerate(x.shape)] if keep_dims else
                          [e for a, e in enumerate(x.shape) if a not in ax], np.float32) for x in xs]
    got, kinds, depths = run(lib, op, xs, axes, keep_dims, dtype, ddof, means, off, moff, off)
    assert got is not None, (what, kinds)
    for i, x in enumerate(xs):
        want, tol = rr.reference(op, x, (rr._axes(x, axes) if x.ndim else None), keep_dims, dtype, ddof,
                                 None if means is None else means[i], depths[i])
        rr.check(got[i], np.asarray(want), tol, (what, rr.NAMES[op], x.dtype, x.shape, axes, keep_dims))
    return kinds


def test_every_operator_and_type(emul):
    rng = np.random.default_rng(1)
    for op in range(8):
        for t in rr.TYPES:
            xs = [_data((7, 9, 3), t, rng), _data((1, 300, 3), t, rng), _data((5, 1, 2), t, rng)]
            for axes in (None, (0, 1), (2,), (-2,)):
                check_all(emul, op, xs, axes, keep_dims=bool(rng.integers(0, 2)), what="types")


def test_sum_dtypes_and_mean_dtypes(emul):
    rng = np.random.default_rng(2)
    xs = [_data((40, 50), np.uint8, rng), _data((3, 700), np.uint8, rng)]
    for d in range(11):                                            # every dtype of sum; UINT8 wraps modulo 256
        check_all(emul, rr.SUM, xs, (1,), dtype=d, what="sum dtype")
    ys = [_data((40, 50), np.int16, rng), _data((6, 13), np.int16, rng)]
    for op in (rr.MEAN, rr.MEAN_SQUARE, rr.RMS):
        for d in (rr.F16, rr.F32, rr.F64):
            check_all(emul, op, ys, (0,), dtype=d, what="mean dtype")
    fs = [_data((30, 40), np.float64, rng)]
    for d in (rr.F16, rr.F32, rr.F64):
        check_all(emul, rr.MEAN, fs, None, dtype=d, what="f64 mean dtype")
        check_all(emul, rr.SUM, fs, (1,), dtype=d, what="f64 sum dtype")
    g, _, _ = run(emul, rr.SUM, [np.full((300,), 200, np.uint8)], dtype=0)
    assert g[0].dtype == np.uint8 and int(g[0]) == (300 * 200) % 256


def test_ranks_0_to_6_and_every_axis_subset_at_ranks_4_and_6(emul):
    rng = np.random.default_rng(3)
    for rank in range(7):
        big = {0: 1, 1: 5000, 2: 90, 3: 20, 4: 8}.get(rank, 5)
        subsets = [c for k in range(rank + 1) for c in itertools.combinations(range(rank), k)]
        if rank not in (4, 6):
            subsets = subsets[::max(1, len(subsets) // 6)] + [tuple(range(rank))]
        for j, sub in enumerate(subsets):
            shapes = [tuple(int(v) for v in rng.integers(1, big + 1, rank)) for _ in range(2)]
            shapes.append(tuple(1 if a % 2 else int(rng.integers(1, big + 1)) for a in range(rank)))
            op = [rr.SUM, rr.MEAN, rr.MAX, rr.STD_DEV, rr.RMS][j % 5]
            t = [np.int16, np.float32, np.uint8, np.float32, np.int32][j % 5]
            xs = [_data(s, t, rng) for s in shapes]
            check_all(emul, op, xs, sub if rank else None, keep_dims=bool(j % 2), what=("rank", rank, sub))


def test_negative_axes_unit_and_zero_extents(emul):
    rng = np.random.default_rng(4)
    for op in (rr.SUM, rr.MEAN, rr.VARIANCE, rr.RMS):
        xs = [_data((4, 0, 3), np.float32, rng), _data((4, 5, 3), np.float32, rng), _data((0, 5, 3), np.float32, rng)]
        check_all(emul, op, xs, (-2,), keep_dims=True, what="zero extents")
        check_all(emul, op, xs, (-3, -1), what="zero extents")
    g, _, _ = run(emul, rr.SUM, [np.zeros((3, 0), np.int32)], (1,))
    assert g[0].tolist() == [0, 0, 0]
    g, _, _ = run(emul, rr.MEAN, [np.zeros((3, 0), np.int32)], (1,))
    assert np.isnan(g[0]).all() and g[0].shape == (3,)
    g, _, _ = run(emul, rr.STD_DEV, [np.zeros((2, 0), np.float32)], (1,), means=[np.zeros(2, np.float32)])
    assert np.isnan(g[0]).all()
    g, _, _ = run(emul, rr.MAX, [np.zeros((0, 4), np.uint8)], (1,))
    assert g[0].shape == (0,)
    _, e, _ = run(emul, rr.MAX, [np.zeros((2, 0), np.uint8)], (1,))
    assert "the reduced axes are empty" in e, e


def test_nan_propagates_through_min_and_max(emul):
    x = np.arange(5000, dtype=np.float32).reshape(50, 100)
    x[17, 33] = np.nan
    for op in (rr.MIN, rr.MAX):
        for axes in (None, (0,), (1,)):
            check_all(emul, op, [x, x[:, :7]], axes, what="nan")


def test_paths_on_both_sides_of_each_threshold(emul):
    rng = np.random.default_rng(5)
    cases = [
        # (shape, axes, expected kinds of the first pass)
        ((40, 32), (0,), COLUMNS),            # I = 32: columns
        ((200, 31), (0,), INNER),             # I = 31, R * I = 6200: inner
        ((66, 31), (0,), COLUMNS),            # R * I = 2046 < 2048: columns
        ((2048,), None, INNER),               # R * I = 2048: inner
        ((2047,), None, SPLIT),               # R * I = 2047: columns, 8 chunks of 256
        ((256,), None, COLUMNS),
        ((256, 40), (0,), COLUMNS),           # R = 256: one chunk
        ((257, 40), (0,), SPLIT),             # R = 257: two chunks
        ((32768,), None, INNER),              # one inner chunk
        ((32769,), None, SPLIT),              # two inner chunks
        ((10923, 3), (0,), SPLIT),            # 3 channels: chunks of 10922 rows
        ((10922, 3), (0,), INNER),
    ]
    for shape, axes, kind in cases:
        for t in (np.uint8, np.float32, np.int64):
            for op in (rr.SUM, rr.MEAN, rr.MIN, rr.STD_DEV):
                xs = [_data(shape, t, rng)]
                kinds = check_all(emul, op, xs, axes, off=int(rng.integers(0, 4)), what=("path", shape, axes))
                assert kinds[0][0] == kind, (shape, axes, kinds)


def test_multi_pass_shapes_differ_per_sample(emul):
    rng = np.random.default_rng(6)
    # HWC per-channel statistics, FHW per-frame, a rank-6 input reduced over axes 0, 2, 4 (three passes)
    xs = [_data((37, 41, 3), np.uint8, rng), _data((1, 300, 3), np.uint8, rng), _data((200, 100, 3), np.uint8, rng)]
    for op in range(8):
        check_all(emul, op, xs, (0, 1), keep_dims=True, what="hwc")
    ys = [_data((3, 5, 7, 4, 6, 2), np.float32, rng), _data((2, 1, 9, 3, 1, 5), np.float32, rng)]
    for op in range(8):
        kinds = check_all(emul, op, ys, (0, 2, 4), what="rank 6")
        assert all(k >= 0 for k in kinds[0]), kinds
    # a long single sample split in the first pass, then reduced again
    zs = [_data((3, 40000, 2), np.float32, rng)]
    for op in (rr.SUM, rr.STD_DEV, rr.MAX):
        check_all(emul, op, zs, (0, 1), what="split then reduce")


def test_unaligned_inputs(emul):
    rng = np.random.default_rng(7)
    for t in (np.uint8, np.int16, np.float32, np.float64):
        xs = [_data((50, 123), t, rng), _data((2500, 3), t, rng)]
        for off in range(16 // np.dtype(t).itemsize):
            for op in (rr.SUM, rr.MEAN_SQUARE, rr.MAX, rr.STD_DEV, rr.VARIANCE):
                check_all(emul, op, xs, (1,), off=off, moff=off % 4, what=("offset", t, off))
                check_all(emul, op, xs, (0,), off=off, moff=off % 4, what=("offset", t, off))


def run_exact(lib, op, xs, cs, axes, keep_dims, off=0, what="", **kw):
    """one batch of exact_data through the host build against exact_reference, byte for byte; returns the kinds"""
    means = [rr.exact_mean(c, x, axes, keep_dims) for x, c in zip(xs, cs)] if op in (rr.STD_DEV, rr.VARIANCE) else None
    got, kinds, _ = run(lib, op, xs, axes, keep_dims, means=means, off=off, moff=off, ooff=off, **kw)
    assert got is not None, (what, kinds)
    for i, x in enumerate(xs):
        want = rr.exact_reference(op, x, axes, keep_dims, mean=None if means is None else means[i], **kw)
        rr.same_bytes(got[i], want, (what, rr.NAMES[op], kw, x.dtype, x.shape, axes, off))
    return kinds


def test_exact_sums_bit_for_bit(emul):
    """float sums, means, std_dev and variance on inputs whose every partial sum is exact: the one right result, byte for byte"""
    rng = np.random.default_rng(8)
    for what, types, ops, shapes, ch, axes, keep in rr.exact_cases(rng):
        for t in types:
            xs, cs = rr.exact_batch(rng, t, shapes, ch, axes)
            for op in ops:
                for kw in rr.VARIANTS.get(op, [{}]):
                    run_exact(emul, op, xs, cs, axes, keep, off=int(rng.integers(0, 16)), what=what, **kw)


def test_exact_sums_see_a_mixed_up_channel(emul):
    """the exact data centres each channel on its own value: a channel's statistics moved to its neighbour are wrong by whole steps"""
    rng = np.random.default_rng(9)
    for t in (np.uint8, np.float32):
        xs, cs = rr.exact_batch(rng, t, [(2500, 3), (700, 5)], 1, (0,))
        for op in (rr.SUM, rr.MEAN, rr.STD_DEV):
            means = [rr.exact_mean(c, x, (0,)) for x, c in zip(xs, cs)] if op == rr.STD_DEV else None
            got, _, _ = run(emul, op, xs, (0,), means=means)
            for i, x in enumerate(xs):
                want = rr.exact_reference(op, x, (0,), mean=None if means is None else means[i])
                rr.same_bytes(got[i], want)
                rolled = np.roll(want, 1)
                assert not np.any(rolled == want), (op, t, want)


def test_random_cases_under_sanitizers(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path / "reduce_fuzz")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-DREDUCE_EMUL_MAIN", SRC, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    for seed in (1, 2, 3):
        r = subprocess.run([exe, "250", str(seed)], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0 and r.stdout.strip() == "ok 250", (r.stdout[-2000:], r.stderr[-3000:])
