"""fn.erase without a GPU:
  * tests/erase_ref.py's rounding pinned (llround ties and the largest double below 0.5);
  * the argument, type, layout, region and fill rules through the operator's argument resolution and plan set-up (dalihTestErase),
    every refusal included;
  * the planner and the kernel bodies compiled for the host (tools/emul/erase_emul.cc), every work item and thread run in reverse
    order, bit for bit against erase_ref: every type x layout, every non-empty subset of erased axes at ranks 3 and 4; 0, 1, 3 and 64
    regions; absolute, normalised and centred coordinates with ties at .5; regions partly and wholly outside, empty, touching,
    overlapping and covering the sample; scalar and per-channel fills in and out of the type's range; empty samples; every byte
    offset of input and output; the band count of many regions;
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
import erase_ref as er  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tools", "emul", "erase_emul.cc")
P64 = C.POINTER(C.c_int64)
DTYPES = (np.uint8, np.uint16, np.uint32, np.uint64, np.int8, np.int16, np.int32, np.int64, np.float16, np.float32, np.float64, np.bool_)
LAYOUTS = ("T", "TC", "ft", "tf", "HW", "HWC", "CHW", "FHWC", "FCHW", "DHWC", "FDHWC")
EXT = {"T": 37, "C": 3, "f": 9, "t": 23, "H": 11, "W": 13, "F": 3, "D": 4}


def data(rng, shape, dt):
    """random bits (NaN payloads included for the float types), 0 / 1 for BOOL"""
    dt = np.dtype(dt)
    if dt == np.bool_:
        return rng.integers(0, 2, shape).astype(np.bool_)
    return rng.integers(0, 256, int(np.prod(shape)) * dt.itemsize, dtype=np.uint8).view(dt).reshape(shape)


def flat(vals):
    return [float(v) for v in np.asarray(vals, np.float32).reshape(-1)]


# ---- argument, type, layout and shape rules (the operator's argument resolution and plan set-up)
def rule(shapes, anchors=None, rshapes=None, layout="", type=0, names=None, axes=None, normalized=-1, norm_anchor=-1, norm_shape=-1,
         centered=0, fill=None):
    s = np.ascontiguousarray(shapes, np.int64).reshape(len(shapes), -1)
    n, nd = s.shape
    anchors = anchors if anchors is not None else [[]] * n
    rshapes = rshapes if rshapes is not None else anchors
    av = (C.c_float * max(1, sum(len(a) for a in anchors)))(*[v for a in anchors for v in a])
    sv = (C.c_float * max(1, sum(len(a) for a in rshapes)))(*[v for a in rshapes for v in a])
    ax = (C.c_int32 * max(1, len(axes or [])))(*(axes or []))
    fv = (C.c_float * max(1, len(fill or [])))(*(fill or []))
    L = backend.lib()
    rc = L.dalihTestErase(type, n, nd, s.ctypes.data_as(P64), layout.encode(), names.encode() if names is not None else None, ax,
                          len(axes) if axes is not None else -1, av, (C.c_int64 * n)(*[len(a) for a in anchors]), sv,
                          (C.c_int64 * n)(*[len(a) for a in rshapes]), normalized, norm_anchor, norm_shape, centered, fv,
                          len(fill) if fill is not None else -1)
    return L.dalihLastError().decode() if rc else None


def test_reference_rounding():
    assert [er.llround(v) for v in (2.5, -2.5, 0.5, -0.5, 1.4999999999999998, 0.49999999999999994, 3.0)] == [3, -3, 1, -1, 1, 0, 3]
    assert er.boxes((10,), [0], [0.25], [0.5], True, True) == [([3], [8])]            # 2.5 -> 3, 7.5 -> 8
    assert er.boxes((10,), [0], [5], [3], centered=True) == [([4], [7])]              # 3.5 -> 4, 6.5 -> 7
    assert er.boxes((10,), [0], [-4], [20]) == [([0], [10])]


def test_arguments_accepted():
    assert rule([[4, 5, 3]], [[1, 1]], [[2, 2]], "HWC") is None
    assert rule([[4, 5, 3]], [[1, 1, 0, 0]], [[2, 2, 1, 1]], "HWC", names="WH") is None
    assert rule([[4, 5]], [[1, 1]], [[2, 2]], "") is None                           # no layout: axes, by default [1, 0]
    assert rule([[4, 5, 3]], [[1]], [[2]], "", axes=[2]) is None
    assert rule([[4, 5, 3], [2, 2, 3]], [[], [0, 0]], [[], [1, 1]], "HWC") is None    # per-sample region counts, 0 included
    assert rule([[4, 5, 3]], [[0, 0]], [[1, 1]], "HWC", fill=[1, 2, 3]) is None
    assert rule([[3, 4, 5]], [[0, 0]], [[1, 1]], "CHW", fill=[1, 2, 3]) is None
    assert rule([[0, 5, 3]], [[0, 0]], [[1, 1]], "HWC") is None
    for t in range(12):
        assert rule([[4, 5]], [[0, 0]], [[1, 1]], "HW", type=t) is None
    assert rule([[2] * 6], [[0]], [[1]], "FDHWCX", names="X") is None
    assert rule([[4, 5]], [[0.5, 0.5]], [[0.5, 0.5]], "HW", normalized=1, norm_anchor=0) is None


def test_refusals_name_the_sample_and_the_argument():
    assert 'axis_names "HX": \'X\' is not an axis of the layout "HWC"' in rule([[4, 5, 3]], layout="HWC", names="HX")
    assert "axis_names names the dimension 0 twice" in rule([[4, 5, 3]], layout="HWC", names="HH")
    assert "axes names the dimension 1 twice" in rule([[4, 5, 3]], axes=[1, 1])
    assert "axis_names names no axis" in rule([[4, 5, 3]], layout="HWC", names="")
    assert "axes names no axis" in rule([[4, 5, 3]], axes=[])
    assert "axes: 3 is not a dimension of the 3-dimensional input 0" in rule([[4, 5, 3]], axes=[3])
    assert "axes: -1 is not a dimension" in rule([[4, 5, 3]], axes=[-1])
    assert 'axis_names "HW" needs a layout, and input 0 has none' in rule([[4, 5]], names="HW")
    assert "'h' is not an axis" in rule([[4, 5]], layout="HW", names="h")                 # layout characters are case-sensitive
    assert 'input 0 has layout "HWC" but 2 dimensions' in rule([[4, 5]], layout="HWC")
    assert 'layout "HWW" of input 0 repeats the axis \'W\'' in rule([[4, 5, 3]], layout="HWW")
    assert "input 0 has 7 dimensions; 1 to 6 are supported" in rule([[1] * 7], axes=[0])
    assert "input 0 has an unsupported type (code 12)" in rule([[4, 5]], layout="HW", type=12)
    assert "sample 1: anchor has 2 values and shape 4" in rule([[4, 5], [4, 5]], [[0, 0], [0, 0]], [[1, 1], [1, 1, 1, 1]], "HW")
    assert "sample 0: anchor and shape have 3 values, not a multiple of the 2 erased axes" in rule([[4, 5]], [[0, 0, 0]], None, "HW")
    assert "sample 0: shape value -1 is a negative extent" in rule([[4, 5]], [[0, 0]], [[1, -1]], "HW")
    assert "sample 0: anchor value nan is not finite" in rule([[4, 5]], [[0, float("nan")]], [[1, 1]], "HW")
    assert "sample 0: shape value inf is not finite" in rule([[4, 5]], [[0, 0]], [[1, float("inf")]], "HW")
    assert "sample 1 of input 0 has a negative extent [4, -5]" in rule([[4, 5], [4, -5]], layout="HW")
    assert "fill_value has 3 values; more than one needs a C axis in the layout of input 0" in rule([[4, 5]], layout="HW", fill=[1, 2, 3])
    assert "fill_value has 3 values, one per channel, but the C axis is erased" in rule([[4, 5, 3]], layout="HWC", names="WC",
                                                                                        fill=[1, 2, 3])
    assert "sample 1: fill_value has 3 values, but the C axis of input 0 has 4 channels" in rule([[4, 5, 3], [4, 5, 4]], layout="HWC",
                                                                                                  fill=[1, 2, 3])
    assert "fill_value has no value" in rule([[4, 5]], layout="HW", fill=[])
    assert "too many elements" in rule([[2 ** 30, 2 ** 30]], layout="HW")


def test_launch_refuses_device_pointers_not_aligned_to_their_element():
    from dali_b200 import capi
    L = capi.lib()
    plan = C.c_void_p()
    capi.check(L.dalib200ErasePlanCreate(C.byref(plan), 1))
    try:
        capi.check(L.dalib200EraseSetup(plan, 5, 1, 3, (C.c_int64 * 3)(4, 5, 3), b"HWC", b"HW", None, 0, (C.c_float * 2)(1, 1),
                                        (C.c_int64 * 1)(2), (C.c_float * 2)(2, 2), (C.c_int64 * 1)(2), 0, 0, 0, (C.c_float * 1)(0), 1))
        for ip, op in ((0x10001, 0x20000), (0x10000, 0x20003)):
            rc = L.dalib200EraseLaunch(plan, (C.c_void_p * 1)(ip), (C.c_void_p * 1)(op), None)
            assert rc != 0 and "sample 0: a device pointer is not aligned to its element size" in L.dalib200GetLastError().decode()
    finally:
        L.dalib200ErasePlanDestroy(plan)


# ---- the host build
@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    so = str(tmp_path_factory.mktemp("er") / "erase_emul.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", SRC, "-o", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


def placed(x, off, keep, fill=0):
    buf = np.full(x.nbytes + 64, fill, np.uint8)
    base = (-buf.ctypes.data) % 16 + 16 + off
    buf[base:base + x.nbytes] = np.ascontiguousarray(x).view(np.uint8).reshape(-1)
    keep.append((buf, base, x.nbytes))
    return buf.ctypes.data + base


def plan(lib, xs, axes, anchors, rshapes=None, fill=(0.0,), layout="", names=None, na=False, ns=False, cen=False, ins=None, outs=None):
    n, nd = len(xs), xs[0].ndim
    rshapes = rshapes if rshapes is not None else anchors
    av = flat([v for a in anchors for v in flat(a)] or [0])
    sv = flat([v for a in rshapes for v in flat(a)] or [0])
    items, bands = (C.c_int64 * n)(), (C.c_int64 * n)()
    err = C.create_string_buffer(512)
    rc = lib.emul_erase(er.TYPES[xs[0].dtype], n, nd, (C.c_int64 * (n * nd))(*[e for x in xs for e in x.shape]), layout.encode(),
                        names.encode() if names is not None else None, (C.c_int32 * len(axes))(*axes), len(axes),
                        (C.c_float * len(av))(*av), (C.c_int64 * n)(*[len(flat(a)) for a in anchors]), (C.c_float * len(sv))(*sv),
                        (C.c_int64 * n)(*[len(flat(a)) for a in rshapes]), int(na), int(ns), int(cen),
                        (C.c_float * len(flat(fill)))(*flat(fill)), len(flat(fill)), ins, outs, items, bands, err, 512)
    assert rc == 0, err.value
    return list(items), list(bands)


def run(lib, xs, axes, anchors, rshapes=None, fill=(0.0,), layout="", names=None, na=False, ns=False, cen=False, offs=(0, 0)):
    """outputs of the host build; sample i's input at byte (offs[0] + i) and output at (offs[1] + 3 i) past a 16-byte boundary, rounded
    down to the element size; the bytes around each output checked"""
    keep, outs = [], []
    ins = [placed(x, (offs[0] + i) % 16 // x.itemsize * x.itemsize, keep) for i, x in enumerate(xs)]
    op = [placed(np.zeros_like(x), (offs[1] + 3 * i) % 16 // x.itemsize * x.itemsize, outs, 0xA5) for i, x in enumerate(xs)]
    plan(lib, xs, axes, anchors, rshapes, fill, layout, names, na, ns, cen, (C.c_void_p * len(xs))(*ins), (C.c_void_p * len(xs))(*op))
    res = []
    for (buf, base, nb), x in zip(outs, xs):
        assert np.all(buf[:base] == 0xA5) and np.all(buf[base + nb:] == 0xA5), "a write outside the output"
        res.append(buf[base:base + nb].view(x.dtype).reshape(x.shape))
    return res


def check(lib, xs, axes, anchors, rshapes=None, fill=(0.0,), layout="", names=None, na=False, ns=False, cen=False, offs=(0, 0)):
    rshapes = rshapes if rshapes is not None else anchors
    got = run(lib, xs, axes, anchors, rshapes, fill, layout, names, na, ns, cen, offs)
    for x, g, a, s in zip(xs, got, anchors, rshapes):
        want = er.erase_ref(x, axes, a, s, fill, layout, na, ns, cen)
        assert g.tobytes() == want.tobytes(), (x.dtype, x.shape, layout, axes, a, s)


def random_regions(rng, shape, axes, k):
    a, s = [], []
    for _ in range(k):
        for ax in axes:
            a.append(float(rng.integers(-3, shape[ax] + 3)))
            s.append(float(rng.integers(0, shape[ax] + 2)))
    return a, s


def test_every_type_layout_and_axis_subset(emul):
    rng = np.random.default_rng(1)
    for lay in LAYOUTS:
        nd = len(lay)
        subsets = [c for r in range(1, nd + 1) for c in itertools.combinations(range(nd), r)] if nd in (3, 4) else \
            [tuple(range(nd)), (nd - 1,), (0,)]
        for sub in subsets:
            for dt in DTYPES:
                axes = list(sub)[::-1] if rng.integers(2) else list(sub)
                shapes = [[EXT[c] for c in lay], [EXT[c] if c == "C" else EXT[c] // 2 + 1 for c in lay]]
                xs = [data(rng, s, dt) for s in shapes]
                regs = [random_regions(rng, s, axes, int(rng.integers(1, 4))) for s in shapes]
                check(emul, xs, axes, [r[0] for r in regs], [r[1] for r in regs], (7.0,), lay, "".join(lay[a] for a in axes),
                      offs=(int(rng.integers(16)), int(rng.integers(16))))


def test_region_counts_0_1_3_and_64(emul):
    rng = np.random.default_rng(2)
    for dt in (np.uint8, np.float32, np.int64):
        x = data(rng, (40, 50, 3), dt)
        for k in (0, 1, 3, 64):
            a, s = random_regions(rng, x.shape, [0, 1], k)
            check(emul, [x, x], [0, 1], [a, a[:2 * (k // 2)]], [s, s[:2 * (k // 2)]], (1.0,), "HWC", "HW")
    seq = data(rng, (5, 20, 30, 2), np.uint16)
    a, s = random_regions(rng, seq.shape, [0, 1, 2], 64)
    check(emul, [seq], [0, 1, 2], [a], [s], (9.0,), "FHWC", "FHW")


def test_normalised_centred_coordinates_and_ties(emul):
    rng = np.random.default_rng(3)
    x = data(rng, (10, 12), np.uint8)
    for na, ns, cen in itertools.product((False, True), repeat=3):
        # ties at .5: 0.25 * 10 = 2.5, 0.75 * 12 = 9; absolute ones 2.5, 3.5
        a = [0.25, 0.75] if na else [2.5, 3.5]
        s = [0.35, 0.125] if ns else [3.0, 2.5]
        check(emul, [x], [0, 1], [a], [s], (255.0,), "HW", "HW", na, ns, cen)
    a = list(rng.random(40).astype(np.float32))
    s = list((rng.random(40) * 0.5).astype(np.float32))
    for cen in (False, True):
        check(emul, [x, data(rng, (7, 3), np.uint8)], [1, 0], [a, a], [s, s], (3.0,), "HW", "WH", True, True, cen)
    # normalised through the argument flags: normalized, with normalized_anchor overriding it
    assert rule([[10, 12]], [[0.5, 0.5]], [[0.2, 0.2]], "HW", normalized=1, norm_anchor=0) is None


def test_regions_outside_empty_touching_overlapping_and_whole(emul):
    rng = np.random.default_rng(4)
    x = data(rng, (16, 20, 3), np.int16)
    cases = {
        "partly outside": ([-3, -4, 10, 15], [6, 8, 10, 10]),
        "wholly outside": ([-10, 0, 16, 0, 0, 20, 0, -9], [5, 20, 4, 20, 16, 3, 16, 9]),
        "empty": ([2, 2, 5, 5], [0, 4, 4, 0]),
        "touching": ([2, 2, 2, 6, 6, 2], [4, 4, 4, 4, 4, 4]),
        "overlapping": ([1, 1, 3, 3, 2, 0], [6, 6, 6, 6, 1, 20]),
        "whole": ([0, 0], [16, 20]),
        "beyond whole": ([-5, -5], [100, 100]),
    }
    for name, (a, s) in cases.items():
        (g,) = run(emul, [x], [0, 1], [a], [s], (-2.0,), "HWC", "HW")
        assert g.tobytes() == er.erase_ref(x, [0, 1], a, s, (-2.0,)).tobytes(), name
    (g,) = run(emul, [x], [0, 1], [[0, 0]], [[16, 20]], (-2.0,), "HWC", "HW")
    assert np.all(g == -2)


def test_scalar_and_per_channel_fills_in_and_out_of_range(emul):
    rng = np.random.default_rng(5)
    fills = [(300.0,), (-5.0,), (1e10,), (-1e30,), (2.5,), (-2.5,), (float("nan"),), (float("inf"),), (70000.0,), (1e-40,)]
    for dt in DTYPES:
        x = data(rng, (9, 17, 3), dt)
        for f in fills:
            check(emul, [x], [0, 1], [[1, 2]], [[5, 9]], f, "HWC", "HW")
        for f in ((1.0, 2.0, 3.0), (300.0, -7.5, float("nan"))):
            check(emul, [x], [0, 1], [[1, 2, 4, 0]], [[5, 9, 5, 17]], f, "HWC", "HW")
            chw = np.ascontiguousarray(np.moveaxis(x, 2, 0))
            check(emul, [chw], [1, 2], [[1, 2, 4, 0]], [[5, 9, 5, 17]], f, "CHW", "HW")
    for c in (1, 2, 3, 4, 5, 7, 16, 17):                                   # patterns that do and do not divide 16 bytes
        for dt in (np.uint8, np.uint16, np.float32, np.float64):
            x = data(rng, (6, 33, c), dt)
            fv = tuple(float(v) for v in range(1, c + 1))
            check(emul, [x], [1], [[3]], [[25]], fv, "HWC", "W", offs=(int(rng.integers(16)), int(rng.integers(16))))
    x = data(rng, (4, 5, 3, 7), np.uint8)                                  # C inside the inner run, not innermost
    check(emul, [x], [0, 1], [[1, 1, 0, 3]], [[3, 3, 4, 1]], (10.0, 20.0, 30.0), "HDCW", "HD")


def test_empty_samples_and_every_byte_offset(emul):
    rng = np.random.default_rng(6)
    xs = [np.zeros((0, 5, 3), np.uint8), data(rng, (4, 5, 3), np.uint8), np.zeros((4, 0, 3), np.uint8), np.zeros((4, 5, 0), np.uint8)]
    check(emul, xs, [0, 1], [[1, 1]] * 4, [[2, 2]] * 4, (5.0,), "HWC", "HW")
    items, _ = plan(emul, xs, [0, 1], [[1, 1]] * 4, None, (5.0,), "HWC", "HW")
    assert items[0] == items[2] == items[3] == 0 and items[1] == 1
    for dt in (np.uint8, np.int16, np.float32, np.float64):
        x = data(rng, (19, 45, 3), dt)
        a, s = random_regions(rng, x.shape, [0, 1], 3)
        for o in range(16):
            for p in (o, (o + 5) % 16):
                check(emul, [x, x], [0, 1], [a, a], [s, s], (1.0, 2.0, 3.0), "HWC", "HW", offs=(o, p))


def test_band_count_of_many_regions(emul):
    rng = np.random.default_rng(7)
    x = data(rng, (200, 300, 3), np.uint8)
    for k in (1, 64):
        a, s = random_regions(rng, x.shape, [0, 1], k)
        _, bands = plan(emul, [x], [0, 1], [a], [s], (0.0,), "HWC", "HW")
        assert 1 <= bands[0] <= 2 * k + 1, (k, bands)
    _, bands = plan(emul, [x], [1], [[5]], [[10]], (0.0,), "HWC", "W")      # no outer erased axis: one band
    assert bands == [1]


def test_random_cases_under_sanitizers(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path / "er_fuzz")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-DERASE_EMUL_MAIN",
                        SRC, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    for seed in (1, 2, 3):
        r = subprocess.run([exe, "300", str(seed)], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0 and r.stdout.strip() == "ok 300", (r.stdout[-2000:], r.stderr[-3000:])
