"""fn.experimental.filter without a GPU:
  * tests/filter_ref.py pinned to cv2.filter2D on float32 data for the four borders cv2 has (anchor order swapped: cv2 takes (x, y)),
    kernels up to 7 x 7 (below cv2's DFT threshold: the check is for indexing, not arithmetic);
  * the argument, type, layout and shape rules through the operator's argument resolution and plan set-up (dalihTestFilter), every
    refusal included;
  * the planner and the kernel bodies compiled for the host (tools/emul/filter_emul.cc), every work item and thread run in reverse
    order, against filter_ref: every type x dtype x border x mode x layout; anchors at every position of 1 x 1 ... 7 x 7 filters and
    non-square filters; filters larger than the sample; bit-exact on exact-sum cases (integer or dyadic kernels on integer data), within
    the gamma_k bound otherwise; per-frame fill values; empty samples and frames; every byte offset;
  * random cases under ASan + UBSan."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from dali_b200 import backend

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import arith_ref as ar  # noqa: E402
import filter_ref as fr  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tools", "emul", "filter_emul.cc")
P64 = C.POINTER(C.c_int64)
BORDER = {b: k for k, b in enumerate(fr.BORDERS)}
MODE = {"same": 0, "valid": 1}
DTYPES = (np.uint8, np.int8, np.uint16, np.int16, np.float16, np.float32)


def data(rng, shape, dt):
    dt = np.dtype(dt)
    if dt.kind in "ui":
        info = np.iinfo(dt)
        return rng.integers(info.min, int(info.max) + 1, shape).astype(dt)
    return (rng.standard_normal(shape) * 100).astype(dt)


def test_reference_is_cv2_filter2d():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(0)
    cvb = {"reflect_101": cv2.BORDER_REFLECT_101, "reflect_1001": cv2.BORDER_REFLECT, "clamp": cv2.BORDER_REPLICATE,
           "constant": cv2.BORDER_CONSTANT}
    for t in range(120):
        fh, fw = (int(v) for v in rng.integers(1, 8, 2))
        h, w = int(rng.integers(fh, 40)), int(rng.integers(fw, 40))
        c = (1, 3, 4)[t % 3]
        x = (rng.standard_normal((h, w, c)) * 50).astype(np.float32)
        f = rng.standard_normal((fh, fw)).astype(np.float32)
        a = (int(rng.integers(0, fh)), int(rng.integers(0, fw))) if t % 2 else (-1, -1)
        for b, code in cvb.items():
            got = cv2.filter2D(x, -1, f, anchor=(a[1], a[0]), borderType=code).reshape(h, w, c)
            v = fr.correlate64(x, f, "HWC", a, b)[0]
            # cv2 sums in float32 in its own order: within twice the bound of one chain
            assert np.all(np.abs(got - v) <= 2 * fr.bound(x, f, "HWC", a, b)[0] + 1e-30), (t, b)


# ---- argument, type, layout and shape rules (the operator's argument resolution and plan set-up)
def rule(shapes, fshapes=None, layout="", in_type=0, dtype=-1, anchors=None, border="reflect_101", mode="same", ftype=9, fnd=2,
         fill_type=-1, fill_counts=None):
    s = np.ascontiguousarray(shapes, np.int64).reshape(len(shapes), -1)
    n, nd = s.shape
    f = np.ascontiguousarray(fshapes if fshapes is not None else [[3, 3]] * n, np.int64)
    a = np.ascontiguousarray(anchors if anchors is not None else [[-1]] * n, np.int32)
    cnt = np.ascontiguousarray(fill_counts if fill_counts is not None else [1] * n, np.int64)
    out = np.zeros((n, nd), np.int64)
    L = backend.lib()
    rc = L.dalihTestFilter(in_type, dtype, n, nd, s.ctypes.data_as(P64), layout.encode(), ftype, fnd, f.ctypes.data_as(P64),
                           a.ctypes.data_as(C.POINTER(C.c_int32)), a.shape[1] if a.ndim == 2 else 1, border.encode(), mode.encode(),
                           fill_type, cnt.ctypes.data_as(P64), out.ctypes.data_as(P64))
    return L.dalihLastError().decode() if rc else [list(r) for r in out]


def test_layouts_output_shapes_and_empty_inputs():
    for lay in fr.LAYOUTS:
        shape = [{"F": 2, "H": 9, "W": 11, "C": 3}[a] for a in lay]
        assert rule([shape], [[3, 5]], lay) == [shape]
        valid = [{"F": 2, "H": 7, "W": 7, "C": 3}[a] for a in lay]
        assert rule([shape], [[3, 5]], lay, mode="valid") == [valid]
    assert rule([[9, 11]]) == [[9, 11]] and rule([[9, 11, 3]]) == [[9, 11, 3]] and rule([[2, 9, 11, 3]]) == [[2, 9, 11, 3]]
    assert rule([[0, 5, 3], [4, 0, 3], [4, 5, 0]], layout="HWC") == [[0, 5, 3], [4, 0, 3], [4, 5, 0]]
    assert rule([[0, 9, 11, 3]], layout="FHWC") == [[0, 9, 11, 3]]
    assert rule([[9, 11, 64]], [[255, 255]], "HWC") == [[9, 11, 64]]
    assert rule([[9, 11]], [[1, 1]], anchors=[[0, 0]]) == [[9, 11]] and rule([[9, 11]], [[3, 5]], anchors=[[2, 4]]) == [[9, 11]]
    assert rule([[4, 5, 3]], [[4, 5]], "HWC", mode="valid", anchors=[[99, 99]]) == [[1, 1, 3]]      # anchor ignored in valid mode
    for t in (0, 4, 1, 5, 8, 9):
        assert rule([[9, 11]], in_type=t, dtype=9) == [[9, 11]] and rule([[9, 11]], in_type=t, dtype=t) == [[9, 11]]
    assert rule([[3, 4, 5, 1]], layout="FHWC", fill_type=0, fill_counts=[3]) == [[3, 4, 5, 1]]


def test_refusals_name_the_problem():
    for t, name in ((2, "UINT32"), (3, "UINT64"), (6, "INT32"), (7, "INT64"), (10, "FLOAT64"), (11, "BOOL")):
        assert f"input 0 must be UINT8, INT8, UINT16, INT16, FLOAT16 or FLOAT, got {name}" in rule([[3, 4]], in_type=t)
    assert "dtype must be the input's type (UINT8) or FLOAT, got INT16" in rule([[3, 4]], dtype=5)
    assert "dtype must be the input's type (FLOAT) or FLOAT, got FLOAT16" in rule([[3, 4]], in_type=9, dtype=8)
    assert "input 1 (the filter) must be FLOAT, got FLOAT64" in rule([[3, 4]], ftype=10)
    assert "input 1 (the filter) must be 2-dimensional (HW), got 3" in rule([[3, 4]], [[3, 3]], fnd=3)
    assert "sample 1 of input 1 (the filter) has extents [0, 3]" in rule([[3, 4], [3, 4]], [[3, 3], [0, 3]])
    assert "sample 0 of input 1 (the filter) has extents [3, 256]" in rule([[3, 4]], [[3, 256]])
    assert "sample 1 of input 0 has 65 channels" in rule([[3, 4, 3], [3, 4, 65]], layout="HWC")
    for lay, nd, what in (("CHW", 3, "channel-first"), ("FCHW", 4, "channel-first"), ("DHW", 3, "volumetric"), ("DHWC", 4, "volumetric"),
                          ("FDHWC", 5, "volumetric"), ("NHWC", 4, "not supported")):
        assert f'layout "{lay}" of input 0 is {what}' in rule([[2] * nd], layout=lay), lay
    assert "cannot infer the layout of 5-dimensional input 0" in rule([[1, 2, 3, 4, 3]])
    assert "cannot infer the layout of 1-dimensional input 0" in rule([[3]])
    assert 'layout "HWC" but 2 dimensions' in rule([[3, 4]], layout="HWC")
    assert 'sample 1 of input 0 [4, 2] is smaller than its 3 x 3 filter in "valid" mode' in rule([[5, 5], [4, 2]], mode="valid")
    assert "sample 0: anchor (3, 1) is outside its 3 x 3 filter" in rule([[5, 5]], anchors=[[3, 1]])
    assert "sample 0: anchor (-2, 1) is outside" in rule([[5, 5]], anchors=[[-2, 1]])
    assert "sample 0: anchor must have one value per filter axis (2), or be [-1]; got 3 values" in rule([[5, 5]], anchors=[[1, 1, 1]])
    assert "anchor must have one value per filter axis" in rule([[5, 5]], anchors=[[1]])
    assert "input 2 (fill_value) must have the type of input 0 (UINT8), got FLOAT" in rule([[5, 5]], fill_type=9)
    assert "sample 1 of input 2 (fill_value) has 2 values; expected 1" in rule([[5, 5], [5, 5]], fill_type=0, fill_counts=[1, 2])
    assert "sample 0 of input 2 (fill_value) has 2 values; expected 1 or one per frame" in rule([[3, 5, 5]], layout="FHW", fill_type=0,
                                                                                              fill_counts=[2])
    assert 'unknown border "mirror"' in rule([[5, 5]], border="mirror")
    assert 'unknown mode "full"' in rule([[5, 5]], mode="full")
    assert "sample 1 of input 0 has a frame of 46341 x 46341 x 1 elements" in rule([[2, 2], [46341, 46341]])
    assert "frame of 1 x 33554432 x 64 elements" in rule([[1, 2 ** 25, 64]], layout="HWC")
    assert rule([[46340, 46341]]) == [[46340, 46341]]
    assert "negative extent" in rule([[3, -4]])


def test_launch_refuses_device_pointers_not_aligned_to_their_element():
    from dali_b200 import capi
    L = capi.lib()
    plan = C.c_void_p()
    capi.check(L.dalib200FilterPlanCreate(C.byref(plan), 1))
    try:
        oshp = (C.c_int64 * 3)()
        capi.check(L.dalib200FilterSetup(plan, 5, 9, 1, 3, (C.c_int64 * 3)(4, 5, 3), b"HWC", 9, 2, (C.c_int64 * 2)(3, 3), None, 0, 0, -1,
                                         None, oshp))
        for ip, op, fp in ((0x10001, 0x20000, 0x30000), (0x10000, 0x20002, 0x30000), (0x10000, 0x20000, 0x30002)):
            rc = L.dalib200FilterLaunch(plan, (C.c_void_p * 1)(ip), (C.c_void_p * 1)(fp), 1, None, 0, (C.c_void_p * 1)(op), None)
            assert rc != 0 and "sample 0: a device pointer is not aligned to its element size" in L.dalib200GetLastError().decode()
    finally:
        L.dalib200FilterPlanDestroy(plan)


# ---- the host build
@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    so = str(tmp_path_factory.mktemp("flt") / "filter_emul.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", SRC, "-o", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


def placed(x, off, keep, fill=0):
    buf = np.full(x.nbytes + 64, fill, np.uint8)
    base = (-buf.ctypes.data) % 16 + 16 + off
    buf[base:base + x.nbytes] = np.ascontiguousarray(x).view(np.uint8).reshape(-1)
    keep.append((buf, base, x.nbytes))
    return buf.ctypes.data + base


def run(lib, xs, fs, layout="", anchors=None, border="reflect_101", mode="same", fills=None, dtype=None, offs=(0, 0)):
    """outputs of the host build; sample i's input (offs[0] + i) and output (offs[1] + 3 i) elements (bytes for 8-bit types) past a
    16-byte boundary, the bytes around each output checked"""
    n, nd = len(xs), xs[0].ndim
    it = fr.TYPES[xs[0].dtype]
    odt = np.dtype(dtype or xs[0].dtype)
    ot = fr.TYPES[odt]
    shp = (C.c_int64 * (n * nd))(*[e for x in xs for e in x.shape])
    fshp = (C.c_int64 * (2 * n))(*[e for f in fs for e in f.shape])
    anc = (C.c_int32 * (2 * n))(*[v for a in (anchors or [(-1, -1)] * n) for v in a])
    oshp = (C.c_int64 * (n * nd))()
    cnt = (C.c_int64 * n)(*[np.asarray(v).size for v in fills] if fills is not None else [0] * n)
    err = C.create_string_buffer(512)
    keep, outs = [], []
    ins = [placed(x, (offs[0] + i) % 16 * (1 if x.itemsize == 1 else 0) + (offs[0] + i) % 4 * x.itemsize * (x.itemsize > 1), keep)
           for i, x in enumerate(xs)]
    fl = [np.ascontiguousarray(f, np.float32) for f in fs]
    fv = [np.ascontiguousarray(np.asarray(v, xs[0].dtype).reshape(-1)) for v in fills] if fills is not None else []
    rc = lib.emul_filter(it, ot, n, nd, shp, layout.encode(), fshp, anc, BORDER[border], MODE[mode], it if fills is not None else -1, cnt,
                         oshp, None, None, None, None, None, err, 512)
    assert rc == 0, err.value
    oshapes = [tuple(oshp[i * nd:(i + 1) * nd]) for i in range(n)]
    op = [placed(np.zeros(s, odt), (offs[1] + 3 * i) % 16 if odt.itemsize == 1 else (offs[1] + 3 * i) % 4 * odt.itemsize, outs, 0xA5)
          for i, s in enumerate(oshapes)]
    rc = lib.emul_filter(it, ot, n, nd, shp, layout.encode(), fshp, anc, BORDER[border], MODE[mode], it if fills is not None else -1, cnt,
                         oshp, (C.c_void_p * n)(*ins), (C.c_void_p * n)(*[f.ctypes.data for f in fl]),
                         (C.c_void_p * n)(*[v.ctypes.data for v in fv]) if fills is not None else None, (C.c_void_p * n)(*op), None, err, 512)
    assert rc == 0, err.value
    res = []
    for (buf, base, nb), s in zip(outs, oshapes):
        assert np.all(buf[:base] == 0xA5) and np.all(buf[base + nb:] == 0xA5), "a write outside the output"
        res.append(buf[base:base + nb].view(odt).reshape(s))
    return res


def exact_kernel(rng, fh, fw, dyadic):
    k = rng.integers(-3, 4, (fh, fw)).astype(np.float32)
    return k / np.float32(4) if dyadic else k


def test_every_type_dtype_border_mode_and_layout_bit_exact(emul):
    rng = np.random.default_rng(1)
    for dt in DTYPES[:4]:                                  # integer data, integer or dyadic kernels: every partial sum is exact
        for dtype in (None, np.float32):
            for border in fr.BORDERS:
                for mode in ("same", "valid"):
                    for lay in fr.LAYOUTS:
                        ext = {"F": 2, "H": 13, "W": 17, "C": 3}
                        shapes = [[ext[a] for a in lay], [ext[a] if a in "FC" else ext[a] // 2 + 4 for a in lay]]
                        xs = [data(rng, s, dt) for s in shapes]
                        if dt in (np.uint16, np.int16):
                            xs = [(x // 64).astype(dt) for x in xs]
                        fs = [exact_kernel(rng, 3, 5, False), exact_kernel(rng, 4, 2, True)]
                        anchors = [(-1, -1), (3, 0)]
                        fills = [np.asarray(7, dt), np.asarray(-1 if dt in (np.int8, np.int16) else 200, dt)] if border == "constant" else None
                        got = run(emul, xs, fs, lay, anchors, border, mode, fills, dtype, (int(rng.integers(16)), int(rng.integers(16))))
                        for x, f, a, g, v in zip(xs, fs, anchors, got, fills or [None] * 2):
                            want = fr.filter_ref(x, f, lay, a, border, mode, v, dtype)
                            assert g.dtype == want.dtype and np.array_equal(g, want), (dt, dtype, border, mode, lay)


def test_float_and_half_data_within_the_bound(emul):
    rng = np.random.default_rng(2)
    for dt in DTYPES:
        for dtype in (None, np.float32):
            for border in fr.BORDERS:
                xs = [data(rng, (21, 34, 3), dt), data(rng, (5, 2, 3), dt)]
                fs = [rng.standard_normal((5, 7)).astype(np.float32), rng.standard_normal((3, 3)).astype(np.float32)]
                got = run(emul, xs, fs, "HWC", None, border, "same", None, dtype)
                for x, f, g in zip(xs, fs, got):
                    assert fr.within(g, x, f, "HWC", (-1, -1), border, "same", None, dtype) == 0, (dt, dtype, border)


def test_anchors_at_every_position_of_1x1_to_7x7_and_non_square_filters(emul):
    rng = np.random.default_rng(3)
    x = data(rng, (9, 11, 2), np.uint8)
    for fh in range(1, 8):
        for fw in range(1, 8):
            f = exact_kernel(rng, fh, fw, True)
            anchors = [(r, s) for r in range(fh) for s in range(fw)]
            for border in fr.BORDERS:
                got = run(emul, [x] * len(anchors), [f] * len(anchors), "HWC", anchors, border, dtype=np.float32)
                for a, g in zip(anchors, got):
                    assert np.array_equal(g, fr.filter_ref(x, f, "HWC", a, border, dtype=np.float32)), (fh, fw, a, border)


def test_filters_larger_than_the_sample_under_every_border(emul):
    rng = np.random.default_rng(4)
    for shape in ((1, 1, 1), (1, 5, 2), (3, 2, 3), (2, 7, 1)):
        x = data(rng, shape, np.int16)
        for fsz in ((15, 9), (31, 1), (1, 23), (40, 40)):
            f = exact_kernel(rng, *fsz, False)
            for border in fr.BORDERS:
                a = (int(rng.integers(fsz[0])), int(rng.integers(fsz[1])))
                (g,) = run(emul, [x], [f], "HWC", [a], border, dtype=np.float32)
                assert np.array_equal(g, fr.filter_ref(x, f, "HWC", a, border, dtype=np.float32)), (shape, fsz, border)


def test_per_frame_fill_values_and_empty_samples_and_frames(emul):
    rng = np.random.default_rng(5)
    seq = data(rng, (4, 10, 12, 3), np.uint8)
    f = exact_kernel(rng, 5, 3, False)
    fills = [np.array([0, 50, 100, 255], np.uint8), np.array(9, np.uint8)]
    got = run(emul, [seq, seq[:2]], [f, f], "FHWC", None, "constant", "same", fills, np.float32)
    for x, g, v in zip([seq, seq[:2]], got, fills):
        assert np.array_equal(g, fr.filter_ref(x, f, "FHWC", (-1, -1), "constant", "same", v, np.float32))
    xs = [np.zeros((0, 5, 3), np.uint8), data(rng, (4, 5, 3), np.uint8), np.zeros((4, 0, 3), np.uint8), np.zeros((4, 5, 0), np.uint8)]
    got = run(emul, xs, [f] * 4, "HWC")
    for x, g in zip(xs, got):
        assert g.shape == x.shape and np.array_equal(g, fr.filter_ref(x, f, "HWC"))
    fs = [np.zeros((0, 6, 7), np.uint8), data(rng, (3, 6, 7), np.uint8)]
    got = run(emul, fs, [f] * 2, "FHW", mode="valid")
    assert [g.shape for g in got] == [(0, 2, 5), (3, 2, 5)] and np.array_equal(got[1], fr.filter_ref(fs[1], f, "FHW", mode="valid"))


def test_every_byte_offset(emul):
    rng = np.random.default_rng(6)
    f = exact_kernel(rng, 3, 3, True)
    for dt in (np.uint8, np.int16, np.float32):
        x = data(rng, (19, 45, 3), dt)
        if dt == np.int16:
            x = (x // 64).astype(dt)
        want = fr.filter_ref(x, f, "HWC", dtype=np.float32) if dt != np.float32 else None
        for a in range(16):
            got = run(emul, [x, x], [f, f], "HWC", dtype=np.float32, offs=(a, (a + 5) % 16))
            for g in got:
                if want is None:
                    assert fr.within(g, x, f, "HWC", dtype=np.float32) == 0
                else:
                    assert np.array_equal(g, want), (dt, a)


def test_random_cases_under_sanitizers(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path / "flt_fuzz")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-DFILTER_EMUL_MAIN", SRC, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    for seed in (1, 2, 3):
        r = subprocess.run([exe, "150", str(seed)], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0 and r.stdout.strip() == "ok 150", (r.stdout[-2000:], r.stderr[-3000:])
