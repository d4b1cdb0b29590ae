"""fn.multi_paste and fn.paste without a GPU:
  * the planner and the kernel bodies compiled for the host (tools/emul/paste_emul.cc), every work item and thread run in reverse
    order, bit for bit against tests/paste_ref.py: all 12 input types into a spread of output types and every type pair once; 0, 1,
    4 (mosaic), 64 and 256 regions; full overlap, nested, edge-touching and zero-size regions; every _rel form with .5 ties; 1, 3, 4 and
    5 channels; every byte offset of input and output; in_ids repeating a sample and naming the output's own index; the multi-input
    form; paste at ratio 1, at paste_x / paste_y 0 and 1 and where min_canvas_size dominates;
  * the band count and host time of 256 regions;
  * every refusal, with its message, through the planner and through the operator's argument resolution (dalihTestMultiPaste);
  * random cases under ASan + UBSan."""
import ctypes as C
import os
import shutil
import subprocess
import sys
import time

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import paste_ref as pr  # noqa: E402
from erase_ref import TYPES  # noqa: E402
from test_erase_cpu import DTYPES, data  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tools", "emul", "paste_emul.cc")
P64 = C.POINTER(C.c_int64)


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    so = str(tmp_path_factory.mktemp("ps") / "paste_emul.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", SRC, "-o", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


def placed(x, off, keep, fill=0):
    buf = np.full(x.nbytes + 64, fill, np.uint8)
    base = (-buf.ctypes.data) % 16 + 16 + off
    buf[base:base + x.nbytes] = np.ascontiguousarray(x).view(np.uint8).reshape(-1)
    keep.append((buf, base, x.nbytes))
    return buf.ctypes.data + base


def setup_args(inputs, args, in_ids, out_sizes, n):
    """the C arrays of a set-up: shapes input-major, in_ids, the six region arguments and output_size"""
    ninputs = len(inputs)
    shapes = [e for inp in inputs for x in inp for e in (x.shape if x.ndim == 3 else (0, 0, 0))]
    ids = idc = None
    if in_ids is not None:
        flat_ids = [int(v) for row in in_ids for v in row] or [0]
        ids = (C.c_int32 * len(flat_ids))(*flat_ids)
        idc = (C.c_int64 * n)(*[len(row) for row in in_ids])
    av = (C.POINTER(C.c_double) * 6)()
    ac = (P64 * 6)()
    keep = []
    for a, name in enumerate(pr.ARGS):
        if name not in args:
            continue
        rows = [np.asarray(v, np.float64).reshape(-1) for v in args[name]]
        vals = np.concatenate(rows + [np.zeros(1)])
        cnt = np.array([len(r) for r in rows], np.int64)
        keep += [vals, cnt]
        av[a] = vals.ctypes.data_as(C.POINTER(C.c_double))
        ac[a] = cnt.ctypes.data_as(P64)
    osz = (C.c_int64 * (2 * n))(*[v for s in out_sizes for v in s]) if out_sizes is not None else None
    return ((C.c_int * ninputs)(*[inp[0].ndim if inp else 3 for inp in inputs]), (C.c_char_p * ninputs)(*[b"HWC"] * ninputs),
            (C.c_int64 * max(1, len(shapes)))(*shapes), ids, idc, av, ac, osz, keep)


def mp_plan(lib, inputs, args=None, in_ids=None, out_sizes=None, dtype=None, ins=None, outs=None, items=None, bands=None, fill=(0.0,)):
    """(rc, message, output shapes) of a set-up of the host build; inputs: per input, its n samples"""
    n = len(inputs[0])
    nd, lay, shp, ids, idc, av, ac, osz, _keep = setup_args(inputs, args or {}, in_ids, out_sizes, n)
    err = C.create_string_buffer(512)
    oshapes = (C.c_int64 * max(1, 3 * n))()
    it = TYPES[inputs[0][0].dtype]
    ot = -1 if dtype is None else TYPES[np.dtype(dtype)]
    rc = lib.emul_paste(it, ot, len(inputs), n, nd, lay, shp, ids, idc, av, ac, osz, (C.c_float * len(fill))(*fill), len(fill), ins, outs,
                        oshapes, items, bands, err, 512)
    return rc, err.value.decode(), [tuple(oshapes[3 * i:3 * i + 3]) for i in range(n)]


def mp_run(lib, inputs, args=None, in_ids=None, out_sizes=None, dtype=None, offs=(0, 0)):
    """outputs of the host build; input sample s at byte (offs[0] + s) past a 16-byte boundary and output i at (offs[1] + 3 i), rounded
    down to the element size; the bytes around each output checked"""
    n = len(inputs[0])
    rc, msg, oshapes = mp_plan(lib, inputs, args, in_ids, out_sizes, dtype)
    assert rc == 0, msg
    odt = np.dtype(dtype or inputs[0][0].dtype)
    keep, outs = [], []
    flat = [x for inp in inputs for x in inp]
    ip = [placed(x, (offs[0] + s) % 16 // x.itemsize * x.itemsize, keep) for s, x in enumerate(flat)]
    op = [placed(np.zeros(s, odt), (offs[1] + 3 * i) % 16 // odt.itemsize * odt.itemsize, outs, 0xA5) for i, s in enumerate(oshapes)]
    rc, msg, _ = mp_plan(lib, inputs, args, in_ids, out_sizes, dtype, (C.c_void_p * len(ip))(*ip), (C.c_void_p * n)(*op))
    assert rc == 0, msg
    res = []
    for (buf, base, nb), s in zip(outs, oshapes):
        assert np.all(buf[:base] == 0xA5) and np.all(buf[base + nb:] == 0xA5), "a write outside the output"
        res.append(buf[base:base + nb].view(odt).reshape(s))
    return res


def mp_check(lib, inputs, args=None, in_ids=None, out_sizes=None, dtype=None, offs=(0, 0)):
    args = args or {}
    n = len(inputs[0])
    got = mp_run(lib, inputs, args, in_ids, out_sizes, dtype, offs)
    for i in range(n):
        srcs = [inputs[0][j] for j in in_ids[i]] if in_ids is not None else [inp[i] for inp in inputs]
        hw = tuple(out_sizes[i]) if out_sizes is not None else inputs[0][0].shape[:2]
        want = pr.multi_paste_ref(srcs, hw, {k: v[i] for k, v in args.items()}, dtype or inputs[0][0].dtype, inputs[0][0].shape[2])
        assert got[i].dtype == want.dtype and got[i].tobytes() == want.tobytes(), (i, inputs[0][0].dtype, dtype)
    return got


def random_regions(rng, src_shapes, out_hw, zero=0.1):
    """absolute in_anchors, shapes and out_anchors of regions inside their sources and the output"""
    ia, sh, oa = [], [], []
    for hs, ws, _ in src_shapes:
        h = 0 if rng.random() < zero else int(rng.integers(0, min(hs, out_hw[0]) + 1))
        w = 0 if rng.random() < zero else int(rng.integers(0, min(ws, out_hw[1]) + 1))
        ia.append([int(rng.integers(0, hs - h + 1)), int(rng.integers(0, ws - w + 1))])
        sh.append([h, w])
        oa.append([int(rng.integers(0, out_hw[0] - h + 1)), int(rng.integers(0, out_hw[1] - w + 1))])
    return np.array(ia).reshape(-1, 2), np.array(sh).reshape(-1, 2), np.array(oa).reshape(-1, 2)


def ids_case(rng, batch, k, out_hw):
    ids = [list(rng.integers(0, len(batch), k)) for _ in batch]
    regs = [random_regions(rng, [batch[j].shape for j in row], out_hw) for row in ids]
    args = {"in_anchors": [r[0] for r in regs], "shapes": [r[1] for r in regs], "out_anchors": [r[2] for r in regs]}
    return ids, args


def test_every_input_type_into_a_spread_of_output_types(emul):
    rng = np.random.default_rng(1)
    for it in DTYPES:
        batch = [data(rng, (13, 21, 3), it), data(rng, (9, 30, 3), it), data(rng, (17, 5, 3), it)]
        ids, args = ids_case(rng, batch, 5, (19, 23))
        for ot in (None, np.uint8, np.int16, np.float16, np.float32, np.int64, np.bool_):
            mp_check(emul, [batch], args, ids, [(19, 23)] * 3, ot, offs=(int(rng.integers(16)), int(rng.integers(16))))


def test_every_type_pair_converts_with_convert_sat(emul):
    rng = np.random.default_rng(2)
    for it in DTYPES:
        batch = [data(rng, (6, 11, 2), it), data(rng, (6, 11, 2), it)]
        for ot in DTYPES:
            ids = [[0, 1], [1, 0]]
            args = {"in_anchors": [[[0, 0], [1, 2]]] * 2, "shapes": [[[6, 11], [4, 7]]] * 2, "out_anchors": [[[0, 0], [2, 3]]] * 2}
            mp_check(emul, [batch], args, ids, None, ot)


def test_region_counts_0_1_4_64_and_256(emul):
    rng = np.random.default_rng(3)
    batch = [data(rng, (40, 52, 3), np.uint8) for _ in range(4)]
    for k in (0, 1, 4, 64, 256):
        ids, args = ids_case(rng, batch, k, (50, 61))
        mp_check(emul, [batch], args, ids, [(50, 61)] * 4)
    # the 4-tile mosaic: each output the four samples' quarters around a centre
    tiles = [data(rng, (32, 32, 3), np.uint8) for _ in range(4)]
    ids = [[0, 1, 2, 3], [3, 2, 1, 0], [1, 1, 1, 1], [2, 0, 3, 1]]
    oa, sh, ia = [], [], []
    for yc, xc in ((32, 32), (17, 45), (40, 21), (32, 9)):
        oa.append([[0, 0], [0, xc], [yc, 0], [yc, xc]])
        sh.append([[yc, xc], [yc, 64 - xc], [64 - yc, xc], [64 - yc, 64 - xc]])
        ia.append([[32 - yc if yc < 32 else 0, 32 - xc if xc < 32 else 0], [0, 0], [0, 0], [0, 0]])
    sh = [[[min(h, 32), min(w, 32)] for h, w in s] for s in sh]
    mp_check(emul, [tiles], {"in_anchors": ia, "shapes": sh, "out_anchors": oa}, ids, [(64, 64)] * 4)


def test_256_regions_band_count_and_host_time(emul):
    rng = np.random.default_rng(4)
    batch = [data(rng, (200, 300, 3), np.uint8) for _ in range(2)]
    ids, args = ids_case(rng, batch, 256, (400, 500))
    items, bands = (C.c_int64 * 2)(), (C.c_int64 * 2)()
    t = time.perf_counter()
    rc, msg, _ = mp_plan(emul, [batch], args, ids, [(400, 500)] * 2, items=items, bands=bands)
    assert rc == 0, msg
    assert time.perf_counter() - t < 2.0
    assert all(1 <= b <= 2 * 256 + 1 for b in bands), list(bands)
    mp_check(emul, [batch], args, ids, [(400, 500)] * 2)


def test_overlaps_nesting_edges_and_zero_size(emul):
    rng = np.random.default_rng(5)
    batch = [data(rng, (20, 24, 3), np.int16) for _ in range(3)]
    cases = {
        "full overlap": ([[0, 0], [0, 0]], [[20, 24], [20, 24]], [[0, 0], [0, 0]]),
        "nested": ([[0, 0], [2, 3], [5, 5]], [[20, 24], [10, 12], [2, 2]], [[0, 0], [4, 4], [8, 9]]),
        "edge-touching": ([[0, 0], [0, 0], [0, 0]], [[10, 12], [10, 12], [10, 12]], [[0, 0], [0, 12], [10, 0]]),
        "zero-size": ([[3, 3], [0, 0], [19, 23]], [[0, 5], [5, 0], [1, 1]], [[20, 24], [0, 0], [0, 0]]),
        "outer edge": ([[0, 0], [0, 0]], [[1, 24], [20, 1]], [[19, 0], [0, 23]]),
    }
    for name, (ia, sh, oa) in cases.items():
        ids = [[0, 1, 2][:len(ia)]] * 3
        mp_check(emul, [batch], {"in_anchors": [ia] * 3, "shapes": [sh] * 3, "out_anchors": [oa] * 3}, ids, None)
    # an output over its own sample's earlier region: a later region on top
    (g, _, _) = mp_check(emul, [batch], {"out_anchors": [[[0, 0], [0, 0]]] * 3}, [[0, 1], [1, 2], [2, 0]], None)
    assert g.tobytes() == batch[1].tobytes()


def test_every_rel_form_with_ties(emul):
    rng = np.random.default_rng(6)
    batch = [data(rng, (10, 14, 3), np.uint8) for _ in range(2)]
    # ties: 0.25 * 10 = 2.5 -> 3, 0.25 * 14 = 3.5 -> 4, 0.65 * 10 = 6.5 -> 7, 0.125 * 20 = 2.5 -> 3, 0.05 * 30 = 1.5 -> 2; 20 x 30 out
    args = {"in_anchors_rel": [[[0.25, 0.25]], [[0.05, 0.0]]], "shapes_rel": [[[0.65, 0.25]], [[0.35, 0.75]]],
            "out_anchors_rel": [[[0.125, 0.05]], [[0.525, 0.55]]]}
    g = mp_check(emul, [batch], args, [[1], [0]], [(20, 30)] * 2)
    ref = pr.regions([batch[1].shape], (20, 30), {k: v[0] for k, v in args.items()})
    assert ref == [(0, 3, 4, 7, 4, 3, 2)], ref
    assert g[0].any()
    for combo in (("in_anchors", "shapes_rel", "out_anchors"), ("in_anchors_rel", "shapes", "out_anchors_rel")):
        a = {"in_anchors": [[[1, 2]]] * 2, "shapes": [[[4, 5]]] * 2, "out_anchors": [[[3, 3]]] * 2,
             "in_anchors_rel": [[[0.15, 0.5]]] * 2, "shapes_rel": [[[0.45, 0.25]]] * 2, "out_anchors_rel": [[[0.025, 0.5]]] * 2}
        mp_check(emul, [batch], {k: a[k] for k in combo}, [[0], [1]], [(20, 30)] * 2)


def test_channels_1_3_4_5_and_every_byte_offset(emul):
    rng = np.random.default_rng(7)
    for c in (1, 3, 4, 5):
        for dt in (np.uint8, np.uint16, np.float32, np.float64):
            batch = [data(rng, (15, 37, c), dt) for _ in range(3)]
            ids, args = ids_case(rng, batch, 4, (21, 41))
            mp_check(emul, [batch], args, ids, [(21, 41)] * 3, offs=(int(rng.integers(16)), int(rng.integers(16))))
    for dt in (np.uint8, np.int16, np.float32, np.float64):
        batch = [data(rng, (19, 45, 3), dt) for _ in range(2)]
        ids, args = ids_case(rng, batch, 3, (23, 50))
        for o in range(16):
            for p in (o, (o + 5) % 16):
                mp_check(emul, [batch], args, ids, [(23, 50)] * 2, offs=(o, p))
                mp_check(emul, [batch], args, ids, [(23, 50)] * 2, np.float16 if dt != np.float16 else np.uint8, offs=(o, p))


def test_in_ids_repeating_a_sample_and_naming_the_own_index(emul):
    rng = np.random.default_rng(8)
    batch = [data(rng, (12, 16, 3), np.uint8) for _ in range(3)]
    ids = [[0, 0, 0], [1, 2, 1], [2, 2, 2]]
    regs = [random_regions(rng, [batch[j].shape for j in row], (12, 16), 0) for row in ids]
    mp_check(emul, [batch], {"in_anchors": [r[0] for r in regs], "shapes": [r[1] for r in regs], "out_anchors": [r[2] for r in regs]},
             ids, None)


def test_multi_input_form(emul):
    rng = np.random.default_rng(9)
    for ninputs in (1, 2, 4, 64):
        inputs = [[data(rng, (9, 11, 3), np.uint8) for _ in range(3)] for _ in range(ninputs)]
        regs = [random_regions(rng, [inp[i].shape for inp in inputs], (14, 15)) for i in range(3)]
        args = {"in_anchors": [r[0] for r in regs], "shapes": [r[1] for r in regs], "out_anchors": [r[2] for r in regs]}
        mp_check(emul, inputs, args, None, [(14, 15)] * 3)
    # without arguments: every input whole at (0, 0), the last on top; without output_size the common shape
    inputs = [[data(rng, (9, 11, 3), np.float32) for _ in range(2)] for _ in range(3)]
    g = mp_check(emul, inputs)
    assert g[1].tobytes() == inputs[2][1].tobytes()


def canvas(lib, xs, ratio, px, py, mc, fill, n_channels=3, ins=None, outs=None):
    n = len(xs)
    f = lambda v: (C.c_float * n)(*([v] * n if np.isscalar(v) else v))  # noqa: E731
    err = C.create_string_buffer(512)
    oshapes = (C.c_int64 * max(1, 3 * n))()
    shp = [e for x in xs for e in x.shape]
    rc = lib.emul_paste_canvas(TYPES[xs[0].dtype], n, xs[0].ndim, b"HWC", (C.c_int64 * max(1, len(shp)))(*shp), n_channels, f(ratio), f(px),
                               f(py), f(mc), (C.c_float * len(fill))(*fill), len(fill), ins, outs, oshapes, err, 512)
    return rc, err.value.decode(), [tuple(oshapes[3 * i:3 * i + 3]) for i in range(n)]


def paste_check(lib, xs, ratio, px=0.5, py=0.5, mc=0.0, fill=(0.0,), off=0):
    rc, msg, oshapes = canvas(lib, xs, ratio, px, py, mc, fill, xs[0].shape[2])
    assert rc == 0, msg
    keep, outs = [], []
    ip = [placed(x, (off + i) % 16, keep) for i, x in enumerate(xs)]
    op = [placed(np.zeros(s, np.uint8), (off + 3 * i) % 16, outs, 0xA5) for i, s in enumerate(oshapes)]
    rc, msg, _ = canvas(lib, xs, ratio, px, py, mc, fill, xs[0].shape[2], (C.c_void_p * len(xs))(*ip), (C.c_void_p * len(xs))(*op))
    assert rc == 0, msg
    per = lambda v, i: v if np.isscalar(v) else v[i]  # noqa: E731
    for i, ((buf, base, nb), s) in enumerate(zip(outs, oshapes)):
        assert np.all(buf[:base] == 0xA5) and np.all(buf[base + nb:] == 0xA5), "a write outside the output"
        want = pr.paste_ref(xs[i], per(ratio, i), per(px, i), per(py, i), per(mc, i), fill)
        assert buf[base:base + nb].tobytes() == want.tobytes() and want.shape == s, (i, s, want.shape)


def test_paste_ratio_positions_and_min_canvas(emul):
    rng = np.random.default_rng(10)
    xs = [rng.integers(0, 256, (h, w, 3), dtype=np.uint8) for h, w in ((30, 30), (17, 41), (1, 1), (0, 5))]
    fill = (123.0, 117.0, 104.0)
    paste_check(emul, xs, 1.0, fill=fill)
    for px in (0.0, 1.0, 0.5, 0.3):
        for py in (0.0, 1.0, 0.7):
            paste_check(emul, xs, 2.5, px, py, fill=fill, off=int(rng.integers(16)))
    paste_check(emul, xs, 1.5, mc=100.0, fill=(9.0,))                        # min_canvas_size dominates
    paste_check(emul, xs, [1.0, 3.7, 4.0, 2.0], [0.0, 0.25, 1.0, 0.5], [1.0, 0.5, 0.0, 0.5], [0.0, 10.0, 3.0, 50.0], fill)
    assert pr.paste_geometry(30, 17, 1.1) == (33, 18, 1, 0)                   # 1.1f * 30 = 33.0000..., 1.1f * 17 = 18.7 -> 18
    gray = [rng.integers(0, 256, (7, 9, 1), dtype=np.uint8)]
    paste_check(emul, gray, 2.0, fill=(300.0,))                               # the fill converted with ConvertSat: 255


def test_refusals_name_the_sample_region_and_argument(emul):
    u8 = lambda *s: np.zeros(s, np.uint8)  # noqa: E731
    b2 = [u8(4, 5, 3), u8(4, 5, 3)]

    def msg(*a, **k):
        rc, m, _ = mp_plan(emul, *a, **k)
        assert rc == 1
        return m
    assert "in_ids is given, so exactly one input is allowed; got 2" in msg([b2, b2], in_ids=[[0], [0]])
    assert "both in_anchors and in_anchors_rel are given" in msg([b2], {"in_anchors": [[[0, 0]]] * 2, "in_anchors_rel": [[[0, 0]]] * 2})
    assert "both shapes and shapes_rel are given" in msg([b2], {"shapes": [[[1, 1]]] * 2, "shapes_rel": [[[0, 0]]] * 2})
    assert "both out_anchors and out_anchors_rel are given" in msg([b2], {"out_anchors": [[[0, 0]]] * 2, "out_anchors_rel": [[[0, 0]]] * 2})
    assert "sample 1, region 0: in_ids 2 is not a sample of the batch of 2" in msg([b2], in_ids=[[0], [2]])
    assert "sample 0, region 0: in_ids -1 is not a sample" in msg([b2], in_ids=[[-1], [0]])
    assert "sample 1: in_anchors has 4 values; its 1 regions need 2 (a [1, 2] tensor)" in msg([b2], {"in_anchors": [[[0, 0]], [[0, 0], [0, 0]]]},
                                                                                                in_ids=[[0], [1]])
    assert "sample 0, region 0: shapes gives the extent (-1, 2), which is negative" in msg([b2], {"shapes": [[[-1, 2]]] * 2}, in_ids=[[0], [1]])
    assert ("sample 0, region 0: in_anchors (1, 1) and shapes (4, 4) leave the source, sample 1 of input 0 (4 x 5)"
            in msg([b2], {"in_anchors": [[[1, 1]]] * 2, "shapes": [[[4, 4]]] * 2}, in_ids=[[1], [0]]))
    assert ("sample 0, region 0: in_anchors (default) (0, 0) and shapes (5, 1) leave the source"
            in msg([b2], {"shapes": [[[5, 1]]] * 2}, in_ids=[[1], [0]]))
    assert ("sample 1, region 0: out_anchors (3, 0) and shapes (default) (4, 5) leave the output (6 x 6)"
            in msg([b2], {"out_anchors": [[[0, 0]], [[3, 0]]]}, in_ids=[[0], [1]], out_sizes=[(6, 6), (6, 6)]))
    assert ("sample 0, region 0: out_anchors_rel (1, 0) and shapes (default)" in
            msg([b2], {"out_anchors_rel": [[[0.25, 0.0]]] * 2}, in_ids=[[0], [1]]))
    assert "sample 0, region 0: in_anchors value 0.5 is not an integer" in msg([b2], {"in_anchors": [[[0.5, 0]]] * 2}, in_ids=[[0], [1]])
    assert "sample 0, region 0: shapes_rel value nan is not finite" in msg([b2], {"shapes_rel": [[[np.nan, 0]]] * 2}, in_ids=[[0], [1]])
    assert ("output_size is not given, and sample 1 of input 0 has the shape [4, 6, 3] where sample 0 of input 0 has [4, 5, 3]"
            in msg([[u8(4, 5, 3), u8(4, 6, 3)]], in_ids=[[0], [1]]))
    assert "sample 1 of input 0 has 4 channels, sample 0 of input 0 has 3" in msg([[u8(4, 5, 3), u8(4, 5, 4)]], in_ids=[[0], [1]])
    assert "sample 0: output_size (-1, 5) has a negative extent" in msg([b2], in_ids=[[0], [1]], out_sizes=[(-1, 5), (4, 5)])
    assert "input 0 has 2 dimensions; HWC images of rank 3 are supported" in msg([[u8(4, 5), u8(4, 5)]], in_ids=[[0], [1]])
    assert "65 inputs; 1 to 64 are supported" in msg([b2] * 65)
    # the layout rule and fill counts, through the planner directly
    n = 1
    err = C.create_string_buffer(512)
    av, ac = (C.POINTER(C.c_double) * 6)(), (P64 * 6)()
    rc = emul.emul_paste(0, -1, 1, n, (C.c_int * 1)(3), (C.c_char_p * 1)(b"CHW"), (C.c_int64 * 3)(3, 4, 5), None, None, av, ac, None,
                         (C.c_float * 1)(0), 1, None, None, None, None, None, err, 512)
    assert rc == 1 and 'input 0 has layout "CHW"; only HWC images' in err.value.decode()
    rc = emul.emul_paste(0, 12, 1, n, (C.c_int * 1)(3), None, (C.c_int64 * 3)(3, 4, 5), None, None, av, ac, None, (C.c_float * 1)(0), 1,
                         None, None, None, None, None, err, 512)
    assert rc == 1 and "dtype has an unsupported type (code 12)" in err.value.decode()
    # paste
    xs = [u8(4, 5, 3)]
    assert "sample 0: ratio 0.5 is less than 1" in canvas(emul, xs, 0.5, 0.5, 0.5, 0.0, (0.0,))[1]
    assert "sample 0: ratio nan is less than 1" in canvas(emul, xs, float("nan"), 0.5, 0.5, 0.0, (0.0,))[1]
    assert "sample 0: paste_x 1.5 is not in [0, 1]" in canvas(emul, xs, 2.0, 1.5, 0.5, 0.0, (0.0,))[1]
    assert "sample 0: paste_y -0.5 is not in [0, 1]" in canvas(emul, xs, 2.0, 0.5, -0.5, 0.0, (0.0,))[1]
    assert "sample 0: min_canvas_size -1 is negative" in canvas(emul, xs, 2.0, 0.5, 0.5, -1.0, (0.0,))[1]
    assert "fill_value has 2 values; one per channel (3), or one for all, is needed" in canvas(emul, xs, 2.0, 0.5, 0.5, 0.0, (0.0, 1.0))[1]
    assert "sample 0 has 3 channels, but n_channels is 4" in canvas(emul, xs, 2.0, 0.5, 0.5, 0.0, (0.0,), 4)[1]
    assert "paste takes UINT8 images" in canvas(emul, [np.zeros((4, 5, 3), np.float32)], 2.0, 0.5, 0.5, 0.0, (0.0,))[1]
    assert "does not fit in an int" in canvas(emul, xs, 1e9, 0.5, 0.5, 0.0, (0.0,))[1]


def test_operator_argument_resolution_and_refusals():
    """dalihTestMultiPaste: the operator's reading of list arguments and dtype, then the plan set-up"""
    from dali_b200 import backend
    L = backend.lib()

    def rule(shp, n=2, ninputs=1, ids=None, dtype=-1, size=None, **args):
        s = np.array([v for _ in range(ninputs) for sh in shp for v in sh], np.int64)
        av = (C.POINTER(C.c_double) * 6)()
        nv = (C.c_int * 6)()
        keep = []
        for a, name in enumerate(pr.ARGS):
            if name in args:
                v = np.asarray(args[name], np.float64).reshape(-1)
                keep.append(v)
                av[a], nv[a] = v.ctypes.data_as(C.POINTER(C.c_double)), len(v)
        oshapes = (C.c_int64 * (3 * n))()
        rc = L.dalihTestMultiPaste(0, dtype, ninputs, n, (C.c_int * ninputs)(*[3] * ninputs), None, s.ctypes.data_as(P64),
                                   (C.c_int64 * max(1, len(ids or [])))(*(ids or [])) if ids is not None else None, len(ids or []), av, nv,
                                   (C.c_int64 * 2)(*size) if size else None, oshapes)
        return (L.dalihLastError().decode() if rc else None), [tuple(oshapes[3 * i:3 * i + 3]) for i in range(n)]
    sh = [(4, 5, 3), (4, 5, 3)]
    assert rule(sh, ids=[0, 1], size=(8, 9), out_anchors=[0, 0, 4, 4]) == (None, [(8, 9, 3)] * 2)
    assert rule(sh, ninputs=3) == (None, [(4, 5, 3)] * 2)
    assert rule(sh, ids=[0], dtype=9)[0] is None
    assert "both shapes and shapes_rel are given" in rule(sh, ids=[0], shapes=[1, 1], shapes_rel=[0.5, 0.5])[0]
    assert "sample 0: in_anchors has 2 values; its 2 regions need 4" in rule(sh, ids=[0, 1], in_anchors=[0, 0])[0]
    assert "invalid dtype 13" in rule(sh, ids=[0], dtype=13)[0]


def test_launch_refuses_device_pointers_not_aligned_to_their_element():
    from dali_b200 import capi
    L = capi.lib()
    plan = C.c_void_p()
    capi.check(L.dalib200PastePlanCreate(C.byref(plan), 1))
    try:
        av, ac = (C.POINTER(C.c_double) * 6)(), (P64 * 6)()
        out = (C.c_int64 * 3)()
        capi.check(L.dalib200PasteSetup(plan, 5, -1, 1, 1, (C.c_int * 1)(3), None, (C.c_int64 * 3)(4, 5, 3), None, None, av, ac, None,
                                        (C.c_float * 1)(0), 1, out))
        assert list(out) == [4, 5, 3]
        for ip, op, what in ((0x10001, 0x20000, "sample 0 of input 0: the input pointer"), (0x10000, 0x20003, "sample 0: the output pointer")):
            rc = L.dalib200PasteLaunch(plan, (C.c_void_p * 1)(ip), (C.c_void_p * 1)(op), None)
            assert rc != 0 and what + " is not aligned to its element size" in L.dalib200GetLastError().decode()
    finally:
        L.dalib200PastePlanDestroy(plan)


def test_random_cases_under_sanitizers(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path / "ps_fuzz")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-DPASTE_EMUL_MAIN",
                        SRC, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    for seed in (1, 2, 3):
        r = subprocess.run([exe, "300", str(seed)], capture_output=True, text=True, timeout=900)
        assert r.returncode == 0 and r.stdout.strip() == "ok 300", (r.stdout[-2000:], r.stderr[-3000:])
