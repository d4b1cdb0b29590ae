"""Arithmetic expressions without a GPU:
  * tests/arith_ref.py pinned against numpy wherever numpy agrees (and the cases where it does not, stated);
  * the Python graph building: the expression_desc strings, fusion and materialisation, constants, device rules and refusals;
  * the planner and the kernel bodies compiled for the host (tools/emul/arith_emul.cc): every operator over every type pair of the
    12 types on edge and random values, bit for bit against arith_ref.py (transcendentals within ULP bounds of a float64
    evaluation), broadcasting, the shape edges of arith_ref.shape_cases (ranks 0-6, broadcast patterns up to 16 operands, empty and
    0-d samples, volumes around the threads and work items) with operands and outputs at unaligned offsets and every output checked
    for stray writes, fn.cast against pointwise_ref's ConvertSat, the planner's limits and refusals, and mutated descriptions under
    ASan + UBSan."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import arith_ref as ar
import pointwise_ref as pr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tools", "emul", "arith_emul.cc")


# ---- the statement against numpy
def test_promotion_agrees_with_numpy_except_where_stated():
    # numpy promotes these differently: it keeps integer precision in a wider float (int16 + float16 -> float32, int32 + float32 ->
    # float64, uint64 + int64 -> float64); the reference picks the float operand's type / caps at INT64
    differ = set()
    for a in ar.TYPES:
        for b in ar.TYPES:
            want = np.result_type(ar.NP[a], ar.NP[b])
            got = ar.NP[ar.promote(a, b)]
            if np.dtype(got) != want:
                differ.add((a, b))
                fa, fb = a in ar.FLOATS, b in ar.FLOATS
                assert fa != fb or {a, b} == {ar.U64, ar.I64} or (a in ar.SIGNED and b == ar.U64) or (b in ar.SIGNED and a == ar.U64), \
                    (ar.NAMES[a], ar.NAMES[b], ar.NAMES[ar.promote(a, b)], want)
    assert (ar.I16, ar.F16) in differ and (ar.I32, ar.F32) in differ and (ar.U64, ar.I64) in differ
    assert ar.promote(ar.U8, ar.I8) == ar.I16 and ar.promote(ar.U32, ar.I32) == ar.I64 and ar.promote(ar.BOOL, ar.I8) == ar.I8
    assert ar.promote(ar.BOOL, ar.U8) == ar.U8 and ar.promote(ar.F16, ar.F64) == ar.F64 and ar.promote(ar.I64, ar.F16) == ar.F16


def test_statement_agrees_with_numpy_on_plain_arithmetic():
    rng = np.random.default_rng(0)
    for t in (ar.U8, ar.I16, ar.I32, ar.U32, ar.F32, ar.F64):
        a, b = ar.random_values(t, 200, rng), ar.random_values(t, 200, rng)
        with np.errstate(all="ignore"):
            for op, f in (("add", np.add), ("sub", np.subtract), ("mul", np.multiply), ("min", np.minimum), ("max", np.maximum)):
                assert ar.same_bits(ar.evaluate(op, [a, b], [t, t]), f(a, b).astype(ar.NP[t])), (op, t)
            if t not in ar.FLOATS:
                nz = np.where((b == 0) | (b == -1), 1, b)          # numpy floors; with trunc it agrees away from x // 0 and MIN // -1
                assert np.array_equal(ar.evaluate("div", [a, nz], [t, t]), np.trunc(a.astype(np.float64) / nz).astype(ar.NP[t])), t
                assert np.array_equal(ar.evaluate("bitxor", [a, b], [t, t]), a ^ b)
    # integer division truncates toward zero (numpy floors), x // 0 is 0, negative powers are 0 except for bases +-1
    assert list(ar.evaluate("div", [np.array([-7, 7, -7, 5], np.int32), np.array([2, -2, 0, 0], np.int32)], [ar.I32, ar.I32])) == [-3, -3, 0, 0]
    assert list(ar.evaluate("pow", [np.array([2, 1, -1, -1, 0], np.int32), np.array([-1, -5, -3, -4, 3], np.int32)], [ar.I32, ar.I32])) == [0, 1, -1, 1, 0]
    # integer overflow wraps; an INT32 constant (a Python int) keeps an INT32 result where numpy's value-based rules would not
    assert ar.evaluate("mul", [np.array([2 ** 30], np.int32), np.int32(4)], [ar.I32, ar.I32])[0] == 0
    assert ar.evaluate("add", [np.array([200], np.uint8), np.int32(100)], [ar.U8, ar.I32]).dtype == np.int32
    # ConvertSat
    x = np.array([0.5, 1.5, 2.5, -0.5, -2.5, 254.5, 255.5, 300.0, -3.0, np.nan], np.float32)
    assert list(ar.convert_sat(x, ar.F32, ar.U8)) == [1, 2, 3, 0, 0, 255, 255, 255, 0, 0]
    assert list(ar.convert_sat(x, ar.F32, ar.I8)) == [1, 2, 3, -1, -3, 127, 127, 127, -3, 0]
    ok = ~np.isnan(x)
    assert np.array_equal(ar.convert_sat(x, ar.F32, ar.U8)[ok], pr.round_sat_u8(x[ok]))
    assert ar.half_sat(np.float32(1e6)) == np.float16(65504) and ar.half_sat(np.float32(2.0 ** -25)) == np.float16(2.0 ** -24)


# ---- graph building
def _define(fn_body, batch=2):
    import nvidia.dali as dali
    pipe = dali.Pipeline(batch_size=batch, num_threads=1, device_id=0)
    with pipe:
        outs = fn_body()
    return pipe, outs


def test_expression_desc_fusion_and_materialisation():
    from nvidia.dali import fn, types, math as dmath
    from dali_b200 import arith
    holder = {}

    def body():
        x = fn.external_source(device="gpu", name="x")
        m = fn.external_source(device="gpu", name="m")
        e = (fn.cast(x, dtype=types.FLOAT) * (1 / 255) - m) / 0.5
        holder["desc"] = arith.describe(e)
        holder["e"] = e
        c = fn.cast(x, dtype=types.INT16)
        holder["mask"] = (x == 3) | (x > 200)
        holder["clamp"] = arith.describe(dmath.clamp(x, 0, 1.5))
        holder["neg"] = arith.describe(-x + x // types.Constant(3, types.INT64))
        return e, c
    pipe, outs = _define(body)
    desc, inputs, ints, reals = holder["desc"]
    assert desc == "fdiv(sub(mul(cast_float32(&0) $0:float32) &1) $1:float32)", desc
    assert [i.name for i in inputs] == ["x", "m"] and ints == [] and reals == [1 / 255, 0.5]
    assert holder["clamp"][0] == "clamp(&0 $0:int32 $0:float32)" and holder["clamp"][2] == [0] and holder["clamp"][3] == [1.5]
    assert holder["neg"][0] == "add(minus(&0) div(&0 $0:int64))", holder["neg"][0]
    assert pipe._nodes == []                                   # nothing materialised until something needs it
    for o in outs:
        arith.materialize(o)
    assert [s for s, _, _ in pipe._nodes] == ["ArithmeticGenericOp", "Cast"]       # one operator per needed expression
    arith.materialize(outs[0])
    assert len(pipe._nodes) == 2                                # materialised once
    # an expression consumed by another operator becomes an input of the later expressions
    e = holder["e"]
    with pipe:
        f = e * 2
    assert arith.describe(f)[0] == "mul(&0 $0:int32)" and arith.describe(f)[1][0] is e


def test_constants_and_types():
    from nvidia.dali import types
    assert types.Constant(3).dtype == types.INT32 and types.Constant(3.0).dtype == types.FLOAT and types.Constant(True).dtype == types.BOOL
    assert types.Constant(7, types.UINT8).dtype == types.UINT8
    from dali_b200 import arith
    holder = {}

    def body():
        from nvidia.dali import fn
        x = fn.external_source(device="gpu")
        holder["d"] = arith.describe(x * -0.0 + 0.0 - types.Constant(2 ** 40, types.INT64) + True)
        return x
    _define(body)
    desc, _, ints, reals = holder["d"]
    assert desc == "add(sub(add(mul(&0 $0:float32) $1:float32) $0:int64) $1:bool)", desc
    assert [repr(v) for v in reals] == ["-0.0", "0.0"] and ints == [2 ** 40, 1]


def test_refusals():
    from nvidia.dali import fn
    import nvidia.dali as dali

    def cpu_only():
        u = fn.random.uniform(range=(0, 1))
        return u * 2
    with pytest.raises(TypeError, match=r"\.gpu\(\)"):
        _define(cpu_only)

    def truth():
        x = fn.external_source(device="gpu")
        if x:
            pass
    with pytest.raises(TypeError, match="truth value"):
        _define(truth)

    def chained():
        x = fn.external_source(device="gpu")
        return 0 < x < 1
    with pytest.raises(TypeError, match="truth value"):
        _define(chained)

    def bad_operand():
        x = fn.external_source(device="gpu")
        return x + "a"
    with pytest.raises(TypeError, match="Unsupported operand"):
        _define(bad_operand)
    # CPU operands: fn.random scalars stay on the CPU, an external source moves to the GPU
    holder = {}

    def mixed():
        x = fn.external_source(device="cpu", name="xc")
        u = fn.random.uniform(range=(0, 1))
        holder["e"] = x * u
        return holder["e"]
    _define(mixed)
    from dali_b200 import arith
    _, inputs, _, _ = arith.describe(holder["e"])
    assert [i.device for i in inputs] == ["gpu", "cpu"]
    assert dali.fn.cast.schema_name == "Cast"


# ---- the host build of the planner and the kernel bodies
@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    so = str(tmp_path_factory.mktemp("arith") / "arith_emul.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", SRC, "-o", so], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(so)


def _at(x, off):
    """a copy of x starting `off` bytes past a 64-byte boundary"""
    x = np.asarray(x)
    buf = np.zeros(x.nbytes + off + 64, np.uint8)
    start = (-buf.ctypes.data) % 64 + off
    y = buf[start:start + x.nbytes].view(x.dtype).reshape(x.shape)
    y[...] = x
    return y


def run(lib, desc, xs, types, scalar=None, ints=(), reals=(), out_offset=0):
    """Evaluates desc over one sample per entry of xs (a list of per-sample input lists); returns (outputs, error).  Each output is
    written `out_offset` bytes past a 64-byte boundary of a buffer filled with 0xA5, whose bytes around the output must stay so."""
    nin = len(types)
    n = len(xs)
    arrs = [[np.asarray(x, ar.NP[t]) for x, t in zip(sample, types)] for sample in xs]
    arrs = [[a if a.flags.c_contiguous else a.copy() for a in sample] for sample in arrs]
    ndims = (C.c_int32 * max(nin, 1))(*[arrs[0][k].ndim if not (scalar and scalar[k]) else 0 for k in range(nin)])
    shp = (C.c_int64 * (n * nin * 6 or 1))()
    for i in range(n):
        for k in range(nin):
            for a, e in enumerate(arrs[i][k].shape):
                shp[(i * nin + k) * 6 + a] = e
    ptrs = (C.c_void_p * (n * nin or 1))(*[arrs[i][k].ctypes.data for i in range(n) for k in range(nin)])
    sc = (C.c_uint8 * max(nin, 1))(*(scalar or [0] * nin))
    iv = (C.c_int64 * max(1, len(ints)))(*ints)
    rv = (C.c_double * max(1, len(reals)))(*reals)
    tv = (C.c_int32 * max(nin, 1))(*types)
    osh, ond, ot = (C.c_int64 * (6 * n))(), C.c_int32(), C.c_int32()
    err = C.create_string_buffer(1024)
    args = (desc.encode(), nin, tv, sc, iv, len(ints), rv, len(reals), n, ndims, shp, ptrs)
    if lib.emul_arith(*args, None, osh, C.byref(ond), C.byref(ot), err, 1024):
        return None, err.value.decode()
    dt = np.dtype(ar.NP[ot.value])
    outs, bufs, starts = [], [], []
    for i in range(n):
        shape = tuple(osh[i * 6 + a] for a in range(ond.value))
        nbytes = int(np.prod(shape, dtype=np.int64)) * dt.itemsize
        bufs.append(np.full(nbytes + out_offset + 128, 0xA5, np.uint8))
        starts.append((-bufs[i].ctypes.data) % 64 + out_offset)
        outs.append(bufs[i][starts[i]:starts[i] + nbytes].view(dt).reshape(shape))
    op = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    assert lib.emul_arith(*args, op, osh, C.byref(ond), C.byref(ot), err, 1024) == 0
    for i, (o, b, s) in enumerate(zip(outs, bufs, starts)):
        assert np.all(b[:s] == 0xA5) and np.all(b[s + o.nbytes:] == 0xA5), ("written outside the output", desc, i)
    return [o.copy() for o in outs], None


ULP_HOST = 4          # glibc's float math functions against a float64 evaluation (FLOAT64: one more for the reference's own rounding)


def _check(op, got, xs, types):
    ar.check(op, got, xs, types, ULP_HOST)


def test_every_op_every_type_pair_bit_exact(emul):
    rng = np.random.default_rng(11)
    unary = [o for o, k in ar.ARITY.items() if k == 1]
    binary = [o for o, k in ar.ARITY.items() if k == 2]
    for ta in ar.TYPES:
        xs = [np.concatenate([ar.edge_values(ta), ar.random_values(ta, 64, rng)])]
        for op in unary:
            (got,), e = run(emul, f"{op}(&0)", [xs], [ta])
            assert e is None, e
            _check(op, got, xs, [ta])
        for tb in ar.TYPES:
            a0, b0 = np.meshgrid(ar.edge_values(ta), ar.edge_values(tb), indexing="ij")
            A = np.concatenate([a0.ravel(), ar.random_values(ta, 64, rng)])
            B = np.concatenate([b0.ravel(), ar.random_values(tb, 64, rng)])
            for op in binary:
                got, e = run(emul, f"{op}(&0 &1)", [[A, B]], [ta, tb])
                if op in ar.INT_ONLY and (ta in ar.FLOATS or tb in ar.FLOATS):
                    assert got is None and "integer or bool operands only" in e, (op, ta, tb, e)
                    continue
                assert e is None, e
                _check(op, got[0], [A, B], [ta, tb])
    for ts in [(ar.U8, ar.I32, ar.I32), (ar.F16, ar.F32, ar.F16), (ar.I64, ar.U8, ar.F64), (ar.BOOL, ar.U16, ar.I8), (ar.U64, ar.I8, ar.U8)]:
        xs = [ar.random_values(t, 200, rng) for t in ts]
        got, e = run(emul, "clamp(&0 &1 &2)", [xs], list(ts))
        _check("clamp", got[0], xs, list(ts))


def test_cast_matrix_and_constants(emul):
    rng = np.random.default_rng(12)
    for tf in ar.TYPES:
        x = np.concatenate([ar.edge_values(tf), ar.random_values(tf, 100, rng)])
        if tf == ar.F32:
            x = np.concatenate([x, np.arange(-300, 300, 0.25, dtype=np.float32)])
        for tt in ar.TYPES:
            (got,), e = run(emul, f"cast_{ar.NAMES[tt]}(&0)", [[x]], [tf])
            assert ar.same_bits(got, ar.convert_sat(x, tf, tt)), (ar.NAMES[tf], ar.NAMES[tt])
    # constants are ConvertSat'ed into their type; a repeated constant shares its slot
    (got,), e = run(emul, "add(add(&0 $0:uint8) $0:uint8)", [[np.array([1, 2], np.int32)]], [ar.I32], ints=[300])
    assert list(got) == [511, 512] and got.dtype == np.int32
    (got,), e = run(emul, "mul(&0 $0:float16)", [[np.array([1, 3], np.float32)]], [ar.F32], reals=[1e6])
    assert list(got) == [65504.0, 196512.0]


def test_broadcasting_scalars_and_errors(emul):
    rng = np.random.default_rng(13)
    img = [rng.integers(0, 256, s, dtype=np.uint8) for s in [(4, 5, 3), (1, 7, 3), (2, 2, 3)]]
    mean = np.array([1.5, 2.5, 3.5], np.float32)
    col = [rng.standard_normal((s[0], 1, 1)).astype(np.float32) for s in [(4,), (1,), (2,)]]
    got, e = run(emul, "fdiv(sub(&0 &1) &2)", [[i, mean, c] for i, c in zip(img, col)], [ar.U8, ar.F32, ar.F32])
    assert e is None, e
    for g, i, c in zip(got, img, col):
        assert ar.same_bits(g, ar.evaluate("fdiv", [ar.evaluate("sub", [i, mean], [ar.U8, ar.F32]), c], [ar.F32, ar.F32]))
    # per-sample scalars (read on the host) beside a tensor, and a 0-d tensor operand
    got, e = run(emul, "mul(&0 &1)", [[np.arange(6, dtype=np.int16).reshape(2, 3), np.array(k - 1, np.int8)] for k in range(3)],
                 [ar.I16, ar.I8], scalar=[0, 1])
    assert [g.tolist() for g in got] == [[[0, -1, -2], [-3, -4, -5]], [[0, 0, 0], [0, 0, 0]], [[0, 1, 2], [3, 4, 5]]]
    # shapes that do not broadcast: the sample and both shapes are named
    _, e = run(emul, "add(&0 &1)", [[np.zeros((4, 3)), np.zeros((4, 3))], [np.zeros((5, 3)), np.zeros((2, 3))]], [ar.F32, ar.F32])
    assert "sample 1" in e and "(5, 3)" in e and "(2, 3)" in e, e


def test_shapes_broadcasts_empty_samples_and_boundaries(emul):
    """arith_ref.shape_cases through the planner and the kernel bodies: ranks 0-6, lower-rank operands, two-way broadcasts, size-1
    output axes, every subset of broadcast axes at rank 4, 16 operands filling the whole stride table, operand shapes that change
    from sample to sample, per-sample scalars, empty and 0-d samples, and volumes around the 4-element threads and 8192-element work
    items for every output element size, both value files, the FLOAT fast path and the generic one."""
    for name, tree, types, scalar, samples in ar.shape_cases(np.random.default_rng(15)):
        outs, e = run(emul, ar.tree_desc(tree), samples, types, scalar=scalar)
        assert e is None, (name, e)
        for i, s in enumerate(samples):
            want_shape = np.broadcast_shapes(*[x.shape for k, x in enumerate(s) if not (scalar and scalar[k])])
            assert outs[i].shape == want_shape, (name, i, outs[i].shape, want_shape)
            ar.tree_check(tree, outs[i], s, types, ULP_HOST)


def test_unaligned_operands_and_outputs(emul):
    """Operands and outputs that break the vector alignment of their element size (the element-by-element branch), next to aligned
    ones, for every element size; the broadcast operand stays aligned."""
    rng = np.random.default_rng(16)
    for name, tree, types, scalar, samples in ar.shape_cases(rng):
        if not name.startswith("volumes"):
            continue
        out_size = np.dtype(ar.NP[ar.tree_type(tree, types)]).itemsize
        for in_step, out_step in ((1, 0), (0, 1), (1, 2), (3, 3)):
            moved = [[_at(x, in_step * x.itemsize) if k < 2 else x for k, x in enumerate(s)] for s in samples]
            outs, e = run(emul, ar.tree_desc(tree), moved, types, scalar=scalar, out_offset=out_step * out_size)
            assert e is None, (name, e)
            for i, s in enumerate(samples):
                ar.tree_check(tree, outs[i], s, types, ULP_HOST)


@pytest.mark.parametrize("desc,msg", [
    ("add(&0)", "expected '&'"), ("add(&0 &1 &0)", "takes 2 operand"), ("foo(&0)", "unknown operator"), ("&5", "does not exist"),
("add(&0 $3:int32)", "integer constant $3 does not exist"), ("add(&0 $0:int33)", "unknown constant type"),
    ("add(&0 &1) x", "unexpected text"), ("bitand(&0 &1)", "integer or bool operands only"), ("div(&1 &0)", "integer or bool operands only"),
    ("cast_float128(&0)", "unknown type"), ("add(" * 70 + "&0" + " &0)" * 70, "nested more than"),
])
def test_planner_refusals(emul, desc, msg):
    _, e = run(emul, desc, [[np.zeros(3, np.int32), np.zeros(3, np.float32)]], [ar.I32, ar.F32])
    assert e is not None and msg in e, (desc, e)


def test_planner_limits(emul):
    x = np.zeros(2, np.int32)
    def tree(leaves):                                           # distinct subexpressions: the planner cannot share them
        if len(leaves) == 1:
            return leaves[0]
        h = len(leaves) // 2
        return f"add({tree(leaves[:h])} {tree(leaves[h:])})"
    xs16 = [x] * 16
    _, e = run(emul, tree([f"{u}(&{k})" for k in range(8) for u in ("minus", "abs")]), [xs16], [ar.I32] * 16)
    assert e is None, e                                          # 8 loads + 16 + 15 operators
    _, e = run(emul, tree([f"{u}(&{k})" for k in range(16) for u in ("minus", "abs")]), [xs16], [ar.I32] * 16)
    assert "more than 64 instructions" in e, e                   # 16 loads + 32 + 31
    _, e = run(emul, "minus($0:int32)", [[x]], [ar.I32], ints=[1])
    assert "no tensor input" in e, e
    many = "&0"
    for k in range(17):
        many = f"add({many} ${k}:int32)"
    _, e = run(emul, many, [[x]], [ar.I32], ints=list(range(17)))
    assert "more than 16 distinct constants" in e, e
    deep = "&0"
    for k in range(9):                                          # the left operands stay live while the right ones are evaluated
        deep = f"add({('minus', 'abs', 'plus')[k % 3]}(&{k // 3}) {deep})"
    _, e = run(emul, deep, [[x, x, x]], [ar.I32] * 3)
    assert "more than 8 live values" in e, e
    _, e = run(emul, "add(&0 &1)", [[np.zeros((1,) * 7), np.zeros(1)]], [ar.F32, ar.F32])
    assert "at most 6 are supported" in e, e


def test_mutated_descriptions_under_sanitizers(tmp_path):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    exe = str(tmp_path / "arith_fuzz")
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-ffp-contract=off", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                        "-DARITH_EMUL_MAIN", SRC, "-o", exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    seeds = ["fdiv(sub(&0 $0:float32) &1)", "clamp(mul(&0 &2) $1:int32 &3)", "cast_int8(add(&3 $2:uint16))", "pow(&2 minus(&0))",
             "bitxor(div(&0 &2) $0:bool)", "atan2(&1 sqrt(&3))", "min(max(&0 &1) cast_float16(&2))"]
    rng = np.random.default_rng(14)
    alphabet = list("&$:() 0123456789_abcdefghijklmnopqrstuvwxyz") + ["float32", "int8", "add(", "&0", "$1:int64", "))", "(("]
    lines = list(seeds)
    for k in range(1500):
        s = list(seeds[k % len(seeds)])
        for _ in range(int(rng.integers(1, 6))):
            p = int(rng.integers(0, len(s) + 1))
            m = int(rng.integers(0, 3))
            if m == 0 and s:
                del s[min(p, len(s) - 1)]
            elif m == 1:
                s.insert(p, str(rng.choice(alphabet)))
            else:
                s[p:p] = s[: int(rng.integers(0, len(s) + 1))]
        lines.append("".join(s).replace("\n", " "))
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="print_stacktrace=1"))
    assert r.returncode == 0 and r.stdout.startswith("ok "), (r.stdout[-500:], r.stderr[-3000:])
    ok, refused = int(r.stdout.split()[1]), int(r.stdout.split()[3])
    assert ok >= len(seeds) and refused > 500, r.stdout


def test_shared_subexpressions_and_constants_end_to_end(emul):
    """Descriptions as the Python front end writes them, evaluated by the host build: a subexpression used twice is evaluated once
    (y = y * y six times is 7 instructions, not 127), UINT64 constants of 2^63 or more keep their bits, integer constants from floats
    and out-of-range values are ConvertSat'ed, FLOAT64 constants keep double precision."""
    from nvidia.dali import fn, types
    from dali_b200 import arith
    holder = {}

    def body():
        x = fn.external_source(device="gpu")
        u = fn.external_source(device="gpu")
        d = fn.external_source(device="gpu")
        y = x * 1.0009765625
        for _ in range(6):
            y = y * y
        holder["sq"] = arith.describe(y)
        holder["u64"] = arith.describe(u & types.Constant(2 ** 64 - 1, types.UINT64))
        holder["hi"] = arith.describe(u + types.Constant(2 ** 63 + 5, types.UINT64))
        holder["ints"] = arith.describe(((x * 0 + types.Constant(2.5, types.INT32)) + types.Constant(-2.5, types.INT16))
                                        * types.Constant(300, types.UINT8) - types.Constant(-7, types.UINT8))
        holder["f64"] = arith.describe(d * types.Constant(0.1, types.FLOAT64))
        return x
    _define(body)
    x = np.array([0.5, 1.0, -1.25, 3.0], np.float32)
    desc, _, ints, reals = holder["sq"]
    (got,), e = run(emul, desc, [[x]], [ar.F32], ints=ints, reals=reals)
    assert e is None, e
    want = x * np.float32(1.0009765625)
    for _ in range(6):
        want = want * want
    assert ar.same_bits(got, want)
    u = np.array([0, 1, 2 ** 63, 2 ** 64 - 1], np.uint64)
    for key, want in (("u64", u), ("hi", u + np.uint64(2 ** 63 + 5))):
        desc, _, ints, reals = holder[key]
        (got,), e = run(emul, desc, [[u]], [ar.U64], ints=ints, reals=reals)
        assert e is None and got.dtype == np.uint64 and np.array_equal(got, want), (key, e, got)
    desc, _, ints, reals = holder["ints"]
    assert ints == [0, 3, -3, 255], ints                         # 0; 2.5 -> 3, -2.5 -> -3, 300 -> 255, -7 -> 0 (ConvertSat)
    (got,), e = run(emul, desc, [[x]], [ar.F32], ints=ints, reals=reals)
    assert e is None and list(got) == [(3 - 3) * 255 - 0] * 4, (desc, ints, got)
    desc, _, ints, reals = holder["f64"]
    d = np.array([1.0, 3.0, 1e-300], np.float64)
    (got,), e = run(emul, desc, [[d]], [ar.F64], ints=ints, reals=reals)
    assert e is None and ar.same_bits(got, d * 0.1), (reals, got)
    assert ar.same_bits(got[:2], np.array([0.1, 0.30000000000000004]))


def test_cpu_operand_that_cannot_move_is_refused_where_written():
    from nvidia.dali import fn

    def body():
        img = fn.external_source(device="gpu")
        b = fn.external_source(device="cpu")
        fn.brightness_contrast(img, brightness=b)                # b is now consumed on the CPU
        return img * b
    with pytest.raises(TypeError, match="cannot be moved to the GPU"):
        _define(body)
