"""numpy statement of the arithmetic-expression rules (DESIGN.md section 2, "Arithmetic expressions and fn.cast").  The reference's
source is not available here, so this file IS the statement for type promotion, result types, integer corner cases and ConvertSat;
tests/test_arith_cpu.py pins it against numpy wherever numpy agrees, and the host build of the kernel bodies (tools/emul/arith_emul.cc)
and the GPU (tests/test_gpu_arith.py, tests/test_gpu_arith_shapes.py) are checked against it bit for bit, the transcendentals within
ULP bounds.

Types are DALIDataType ids.  Every node is computed in its own type: integers wrap, a BOOL result is "value != 0", FLOAT16 nodes are
computed in float32 and rounded to binary16 (to nearest even) after every operator."""
import numpy as np

U8, U16, U32, U64, I8, I16, I32, I64, F16, F32, F64, BOOL = range(12)
TYPES = list(range(12))
NP = {U8: np.uint8, U16: np.uint16, U32: np.uint32, U64: np.uint64, I8: np.int8, I16: np.int16, I32: np.int32, I64: np.int64,
      F16: np.float16, F32: np.float32, F64: np.float64, BOOL: np.bool_}
NAMES = {U8: "uint8", U16: "uint16", U32: "uint32", U64: "uint64", I8: "int8", I16: "int16", I32: "int32", I64: "int64",
         F16: "float16", F32: "float32", F64: "float64", BOOL: "bool"}
FLOATS = (F16, F32, F64)
SIGNED = (I8, I16, I32, I64)
BITS = {U8: 8, U16: 16, U32: 32, U64: 64, I8: 8, I16: 16, I32: 32, I64: 64, F16: 16, F32: 32, F64: 64, BOOL: 1}

SAME = ("add", "sub", "mul", "pow", "min", "max", "clamp", "abs", "plus", "minus")
FLOAT_FUNCS = ("fabs", "floor", "ceil", "sqrt", "rsqrt", "cbrt", "exp", "log", "log2", "log10", "sin", "cos", "tan", "asin", "acos",
               "atan", "sinh", "cosh", "tanh", "asinh", "acosh", "atanh", "fdiv", "fpow", "atan2")
INT_ONLY = ("div", "bitand", "bitor", "bitxor")
CMP = ("eq", "neq", "lt", "leq", "gt", "geq")
ARITY = {**{k: 1 for k in ("abs", "plus", "minus") + FLOAT_FUNCS}, **{k: 2 for k in ("add", "sub", "mul", "pow", "min", "max", "fdiv",
         "fpow", "atan2") + INT_ONLY + CMP}, "clamp": 3}
# exact in every type (bit for bit); the others are transcendental: within ULP bounds
EXACT = SAME + INT_ONLY + CMP + ("fabs", "floor", "ceil", "sqrt", "rsqrt", "fdiv")


def promote(a, b):
    """Same type -> it.  A float with a non-float -> the float; two floats -> the wider.  Two signed or two unsigned -> the wider
    (BOOL is the narrowest unsigned type).  Signed intX with unsigned uintY: intX if X > Y, else int(2Y), capped at INT64."""
    if a == b:
        return a
    if a in FLOATS or b in FLOATS:
        if a in FLOATS and b in FLOATS:
            return a if BITS[a] >= BITS[b] else b
        return a if a in FLOATS else b
    if (a in SIGNED) == (b in SIGNED):
        return a if BITS[a] >= BITS[b] else b
    s, u = (a, b) if a in SIGNED else (b, a)
    if BITS[s] > BITS[u]:
        return s
    return {8: I16, 16: I32}.get(BITS[u], I64)


def compute_type(op, types):
    """The type the operands are converted to before the operator."""
    t = types[0]
    for u in types[1:]:
        t = promote(t, u)
    if op in FLOAT_FUNCS and t not in FLOATS:
        t = F32
    return t


def result_type(op, types):
    if op.startswith("cast_"):
        return {v: k for k, v in NAMES.items()}[op[5:]]
    if op in INT_ONLY and any(t in FLOATS for t in types):
        raise TypeError(f"{op}: integer or bool operands only")
    return BOOL if op in CMP else compute_type(op, types)


# ---- conversions
def _wrap_int(x, t):
    """a Python integer reduced to type t (two's complement wrap; BOOL: != 0)"""
    if t == BOOL:
        return x != 0
    mod = 1 << BITS[t]
    x %= mod
    return x - mod if t in SIGNED and x >= mod // 2 else x


def cvt(a, frm, to):
    """The value conversion of a promotion: integer widening / re-interpretation, integer -> float (to nearest), float -> wider float.
    FLOAT16 targets go through float32 (exact below 2^24, and every larger integer overflows binary16 either way)."""
    a = np.asarray(a)
    if to in FLOATS:
        if to == F16:
            return a.astype(np.float32).astype(np.float16)
        return a.astype(NP[to])
    return np.array([_wrap_int(int(v), to) for v in a.astype(object).ravel()], NP[to]).reshape(a.shape)


def _round_half_away(x):
    x = np.asarray(x, np.float64)
    big = np.abs(x) >= 2.0 ** 52
    with np.errstate(invalid="ignore"):
        r = np.copysign(np.floor(np.abs(x) + 0.5), x)
    return np.where(big, x, r)


def half_sat(x):
    """float32 -> binary16 as ConvertSat<float16>: clamped to +-65504, to nearest with ties away from zero (NaN stays NaN)"""
    x = np.asarray(x, np.float32).astype(np.float64)
    c = np.clip(x, -65504.0, 65504.0)
    m, e = np.frexp(np.abs(c))                     # |c| = m 2^e, m in [0.5, 1)
    q = np.ldexp(1.0, np.maximum(e - 11, -24))     # the binary16 quantum at |c|
    r = np.copysign(np.floor(np.abs(c) / q + 0.5) * q, c)
    return np.where(np.isnan(x), np.nan, r).astype(np.float16)


def convert_sat(a, frm, to):
    """ConvertSat<to>(a): floats round half away from zero (NaN -> 0) and saturate; integers saturate; BOOL is != 0; -> FLOAT16 via
    float32 and half_sat; FLOAT64 -> FLOAT to nearest; integers -> floats to nearest."""
    a = np.asarray(a)
    if to == BOOL:
        return a != 0
    if to in FLOATS:
        if to == F16:
            return half_sat(a.astype(np.float32))
        return a.astype(NP[to])
    info = np.iinfo(NP[to])
    if frm in FLOATS:
        r = _round_half_away(a.astype(np.float64))
        out = np.zeros(a.shape, NP[to])
        ok = ~np.isnan(r)
        hi = r >= float(info.max) if BITS[to] < 64 else r >= 2.0 ** (63 if to == I64 else 64)
        lo = r <= float(info.min)
        mid = ok & ~hi & ~lo
        out[ok & hi] = info.max
        out[ok & lo] = info.min
        out[mid] = r[mid].astype(NP[to])
        return out
    v = [int(x) for x in np.asarray(a).astype(object).ravel()]
    return np.array([min(max(x, info.min), info.max) for x in v], NP[to]).reshape(a.shape)


# ---- operators
def _int_op(op, xs, t):
    """integer / bool operator in compute type t (Python integers, wrapped at the end)"""
    shape = np.broadcast(*xs).shape
    vals = [np.broadcast_to(np.asarray(x, object), shape).ravel() for x in xs]
    out = []
    for k in range(int(np.prod(shape)) if shape else 1):
        a = int(vals[0][k])
        b = int(vals[1][k]) if len(vals) > 1 else 0
        c = int(vals[2][k]) if len(vals) > 2 else 0
        if op == "plus": r = a
        elif op == "minus": r = -a
        elif op == "abs": r = abs(a)
        elif op == "add": r = a + b
        elif op == "sub": r = a - b
        elif op == "mul": r = a * b
        elif op == "div":
            r = 0 if b == 0 else (abs(a) // abs(b)) * (1 if (a < 0) == (b < 0) else -1)
        elif op == "pow":
            if b < 0:
                r = 1 if a == 1 else (-1 if b % 2 else 1) if a == -1 else 0
            else:
                r = pow(a, b, 1 << 64)
        elif op == "min": r = b if b < a else a
        elif op == "max": r = b if a < b else a
        elif op == "clamp": r = b if a < b else (c if c < a else a)
        elif op == "bitand": r = a & b
        elif op == "bitor": r = a | b
        elif op == "bitxor": r = a ^ b
        elif op in CMP:
            r = {"eq": a == b, "neq": a != b, "lt": a < b, "leq": a <= b, "gt": a > b, "geq": a >= b}[op]
        else:
            raise ValueError(op)
        out.append(r if op in CMP else _wrap_int(r, t))
    return np.array(out, NP[BOOL] if op in CMP else NP[t]).reshape(shape)


_F = {"fabs": np.abs, "abs": np.abs, "floor": np.floor, "ceil": np.ceil, "sqrt": np.sqrt, "cbrt": np.cbrt, "exp": np.exp, "log": np.log,
      "log2": np.log2, "log10": np.log10, "sin": np.sin, "cos": np.cos, "tan": np.tan, "asin": np.arcsin, "acos": np.arccos,
      "atan": np.arctan, "sinh": np.sinh, "cosh": np.cosh, "tanh": np.tanh, "asinh": np.arcsinh, "acosh": np.arccosh, "atanh": np.arctanh}


def _float_op(op, xs, ft):
    """float operator on arrays of numpy type ft (float32 or float64)"""
    a = xs[0]
    b = xs[1] if len(xs) > 1 else None
    c = xs[2] if len(xs) > 2 else None
    if op == "plus": return a.copy()
    if op == "minus": return -a
    if op == "add": return a + b
    if op == "sub": return a - b
    if op == "mul": return a * b
    if op == "fdiv": return a / b
    if op == "rsqrt": return ft(1) / np.sqrt(a)
    if op in ("pow", "fpow"): return np.power(a, b)
    if op == "atan2": return np.arctan2(a, b)
    if op == "min": return np.where(b < a, b, a)
    if op == "max": return np.where(a < b, b, a)
    if op == "clamp": return np.where(a < b, b, np.where(c < a, c, a))
    if op in CMP:
        return {"eq": a == b, "neq": a != b, "lt": a < b, "leq": a <= b, "gt": a > b, "geq": a >= b}[op]
    return _F[op](a)


def evaluate(op, xs, types):
    """op applied to operand arrays xs of the given types (numpy broadcasting), in the reference's type rules."""
    rt = result_type(op, types)
    if op.startswith("cast_"):
        return convert_sat(xs[0], types[0], rt)
    ct = compute_type(op, types)
    ys = [cvt(np.asarray(x, NP[t]), t, ct) for x, t in zip(xs, types)]
    if ct in FLOATS:
        ft = np.float64 if ct == F64 else np.float32
        with np.errstate(all="ignore"):
            r = _float_op(op, [np.asarray(y).astype(ft) for y in ys], ft)
        if op in CMP:
            return np.asarray(r, np.bool_)
        return np.asarray(r, ft).astype(np.float16) if ct == F16 else np.asarray(r, ft)
    return _int_op(op, ys, ct)


def edge_values(t):
    """0, +-1, min, max and for floats NaN, +-inf, -0.0 and (float16) subnormals"""
    if t == BOOL:
        return np.array([False, True])
    if t in FLOATS:
        fi = np.finfo(NP[t])
        v = [0.0, -0.0, 1.0, -1.0, float(fi.max), -float(fi.max), float(fi.tiny), np.inf, -np.inf, np.nan, 0.5, -2.5, 3.0, 1e-3]
        if t == F16:
            v += [2.0 ** -24, -(2.0 ** -20), 65504.0, 1000.5]
        return np.array(v, NP[t])
    ii = np.iinfo(NP[t])
    v = [0, 1, ii.max, ii.min, 2, 3, ii.max - 1, 7]
    if t in SIGNED:
        v += [-1, -2, ii.min + 1, -7]
    return np.array(v, NP[t])


def random_values(t, n, rng):
    if t == BOOL:
        return rng.integers(0, 2, n).astype(np.bool_)
    if t in FLOATS:
        return (rng.standard_normal(n) * rng.choice([1, 10, 300], n)).astype(NP[t])
    ii = np.iinfo(NP[t])
    return rng.integers(int(ii.min), int(ii.max), n, dtype=np.int64 if t != U64 else np.uint64, endpoint=True).astype(NP[t])


def same_bits(got, want):
    """bit equality, any NaN equal to any NaN"""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype != want.dtype or got.shape != want.shape:
        return False
    if got.dtype.kind == "f":
        both_nan = np.isnan(got) & np.isnan(want)
        return bool(np.all(both_nan | (got.view(np.dtype(f"u{got.itemsize}")) == want.view(np.dtype(f"u{want.itemsize}")))))
    return bool(np.array_equal(got, want))


def _transcendental(op, ct):
    return not op.startswith("cast_") and (op not in EXACT or (op == "pow" and ct in FLOATS))


# CUDA C Programming Guide, "Mathematical Functions" appendix: maximum ULP errors (float / double), without fast math
ULP32 = {"cbrt": 1, "exp": 2, "log": 1, "log2": 1, "log10": 2, "sin": 2, "cos": 2, "tan": 4, "asin": 2, "acos": 2, "atan": 2,
         "sinh": 3, "cosh": 2, "tanh": 2, "asinh": 3, "acosh": 4, "atanh": 3, "pow": 4, "fpow": 4, "atan2": 3}
ULP64 = {"cbrt": 1, "exp": 1, "log": 1, "log2": 1, "log10": 1, "sin": 2, "cos": 2, "tan": 2, "asin": 2, "acos": 2, "atan": 2,
         "sinh": 2, "cosh": 1, "tanh": 1, "asinh": 2, "acosh": 2, "atanh": 2, "pow": 2, "fpow": 2, "atan2": 2}


def check(op, got, xs, types, ulp=None):
    """got is op applied to xs: bit for bit where the result is exact, else within the ULP bound of a float64 evaluation (ULP32 /
    ULP64 by default, `ulp` when given; FLOAT16 within 1; FLOAT64 one more for the float64 reference's own rounding)."""
    rt = result_type(op, types)
    want = evaluate(op, xs, types)
    assert got.dtype == want.dtype and got.shape == want.shape, (op, types, got.dtype, want.dtype, got.shape, want.shape)
    ct = compute_type(op, types)
    if not _transcendental(op, ct):
        assert same_bits(got, want), (op, [NAMES[t] for t in types], np.argwhere(~((got == want) | (want != want)))[:4])
        return
    ys = [cvt(np.asarray(x, NP[t]), t, ct).astype(np.float64) for x, t in zip(xs, types)]
    with np.errstate(all="ignore"):
        ref = _float_op(op, ys, np.float64)
    if rt == F16:
        bound = 1.0
    elif ulp is not None:
        bound = ulp + (rt == F64)
    else:
        bound = ULP64[op] + 1 if rt == F64 else ULP32[op]
    err = ulp_error(got, ref, rt)
    assert np.all(err <= bound), (op, [NAMES[t] for t in types], float(np.max(err)), bound)


# ---- expression trees: ("add", ("mul", 0, 1), 2) is add(mul(&0 &1) &2); a leaf k is input k
def tree_desc(tree):
    if isinstance(tree, int):
        return f"&{tree}"
    return f"{tree[0]}({' '.join(tree_desc(t) for t in tree[1:])})"


def tree_type(tree, types):
    return types[tree] if isinstance(tree, int) else result_type(tree[0], [tree_type(t, types) for t in tree[1:]])


def tree_eval(tree, xs, types):
    """(value, type) of the tree over the operand arrays xs, every node evaluated by evaluate() (numpy broadcasting)."""
    if isinstance(tree, int):
        return np.asarray(xs[tree], NP[types[tree]]), types[tree]
    kids = [tree_eval(t, xs, types) for t in tree[1:]]
    op = tree[0]
    tt = [t for _, t in kids]
    return evaluate(op, [v for v, _ in kids], tt), result_type(op, tt)


def tree_check(tree, got, xs, types, ulp=None):
    """got is the tree over xs: its operands evaluated exactly, the root held to check() (so a transcendental root is bounded)."""
    if isinstance(tree, int):
        assert same_bits(got, np.asarray(xs[tree], NP[types[tree]]))
        return
    kids = [tree_eval(t, xs, types) for t in tree[1:]]
    check(tree[0], got, [v for v, _ in kids], [t for _, t in kids], ulp)


def _rand(t, shape, rng):
    return random_values(t, int(np.prod(shape, dtype=np.int64)), rng).reshape(shape)


def _ones_at(shape, mask):
    """shape with the axes in bit mask `mask` (bit a: axis a) set to 1"""
    return tuple(1 if (mask >> a) & 1 else e for a, e in enumerate(shape))


# sample volumes around the kernel's 4-element threads and 8192-element work items
VOLUMES = (1, 3, 4, 5, 8191, 8192, 8193, 3 * 8192 + 5)


def shape_cases(rng, big=False):
    """[(name, tree, types, scalar flags, samples)]: expressions whose result depends on the operands' shapes rather than their types.
    samples[i][k] is operand k of sample i (a 0-d array for a per-sample scalar).  Every operator is exact except the root of the
    atan2 case.  big: the float cases also get a 1080p x 3 sample (the integer reference loops in Python)."""
    cases = []
    # ranks 0-6: a full operand, one with random unit axes, one of lower rank (the trailing half of the axes)
    for r in range(7):
        samples = []
        for _ in range(3):
            s = tuple(int(v) for v in rng.integers(1, 5 if r < 5 else 4, r))
            samples.append([_rand(I16, s, rng), _rand(F32, _ones_at(s, int(rng.integers(0, 1 << r))), rng),
                            _rand(U8, s[r - r // 2:], rng)])
        cases.append((f"rank {r}", ("mul", ("add", 0, 1), 2), [I16, F32, U8], None, samples))
    # operands of lower rank than the output, each broadcast along the leading axes
    cases.append(("lower ranks", ("add", ("add", ("mul", 0, 1), 2), 3), [U16, I32, U8, I8], None,
                  [[_rand(U16, (2, 3, 4, 5), rng), _rand(I32, (5,), rng), _rand(U8, (4, 1), rng), _rand(I8, (3, 1, 1), rng)],
                   [_rand(U16, (1, 2, 7, 3), rng), _rand(I32, (1,), rng), _rand(U8, (7, 3), rng), _rand(I8, (2, 1, 3), rng)]]))
    # two-way broadcasts: neither operand has the output's shape
    hw = [(5, 7), (1, 9), (6, 1), (1, 1), (33, 130)]
    cases.append(("(H, 1) + (1, W)", ("add", 0, 1), [F32, F32], None, [[_rand(F32, (h, 1), rng), _rand(F32, (1, w), rng)] for h, w in hw]))
    cases.append(("(H, 1) - (1, W) u8", ("sub", 0, 1), [U8, U8], None, [[_rand(U8, (h, 1), rng), _rand(U8, (1, w), rng)] for h, w in hw]))
    fhwc = [(3, 4, 5, 3), (1, 9, 2, 1), (2, 1, 1, 4), (4, 6, 7, 2)]
    cases.append(("(F, 1, W, 1) * (1, H, 1, C)", ("mul", 0, 1), [F16, F16], None,
                  [[_rand(F16, (f, 1, w, 1), rng), _rand(F16, (1, h, 1, c), rng)] for f, h, w, c in fhwc]))
    # size-1 output axes
    cases.append(("size-1 output axes", ("sub", 0, 1), [I32, I32], None,
                  [[_rand(I32, (4, 1, 5), rng), _rand(I32, (4, 1, 1), rng)], [_rand(I32, (1, 1, 1), rng), _rand(I32, (1, 1, 1), rng)],
                   [_rand(I32, (1, 1, 9), rng), _rand(I32, (1, 1, 9), rng)], [_rand(I32, (3, 1, 1), rng), _rand(I32, (1, 1, 1), rng)]]))
    # every subset of broadcast axes at rank 4, one subset per sample: x broadcasts the subset, y its complement, z is full
    full = (3, 2, 5, 4)
    cases.append(("rank-4 broadcast subsets", ("sub", ("mul", 0, 1), 2), [F32, F32, F32], None,
                  [[_rand(F32, _ones_at(full, m), rng), _rand(F32, _ones_at(full, 15 & ~m), rng), _rand(F32, full, rng)]
                   for m in range(16)]))
    # 16 tensor operands over 6 axes, each broadcasting a different subset: the whole stride table
    masks = [0, 1, 2, 4, 8, 16, 32, 63, 5, 10, 20, 40, 21, 42, 7, 56]
    ops = ("add", "mul", "bitxor", "sub")
    tree = 0
    for k in range(1, 16):
        tree = (ops[k % 4], tree, k)
    samples = []
    for j, shape in enumerate([(3, 2, 4, 3, 2, 5), (2, 3, 2, 5, 3, 2)]):
        samples.append([_rand(I32, _ones_at(shape, masks[(k + j) % 16]), rng) for k in range(16)])
    cases.append(("16 operands, 6 axes", tree, [I32] * 16, None, samples))
    # the same input broadcasts in some samples and not in others
    cases.append(("per-sample operand shapes", ("add", ("mul", 0, 1), 2), [U8, U8, I16], None,
                  [[_rand(U8, (4, 3), rng), _rand(U8, s1, rng), _rand(I16, s2, rng)]
                   for s1, s2 in (((4, 3), (3,)), ((1, 3), (1,)), ((4, 1), (3,)), ((1, 1), (1,)))]))
    # per-sample scalars (read on the host) between broadcast tensors, narrow and wide
    cases.append(("scalars and broadcasts", ("min", ("mul", ("sub", 0, 2), 1), 3), [F32, I32, F32, F32], [0, 1, 0, 1],
                  [[_rand(F32, (h, 4), rng), _rand(I32, (), rng), _rand(F32, (1, 4), rng), _rand(F32, (), rng)] for h in (5, 1, 3)]))
    cases.append(("scalars and broadcasts, 64-bit", ("add", ("mul", 0, 1), 2), [U16, I64, U8], [0, 1, 0],
                  [[_rand(U16, (h, 5), rng), _rand(I64, (), rng), _rand(U8, (5,), rng)] for h in (4, 1, 2)]))
    # empty samples (an extent of 0 broadcast against 1) between non-empty ones
    pairs = [((3, 4), (1, 4)), ((0, 4), (1, 4)), ((5, 1), (1, 0)), ((2, 3), (2, 1)), ((0, 1), (1, 0)), ((1, 1), (1, 1)), ((0, 0), (0, 1)),
             ((7, 9), (7, 9))]
    cases.append(("empty samples", ("add", 0, 1), [U8, F32], None, [[_rand(U8, a, rng), _rand(F32, b, rng)] for a, b in pairs]))
    cases.append(("all 0-d", ("fdiv", ("add", 0, 1), 1), [F64, F64], None, [[_rand(F64, (), rng), _rand(F64, (), rng)] for _ in range(5)]))
    cases.append(("every sample empty", ("add", 0, 1), [I16, I16], None,
                  [[_rand(I16, a, rng), _rand(I16, b, rng)] for a, b in (((0, 3), (1, 3)), ((4, 0), (4, 1)), ((0, 0), (1, 1)))]))
    # sample volumes around the 4-element threads and the work items, every element size, both value files, the FLOAT fast path
    # and the generic path; a linear pair beside a broadcast third operand
    for name, tree, types in (("u8", ("sub", ("add", 0, 1), 2), [U8] * 3), ("i16", ("sub", ("add", 0, 1), 2), [I16] * 3),
                              ("f16", ("sub", ("add", 0, 1), 2), [F16] * 3), ("f32", ("sub", ("mul", 0, 1), 2), [F32] * 3),
                              ("i32", ("sub", ("mul", 0, 1), 2), [I32] * 3), ("f64", ("sub", ("add", 0, 1), 2), [F64] * 3),
                              ("i64", ("sub", ("mul", 0, 1), 2), [I64] * 3), ("bool", ("lt", ("add", 0, 2), 1), [U8] * 3),
                              ("narrow", ("cast_int32", ("add", 0, ("mul", 1, 2))), [I32] * 3),
                              ("wide", ("cast_int32", ("add", 0, ("mul", 1, 2))), [I32, I64, I32]),
                              ("atan2", ("atan2", ("add", 0, 2), 1), [F32] * 3)):
        vs = VOLUMES + ((1080 * 1920 * 3,) if big and types[0] in FLOATS else ())
        cases.append((f"volumes {name}", tree, types, None,
                      [[_rand(types[0], (v,), rng), _rand(types[1], (v,), rng), _rand(types[2], (1,), rng)] for v in vs]))
    return cases


def ulp_error(got, ref64, t):
    """|got - ref64| in units of the last place of type t at ref64.  Where ref64 rounds to an infinity or is NaN in t, got must be
    that value (error 0, else inf)."""
    got = np.asarray(got).astype(np.float64)
    ref64 = np.asarray(ref64, np.float64)
    fi = np.finfo(NP[t])
    with np.errstate(all="ignore"):
        r = ref64.astype(NP[t]).astype(np.float64)     # the reference in t (overflow to infinity as t has it)
        e = np.floor(np.log2(np.maximum(np.abs(ref64), float(fi.tiny))))
        ulp = np.ldexp(1.0, (np.minimum(e, fi.maxexp - 1) - fi.nmant).astype(int))
        err = np.abs(got - ref64) / ulp
    special = np.isnan(r) | np.isinf(r)
    agree = (np.isnan(got) & np.isnan(r)) | (got == r)
    err = np.where(special, np.where(agree, 0.0, np.inf), np.where(np.isfinite(got), err, np.inf))
    return err
