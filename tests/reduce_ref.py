"""A numpy statement of fn.reductions.* (DESIGN.md section 2): the type rules, the exact results (min / max, integer sums, and
sum / mean / mean_square / rms of 8- and 16-bit integers: an exact 64-bit sum, then one rounding), and for floating-point accumulation
a float64 result with the error bound of the planner's accumulation tree: depth * u * sum|t| for the sum of the terms t, where u is
the unit roundoff of the accumulator (2^-24 for FLOAT, 2^-53 for FLOAT64) and depth the number of additions on the longest path of
the tree (dalib200ReducePlanGetPaths), plus the final division, square root and rounding to the output type.

That bound is loose where the kernel is busiest, so `exact_data` builds inputs on which every partial sum is exact in any order,
and `exact_reference` states the one right result for them, down to the last bit (compared with `same_bytes`)."""
import numpy as np

TYPES = [np.uint8, np.uint16, np.uint32, np.uint64, np.int8, np.int16, np.int32, np.int64, np.float16, np.float32, np.float64]
CODE = {np.dtype(t): k for k, t in enumerate(TYPES)}
MIN, MAX, SUM, MEAN, MEAN_SQUARE, RMS, STD_DEV, VARIANCE = range(8)
NAMES = ["min", "max", "sum", "mean", "mean_square", "rms", "std_dev", "variance"]
F16, F32, F64 = 8, 9, 10


def is_int(code):
    return 0 <= code <= 7


def resolve(op, in_code, dtype=None):
    """(output type code, accumulator: 'int' | 'f32' | 'f64'), or raises ValueError as the operator refuses"""
    if in_code == 11:
        raise ValueError("BOOL")
    narrow = is_int(in_code) and np.dtype(TYPES[in_code]).itemsize <= 2
    if op in (MIN, MAX):
        return in_code, "int" if is_int(in_code) else ("f64" if in_code == F64 else "f32")
    if op == SUM:
        out = dtype if dtype is not None else (3 if in_code <= 3 else 7) if is_int(in_code) else (F64 if in_code == F64 else F32)
        if is_int(out) and not is_int(in_code):
            raise ValueError("integer dtype needs an integer input")
        return out, "int" if is_int(out) or narrow else ("f64" if out == F64 else "f32")
    if op in (MEAN, MEAN_SQUARE, RMS):
        out = dtype if dtype is not None else (F64 if in_code == F64 else F32)
        if out not in (F16, F32, F64):
            raise ValueError("dtype must be a float type")
        return out, "int" if narrow else ("f64" if out == F64 else "f32")
    return F32, "f32"


def _axes(x, axes):
    return tuple(range(x.ndim)) if axes is None else tuple(a % x.ndim for a in axes)


def reference(op, x, axes=None, keep_dims=False, dtype=None, ddof=0, mean=None, depth=0):
    """(want, tol): want in the output type; tol None for exact results, else the float64 bound per element"""
    code = CODE[x.dtype]
    out, acc = resolve(op, code, dtype)
    ot = TYPES[out]
    ax = _axes(x, axes)
    n = int(np.prod([x.shape[a] for a in ax], dtype=np.int64))
    if op in (MIN, MAX):
        f = np.min if op == MIN else np.max
        return f(x, axis=ax, keepdims=keep_dims).astype(ot), None
    if acc == "int":
        wide = x.astype(np.uint64 if code <= 3 else np.int64)
        t = wide * wide if op in (MEAN_SQUARE, RMS) else wide
        s = np.sum(t, axis=ax, keepdims=keep_dims, dtype=t.dtype)
        with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
            if op == SUM:
                return (s.astype(ot) if is_int(out) else s.astype(np.float64).astype(ot)), None
            v = s.astype(np.float64) / np.float64(n)
            if op == RMS:
                v = np.sqrt(v)
            return v.astype(ot), None
    u = 2.0 ** -24 if acc == "f32" else 2.0 ** -53
    at = np.float32 if acc == "f32" else np.float64
    xv = x.astype(at).astype(np.float64)                       # the device converts every element to the accumulator first
    ou = {F16: 2.0 ** -11, F32: 2.0 ** -24, F64: 2.0 ** -53}[out]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if op in (STD_DEV, VARIANCE):
            m = np.asarray(mean, np.float32).astype(np.float64).reshape(np.sum(x, axis=ax, keepdims=True).shape)
            t = (xv - m) ** 2
            extra = 3
            div = max(1, n - ddof)
        else:
            t = xv * xv if op in (MEAN_SQUARE, RMS) else xv
            extra = 1 if op in (MEAN_SQUARE, RMS) else 0
            div = n
        s = np.sum(t, axis=ax, keepdims=keep_dims)
        e = (depth + extra) * u * np.sum(np.abs(t), axis=ax, keepdims=keep_dims)
        if op == SUM:
            return s, e + ou * np.abs(s)
        v = s / np.float64(div)
        ev = e / div + u * np.abs(v)
        if n == 0:
            v = np.full_like(v, np.nan)
        if op in (RMS, STD_DEV):
            return np.sqrt(v), np.sqrt(ev) + (u + ou) * np.sqrt(np.abs(v))
        return v, ev + ou * np.abs(v)


def random_data(shape, dt, rng):
    """random values of type dt: standard_normal * 10 + 3 for floats; integers over the whole range, or within +-2^20 for 32- and
    64-bit ones, whose squares would leave the range of FLOAT"""
    dt = np.dtype(dt)
    if dt.kind == "f":
        return (rng.standard_normal(shape) * 10 + 3).astype(dt)
    info = np.iinfo(dt)
    lo, hi = (max(info.min, -(1 << 20)), 1 << 20) if dt.itemsize >= 4 else (info.min, info.max)
    return rng.integers(lo, hi, shape, dtype=dt, endpoint=True)


# ---- exact-sum inputs: every partial sum exact in any order of addition, so a float result has one right value
EXACT = 1 << 24            # the integers a FLOAT holds exactly


def exact_data(shape, dtype, channel_axis, rng, count=None, terms=("x", "sq", "dev")):
    """(x, centres): x of `shape` and `dtype` whose sums are exact for the term kinds named in `terms` ("x": the values, "sq": their
    squares, "dev": (x - centre)^2) over any reduced set of at most `count` elements (default: all of x).  Values are integers, or
    multiples of 1/4 for float types.  Channel c along `channel_axis` (None: one channel) is centred on its own value, so that mixing
    channels up is wrong by whole steps; `centres` (float32, shape 1 but for the channel axis) is the exact centre of each element,
    the `mean` input that keeps (x - m)^2 exact.  Integers k = x / g and k^2 must stay under 2^24 / count summed, as FLOAT needs."""
    dt = np.dtype(dtype)
    g = 0.25 if dt.kind == "f" else 1.0
    n = max(1, int(np.prod(shape, dtype=np.int64)) if count is None else count)
    assert n <= EXACT, n
    lim = EXACT // n                                    # largest |k| (or k^2) a term may reach
    if dt.kind == "f":
        top = 2048 if dt == np.float16 else EXACT - 1  # integers k whose k / 4 the type holds
        lo = -top
    else:
        info = np.iinfo(dt)
        top, lo = min(int(info.max), EXACT - 1), max(int(info.min), -(EXACT - 1))
    if "sq" in terms:
        amp = int(np.sqrt(lim))
    elif "x" in terms:
        amp = lim
    else:
        amp = top
    hi, lo = min(top, amp), max(lo, -amp)
    C = 1 if channel_axis is None else shape[channel_axis]
    width = (hi - lo + 1) // max(C, 1)                  # the range is cut into C slots of `width` values, one per channel
    assert width >= 1, ("too few exact values for the channels", shape, dtype, count, terms)
    spread = (width - 1) // 2
    if "dev" in terms:
        spread = min(spread, int(np.sqrt(lim)))
    cshape = [1] * len(shape)
    if channel_axis is not None:
        cshape[channel_axis] = C
    ck = (lo + (width - 1) // 2 + width * np.arange(C, dtype=np.int64)).reshape(cshape)
    k = ck + rng.integers(-spread, spread, shape, dtype=np.int64, endpoint=True)
    return (k * g).astype(dt), (ck * g).astype(np.float32)


def _exact_terms(op, x, acc, mean, ax):
    """the terms of the sum as float64 (exact) and the accumulator limit, asserting the exactness condition per reduced set"""
    at = np.float32 if acc == "f32" else np.float64
    xv = x.astype(at)
    assert np.array_equal(xv.astype(np.float64), x.astype(np.float64)), "a value the accumulator does not hold exactly"
    xv = xv.astype(np.float64)
    if op in (STD_DEV, VARIANCE):
        m = np.asarray(mean, np.float32).astype(np.float64).reshape(np.sum(x, axis=ax, keepdims=True).shape)
        t = (xv - m) ** 2
    elif op in (MEAN_SQUARE, RMS):
        t = xv * xv
    else:
        t = xv
    if t.size:
        q = 0
        while q < 60 and not np.array_equal(t * 2.0 ** q, np.floor(t * 2.0 ** q)):
            q += 1
        limit = EXACT if acc == "f32" else 1 << 53
        worst = float(np.max(np.sum(np.abs(t), axis=ax))) * 2.0 ** q
        assert worst <= limit, ("inexact: the terms of a reduced set add up past the accumulator's integers", worst, limit)
        assert np.array_equal(t.astype(at).astype(np.float64), t), "a term the accumulator does not hold exactly"
    return t


def exact_reference(op, x, axes=None, keep_dims=False, dtype=None, ddof=0, mean=None):
    """the result in the output type, exactly: the exact sum of the terms (asserted: every term exact in the accumulator, the terms'
    magnitudes of each reduced set adding up to at most 2^24 steps of their granularity for FLOAT, 2^53 for FLOAT64, at most 2^24
    elements) followed by the one rounding red_final performs -- a FLOAT accumulator divides in float32 and takes float32 square
    roots, an integer or FLOAT64 one divides in float64, and a FLOAT16 output is rounded from that."""
    code = CODE[x.dtype]
    out, acc = resolve(op, code, dtype)
    ot = TYPES[out]
    ax = _axes(x, axes)
    n = int(np.prod([x.shape[a] for a in ax], dtype=np.int64))
    if op in (MIN, MAX) or acc == "int":
        return reference(op, x, axes, keep_dims, dtype, ddof, mean)[0]
    assert n <= EXACT, n
    t = _exact_terms(op, x, acc, mean, ax)
    s = np.sum(t, axis=ax, keepdims=keep_dims)            # exact: every partial sum is
    with np.errstate(invalid="ignore", divide="ignore"):
        if op == SUM:
            return np.asarray(s.astype(np.float32) if acc == "f32" else s).astype(np.float64).astype(ot)
        div = max(1, n - ddof) if op in (STD_DEV, VARIANCE) else n
        if acc == "f32":
            v = np.asarray(s, np.float32) / np.float32(div)
            if op in (RMS, STD_DEV):
                v = np.sqrt(v)
        else:
            v = np.asarray(s, np.float64) / np.float64(div)
            if op == RMS:
                v = np.sqrt(v)
    if n == 0:
        v = np.full_like(v, np.nan)
    return np.asarray(v).astype(np.float64).astype(ot)


def exact_mean(centres, x, axes=None, keep_dims=False):
    """the `mean` input of std_dev / variance for exact_data's x: its centres over the output (channel axis kept, or one channel)"""
    ax = _axes(x, axes)
    m = np.broadcast_to(centres, tuple(1 if a in ax else e for a, e in enumerate(x.shape)))
    return np.ascontiguousarray(m if keep_dims else m.reshape([e for a, e in enumerate(m.shape) if a not in ax]), np.float32)


# each threshold of the planner from both sides, as [R, I] reduced over R (csrc/reduce_plan.h): columns, inner and split
PATH_SHAPES = [(40, 32), (200, 31), (66, 31), (2048, 1), (2047, 1), (256, 1), (256, 40), (257, 40), (32768, 1), (32769, 1),
               (10923, 3), (10922, 3)]
VARIANTS = {SUM: [{}, {"dtype": F64}], MEAN: [{}, {"dtype": F16}, {"dtype": F64}], MEAN_SQUARE: [{}, {"dtype": F64}],
            RMS: [{}, {"dtype": F16}, {"dtype": F64}], STD_DEV: [{"ddof": 0}, {"ddof": 1}], VARIANCE: [{"ddof": 0}, {"ddof": 1}]}


def exact_cases(rng):
    """(what, types, ops, shapes, channel axis, axes, keep_dims) of the exact-sum batches both suites run: per-channel statistics of
    HWC, every path on both sides of its threshold, all axes at once, a three-pass rank-6 reduction, a split first pass of two further
    passes, and a sample whose reduced axes are empty"""
    ints = [np.uint8, np.uint16, np.uint32, np.uint64, np.int8, np.int16, np.int32, np.int64]
    floats = [np.float16, np.float32, np.float64]
    every = list(range(8))
    return [
        ("hwc", ints + floats, every, [(37, 41, 3), (1, 300, 3), (200, 100, 3)], 2, (0, 1), True),
        ("all axes", [np.int8, np.uint32] + floats, every, [(7, 9, 3), (50, 1, 2), (1, 1, 1)], None, None, False),
        ("paths", [np.uint8, np.int16, np.float16, np.float32, np.int64, np.float64], every, PATH_SHAPES, 1, (0,), False),
        ("rank 6", [np.float32, np.int16], every, [(3, 5, 7, 4, 6, 2), (2, 1, 9, 3, 1, 5)], 3, (0, 2, 4), False),
        ("split first of three passes", [np.float32, np.uint8], every, [(3, 2, 5, 4, 600, 2), (2, 3, 2, 1, 3000, 3)], 5, (0, 2, 4), True),
        ("split then reduce", [np.float32], every, [(3, 40000, 2)], 2, (0, 1), False),
        ("empty", [np.float32, np.int32], [SUM, MEAN, MEAN_SQUARE, RMS, STD_DEV, VARIANCE], [(4, 0, 3), (4, 5, 3), (0, 5, 3)], 2, (1,), True),
    ]


def exact_batch(rng, t, shapes, channel_axis, axes):
    """exact_data for each shape of a batch, sized to its reduced count: (xs, centres)"""
    xs, cs = [], []
    for s in shapes:
        ax = tuple(range(len(s))) if axes is None else axes
        x, c = exact_data(s, t, channel_axis, rng, count=int(np.prod([s[a] for a in ax], dtype=np.int64)))
        xs.append(x)
        cs.append(c)
    return xs, cs


def same_bytes(got, want, what=""):
    """got and want of one type and shape, byte for byte; a NaN matches any NaN"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
    g, w = got.copy(), want.copy()
    if g.dtype.kind == "f":
        nan = np.isnan(w)
        assert np.array_equal(np.isnan(g), nan), (what, "NaN at other places", g[np.isnan(g) != nan][:5], w[np.isnan(g) != nan][:5])
        g[nan] = 0
        w[nan] = 0
    bad = g.reshape(-1).view(np.uint8).reshape(g.size, g.itemsize) != w.reshape(-1).view(np.uint8).reshape(w.size, w.itemsize)
    idx = np.flatnonzero(bad.any(axis=1))
    assert idx.size == 0, (what, "differs at", idx[:5], g.reshape(-1)[idx[:5]], w.reshape(-1)[idx[:5]], idx.size)


def check(got, want, tol, what=""):
    got = np.asarray(got)
    if tol is None:
        assert got.dtype == want.dtype and got.shape == want.shape, (what, got.dtype, want.dtype, got.shape, want.shape)
        if got.dtype.kind == "f":
            assert np.array_equal(got, want, equal_nan=True), (what, got, want)
        else:
            assert np.array_equal(got, want), (what, got, want)
        return
    assert got.shape == want.shape, (what, got.shape, want.shape)
    g = got.astype(np.float64)
    nan = np.isnan(want)
    assert np.array_equal(np.isnan(g), nan), (what, g, want)
    with np.errstate(invalid="ignore"):
        bad = ~nan & ~(np.abs(g - want) <= tol)
    assert not bad.any(), (what, g[bad][:5], want[bad][:5], np.asarray(tol)[bad][:5] if np.ndim(tol) else tol)
