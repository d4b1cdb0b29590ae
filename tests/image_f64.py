"""float64 statements of the image operators on the benchmark's path (resize in any number of spatial axes, warp_affine, crop_mirror_normalize,
the colour twist behind hsv / color_twist / brightness_contrast, the BT.601 YCbCr conversions) and of the mel filter bank's weights, each
written from the operation's definition, with an error bound per output element that says what a single-precision evaluation can be off by.

The bit-exact GPU tests compare the kernels with oracle/imgproc_oracle.c, a second float32 restatement of the same reading of the reference.
A mistake shared by both (a pixel centre, an antialias radius, a flipped region of interest, a hue sign, a YIQ constant) passes them.  These
statements share neither the restatement's code nor its operation order; tests/test_image_f64_cpu.py shows that the restatement meets every
bound with 4x margin and that plausible mistakes are rejected, and tests/test_gpu_image_f64.py holds the kernels to the same bounds.

U = 2^-24 is the unit round-off of float32.  Functions return (value, bound) in float64, or the set of acceptable answers where an output is
an index choice (nearest neighbour).  None of them calls oracle/ or the library."""
import itertools
import math

import numpy as np

U = 2.0 ** -24

F_NN, F_LINEAR, F_TRIANGULAR, F_GAUSSIAN, F_CUBIC, F_LANCZOS3 = range(6)


# ------------------------------------------------------------------------------------------------------------------------ checks
def _pick(got, ref, bound):
    """ref (and bound) may be lists of acceptable float64 answers with their bounds: per element, the answer got is relatively closest to."""
    got = np.asarray(got, np.float64)
    refs = ref if isinstance(ref, list) else [ref]
    bounds = bound if isinstance(bound, list) else [bound] * len(refs)
    refs = [np.broadcast_to(np.asarray(r, np.float64), got.shape) for r in refs]
    bounds = [np.broadcast_to(np.asarray(b, np.float64), got.shape) for b in bounds]
    score = lambda r, b: np.where(np.abs(got - r) <= b, np.abs(got - r) / np.where(b > 0, b, 1.0), np.inf)
    best, bb = refs[0], bounds[0]
    for r, b in zip(refs[1:], bounds[1:]):
        better = score(r, b) < score(best, bb)
        best, bb = np.where(better, r, best), np.where(better, b, bb)
    return got, best, bb


def check(got, ref, bound, what=""):
    """|got - ref| <= bound everywhere (ref: one answer or a list of acceptable ones); returns the largest |got - ref| / bound (0.0
    where every bound is 0)."""
    got, ref, bound = _pick(got, ref, bound)
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound, first at {i}: got {got[i]!r}, "
                             f"float64 {ref[i]!r}, |diff| {err[i]:.3e} > bound {bound[i]:.3e}")
    nz = bound > 0
    return float((err[nz] / bound[nz]).max()) if nz.any() else 0.0


def check_u8(got, ref, bound, what=""):
    """A u8 store of a float within `bound` of ref: got is a rounding (half-even or half-away, both are used) of some value in
    [ref - bound, ref + bound], saturated to [0, 255].  So |got - clamp(ref)| <= 1/2 + bound, and got equals the rounded value wherever
    ref is farther than the bound from a half-integer.  ref / bound may be lists of acceptable answers.  Returns the largest
    (|got - clamp(ref)| - 1/2) / bound (0.0 when none exceeds 1/2)."""
    got = np.asarray(got, np.float64)
    refs = ref if isinstance(ref, list) else [ref]
    bounds = bound if isinstance(bound, list) else [bound] * len(refs)
    ok = np.zeros(got.shape, bool)
    excess = np.full(got.shape, np.inf)
    for r, b in zip(refs, bounds):
        r, b = np.broadcast_to(np.asarray(r, np.float64), got.shape), np.broadcast_to(np.asarray(b, np.float64), got.shape)
        inside = (got >= np.clip(np.ceil(r - b - 0.5), 0, 255)) & (got <= np.clip(np.floor(r + b + 0.5), 0, 255))
        ex = np.maximum(np.abs(got - np.clip(r, 0, 255)) - 0.5, 0.0) / np.where(b > 0, b, np.inf)
        excess = np.where(inside, np.minimum(excess, ex), excess)
        ok |= inside
    if not ok.all():
        i = tuple(int(v) for v in np.argwhere(~ok)[0])
        r0, b0 = np.broadcast_to(np.asarray(refs[0], np.float64), got.shape), np.broadcast_to(np.asarray(bounds[0], np.float64), got.shape)
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.size} u8 outputs outside the band, first at {i}: got {got[i]!r}, "
                             f"float64 {r0[i]!r}, bound {b0[i]:.3e}")
    return float(np.nan_to_num(excess, posinf=0.0).max()) if excess.size else 0.0


def check_f16(got, ref, bound, what=""):
    """An fp16 store (saturated to +-65504) of a float within `bound` of ref: within 1/2 ulp_fp16 + bound of the clamped value, and equal to
    its fp16 rounding wherever it is farther than the bound from a tie.  Returns the largest (|got - clamp(ref)| - ulp / 2) / bound."""
    got = np.asarray(got, np.float64)
    ref, bound = np.broadcast_arrays(np.asarray(ref, np.float64), np.asarray(bound, np.float64))
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    rc = np.clip(ref, -65504.0, 65504.0)
    h = rc.astype(np.float16)
    hf = h.astype(np.float64)
    with np.errstate(over="ignore"):
        up = np.nextafter(h, np.float16(np.inf)).astype(np.float64)
        dn = np.nextafter(h, np.float16(-np.inf)).astype(np.float64)
    up = np.where(np.isfinite(up), up, hf + 32)                      # beyond +-65504 the next fp16 would be 65536: ulp 32
    dn = np.where(np.isfinite(dn), dn, hf - 32)
    ulp = np.maximum(up - hf, hf - dn)
    tie_dist = np.minimum(np.abs(rc - (hf + up) / 2), np.abs(rc - (hf + dn) / 2))
    err = np.abs(got - rc)
    bad = err > ulp / 2 + bound
    bad |= (tie_dist > bound) & (got != hf)
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} fp16 outputs wrong, first at {i}: got {got[i]!r}, float64 {ref[i]!r}, "
                             f"rounded {hf[i]!r}, bound {bound[i]:.3e}")
    excess = err - ulp / 2
    nz = (bound > 0) & (excess > 0)
    return float((excess[nz] / bound[nz]).max()) if nz.any() else 0.0


def check_choice(got, candidates, what=""):
    """got[i] equals candidates[k][i] for some k (nearest-neighbour index choices)."""
    got = np.asarray(got)
    ok = np.zeros(got.shape, bool)
    for c in candidates:
        ok |= got == np.asarray(c)
    if not ok.all():
        i = tuple(int(v) for v in np.argwhere(~ok)[0])
        raise AssertionError(f"{what}: {int((~ok).sum())} of {ok.size} outputs are none of the accepted pixels, first at {i}: got {got[i]!r}, "
                             f"accepted {[np.asarray(c)[i] for c in candidates]}")


# ------------------------------------------------------------------------------------------------------------------------ resize
# The filters as the reference tabulates them: (knots, half-extent A of the closed form's argument).  Knot i of n sits at
# a_i = (2 i / (n - 1) - 1) A and holds the closed form there; the interpolant is piecewise linear and falls to zero one knot beyond each
# end (dali/kernels/imgproc/resample/resampling_filters.cu:66-118, resampling_filters.cuh:48-67).
_TABLE = {F_LINEAR: (3, 1.0), F_TRIANGULAR: (3, 1.0), F_GAUSSIAN: (65, 2.0), F_CUBIC: (129, 2.0), F_LANCZOS3: (193, 3.0)}


def keys_cubic(a, alpha=-0.5):
    a = np.abs(np.asarray(a, np.float64))
    near = (alpha + 2) * a ** 3 - (alpha + 3) * a ** 2 + 1
    far = alpha * a ** 3 - 5 * alpha * a ** 2 + 8 * alpha * a - 4 * alpha
    return np.where(a <= 1, near, np.where(a < 2, far, 0.0))


def lanczos(a, lobes=3):
    a = np.asarray(a, np.float64)
    return np.where(np.abs(a) < lobes, np.sinc(a) * np.sinc(a / lobes), 0.0)


def closed_form(ftype, a):
    """The continuous filter in its own argument: triangle, exp(-a^2), Keys cubic (a = -1/2), Lanczos-3."""
    a = np.asarray(a, np.float64)
    if ftype in (F_LINEAR, F_TRIANGULAR):
        return np.maximum(0.0, 1 - np.abs(a))
    if ftype == F_GAUSSIAN:
        return np.exp(-a * a)
    if ftype == F_CUBIC:
        return keys_cubic(a)
    assert ftype == F_LANCZOS3, ftype
    return lanczos(a)


def knots(ftype, form=closed_form):
    n, A = _TABLE[ftype]
    k = form(ftype, (2 * np.arange(n) / (n - 1) - 1) * A)
    return np.concatenate(([0.0], k, [0.0]))                              # the zero knots at -1 and n


def _second_derivative_max(ftype, form=closed_form):
    """max |d^2 F / dt^2| in knot units (knot spacing 1), from a fine grid of the closed form."""
    n, A = _TABLE[ftype]
    g = np.linspace(-A, A, 200001)
    h = g[1] - g[0]
    d2 = np.abs(np.diff(form(ftype, g), 2)) / h ** 2
    return float(d2.max()) * (2 * A / (n - 1)) ** 2


def default_radius(ftype, antialias, in_size, out_size):
    """params.h:40-56: with antialias and a shrinking axis the radius scales with in / out."""
    aa = antialias and in_size > out_size
    r = in_size / out_size if out_size else 1.0
    if ftype in (F_TRIANGULAR, F_GAUSSIAN):
        return r if aa else 1.0
    if ftype == F_CUBIC:
        return 2 * r if aa else 2.0
    if ftype == F_LANCZOS3:
        return 3 * r if aa else 3.0
    return 1.0


def select_filter(n, m, roi, min_filter, mag_filter):
    """(type, width in source pixels) of one axis: minification when m < |r1 - r0|; linear with antialias becomes triangular, triangular
    without antialias becomes linear; a zero radius takes the default; the width is the span of the table in source pixels."""
    r0, r1 = (0.0, float(n)) if roi is None else roi
    span = abs(float(np.float32(r1) - np.float32(r0))) if roi is not None else float(n)
    ftype, aa, radius = min_filter if m < span else mag_filter
    if aa and ftype == F_LINEAR:
        ftype = F_TRIANGULAR
    elif not aa and ftype == F_TRIANGULAR:
        ftype = F_LINEAR
    if ftype == F_NN:
        return F_NN, 0.0
    if radius == 0:
        radius = default_radius(ftype, aa, span, m)
    if ftype == F_LINEAR:
        width = 2.0
    elif ftype in (F_TRIANGULAR, F_GAUSSIAN):
        width = max(1.0, 2 * radius)                                     # Gaussian: 4 sqrt(2) sigma, sigma = radius / (2 sqrt(2))
    elif ftype == F_CUBIC:
        width = 2 * max(2.0, radius)
    else:
        width = 2 * max(3.0, radius)
    return ftype, width


def _support(ftype, width):
    """Taps per output: ceil of the width as the reference's float arithmetic gives it ((n - 1) / ((n - 1) / width)); a filter whose
    support exceeds 8192 is rescaled to a width of 8192 (resampling_setup.cc)."""
    n = _TABLE[ftype][0]
    f32 = np.float32
    s = int(math.ceil(f32(n - 1) / f32(f32(n - 1) / f32(width))))
    if s > 8192:
        width = 8192.0
        s = int(math.ceil(f32(n - 1) / f32(f32(n - 1) / f32(width))))
    return s, width


class Axis:
    """One axis of a resize as sparse taps: idx [m, T] (source rows, clamped), w [m, T] (the float64 weights), dw [m, T] (per-tap bound on
    |w_float - w|, position and table errors included), support S (the float32 accumulation term counts S + 2 roundings)."""

    def __init__(self, idx, w, dw, support, ftype, width, alts):
        self.idx, self.w, self.dw, self.support, self.ftype, self.width, self.alts = idx, w, dw, support, ftype, width, alts


def axis_taps(n, m, roi=None, min_filter=(F_LINEAR, 1, 0.0), mag_filter=(F_LINEAR, 1, 0.0), exact=False, accumulated=False, form=None):
    """The taps of one axis of extent n resized to m over roi = (r0, r1) (None: the whole axis; r1 < r0 flips it).

    s = (r1 - r0) / m, the centre of output x is c = r0 + (x + 1/2) s, source sample j sits at j + 1/2.  A filter of width W (source
    pixels) gives sample j the weight F((j + 1/2 - c) / (W / 2)) normalised to sum 1 over the window of `support` taps starting at
    ceil(c - 1/2 - W / 2); the source index is clamped to [0, n - 1].  F is the table's piecewise-linear interpolant (exact=False) or the
    continuous filter (exact=True, the bound gains the interpolation error h^2 / 8 max|F''| per tap).  NN takes floor(c) (clamped).

    Bound per tap: the float32 position sx0f = x s + (r0 + s / 2 - 1/2 - W / 2) is off by delta <= 8u (max(|r0|, |r1|, n) + W + 1) (the scale,
    the product and four additions); the table coordinate (j - sx0f) (n_k - 1) / W gains u (k + 1) from f0 + k and 6u of its own size from the
    float scale, width and product, and 3u (n_k - 1) / 2 from the float anchor.  That times the local knot slope, plus 4u of the local knot
    size for the knots themselves and the interpolation, is the raw coefficient error e_k; normalising by the float sum adds (S + 2) u w_k,
    and (e_k + w_k sum e) / sum c.  Where c - 1/2 - W / 2 is within delta of an integer the float window may start one tap later or earlier:
    Axis.alts holds the weights of that other window (NN: the neighbouring pixel) for those outputs.  `accumulated`: the reference accumulates an NN coordinate (sy += scale), so its
    delta grows by u max|c| per output."""
    r0, r1 = (0.0, float(n)) if roi is None else (float(np.float32(roi[0])), float(np.float32(roi[1])))
    ftype, width = select_filter(n, m, roi, min_filter, mag_filter)
    s = (r1 - r0) / m
    x = np.arange(m, dtype=np.float64)
    c = r0 + (x + 0.5) * s
    mag = max(abs(r0), abs(r1), float(n))
    if ftype == F_NN:
        delta = 8 * U * (mag + 1) + (x * U * (mag + abs(s)) if accumulated else 0.0)
        i = np.floor(c)
        idx = np.clip((i[:, None] + np.arange(-1, 2)).astype(np.int64), 0, n - 1)
        w = np.zeros((m, 3)); w[:, 1] = 1
        alts = []
        for side, amb in ((0, np.floor(c - delta) != i), (2, np.floor(c + delta) != i)):
            if amb.any():
                wa = w.copy()
                wa[amb] = 0
                wa[amb, side] = 1
                alts.append((wa, np.zeros((m, 3))))
        return Axis(idx, w, np.zeros((m, 3)), 1, ftype, 0.0, alts)
    S, width = _support(ftype, width)
    nk = _TABLE[ftype][0]
    K = knots(ftype, form or closed_form)
    fscale = (nk - 1) / width
    delta = 8 * U * (mag + width + 1)
    v = c - 0.5 - width / 2
    start = np.ceil(v)
    lo_start = np.ceil(v - delta)
    hi_start = np.ceil(v + delta)
    base = lo_start
    T = S + int((hi_start - lo_start).max()) if m else S
    j = base[:, None] + np.arange(T)[None, :]
    t = (j + 0.5 - c[:, None] + width / 2) * fscale                        # table coordinate, knot i at t = i
    D = np.abs(np.diff(K))
    Dloc = np.maximum(np.maximum(np.concatenate(([0.0], D[:-1])), D), np.concatenate((D[1:], [0.0])))
    Kabs = np.maximum(np.abs(K[:-1]), np.abs(K[1:]))

    def F(tt):
        if exact:
            n_, A = _TABLE[ftype]
            a = (2 * tt / (n_ - 1) - 1) * A
            inside = (tt >= 0) & (tt <= n_ - 1)
            ramp = np.interp(tt, np.arange(-1, n_ + 1), K)                   # the table's ramp to zero beyond the end knots
            return np.where(inside, (form or closed_form)(ftype, a), ramp)
        return np.interp(tt, np.arange(-1, nk + 1), K)

    def window(st):
        inwin = (j >= st[:, None]) & (j < st[:, None] + S)
        raw = np.where(inwin, F(t), 0.0)
        ssum = raw.sum(axis=1, keepdims=True)
        return inwin, raw, ssum, np.where(ssum != 0, raw / np.where(ssum != 0, ssum, 1.0), 0.0)

    seg = np.clip(np.floor(t).astype(np.int64) + 1, 0, D.size - 1)          # segment index in the zero-extended knot list
    d2 = _second_derivative_max(ftype, form or closed_form) / 8 + 4 * U if exact else 0.0

    def weights(st):
        """(w, dw) of the window that starts at st."""
        inwin, raw, ssum, w = window(st)
        k = j - st[:, None]
        dt = fscale * (delta + U * (np.abs(k) + 1)) + 6 * U * np.abs(t) + 3 * U * (nk - 1) / 2
        e = np.where(inwin, Dloc[seg] * dt + 4 * U * Kabs[seg] + d2, 0.0)
        safe = np.where(ssum != 0, np.abs(ssum), np.inf)
        return w, (e + np.abs(w) * e.sum(axis=1, keepdims=True)) / safe + (S + 2) * U * np.abs(w)

    w, dw = weights(start)
    alts = []
    for st in (lo_start, hi_start):
        amb = st != start
        if amb.any():
            wa, dwa = weights(st)
            alts.append((np.where(amb[:, None], wa, w), np.where(amb[:, None], dwa, dw)))
    idx = np.clip(j.astype(np.int64), 0, n - 1)
    return Axis(idx, w, dw, S, ftype, width, alts)


def _apply(x, axes, weights):
    """sum over the taps of every axis of weights[a] x[idx], axes in any order (float64: the order does not matter at this precision)."""
    y = np.asarray(x, np.float64)
    order = sorted(range(len(axes)), key=lambda a: axes[a].idx.shape[0] / max(1, y.shape[a]))
    for a in order:
        ax, wt = axes[a], weights[a]
        m, T = ax.idx.shape
        g = np.take(y, ax.idx.reshape(-1), axis=a)
        g = g.reshape(y.shape[:a] + (m, T) + y.shape[a + 1:])
        shape = [1] * g.ndim
        shape[a], shape[a + 1] = m, T
        y = (g * wt.reshape(shape)).sum(axis=a + 1)
    return y


def resize(x, out_shape, rois=None, min_filter=(F_LINEAR, 1, 0.0), mag_filter=(F_LINEAR, 1, 0.0), exact=False, form=None,
           full_shape=None, origin=None):
    """Resize of x [spatial..., C] to out_shape (spatial) as the tensor product of the per-axis weights of axis_taps(); rois: per axis
    None or (r0, r1); filters: one (type, antialias, radius) for every axis or a list per axis.  Every axis but the last (x) is treated as
    an accumulated nearest-neighbour coordinate.  The value does not depend on which axis a kernel processes first.

    Returns ([value, alternatives...], [bound, ...]): the alternatives are the values with another tap window (or NN pixel) on some axis,
    for the outputs where the float position may pick it; every other output equals the value there.  Bound of each: (sum over axes of
    (S_a + 2)) u sum |w| |x| for the float32 accumulation of the passes (each pass sums S products; its input carries the error of the
    pass before, weighted by this pass's |w|), plus sum over axes a of (dw_a x |w_other|) |x| for the weights.

    full_shape / origin: x is the block at `origin` of a larger image of spatial shape `full_shape` (positions, clamping and the bound's
    position error are those of the whole image); every tap the outputs read must lie inside the block."""
    x = np.asarray(x)
    nd = len(out_shape)
    full_shape = full_shape or x.shape[:nd]
    origin = origin or [0] * nd
    rois = rois or [None] * nd
    per = lambda f: f if isinstance(f, list) else [f] * nd
    mins, mags = per(min_filter), per(mag_filter)
    axes = [axis_taps(int(full_shape[a]), int(out_shape[a]), rois[a], mins[a], mags[a], exact, accumulated=(a < nd - 1), form=form)
            for a in range(nd)]
    for a in range(nd):
        if origin[a]:
            axes[a].idx = axes[a].idx - int(origin[a])
            used = (np.abs(axes[a].w) + sum(np.abs(w) for w, _ in axes[a].alts)) > 0
            assert axes[a].idx[used].min() >= 0 and axes[a].idx[used].max() < x.shape[a], "a tap lies outside the block"
            axes[a].idx = np.clip(axes[a].idx, 0, x.shape[a] - 1)
    xa = np.abs(x.astype(np.float64))
    acc = sum(a.support + 2 for a in axes) * U
    values, bounds = [], []
    for combo in itertools.product(*[[(a.w, a.dw)] + a.alts for a in axes]):
        ws = [c[0] for c in combo]
        values.append(_apply(x, axes, ws))
        bound = acc * _apply(xa, axes, [np.abs(w) for w in ws])
        for k in range(nd):
            bound = bound + _apply(xa, axes, [combo[a][1] if a == k else np.abs(ws[a]) for a in range(nd)])
        bounds.append(bound)
    return values, bounds


# ------------------------------------------------------------------------------------------------------------------------ warp
def warp_affine(img, M, out_hw=None, interp=1, fill=None):
    """Affine warp with the dst->src 2x3 matrix M: output (x, y) samples the source at p = M (x + 1/2, y + 1/2) in float64.  NN takes the
    pixel at floor(p); bilinear interpolates the corners at floor(p - 1/2) and floor(p - 1/2) + 1.  Taps outside the source take the
    nearest edge pixel (fill None) or ConvertSat<u8>(fill) (the fill rounded half away from zero and saturated).

    Bound: the reference walks float32 coordinates per row, re-anchored every 256 outputs (anchor + 256 dsx per block, then + dsx per pixel);
    its error is at most u (4 |p|_0 + (x // 256 + x % 256 + 2) R) per axis, |p|_0 the magnitude of the anchor's terms and R the largest
    |coordinate| along the row.  Twice that (the coordinate) times the largest difference between the samples around the taps (a 4 x 4 block
    holds every cell the coordinate can move into), plus 8u of the largest sample for the lerps, bounds a bilinear output.
    NN: returns the candidate pixels instead (interp=0): floor(p +- delta) on each axis."""
    img = np.asarray(img)
    H, W, C = img.shape
    oh, ow = out_hw or (H, W)
    M = np.asarray(M, np.float64).reshape(2, 3)                          # a float32 matrix converts exactly
    ys, xs = np.meshgrid(np.arange(oh, dtype=np.float64), np.arange(ow, dtype=np.float64), indexing="ij")
    px = M[0, 0] * (xs + 0.5) + M[0, 1] * (ys + 0.5) + M[0, 2]
    py = M[1, 0] * (xs + 0.5) + M[1, 1] * (ys + 0.5) + M[1, 2]
    steps = xs // 256 + xs % 256 + 2
    fillv = None if fill is None else float(min(255.0, max(0.0, math.floor(abs(float(np.float32(fill))) + 0.5) * math.copysign(1, fill))))
    src = img.astype(np.float64)

    def fetch(ix, iy):
        inside = (ix >= 0) & (ix < W) & (iy >= 0) & (iy < H)
        v = src[np.clip(iy, 0, H - 1), np.clip(ix, 0, W - 1)]
        if fillv is not None:
            v = np.where(inside[..., None], v, fillv)
        return v

    deltas = []
    for r in range(2):
        p0 = np.abs(M[r, 2]) + np.abs(M[r, 0]) * 0.5 + np.abs(M[r, 1]) * (ys + 0.5)
        R = np.abs(M[r, 2]) + np.abs(M[r, 0]) * ow + np.abs(M[r, 1]) * (ys + 1)
        deltas.append(2 * U * (4 * p0 + steps * R))
    dx, dy = deltas
    if interp == 0:
        cands = []
        for ox in (-1, 0, 1):
            for oy in (-1, 0, 1):
                ix = np.floor(px + ox * dx).astype(np.int64)
                iy = np.floor(py + oy * dy).astype(np.int64)
                cands.append(fetch(ix, iy))
        return cands
    fx, fy = px - 0.5, py - 0.5
    x0, y0 = np.floor(fx).astype(np.int64), np.floor(fy).astype(np.int64)
    qx, qy = (fx - x0)[..., None], (fy - y0)[..., None]
    s00, s01, s10, s11 = fetch(x0, y0), fetch(x0 + 1, y0), fetch(x0, y0 + 1), fetch(x0 + 1, y0 + 1)
    value = (s00 * (1 - qx) + s01 * qx) * (1 - qy) + (s10 * (1 - qx) + s11 * qx) * qy
    hi = np.full(value.shape, -np.inf)
    lo = np.full(value.shape, np.inf)
    for ox in range(-1, 3):
        for oy in range(-1, 3):
            s = fetch(x0 + ox, y0 + oy)
            hi, lo = np.maximum(hi, s), np.minimum(lo, s)
    bound = (dx + dy)[..., None] * (hi - lo) + 8 * U * np.maximum(np.abs(hi), np.abs(lo))
    return value, bound


def rotation_matrix(angle_deg, in_hw, out_hw):
    """dst->src matrix of fn.rotate by angle_deg about the centres of the two canvases: src = c_in + R(angle) (dst - c_out), with
    R(t) = [[cos t, -sin t], [sin t, cos t]] applied to (x, y), y pointing down (dali/operators/image/remap/rotate_params.h)."""
    a = math.radians(float(angle_deg))
    c, s = math.cos(a), math.sin(a)
    cx_i, cy_i = in_hw[1] / 2, in_hw[0] / 2
    cx_o, cy_o = out_hw[1] / 2, out_hw[0] / 2
    return np.array([[c, -s, cx_i - c * cx_o + s * cy_o], [s, c, cy_i - s * cx_o - c * cy_o]])


# ------------------------------------------------------------------------------------------------------------------------ CMN
def crop_mirror_normalize(img, anchor=(0, 0), crop=None, mirror=False, mean=0.0, std=1.0, scale=1.0, shift=0.0, layout="CHW",
                          pad_channels=None, fill=0.0):
    """(x - mean) * scale / std + shift per channel in float64 from the user's arguments; the crop window (which may stick out of the
    image), the horizontal mirror of the cropped window, the padded channels and the layout are plain indexing; out-of-image pixels and
    padded channels hold the fill value exactly.

    Bound: the kernel receives mean' = mean - shift std / scale and inv = scale / std in float32, computed from the float32 user arguments:
    mean' is off by u (|mean| + 3 |shift std / scale| + |mean'|), inv by 3u relative; the output fl(fl(x - mean') inv) adds u |x - mean'|
    inv and u |v|.  In all u ((|mean| + 3 |shift std / scale| + |mean'|) inv + 5 |x - mean'| inv + |v|) to first order, doubled (as
    tests/audio_tail_f64.py does): when the shift dominates, every rounding acts on the same magnitude.  Filled elements have bound 0."""
    img = np.asarray(img)
    H, W, C = img.shape
    ch, cw = crop or (H, W)
    ay, ax = anchor
    oc = pad_channels or C
    mean = np.broadcast_to(np.asarray(mean, np.float64), (C,))
    std = np.broadcast_to(np.asarray(std, np.float64), (C,))
    inv = scale / std
    meanp = mean - shift * std / scale
    ys = ay + np.arange(ch)
    xs = ax + (np.arange(cw)[::-1] if mirror else np.arange(cw))
    inside = ((ys >= 0) & (ys < H))[:, None] & ((xs >= 0) & (xs < W))[None, :]
    px = img[np.clip(ys, 0, H - 1)][:, np.clip(xs, 0, W - 1)].astype(np.float64)
    fillv = np.broadcast_to(np.asarray(fill, np.float64), (oc,)) if np.ndim(fill) else np.full(oc, float(fill))
    val = np.empty((ch, cw, oc))
    bnd = np.zeros((ch, cw, oc))
    for c in range(oc):
        if c < C:
            v = (px[..., c] - meanp[c]) * inv[c]
            b = 2 * U * ((abs(mean[c]) + 3 * abs(shift * std[c] / scale) + abs(meanp[c])) * abs(inv[c]) + 6 * np.abs(v))   # |x - mean'| inv = |v|
            val[..., c] = np.where(inside, v, fillv[c])
            bnd[..., c] = np.where(inside, b, 0.0)
        else:
            val[..., c] = fillv[c]
    if layout == "CHW":
        val, bnd = val.transpose(2, 0, 1), bnd.transpose(2, 0, 1)
    return val, bnd


# ------------------------------------------------------------------------------------------------------------------------ colour
RGB2YIQ = np.array([[0.299, 0.587, 0.114], [0.596, -0.274, -0.321], [0.211, -0.523, 0.311]])


def twist_matrix(hue=0.0, saturation=1.0, value=1.0, brightness=1.0, contrast=1.0, half_range=128.0, yiq=RGB2YIQ, inverse=np.linalg.inv):
    """M = B C YIQ^-1 H(hue) S V YIQ, T = (half_range - half_range contrast) brightness, in float64 from the nine YIQ constants; H rotates
    the (I, Q) plane: [[1, 0, 0], [0, cos h, sin h], [0, -sin h, cos h]] (dali/operators/image/color/color_twist.h)."""
    h = math.radians(float(np.float32(hue)))
    Hm = np.array([[1, 0, 0], [0, math.cos(h), math.sin(h)], [0, -math.sin(h), math.cos(h)]])
    f = lambda v: float(np.float32(v))
    Mx = f(brightness) * f(contrast) * inverse(yiq) @ Hm @ np.diag([1, f(saturation), f(saturation)]) * f(value) @ yiq
    T = (f(half_range) - f(half_range) * f(contrast)) * f(brightness)
    return Mx, np.full(3, T)


def twist(img, hue=0.0, saturation=1.0, value=1.0, brightness=1.0, contrast=1.0, half_range=128.0, **kw):
    """linear_transform() of twist_matrix(); the offset's bound counts its largest term, half_range * max(1, |contrast|) |brightness|."""
    M, T = twist_matrix(hue, saturation, value, brightness, contrast, half_range, **kw)
    f = lambda v: abs(float(np.float32(v)))
    return linear_transform(img, M, T, f(half_range) * max(1.0, f(contrast)) * f(brightness))


def linear_transform(img, M, T, t_mag=None):
    """out = M x + T per pixel; M and T are the float64 statement (twist_matrix).

    Bound: the float32 host construction of M (five 3 x 3 products, a float inverse, float YIQ constants, cosf / sinf) is off by at most
    40u max|M_ij| per entry, times sum |x_j|; the pixel's three products and three additions are 3u sum |M_ij x_j| + u |out|; the float
    offset (half_range - half_range contrast) brightness is three roundings, at most 3u t_mag (t_mag: the magnitude of its largest term,
    given by the caller, |T| by default).  Doubled, as a first-order bound: a pixel of zeros leaves only the offset's three roundings,
    which a float32 evaluation comes within 0.4 of."""
    x = np.asarray(img, np.float64)
    M = np.asarray(M, np.float64)
    T = np.asarray(T, np.float64)
    t_mag = np.abs(T) if t_mag is None else t_mag
    v = x @ M.T + T
    bound = 2 * (40 * U * np.abs(M).max() * np.abs(x).sum(axis=-1, keepdims=True) + 3 * U * (np.abs(x) @ np.abs(M).T) + 3 * U * t_mag
                 + U * np.abs(v))
    return v, bound


KR, KB = 0.299, 0.114
KG = 1 - KR - KB


def rgb_to_ycbcr(rgb):
    """BT.601 studio range: Y = 16 + 219/255 (Kr R + Kg G + Kb B), Cb = 128 + 224/255 (B - Y') / (2 (1 - Kb)), Cr likewise with R, Kr;
    bound 6u of the sum of the magnitudes of the terms."""
    x = np.asarray(rgb, np.float64)
    R, G, B = x[..., 0], x[..., 1], x[..., 2]
    yp = KR * R + KG * G + KB * B
    Y = 16 + 219 / 255 * yp
    Cb = 128 + 224 / 255 * (B - yp) / (2 * (1 - KB))
    Cr = 128 + 224 / 255 * (R - yp) / (2 * (1 - KR))
    mag = (np.abs(R) + np.abs(G) + np.abs(B)) + 128
    return np.stack([Y, Cb, Cr], -1), np.stack([6 * U * mag] * 3, -1)


def ycbcr_to_rgb(ycc):
    """The inverse of rgb_to_ycbcr, in float64."""
    x = np.asarray(ycc, np.float64)
    yp = (x[..., 0] - 16) * 255 / 219
    tb, tr = (x[..., 1] - 128) * 255 / 224, (x[..., 2] - 128) * 255 / 224
    R = yp + 2 * (1 - KR) * tr
    B = yp + 2 * (1 - KB) * tb
    G = yp - 2 * KB * (1 - KB) / KG * tb - 2 * KR * (1 - KR) / KG * tr
    mag = np.abs(yp) + 3 * (np.abs(tb) + np.abs(tr))
    return np.stack([R, G, B], -1), np.stack([8 * U * mag] * 3, -1)


def ycbcr_to_gray(ycc):
    x = np.asarray(ycc, np.float64)
    v = (x[..., :1] - 16) * 255 / 219
    return v, 6 * U * (np.abs(x[..., :1]) + 16) * 255 / 219


def gray_to_ycbcr(g):
    x = np.asarray(g, np.float64)[..., :1]
    Y = 16 + 219 / 255 * x
    return np.concatenate([Y, np.full_like(Y, 128.0), np.full_like(Y, 128.0)], -1), np.concatenate([4 * U * (Y + 16), 0 * Y, 0 * Y], -1)


# ------------------------------------------------------------------------------------------------------------------------ mel
def hz_to_mel(f, htk):
    f = np.asarray(f, np.float64)
    if htk:
        return 1127.0 * np.log1p(f / 700.0)
    return np.where(f >= 1000, 15.0 + np.log(np.maximum(f, 1e-300) / 1000) * 27 / math.log(6.4), f * 3 / 200)


def mel_to_hz(m, htk):
    m = np.asarray(m, np.float64)
    if htk:
        return 700.0 * np.expm1(m / 1127.0)
    return np.where(m >= 15, 1000 * np.exp((m - 15) * math.log(6.4) / 27), m * 200 / 3)


def _dfdm(f, htk):
    f = np.asarray(f, np.float64)
    if htk:
        return (f + 700) / 1127
    return np.where(f >= 1000, f * math.log(6.4) / 27, 200 / 3)


def mel_weights(nbin, nfilter, sample_rate, freq_low=0.0, freq_high=0.0, htk=False, normalize=True):
    """[nfilter, nbin] weights: nfilter + 2 edges equally spaced on the mel scale (HTK: 1127 ln(1 + f / 700); Slaney: linear below 1 kHz at
    200/3 Hz per mel, logarithmic above with 27 mels per factor 6.4), triangle i rising from edge i to i + 1 and falling to i + 2,
    sampled at the bin frequencies k sr / nfft (nfft = 2 (nbin - 1)) from ceil(freq_low / step) up to the bin of freq_high; Slaney
    normalisation multiplies triangle i by 2 / (f_{i+2} - f_i).  freq_high <= 0 means sr / 2.

    Bound per weight: the float32 edges are off by df_i <= (6u |mel_high| + u |m_i|) df/dmel + 6u (f_i + 700) (h2m / m2h in float); a
    triangle side of width f_{i+1} - f_i then moves by 2 (df_i + df_{i+1}) / width, plus 4u for the weight's own roundings; normalisation
    adds (df_i + df_{i+2}) / (f_{i+2} - f_i) + 2u relative.  Doubled, as a first-order bound."""
    if freq_high <= 0:
        freq_high = sample_rate / 2
    f32 = lambda v: float(np.float32(v))
    sr, fl, fh = f32(sample_rate), f32(freq_low), f32(freq_high)
    nfft = 2 * (nbin - 1)
    mlo, mhi = float(hz_to_mel(fl, htk)), float(hz_to_mel(fh, htk))
    mel = mlo + (mhi - mlo) * np.arange(nfilter + 2) / (nfilter + 1)
    f = mel_to_hz(mel, htk)
    df = (6 * U * max(abs(mhi), abs(mlo)) + U * np.abs(mel)) * _dfdm(f, htk) + 6 * U * (f + 700)
    step = sr / nfft
    k = np.arange(nbin)
    fk = k * step
    kb0 = math.ceil(fl / step)
    kb1 = min(math.ceil(fh / step), nbin)
    live = (k >= kb0) & (k < kb1)
    W = np.zeros((nfilter, nbin))
    B = np.zeros((nfilter, nbin))
    for i in range(nfilter):
        a, b, c = f[i], f[i + 1], f[i + 2]
        up = (fk - a) / (b - a)
        dn = (c - fk) / (c - b)
        w = np.clip(np.minimum(up, dn), 0, None)
        near = (fk > a - df[i]) & (fk < c + df[i + 2])
        e = np.where(fk <= b, 2 * (df[i] + df[i + 1]) / (b - a), 2 * (df[i + 1] + df[i + 2]) / (c - b)) + 4 * U
        nf = 2 / (c - a) if normalize else 1.0
        enf = ((df[i] + df[i + 2]) / (c - a) + 2 * U) if normalize else 0.0
        W[i] = np.where(live, w * nf, 0.0)
        B[i] = np.where(live & near, 2 * nf * (e + w * enf), 0.0)
    return W, B
