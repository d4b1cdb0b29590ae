"""float64 statements of the audio-tail operators (to_decibels, MFCC, normalize, nonsilent_region, audio_resample), each written from
the operation's definition, with an error bound per output element that says what a single-precision evaluation can be off by.

The bit-exact GPU tests compare the kernels with oracle/audio_oracle.c, a second float32 restatement of the same reading of the
reference.  A mistake shared by both (a tap range, a window centre, a DCT convention, a lifter index, the window adjustment of the
non-silent region) passes them.  These statements do not share the restatement's code or its operation order, so they catch such a
mistake; tests/test_audio_tail_f64_cpu.py shows that a plain float32 evaluation meets every bound with 4x margin and that plausible
arithmetic mistakes are rejected, and tests/test_gpu_audio_tail_f64.py holds the kernels to the same bounds.

U = 2^-24 is the unit round-off of float32.  Each function returns (value, bound); value is float64, bound is >= 0 elementwise."""
import math

import numpy as np

U = 2.0 ** -24
LN10 = math.log(10.0)


def check(got, ref, bound, what=""):
    """|got - ref| <= bound everywhere (bound 0 means exact equality).  Returns the largest |got - ref| / bound over elements with a
    non-zero bound (0.0 when there is none), so that callers can report how close to the bound a kernel comes."""
    got = np.asarray(got, np.float64)
    ref, bound = np.broadcast_arrays(np.asarray(ref, np.float64), np.asarray(bound, np.float64))
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = np.abs(got - ref)
    bad = ~(err <= bound)
    if bad.any():
        i = tuple(int(v) for v in np.argwhere(bad)[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} elements outside the bound, first at {i}: got {got[i]!r}, "
                             f"float64 {ref[i]!r}, |diff| {err[i]:.3e} > bound {bound[i]:.3e}")
    nz = bound > 0
    return float((err[nz] / bound[nz]).max()) if nz.any() else 0.0


# ------------------------------------------------------------------------------------------------------------------ ToDecibels
def to_decibels(x, multiplier=10.0, reference=None, cutoff_db=-200.0):
    """m * log10(max(x / s_ref, 10^(cutoff / m))) (dali/kernels/signal/decibel/decibel_calculator.h:25-56, to_decibels_op.h:41-50).
    s_ref = `reference`, or the sample maximum when it is None -- 1 when that maximum is <= 0 (no positive value to refer to).
    The cut-off ratio is the float32 value the operator uses, so that clamped elements compare at the float cut-off.

    Bound: twice the first-order worst case of a float32 evaluation.  The ratio x * (1 / s_ref) is two float roundings
    (|m| * 2u / ln 10 after the logarithm), the cut-off ratio one more (|m| * u / ln 10, plus u * |cutoff| for the rounded exponent
    cutoff / m); log2f (1 ulp), log10(2) in float, m * log10(2) and the final product are relative roundings of the result (5u * |out|).
    A float32 evaluation comes within 0.4 of that worst case, so the factor 2 leaves the 4x margin the CPU test asserts."""
    m = float(np.float32(multiplier))
    a = np.asarray(x, np.float64)
    if reference is None:
        s = float(a.max()) if a.size else 0.0
        s = s if s > 0 else 1.0
    else:
        s = float(np.float32(reference))
    min_ratio = float(np.float32(10.0 ** (float(np.float32(cutoff_db)) / m)))
    if min_ratio == 0.0:
        min_ratio = float(np.nextafter(np.float32(0), np.float32(1)))
    out = m * np.log10(np.maximum(a / s, min_ratio))
    bound = 2 * (5 * U * np.abs(out) + abs(m) * 3 * U / LN10 + U * abs(float(cutoff_db)))
    return out, bound


# ------------------------------------------------------------------------------------------------------------------------ MFCC
def dct_matrix(nfeat, ndct, dct_type, normalize=False):
    """c(k, n), float64, k < ndct, n < nfeat (dali/kernels/signal/dct/table.h:27-112 states the same four definitions):
      I    X_k = x_0 / 2 + (-1)^k x_{N-1} / 2 + sum_{n=1}^{N-2} x_n cos(pi k n / (N - 1))
      II   X_k = sum_n x_n cos(pi (n + 1/2) k / N)                  ortho: * 1 / sqrt(N) for k = 0, sqrt(2 / N) otherwise
      III  X_k = x_0 / 2 + sum_{n>=1} x_n cos(pi n (k + 1/2) / N)    ortho: x_0 / sqrt(N) + sqrt(2 / N) * sum_{n>=1}
      IV   X_k = sum_n x_n cos(pi (n + 1/2) (k + 1/2) / N)           ortho: * sqrt(2 / N)
    i.e. half of scipy.fft.dct(type=t) unnormalised, and scipy's norm="ortho" otherwise."""
    N = int(nfeat)
    k = np.arange(ndct, dtype=np.float64)[:, None]
    n = np.arange(N, dtype=np.float64)[None, :]
    if dct_type == 1:
        assert not normalize and N > 1
        c = np.cos(np.pi * k * n / (N - 1))
        c[:, 0] *= 0.5
        c[:, N - 1] *= 0.5
    elif dct_type == 2:
        c = np.cos(np.pi * (n + 0.5) * k / N)
        if normalize:
            c *= math.sqrt(2.0 / N)
            c[0] = 1.0 / math.sqrt(N)
    elif dct_type == 3:
        c = np.cos(np.pi * n * (k + 0.5) / N)
        if normalize:
            c *= math.sqrt(2.0 / N)
            c[:, 0] = 1.0 / math.sqrt(N)
        else:
            c[:, 0] = 0.5
    else:
        assert dct_type == 4, dct_type
        c = np.cos(np.pi * (n + 0.5) * (k + 0.5) / N)
        if normalize:
            c *= math.sqrt(2.0 / N)
    return c


def lifter_coeffs(ndct, lifter):
    """1 + L/2 * sin(pi (k + 1) / L) for k < ndct (dali/operators/audio/mfcc/mfcc.h:36-41); all ones for L = 0."""
    L = float(np.float32(lifter))
    if L == 0:
        return np.ones(ndct)
    return 1.0 + L / 2 * np.sin(np.pi * (np.arange(ndct) + 1.0) / L)


def mfcc(x, n_mfcc=20, dct_type=2, normalize=False, lifter=0.0):
    """lift[k] * sum_n c(k, n) x[n, t] along axis 0 of x[nfeat, frames]; n_mfcc above nfeat is clipped to nfeat.

    Bound: twice the first-order worst case of a float32 evaluation in any summation order.  The table entries are float roundings of
    c(k, n) (u / 2 each), each product and each of the nfeat - 1 additions one rounding, the lifter product one more:
    |lift_k| (nfeat + 3) u sum_n |c(k, n) x[n, t]|.  The float lifter itself is off by |L / 2| (2.5u * pi (k + 1) / |L| + 2u) + u |lift_k|
    (argument, sinf, product and sum roundings), times |sum_n c x|.  Sums of a few terms come within 0.4 of the worst case, so the
    factor 2 leaves the 4x margin the CPU test asserts.  A column of zeros gives exactly 0."""
    a = np.asarray(x, np.float64)
    nfeat = a.shape[0]
    ndct = min(int(n_mfcc), nfeat)
    c = dct_matrix(nfeat, ndct, dct_type, normalize)
    lift = lifter_coeffs(ndct, lifter)[:, None]
    y = c @ a
    mag = np.abs(c) @ np.abs(a)
    L = float(np.float32(lifter))
    dlift = 0.0 if L == 0 else abs(L / 2) * (2.5 * U * np.pi * (np.arange(ndct)[:, None] + 1) / abs(L) + 2 * U) + U * np.abs(lift)
    return lift * y, 2 * (np.abs(lift) * (nfeat + 3) * U * mag + dlift * np.abs(y))


# ------------------------------------------------------------------------------------------------------------------- Normalize
def _groups(a, axes):
    """[groups, count] view of a 1-D or 2-D sample for the reduced axes (None: all), and the function that puts it back."""
    if a.ndim == 1 or axes is None or sorted(axes) == [0, 1]:
        return a.reshape(1, -1), lambda g: g.reshape(a.shape)
    if list(axes) == [1]:
        return a, lambda g: g
    assert list(axes) == [0], axes
    return a.T, lambda g: g.T


def normalize(x, axes=None, ddof=0, epsilon=0.0, scale=1.0, shift=0.0):
    """(x - mean) * scale / sqrt(var + eps) + shift over the reduced axes, var = sum (x - mean)^2 / max(1, count - ddof); a group whose
    divisor sqrt(var + eps) is 0 gives `shift` (dali/operators/math/normalize: the multiplier is 0 then).

    Bound, for a float32 evaluation that sums the deviations from the group's first element x0 in 256 interleaved sequential partial
    sums joined by a tree (the order of audio_tail.cu's normalize_kernel; a pairwise or a shorter sequential sum does better):
      mean    d_mu <= (n / 256 + 16) u A,  A = mean |x - x0|
      each deviation  e_i <= u |x_i - x0| + d_mu + u |x_i - mean|
      variance  d_var <= ((n / 256 + 16) u var' + 2 mean(|x - mean| e) + mean(e^2)) * n / (n - ddof),  var' = the sum of squares / n
      multiplier  rel <= d_var / (2 (var + eps)) + 3u
      output  |mul| e_i + |x_i - mean| |mul| rel + u |(x_i - mean) mul| + u |out_i|.
    A group whose values are all equal has var = 0: with eps = 0 it must give `shift` exactly."""
    a = np.asarray(x, np.float64)
    g, back = _groups(a, axes)
    n = g.shape[1]
    f32 = np.float32
    scale, shift, eps = float(f32(scale)), float(f32(shift)), float(f32(epsilon))
    mean = g.mean(axis=1, keepdims=True)
    dev = g - mean
    const = (g.max(axis=1, keepdims=True) == g.min(axis=1, keepdims=True)) if n else np.ones((g.shape[0], 1), bool)
    dev = np.where(const, 0.0, dev)
    div = max(1, n - ddof)
    var = np.where(const, 0.0, (dev ** 2).sum(axis=1, keepdims=True) / div)
    sd = np.sqrt(var + eps)
    mul = np.where(sd != 0, scale / np.where(sd != 0, sd, 1.0), 0.0)
    out = dev * mul + shift
    # bound
    k = n / 256 + 16
    x0 = g[:, :1]
    A = np.abs(g - x0).mean(axis=1, keepdims=True) if n else np.zeros_like(x0)
    d_mu = k * U * A
    e = U * np.abs(g - x0) + d_mu + U * np.abs(dev)
    var_sum = (dev ** 2).mean(axis=1, keepdims=True) if n else np.zeros_like(x0)
    d_var = (k * U * var_sum + 2 * (np.abs(dev) * e).mean(axis=1, keepdims=True) + (e ** 2).mean(axis=1, keepdims=True)) * n / div \
        if n else np.zeros_like(x0)
    with np.errstate(divide="ignore", invalid="ignore"):
        rel = np.where(var + eps > 0, d_var / (2 * (var + eps)), 0.0) + 3 * U
    bound = np.abs(mul) * e + np.abs(dev * mul) * (rel + U) + U * np.abs(out)
    bound = np.where(mul == 0, 0.0, bound)          # divisor 0: the multiplier is 0 and the output is `shift`, exactly
    return back(out), back(bound)


# ------------------------------------------------------------------------------------------------------------- NonsilentRegion
def nonsilent_band(x, cutoff_db=-60.0, window_length=2048, reference_power=None, reset_interval=8192):
    """The non-silent region of a clip, as the interval of answers a float32 running-sum evaluation may give.

    Definition (dali/operators/audio/nonsilence_op.h:60-130, dali/kernels/signal/moving_mean_square.cc:55-77): W = min(window_length,
    n); mms[t] = sum_{j = max(0, t - W + 1)}^{t} x_j^2 / W (always divided by W, also for the partial windows at the start);
    threshold = ref * 10^(cutoff_db / 10), ref = max(mms) or `reference_power`; lo / hi = first / last t with mms[t] >= threshold;
    begin = max(lo - (W - 1), 0) (the non-silent sample sits somewhere inside the window that reported it), length = hi - begin + 1;
    (0, 0) when no t qualifies.

    The reference keeps the window sum as a running float sum (add the new square, subtract the oldest), restarted every
    `reset_interval` samples from the W - 1 squares before the restart.  Its error at t grows by at most
    u (2 S_t + x_t^2 + x_{t-W+1}^2) per step (the two sums, the two squares) and is amplified by (1 + 2u) per step; the restart sum
    of W - 1 squares is off by at most 2 (W - 1) u S.  With E_t the resulting bound on |mms_f32[t] - mms[t]| and E_thr the one on
    the float threshold, t is certainly above if mms[t] - E_t >= thr + E_thr and certainly below if mms[t] + E_t < thr - E_thr.

    Returns dict(begin=(lo, hi), end=(lo, hi), empty_possible, nonempty_possible): the float32 answer (begin, begin + length - 1) has
    begin and end in these closed ranges; outside the band the answer is exact."""
    from scipy.signal import lfilter
    a = np.asarray(x, np.float32).astype(np.float64)
    n = a.size
    assert n > 0
    W = min(int(window_length), n)
    interval = n if reset_interval == -1 else int(reset_interval)
    sq = a * a
    cs = np.concatenate(([0.0], np.cumsum(sq)))
    t = np.arange(n)
    S = cs[t + 1] - cs[np.maximum(0, t - W + 1)]
    S = np.maximum(S, 0.0)
    mms = S / W
    old = np.where(t - W + 1 >= 0, sq[np.maximum(t - W + 1, 0)], 0.0)
    b = U * (2 * S + sq + old)
    e = np.empty(n)
    amp = 1 + 2 * U
    for r in range(0, n, interval):
        r1 = min(n, r + interval)
        e0 = 2 * (W - 1) * U * (S[r - 1] if r > 0 else 0.0)
        e[r:r1] = lfilter([1.0], [1.0, -amp], b[r:r1], zi=[amp * e0])[0]
    E = e / W * (1 + 2 * U) + 2 * U * mms
    c = float(np.float32(cutoff_db))
    factor = 10.0 ** (c / 10)
    if reference_power is None:
        ref, dref = float(mms.max()), float(E.max())
    else:
        ref, dref = float(np.float32(reference_power)), 0.0
    thr = ref * factor
    e_thr = factor * dref + thr * (LN10 * 1.5 * U * abs(c) / 10 + 4 * U)
    sure = mms - E >= thr + e_thr
    maybe = mms + E >= thr - e_thr
    res = dict(empty_possible=not sure.any(), nonempty_possible=bool(maybe.any()), W=W)
    if maybe.any():
        fm, fs = int(np.argmax(maybe)), (int(np.argmax(sure)) if sure.any() else n - 1)
        lm, ls = n - 1 - int(np.argmax(maybe[::-1])), (n - 1 - int(np.argmax(sure[::-1])) if sure.any() else 0)
        res["begin"] = (max(fm - (W - 1), 0), max(fs - (W - 1), 0))
        res["end"] = (ls, lm)
    return res


def check_nonsilent(got, band, what=""):
    """got = (begin, length) of a float32 evaluation against nonsilent_band(); returns the width of the band it was checked in."""
    begin, length = int(got[0]), int(got[1])
    if length == 0:
        assert band["empty_possible"], (what, got, band)
        return 0
    assert band["nonempty_possible"], (what, got, band)
    end = begin + length - 1
    b0, b1 = band["begin"]
    e0, e1 = band["end"]
    assert b0 <= begin <= b1 and e0 <= end <= e1, (what, "begin", begin, (b0, b1), "end", end, (e0, e1))
    return max(b1 - b0, e1 - e0)


# ----------------------------------------------------------------------------------------------------------------- AudioResample
def resample_lobes(quality):
    """ResamplingParams::FromQuality (dali/operators/audio/resampling_params.h:27-30): round(0.007 q^2 - 0.09 q + 3)."""
    q = float(np.float32(quality))
    return int(math.floor(0.007 * q * q - 0.09 * q + 3 + 0.5))


def window_exact(x, lobes):
    """The Hann-windowed sinc of dali/kernels/signal/resampling.h:73-96 as a function: sinc(x) * (1 + cos(pi x 64 / coeffs)) / 2,
    coeffs = 64 lobes + 1 (the envelope reaches 0 just beyond |x| = lobes); 0 for |x| >= lobes."""
    coeffs = 64 * lobes + 1
    x = np.asarray(x, np.float64)
    w = np.sinc(x) * 0.5 * (1 + np.cos(np.pi * x * (coeffs - 1) / (lobes * coeffs)))
    return np.where(np.abs(x) < lobes, w, 0.0)


def window_knots(lobes):
    """(x_j, w(x_j)) of the lookup table: coeffs = 64 lobes + 1 knots 1/32 apart, centred on 0."""
    coeffs = 64 * lobes + 1
    xj = (np.arange(coeffs) - 32 * lobes) / 32.0
    return xj, np.sinc(xj) * 0.5 * (1 + np.cos(np.pi * xj * (coeffs - 1) / (lobes * coeffs)))


def resampled_length(n, in_rate, out_rate):
    return int(math.ceil(n * float(out_rate) / float(in_rate)))


def source_positions(out_idx, scale):
    """(in_block_i, p) of each output: the reference splits the output into blocks of 256 and, per block starting at output b,
    accumulates the float32 source position p = (b scale - floor(b scale)) + j * fscale step by step (resampling_cpu.cc:131-136);
    the taps of output b + j are in_block_i + i around p."""
    out_idx = np.asarray(out_idx, np.int64)
    fscale = np.float32(scale)
    blocks = np.unique(out_idx // 256)
    base = np.empty(blocks.size, np.int64)
    pos = np.empty((blocks.size, 256), np.float32)
    for k, blk in enumerate(blocks):
        f = float(blk * 256) * scale
        base[k] = math.floor(f)
        steps = np.full(256, fscale, np.float32)
        steps[0] = np.float32(f - base[k])
        pos[k] = np.add.accumulate(steps, dtype=np.float32)
    k = np.searchsorted(blocks, out_idx // 256)
    return base[k], pos[k, out_idx % 256].astype(np.float64)


def audio_resample(x, in_rate, out_rate, quality=50.0, out_length=None, out_idx=None, exact=False):
    """y[o] = sum over taps i in [ceil(p) - lobes, ceil(p) + lobes) that lie inside the input of x[in_block_i + i] w(i - p)
    (dali/kernels/signal/resampling_cpu.cc:120-230), p and in_block_i from source_positions(), in float64.  x: [n] or [n, channels];
    out_idx: the outputs to evaluate (default all).  Output length ceil(n * out_rate / in_rate) unless out_length is given.

    w is the lookup table's linear interpolation of the float64 knots (exact=False), or the windowed sinc itself (exact=True).
    Bound per output and channel, over its taps:
      sum |x_i| (eps_fi * slope_i + 10u) + (taps + 3) u sum |x_i w_i|            (lookup form)
    eps_fi = (128 lobes + 66) u knots is the error of the float table coordinate x * 32 + center (x = i - p in float, accumulated
    over the taps, then the product and the sum), slope_i the largest knot-to-knot change around the tap's knot, 10u the float
    rounding of the knots and of the interpolation; the sum is one rounding per product and per addition.  exact=True adds the
    interpolation error of the table, h^2 / 8 max |w''| |x_i| per tap with h = 1/32."""
    a = np.asarray(x, np.float32)
    mono = a.ndim == 1
    a2 = a.reshape(a.shape[0], 1 if mono else a.shape[1]).astype(np.float64)
    n, C = a2.shape
    scale = float(in_rate) / float(out_rate)
    n_out = int(out_length) if out_length is not None else resampled_length(n, in_rate, out_rate)
    idx = np.arange(n_out, dtype=np.int64) if out_idx is None else np.asarray(out_idx, np.int64)
    lobes = resample_lobes(quality)
    xj, K = window_knots(lobes)
    D = np.abs(np.diff(K))
    Dloc = np.maximum(np.maximum(np.concatenate(([0.0], D[:-1])), D), np.concatenate((D[1:], [0.0])))   # segments j-1, j, j+1
    eps_fi = (128 * lobes + 66) * U
    if exact:
        g = np.linspace(-lobes, lobes, 4096 * lobes + 1)
        h = g[1] - g[0]
        w2 = np.abs(np.diff(window_exact(g, lobes), 2)) / h ** 2
        interp_err = (1 / 32) ** 2 / 8 * float(w2.max())
    y = np.zeros((idx.size, C))
    bound = np.zeros((idx.size, C))
    for s in range(0, idx.size, 8192):
        o = idx[s:s + 8192]
        if o.size == 0:
            continue
        base, p = source_positions(o, scale)
        xc = np.ceil(p).astype(np.int64)
        taps = np.arange(-lobes, lobes)[None, :] + xc[:, None]            # relative to base
        absi = taps + base[:, None]
        valid = (absi >= 0) & (absi < n)
        xw = taps - p[:, None]                                             # exact in float64
        if exact:
            w = window_exact(xw, lobes)
        else:
            w = np.interp(xw, xj, K)
        w = np.where(valid, w, 0.0)
        j = np.clip(np.floor(xw * 32 + 32 * lobes).astype(np.int64), 0, D.size - 1)
        per_tap = np.where(valid, eps_fi * Dloc[j] + 10 * U + (interp_err if exact else 0.0), 0.0)
        T = valid.sum(axis=1)[:, None]
        v = a2[np.clip(absi, 0, max(n - 1, 0))] if n else np.zeros(absi.shape + (C,))
        v = np.where(valid[..., None], v, 0.0)                              # [outs, taps, C]
        y[s:s + o.size] = np.einsum("otc,ot->oc", v, w)
        bound[s:s + o.size] = np.einsum("otc,ot->oc", np.abs(v), per_tap) + (T + 3) * U * np.einsum("otc,ot->oc", np.abs(v), np.abs(w))
    if mono:
        return y[:, 0], bound[:, 0]
    return y, bound


def check_indices(n_out, lobes_, rng, extra=2000):
    """The outputs a long clip is checked at: every output within two lobes of a 256-block boundary and of both ends, and a seeded
    random subset of `extra` more."""
    span = 2 * lobes_ + 2
    near = [np.arange(0, min(n_out, span)), np.arange(max(0, n_out - span), n_out)]
    for b in range(256, n_out, 256):
        near.append(np.arange(max(0, b - span), min(n_out, b + span)))
    near.append(rng.integers(0, max(n_out, 1), extra) if n_out else np.zeros(0, np.int64))
    return np.unique(np.concatenate(near).astype(np.int64))
