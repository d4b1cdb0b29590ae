"""CPU checks of the float64 audio-tail statements (tests/audio_tail_f64.py): each is pinned to an independent form (scipy's DCTs,
closed forms, the reference's known answers), the plain-C restatements behind the bit-exact GPU tests (oracle/audio_oracle.c, po.*)
meet every bound with 4x margin on the edge matrix of tests/test_gpu_audio_tail_f64.py, and for each operator a plausible arithmetic
mistake, applied to a float32 numpy statement of the operation, is rejected by the bound."""
import numpy as np
import pytest
import scipy.fft

import audio_tail_f64 as F
from oracle import pyoracle as po

U = F.U
f32 = np.float32


def _clip(rng, n, sr=16000):
    t = np.arange(n) / sr
    x = sum(rng.uniform(0.05, 0.3) * np.sin(2 * np.pi * rng.uniform(50, 7000) * t + rng.uniform(0, 6)) for _ in range(5))
    return np.clip(x + 0.05 * rng.normal(0, 1, n), -1, 1).astype(np.float32)


def _margin(got, ref, bound, what):
    r = F.check(got, ref, bound, what)
    assert r <= 0.25, (what, r)
    return r


def _rejected(got, ref, bound, what):
    with pytest.raises(AssertionError):
        F.check(got, ref, bound, what)


# ------------------------------------------------------------------------------------------------------- independent forms
@pytest.mark.parametrize("N", [2, 3, 8, 33, 80, 128])
def test_dct_matrix_equals_scipy(N):
    rng = np.random.default_rng(N)
    x = rng.normal(0, 1, (N, 5))
    for t, norm in ((1, False), (2, False), (2, True), (3, False), (3, True), (4, False), (4, True)):
        if t == 1 and N < 2:
            continue
        want = scipy.fft.dct(x, type=t, axis=0, norm="ortho" if norm else None)
        if not norm:
            want = want / 2
        assert np.allclose(F.dct_matrix(N, N, t, norm) @ x, want, rtol=0, atol=1e-12 * np.abs(want).max()), (N, t, norm)


def test_lifter_and_clipping():
    # mfcc.h:36-41: 1 + L/2 sin(pi (k + 1) / L); L = 2 -> 2, 1, 0, 1, 2, ...
    assert np.allclose(F.lifter_coeffs(5, 2.0), [2, 1, 0, 1, 2], atol=1e-15)
    y, _ = F.mfcc(np.ones((4, 2)), n_mfcc=9)                     # n_mfcc above nfeat: clipped to nfeat
    assert y.shape == (4, 2) and np.allclose(y[:, 0], [4, 0, 0, 0], atol=1e-12)


def test_known_answers_on_restatement_and_statements():
    """The known answers of the reference-shim tests, run against po.* (no reference build needed) and the float64 statements."""
    x = np.array([[1.0, 10.0, 100.0, 1e-30]], np.float32)
    for d in (po.to_decibels(x, 10.0, 1.0, -80.0), F.to_decibels(x, 10.0, 1.0, -80.0)[0]):
        assert np.allclose(d, [[0.0, 10.0, 20.0, -80.0]], atol=1e-5)
    for d in (po.to_decibels(x, 20.0, None, -200.0), F.to_decibels(x, 20.0, None, -200.0)[0]):
        assert np.allclose(d[0, :3], [-40.0, -20.0, 0.0], atol=1e-4)
    m = np.full((8, 3), 2.0, np.float32)
    for c in (po.mfcc(m, 4, 2, False), F.mfcc(m, 4, 2, False)[0]):
        assert c.shape == (4, 3) and np.allclose(c[0], 16.0) and np.abs(c[1:]).max() < 1e-4
    # nonsilence_op.h's example: [0, 0, 0, 0, 50, 50, 0, 0], window 1 -> (4, 2)
    b = np.array([0, 0, 0, 0, 50, 50, 0, 0], np.float32)
    assert po.nonsilent_region(b, -3.0, 1, None, -1) == (4, 2)
    band = F.nonsilent_band(b, -3.0, 1, None, -1)
    assert band["begin"] == (4, 4) and band["end"] == (5, 5)
    # digital silence: threshold 0 with the default reference -> the whole buffer; with a fixed reference -> empty
    z = np.zeros(100, np.float32)
    assert po.nonsilent_region(z, window_length=4, reset_interval=-1) == (0, 100)
    assert F.nonsilent_band(z, window_length=4, reset_interval=-1)["begin"] == (0, 0)
    assert F.nonsilent_band(z, window_length=4, reset_interval=-1)["end"] == (99, 99)
    assert po.nonsilent_region(z, window_length=4, reference_power=1.0, reset_interval=-1)[1] == 0
    assert not F.nonsilent_band(z, window_length=4, reference_power=1.0, reset_interval=-1)["nonempty_possible"]
    # a burst of ones at 400..499, window 16, -20 dB: windows reach 1 % of the maximum mean square (1.0) once they hold 1 sample of
    # 16 (1/16 > 1/100): lo = 400, begin = 400 - 15; the last window holding a burst sample ends at 499 + 15
    x = np.zeros(1000, np.float32)
    x[400:500] = 1.0
    for rp in (None, 1.0):
        assert po.nonsilent_region(x, -20.0, 16, rp, -1) == (385, 514 - 385 + 1)
        band = F.nonsilent_band(x, -20.0, 16, rp, -1)
        assert band["begin"] == (385, 385) and band["end"] == (514, 514)


def test_resample_known_answers():
    rng = np.random.default_rng(0)
    x = rng.uniform(-1, 1, 2000).astype(np.float32)
    # equal rates: the window is sampled at integers -> the signal itself, within the lookup bound
    y, bnd = F.audio_resample(x, 16000.0, 16000.0)
    F.check(po.audio_resample(x, 16000.0, 16000.0), y, bnd, "po equal rates")
    F.check(x, y, bnd, "identity")
    assert np.abs(y - x).max() < 1e-6
    assert po.audio_resample(x, 16000.0, 44100.0).shape == (F.resampled_length(2000, 16000, 44100),) == (5513,)
    assert po.audio_resample(x, 44100.0, 16000.0).shape == (F.resampled_length(2000, 44100, 16000),) == (726,)
    # a slow sine survives 2x up-sampling
    s = np.sin(2 * np.pi * np.arange(4000) / 200).astype(np.float32)
    want = np.sin(2 * np.pi * (np.arange(8000) / 2.0) / 200)
    for u in (po.audio_resample(s, 1.0, 2.0, 90.0), F.audio_resample(s, 1.0, 2.0, 90.0)[0], F.audio_resample(s, 1.0, 2.0, 90.0, exact=True)[0]):
        assert u.shape == (8000,) and np.abs(u[100:-100] - want[100:-100]).max() < 2e-3
    # interleaved stereo: channels resampled independently
    st = np.stack([s, -s], axis=1)
    v = po.audio_resample(st, 1.0, 2.0, 90.0)
    assert v.shape == (8000, 2) and np.abs(v[:, 0] + v[:, 1]).max() < 1e-6
    y2, _ = F.audio_resample(st, 1.0, 2.0, 90.0)
    assert np.array_equal(y2[:, 0], -y2[:, 1])


# ------------------------------------------------------------------------------------------- restatements within the bounds
def test_to_decibels_restatement_within_bound():
    rng = np.random.default_rng(1)
    big = (np.abs(rng.normal(0, 1, 10 ** 6)) ** 2).astype(np.float32)
    big[-1] = 50.0                                                       # the maximum in the last 4096-element item
    samples = [big, np.zeros(300, np.float32), -np.abs(rng.normal(0, 1, 500)).astype(np.float32),
               (np.abs(rng.normal(0, 1, (80, 129))) ** 2).astype(np.float32)]
    samples[3][:, 7] = 0
    for s in samples:
        for args in ((10.0, None, -200.0), (20.0, None, -80.0), (10.0, 0.5, -60.0), (20.0, 2.0, -100.0)):
            _margin(po.to_decibels(s, *args), *F.to_decibels(s, *args), what=("todb", s.shape, args))


def test_mfcc_restatement_within_bound():
    rng = np.random.default_rng(2)
    for nfeat in (1, 2, 80, 128, 400):
        x = rng.normal(0, 4, (nfeat, 129)).astype(np.float32)
        x[:, 3] = 0
        for t, norm in ((1, False), (2, False), (2, True), (3, False), (3, True), (4, False), (4, True)):
            if t == 1 and nfeat < 2:
                continue
            for n_mfcc, lift in ((nfeat + 5, 0.0), (min(nfeat, 128), 22.0), (13, 2.0)):
                got = po.mfcc(x, n_mfcc, t, norm, lift)
                ref, bnd = F.mfcc(x, n_mfcc, t, norm, lift)
                _margin(got, ref, bnd, ("mfcc", nfeat, t, norm, n_mfcc, lift))
                assert np.all(got[:, 3] == 0)


def normalize_f32(x, axes=None, ddof=0, epsilon=0.0, scale=1.0, shift=0.0, pivot=True, use_ddof=True):
    """float32 numpy statement of normalize in the order the bound is stated for: deviations from the group's first element summed
    in 256 interleaved sequential partial sums, then a tree."""
    a = np.asarray(x, np.float32)
    g, back = F._groups(a, axes)
    out = np.empty_like(g)
    n = g.shape[1]

    def tsum(v):                                                         # v: [n] float32
        pad = np.zeros(-(-n // 256) * 256, np.float32)
        pad[:n] = v
        part = np.add.accumulate(pad.reshape(-1, 256), axis=0, dtype=np.float32)[-1].reshape(8, 32)
        for o in (16, 8, 4, 2, 1):                                       # butterfly inside each warp of 32, then the 8 warps in order
            part = (part[:, :o] + part[:, o:2 * o]).astype(np.float32)
        return np.add.accumulate(part[:, 0], dtype=np.float32)[-1]
    for r in range(g.shape[0]):
        v = g[r] - (g[r, 0] if pivot else f32(0))
        mean = f32(tsum(v) / f32(n))
        d = (v - mean).astype(np.float32)
        var = f32(tsum(d * d) / f32(max(1, n - (ddof if use_ddof else 0))))
        sd = np.sqrt(f32(var + f32(epsilon)), dtype=np.float32)
        mul = f32(f32(scale) / sd) if sd != 0 else f32(0)
        out[r] = d * mul + f32(shift)
    return back(out)


NORMALIZE_CASES = [
    (lambda rng: (0.3 + 0.1 * rng.normal(0, 1, 16000)).astype(np.float32), dict()),
    (lambda rng: (-2.0 + 0.05 * rng.normal(0, 1, 300000)).astype(np.float32), dict(ddof=1, scale=2.0, shift=0.5)),
    (lambda rng: rng.normal(3, 2, (40, 43)).astype(np.float32), dict(axes=[1], ddof=1, epsilon=1e-3)),
    (lambda rng: rng.normal(3, 2, (40, 43)).astype(np.float32), dict(axes=[0], scale=2.0, shift=0.5)),
    (lambda rng: rng.normal(3, 2, (40, 43)).astype(np.float32), dict()),
]


def test_normalize_statement_within_bound():
    rng = np.random.default_rng(3)
    for make, kw in NORMALIZE_CASES:
        x = make(rng)
        ref, bnd = F.normalize(x, **kw)
        _margin(normalize_f32(x, **kw), ref, bnd, ("normalize", x.shape, kw))
    # constant rows: exactly `shift` (with and without epsilon)
    c = np.tile(np.float32([0.1, 0.7, 1 / 3, 3333.3333, -2.5e-3])[:, None], (1, 300))
    for kw in (dict(axes=[1]), dict(axes=[1], epsilon=1e-6, shift=0.25)):
        ref, bnd = F.normalize(c, **kw)
        assert np.all(ref == kw.get("shift", 0.0)) and np.all(bnd <= U * abs(kw.get("shift", 0.0)))
        F.check(normalize_f32(c, **kw), ref, bnd, ("constant", kw))


def _nonsilent_clips(rng):
    clips = []
    for n, lead, trail in ((40000, 6000, 9000), (16000, 0, 3000), (30000, 12345, 0), (1000, 300, 200), (20000, 0, 0)):
        x = (0.4 * np.sin(np.arange(n) * 0.05) + 0.05 * rng.normal(0, 1, n)).astype(np.float32)
        x[:lead] = (1e-5 * rng.normal(0, 1, lead)).astype(np.float32)
        if trail:
            x[n - trail:] = (1e-5 * rng.normal(0, 1, trail)).astype(np.float32)
        clips.append(x)
    return clips


def test_nonsilent_restatement_within_band():
    rng = np.random.default_rng(4)
    for x in _nonsilent_clips(rng) + [np.zeros(5000, np.float32)]:
        for kw in (dict(), dict(cutoff_db=-40.0, window_length=512, reset_interval=2048), dict(window_length=60000, reset_interval=-1),
                   dict(cutoff_db=-45.0, window_length=3000, reference_power=0.02, reset_interval=-1), dict(reference_power=1e-3)):
            F.check_nonsilent(po.nonsilent_region(x, **kw), F.nonsilent_band(x, **kw), (x.size, kw))


@pytest.mark.parametrize("q", [0.0, 50.0, 100.0])
def test_resample_restatement_within_bound(q):
    """The lookup form with 4x margin; the exact form within its bound (the interpolation error h^2/8 max|w''| is a bound the
    table's own error comes close to, 0.7 of it at quality 0)."""
    rng = np.random.default_rng(5)
    for C in (1, 2, 3, 5, 8):
        for ir, orr in ((8000.0, 48000.0), (48000.0, 8000.0), (44100.0, 16000.0)):
            x = rng.uniform(-1, 1, (3001, C)).astype(np.float32)
            x = x[:, 0] if C == 1 else x
            got = po.audio_resample(x, ir, orr, q)
            _margin(got, *F.audio_resample(x, ir, orr, q), what=("resample", q, C, ir, orr))
            F.check(got, *F.audio_resample(x, ir, orr, q, exact=True), what=("resample exact", q, C, ir, orr))
    x = rng.uniform(-1, 1, 5).astype(np.float32)                       # shorter than the window, output longer than natural
    for L in (3, 40):
        got = po.audio_resample(x, 5.0, float(L), q, out_length=L)
        _margin(got, *F.audio_resample(x, 5.0, float(L), q, out_length=L), what=("short", q, L))


# ----------------------------------------------------------------------------------------------- the bounds discriminate
def test_mutations_are_rejected():
    rng = np.random.default_rng(6)
    # to_decibels: the cut-off ratio taken as 10^(cutoff / 10) whatever the multiplier
    s = (np.abs(rng.normal(0, 1, 4000)) ** 2).astype(np.float32)
    s[:50] = 1e-12
    ref, bnd = F.to_decibels(s, 20.0, None, -80.0)
    mx = s.max()
    bad = f32(20 * np.log10(2)) * np.log2(np.maximum(f32(10 ** (-80 / 10)), s * (f32(1) / mx))).astype(np.float32)
    _rejected(bad, ref, bnd, "todb cut-off")
    # MFCC: lifter index k instead of k + 1, and DCT-III without the halved x_0
    x = rng.normal(0, 1, (40, 64)).astype(np.float32)
    ref, bnd = F.mfcc(x, 13, 2, False, 22.0)
    c = F.dct_matrix(40, 13, 2).astype(np.float32)
    lift_k = (1 + f32(11.0) * np.sin(f32(np.pi / 22) * np.arange(13, dtype=np.float32))).astype(np.float32)
    _rejected((c @ x) * lift_k[:, None], ref, bnd, "mfcc lifter index")
    ref, bnd = F.mfcc(x, 20, 3, False)
    c3 = F.dct_matrix(40, 20, 3)
    c3[:, 0] = 1.0
    _rejected(c3.astype(np.float32) @ x, ref, bnd, "dct3 x0")
    # normalize: ddof ignored; the sums without the first-element pivot (a constant row comes out +-scale)
    xr = rng.normal(3, 2, (40, 43)).astype(np.float32)
    ref, bnd = F.normalize(xr, axes=[1], ddof=1)
    _rejected(normalize_f32(xr, axes=[1], ddof=1, use_ddof=False), ref, bnd, "ddof")
    cst = np.tile(np.float32([0.1, 0.7, 1 / 3])[:, None], (1, 300))
    ref, bnd = F.normalize(cst, axes=[1])
    _rejected(normalize_f32(cst, axes=[1], pivot=False), ref, bnd, "no pivot")
    # nonsilent_region: the window - 1 adjustment dropped, and partial windows divided by the samples seen
    b = np.zeros(3000, np.float32)
    b[1200:1700] = 0.5
    band = F.nonsilent_band(b, -30.0, 64, None, -1)
    lo, l = po.nonsilent_region(b, -30.0, 64, None, -1)
    with pytest.raises(AssertionError):
        F.check_nonsilent((lo + 63, l - 63), band, "no window adjustment")
    e = np.zeros(3000, np.float32)
    e[:40] = 0.5                                                       # a burst at the very start: partial windows decide
    band = F.nonsilent_band(e, -20.0, 512, None, -1)
    t = np.arange(3000)
    sq = np.cumsum(e.astype(np.float64) ** 2)
    mms_seen = (sq - np.concatenate((np.zeros(512), sq[:-512]))) / np.minimum(t + 1, 512)
    hit = np.nonzero(mms_seen >= mms_seen.max() * 0.01)[0]
    with pytest.raises(AssertionError):
        F.check_nonsilent((max(hit[0] - 511, 0), hit[-1] - max(hit[0] - 511, 0) + 1), band, "partial windows / count")
    # audio_resample: window centre one knot off, tap range one short
    x = rng.uniform(-1, 1, 2000).astype(np.float32)
    ref, bnd = F.audio_resample(x, 16000.0, 44100.0, 0.0)
    lobes = F.resample_lobes(0.0)
    xj, K = F.window_knots(lobes)
    for shift_knots, drop_last in ((1, False), (0, True)):
        base, p = F.source_positions(np.arange(ref.size), 16000.0 / 44100.0)
        xc = np.ceil(p).astype(np.int64)
        hi = lobes - (1 if drop_last else 0)
        taps = np.arange(-lobes, hi)[None, :] + xc[:, None]
        absi = taps + base[:, None]
        ok = (absi >= 0) & (absi < x.size)
        xw = (taps - p[:, None]).astype(np.float32)
        w = np.interp(xw + shift_knots / 32.0, xj, K).astype(np.float32)
        v = np.where(ok, x[np.clip(absi, 0, x.size - 1)], 0).astype(np.float32)
        bad = np.add.accumulate(v * w, axis=1, dtype=np.float32)[:, -1]
        _rejected(bad, ref, bnd, ("resample", shift_knots, drop_last))
