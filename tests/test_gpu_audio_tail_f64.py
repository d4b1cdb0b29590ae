"""-m gpu: fn.to_decibels, fn.mfcc, fn.normalize, fn.nonsilent_region and fn.audio_resample against the float64 statements of
tests/audio_tail_f64.py, element by element within the stated bounds, on batches that mix the edges where these kernels can go wrong
(many-item maxima, empty samples, every DCT type, tables beyond 48 KB, 1-D and constant normalize groups, windows longer than the clip,
long clips without restarts, 3..8 channels, clips shorter than the resampling window).  The bit-exact comparisons with the plain-C
restatement stay in tests/test_gpu_warp_color_audio.py; these add a check that does not share its reading of the reference.

Each test prints the largest |GPU - float64| / bound it saw (nonsilent_region: the widest band it was checked in)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import audio_tail_f64 as F  # noqa: E402

DCT_CFGS = ((1, False), (2, False), (2, True), (3, False), (3, True), (4, False), (4, True))


def _run(batch, sources, build):
    """One pipeline run: sources = list of (batch list, device, layout); build(fn, *nodes) returns the outputs."""
    from dali_b200 import fn, pipeline_def

    @pipeline_def(batch_size=batch, num_threads=1, device_id=0)
    def pipe():
        nodes = [fn.external_source(source=(lambda s: lambda i: s)(s), device=dev, **({"layout": lay} if lay else {}))
                 for s, dev, lay in sources]
        return build(fn, *nodes)
    p = pipe()
    p.build()
    return [[np.asarray(o[i]) for i in range(batch)] for o in (x.as_cpu() for x in p.run())]


def _report(name, r):
    print(f"\n[ratio] {name}: {r:.3g}")


def _clip(rng, n, sr=16000, dc=0.0):
    t = np.arange(n) / sr
    x = sum(rng.uniform(0.05, 0.3) * np.sin(2 * np.pi * rng.uniform(50, 7000) * t + rng.uniform(0, 6)) for _ in range(3))
    return (dc + x + 0.05 * rng.normal(0, 1, n)).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------------------ MFCC
@pytest.mark.parametrize("nfeat", [1, 2, 80, 128, 400])
def test_mfcc_every_type_against_float64(nfeat):
    """Frame counts 0, 1, 127, 128, 129 and 10 000 in one batch; every DCT type with and without normalize, lifter 0 / 22;
    n_mfcc above nfeat (clipped), and for nfeat 128 ndct 1, 32, 33 and 128 (a 64 KB table: dynamic shared memory); nfeat 400 with
    128 coefficients is a table of exactly 200 KB."""
    rng = np.random.default_rng(100 + nfeat)
    frames = (0, 1, 127, 128, 129, 10000)
    xs = [rng.normal(0, 4, (nfeat, t)).astype(np.float32) for t in frames]
    xs[4][:, 5] = 0.0                                                   # a zero column: exactly 0 out
    cfgs = []
    for t, norm in DCT_CFGS:
        if t == 1 and nfeat < 2:
            continue
        for lift in (0.0, 22.0):
            cfgs.append((min(nfeat + 5, 128), t, norm, lift))
    if nfeat == 128:
        cfgs += [(k, 2, False, 0.0) for k in (1, 32, 33)] + [(128, 3, True, 5.0)]
    outs = _run(len(xs), [(xs, "gpu", "ft")], lambda fn, x: tuple(
        fn.mfcc(x, n_mfcc=k, dct_type=t, normalize=nm, lifter=lf) for k, t, nm, lf in cfgs))
    worst = 0.0
    for (k, t, nm, lf), out in zip(cfgs, outs):
        for x, o in zip(xs, out):
            ref, bnd = F.mfcc(x, k, t, nm, lf)
            worst = max(worst, F.check(o, ref, bnd, ("mfcc", nfeat, x.shape, k, t, nm, lf)))
        assert np.all(out[4][:, 5] == 0)
    _report(f"mfcc nfeat={nfeat}", worst)


def test_mfcc_table_over_200kb_rejected():
    x = [np.zeros((400, 3), np.float32)]
    with pytest.raises(Exception, match="does not fit shared memory"):
        _run(1, [(x, "gpu", "ft")], lambda fn, x: (fn.mfcc(x, n_mfcc=200),))


# ------------------------------------------------------------------------------------------------------------------ ToDecibels
def test_to_decibels_against_float64():
    """A sample of 10^6 elements (245 items of 4096) whose maximum sits in its last item, an all-zero sample, a sample <= 0
    everywhere, empty samples inside the batch, and both multipliers with and without `reference`."""
    rng = np.random.default_rng(200)
    big = (np.abs(rng.normal(0, 1, 10 ** 6)) ** 2).astype(np.float32)
    big[-3] = 75.0
    xs = [np.zeros(0, np.float32), big, np.zeros(5000, np.float32), -np.abs(rng.normal(0, 1, 9000)).astype(np.float32),
          np.zeros(0, np.float32), (np.abs(rng.normal(0, 1, 80 * 129)) ** 2).astype(np.float32) * 1e-3, np.zeros(0, np.float32)]
    xs[5][::7] = 0.0
    cfgs = ((10.0, None, -200.0), (20.0, None, -80.0), (10.0, 0.5, -60.0), (20.0, 2.0, -100.0))
    outs = _run(len(xs), [(xs, "gpu", None)], lambda fn, x: tuple(
        fn.to_decibels(x, multiplier=m, cutoff_db=c, **({} if r is None else {"reference": r})) for m, r, c in cfgs))
    worst = 0.0
    for (m, r, c), out in zip(cfgs, outs):
        for x, o in zip(xs, out):
            worst = max(worst, F.check(o, *F.to_decibels(x, m, r, c), what=("todb", x.size, m, r, c)))
    _report("to_decibels", worst)


# ------------------------------------------------------------------------------------------------------------------- Normalize
def test_normalize_1d_against_float64():
    """1-D clips of 16 000 to 9.6 M samples with a DC offset (one group per clip), with and without ddof / scale / shift."""
    rng = np.random.default_rng(300)
    xs = [_clip(rng, 16000, dc=0.3), _clip(rng, 160000, dc=-2.0), _clip(rng, 9600000, dc=0.5), _clip(rng, 1000, dc=100.0)]
    cfgs = (dict(), dict(ddof=1, scale=2.0, shift=0.5), dict(epsilon=1e-4))
    outs = _run(len(xs), [(xs, "gpu", None)], lambda fn, x: tuple(fn.normalize(x, **kw) for kw in cfgs))
    worst = 0.0
    for kw, out in zip(cfgs, outs):
        for x, o in zip(xs, out):
            worst = max(worst, F.check(o, *F.normalize(x, **kw), what=("normalize 1-D", x.size, kw)))
    _report("normalize 1-D", worst)


def test_normalize_2d_rows_columns_constant_against_float64():
    """Per row, per column and whole-sample groups, with constant rows and columns (sd = 0: exactly `shift` without epsilon, and
    with it), ddof, scale and shift."""
    rng = np.random.default_rng(301)
    xs = []
    for r, c in ((40, 25), (64, 1000), (3, 70000), (257, 5)):
        x = rng.normal(3, 2, (r, c)).astype(np.float32)
        x[:, 2] = np.float32(1 / 3)                                     # a constant column (but for row 1)
        x[1] = np.float32(0.1)                                          # a constant row
        xs.append(x)
    xs.append(np.full((6, 300), np.float32(0.7)))                       # constant everywhere
    cfgs = ((None, dict()), ([1], dict()), ([1], dict(ddof=1, epsilon=1e-3)), ([0], dict(scale=2.0, shift=0.5)),
            ([0], dict(ddof=1)), ([1], dict(epsilon=1e-6, shift=-1.0)))
    outs = _run(len(xs), [(xs, "gpu", "ft")], lambda fn, x: tuple(
        fn.normalize(x, **kw) if ax is None else fn.normalize(x, axes=ax, **kw) for ax, kw in cfgs))
    worst = 0.0
    for (ax, kw), out in zip(cfgs, outs):
        for x, o in zip(xs, out):
            worst = max(worst, F.check(o, *F.normalize(x, ax, **kw), what=("normalize 2-D", x.shape, ax, kw)))
        if ax == [1] and not kw.get("epsilon"):
            assert np.all(out[0][1] == kw.get("shift", 0.0))             # the constant row gives `shift`
    _report("normalize 2-D", worst)


# ------------------------------------------------------------------------------------------------------------- NonsilentRegion
def test_nonsilent_region_against_float64_band():
    """A 10-minute clip (9.6 M samples) with reset_interval -1 and 8192, a clip shorter than the window, per-sample cutoff_db, a fixed
    reference_power and digital silence; each answer lies in the band of answers a float running sum may give, and where the band
    is a single answer it is that answer."""
    rng = np.random.default_rng(400)
    n10 = 16000 * 600
    long = (0.3 * np.sin(np.arange(n10) * 0.01) * (1 + 0.5 * np.sin(np.arange(n10) * 1e-5)) + 0.02 * rng.normal(0, 1, n10)).astype(np.float32)
    long[:800000] = (1e-5 * rng.normal(0, 1, 800000)).astype(np.float32)
    long[-1200000:] = (1e-5 * rng.normal(0, 1, 1200000)).astype(np.float32)
    clips = [long]
    for n, lead, trail in ((40000, 6000, 9000), (1000, 300, 200), (3000, 0, 0), (20000, 0, 5000)):
        x = (0.4 * np.sin(np.arange(n) * 0.05) + 0.05 * rng.normal(0, 1, n)).astype(np.float32)
        x[:lead] = (1e-5 * rng.normal(0, 1, lead)).astype(np.float32)
        if trail:
            x[n - trail:] = (1e-5 * rng.normal(0, 1, trail)).astype(np.float32)
        clips.append(x)
    clips[3][:] = 0.0                                                   # digital silence
    cut = [np.float32(v) for v in (-60, -40, -50, -60, -30)]
    cfgs = (dict(), dict(cutoff_db="per-sample", window_length=4096, reset_interval=8192), dict(window_length=2048, reset_interval=-1),
            dict(cutoff_db=-45.0, window_length=512, reference_power=0.02, reset_interval=-1))
    n = len(clips)

    def build(fn, x, c):
        outs = []
        for kw in cfgs:
            kw = dict(kw)
            if kw.get("cutoff_db") == "per-sample":
                kw["cutoff_db"] = c
            outs += list(fn.nonsilent_region(x, **kw))
        return tuple(outs)
    outs = _run(n, [(clips, "gpu", None), (cut, "cpu", None)], build)
    widest = 0
    for k, kw in enumerate(cfgs):
        for i, x in enumerate(clips):
            got = (int(outs[2 * k][i].reshape(-1)[0]), int(outs[2 * k + 1][i].reshape(-1)[0]))
            a = dict(kw)
            if a.get("cutoff_db") == "per-sample":
                a["cutoff_db"] = float(cut[i])
            a.setdefault("cutoff_db", -60.0)
            a.setdefault("window_length", 2048)
            a.setdefault("reset_interval", 8192)
            widest = max(widest, F.check_nonsilent(got, F.nonsilent_band(x, **a), ("nonsilent", x.size, a)))
    print(f"\n[band] nonsilent_region: widest band {widest} samples")


# --------------------------------------------------------------------------------------------------------------- AudioResample
def _resample_check(outs, xs, specs, name):
    worst = 0.0
    for o, x, (ir, orr, q, L) in zip(outs, xs, specs):
        ref, bnd = F.audio_resample(x, ir, orr, q, out_length=L)
        worst = max(worst, F.check(o, ref, bnd, (name, x.shape, ir, orr, q, L)))
    return worst


@pytest.mark.parametrize("q", [0.0, 50.0, 100.0])
def test_audio_resample_mono_against_float64(q):
    """8k <-> 48k and 44.1k -> 16k, `scale`, `out_length` shorter and longer than natural; clips of 1 sample, fewer samples than
    lobes and 0 samples (out_length 0); every output checked."""
    rng = np.random.default_rng(500 + int(q))
    lens = (24000, 48000, 88200, 1, 5, 0)
    rates = ((8000.0, 48000.0), (48000.0, 8000.0), (44100.0, 16000.0), (8000.0, 48000.0), (48000.0, 8000.0), (44100.0, 16000.0))
    xs = [_clip(rng, n) for n in lens]
    ol = [np.int64(v) for v in (100000, 9000, 40000, 3, 1, 0)]
    ir = [np.float32(r[0]) for r in rates]
    orr = [np.float32(r[1]) for r in rates]
    n = len(xs)
    a, b, c = _run(n, [(xs, "gpu", None), (ir, "cpu", None), (orr, "cpu", None), (ol, "cpu", None)], lambda fn, x, i, o, l: (
        fn.audio_resample(x, in_rate=i, out_rate=o, quality=q), fn.audio_resample(x, scale=0.37, quality=q),
        fn.audio_resample(x, out_length=l, quality=q)))
    worst = _resample_check(a, xs, [(float(i), float(o), q, None) for i, o in zip(ir, orr)], "rates")
    worst = max(worst, _resample_check(b, xs, [(1.0, float(np.float32(0.37)), q, None)] * n, "scale"))
    worst = max(worst, _resample_check(c, xs, [(float(x.shape[0]) if x.shape[0] else 1.0, float(L) if L else 1.0, q, int(L))
                                              for x, L in zip(xs, ol)], "out_length"))
    _report(f"audio_resample mono q={q}", worst)


@pytest.mark.parametrize("q", [0.0, 50.0, 100.0])
def test_audio_resample_channels_against_float64(q):
    """Interleaved 2, 3, 5 and 8 channels (the multi-channel path handles up to 8), up and down."""
    rng = np.random.default_rng(600 + int(q))
    chans = (2, 3, 5, 8)
    xs = [np.stack([_clip(rng, n) for _ in range(C)], axis=1) for n, C in zip((4000, 3001, 2500, 1000), chans)]
    rates = ((8000.0, 48000.0), (48000.0, 8000.0), (44100.0, 16000.0), (16000.0, 44100.0))
    ir = [np.float32(r[0]) for r in rates]
    orr = [np.float32(r[1]) for r in rates]
    (a,) = _run(len(xs), [(xs, "gpu", None), (ir, "cpu", None), (orr, "cpu", None)], lambda fn, x, i, o: (
        fn.audio_resample(x, in_rate=i, out_rate=o, quality=q),))
    _report(f"audio_resample channels q={q}", _resample_check(a, xs, [(float(i), float(o), q, None) for i, o in zip(ir, orr)], "channels"))


def test_audio_resample_long_clip_block_boundaries():
    """A minute at 44.1 kHz to 16 kHz (958 k outputs): every output within two lobes of a 256-output block boundary and of both
    ends, and a seeded random subset; the exact windowed sinc within its interpolation bound as well."""
    rng = np.random.default_rng(700)
    x = _clip(rng, 44100 * 60)
    (a,) = _run(1, [([x], "gpu", None)], lambda fn, s: (fn.audio_resample(s, in_rate=44100.0, out_rate=16000.0, quality=50.0),))
    out = a[0]
    assert out.shape == (F.resampled_length(x.size, 44100.0, 16000.0),)
    idx = F.check_indices(out.size, F.resample_lobes(50.0), rng)
    ref, bnd = F.audio_resample(x, 44100.0, 16000.0, 50.0, out_idx=idx)
    r = F.check(out[idx], ref, bnd, "long clip")
    ref, bnd = F.audio_resample(x, 44100.0, 16000.0, 50.0, out_idx=idx, exact=True)
    F.check(out[idx], ref, bnd, "long clip exact window")
    _report("audio_resample long clip", r)
