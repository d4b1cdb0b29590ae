"""-m gpu: every STFT kernel checked frame by frame against a float64 DFT of the same float32 windowed frame.

A power spectrum spans many decades, so a bound relative to the spectrogram's maximum says nothing about quiet frames or quiet
bins.  Here each frame f gets a bound of its own, on amplitudes A = sqrt(P) (power 2) or A = |X| (power 1):

    |A_gpu - A_ref| <= 8 * ceil(log2 nfft) * 2^-24 * sqrt(nfft) * ||x_f||_2  +  2^-22 * A_ref

x_f = frame f's float32 windowed samples in the nfft buffer.  A frame whose windowed samples are all zero must come out exactly 0.
The constant is not tuned to the kernels: every check first asserts that scipy's float32 FFT of each frame on its own meets the
bound with 4x margin, so the bound states what a single-precision FFT of one frame achieves.  With power 2 the output is |X|^2 in
float32, which cannot resolve a power below the subnormal spacing 2^-149: each side's rounding of P moves A by up to 2^-74.5,
so that much is added for power 2 (it only matters for frames around 1e-19 and below).

The two FFT kernels pack two real frames into one complex transform (frame 2p real part, 2p + 1 imaginary part).  The signals are
built so that all-zero frames and frames 120 dB below their partner sit on either side of such a pair."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.fft

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
from oracle import pyoracle as po  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
P2_FLOOR = 2 * 2.0 ** -74.5


def _cfg(nfft, window_length=None, window_step=None, power=2, layout="ft", padding="reflect"):
    W = window_length or nfft
    return dict(nfft=nfft, window_length=W, window_step=window_step or max(1, W // 4), power=power, layout=layout,
                center=padding != "none", reflect=padding == "reflect")


def _id(c):
    pad = "reflect" if c["reflect"] and c["center"] else ("zero" if c["center"] else "none")
    return f"n{c['nfft']}-w{c['window_length']}-s{c['window_step']}-p{c['power']}-{c['layout']}-{pad}"


# --------------------------------------------------------------------------------------------------------- reference framing
def frames(sig, nfft, window_length, window_step, center=True, reflect=True, **_):
    """float32 [nwin, nfft]: frame f's windowed samples placed at (nfft - window_length) / 2 of the nfft buffer."""
    W, S = window_length, window_step
    c = W // 2 if center else 0
    nwin = po.num_windows(sig.size, W, S, center)
    x = np.pad(sig, (c, W), mode="reflect" if reflect else "constant") if center else sig      # np.pad's reflect is reflect-101
    t = np.arange(nwin)[:, None] * S + np.arange(W)[None, :]
    out = np.zeros((nwin, nfft), np.float32)
    s0 = (nfft - W) // 2
    out[:, s0:s0 + W] = x[t] * po.hann_window(W)                                 # float32 products, as the kernels form them
    return out


def amplitude(spec, power, layout, **_):
    a = np.asarray(spec, np.float64)
    a = a.T if layout == "ft" else a
    return np.sqrt(a) if power == 2 else a


def check_frames(sig, got, cfg, what=""):
    """Per-frame bound of the module docstring; also pins the framing and calibrates the bound (see there)."""
    nfft = cfg["nfft"]
    fr = frames(sig, **cfg)
    want = po.spectrogram(sig, **cfg)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    a_ref, a_got = amplitude(want, **cfg), amplitude(got, **cfg)
    norm = np.linalg.norm(fr.astype(np.float64), axis=1)
    floor = np.where(norm > 0, P2_FLOOR, 0.0)[:, None] if cfg["power"] == 2 else 0.0
    fft_term = (8 * math.ceil(math.log2(nfft)) * U * math.sqrt(nfft) * norm)[:, None]
    # the framing above is the oracle's: numpy's float64 DFT of these frames reproduces it
    a64 = np.abs(np.fft.rfft(fr.astype(np.float64), axis=1))
    assert np.all(np.abs(a64 - a_ref) <= 2 * U * a64 + 1e-12 * norm[:, None] + floor), (what, "framing differs from the oracle")
    # calibration: a float32 FFT of each frame on its own stays within a quarter of the bound
    a32 = np.abs(scipy.fft.rfft(fr, axis=1).astype(np.complex128))
    cal = np.abs(a32 - a64) / np.maximum(fft_term + 4 * U * a64, 1e-300)
    assert cal.max() <= 0.25, (what, "scipy float32 FFT vs bound", float(cal.max()))
    # the kernel
    zero = norm == 0
    assert not np.any(a_got[zero]), (what, "all-zero frames with a non-zero output", np.nonzero(np.any(a_got[zero] != 0, axis=1))[0],
                                     np.nonzero(zero)[0])
    bound = fft_term + 4 * U * a_ref + floor
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(bound > 0, np.abs(a_got - a_ref) / bound, np.where(a_got == a_ref, 0.0, np.inf))
    if not ratio.max() <= 1.0:
        f, k = np.unravel_index(np.argmax(ratio), ratio.shape)
        p = f ^ 1
        raise AssertionError(f"{what}: frame {f} bin {k}: |A_gpu - A_ref| = {abs(a_got[f, k] - a_ref[f, k]):.3e} is {ratio[f, k]:.3g} x the "
                             f"bound; ||x_f|| = {norm[f]:.3e}, pair partner {p}: ||x|| = {norm[p] if p < len(norm) else 0.0:.3e}; "
                             f"{int(np.sum(ratio.max(axis=1) > 1))} of {len(norm)} frames over the bound")
    return fr


# --------------------------------------------------------------------------------------------------------- signals
def _loud(rng, n, amp=1.0):
    t = np.arange(n)
    return (amp * (0.3 * rng.normal(0, 1, n) + 0.5 * np.sin(2 * np.pi * rng.uniform(0.01, 0.45) * t + rng.uniform(0, 6)))).astype(np.float32)


def signals(cfg, seed, batch=44):
    """Zero-padded bursts and 120 dB steps on both sides of a frame pair, an all-zero clip, DC, Nyquist, an impulse, tones at bins
    1 and nfft/2 - 1, amplitudes 1e-20 .. 1e3, the short lengths (1, 2, 3, < half a window, one window, one window + 1), and
    mixed-length noise up to `batch` clips."""
    rng = np.random.default_rng(seed)
    N, W, S, center = cfg["nfft"], cfg["window_length"], cfg["window_step"], cfg["center"]
    c = W // 2 if center else 0
    tail = 2 * W + 3 * S
    z_odd = next(z for z in range(3, 1 << 30, 2) if z * S - c >= 1)
    b_even = 2 * S - c + W                   # frames 0..2 end before b_even, frame 3 reaches past it
    e_odd = z_odd * S - c                    # frame z_odd - 1 reaches below e_odd, frames >= z_odd start at or after it
    sigs = []
    for quiet in (0.0, 1e-6):
        sigs.append(np.concatenate([_loud(rng, b_even, quiet), _loud(rng, tail)]))          # quiet frame 2, loud partner 3
        sigs.append(np.concatenate([_loud(rng, e_odd), _loud(rng, tail, quiet)]))           # loud frame z_odd - 1, quiet partner z_odd
    L = W + 4 * S
    t = np.arange(L)
    sigs.append(np.zeros(L, np.float32))
    sigs.append(np.full(L, 0.7, np.float32))
    sigs.append((0.7 * (-1.0) ** t).astype(np.float32))
    imp = np.zeros(L, np.float32)
    imp[W + S // 2 + 1] = 0.9
    sigs.append(imp)
    for k in sorted({1, N // 2 - 1}):
        sigs.append((0.6 * np.cos(2 * np.pi * k * t / N + rng.uniform(0, 6))).astype(np.float32))
    for amp in (1e-20, 1e-10, 1e-3, 1e3):
        sigs.append(_loud(rng, L, amp))
    lens = (1, 2, 3, max(1, W // 2 - 1), W, W + 1) if center else (W, W + 1, W + S, W + 2 * S + 1)
    sigs += [_loud(rng, n) for n in lens]
    lo = 1 if center else W
    while len(sigs) < batch:
        sigs.append(_loud(rng, int(rng.integers(lo, W + 6 * S)), float(10.0 ** rng.uniform(-3, 1))))
    return sigs


def _check_pairs_covered(frs):
    """The batch holds an all-zero frame as the even and as the odd member of a pair whose partner is not zero, and likewise a
    frame 80+ dB below its partner (the signal steps by 120 dB; the partner's window only partly covers the loud side)."""
    seen = set()
    for fr in frs:
        e = np.linalg.norm(fr.astype(np.float64), axis=1)
        for f in range(len(e) - (len(e) & 1)):
            p = f ^ 1
            if e[p] > 0 and e[f] == 0:
                seen.add(("zero", f & 1))
            elif e[f] > 0 and e[p] >= 1e4 * e[f]:
                seen.add(("quiet", f & 1))
    assert seen == {("zero", 0), ("zero", 1), ("quiet", 0), ("quiet", 1)}, seen


def _gpu(sigs, cfg):
    """Spectrogram launch with the profiled kernel names."""
    import gpu_helpers as g
    capi.profiling(True)
    capi.profiling_collect()
    got = g.spectrogram(sigs, **cfg)
    names = {k for k, _ in capi.profiling_collect()}
    capi.profiling(False)
    return got, names


def _run_and_check(cfg, kernel, seed, batch=44):
    sigs = signals(cfg, seed, batch)
    got, names = _gpu(sigs, cfg)
    frs = [check_frames(s, o, cfg, f"clip {i} (len {s.size})") for i, (s, o) in enumerate(zip(sigs, got))]
    _check_pairs_covered(frs)
    assert kernel in names, (kernel, names)


# --------------------------------------------------------------------------------------------------------- spectrogram1024
CFG_1024 = [_cfg(1024, 1024, 256), _cfg(1024, 1024, 256, power=1, layout="tf", padding="zero"), _cfg(1024, 1024, 512, padding="none"),
            _cfg(1024, 1000, 250), _cfg(1024, 512, 128, power=1, padding="zero"), _cfg(1024, 512, 200, layout="tf", padding="none")]


@pytest.mark.parametrize("cfg", CFG_1024, ids=_id)
def test_spectrogram1024_per_frame(cfg):
    """The register-resident 32 x 32 FFT: window 1024 (interior fast path and border path) and windows 1000 / 512 (in_win_start
    not 0), both paddings and none, power 1 / 2, both layouts."""
    _run_and_check(cfg, "spectrogram_stft", 1024 + CFG_1024.index(cfg))


@pytest.mark.parametrize("cfg", [c for c in CFG_1024 if c["layout"] == "ft"], ids=_id)
def test_spectrogram1024_fused_with_mel_per_frame(cfg):
    """STFT -> mel in one kernel: the spectrogram it writes meets the per-frame bound and equals the stand-alone launch bit for
    bit, its mel (spectrogram kept or not) equals the mel kernel applied to that spectrogram bit for bit, and the mel of an all-zero
    frame is exactly 0."""
    import gpu_helpers as g
    sigs = signals(cfg, 2048)
    spec, names0 = _gpu(sigs, cfg)
    chain = g.mel_filter_bank(spec, 128, 16000.0, 0.0, 8000.0)
    capi.profiling(True)
    capi.profiling_collect()
    fs, fm = g.spectrogram_mel_fused(sigs, **cfg)
    _, fm2 = g.spectrogram_mel_fused(sigs, keep_spectrogram=False, **cfg)
    names = [k for k, _ in capi.profiling_collect()]
    capi.profiling(False)
    for i, (s, a, b, c, d, e) in enumerate(zip(sigs, spec, chain, fs, fm, fm2)):
        fr = check_frames(s, c, cfg, f"clip {i} (len {s.size})")
        zero = ~np.any(fr, axis=1)
        assert not np.any(d[:, zero]) and not np.any(e[:, zero]), (i, "mel of all-zero frames is not 0")
        assert np.array_equal(a.view(np.uint32), c.view(np.uint32)), i
        assert np.array_equal(b.view(np.uint32), d.view(np.uint32)) and np.array_equal(b.view(np.uint32), e.view(np.uint32)), i
    assert "spectrogram_stft" in names0 and names.count("spectrogram_mel_fused") == 2, (names0, names)


# --------------------------------------------------------------------------------------------------------- spectrogram_kernel
_VARIANTS = [dict(power=2, layout="ft", padding="reflect"), dict(power=1, layout="tf", padding="zero"),
             dict(power=2, layout="tf", padding="none"), dict(power=1, layout="ft", padding="reflect"),
             dict(power=2, layout="ft", padding="zero"), dict(power=1, layout="tf", padding="none")]
CFG_RADIX2 = [_cfg(n, n if i % 3 else max(1, 3 * n // 4), **_VARIANTS[i % len(_VARIANTS)])
              for i, n in enumerate((2, 4, 8, 16, 32, 64, 128, 256, 512, 2048, 4096, 8192))]


@pytest.mark.parametrize("cfg", CFG_RADIX2, ids=_id)
def test_spectrogram_radix2_per_frame(cfg):
    """The shared-memory radix-2 FFT, every power of two but 1024: odd and even log2(nfft); at 8192 two frames per CTA and more
    than 96 KB of shared memory."""
    _run_and_check(cfg, "spectrogram_stft_radix2", 2 + CFG_RADIX2.index(cfg))


CFG_RADIX2_1024 = [_cfg(1024, 1024, 256), _cfg(1024, 1000, 250, power=1, layout="tf", padding="zero"),
                   _cfg(1024, 512, 200, padding="none")]


@pytest.mark.skipif(not os.environ.get("DALIB200_STFT_RADIX2"), reason="run by test_spectrogram_radix2_at_nfft1024 in a child process")
@pytest.mark.parametrize("cfg", CFG_RADIX2_1024, ids=_id)
def test_spectrogram_radix2_at_nfft1024_child(cfg):
    _run_and_check(cfg, "spectrogram_stft_radix2", 3 + CFG_RADIX2_1024.index(cfg))


def test_spectrogram_radix2_at_nfft1024():
    """nfft = 1024 takes the radix-2 kernel only with DALIB200_STFT_RADIX2 set, which is read once per process: the cases run in a
    child process."""
    env = dict(os.environ, DALIB200_STFT_RADIX2="1")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-q", "-m", "gpu", "-p", "no:cacheprovider",
                        "-k", "radix2_at_nfft1024_child"], capture_output=True, text=True, timeout=900, env=env, cwd=ROOT)
    tail = r.stdout[-4000:] + r.stderr[-2000:]
    assert r.returncode == 0 and f"{len(CFG_RADIX2_1024)} passed" in r.stdout, tail


# --------------------------------------------------------------------------------------------------------- spectrogram_dft
CFG_DFT = [_cfg(3, 3, 1), _cfg(5, 4, 2, power=1, layout="tf", padding="zero"), _cfg(400, 400, 160, padding="none"),
           _cfg(1000, 800, 250, power=1), _cfg(4095, 4000, 2000, layout="tf")]


@pytest.mark.parametrize("cfg", CFG_DFT, ids=_id)
def test_spectrogram_dft_per_frame(cfg):
    """nfft not a power of two: the direct DFT transforms one frame at a time."""
    _run_and_check(cfg, "spectrogram_dft", 5 + CFG_DFT.index(cfg), batch=44 if cfg["nfft"] < 4000 else 20)


# --------------------------------------------------------------------------------------------------------- through the pipeline
def _tail(name):
    return getattr(po, "ref_" + name) if po.have_ref() else getattr(po, name)


def test_pipeline_silent_frames_mel_and_decibels():
    """spectrogram -> mel_filter_bank -> to_decibels with the spectrogram consumed only by the mel filters (the executor runs the
    fused STFT -> mel kernel) on zero-padded clips: on every frame whose windowed samples are all zero the mel output is exactly 0
    and the dB value equals the reference chain's (the cut-off) within ToDecibels' stated 1e-5 dB."""
    from dali_b200 import fn, pipeline_def
    rng = np.random.default_rng(90)
    clips = []
    for lead, n, trail in ((4100, 16000, 6000), (4096 + 512, 7000, 3 * 256), (0, 9000, 5000), (3000, 1, 3000), (2048, 300, 0)):
        clips.append(np.concatenate([np.zeros(lead, np.float32), _loud(rng, n), np.zeros(trail, np.float32)]))
    clips.append(np.zeros(5000, np.float32))
    cfg = _cfg(1024, 1024, 256)

    @pipeline_def(batch_size=len(clips), num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: clips, device="gpu")
        m = fn.mel_filter_bank(fn.spectrogram(x, nfft=1024, window_length=1024, window_step=256), nfilter=128, sample_rate=16000.0)
        return m, fn.to_decibels(m)
    p = pipe()
    p.build()
    capi.profiling(True)
    capi.profiling_collect()
    mel, db = [o.as_cpu() for o in p.run()]
    names = {k for k, _ in capi.profiling_collect()}
    capi.profiling(False)
    nzero = 0
    for i, s in enumerate(clips):
        zero = ~np.any(frames(s, **cfg), axis=1)
        nzero += int(zero.sum())
        m, d = np.asarray(mel[i]), np.asarray(db[i])
        ref_mel = po.mel_filter_bank(po.spectrogram(s, **cfg), 128, 16000.0, 0.0, 8000.0)
        ref_db = _tail("to_decibels")(ref_mel)
        assert m.shape == ref_mel.shape and d.shape == ref_db.shape, i
        assert not np.any(m[:, zero]), (i, "mel of all-zero frames is not 0", np.nonzero(np.any(m[:, zero] != 0, axis=0))[0])
        assert np.allclose(d[:, zero], ref_db[:, zero], rtol=1e-6, atol=1e-5), (i, float(np.abs(d[:, zero] - ref_db[:, zero]).max()))
    assert nzero >= 40, nzero
    assert "spectrogram_mel_fused" in names, names


# --------------------------------------------------------------------------------------------------------- plan reuse
def test_spectrogram_plan_set_up_again():
    """One plan set up again through nfft 1024 -> 512 -> 4095 -> 1024 -> 8192 with window lengths that shrink and grow (the
    plan's twiddle and window caches): every output equals a fresh plan's bit for bit."""
    import gpu_helpers as g
    rng = np.random.default_rng(91)
    sigs = [_loud(rng, n) for n in (9000, 4001, 700)]
    plan = capi.Plan("Spectrogram", len(sigs))
    for cfg, n in ((_cfg(1024, 1024, 256), 3), (_cfg(512, 400, 160, power=1, layout="tf"), 2), (_cfg(4095, 4000, 1000, padding="zero"), 3),
                   (_cfg(1024, 700, 256, padding="none"), 2), (_cfg(1024, 1024, 256, power=1), 3), (_cfg(8192, 5000, 1000), 1)):
        again = g.spectrogram(sigs[:n], plan=plan, **cfg)
        fresh = g.spectrogram(sigs[:n], **cfg)
        for i, (a, b) in enumerate(zip(again, fresh)):
            assert a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32)), (_id(cfg), i)
