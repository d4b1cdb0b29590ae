"""-m gpu parity tests for WarpAffine, Hsv / linear colour transform, ColorSpaceConversion, Spectrogram and
MelFilterBank: CUDA path (through the C-ABI) vs the oracle."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from dali_b200 import capi  # noqa: E402
from oracle import pyoracle as po  # noqa: E402


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def _rot(rng, h, w):
    ang, s = rng.uniform(-0.5, 0.5), rng.uniform(0.7, 1.4)
    c, si = np.cos(ang) * s, np.sin(ang) * s
    cx, cy = w / 2, h / 2
    return np.float32([[c, -si, cx - c * cx + si * cy + rng.uniform(-5, 5)], [si, c, cy - si * cx - c * cy + rng.uniform(-5, 5)]])


def test_warp_golden(golden_dir):
    import gpu_helpers as g
    gz = np.load(os.path.join(golden_dir, "warp_color_ref.npz"))
    img, M = gz["in"], gz["M"]
    for interp in (0, 1):
        for fill, fn in ((None, "clamp"), (0.0, "fill0")):
            (out,) = g.warp_affine([img], [M], None, interp, fill)
            assert np.array_equal(out, gz[f"out_{interp}_{fn}"]), (interp, fn)


def test_warp_random_batch_bit_exact():
    """Includes outputs wider than 256 px: the reference's incremental coordinates are replayed exactly."""
    import gpu_helpers as g
    rng = np.random.default_rng(51)
    for interp in (0, 1):
        for fill in (None, 42.0):
            for odt in (np.uint8, np.float32):
                imgs, mats, outs = [], [], []
                for it in range(10):
                    H, W = [int(v) for v in rng.integers(2, 400, 2)]
                    C = 3 if it % 4 else 1
                    imgs.append(rng.integers(0, 256, (H, W, C)).astype(np.uint8))
                    mats.append(_rot(rng, H, W))
                    outs.append((int(rng.integers(1, 300)), int(rng.integers(1, 900))) if it % 2 else (H, W))
                got = g.warp_affine(imgs, mats, outs, interp, fill, odt)
                for im, M, hw, o in zip(imgs, mats, outs, got):
                    want = po.warp_affine(im, M, hw, interp, fill, odt)
                    assert np.array_equal(bits(o), bits(want)), (im.shape, hw, interp, fill, odt)


def test_warp_c3_frame():
    import gpu_helpers as g
    rng = np.random.default_rng(52)
    img = rng.integers(0, 256, (720, 1280, 3)).astype(np.uint8)
    M = _rot(rng, 720, 1280)
    (o,) = g.warp_affine([img], [M], None, 1, 0.0)
    assert np.array_equal(o, po.warp_affine(img, M, None, 1, 0.0))


def test_warp_tensor_map_tma_path():
    """Bilinear u8 3-channel batches take the band kernel (anchored coordinate replay); uniform batches at a constant stride
    additionally get their source boxes staged in shared memory by tiled TMA loads through a tensor map (cp.async.bulk.tensor);
    pixels at the border, or whose footprint is not inside the box (large angles, down-scaling maps), fall back per pixel.
    Everything stays bit-exact, for both border modes and for output sizes that are not tile multiples."""
    import gpu_helpers as g
    rng = np.random.default_rng(57)
    for (H, W), out_hw in (((360, 640), None), ((200, 448), (173, 301)), ((96, 1280), (96, 1277))):
        n = 5
        imgs = [rng.integers(0, 256, (H, W, 3)).astype(np.uint8) for _ in range(n)]
        mats = []
        for k, (deg, sc) in enumerate(((3.0, 1.0), (-9.0, 1.04), (40.0, 1.0), (1.0, 2.2), (0.0, 1.0))):
            a = np.deg2rad(deg)
            c, si = np.cos(a) * sc, np.sin(a) * sc
            cx, cy = W / 2, H / 2
            mats.append(np.float32([[c, -si, cx - c * cx + si * cy + 0.37 * k], [si, c, cy - si * cx - c * cy - 0.21 * k]]))
        outs = [out_hw] * n if out_hw else None
        for fill in (None, 17.0):
            got, path = g.warp_affine(imgs, mats, outs, 1, fill, np.uint8, contiguous=True, want_path=True)
            assert path == 1
            for im, M, o in zip(imgs, mats, got):
                assert np.array_equal(o, po.warp_affine(im, M, out_hw, 1, fill, np.uint8)), ((H, W), out_hw, fill)
        # nearest-neighbour and float outputs keep the generic kernel
        got, path = g.warp_affine(imgs, mats, outs, 0, None, np.uint8, contiguous=True, want_path=True)
        assert path == 0
        for im, M, o in zip(imgs, mats, got):
            assert np.array_equal(o, po.warp_affine(im, M, out_hw, 0, None, np.uint8))
    # rows that are not a multiple of 16 bytes cannot be described by a tensor map: generic kernel
    imgs = [rng.integers(0, 256, (64, 301, 3)).astype(np.uint8) for _ in range(2)]
    mats = [np.float32([[1, 0.02, 0.5], [-0.02, 1, 0.25]])] * 2
    got, path = g.warp_affine(imgs, mats, None, 1, None, np.uint8, contiguous=True, want_path=True)
    assert path == 0
    for im, M, o in zip(imgs, mats, got):
        assert np.array_equal(o, po.warp_affine(im, M, None, 1, None, np.uint8))


def test_hsv_and_linear_transform():
    import gpu_helpers as g
    rng = np.random.default_rng(53)
    imgs, Ms, Ts = [], [], []
    for it in range(12):
        H, W = [int(v) for v in rng.integers(1, 200, 2)]
        imgs.append(rng.integers(0, 256, (H, W, 3)).astype(np.uint8))
        M, T = g.color_twist_matrix(rng.uniform(-30, 30), rng.uniform(0.7, 1.3), rng.uniform(0.8, 1.2))
        Mo, To = po.color_twist_matrix(0, 1, 1)
        Ms.append(M); Ts.append(T)
    for odt in (np.uint8, np.float32):
        got = g.linear_transform(imgs, Ms, Ts, odt)
        for im, M, T, o in zip(imgs, Ms, Ts, got):
            assert np.array_equal(bits(o), bits(po.linear_transform(im, M, T, odt)))
    # identity
    Mi, Ti = g.color_twist_matrix(0.0, 1.0, 1.0)
    (o,) = g.linear_transform([imgs[0]], [Mi], [Ti])
    assert np.array_equal(o, imgs[0])


def test_hsv_golden(golden_dir):
    import gpu_helpers as g
    gz = np.load(os.path.join(golden_dir, "warp_color_ref.npz"))
    for i, (h, s, v) in enumerate(gz["hsv_args"]):
        M, T = g.color_twist_matrix(float(h), float(s), float(v))
        assert np.array_equal(M, gz[f"hsv_M_{i}"])
        (o,) = g.linear_transform([gz["in"]], [M], [T])
        assert np.array_equal(o, gz[f"hsv_out_{i}"])


def test_color_space_conversion_all_pairs():
    import gpu_helpers as g
    rng = np.random.default_rng(54)
    cube = np.stack(np.meshgrid(np.arange(0, 256, 5), np.arange(0, 256, 3), np.arange(0, 256, 7), indexing="ij"), -1)
    cube = cube.reshape(-1, 1, 3).astype(np.uint8)
    rgb = [cube, rng.integers(0, 256, (33, 47, 3)).astype(np.uint8), rng.integers(0, 256, (1, 1, 3)).astype(np.uint8)]
    gray = [np.arange(256, dtype=np.uint8).reshape(16, 16, 1), rng.integers(0, 256, (5, 7, 1)).astype(np.uint8)]
    T = {"RGB": (capi.RGB, po.IT_RGB), "BGR": (capi.BGR, po.IT_BGR), "GRAY": (capi.GRAY, po.IT_GRAY), "YCbCr": (capi.YCbCr, po.IT_YCBCR)}
    for a in T:
        for b in T:
            ins = gray if a == "GRAY" else rgb
            got = g.csc(ins, T[a][0], T[b][0])
            for im, o in zip(ins, got):
                assert np.array_equal(o, po.csc(im, T[a][1], T[b][1])), (a, b)


def _clip(rng, n, sr=16000):
    t = np.arange(n) / sr
    x = sum(rng.uniform(0.05, 0.3) * np.sin(2 * np.pi * rng.uniform(50, 7000) * t + rng.uniform(0, 6)) for _ in range(5))
    return np.clip(x + 0.05 * rng.normal(0, 1, n), -1, 1).astype(np.float32)


@pytest.mark.parametrize("cfg", [dict(nfft=1024, window_length=1024, window_step=256), dict(nfft=1024, window_length=512, window_step=256),
                                 dict(nfft=512, window_length=400, window_step=160, center=False),
                                 dict(nfft=2048, window_length=2048, window_step=512, reflect=False),
                                 dict(nfft=256, window_length=256, window_step=64, power=1, layout="tf")])
def test_spectrogram_vs_oracle(cfg):
    """Stated tolerance: 2e-4 of the spectrogram maximum (the reference's own STFT GPU test bound,
    dali/kernels/signal/fft/stft_gpu_test.cu:246: EqualEpsRel(2e-5, 2e-4)); the oracle is a double-precision DFT."""
    import gpu_helpers as g
    rng = np.random.default_rng(61)
    sigs = [_clip(rng, n) for n in (16000, 4000, 2048 + 7, 33001)]
    got = g.spectrogram(sigs, **cfg)
    for s, o in zip(sigs, got):
        want = po.spectrogram(s, **cfg)
        assert o.shape == want.shape
        assert np.abs(o - want).max() <= 2e-4 * want.max()
        # and far tighter in practice
        assert np.abs(o - want).max() <= 5e-6 * want.max()


@pytest.mark.parametrize("cfg", [dict(nfft=1024, window_length=1024, window_step=256), dict(nfft=1024, window_length=800, window_step=200, reflect=False),
                                 dict(nfft=1024, window_length=1024, window_step=512, center=False), dict(nfft=1024, window_length=1024, window_step=160, power=1)])
def test_spectrogram_mel_fused_kernel(cfg):
    """STFT -> mel in one kernel (nfft = 1024: register-resident 32 x 32 FFT, power spectrum parked in shared memory): the
    spectrogram it can optionally write equals the stand-alone spectrogram launch bit for bit, the mel output equals the stand-alone
    mel kernel applied to that spectrogram bit for bit (same summation order), with and without materialising the spectrogram; odd
    window counts, clips shorter than a window (reflect padding) and several clips per batch included."""
    import gpu_helpers as g
    rng = np.random.default_rng(77)
    lens = (16000, 5000, 40001, 1500) if cfg.get("center", True) else (16000, 5000, 40001, 2049)
    sigs = [_clip(rng, n) for n in lens]
    spec = g.spectrogram(sigs, **cfg)
    mel = g.mel_filter_bank(spec, 128, 16000.0, 0.0, 8000.0)
    fs, fm = g.spectrogram_mel_fused(sigs, **cfg)
    _, fm2 = g.spectrogram_mel_fused(sigs, keep_spectrogram=False, **cfg)
    for a, b, c, d, e in zip(spec, mel, fs, fm, fm2):
        assert np.array_equal(bits(a), bits(c))
        assert np.array_equal(bits(b), bits(d)) and np.array_equal(bits(b), bits(e))
    for s_, got in zip(sigs, spec):                       # and the new FFT against the oracle, at the stated tolerance
        want = po.spectrogram(s_, **cfg)
        assert np.abs(got - want).max() <= 2e-4 * max(1e-30, np.abs(want).max())


def test_spectrogram_c4_shape_and_unsupported():
    import gpu_helpers as g
    rng = np.random.default_rng(62)
    (o,) = g.spectrogram([_clip(rng, 160000)], nfft=1024, window_length=1024, window_step=256)
    assert o.shape == (513, 626)
    with pytest.raises(capi.DaliB200Error, match="powers of two"):
        g.spectrogram([_clip(rng, 20000)], nfft=5000, window_length=5000, window_step=160)


@pytest.mark.parametrize("cfg", [dict(nfft=400, window_length=400, window_step=160), dict(nfft=600, window_length=500, window_step=200, center=False),
                                 dict(nfft=1000, window_length=1000, window_step=250, power=1, layout="tf", reflect=False)])
def test_spectrogram_non_power_of_two_nfft(cfg):
    """nfft that is not a power of two (the reference's FFTS complex path): direct DFT kernel, same stated tolerance."""
    import gpu_helpers as g
    rng = np.random.default_rng(64)
    sigs = [_clip(rng, n) for n in (16000, 4000, 1003)]
    got = g.spectrogram(sigs, **cfg)
    for s, o in zip(sigs, got):
        want = po.spectrogram(s, **cfg)
        assert o.shape == want.shape
        assert np.abs(o - want).max() <= 5e-6 * want.max()


def test_mel_filter_bank_bit_exact():
    import gpu_helpers as g
    rng = np.random.default_rng(63)
    specs = [po.spectrogram(_clip(rng, n), nfft=1024, window_length=1024, window_step=256) for n in (16000, 5000, 160000)]
    for (nf, sr, fl, fh, formula, norm) in [(128, 16000.0, 0.0, 8000.0, "slaney", True), (80, 16000.0, 20.0, 7600.0, "htk", False),
                                            (64, 44100.0, 0.0, 0.0, "slaney", True), (40, 22050.0, 100.0, 9000.0, "htk", True)]:
        got = g.mel_filter_bank(specs, nf, sr, fl, fh, formula, norm)
        for s, o in zip(specs, got):
            assert np.array_equal(bits(o), bits(po.mel_filter_bank(s, nf, sr, fl, fh, formula, norm))), (nf, formula)


def _mel_f64(spec, nf, sr, fl, fh, formula, norm):
    """The float64 mel filter bank (tests/image_f64.py mel_weights: triangles between mel-spaced edges at the bin frequencies) applied to
    a spectrogram, and its bound: the weights' own bound times the powers, plus 2 (nterms + 16) u sum_b w P for the float32 sums
    (nterms = the filter's non-zero weights; u = 2^-24; 16 for the ~2^-21 split products of the tensor-core path)."""
    import image_f64 as F
    W, B = F.mel_weights(spec.shape[0], nf, sr, fl, fh, formula == "htk", norm)
    P = spec.astype(np.float64)
    nterms = (W != 0).sum(axis=1, keepdims=True)
    want = W @ P
    return want, B @ P + 2 * (nterms + 16) * 2.0 ** -24 * want


def test_mel_filter_bank_default_path_f64():
    """The default (banded, non-tensor-core) mel kernel against the float64 statement of the weights, within the bound."""
    import gpu_helpers as g
    import image_f64 as F
    rng = np.random.default_rng(65)
    specs = [po.spectrogram(_clip(rng, n), nfft=1024, window_length=1024, window_step=256) for n in (16000, 5000)]
    specs[0][:, 10:20] *= np.float32(1e-12)
    for (nf, sr, fl, fh, formula, norm) in [(128, 16000.0, 0.0, 8000.0, "slaney", True), (80, 16000.0, 20.0, 7600.0, "htk", False),
                                            (200, 44100.0, 0.0, 0.0, "slaney", True), (13, 22050.0, 100.0, 9000.0, "htk", True)]:
        got = g.mel_filter_bank(specs, nf, sr, fl, fh, formula, norm)
        for s, o in zip(specs, got):
            want, tol = _mel_f64(s, nf, sr, fl, fh, formula, norm)
            F.check(o, want, tol, (nf, formula))


def test_mel_filter_bank_tensor_core_path():
    """The optional dense-GEMM path on the tensor cores (TF32 x 3 split, FP32 accumulate): same weights, different summation
    order.  Weights and powers are >= 0, so every output element gets a bound relative to its own float64 value,
    2 (nterms + 16) u sum_b w P against the float32 weights the kernel multiplies (nterms = the filter's non-zero weights; u = 2^-24; 16
    for the ~2^-21 split products): a bound relative to the row maximum would not see a wrong quiet frame, and frames 120 dB below the
    rest are included.  The same outputs are also held to the float64 statement of the weights (_mel_f64), which does not rest on the
    restatement's weights.  Also nfilter not a multiple of 16 / above 128 and window counts that are not multiples of the 64-column tile."""
    import gpu_helpers as g
    import image_f64 as F
    rng = np.random.default_rng(64)
    specs = [po.spectrogram(_clip(rng, n), nfft=1024, window_length=1024, window_step=256) for n in (16000, 5000, 160000, 700)]
    specs[0][:, 10:20] *= np.float32(1e-12)                             # 120 dB below the other frames
    specs[2][:, 63:66] *= np.float32(1e-12)
    specs[2][:, 300] = 0.0
    for (nf, sr, fl, fh, formula, norm) in [(128, 16000.0, 0.0, 8000.0, "slaney", True), (80, 16000.0, 20.0, 7600.0, "htk", False),
                                            (200, 44100.0, 0.0, 0.0, "slaney", True), (13, 22050.0, 100.0, 9000.0, "htk", True)]:
        got = g.mel_filter_bank(specs, nf, sr, fl, fh, formula, norm, tensor_cores=True)
        W = po.mel_weights(specs[0].shape[0], nf, sr, fl, fh, formula, norm).astype(np.float64)
        nterms = (W != 0).sum(axis=1, keepdims=True)
        for s, o in zip(specs, got):
            want64, tol64 = _mel_f64(s, nf, sr, fl, fh, formula, norm)
            F.check(o, want64, tol64, (nf, formula, "float64 weights"))
            want = W @ s.astype(np.float64)
            tol = 2 * (nterms + 16) * 2.0 ** -24 * want
            err = np.abs(o - want)
            assert o.shape == want.shape and np.all(err <= tol), (nf, formula, float((err / np.maximum(tol, 1e-300)).max()))


def test_audio_golden(golden_dir):
    import gpu_helpers as g
    gz = np.load(os.path.join(golden_dir, "audio_ref.npz"))
    (spec,) = g.spectrogram([gz["sig"]], nfft=1024, window_length=512, window_step=256)
    want = gz["spec_nfft1024_power2_float64"]
    assert np.abs(spec - want).max() <= 5e-6 * want.max()
    s32 = want.astype(np.float32)
    (m,) = g.mel_filter_bank([s32], 128, 16000.0, 0.0, 8000.0, "slaney", True)
    assert np.array_equal(bits(m), bits(gz["mel_128_16k_slaney_norm"]))
    (m2,) = g.mel_filter_bank([s32], 40, 16000.0, 20.0, 7600.0, "htk", False)
    assert np.array_equal(bits(m2), bits(gz["mel_40_16k_htk_nonorm"]))


# ------------------------------------------------------------------------------------------------------------------
# audio tail (SURVEY 8f rank 3): to_decibels, mfcc, normalize through the public API
def _tail(name):
    """The compiled reference kernel when oracle/_ref is present, else the plain-C restatement of oracle/audio_oracle.c.  The
    restatement is pinned bit for bit against the compiled reference by tests/test_audio_tail_ref_cpu.py only where oracle/_ref exists;
    everywhere, it and the kernels are held to the float64 statements of tests/audio_tail_f64.py (tests/test_audio_tail_f64_cpu.py,
    tests/test_gpu_audio_tail_f64.py)."""
    return getattr(po, "ref_" + name) if po.have_ref() else getattr(po, name)



def _audio_pipe(batch, source, build):
    from dali_b200 import fn, pipeline_def

    @pipeline_def(batch_size=batch, num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: source, device="gpu", layout="ft")
        return build(fn, x)
    p = pipe()
    p.build()
    return [o.as_cpu() for o in p.run()]


def test_to_decibels_and_mfcc_match_reference_cpu_kernels():
    rng = np.random.default_rng(9)
    mels = [np.abs(rng.normal(0, 1, (80, 37 + 50 * i))).astype(np.float32) ** 2 + 1e-9 for i in range(3)]
    mels[1][3, 5] = 0.0                                                  # below the cut-off
    a, b, c, d, e = _audio_pipe(3, mels, lambda fn, x: (
        fn.to_decibels(x), fn.to_decibels(x, multiplier=20.0, reference=0.5, cutoff_db=-60.0),
        fn.mfcc(fn.to_decibels(x, reference=1.0, cutoff_db=-80.0), n_mfcc=13, dct_type=2, normalize=True, lifter=22.0),
        fn.mfcc(x, n_mfcc=40, dct_type=3), fn.mfcc(x, n_mfcc=7, dct_type=1)))
    for i, m in enumerate(mels):
        # stated tolerance of ToDecibels: device log2f vs glibc log2f, 1e-5 dB absolute + 1e-6 relative
        assert np.allclose(a[i], _tail("to_decibels")(m), rtol=1e-6, atol=1e-5), i
        assert np.allclose(b[i], _tail("to_decibels")(m, 20.0, 0.5, -60.0), rtol=1e-6, atol=1e-5), i
        db = _tail("to_decibels")(m, 10.0, 1.0, -80.0)
        want = _tail("mfcc")(db, 13, 2, True, 22.0)
        assert c[i].shape == want.shape and np.allclose(c[i], want, rtol=0, atol=2e-4 * np.abs(want).max()), i     # inherits the dB tolerance
        assert np.array_equal(d[i], _tail("mfcc")(m, 40, 3)), i           # the DCT itself is bit-exact (same order, same tables)
        assert np.array_equal(e[i], _tail("mfcc")(m, 7, 1)), i
    # the DCT on identical inputs, with liftering: bit-exact
    (f,) = _audio_pipe(3, mels, lambda fn, x: (fn.mfcc(x, n_mfcc=20, lifter=10.0),))
    for i, m in enumerate(mels):
        assert np.array_equal(f[i], _tail("mfcc")(m, 20, 2, False, 10.0)), i


def test_normalize_axes_ddof_epsilon():
    rng = np.random.default_rng(10)
    xs = [rng.normal(3.0, 2.0, (40, 25 + 9 * i)).astype(np.float32) for i in range(3)]
    a, b, c = _audio_pipe(3, xs, lambda fn, x: (fn.normalize(x), fn.normalize(x, axes=[1], ddof=1, epsilon=1e-3),
                                                fn.normalize(x, axis_names="f", scale=2.0, shift=0.5)))
    import audio_tail_f64 as F
    for i, x in enumerate(xs):
        # per-element bounds derived from the conditioning of each group (tests/audio_tail_f64.py)
        F.check(a[i], *F.normalize(x), what=("all", i))
        F.check(b[i], *F.normalize(x, [1], ddof=1, epsilon=1e-3), what=("rows", i))
        F.check(c[i], *F.normalize(x, [0], scale=2.0, shift=0.5), what=("columns", i))


def test_nonsilent_region_matches_reference():
    """fn.nonsilent_region: the moving mean square is a running float sum restarted every `reset_interval` samples -- replayed as the
    same serial recurrence per interval (bit-exact), so (begin, length) equal the reference's for every sample, including all-silent
    clips, clips shorter than the window, a fixed reference power and per-sample cut-offs."""
    from dali_b200 import fn, pipeline_def
    rng = np.random.default_rng(12)
    clips = []
    for n, lead, trail in ((40000, 6000, 9000), (16000, 0, 3000), (30000, 12345, 0), (5000, 0, 0), (1000, 300, 200), (20000, 0, 0)):
        x = (0.4 * np.sin(np.arange(n) * 0.05) + 0.05 * rng.normal(0, 1, n)).astype(np.float32)
        x[:lead] = (1e-5 * rng.normal(0, 1, lead)).astype(np.float32)
        if trail:
            x[n - trail:] = (1e-5 * rng.normal(0, 1, trail)).astype(np.float32)
        clips.append(x)
    clips[3][:] = 0.0                                                   # rest is silence
    cut = [np.float32(v) for v in (-60, -40, -50, -60, -30, -80)]
    n = len(clips)

    @pipeline_def(batch_size=n, num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: clips, device="gpu")
        c = fn.external_source(source=lambda i: cut)
        b0, l0 = fn.nonsilent_region(x)
        b1, l1 = fn.nonsilent_region(x, cutoff_db=c, window_length=512, reset_interval=2048)
        b2, l2 = fn.nonsilent_region(x, cutoff_db=-45.0, window_length=3000, reference_power=0.02, reset_interval=-1)
        return b0, l0, b1, l1, b2, l2
    p = pipe()
    p.build()
    outs = [o.as_cpu() for o in p.run()]
    for i, x in enumerate(clips):
        got = [(int(np.asarray(outs[2 * k][i]).reshape(-1)[0]), int(np.asarray(outs[2 * k + 1][i]).reshape(-1)[0])) for k in range(3)]
        want = [_tail("nonsilent_region")(x), _tail("nonsilent_region")(x, float(cut[i]), 512, None, 2048),
                _tail("nonsilent_region")(x, -45.0, 3000, 0.02, -1)]
        for k in range(3):
            if want[k][1] == 0:
                assert got[k][1] == 0, (i, k, got[k], want[k])           # begin is undefined for an all-silent clip
            else:
                assert got[k] == want[k], (i, k, got[k], want[k])


def test_audio_resample_matches_reference():
    """fn.audio_resample: windowed-sinc resampling with the reference's operation order (four partial sums + scalar tail for one
    channel, in-order taps for several; float source position accumulated per block of 256 outputs) -> bit-exact against the
    compiled reference kernel for up- and down-sampling, `scale`, `out_length`, several qualities, mono and interleaved stereo."""
    from dali_b200 import fn, pipeline_def
    rng = np.random.default_rng(13)
    mono = [_clip(rng, n) for n in (16000, 4001, 700, 25000)]
    stereo = [np.stack([_clip(rng, n), _clip(rng, n)], axis=1) for n in (3000, 9000, 512, 12345)]
    n = len(mono)
    in_r = [np.float32(v) for v in (16000, 44100, 8000, 22050)]
    out_r = [np.float32(v) for v in (44100, 16000, 16000, 8000)]
    lens = [np.int64(v) for v in (12000, 1234, 3000, 5)]

    @pipeline_def(batch_size=n, num_threads=1, device_id=0)
    def pipe():
        x = fn.external_source(source=lambda i: mono, device="gpu")
        s = fn.external_source(source=lambda i: stereo, device="gpu")
        ir = fn.external_source(source=lambda i: in_r)
        orr = fn.external_source(source=lambda i: out_r)
        ol = fn.external_source(source=lambda i: lens)
        return (fn.audio_resample(x, in_rate=ir, out_rate=orr), fn.audio_resample(x, scale=0.37, quality=90.0),
                fn.audio_resample(x, out_length=ol, quality=10.0), fn.audio_resample(s, in_rate=ir, out_rate=orr),
                fn.audio_resample(s, scale=2.5, quality=0.0))
    p = pipe()
    p.build()
    a, b, c, d, e = [o.as_cpu() for o in p.run()]
    for i in range(n):
        assert np.array_equal(bits(a[i]), bits(_tail("audio_resample")(mono[i], float(in_r[i]), float(out_r[i])))), i
        assert np.array_equal(bits(b[i]), bits(_tail("audio_resample")(mono[i], 1.0, float(np.float32(0.37)), 90.0))), i
        L = int(lens[i])
        assert np.array_equal(bits(c[i]), bits(_tail("audio_resample")(mono[i], float(mono[i].shape[0]), float(L), 10.0, out_length=L))), i
        assert np.array_equal(bits(d[i]), bits(_tail("audio_resample")(stereo[i], float(in_r[i]), float(out_r[i])))), i
        assert np.array_equal(bits(e[i]), bits(_tail("audio_resample")(stereo[i], 1.0, 2.5, 0.0))), i
