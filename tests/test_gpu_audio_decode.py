"""-m gpu: fn.decoders.audio on WAV and FLAC.

The corpus of tests/audio_streams.py decodes bit-exactly against the samples its encoder was given (FLOAT / INT16 / INT32), and so does a
10-minute stereo 48 kHz FLAC clip.  The downmix equals the float32 statement of the reference's expression bit for bit and a float64 mean
within a stated bound.  sample_rate=16000 equals fn.audio_resample applied to the decoder's own un-resampled output.  Corrupt streams
raise "Failed to decode sample #i" while the others decode.  fn.readers.file feeds files through DALIGenericIterator, and the Jasper
front-end run from FLAC files gives the bits of the same chain fed the encoder's samples."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import audio_streams as aus  # noqa: E402
from dali_b200 import fn, pipeline_def, types  # noqa: E402
from test_audio_decode_cpu import FLOAT, INT16, INT32, expected  # noqa: E402

_DT = {FLOAT: types.FLOAT, INT16: types.INT16, INT32: types.INT32}


def _decode(streams, **kw):
    @pipeline_def(batch_size=len(streams), num_threads=1, device_id=0)
    def pipe():
        return fn.decoders.audio(fn.external_source(source=lambda i: streams), **kw)
    p = pipe()
    p.build()
    audio, rate = p.run()
    return audio.as_cpu(), [float(r) for r in rate.as_cpu()], audio.layout()


def _same(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, (what, a.shape, b.shape, a.dtype, b.dtype)
    assert np.array_equal(a.view(np.uint8), b.view(np.uint8)), (what, int(np.sum(a != b)))


@pytest.mark.parametrize("dtype", [FLOAT, INT16, INT32])
def test_corpus_bit_exact(dtype):
    corpus = [c for c in aus.corpus() if not (dtype != FLOAT and c[2].dtype == np.float32)]
    streams = [np.frombuffer(s, np.uint8) for _, s, _, _ in corpus]
    out, rates, layout = _decode(streams, dtype=_DT[dtype])
    assert layout == "TC"
    for (name, s, x, bits), got in zip(corpus, out):
        _same(got, expected(x, bits, dtype), name)


def test_downmix_exact_and_near_the_mean():
    corpus = aus.corpus()
    streams = [np.frombuffer(s, np.uint8) for _, s, _, _ in corpus]
    out, rates, layout = _decode(streams, downmix=True)
    assert layout == "T"
    for (name, s, x, bits), got in zip(corpus, out):
        want = expected(x, bits, FLOAT, downmix=True)[:, 0]
        _same(got, want, name)
        f = expected(x, bits, FLOAT).astype(np.float64)
        # C products and C - 1 sums, each rounded once: |error| <= C * 2^-24 * max|x| (|x| <= 1.5 in the float WAVs)
        C = f.shape[1]
        assert np.all(np.abs(got - f.mean(1)) <= C * 2.0 ** -24 * max(1.0, np.abs(f).max())), name


def test_resampling_equals_audio_resample_on_the_decoders_output():
    rng = np.random.default_rng(5)
    items = []
    for rate, C, bits in ((44100, 2, 16), (48000, 1, 24), (22050, 3, 8), (8000, 2, 16), (16000, 1, 16)):
        x = aus.signal(3 * rate // 10, C, bits, rng)
        items.append((aus.flac(x, bits, rate, [576] * (len(x) // 576) + [len(x) % 576]) if len(x) % 576 else
                       aus.flac(x, bits, rate, [576] * (len(x) // 576)), rate))
    items.append((aus.wav_pcm(aus.signal(5000, 2, 16, rng), 16, 11025), 11025))
    streams = [np.frombuffer(s, np.uint8) for s, _ in items]
    raw, raw_rates, _ = _decode(streams, downmix=True)
    assert raw_rates == [float(r) for _, r in items]
    res, rates, _ = _decode(streams, downmix=True, sample_rate=16000.0)
    assert rates == [16000.0] * len(items)
    for i, (s, r) in enumerate(items):
        want = _audio_resample(raw[i], r, 16000.0) if r != 16000 else raw[i]
        assert len(res[i]) == math.ceil(len(raw[i]) * 16000.0 / r)
        _same(res[i], want, (i, r))


def _audio_resample(x, in_rate, out_rate):
    """fn.audio_resample of one float signal on the GPU"""
    @pipeline_def(batch_size=1, num_threads=1, device_id=0)
    def pipe():
        return fn.audio_resample(fn.external_source(source=lambda k: [x], device="gpu"), in_rate=float(in_rate), out_rate=float(out_rate))
    p = pipe()
    p.build()
    return p.run()[0].as_cpu()[0]


def test_per_sample_rates():
    rng = np.random.default_rng(6)
    xs = [aus.signal(4000, 1, 16, rng) for _ in range(3)]
    streams = [np.frombuffer(aus.wav_pcm(x, 16, 22050), np.uint8) for x in xs]
    targets = [np.array(v, np.float32) for v in (8000, 16000, 44100)]

    @pipeline_def(batch_size=3, num_threads=1, device_id=0)
    def pipe():
        sr = fn.external_source(source=lambda i: targets)
        return fn.decoders.audio(fn.external_source(source=lambda i: streams), sample_rate=sr, downmix=True)
    p = pipe()
    p.build()
    audio, rate = p.run()
    got = audio.as_cpu()
    assert [float(r) for r in rate.as_cpu()] == [8000.0, 16000.0, 44100.0]
    raw, _, _ = _decode(streams, downmix=True)
    for x, g, t, r in zip(xs, got, targets, raw):
        assert len(g) == math.ceil(4000 * float(t) / 22050)
        _same(g, _audio_resample(r, 22050, float(t)), float(t))


@pytest.mark.parametrize("kw", [dict(downmix=True), dict(sample_rate=16000.0)])
@pytest.mark.parametrize("dtype", [types.INT16, types.INT32])
def test_integer_output_with_downmix_or_resampling_is_refused_when_the_operator_is_built(dtype, kw):
    streams = [np.frombuffer(aus.corpus()[0][1], np.uint8)]

    @pipeline_def(batch_size=1, num_threads=1, device_id=0)
    def pipe():
        return fn.decoders.audio(fn.external_source(source=lambda i: streams), dtype=dtype, **kw)
    p = pipe()
    try:
        p.build()
        raised = ""
    except Exception as e:  # noqa: BLE001 -- the operator's construction error, checked by its message
        raised = str(e)
    assert "integer output (INT16 / INT32) is not available with `downmix` or `sample_rate`" in raised, raised


def test_long_stereo_clip_bit_exact():
    """10 minutes of 48 kHz stereo 16-bit FLAC (verbatim frames written column-wise, CRC-16 for all frames at once)"""
    rng = np.random.default_rng(10)
    T, bs = 48000 * 600, 4096
    x = (rng.integers(-3000, 3000, (T, 2)) + (8000 * np.sin(np.arange(T) * 0.01))[:, None]).astype(np.int16)
    nfr = (T + bs - 1) // bs
    frames = []
    for k in range(nfr):
        blk = x[k * bs:(k + 1) * bs]
        n = len(blk)
        code = 12 if n == bs else 7
        h = bytearray([0xFF, 0xF8, (code << 4) | 10, (1 << 4) | (4 << 1)]) + aus.utf8_number(k)
        if code == 7:
            h += (n - 1).to_bytes(2, "big")
        h.append(aus.crc8(h))
        frames.append(bytes(h) + b"\x02" + blk[:, 0].astype(">i2").tobytes() + b"\x02" + blk[:, 1].astype(">i2").tobytes())
    crcs = aus.crc16_many(frames)
    s = b"fLaC" + aus.meta_block(0, aus.streaminfo(bs, bs, 48000, 2, 16, T), True) + b"".join(f + c.to_bytes(2, "big") for f, c in zip(frames, crcs))
    out, rates, _ = _decode([np.frombuffer(s, np.uint8)], dtype=types.INT16)
    assert rates == [48000.0]
    _same(out[0], x, "10 min clip")


def test_corrupt_samples_raise_while_others_decode():
    good = aus.corpus()[0]
    for name, bad in aus.corrupt():
        streams = [np.frombuffer(good[1], np.uint8), np.frombuffer(bad, np.uint8)]
        try:
            _decode(streams)
            raised = ""
        except Exception as e:  # noqa: BLE001 -- the executor's error, checked by its message
            raised = str(e)
        assert "Failed to decode sample #1" in raised, (name, raised)
    out, _, _ = _decode([np.frombuffer(good[1], np.uint8)] * 2)
    _same(out[1], expected(good[2], good[3]), "good after corrupt")


def test_refusals_name_the_sample():
    good = aus.corpus()[0][1]
    for name, s, code, why in aus.refused()[:6]:
        with pytest.raises(Exception, match="sample 1"):
            _decode([np.frombuffer(good, np.uint8), np.frombuffer(s, np.uint8)])


def _write_files(tmp_path, rng):
    (tmp_path / "a").mkdir()
    want = []
    for k, (C, bits, kind) in enumerate(((1, 16, "flac"), (2, 16, "wav"), (2, 24, "flac"), (3, 8, "wav"), (1, 16, "flac"), (2, 16, "flac"))):
        x = aus.signal(16000 + 1234 * k, C, bits, rng)
        if kind == "flac":
            n = len(x)
            s = aus.flac(x, bits, 16000, [4096] * (n // 4096) + [n % 4096], assign=lambda f: 10 if C == 2 else C - 1,
                         spec=lambda f, c, b: {"kind": "lpc", "order": 8, "precision": 12, "porder": 0 if len(b) % 4 else 2})
        else:
            s = aus.wav_pcm(x, bits, 16000)
        (tmp_path / "a" / f"clip{k}.{kind}").write_bytes(s)
        want.append((x, bits))
    return want


def test_readers_file_and_generic_iterator(tmp_path):
    from dali_b200.plugin.pytorch import DALIGenericIterator
    want = _write_files(tmp_path, np.random.default_rng(12))

    @pipeline_def(batch_size=len(want), num_threads=1, device_id=0)
    def pipe():
        data, label = fn.readers.file(file_root=str(tmp_path), name="Reader")
        audio, sr = fn.decoders.audio(data, downmix=True, dtype=types.FLOAT)
        return audio, sr, label
    p = pipe()
    p.build()
    audio, sr, _ = p.run()
    for (x, bits), got in zip(want, audio.as_cpu()):
        _same(got, expected(x, bits, FLOAT, downmix=True)[:, 0], "reader")

    @pipeline_def(batch_size=len(want), num_threads=1, device_id=0)
    def padded():
        data, label = fn.readers.file(file_root=str(tmp_path), name="Reader")
        audio, sr = fn.decoders.audio(data, downmix=True)
        return fn.pad(audio, fill_value=0.0), sr
    it = DALIGenericIterator([padded()], ["audio", "sr"], reader_name="Reader")
    batch = next(iter(it))[0]
    n = max(len(x) for x, _ in want)
    assert tuple(batch["audio"].shape) == (len(want), n) and batch["sr"].cpu().tolist() == [16000.0] * len(want)
    for k, (x, bits) in enumerate(want):
        _same(batch["audio"][k, :len(x)].cpu().numpy(), expected(x, bits, FLOAT, downmix=True)[:, 0], "iterator")


def test_jasper_front_end_from_flac_files(tmp_path):
    want = _write_files(tmp_path, np.random.default_rng(13))
    feed = [expected(x, bits, FLOAT, downmix=True)[:, 0] for x, bits in want]

    def chain(x):
        x = fn.preemphasis_filter(x)
        x = fn.spectrogram(x, nfft=512, window_length=320, window_step=160)
        x = fn.mel_filter_bank(x, sample_rate=16000.0, nfilter=64)
        x = fn.to_decibels(x, multiplier=math.log(10), reference=1.0, cutoff_db=math.log(1e-20))
        x = fn.normalize(x, axes=[1])
        return fn.pad(x, axes=[1], fill_value=0.0, align=16)

    @pipeline_def(batch_size=len(want), num_threads=1, device_id=0)
    def from_files():
        data, _ = fn.readers.file(file_root=str(tmp_path))
        audio, _ = fn.decoders.audio(data, downmix=True, sample_rate=16000)
        return chain(audio)

    @pipeline_def(batch_size=len(want), num_threads=1, device_id=0)
    def from_samples():
        return chain(fn.external_source(source=lambda i: feed, device="gpu"))
    outs = []
    for mk in (from_files, from_samples):
        p = mk()
        p.build()
        outs.append(p.run()[0].as_cpu())
    for a, b in zip(*outs):
        _same(a, b, "jasper")
