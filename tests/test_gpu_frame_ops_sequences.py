"""-m gpu: the frame operators on sequences whose samples differ in frame count and frame size, with outputs of more than one byte
per element, so that the frames of each sample lie at strides of their own in the output.  Every output frame must equal, bit for bit,
the same operator applied to that frame as a sample of its own: a frame placed at the wrong offset fails the comparison."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIMS = ((3, 37, 53), (1, 20, 16), (4, 9, 30))          # (frames, H, W) of each sample


def _sequences(channel_first=False):
    rng = np.random.default_rng(11)
    return [rng.integers(0, 256, (f, 3, h, w) if channel_first else (f, h, w, 3), dtype=np.uint8) for f, h, w in DIMS]


def _run(batch, layout, op, keep=None):
    """op(fn, types, x) on the GPU batch `batch` of layout `layout`; the output samples as numpy arrays.  keep collects the pipelines
    whose random state must stay their own until the test ends."""
    from dali_b200 import fn, pipeline_def, types

    @pipeline_def(batch_size=len(batch), num_threads=1, device_id=0)
    def pipe():
        return op(fn, types, fn.external_source(source=lambda i: batch, device="gpu", layout=layout))
    p = pipe()
    p.build()
    (out,) = [o.as_cpu() for o in p.run()]
    if keep is not None:
        keep.append(p)
    return [np.asarray(out[i]) for i in range(len(batch))]


def _assert_same(got, want, what):
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, got.dtype, want.shape, want.dtype)
    assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), what


def _check_per_frame(op, seq_layout, frame_layout, channel_first=False, frame_op=None):
    """op on the sequences against frame_op (default: op) on their frames as one batch"""
    seqs = _sequences(channel_first)
    got = _run(seqs, seq_layout, op)
    frames = [s[f] for s in seqs for f in range(s.shape[0])]
    want = iter(_run(frames, frame_layout, frame_op or op))
    for i, s in enumerate(seqs):
        assert got[i].shape[0] == s.shape[0], (i, got[i].shape)
        for f in range(s.shape[0]):
            _assert_same(got[i][f], next(want), (i, f))


def test_rotate_float_sequences():
    _check_per_frame(lambda fn, types, x: fn.rotate(x, angle=33.0, dtype=types.FLOAT), "FHWC", "HWC")


def test_warp_affine_float_sequences():
    m = [1.1, 0.2, -3.0, -0.15, 0.9, 2.5]
    _check_per_frame(lambda fn, types, x: fn.warp_affine(x, matrix=m, dtype=types.FLOAT), "FHWC", "HWC")


@pytest.mark.parametrize("seq_layout,frame_layout", [("FHWC", "HWC"), ("FCHW", "CHW")])
def test_resize_float_sequences(seq_layout, frame_layout):
    _check_per_frame(lambda fn, types, x: fn.resize(x, resize_shorter=24, dtype=types.FLOAT), seq_layout, frame_layout,
                     channel_first=seq_layout == "FCHW")


def test_crop_mirror_normalize_padded_fchw_float16_sequences():
    def cmn(layout):
        return lambda fn, types, x: fn.crop_mirror_normalize(x, output_layout=layout, pad_output=True, dtype=types.FLOAT16,
                                                             mean=[10.0, 20.0, 30.0], std=[2.0, 3.0, 4.0])
    _check_per_frame(cmn("FCHW"), "FHWC", "HWC", frame_op=cmn("CHW"))


def test_random_resized_crop_float_sequences():
    """One window per sample: the reference for frame f is a pipeline with the same seed whose batch position i holds frame f of
    sample i (the last frame of a shorter sample), so that each position draws the window of its sample."""
    def op(fn, types, x):
        return fn.random_resized_crop(x, size=[20, 24], seed=4321, dtype=types.FLOAT)
    seqs = _sequences()
    keep = []
    got = _run(seqs, "FHWC", op, keep)
    for f in range(max(s.shape[0] for s in seqs)):
        want = _run([s[min(f, s.shape[0] - 1)] for s in seqs], "HWC", op, keep)
        for i, s in enumerate(seqs):
            assert got[i].shape[0] == s.shape[0], (i, got[i].shape)
            if f < s.shape[0]:
                _assert_same(got[i][f], want[i], (i, f))
