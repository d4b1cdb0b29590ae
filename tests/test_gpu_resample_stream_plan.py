"""-m gpu: one Resample plan set up again and again with different batches.  The streaming kernel's walk records live in the
plan's table arena, built per distinct vertical axis at set-up and uploaded only when the arena changes; a stale or mis-indexed
record shows up as a wrong output row.  Every output is compared with the oracle bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import pyoracle as po  # noqa: E402


def bits(a):
    return np.ascontiguousarray(a).view(np.uint8)


def test_resample_stream_records_across_setups():
    import gpu_helpers as g
    from dali_b200 import capi
    rng = np.random.default_rng(90)
    plan = capi.Plan("Resample", 6)
    c2 = (po.F_LINEAR, 1, 0.0)
    gauss = (po.F_GAUSSIAN, 1, 0.0)
    mag = (po.F_LINEAR, 0, 0.0)

    def u8(*shape):
        return rng.integers(0, 256, shape).astype(np.uint8)

    setups = [
        # C2: 1080p -> 224 x 224, triangular antialias, u8
        ([u8(1080, 1920, 3) for _ in range(3)], [(224, 224)] * 3, c2, np.uint8, [1, 1, 1]),
        # another output size and filter, f32 out, a 1-channel sample next to 3-channel ones
        ([u8(720, 1280, 3), u8(700, 960, 1), u8(720, 1280, 3)], [(180, 250), (97, 333), (180, 250)], gauss, np.float32, [1, 1, 1]),
        # back to C2, twice (the second set-up leaves the uploaded arena as it is)
        ([u8(1080, 1920, 3) for _ in range(2)], [(224, 224)] * 2, c2, np.uint8, [1, 1]),
        ([u8(1080, 1920, 3) for _ in range(2)], [(224, 224)] * 2, c2, np.uint8, [1, 1]),
        # streamed and non-streamed samples in one batch: rows not 16-byte aligned, an upscale, two streamed down-scales
        ([u8(1080, 1921, 3), u8(1080, 1920, 3), u8(60, 80, 3), u8(720, 1280, 3)], [(224, 224), (224, 224), (150, 170), (180, 250)], c2,
         np.uint8, [0, 1, 0, 1]),
    ]
    for k, (imgs, hws, fm, odt, want_paths) in enumerate(setups):
        got, paths = g.resample(imgs, hws, fm, mag, odt, plan=plan, want_path=True)
        assert paths == want_paths, (k, paths)
        for i, (img, hw, o) in enumerate(zip(imgs, hws, got)):
            want = po.resample(img, hw, fm, mag, odt)
            assert np.array_equal(bits(o), bits(want)), (k, i, img.shape, hw, int((o != want).sum()))
