"""-m gpu: the phases of the coefficient write pass (H3 in jpeg.cu) at the subsequence boundaries where one thread hands over to the
next.  A thread skips the tail of the block open at its entry, writes the blocks that start in its subsequence and finishes the last
one behind it; the DC difference of a block travels through the block buffer to the DC array.  The streams are cv2-encoded 4:2:0
images without restarts and with restart intervals of 1 and 2 MCUs (several units per image).  The sequential model of
tests/jpeg_entropy_streams.py finds, at every subsequence size, boundaries that fall
  * exactly at the start of a block (the thread has nothing to skip),
  * inside or right behind a DC symbol (the thread enters at zig-zag position 1),
  * inside a pair step (two AC symbols of one lookup): at its second symbol, or inside its second symbol,
  * inside the last block of a unit (the thread skips it and meets the pad bits and the unit's block limit),
and each kind must occur, so that a stream that drifts away from an edge fails instead of testing something easier.  The decoded
coefficients must equal the oracle's and the pixels cv2.imdecode's, as in the other JPEG tests."""
import functools

import numpy as np
import pytest

import jpeg_entropy_streams as E

pytestmark = pytest.mark.gpu

LUT_BITS = 11          # kAcLutBits: a pair is stored where the first symbol and the second code fit in the index
KINDS = ("block start", "dc", "pair second symbol", "inside pair", "last block of a unit")


@functools.lru_cache(maxsize=None)
def _streams():
    import cv2
    rng = np.random.default_rng(7)
    out = []
    for rst, (h, w), q in ((0, (200, 328), 90), (1, (136, 248), 90), (2, (152, 216), 95), (1, (96, 120), 75), (2, (120, 176), 85)):
        lo = rng.uniform(0, 255, (h // 16 + 2, w // 16 + 2, 3)).astype(np.float32)
        img = np.clip(cv2.resize(lo, (w, h), interpolation=cv2.INTER_CUBIC) + rng.normal(0, 6, (h, w, 3)), 0, 255).astype(np.uint8)
        ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_RST_INTERVAL, rst])
        assert ok
        out.append(enc.tobytes())
    return out


def _pair_starts(u, P, Cs, Zs):
    """symbols that start a pair step: an AC symbol that is not an EOB, leaves its block open, and whose bits and the next code fit
    in the LUT index (jpeg_huff_core.h BuildDeviceTable / pair_threshold)"""
    steps = [u._step(int(P[i]), int(Cs[i]), int(Zs[i])) for i in range(len(P) - 1)]
    pair = np.zeros(len(P), bool)
    for i in range(len(steps) - 1):
        bits, adv, _, _ = steps[i]
        if Zs[i] == 0 or adv == 64 or bits >= LUT_BITS or Zs[i] + adv >= 64 or P[i] + LUT_BITS > u.clean_bits:
            continue
        pair[i] = bits + steps[i + 1][3] <= LUT_BITS
    return pair


def _boundary_kinds(stream, S):
    """the kinds of boundary (KINDS) that the subsequences of S bits of the stream's units meet"""
    seen = set()
    for u in E.units(stream):
        P, Cs, Zs, _ = u.walk()
        pair = _pair_starts(u, P, Cs, Zs)
        starts = P[:-1][Zs[:-1] == 0]
        last = (int(starts[u.nblocks - 1]), int(starts[u.nblocks]) if len(starts) > u.nblocks else int(P[-1]))
        for k in range(1, u.nsub(S)):
            b = k * S
            j = int(np.searchsorted(P, b))                        # the first symbol the next thread decodes
            if P[j] == b and Zs[j] == 0:
                seen.add("block start")
            if j >= 1 and Zs[j] == 1 and Zs[j - 1] == 0:
                seen.add("dc")
            if j >= 1 and pair[j - 1]:
                seen.add("pair second symbol")
            if j >= 2 and pair[j - 2] and P[j - 1] < b:
                seen.add("inside pair")
            if last[0] < b < last[1]:
                seen.add("last block of a unit")
    return seen


def _oracle(s):
    import cv2
    img = cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR)
    assert img is not None
    return E.mcu_order(s).reshape(-1), np.ascontiguousarray(img[..., ::-1])


@pytest.mark.parametrize("sub_bytes", E.SUB_BYTES)
def test_write_phases_at_subsequence_boundaries(sub_bytes, monkeypatch):
    import gpu_helpers as g
    streams = _streams()
    seen = set().union(*(_boundary_kinds(s, 8 * sub_bytes) for s in streams))
    assert seen == set(KINDS), f"{sub_bytes} B subsequences miss {set(KINDS) - seen}"
    assert {len(E.units(s)) > 1 for s in streams} == {True, False}
    monkeypatch.setenv("DALIB200_JPEG_SUBSEQ_BYTES", str(sub_bytes))
    outs, status, plan = g.jpeg_decode(streams, want_coefs=True)
    assert status == [0] * len(streams)
    for i, s in enumerate(streams):
        coefs, px = _oracle(s)
        got = g.jpeg_coefs(plan, i, coefs.size)
        bad = np.nonzero((got != coefs).reshape(-1, 64).any(1))[0]
        assert bad.size == 0, f"{sub_bytes} B, sample {i}: {bad.size} blocks differ, the first {bad[:8].tolist()}"
        assert np.array_equal(outs[i], px), f"{sub_bytes} B, sample {i}: pixels differ from cv2.imdecode"
