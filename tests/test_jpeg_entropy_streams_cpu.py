"""The crafted entropy-stage streams of tests/jpeg_entropy_streams.py without a GPU: cv2 and the oracle accept every one, the model's
sequential decode equals the oracle's coefficients, and every placement a GPU case states holds."""
import numpy as np
import pytest

import jpeg_entropy_streams as E


def _accepts(s):
    import cv2
    from oracle import pyoracle as po
    img = cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR)
    assert img is not None
    assert np.array_equal(po.jpeg_decode(s), img[..., ::-1])
    assert np.array_equal(E.coefficients(s), E.mcu_order(s))


def test_constants_are_read_from_the_sources():
    assert (E.SYNC_THREADS, E.WRITE_THREADS, E.MAX_CHAIN_LEN, E.CHUNK_BYTES) == (256, 384, 4095, 4096) and E.CLEAN_PAD >= 16


def test_stuffing_stream():
    s, notes = E.stuffing_stream()
    _accepts(s)
    us = E.units(s)
    assert len(us) == 15
    for u in range(6):
        assert notes[u] == ("ff", 4093 + u) and us[u].raw[4093 + u:4095 + u] == b"\xff\x00"
    assert us[7].raw[8191:8193] == b"\xff\x00"
    assert [len(us[u].raw) for u in range(8, 13)] == [4095, 4096, 4097, 8191, 8193]
    assert us[6].raw[4093:4095] == b"\xff\x00" and us[6].raw[4096:4098] == b"\xff\x00"
    assert 2 * us[13].raw.count(b"\xff\x00") > len(us[13].raw) // 2


@pytest.mark.parametrize("fill", [0, 1, 3])
def test_small_units_and_fill_bytes(fill):
    s, sizes = E.small_units_stream(fill=fill)
    _accepts(s)
    us = E.units(s)
    assert [len(u.raw) - fill for u in us[:-1]] == sizes[:-1]
    if fill == 0:
        assert {u.raw_off % 16 for u in us} == set(range(16))


@pytest.mark.parametrize("sub_bytes", E.SUB_BYTES)
def test_subsequence_and_sync_edge_streams(sub_bytes):
    for n in (255, 513):
        s = E.subseq_stream(n, sub_bytes)
        _accepts(s)
        u = E.units(s)[0]
        assert u.nsub(8 * sub_bytes) == n and len(u.clean) == n * sub_bytes
    s = E.sync_edge_stream(sub_bytes)
    _accepts(s)
    us = E.units(s)
    assert sum(-(-len(u.raw) // sub_bytes) for u in us[:5]) == E.SYNC_THREADS - 1


@pytest.mark.parametrize("P", [256, 512, 768, 33 * 64, 301 * 4, 4097, 4543])
def test_zero_streams(P):
    sampling, _, _ = E.zero_layout(P)
    s = E.zero_stream(P, 24)
    _accepts(s)
    u = E.units(s)[0]
    P_bits, Cs, Zs, _ = u.walk()
    bpm = sum(hs * vs for hs, vs in sampling)
    assert int(P_bits[Zs == 0][bpm]) == P                          # the MCU is exactly P bits long


@pytest.mark.parametrize("P,S", [(256, 256), (512, 256), (768, 512), (33 * 64, 1024), (33 * 64, 256)])
def test_model_chain_matches_closed_form(P, S):
    """the generic model (speculative decoders run until they meet the true one) and the closed form of an all-zero segment agree"""
    L = E.zero_chain(P, S)
    s = E.zero_stream(P, -(-(L + 8) * S // P) + 4)
    u = E.units(s)[0]
    assert u.chain(S) == L
    for o in range(1, min(L, 5)):
        assert u.sync(o, S, bound=L + 2) is None or u.sync(o, S) >= L


def test_model_speculative_exit_of_a_natural_stream():
    """on a natural stream every speculative decoder synchronises within a few subsequences, and the one started at subsequence 0 is
    the true decoder"""
    import cv2
    import gpu_helpers as g
    s = cv2.imencode(".jpg", g.synth_image(96, 128, 3), [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes()
    _accepts(s)
    u = E.units(s)[0]
    pos, c, z, nb = u.exits(256)
    assert u.spec_exit(0, 256) == (int(pos[0]), int(c[0]), int(z[0]))
    assert 1 <= u.chain(256) <= 8
    assert int(nb.sum()) >= u.nblocks


def test_pad_and_write_edge_streams():
    s = E.pad_stream()
    _accepts(s)
    assert [u.pad_bits() for u in E.units(s)] == [1, 2, 3, 4, 5, 6, 7, 0]
    for sub_bytes in E.SUB_BYTES:
        s = E.write_edge_stream(sub_bytes)
        _accepts(s)
        starts = E.units(s)[0].walk()[0][:-1][E.units(s)[0].walk()[2][:-1] == 0]
        for j in (E.WRITE_THREADS - 1, 2 * E.WRITE_THREADS - 1):
            assert (j + 1) * 8 * sub_bytes - 8 in starts


def test_walk_paths_and_planner_rule():
    """which tables the chain walk reads, as the plan numbers its table sets; the subsequence size the plan picks"""
    import cv2
    import gpu_helpers as g
    img = g.synth_image(32, 48, 1)
    jpg, prog = cv2.imencode(".jpg", img)[1].tobytes(), cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    png = cv2.imencode(".png", img)[1].tobytes()
    a, b = E.zero_stream(256, 4), E.zero_stream(768, 4)
    assert E.walk_paths([a, b, a]) == ["shared", "global", "shared"]
    assert E.walk_paths([jpg, a, jpg]) == ["shared", "global", "shared"]
    assert E.walk_paths([prog, a]) == [None, "global"] and E.walk_paths([png, a, b]) == [None, "shared", "global"]
    assert E.planner_sub_bytes([100]) == 32 and E.planner_sub_bytes([1 << 30]) == 1 << (E.MAX_LOG2_SUB - 3)
