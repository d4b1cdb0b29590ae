"""-m gpu: the baseline entropy stage of jpeg.cu (U1 - U3 un-stuffing, H1 speculative decode, H2a chain walk, H2b block-count scan,
H3 coefficient write, D1 DC prediction) on streams built to land on its own boundaries (tests/jpeg_entropy_streams.py), at every
subsequence size.  Every sample of every batch is checked three ways: its quantised coefficients in MCU order equal the oracle's, its
pixels equal cv2.imdecode, and its status is 0.  Every case asserts through the model of the synchronisation that it reaches the edge it
is written for, so that a case that drifts away fails instead of testing something easier."""
import functools

import numpy as np
import pytest

import jpeg_entropy_streams as E

pytestmark = pytest.mark.gpu


@functools.lru_cache(maxsize=None)
def _oracle(s):
    import cv2
    img = cv2.imdecode(np.frombuffer(s, np.uint8), cv2.IMREAD_COLOR)
    assert img is not None
    coefs = E.mcu_order(s).reshape(-1) if isinstance(E.table_key(s), tuple) else None     # baseline samples: the oracle's blocks
    return coefs, np.ascontiguousarray(img[..., ::-1])


def _decode_and_check(streams, sub_bytes, monkeypatch, what):
    import gpu_helpers as g
    if sub_bytes is None:
        monkeypatch.delenv("DALIB200_JPEG_SUBSEQ_BYTES", raising=False)
    else:
        monkeypatch.setenv("DALIB200_JPEG_SUBSEQ_BYTES", str(sub_bytes))
    outs, status, plan = g.jpeg_decode(streams, want_coefs=True)
    assert status == [0] * len(streams), f"{what} at {sub_bytes} B: status {status}"
    for i, s in enumerate(streams):
        coefs, px = _oracle(s)
        if coefs is not None:
            got = g.jpeg_coefs(plan, i, coefs.size)
            bad = np.nonzero((got != coefs).reshape(-1, 64).any(1))[0]
            assert bad.size == 0, f"{what} at {sub_bytes} B, sample {i}: {bad.size} blocks differ, the first {bad[:8].tolist()}"
        assert np.array_equal(outs[i], px), f"{what} at {sub_bytes} B, sample {i}: pixels differ from cv2.imdecode"


def _first_subseq(us, sub_bytes):
    """image-local first subsequence of every unit: the plan counts ceil(raw length / subsequence) per unit"""
    out, k = [], 0
    for u in us:
        out.append(k)
        k += -(-len(u.raw) // sub_bytes)
    return out


@pytest.mark.parametrize("sub_bytes", E.SUB_BYTES)
def test_unstuffing_chunks_and_units(sub_bytes, monkeypatch):
    """U1 - U3: 0xFF 0x00 at raw bytes 4093 .. 4098 and 8191 of a unit, pairs on both sides of the chunk boundary, units of 4095 /
    4096 / 4097 / 8191 / 8193 bytes, a unit that is mostly stuffing, units of 1 .. 8 bytes at every staged offset mod 16, and 0xFF fill
    bytes before every RSTn and the EOI"""
    stuffed, notes = E.stuffing_stream()
    us = E.units(stuffed)
    for u, (what, where) in notes.items():
        raw = us[u].raw
        if what == "ff":
            assert raw[where:where + 2] == b"\xff\x00", (u, where)
            assert min(where % E.CHUNK_BYTES, E.CHUNK_BYTES - where % E.CHUNK_BYTES) <= 3      # within 3 bytes of a chunk boundary
        elif what == "ff2":
            assert raw[where:where + 5] == b"\xff\x00" + raw[where + 2:where + 3] + b"\xff\x00" and where < E.CHUNK_BYTES <= where + 3
        elif what == "len":
            assert len(raw) == where and len(us[u].clean) == where
        else:
            assert 2 * raw.count(b"\xff\x00") > len(raw) // 2
    assert any(len(u.clean) % 16 == 0 and len(u.clean) >= E.CHUNK_BYTES for u in us)
    small, sizes = E.small_units_stream()
    filled, _ = E.small_units_stream(fill=2)
    su = E.units(small)
    assert [len(u.raw) for u in su] == sizes and {u.raw_off % 16 for u in su} == set(range(16))
    assert all(u.raw.endswith(b"\xff\xff") for u in E.units(filled)[:-1])
    _decode_and_check([stuffed, small, filled], sub_bytes, monkeypatch, "un-stuffing")


@pytest.mark.parametrize("sub_bytes", E.SUB_BYTES)
def test_subsequence_counts_around_sync_blocks(sub_bytes, monkeypatch):
    """H1: one-unit images of 255 / 256 / 257 / 511 / 512 / 513 subsequences, in one batch"""
    counts = (E.SYNC_THREADS - 1, E.SYNC_THREADS, E.SYNC_THREADS + 1, 2 * E.SYNC_THREADS - 1, 2 * E.SYNC_THREADS, 2 * E.SYNC_THREADS + 1)
    streams = [E.subseq_stream(n, sub_bytes) for n in counts]
    assert [E.units(s)[0].nsub(8 * sub_bytes) for s in streams] == list(counts)
    _decode_and_check(streams, sub_bytes, monkeypatch, "subsequence counts")


@pytest.mark.parametrize("sub_bytes", E.SUB_BYTES)
def test_unit_and_widest_block_at_the_sync_block_edge(sub_bytes, monkeypatch):
    """H1 / H3: a restart unit that begins in the last column of sync block 0, and in it the widest block (16-bit codes, the largest
    magnitudes) starting 8 bits before the end of that column: H1's last thread decodes its first symbols from the look-ahead column
    staged behind the sync block, H3 completes it 208 bytes into sync block 1"""
    s = E.sync_edge_stream(sub_bytes)
    us = E.units(s)
    first = _first_subseq(us, sub_bytes)
    assert first[5] == E.SYNC_THREADS - 1
    P, Cs, Zs, _ = us[5].walk()
    starts = P[Zs == 0]
    k = int(np.nonzero(starts < 8 * sub_bytes)[0][-1])              # the last block that starts in the unit's first column
    assert starts[k + 1] - starts[k] == 1665 and starts[k + 1] > 8 * sub_bytes + 8 * 200
    _decode_and_check([s], sub_bytes, monkeypatch, "sync-block edge")


def _chain_streams(S):
    """all-zero segments whose true chain stops after exactly L subsequences: L = 1, 2, 3, 33, 301, kMaxChainLen and kMaxChainLen + 2
    (odd MCU lengths above 4096 bits, so no speculative decoder synchronises before), and the 4:2:0 MCU of 4543 bits"""
    out = []
    for L, P in ((1, 256), (2, 2 * S), (3, 768), (33, 33 * 64), (301, 301 * 4), (E.MAX_CHAIN_LEN, E.MAX_CHAIN_LEN),
                 (E.MAX_CHAIN_LEN + 2, E.MAX_CHAIN_LEN + 2), (4543, 4543)):
        assert E.zero_chain(P, S) == L, (P, S)
        nmcu = -(-(L + 40) * 1024 // P) if L > 400 else -(-(L + 40) * S // P) + 16
        out.append((L, E.zero_stream(P, nmcu)))
    return out


@functools.lru_cache(maxsize=None)
def _chains(S):
    return _chain_streams(S)


def _lead(kind):
    import cv2
    import gpu_helpers as gh
    img = gh.synth_image(64, 96, 5)
    if kind == "jpeg":
        return cv2.imencode(".jpg", img)[1].tobytes()
    if kind == "prog":
        return cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    return cv2.imencode(".png", img)[1].tobytes()


@pytest.mark.parametrize("lead", [None, "jpeg", "prog", "png"])
@pytest.mark.parametrize("sub_bytes", E.SUB_BYTES)
def test_chain_lengths(sub_bytes, lead, monkeypatch):
    """H2a: true chains of exactly 1, 2, 3, 33, 301, 4095 and more than 4095 subsequences (the walk's three launches, chains across
    sync blocks, and a chain that outgrows the 12-bit priority).  Every crafted stream has tables of its own.  lead None: each stream is
    decoded alone, so that it is sample 0 and every walk reads the tables from shared memory (the path natural batches take); lead
    "jpeg" / "prog" / "png": one batch behind a baseline JPEG of other tables, a progressive JPEG or a PNG, so that the walks read the
    tables from global memory (behind the PNG, whose table index is 0, the first stream keeps the shared path)"""
    if lead in ("prog", "png") and sub_bytes != 32:
        pytest.skip("the progressive and PNG leads run at 32 B")
    S = 8 * sub_bytes
    assert (S >> 5) + 4 <= E.TAIL_COL_WORDS                       # the shared path's private column holds the subsequence
    cases = _chains(S)
    for L, s in cases:
        u = E.units(s)[0]
        assert u.nsub(S) > L + 1, (L, u.nsub(S))
        if L <= 33:
            assert u.chain(S) == L                                # the generic model agrees with the closed form
    assert max(L for L, _ in cases) > E.MAX_CHAIN_LEN
    if lead is None:
        for L, s in cases:
            assert E.walk_paths([s]) == ["shared"]
            _decode_and_check([s], sub_bytes, monkeypatch, f"chain of {L} (shared tables)")
        return
    streams = [_lead(lead)] + [s for _, s in cases]
    want = {"jpeg": ["shared"] + ["global"] * len(cases), "prog": [None] + ["global"] * len(cases),
            "png": [None, "shared"] + ["global"] * (len(cases) - 1)}[lead]
    assert E.walk_paths(streams) == want
    _decode_and_check(streams, sub_bytes, monkeypatch, f"chain lengths (lead {lead}, global tables)")


@pytest.mark.parametrize("sub_bytes", E.SUB_BYTES)
def test_blocks_across_write_blocks(sub_bytes, monkeypatch):
    """H2b / H3: the widest block starts in the last subsequence of write blocks 0 and 1 (image subsequences WRITE_THREADS - 1 and
    2 WRITE_THREADS - 1) and spans up to 8 subsequences, the ones behind its first holding no block start"""
    S = 8 * sub_bytes
    s = E.write_edge_stream(sub_bytes)
    u = E.units(s)[0]
    P, Cs, Zs, _ = u.walk()
    starts = P[:-1][Zs[:-1] == 0]
    for j in (E.WRITE_THREADS - 1, 2 * E.WRITE_THREADS - 1):
        i = int(np.nonzero((starts >= j * S) & (starts < (j + 1) * S))[0][-1])
        assert starts[i] == (j + 1) * S - 8 and starts[i + 1] - starts[i] == 1665
        last = int(starts[i + 1]) // S
        assert last - j == -(-(1665 - 8) // S) and not np.any((starts >= (j + 1) * S) & (starts < last * S))
    assert -(-(1665 - 8) // 256) + 1 == 8                         # at 32 B the block touches 8 subsequences
    _decode_and_check([s], sub_bytes, monkeypatch, "write-block edge")


@pytest.mark.parametrize("sub_bytes", E.SUB_BYTES)
def test_pad_bits_fill_and_trailing_bytes(sub_bytes, monkeypatch):
    """H2b / H3: pad bits of every length 1 - 7 that decode into extra symbols, 0xFF fill before RSTn and EOI, zeros and a second JPEG behind the EOI; the
    samples sit next to each other in one batch, so a coefficient that leaks into a neighbour is seen"""
    import cv2
    import gpu_helpers as gh
    base = E.subseq_stream(37, sub_bytes)
    assert base.endswith(b"\xff\xd9")
    second = cv2.imencode(".jpg", gh.synth_image(24, 40, 7))[1].tobytes()
    filled, _ = E.small_units_stream(fill=3)
    padded = E.pad_stream()
    pu = E.units(padded)
    assert [u.pad_bits() for u in pu[:7]] == list(range(1, 8)) and all(u.extra_symbols() > 0 for u in pu[:7])
    streams = [base, base + bytes(300), base[:-2] + b"\xff\xff\xff\xd9", base + second, filled, padded]
    for s in streams[1:]:
        assert sum(u.extra_symbols() for u in E.units(s)) > 0      # symbols decoded behind the last block of some unit
    _decode_and_check(streams, sub_bytes, monkeypatch, "pad / fill / trailing bytes")


def _tiny_blocks_stream(rst=0):
    """D1 / H2b: gray 2048 x 1040 (33280 blocks, one component).  First half: 2-bit blocks (DC category 0 '0', EOB '0') with a DC
    difference of -2047 / +2047 in every 700th block (runs long enough to fill a 128-byte subsequence with 512 blocks); second half:
    +2047 in every other block, so that the DC sum wraps int16 many times; rst: a 1-MCU restart interval on a smaller frame instead
    (more than 1024 segments)"""
    tabs = {0x00: [(1, 0), (2, 11)], 0x10: [(1, 0x00)]}
    if rst:
        st = E.Stream(200, 352, E.GRAY, tabs, E.SEL0, rst=1)
    else:
        st = E.Stream(1040, 2048, E.GRAY, tabs, E.SEL0)
    for k in range(st.nblocks):
        if k < st.nblocks // 2 and k % 700 == 350:
            st.add([(11, "00000000000" if k % 1400 == 350 else "11111111111"), (0x00, "")])
        elif k >= st.nblocks // 2 and k % 2:
            st.add([(11, "11111111111"), (0x00, "")])
        else:
            st.add([(0, ""), (0x00, "")])
    return st.finish()


@pytest.mark.parametrize("sub_bytes", E.SUB_BYTES)
def test_tiny_blocks_and_dc_prediction(sub_bytes, monkeypatch):
    """H2b / H3 / D1: subsequences full of 2-bit blocks, a component of more than 32 x 1024 blocks whose DC sum wraps int16, and a
    1-MCU restart interval with more than 1024 segments"""
    big, segs = _tiny_blocks_stream(), _tiny_blocks_stream(rst=1)
    u = E.units(big)[0]
    assert u.nblocks > 32 * 1024
    assert int(u.exits(8 * sub_bytes)[3].max()) == 8 * sub_bytes // 2
    dc = E.coefficients(big)[:, 0].astype(np.int64)
    half = u.nblocks // 2
    assert np.count_nonzero(np.diff(dc[:half])) >= half // 700 and np.any(np.diff(dc[half:]) < 0)    # DC moves in both halves; it wraps
    assert len(E.units(segs)) > 1024
    _decode_and_check([big, segs], sub_bytes, monkeypatch, "tiny blocks / DC")


def test_planner_picks_128_bytes(monkeypatch):
    """a batch just large enough that the planner picks 128-byte subsequences on its own (its rule and threshold read from jpeg.cu),
    with long chains in it"""
    stuffed, _ = E.stuffing_stream()
    long_chain = _chains(1024)[-2][1]
    streams = [long_chain] * 8 + [stuffed] * 8
    while E.planner_sub_bytes(map(len, streams)) < 128:
        streams += [stuffed, long_chain]
    assert E.planner_sub_bytes(map(len, streams)) == 128 and E.planner_sub_bytes(map(len, streams[:-2])) < 128
    _decode_and_check(streams, None, monkeypatch, "planner's size")
