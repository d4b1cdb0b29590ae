"""decoders.audio without a GPU: the host-compiled planner and kernel bodies (tools/emul/audio_decode_emul.cc) against the samples the
encoder of tests/audio_streams.py was given, in FLOAT / INT16 / INT32 and with the downmix; every refusal code; every corruption class;
mutated streams under ASan + UBSan; false syncs; and the corpus itself (coverage from its parsed headers, WAV against scipy)."""
import ctypes as C
import os
import shutil
import struct
import subprocess

import numpy as np
import pytest

import audio_streams as aus

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tools", "emul", "audio_decode_emul.cc")
FLOAT, INT16, INT32 = 9, 5, 6


def _build(tmp, flags):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp / "libaudioemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-shared", "-fPIC", "-Wall", "-ffp-contract=off", "-I/usr/local/cuda/include"] + flags + [EMUL, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    lib = C.CDLL(_build(tmp_path_factory.mktemp("audio_emul"), ["-O2"]))
    lib.emul_audio_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def emul_decode(lib, s, downmix=False, dtype=FLOAT):
    """(status, output): the planner's status, or 0 / -1 (the sample's status) with the output"""
    info = (C.c_int64 * 5)()
    rc = lib.emul_audio_decode(s, len(s), int(downmix), dtype, None, info)
    if rc:
        return rc, None
    T, ch = info[4], info[2]
    out = np.zeros((T, 1 if downmix else ch), {FLOAT: np.float32, INT16: np.int16, INT32: np.int32}[dtype])
    return lib.emul_audio_decode(s, len(s), int(downmix), dtype, out.ctypes.data if out.size else 1, info), out


def expected(x, bits, dtype=FLOAT, downmix=False):
    """libsndfile's reads as restated in DESIGN section 2: x / 2^(b-1) (32-bit: RN(float(x)) * 2^-31), float WAV copied; integer reads
    shifted to 16 / 32 bits; the downmix as float32 products and sums rounded one by one"""
    if x.dtype == np.float32:
        f = x
    elif dtype == FLOAT:
        f = x.astype(np.float32) * np.float32(2.0 ** -(bits - 1))
    else:
        ob = 16 if dtype == INT16 else 32
        y = x.astype(np.int64) << (ob - bits) if ob >= bits else x.astype(np.int64) >> (bits - ob)
        return y.astype(np.int16 if dtype == INT16 else np.int32)
    if not downmix:
        return f
    w = np.float32(1) / np.float32(f.shape[1])
    s = f[:, 0] * w
    for c in range(1, f.shape[1]):
        s = s + f[:, c] * w
    return s[:, None]


def test_emulated_decode_of_the_corpus(emul):
    for name, s, x, bits in aus.corpus():
        for dtype in (FLOAT, INT16, INT32):
            if x.dtype == np.float32 and dtype != FLOAT:
                assert emul_decode(emul, s, dtype=dtype)[0] == aus.UNSUPPORTED, name
                continue
            st, out = emul_decode(emul, s, dtype=dtype)
            want = expected(x, bits, dtype)
            assert st == 0 and out.dtype == want.dtype and np.array_equal(out.view(np.uint8), want.view(np.uint8)), (name, dtype, st)
        st, out = emul_decode(emul, s, downmix=True)
        want = expected(x, bits, FLOAT, downmix=True)
        assert st == 0 and np.array_equal(out.view(np.uint32), want.view(np.uint32)), (name, "downmix")


def test_emulated_refusals(emul):
    for name, s, code, why in aus.refused():
        assert emul_decode(emul, s)[0] == code, (name, why)


def test_emulated_corruption_sets_the_status(emul):
    for name, s in aus.corrupt():
        assert emul_decode(emul, s)[0] == -1, name


def test_wav_data_chunk_longer_than_the_file_decodes_the_whole_frames_present(emul):
    x = aus.signal(300, 2, 16, np.random.default_rng(3))
    s = aus.wav_pcm(x, 16, 8000)
    s = s[:40] + struct.pack("<I", 10 ** 6) + s[44:-3]            # claims 1 MB, the last frame is cut short
    st, out = emul_decode(emul, s, dtype=INT16)
    assert st == 0 and np.array_equal(out, x[:299].astype(np.int16))


def _salted_stream(rng):
    """frames whose verbatim data holds whole valid frames of the same stream (header, CRC-8, CRC-16 included): false syncs that parse"""
    x = aus.signal(4096, 1, 16, rng)
    inner = []
    aus.flac(x[:256], 16, 16000, [256], spec=lambda k, c, b: {"kind": "fixed", "order": 1}, frames_out=inner)
    fake = np.frombuffer(inner[0] + bytes(len(inner[0]) & 1), ">i2").astype(np.int64)
    y = x.copy()
    for k in range(4):                                            # each frame of 1024 carries the fake frame in its verbatim samples
        y[k * 1024 + 1:k * 1024 + 1 + len(fake), 0] = fake
    s = aus.flac(y, 16, 16000, [1024] * 4, spec=lambda k, c, b: {"kind": "verbatim"})
    return s, y


def test_false_syncs_inside_frames_do_not_reach_the_output(emul):
    s, y = _salted_stream(np.random.default_rng(9))
    st, out = emul_decode(emul, s, dtype=INT16)
    assert st == 0 and np.array_equal(out[:, 0], y[:, 0].astype(np.int16))


def _flooded_stream(n_false, rng):
    """four verbatim frames of 1024 samples whose data holds n_false valid frame HEADERS (sync, codes, CRC-8) of the same stream"""
    x = aus.signal(4096, 1, 16, rng)
    inner = []
    aus.flac(x[:256], 16, 16000, [256], spec=lambda k, c, b: {"kind": "verbatim"}, frames_out=inner)
    hdr = np.frombuffer(inner[0][:6], ">i2").astype(np.int64)         # 6 header bytes = 3 samples
    y = x.copy()
    for j in range(n_false):
        k, o = divmod(j, 1024 // 4 - 1)
        y[k * 1024 + 1 + 4 * o:k * 1024 + 4 + 4 * o, 0] = hdr
    return aus.flac(y, 16, 16000, [1024] * 4, spec=lambda k, c, b: {"kind": "verbatim"}), y


def test_candidate_cap(emul):
    """more header candidates than the stream's cap (2 x (ceil(T / min_block) + 1) + 64 = 74 here) fail the sample cleanly; fewer
    still decode exactly"""
    rng = np.random.default_rng(21)
    s, y = _flooded_stream(40, rng)
    st, out = emul_decode(emul, s, dtype=INT16)
    assert st == 0 and np.array_equal(out[:, 0], y[:, 0].astype(np.int16))
    s, y = _flooded_stream(200, rng)
    assert emul_decode(emul, s, dtype=INT16)[0] == -1


def test_mutated_streams_under_asan_ubsan(tmp_path):
    """1 500 mutated corpus streams through the host-compiled decode with AddressSanitizer and UndefinedBehaviorSanitizer: no report"""
    out = _build(tmp_path, ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-fno-omit-frame-pointer"])
    rng = np.random.default_rng(77)
    bases = [s for _, s, _, _ in aus.corpus() if len(s) < 40000] + [s for _, s in aus.corrupt()] + [_salted_stream(rng)[0]]
    cases = []
    for i in range(1500):
        b = bytearray(bases[i % len(bases)])
        kind = i % 4
        if kind == 0:
            for _ in range(1 + rng.integers(8)):
                b[rng.integers(len(b))] ^= 1 << int(rng.integers(8))
        elif kind == 1:
            b = b[:rng.integers(1, len(b))]
        elif kind == 2:
            p = rng.integers(len(b))
            b[p:p + 8] = rng.integers(0, 256, 8).astype(np.uint8).tobytes()
        else:
            p = rng.integers(len(b))
            b[p:p] = bytes([0xFF, 0xF8]) + rng.integers(0, 256, 14).astype(np.uint8).tobytes()
        cases.append(bytes(b))
    data = tmp_path / "cases.bin"
    with open(data, "wb") as f:
        for c in cases:
            f.write(struct.pack("<I", len(c)) + c)
    drv = tmp_path / "drive.py"
    drv.write_text(
        "import ctypes as C, struct, sys\n"
        f"lib = C.CDLL({out!r})\n"
        "lib.emul_audio_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_void_p]\n"
        f"d = open({str(data)!r}, 'rb').read(); p = 0; n = 0\n"
        "info = (C.c_int64 * 5)()\n"
        "while p < len(d):\n"
        "    L = struct.unpack_from('<I', d, p)[0]; s = d[p + 4:p + 4 + L]; p += 4 + L\n"
        "    for dm in (0, 1):\n"
        "        if lib.emul_audio_decode(s, len(s), dm, 9, None, info) == 0 and info[4] * info[2] < 1 << 22:\n"
        "            buf = C.create_string_buffer(max(4, 4 * info[4] * info[2]))\n"
        "            lib.emul_audio_decode(s, len(s), dm, 9, buf, info)\n"
        "    n += 1\n"
        "print('ran', n)\n")
    asan = subprocess.run(["g++", "-print-file-name=libasan.so"], capture_output=True, text=True).stdout.strip()
    env = dict(os.environ, LD_PRELOAD=asan, ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="halt_on_error=1:print_stacktrace=1")
    r = subprocess.run(["python3", str(drv)], capture_output=True, text=True, env=env, timeout=1200)
    assert r.returncode == 0 and "ran 1500" in r.stdout, (r.stdout[-2000:], r.stderr[-4000:])
    assert "runtime error" not in r.stderr and "AddressSanitizer" not in r.stderr, r.stderr[-4000:]


# ---- the corpus itself
def _flac_audio_region(s):
    """(metadata block types, offset of the first frame) read back from the stream's container"""
    p = 0
    if s[:3] == b"ID3":
        p = 10 + ((s[6] << 21) | (s[7] << 14) | (s[8] << 7) | s[9])
    p += 4
    blocks = []
    while True:
        t, last, L = s[p] & 127, s[p] & 128, int.from_bytes(s[p + 1:p + 4], "big")
        blocks.append(t)
        p += 4 + L
        if last:
            break
    return blocks, p


def _frame_header_len(s, i):
    """length of the frame header at i (through its CRC-8 byte) read from its codes, or 0 when it is not one"""
    if not (s[i] == 0xFF and (s[i + 1] & 0xFE) == 0xF8):
        return 0
    b = s[i + 4]
    n = 1 if b < 0x80 else 8 - (b ^ 0xFF).bit_length()              # UTF-8-like: the leading one bits count the bytes
    p = i + 4 + n
    bs, rc = s[i + 2] >> 4, s[i + 2] & 15
    p += {6: 1, 7: 2}.get(bs, 0) + {12: 1, 13: 2, 14: 2}.get(rc, 0)
    return p + 1 - i if p < len(s) and aus.crc8(s[i:p]) == s[p] else 0


def test_corpus_covers_what_it_claims():
    """block-size, sample-rate, channel-assignment and bits-per-sample codes and blocking strategies, read from every frame header
    whose CRC-8 holds (the encoder's frames follow each other; a false sync in the data would need a matching CRC-8 too)"""
    seen = {"bs": set(), "rate": set(), "assign": set(), "bits_code": set(), "bits": set(), "variable": set(), "meta": set(), "id3": False}
    for name, s, x, bits in aus.corpus():
        if not name.startswith("flac"):
            continue
        seen["bits"].add(bits)
        seen["id3"] |= s[:3] == b"ID3"
        meta, p = _flac_audio_region(s)
        seen["meta"].update(meta)
        for i in range(p, len(s) - 8):
            if _frame_header_len(s, i):
                seen["variable"].add(s[i + 1] & 1)
                seen["bs"].add(s[i + 2] >> 4)
                seen["rate"].add(s[i + 2] & 15)
                seen["assign"].add(s[i + 3] >> 4)
                seen["bits_code"].add((s[i + 3] >> 1) & 7)
    assert seen["bs"] >= set(range(1, 16)) and seen["rate"] >= set(range(0, 15)) and seen["assign"] >= {0, 1, 2, 5, 7, 8, 9, 10}
    assert seen["bits_code"] >= {0, 1, 4, 6} and seen["bits"] == {8, 16, 24} and seen["variable"] == {0, 1}
    assert seen["id3"] and {0, 1, 4} <= seen["meta"]


def test_encoder_coverage_of_subframes_and_partitions(monkeypatch):
    """every subframe type, LPC order 1..32 at several precisions and shifts, both residual methods, escapes and partition orders 0..8"""
    got = {"kind": set(), "fixed": set(), "lpc": set(), "prec": set(), "method": set(), "porder": set(), "escape": False, "wasted": False}
    orig = aus.subframe

    def spy(bw, x, sb, spec, rng):
        got["kind"].add(spec["kind"])
        if spec["kind"] == "fixed":
            got["fixed"].add(spec["order"])
        if spec["kind"] == "lpc":
            got["lpc"].add(spec["order"])
            got["prec"].add(spec.get("precision", 12))
        if spec["kind"] in ("fixed", "lpc"):
            got["method"].add(spec.get("method", 0))
            got["porder"].add(spec.get("porder", 0))
            got["escape"] |= bool(spec.get("escape"))
        got["wasted"] |= bool(spec.get("wasted"))
        return orig(bw, x, sb, spec, rng)
    monkeypatch.setattr(aus, "subframe", spy)
    aus.corpus()
    assert got["lpc"] == set(range(1, 33))
    assert got["kind"] == {"constant", "verbatim", "fixed", "lpc"} and got["fixed"] == {0, 1, 2, 3, 4}
    assert got["method"] == {0, 1} and got["porder"] >= set(range(0, 9)) and got["escape"] and got["wasted"]
    assert len(got["prec"]) >= 4


def test_wav_streams_read_back_by_scipy():
    wavfile = pytest.importorskip("scipy.io.wavfile")
    import io
    for name, s, x, bits in aus.corpus():
        if not name.startswith("wav") or bits == 24:
            continue
        rate, y = wavfile.read(io.BytesIO(s))
        y = y.reshape(len(y), -1)
        want = (x + 128).astype(np.uint8) if bits == 8 else x
        assert np.array_equal(y.astype(np.float64), np.asarray(want, np.float64)), name
