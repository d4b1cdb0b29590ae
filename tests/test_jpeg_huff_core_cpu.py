"""The first-level Huffman tables of the JPEG entropy passes and the step rule that may decode two symbols per lookup
(dali_b200/csrc/jpeg_huff_core.h), run on the host through tools/emul/jpeg_huff_emul.cc:
  - every index of every AC table, at every zig-zag position 1..63 and with the limit inside, at and just behind the first symbol,
    against a plain one-symbol decoder written here: a step must give exactly the state (bits, zig-zag position) of one or of two
    single steps, take the pair whenever the table can hold it, the block stays open after the first symbol and the limit is at
    least 11 bits (the index width) away, and store every coefficient's value at its zig-zag index;
  - the standard tables (T.81 K.3), the optimised tables cv2 writes for the benchmark image, a table with codes of every length 1..16
    and a table whose codes are all longer than the index;
  - random bit streams and the benchmark image's entropy data, decoded span by span with pairs and one symbol per step: the state
    after every span and the coefficients must agree."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMUL = os.path.join(ROOT, "tools", "emul", "jpeg_huff_emul.cc")
sys.path.insert(0, ROOT)

AC_BITS = 11

# T.81 K.3.3.2: luminance and chrominance AC tables; K.3.3.1: DC tables
STD_DC_BITS = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], [0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0])
STD_DC_VALS = (list(range(12)), list(range(12)))
STD_AC_BITS = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7D], [0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77])
STD_AC_VALS = (bytes.fromhex(
    "01020300041105122131410613516107227114328191a1082342b1c11552d1f02433627282090a161718191a25262728292a3435363738393a434445464748494a"
    "535455565758595a636465666768696a737475767778797a838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4c5c6c7"
    "c8c9cad2d3d4d5d6d7d8d9dae1e2e3e4e5e6e7e8e9eaf1f2f3f4f5f6f7f8f9fa"), bytes.fromhex(
    "000102031104052131061241510761711322328108144291a1b1c109233352f0156272d10a162434e125f11718191a262728292a35363738393a434445464748"
    "494a535455565758595a636465666768696a737475767778797a82838485868788898a92939495969798999aa2a3a4a5a6a7a8a9aab2b3b4b5b6b7b8b9bac2c3c4"
    "c5c6c7c8c9cad2d3d4d5d6d7d8d9dae2e3e4e5e6e7e8e9eaf2f3f4f5f6f7f8f9fa"))

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
                   62, 63])


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp_path_factory.mktemp("huff_emul") / "libhuffemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", "-shared", "-fPIC", EMUL, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    lib = C.CDLL(out)
    lib.emul_build.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    lib.emul_steps.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.emul_decode.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_uint32,
                                C.c_void_p, C.c_int]
    return lib


def _ptr(a):
    return a.ctypes.data_as(C.c_void_p)


def _table(bits16, vals):
    """(bits[0..16] with bits[0] unused, vals[256]) as the builder takes them"""
    b = np.zeros(17, np.uint8)
    b[1:] = bits16
    v = np.zeros(256, np.uint8)
    v[:len(vals)] = list(vals)
    return b, v


def _decoder(bits, vals):
    """one-symbol decoder: the 16-bit window -> (code length, symbol); a window that matches no code takes 17 bits, symbol 0"""
    ln = np.full(65536, 17, np.int64)
    sym = np.zeros(65536, np.int64)
    code = k = 0
    for l in range(1, 17):
        for _ in range(int(bits[l])):
            lo = code << (16 - l)
            ln[lo:lo + (1 << (16 - l))] = l
            sym[lo:lo + (1 << (16 - l))] = vals[k]
            code += 1
            k += 1
        code <<= 1
    return ln, sym


def _extend(bits, s):
    return np.where((s > 0) & (bits < (1 << np.maximum(s - 1, 0))), bits - (1 << s) + 1, bits)


def _ac_symbol(dec, hi, at):
    """the AC symbol at bit `at` of the 32-bit windows hi (at + 16 <= 32 wherever it is used): length, bits, size, advance, value"""
    ln, sym = dec
    w = (hi << at) & 0xFFFFFFFF
    l = ln[w >> 16]
    sy = sym[w >> 16]
    s, r = sy & 15, sy >> 4
    adv = np.where(s == 0, np.where(r == 15, 16, 64), r + 1)
    tb = l + s
    mag = ((w << np.minimum(l, 31)) & 0xFFFFFFFF) >> np.maximum(32 - s, 0)
    mag = np.where(s == 0, 0, mag)
    return l, tb, s, adv, _extend(mag, s)


def _tables():
    import cv2
    from bench import H, W, synth_image
    out = {"k3_luma": _table(STD_AC_BITS[0], STD_AC_VALS[0]), "k3_chroma": _table(STD_AC_BITS[1], STD_AC_VALS[1])}
    ok, enc = cv2.imencode(".jpg", synth_image(H, W, 0), [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_OPTIMIZE, 1])
    assert ok
    dht = _parse(enc.tobytes())[0]
    out["cv2_opt_luma"] = dht[(1, 0)]
    out["cv2_opt_chroma"] = dht[(1, 1)]
    # codes of every length 1..16 (the all-ones code of each length is the prefix of the next), then one more of length 16
    out["every_length"] = _table([1] * 15 + [2], [(i * 37 + 1) & 0xFF for i in range(17)])
    # every code longer than the index: 12..16 bits
    out["all_long"] = _table([0] * 11 + [1, 2, 4, 8, 16], [(i * 53 + 0x11) & 0xFF for i in range(31)])
    return out


def _parse(buf):
    """DHT tables {(class, id): (bits, vals)}, SOF components, SOS table selectors and the un-stuffed entropy data of a baseline
    stream without restart markers"""
    i, dht, comps, sel = 2, {}, None, None
    while True:
        assert buf[i] == 0xFF
        m, L = buf[i + 1], buf[i + 2] << 8 | buf[i + 3]
        seg = buf[i + 4:i + 2 + L]
        if m == 0xC4:
            k = 0
            while k < len(seg):
                tc, th = seg[k] >> 4, seg[k] & 15
                n = sum(seg[k + 1:k + 17])
                dht[(tc, th)] = _table(list(seg[k + 1:k + 17]), seg[k + 17:k + 17 + n])
                k += 17 + n
        elif m == 0xC0:
            comps = [(seg[7 + 3 * c] >> 4) * (seg[7 + 3 * c] & 15) for c in range(seg[5])]
        elif m == 0xDA:
            sel = [(seg[2 + 2 * c] >> 4, seg[2 + 2 * c] & 15) for c in range(seg[0])]
            data = buf[i + 2 + L:]
            break
        i += 2 + L
    out, k = bytearray(), 0
    while k < len(data):
        if data[k] == 0xFF:
            if data[k + 1] != 0:
                break
            k += 1
        out.append(data[k])
        k += 1
    return dht, comps, sel, bytes(out)


@pytest.mark.parametrize("name", ["k3_luma", "k3_chroma", "cv2_opt_luma", "cv2_opt_chroma", "every_length", "all_long"])
def test_every_entry_every_state(emul, name):
    bits, vals = _tables()[name]
    lut = np.zeros(1 << AC_BITS, np.uint32)
    emul.emul_build(_ptr(bits), _ptr(vals), 0, _ptr(lut))
    dec = _decoder(bits, vals)
    rng = np.random.default_rng(7)
    # every index, the 21 bits behind it at random (four draws), then all ones and all zeros
    idx = np.repeat(np.arange(1 << AC_BITS, dtype=np.int64), 6)
    tail = rng.integers(0, 1 << 21, idx.size)
    tail[4::6] = (1 << 21) - 1
    tail[5::6] = 0
    hi = (idx << 21) | tail
    l1, tb1, s1, adv1, v1 = _ac_symbol(dec, hi, 0)
    first_level = l1 <= AC_BITS
    assert ((lut[idx] == 0) == ~first_level).all(), "an entry must be 0 exactly where the code is longer than the index or invalid"
    # the second symbol, where the first one leaves room for a code inside the index
    at2 = np.where(first_level & (tb1 < AC_BITS), tb1, 0)
    l2, tb2, s2, adv2, v2 = _ac_symbol(dec, hi, at2)
    has_pair = first_level & (adv1 != 64) & (tb1 < AC_BITS) & (tb1 + l2 <= AC_BITS)
    assert has_pair.any() or name == "all_long"
    npairs = 0
    for z in range(1, 64):
        for room_kind in range(6):
            room = [tb1 - 1, tb1, tb1 + 1, np.full_like(tb1, AC_BITS - 1), np.full_like(tb1, AC_BITS),
                    np.full_like(tb1, 32)][room_kind]
            room = np.maximum(room, 1)          # a decoder only looks up a symbol that starts before its limit
            out = np.zeros((idx.size, 8), np.int32)
            zz = np.full(idx.size, z, np.int32)
            emul.emul_steps(_ptr(lut), idx.size, _ptr(hi.astype(np.uint32)), _ptr(zz), _ptr(room.astype(np.uint32)), _ptr(out))
            # the second symbol must start before the limit; within kAcLutBits of it no pair is taken at all
            pair = has_pair & (z + adv1 < 64) & (room >= AC_BITS)
            assert (~pair | (tb1 < room)).all()
            npairs += int(pair.sum())
            want_tb = np.where(first_level, np.where(pair, tb1 + tb2, tb1), 0)
            want_adv = np.where(first_level, np.where(pair, adv1 + adv2, adv1), 0)
            np.testing.assert_array_equal(out[:, 0], want_tb, err_msg=f"{name} z={z} bits consumed")
            np.testing.assert_array_equal(out[:, 1], want_adv, err_msg=f"{name} z={z} zig-zag advance")
            # stores: the first symbol of a pair at z + adv1 - 1; the step's last symbol at min(z + adv - 1, 63)
            st1 = pair & (s1 > 0)
            np.testing.assert_array_equal(out[:, 2], np.where(st1, z + adv1 - 1, -1), err_msg=f"{name} z={z}")
            np.testing.assert_array_equal(out[:, 3], np.where(st1, v1, 0), err_msg=f"{name} z={z}")
            s_last = np.where(pair, s2, s1)
            st2 = first_level & (s_last > 0)
            last_zz = np.minimum(z + want_adv - 1, 63)
            np.testing.assert_array_equal(out[:, 4], np.where(st2, last_zz, -1), err_msg=f"{name} z={z}")
            np.testing.assert_array_equal(out[:, 5], np.where(st2, np.where(pair, v2, v1), 0), err_msg=f"{name} z={z}")
            # a pair's first store lands before 63 and before the second's: natural indices stay distinct
            assert (ZIGZAG[out[st1 & st2, 2]] != ZIGZAG[out[st1 & st2, 4]]).all()
    assert npairs > 0 or name == "all_long"


def _decode_spans(emul, data, tables, tsel, bpm, span_bits, pairs, nblocks):
    bits = np.concatenate([t[0] for t in tables])
    vals = np.concatenate([t[1] for t in tables])
    coef = np.zeros((nblocks, 64), np.int16)
    st = np.zeros(5, np.uint32)
    states = []
    buf = np.frombuffer(data, np.uint8)
    total = 8 * len(data)
    for end in list(range(span_bits, total, span_bits)) + [total]:
        emul.emul_decode(_ptr(buf), len(data), _ptr(bits), _ptr(vals), _ptr(tsel), bpm, _ptr(st), pairs, end, _ptr(coef), nblocks)
        states.append(tuple(int(x) for x in st[:4]))
    return states, int(st[4]), coef


def test_random_streams_pairs_equal_single_steps(emul):
    """random bits: long codes, invalid codes, runs past coefficient 63 and blocks that fill 63 without an EOB all occur"""
    t = _tables()
    dc = [_table(STD_DC_BITS[0], STD_DC_VALS[0]), _table(STD_DC_BITS[1], STD_DC_VALS[1])]
    rng = np.random.default_rng(11)
    y, cbcr = 0, 1 | (1 << 8)                        # dc table | ac table << 8 of a block
    cases = [((t["k3_luma"], t["k3_chroma"]), [y, y, y, y, cbcr, cbcr], 256), ((t["cv2_opt_luma"], t["every_length"]), [y, cbcr, cbcr], 1024),
             ((t["all_long"], t["k3_chroma"]), [y], 512), ((t["every_length"], t["cv2_opt_chroma"]), [y, y, cbcr, cbcr], 97)]
    for case, (ac, tsel, span) in enumerate(cases):
        tsel = np.array(tsel, np.int32)
        bpm = len(tsel)
        data = rng.integers(0, 256, 4096, dtype=np.uint8).tobytes()
        a = _decode_spans(emul, data, dc + list(ac), tsel, bpm, span, 0, 4096)
        b = _decode_spans(emul, data, dc + list(ac), tsel, bpm, span, 1, 4096)
        assert a[0] == b[0], f"case {case}: states differ"
        np.testing.assert_array_equal(a[2], b[2], err_msg=f"case {case}")


def test_benchmark_image_pairs_equal_single_steps(emul):
    import cv2
    from bench import H, W, synth_image
    ok, enc = cv2.imencode(".jpg", synth_image(H, W, 0), [cv2.IMWRITE_JPEG_QUALITY, 90])
    assert ok
    dht, comps, sel, data = _parse(enc.tobytes())
    tables = [dht[(0, 0)], dht[(0, 1)], dht[(1, 0)], dht[(1, 1)]]
    tsel = np.array([sel[ci][0] | (sel[ci][1] << 8) for ci, n in enumerate(comps) for _ in range(n)], np.int32)
    bpm = len(tsel)
    nblocks = ((H + 15) // 16) * ((W + 15) // 16) * bpm
    single, steps1, c1 = _decode_spans(emul, data, tables, tsel, bpm, 1024, 0, nblocks)
    paired, steps2, c2 = _decode_spans(emul, data, tables, tsel, bpm, 1024, 1, nblocks)
    assert single == paired
    assert single[-1][3] >= nblocks                 # every block decoded (the pad bits behind the last one may add a few)
    np.testing.assert_array_equal(c1, c2)
    assert steps2 < 0.7 * steps1, (steps1, steps2)  # about 0.64 lookups per symbol at q90
