"""Seeded PNG streams for the decoder tests, written from numpy arrays.

`encode` controls what a PNG decoder has to handle: colour type and bit depth, palette / tRNS, the filter type of every row (0..4 or
a seeded mix), the zlib level and strategy (level 0 = stored blocks, Z_FIXED, Z_HUFFMAN_ONLY, Z_RLE, default), how the zlib stream is
split over IDAT chunks (including 1-byte and zero-length chunks), Adam7 interlacing and an eXIf orientation.  `corpus()` is the set
the tests decode, with streams written by cv2 and Pillow beside ours; `corrupt()` makes one stream of each class libpng rejects.
"""
import io
import struct
import zlib

import numpy as np

SIG = b"\x89PNG\r\n\x1a\n"
ADAM7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]
SPP = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}


def chunk(t, d, bad_crc=False):
    c = zlib.crc32(t + d) & 0xFFFFFFFF
    return struct.pack(">I", len(d)) + t + d + struct.pack(">I", c ^ (1 if bad_crc else 0))


def exif_block(orientation):
    return b"MM\x00\x2a\x00\x00\x00\x08\x00\x01" + struct.pack(">HHIHH", 0x0112, 3, 1, orientation, 0) + b"\x00\x00\x00\x00"


def pack_rows(a, depth):
    """a: (h, w, spp) sample values -> the packed bytes of each row"""
    if depth == 16:
        return [r.astype(">u2").tobytes() for r in a]
    if depth == 8:
        return [r.astype(np.uint8).tobytes() for r in a]
    per = 8 // depth
    rows = []
    for r in a[..., 0]:
        nb = (len(r) * depth + 7) // 8
        v = np.zeros(nb * per, np.int64)
        v[:len(r)] = r
        v = v.reshape(nb, per)
        b = np.zeros(nb, np.int64)
        for k in range(per):
            b |= v[:, k] << (8 - depth * (k + 1))
        rows.append(b.astype(np.uint8).tobytes())
    return rows


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_row(f, cur, prev, bpp):
    c = np.frombuffer(cur, np.uint8).astype(np.int32)
    p = np.frombuffer(prev, np.uint8).astype(np.int32) if prev is not None else np.zeros_like(c)
    a = np.zeros_like(c)
    a[bpp:] = c[:-bpp] if len(c) > bpp else a[bpp:]
    ul = np.zeros_like(c)
    ul[bpp:] = p[:-bpp] if len(c) > bpp else ul[bpp:]
    pred = [np.zeros_like(c), a, p, (a + p) >> 1, _paeth(a, p, ul)][f]
    return bytes([f]) + ((c - pred) & 255).astype(np.uint8).tobytes()


def scanlines(a, depth, ctype, interlace=False, filters=0, seed=0):
    """the filtered scanlines (filter byte first) of all passes"""
    rng = np.random.default_rng(seed)
    bpp = max(1, SPP[ctype] * depth // 8)
    out = []
    passes = ADAM7 if interlace else [(0, 0, 1, 1)]
    for x0, y0, dx, dy in passes:
        sub = a[y0::dy, x0::dx]
        if sub.shape[0] == 0 or sub.shape[1] == 0:
            continue
        prev = None
        for r in pack_rows(sub, depth):
            f = int(rng.integers(0, 5)) if filters == "mixed" else int(filters)
            out.append(filter_row(f, r, prev, bpp))
            prev = r
    return b"".join(out)


def split_idat(z, split):
    if split is None:
        return [z]
    if isinstance(split, int):
        return [z[i:i + split] for i in range(0, len(z), split)] or [b""]
    parts, o = [], 0
    for n in split:
        parts.append(z[o:o + n])
        o += n
    return parts + [z[o:]]


def encode(a, ctype, depth, *, filters=0, level=6, strategy=zlib.Z_DEFAULT_STRATEGY, split=None, interlace=False, palette=None,
           trns=None, exif=None, exif_after=False, seed=0, raw=None):
    """a: (h, w, spp) sample values.  raw: replaces the scanlines (corruption tests)"""
    h, w = a.shape[:2]
    if raw is None:
        raw = scanlines(a, depth, ctype, interlace, filters, seed)
    zo = zlib.compressobj(level, zlib.DEFLATED, 15, 9, strategy)
    z = zo.compress(raw) + zo.flush()
    s = SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, int(interlace)))
    if palette is not None:
        s += chunk(b"PLTE", np.asarray(palette, np.uint8).tobytes())
    if trns is not None:
        s += chunk(b"tRNS", bytes(trns))
    if exif is not None and not exif_after:
        s += chunk(b"eXIf", exif_block(exif))
    s += b"".join(chunk(b"IDAT", part) for part in split_idat(z, split))
    if exif is not None and exif_after:
        s += chunk(b"eXIf", exif_block(exif))
    return s + chunk(b"IEND", b"")


def samples(h, w, ctype, depth, seed):
    """smooth-ish content plus noise, so that every filter type and match length occurs"""
    rng = np.random.default_rng(seed)
    hi = (1 << depth) - 1
    y, x = np.mgrid[0:h, 0:w]
    base = (x * 7 + y * 3) % (hi + 1) if depth < 8 else ((x * 37 + y * 11) * hi // max(1, 37 * w + 11 * h))
    n = SPP[ctype]
    a = np.stack([base] * n, -1).astype(np.int64)
    noise = rng.integers(0, hi + 1, a.shape)
    mask = rng.random(a.shape) < 0.3
    return np.where(mask, noise, a)


def _cv2_stream(a, **kw):
    import cv2
    ok, b = cv2.imencode(".png", a, [cv2.IMWRITE_PNG_COMPRESSION, kw.get("level", 3)])
    assert ok
    return b.tobytes()


def _pil_stream(img, **kw):
    buf = io.BytesIO()
    img.save(buf, format="PNG", **kw)
    return buf.getvalue()


def corpus(seed=0):
    """[(name, stream)]: every legal colour type / bit depth, filters, deflate strategies, IDAT splits, Adam7, palettes, cv2 and
    Pillow writers"""
    out = []
    legal = [(0, 1), (0, 2), (0, 4), (0, 8), (0, 16), (2, 8), (2, 16), (3, 1), (3, 2), (3, 4), (3, 8), (4, 8), (4, 16), (6, 8), (6, 16)]
    k = seed
    for ct, d in legal:
        for h, w in ((13, 29), (1, 1), (9, 3)):
            k += 1
            a = samples(h, w, ct, d, k)
            pal = None
            if ct == 3:
                npal = 1 << d
                pal = np.random.default_rng(k).integers(0, 256, (npal, 3))
            for il in (False, True):
                out.append((f"ct{ct}_d{d}_{h}x{w}_il{int(il)}",
                            encode(a, ct, d, filters="mixed", interlace=il, palette=pal, seed=k)))
    a = samples(40, 57, 2, 8, 99)
    for f in range(5):
        out.append((f"filter{f}", encode(a, 2, 8, filters=f)))
    strategies = [("stored", 0, zlib.Z_DEFAULT_STRATEGY), ("fixed", 6, zlib.Z_FIXED), ("huffman", 6, zlib.Z_HUFFMAN_ONLY),
                  ("rle", 6, zlib.Z_RLE), ("default9", 9, zlib.Z_DEFAULT_STRATEGY)]
    for name, lvl, st in strategies:
        out.append((f"zlib_{name}", encode(a, 2, 8, filters="mixed", level=lvl, strategy=st, seed=3)))
    big = samples(300, 400, 2, 8, 7)          # more than 32 KiB of scanlines: distances span the whole window, stored blocks split
    out.append(("big_stored", encode(big, 2, 8, filters="mixed", level=0, seed=4)))
    out.append(("big_default", encode(big, 2, 8, filters="mixed", seed=4)))
    out.append(("split1", encode(a, 2, 8, filters="mixed", split=1, seed=5)))
    out.append(("split_zero", encode(a, 2, 8, filters="mixed", split=[0, 1, 0, 7, 0, 0, 300], seed=5)))
    out.append(("split_big_stored", encode(big, 2, 8, level=0, split=1000, seed=6)))
    # palette with tRNS and an index past the palette's end (libpng reads black)
    idx = np.random.default_rng(11).integers(0, 256, (17, 23, 1))
    out.append(("palette_oob", encode(idx, 3, 8, palette=np.random.default_rng(12).integers(0, 256, (100, 3)), trns=[0, 128, 255])))
    out.append(("rgba_trns_gray", encode(samples(8, 8, 0, 8, 13), 0, 8, trns=[0, 7])))
    out.append(("surplus", encode(a, 2, 8, raw=scanlines(a, 8, 2) + b"\x00" * 100)))
    out += [(n, st) for n, st, ok in zlib_tails() if ok]
    out.append(("colours_all", encode(np.random.default_rng(14).integers(0, 256, (64, 64, 3)), 2, 8)))
    # other writers
    import cv2
    from PIL import Image
    rng = np.random.default_rng(15)
    img = rng.integers(0, 256, (31, 45, 3), dtype=np.uint8)
    img[::2] = img[::2] // 16 * 16
    out.append(("cv2_bgr", _cv2_stream(img)))
    out.append(("cv2_gray", _cv2_stream(img[..., 0])))
    out.append(("cv2_bgra", _cv2_stream(np.dstack([img, img[..., :1]]), level=9)))
    out.append(("cv2_16", _cv2_stream((img.astype(np.uint16) * 257 + 3))))
    pim = Image.fromarray(img)
    out.append(("pil_palette", _pil_stream(pim.quantize(77))))
    out.append(("pil_1bit", _pil_stream(pim.convert("1"))))
    out.append(("pil_la", _pil_stream(pim.convert("LA"))))
    out.append(("pil_rgba_opt", _pil_stream(pim.convert("RGBA"), optimize=True)))
    return out


def _fixed_block_stream(codes):
    """zlib stream of one final fixed-Huffman block whose symbols are given as (code, nbits) pairs sent MSB first"""
    bits = [1, 1, 0]                                    # BFINAL, BTYPE = 01 (LSB first)
    for code, n in codes:
        bits += [(code >> (n - 1 - i)) & 1 for i in range(n)]
    bits += [0] * (-len(bits) % 8)
    body = bytes(sum(b << i for i, b in enumerate(bits[j:j + 8])) for j in range(0, len(bits), 8))
    return b"\x78\x01" + body + b"\x00" * 8


def _with_zlib(a, ct, d, z):
    h, w = a.shape[:2]
    return SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, d, ct, 0, 0, 0)) + chunk(b"IDAT", z) + chunk(b"IEND", b"")


def _lsb(v, n):
    return [(v >> i) & 1 for i in range(n)]


def _msb(c, n):
    return [(c >> (n - 1 - i)) & 1 for i in range(n)]


def _pack_bits(bits):
    bits = bits + [0] * (-len(bits) % 8)
    return bytes(sum(b << k for k, b in enumerate(bits[j:j + 8])) for j in range(0, len(bits), 8))


def zlib_tails():
    """[(name, stream, cv2 decodes it)]: what follows the image's last byte in the zlib stream, probed against cv2 4.13.  An empty
    final block or a final dynamic block that codes only its end-of-block symbol (a single length-1 literal / length code) after
    the image, with a good or a bad Adler-32; more data than the image needs, then a bad trailer, a malformed block, no trailer or
    data cut short; the image's data without a trailer."""
    a = samples(6, 7, 2, 8, 1)
    raw = scanlines(a, 8, 2)
    ad = struct.pack(">I", zlib.adler32(raw))
    bad_ad = bytes([ad[0] ^ 1]) + ad[1:]
    stored = b"\x00" + struct.pack("<HH", len(raw), len(raw) ^ 0xFFFF) + raw          # non-final stored block
    empty_final = b"\x01" + struct.pack("<HH", 0, 0xFFFF)
    # final dynamic block: code-length code {1: 1 bit, 0: 2, 18: 2}; 256 zeros (18 x 138, 18 x 118), a 1 for symbol 256, one
    # distance length 0; then the end-of-block code 0
    order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
    bits = [1] + _lsb(2, 2) + _lsb(0, 5) + _lsb(0, 5) + _lsb(14, 4)
    for sym in order[:18]:
        bits += _lsb({18: 2, 0: 2, 1: 1}.get(sym, 0), 3)
    bits += _msb(0b11, 2) + _lsb(138 - 11, 7) + _msb(0b11, 2) + _lsb(118 - 11, 7) + _msb(0, 1) + _msb(0b10, 2) + _msb(0, 1)
    eob_only = _pack_bits(bits)
    raw2 = raw + b"\x00" * 50
    ad2 = struct.pack(">I", zlib.adler32(raw2))
    st2 = b"\x01" + struct.pack("<HH", len(raw2), len(raw2) ^ 0xFFFF) + raw2
    st2_open = b"\x00" + st2[1:]
    exact_final = b"\x01" + stored[1:]
    cases = [("empty_final_block", stored + empty_final + ad, True), ("empty_final_block_bad_adler", stored + empty_final + bad_ad, False),
             ("eob_only_block", stored + eob_only + ad, True), ("eob_only_block_bad_adler", stored + eob_only + bad_ad, False),
             ("surplus_bad_adler", st2 + bytes([ad2[0] ^ 1]) + ad2[1:], True), ("surplus_bad_block", st2_open + b"\x07" + ad2, True),
             ("surplus_no_trailer", st2, False), ("surplus_cut", st2[:-20], False), ("exact_no_trailer", exact_final, False)]
    return [(n, _with_zlib(a, 2, 8, b"\x78\x01" + z), ok) for n, z, ok in cases]


def corrupt():
    """[(name, stream)]: one stream of each class cv2.imdecode rejects"""
    a = samples(20, 30, 2, 8, 21)
    good = encode(a, 2, 8, filters="mixed", seed=21)
    raw = scanlines(a, 8, 2, filters="mixed", seed=21)
    z = zlib.compress(raw)
    i = good.index(b"IDAT")
    out = []
    s = bytearray(good)
    n = struct.unpack(">I", s[i - 4:i])[0]
    s[i + 4 + n] ^= 1                                    # last byte of the IDAT CRC
    out.append(("idat_crc", bytes(s)))
    out.append(("adler", _with_zlib(a, 2, 8, z[:-1] + bytes([z[-1] ^ 1]))))
    out.append(("truncated", _with_zlib(a, 2, 8, z[:len(z) // 2])))
    out.append(("filter5", encode(a, 2, 8, raw=bytes([5]) + raw[1:])))
    out.append(("distance", _with_zlib(a, 2, 8, _fixed_block_stream([(0b0000001, 7), (0, 5)]))))       # length 3, distance 1 at 0
    out.append(("undefined_symbol", _with_zlib(a, 2, 8, _fixed_block_stream([(0x30 + 65, 8), (0b11000110, 8)]))))   # 'A', 286
    # dynamic block whose code-length code is over-subscribed (19 codes of length 1)
    bits = [1, 0, 1] + [0] * 5 + [0] * 5 + [1, 1, 1, 1] + [1, 0, 0] * 19
    bits += [0] * (-len(bits) % 8)
    body = bytes(sum(b << k for k, b in enumerate(bits[j:j + 8])) for j in range(0, len(bits), 8))
    out.append(("code_lengths", _with_zlib(a, 2, 8, b"\x78\x01" + body + b"\x00" * 8)))
    out.append(("no_iend", good[:-12]))
    s = bytearray(good)
    s[29] ^= 1                                           # IHDR CRC
    out.append(("ihdr_crc", bytes(s)))
    out.append(("critical_chunk", good[:33] + chunk(b"ABCD", b"x") + good[33:]))
    # 2^29 x 1 RGBA 16-bit: rows of 4 GiB (libpng: at most 1000000 pixels per side)
    out.append(("wide", SIG + chunk(b"IHDR", struct.pack(">IIBBBBB", 1 << 29, 1, 16, 6, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(b"\x00")) +
                chunk(b"IEND", b"")))
    out += [(n, st) for n, st, ok in zlib_tails() if not ok]
    zz = zlib.compress(raw)
    out.append(("idat_gap", SIG + good[8:33] + chunk(b"IDAT", zz[:9]) + chunk(b"tEXt", b"a\x00b") + chunk(b"IDAT", zz[9:]) +
                chunk(b"IEND", b"")))
    return out
