"""Seeded TIFF writer for the tests: its own LZW (MSB-first, early change, as libtiff writes it) and PackBits encoders, zlib for
Deflate, so that strips down to one row, tiles with padded edges, PlanarConfiguration 2, both byte orders, every supported photometric
and bit depth, and crafted corruptions can be written -- Pillow and cv2 write only some of these.  corpus() also holds cv2- and
Pillow-written files; data_corrupt() and plan_corrupt() hold one stream per corruption class."""
import io
import struct
import zlib

import numpy as np


class _Bits:
    def __init__(self):
        self.out, self.acc, self.n = bytearray(), 0, 0

    def put(self, v, w):
        self.acc = (self.acc << w) | v
        self.n += w
        while self.n >= 8:
            self.n -= 8
            self.out.append((self.acc >> self.n) & 255)

    def done(self):
        if self.n:
            self.out.append((self.acc << (8 - self.n)) & 255)
        return bytes(self.out)


def lzw(data, clear_first=True):
    """libtiff's LZWEncode: Clear first, a Clear when the table reaches 4094 entries, the code width grows one code early, EOI last"""
    b = _Bits()
    width, maxcode, free = 9, 511, 258
    if clear_first:
        b.put(256, 9)
    if not data:
        b.put(257, 9)
        return b.done()
    table = {}
    ent = data[0]
    for c in data[1:]:
        key = (ent, c)
        if key in table:
            ent = table[key]
            continue
        b.put(ent, width)
        ent = c
        table[key] = free
        free += 1
        if free == 4094:
            b.put(256, width)
            table, free, width, maxcode = {}, 258, 9, 511
        elif free > maxcode:
            width += 1
            maxcode = (1 << width) - 1
    b.put(ent, width)
    free += 1
    if free == 4094:
        b.put(256, width)
        width = 9
    elif free > maxcode:
        width += 1
    b.put(257, width)
    return b.done()


def packbits(data):
    out, i, n = bytearray(), 0, len(data)
    while i < n:
        j = i
        while j + 1 < n and data[j + 1] == data[i] and j - i < 127:
            j += 1
        if j - i >= 2:
            out += bytes([257 - (j - i + 1), data[i]])
            i = j + 1
            continue
        j = i
        while j < n and j - i < 128 and not (j + 2 < n and data[j] == data[j + 1] == data[j + 2]):
            j += 1
        out.append(j - i - 1)
        out += data[i:j]
        i = j
    return bytes(out)


def _pack_rows(a, bps, big_endian):
    """(rows, width, samples) sample values -> packed rows, each padded to a byte"""
    rows, w, c = a.shape
    if bps == 16:
        return a.astype(">u2" if big_endian else "<u2").reshape(rows, -1).view(np.uint8).reshape(rows, -1)
    if bps == 8:
        return a.astype(np.uint8).reshape(rows, -1)
    flat = a.reshape(rows, w * c).astype(np.uint8)
    bits = np.unpackbits(flat[..., None], axis=-1)[..., 8 - bps:].reshape(rows, -1)
    return np.packbits(bits, axis=-1)


def _predict(a, bps):
    d = a.astype(np.int64).copy()
    d[:, 1:] -= a[:, :-1].astype(np.int64)
    return (d % (1 << bps)).astype(np.uint32)


def encode(a, photometric, bps, compression=5, predictor=1, planar=1, rows_per_strip=None, tile=None, big_endian=False,
           extra=None, colormap=None, orientation=None, extra_tags=(), lzw_clear_first=True):
    """a: (H, W, spp) sample values.  Returns the bytes of a classic TIFF holding one image."""
    a = np.asarray(a)
    if a.ndim == 2:
        a = a[..., None]
    H, W, spp = a.shape
    e = ">" if big_endian else "<"
    planes = [a[..., k:k + 1] for k in range(spp)] if planar == 2 else [a]
    if tile:
        tw, th = tile
        rects = [(x, y, tw, th) for y in range(0, H, th) for x in range(0, W, tw)]
    else:
        rps = rows_per_strip or H
        rects = [(0, y, W, min(rps, H - y)) for y in range(0, H, rps)]
    segs = []
    for pl in planes:
        for x, y, w, h in rects:
            blk = np.zeros((h, w, pl.shape[2]), np.uint32)
            src = pl[y:y + h, x:x + w]
            blk[:src.shape[0], :src.shape[1]] = src
            if predictor == 2:
                blk = _predict(blk, bps)
            raw = _pack_rows(blk, bps, big_endian).tobytes()
            if compression == 5:
                raw = lzw(raw, lzw_clear_first)
            elif compression in (8, 32946):
                raw = zlib.compress(raw, 6)
            elif compression == 32773:
                raw = packbits(raw)
            segs.append(raw)
    tags = {256: (4, [W]), 257: (4, [H]), 258: (3, [bps] * spp), 259: (3, [compression]), 262: (3, [photometric]),
            277: (3, [spp]), 284: (3, [planar])}
    if predictor != 1:
        tags[317] = (3, [predictor])
    if extra is not None:
        tags[338] = (3, list(extra))
    if colormap is not None:
        tags[320] = (3, list(np.asarray(colormap, np.uint32).T.reshape(-1)))
    if orientation is not None:
        tags[274] = (3, [orientation])
    for k, v in extra_tags:
        tags[k] = v
    body = bytearray(b"MM\0*" if big_endian else b"II*\0") + b"\0\0\0\0"
    offs = []
    for s in segs:
        offs.append(len(body))
        body += s
        if len(body) & 1:
            body += b"\0"
    if tile:
        tags[322] = (3, [tile[0]])
        tags[323] = (3, [tile[1]])
        tags[324] = (4, offs)
        tags[325] = (4, [len(s) for s in segs])
    else:
        tags[278] = (4, [rows_per_strip or H])
        tags[273] = (4, offs)
        tags[279] = (4, [len(s) for s in segs])
    entries = []
    for k in sorted(tags):
        t, v = tags[k]
        fmt = "H" if t == 3 else "I"
        data = struct.pack(e + fmt * len(v), *[int(x) for x in v])
        if len(data) <= 4:
            entries.append((k, t, len(v), data.ljust(4, b"\0"), None))
        else:
            entries.append((k, t, len(v), None, len(body)))
            body += data
            if len(body) & 1:
                body += b"\0"
    ifd = len(body)
    body[4:8] = struct.pack(e + "I", ifd)
    body += struct.pack(e + "H", len(entries))
    for k, t, n, inline, off in entries:
        body += struct.pack(e + "HHI", k, t, n) + (inline if inline is not None else struct.pack(e + "I", off))
    body += b"\0\0\0\0"
    return bytes(body)


def samples(h, w, spp, bps, seed):
    """smooth-ish content with noise, so that every codec has runs and literals"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    top = (1 << bps) - 1
    base = np.stack([(x * (k + 1) * 7 + y * (3 - k % 3) * 5) for k in range(spp)], -1)
    noise = rng.integers(0, max(2, top // 16 + 1), (h, w, spp))
    a = (base * max(1, top // 255) + noise) % (top + 1)
    a[: h // 3, : w // 4] = rng.integers(0, top + 1, spp)          # a flat patch (PackBits runs, long LZW strings)
    return a.astype(np.uint32)


def palette(bps, seed, wide=True):
    rng = np.random.default_rng(seed)
    m = rng.integers(0, 256, (1 << bps, 3))
    return m * 257 if wide else m


def _cv2(img, ext=".tiff", params=()):
    import cv2
    ok, b = cv2.imencode(ext, img, list(params))
    assert ok
    return b.tobytes()


def _pil(arr, mode, **kw):
    from PIL import Image
    bio = io.BytesIO()
    Image.fromarray(arr, mode).save(bio, "TIFF", **kw) if mode else Image.fromarray(arr).save(bio, "TIFF", **kw)
    return bio.getvalue()


def corpus():
    """(name, stream) pairs the decoder must decode exactly as cv2.imdecode does"""
    out = []
    k = 0
    for comp in (1, 5, 8, 32946, 32773):
        for pred in (1, 2):
            for photometric, spp, bps, extra in [(1, 1, 8, None), (2, 3, 8, None), (2, 4, 8, (2,)), (2, 4, 8, (1,)), (1, 2, 8, (2,)),
                                                 (2, 3, 16, None), (1, 1, 16, None), (0, 1, 8, None), (2, 4, 16, (2,)), (0, 1, 16, None)]:
                if pred == 2 and comp == 32773 and bps == 16:
                    continue
                k += 1
                be = k % 3 == 0
                layout = [dict(rows_per_strip=1), dict(rows_per_strip=5), dict(tile=(16, 16)), dict(), dict(tile=(32, 16))][k % 5]
                if "tile" in layout and (comp == 1 or (bps == 16 and spp == 1)):
                    layout = dict(rows_per_strip=2)
                planar = 2 if (spp > 1 and k % 4 == 1) else 1
                h, w = 19 + k % 7, 23 + k % 11
                out.append((f"c{comp}_p{pred}_ph{photometric}_s{spp}_b{bps}_e{extra}_{k}",
                            encode(samples(h, w, spp, bps, k), photometric, bps, comp, pred, planar, big_endian=be, extra=extra, **layout)))
    for photometric in (0, 1):
        for bps in (1,):
            for comp in (1, 5, 32773, 8):
                k += 1
                lay = dict(tile=(16, 32)) if k % 3 == 0 and comp != 1 else dict(rows_per_strip=3)
                out.append((f"gray{bps}_ph{photometric}_c{comp}", encode(samples(21, 37, 1, bps, k), photometric, bps, comp,
                                                                         big_endian=k % 2 == 0, **lay)))
    for bps in (1, 4, 8):
        for wide in (True, False):
            for comp in (1, 5, 8):
                k += 1
                out.append((f"palette{bps}_{wide}_c{comp}", encode(samples(17, 29, 1, bps, k), 3, bps, comp, colormap=palette(bps, k, wide),
                                                                   rows_per_strip=4, big_endian=k % 2 == 0)))
    # 2-row strips that LZW-code 2^13+ bytes (the table fills, Clear, and restarts)
    big = samples(40, 400, 3, 8, 99)
    big[::2] = np.random.default_rng(5).integers(0, 256, big[::2].shape)
    out.append(("lzw_table_full", encode(big, 2, 8, 5, rows_per_strip=20)))
    # cv2 and Pillow
    import cv2
    rng = np.random.default_rng(11)
    img = (samples(45, 61, 3, 8, 12)).astype(np.uint8)
    out.append(("cv2_rgb", _cv2(img)))
    out.append(("cv2_gray", _cv2(img[..., 0])))
    out.append(("cv2_rgba", _cv2(np.dstack([img, rng.integers(0, 256, img.shape[:2]).astype(np.uint8)]))))
    out.append(("cv2_rgb16", _cv2((samples(33, 47, 3, 16, 13)).astype(np.uint16))))
    out.append(("cv2_gray16", _cv2((samples(33, 47, 1, 16, 14))[..., 0].astype(np.uint16))))
    out.append(("cv2_rgb_nocomp", _cv2(img, params=(cv2.IMWRITE_TIFF_COMPRESSION, 1))))
    out.append(("pil_rgb", _pil(img, "RGB")))
    out.append(("pil_gray16", _pil(samples(30, 40, 1, 16, 15)[..., 0].astype(np.uint16), "I;16")))
    out.append(("pil_palette", _pil(img[..., 0] % 200, "P")))
    out.append(("pil_rgb_deflate", _pil(img, "RGB", compression="tiff_adobe_deflate")))
    out.append(("pil_rgb_packbits", _pil(img, "RGB", compression="packbits")))
    out.append(("pil_bilevel", _pil(img[..., 0] > 100, "1")))
    out.append(("pil_rgba", _pil(np.dstack([img, img[..., 1]]), "RGBA")))
    return out


def _patch_tag(s, tag, value):
    """rewrites the first value of an inline tag"""
    e = ">" if s[:2] == b"MM" else "<"
    ifd = struct.unpack(e + "I", s[4:8])[0]
    n = struct.unpack(e + "H", s[ifd:ifd + 2])[0]
    b = bytearray(s)
    for i in range(n):
        o = ifd + 2 + 12 * i
        t, ty = struct.unpack(e + "HH", s[o:o + 4])
        if t == tag:
            b[o + 8:o + 12] = struct.pack(e + ("H" if ty == 3 else "I"), value).ljust(4, b"\0")
            return bytes(b)
    raise KeyError(tag)


def _seg0(s):
    e = ">" if s[:2] == b"MM" else "<"
    ifd = struct.unpack(e + "I", s[4:8])[0]
    n = struct.unpack(e + "H", s[ifd:ifd + 2])[0]
    for i in range(n):
        o = ifd + 2 + 12 * i
        t, ty, c = struct.unpack(e + "HHI", s[o:o + 8])
        if t in (273, 324):
            v = struct.unpack(e + "I", s[o + 8:o + 12])[0]
            return v if c == 1 else struct.unpack(e + "I", s[v:v + 4])[0]


def data_corrupt():
    """streams the planner accepts whose segment data is bad: (name, stream); each is a per-sample decode error in cv2 and here"""
    a = samples(12, 20, 3, 8, 21)
    out = []
    one = lambda comp, **kw: encode(a, 2, 8, comp, rows_per_strip=12, **kw)
    s = one(5)
    o = _seg0(s)
    out.append(("lzw_eoi_early", s[:o] + lzw(bytes(a.astype(np.uint8).reshape(-1)[:300])) + s[o + len(lzw(bytes(a.astype(np.uint8).reshape(-1)[:300]))):]))
    b = bytearray(s)
    b[o + 40] ^= 0xFF
    b[o + 41] ^= 0xFF
    out.append(("lzw_bad_code", bytes(b)))
    out.append(("lzw_truncated", _patch_tag(s, 279, 100)))
    out.append(("lzw_no_clear", one(5, lzw_clear_first=False)))
    s = one(8)
    out.append(("deflate_truncated", _patch_tag(s, 279, 60)))
    b = bytearray(s)
    o = _seg0(s)
    b[o] = 0x79
    out.append(("deflate_header", bytes(b)))
    b = bytearray(s)
    n = struct.unpack("<I", _tag_bytes(s, 279))[0]
    b[o + n - 1] ^= 1
    out.append(("deflate_adler", bytes(b)))
    s = one(32773)
    out.append(("packbits_truncated", _patch_tag(s, 279, 30)))
    s = one(1)
    out.append(("raw_truncated", _patch_tag(s, 279, 100)))
    return out


def _tag_bytes(s, tag):
    e = ">" if s[:2] == b"MM" else "<"
    ifd = struct.unpack(e + "I", s[4:8])[0]
    n = struct.unpack(e + "H", s[ifd:ifd + 2])[0]
    for i in range(n):
        o = ifd + 2 + 12 * i
        if struct.unpack(e + "H", s[o:o + 2])[0] == tag:
            return s[o + 8:o + 12]


def plan_corrupt():
    """streams whose IFD or segment table is malformed or unsupported: (name, stream).  The plan set-up fails for every one.  cv2
    rejects those named in CV2_REJECTS too; the others it decodes, where the decoder refuses what it does not support (DESIGN 2)."""
    a = samples(12, 20, 3, 8, 22)
    s = encode(a, 2, 8, 5, rows_per_strip=4)
    out = [("truncated_ifd", s[:-20]),
           ("segment_outside", _patch_tag(encode(a, 2, 8, 1), 273, len(s) + 100)),
           ("bigtiff", b"II+\0" + s[4:]),
           ("jpeg_compression", _patch_tag(s, 259, 7)),
           ("fill_order_2", encode(a, 2, 8, 5, rows_per_strip=4, extra_tags=[(266, (3, [2]))])),
           ("float_samples", encode(a, 2, 8, 5, rows_per_strip=4, extra_tags=[(339, (3, [3, 3, 3]))])),
           ("predictor_3", _patch_tag(encode(a, 2, 8, 5, 2, rows_per_strip=4), 317, 3)),
           ("cmyk", _patch_tag(encode(samples(12, 20, 4, 8, 3), 2, 8, 5), 262, 5)),
           ("ycbcr", _patch_tag(s, 262, 6)),
           ("too_wide", _patch_tag(encode(a, 2, 8, 1), 256, (1 << 20) + 1)),
           ("too_many_pixels", _patch_tag(_patch_tag(encode(a, 2, 8, 1), 256, 40000), 257, 30000)),
           ("oversized_tile", _patch_tag(_patch_tag(encode(samples(2, 2, 3, 8, 5), 2, 8, 5, tile=(16, 16)), 322, 32768), 323, 16384)),
           ("gray2", encode(samples(12, 20, 1, 2, 4), 1, 2, 5)),
           ("gray4", encode(samples(12, 20, 1, 4, 4), 1, 4, 5)),
           ("palette2", encode(samples(12, 20, 1, 2, 4), 3, 2, 5, colormap=palette(2, 1))),
           ("raw_tiles", encode(a, 2, 8, 1, tile=(16, 16))),
           ("gray16_tiles", encode(samples(12, 20, 1, 16, 4), 1, 16, 5, tile=(16, 16))),
           ("old_lzw", _old_lzw(s))]
    return out


# plan_corrupt() streams cv2.imdecode rejects as well (None, or an error for the size limits)
CV2_REJECTS = {"truncated_ifd", "segment_outside", "bigtiff", "jpeg_compression", "float_samples", "predictor_3", "too_wide",
               "too_many_pixels", "oversized_tile", "gray2", "gray4", "palette2", "raw_tiles"}


def _old_lzw(s):
    b = bytearray(s)
    o = _seg0(s)
    b[o], b[o + 1] = 0, 1
    return bytes(b)
