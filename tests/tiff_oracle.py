"""numpy restatement of what cv2.imdecode (OpenCV 4.13 / libtiff 4.7) makes of a TIFF stream with IMREAD_COLOR and IMREAD_GRAYSCALE;
tests/test_tiff_cpu.py pins it against cv2 on the corpus of tests/tiff_streams.py.

cv2 decodes 8-bit output through libtiff's TIFFReadRGBA* and converts RGBA to BGR (alpha dropped) or to gray.  The rules:
  * a segment (strip or tile of one plane) decodes to exactly its size; surplus input is ignored, a short segment is an error, and an
    error anywhere fails the image.  LZW is libtiff's decoder (a first code that is not Clear is rejected here, see DESIGN 2);
    Deflate stops once the segment is full (a bad block header or Adler-32 met before that is an error); PackBits clips a run at the
    segment's end.
  * gray (contiguous): 1/8 bits -> v * 255 // (2^bps - 1), MinIsWhite (2^bps - 1 - v) * 255 // (2^bps - 1); 16 bits -> high byte
    (MinIsWhite 255 - high byte).  An extra sample is dropped.  1-bit gray is {0, 255}.  cv2 rejects 2- and 4-bit gray, 2-bit palette
    and uncompressed tiles; it reads 16-bit gray tiles otherwise, and those are rejected here.
  * Predictor applies to LZW and Deflate only; with no compression or PackBits the tag is ignored.
  * a corrupt segment: cv2 returns an image with whatever libtiff's RGBA reader (stoponerr = 0) left in its buffer; decode() returns
    None, as the decoder fails the sample (DESIGN 2).
  * RGB, and gray + extra sample in PlanarConfiguration 2 (libtiff reads it as RGB with R = G = B, without MinIsWhite inversion):
    16 bits -> (v + 128) // 257; ExtraSamples = 2 (unassociated alpha) premultiplies: (c * a + 127) // 255 on the 8-bit values;
    associated or unspecified alpha is dropped.
  * palette: the ColorMap's high bytes, or its values when every entry is below 256 (libtiff's 8-bit ColorMap guess).
  * GRAY of a colour pixel: (1868 B + 9617 G + 4899 R + 8192) >> 14.
  * Orientation (tag 274) is returned, to be applied as orient() does.
decode() returns (rgb, gray, orientation) or None where cv2 returns None."""
import struct
import zlib

import numpy as np

from png_oracle import orient  # noqa: F401  (EXIF orientation as cv2.imdecode applies it)

GRAY = (4899, 9617, 1868)


def _lzw(src, total):
    out = bytearray()
    acc = nb = pos = 0
    width, mask, k = 9, 511, -1
    start = []
    while len(out) < total:
        while nb < width:
            if pos >= len(src):
                return None
            acc = (acc << 8) | src[pos]
            pos += 1
            nb += 8
        nb -= width
        code = (acc >> nb) & ((1 << width) - 1)
        if code == 257:
            return None
        if code == 256:
            k, width, mask, start = 0, 9, 511, []
            continue
        if k < 0:
            return None
        fr = 257 + k
        if k == 0:
            if code > 255:
                return None
        else:
            if fr >= 5119 or (code > 255 and code > fr):
                return None
            if fr + 1 > mask - 1 and width < 12:
                width += 1
                mask = (1 << width) - 1
        start.append(len(out))
        k += 1
        if code < 256:
            out.append(code)
            continue
        j = code - 258
        s0 = start[j]
        n = start[j + 1] - s0 + 1
        for i in range(n):
            if len(out) >= total:
                break
            out.append(out[s0 + i])
    return bytes(out[:total])


def _packbits(src, total):
    out, pos = bytearray(), 0
    while pos < len(src) and len(out) < total:
        c = src[pos] - 256 if src[pos] >= 128 else src[pos]
        pos += 1
        if c == -128:
            continue
        if c < 0:
            if pos >= len(src):
                break
            out += bytes([src[pos]]) * min(1 - c, total - len(out))
            pos += 1
        else:
            m = min(c + 1, total - len(out))
            if m > len(src) - pos:
                break
            out += src[pos:pos + m]
            pos += m
    return bytes(out) if len(out) >= total else None


def _inflate(src, total):
    try:
        d = zlib.decompressobj()
        out = d.decompress(src, total)
    except zlib.error:
        return None
    return out if len(out) == total else None


def _parse(s):
    if len(s) < 8 or s[:4] not in (b"II*\0", b"MM\0*"):
        return None
    e = ">" if s[0:1] == b"M" else "<"
    ifd = struct.unpack(e + "I", s[4:8])[0]
    if ifd + 2 > len(s):
        return None
    n = struct.unpack(e + "H", s[ifd:ifd + 2])[0]
    if n == 0 or ifd + 2 + 12 * n > len(s):
        return None
    tags = {}
    for i in range(n):
        o = ifd + 2 + 12 * i
        t, ty, c = struct.unpack(e + "HHI", s[o:o + 8])
        if ty not in (3, 4):
            continue
        sz = 2 if ty == 3 else 4
        off = o + 8 if c * sz <= 4 else struct.unpack(e + "I", s[o + 8:o + 12])[0]
        if off + c * sz > len(s):
            return None
        tags[t] = list(struct.unpack(e + ("H" if ty == 3 else "I") * c, s[off:off + c * sz]))
    return e, tags


def decode(s):
    p = _parse(s)
    if p is None:
        return None
    e, t = p
    g = lambda k, d: t.get(k, [d])[0]
    W, H = g(256, 0), g(257, 0)
    spp, bps, comp, pred, planar = g(277, 1), g(258, 1), g(259, 1), g(317, 1), g(284, 1)
    ph = g(262, -1)
    if W == 0 or H == 0 or W > 1 << 20 or H > 1 << 20 or W * H > 1 << 30:
        return None
    if comp not in (1, 5, 8, 32946, 32773) or g(266, 1) != 1 or pred not in (1, 2) or any(v != 1 for v in t.get(339, [1])):
        return None
    ok = ((ph in (0, 1) and ((spp == 1 and bps in (1, 8, 16)) or (spp == 2 and bps in (8, 16)))) or
          (ph == 2 and spp in (3, 4) and bps in (8, 16)) or (ph == 3 and spp == 1 and bps in (1, 4, 8)))
    if not ok or (pred == 2 and bps not in (8, 16)):
        return None
    if comp not in (5, 8, 32946):
        pred = 1                      # libtiff applies Predictor to LZW and Deflate only
    if spp == 1:
        planar = 1
    planes = spp if planar == 2 else 1
    psp = 1 if planar == 2 else spp
    tiled = 322 in t
    if tiled and (comp == 1 or (bps == 16 and ph != 2 and spp == 1)):
        return None
    sw, sh = (g(322, 0), g(323, 0)) if tiled else (W, min(g(278, 0xFFFFFFFF), H))
    if tiled and (sw > max(512, -(-W // 16) * 16) or sh > max(512, -(-H // 16) * 16)):
        return None                   # refused by the decoder: a tile far beyond the image only claims decode scratch
    offs, cnts = (t.get(324), t.get(325)) if tiled else (t.get(273), t.get(279))
    across, down = -(-W // sw), -(-H // sh)
    if offs is None or cnts is None or len(offs) != across * down * planes or len(cnts) != len(offs):
        return None
    rb = (sw * psp * bps + 7) // 8
    full = np.zeros((planes, down * sh, across * sw, psp), np.uint32)
    for k, (o, n) in enumerate(zip(offs, cnts)):
        if o + n > len(s):
            return None
        src = s[o:o + n]
        if comp == 5 and len(src) >= 2 and src[0] == 0 and src[1] & 1:
            return None
        pl, r = divmod(k, across * down)
        sy, sx = divmod(r, across)
        rows = sh if tiled else min(sh, H - sy * sh)
        total = rows * rb
        dec = (_lzw(src, total) if comp == 5 else _inflate(src, total) if comp in (8, 32946) else _packbits(src, total) if comp == 32773
               else (src[:total] if len(src) >= total else None))
        if dec is None:
            return None
        a = np.frombuffer(dec, np.uint8).reshape(rows, rb)
        if bps == 16:
            v = a.view(e + "u2").astype(np.uint32).reshape(rows, sw, psp)
        elif bps == 8:
            v = a.astype(np.uint32).reshape(rows, sw, psp)
        else:
            v = np.unpackbits(a, axis=1).reshape(rows, -1)[:, :sw * psp * bps].reshape(rows, sw * psp, bps)
            v = (v.astype(np.uint32) << np.arange(bps - 1, -1, -1, dtype=np.uint32)).sum(-1).reshape(rows, sw, psp)
        if pred == 2:
            v = np.cumsum(v.astype(np.int64), axis=1) % (1 << bps)
        full[pl, sy * sh:sy * sh + rows, sx * sw:(sx + 1) * sw] = v
    smp = np.concatenate(list(full), -1)[:H, :W] if planar == 2 else full[0, :H, :W]
    smp = smp.astype(np.int64)
    to8 = (lambda v: (v + 128) // 257) if bps == 16 else (lambda v: v)
    if ph == 3:
        cm = np.array(t.get(320, []), np.int64)
        if cm.size != 3 << bps:
            return None
        cm = cm.reshape(3, -1).T
        cm = cm >> 8 if (cm >= 256).any() else cm
        rgb = cm[smp[..., 0]]
    elif ph == 2 or planar == 2:
        c = [to8(smp[..., k]) for k in ((0, 1, 2) if ph == 2 else (0, 0, 0))]
        extra = t.get(338, [])
        if extra and extra[0] == 2:
            a = to8(smp[..., 3 if ph == 2 else 1])
            c = [(x * a + 127) // 255 for x in c]
        rgb = np.stack(c, -1)
    else:
        rng = 255 if bps == 16 else (1 << bps) - 1
        v = smp[..., 0] >> 8 if bps == 16 else smp[..., 0]
        v = ((rng - v) if ph == 0 else v) * 255 // rng
        rgb = np.stack([v] * 3, -1)
    gray = (GRAY[2] * rgb[..., 2] + GRAY[1] * rgb[..., 1] + GRAY[0] * rgb[..., 0] + 8192) >> 14
    o = g(274, 1)
    return rgb.astype(np.uint8), gray.astype(np.uint8), o if 1 <= o <= 8 else 1
