"""numpy restatement of the PNG decode of decoders.image, pinned bit-exactly against cv2.imdecode (OpenCV 4.13 / libpng) by
tests/test_png_cpu.py: chunk walk with CRC checks, zlib inflate, unfilter, then cv2's conversion rules:

  * 1/2/4-bit gray scales to 8 bits (v * 255 / (2^depth - 1)); a palette index reads PLTE, black past its end;
  * 16-bit samples keep their high byte (v >> 8); alpha is dropped without compositing;
  * IMREAD_GRAYSCALE of an 8-bit colour or palette pixel: (9797 R + 19234 G + 3737 B) >> 15, truncating;
  * IMREAD_GRAYSCALE of a 16-bit colour pixel: ((9797 R + 19234 G + 3737 B + 16384) >> 15) >> 8 on the 16-bit samples;
  * the stream must hold the whole image and run to its end; behind the image a malformed block or a bad Adler-32 fails,
    unless the stream holds more than the image needs.

decode(stream) -> (rgb HxWx3 uint8, gray HxW uint8, orientation), or None where cv2 rejects the stream."""
import struct
import zlib

import numpy as np

from png_streams import ADAM7, SPP

GRAY8 = (9797, 19234, 3737)


def _chunks(s):
    if s[:8] != b"\x89PNG\r\n\x1a\n":
        return None
    pos, out = 8, []
    while pos + 12 <= len(s):
        n = struct.unpack(">I", s[pos:pos + 4])[0]
        t, d = s[pos + 4:pos + 8], s[pos + 8:pos + 8 + n]
        if pos + 12 + n > len(s):
            return None
        ok = zlib.crc32(t + d) & 0xFFFFFFFF == struct.unpack(">I", s[pos + 8 + n:pos + 12 + n])[0]
        out.append((t, d, ok))
        pos += 12 + n
        if t == b"IEND":
            return out
    return None


def _exif_orientation(d):
    if len(d) < 8 or d[:2] not in (b"II", b"MM"):
        return 1
    e = "<" if d[:2] == b"II" else ">"
    ifd = struct.unpack(e + "I", d[4:8])[0]
    if ifd + 2 > len(d):
        return 1
    for k in range(struct.unpack(e + "H", d[ifd:ifd + 2])[0]):
        o = ifd + 2 + 12 * k
        if o + 12 > len(d):
            return 1
        if struct.unpack(e + "H", d[o:o + 2])[0] == 0x0112:
            v = struct.unpack(e + "H", d[o + 8:o + 10])[0]
            return v if 1 <= v <= 8 else 1
    return 1


def _inflate(z, need):
    """zlib fed byte by byte, as libpng sees it: the data running out before the stream's end fails; an error behind the image's
    last byte fails unless more than the image was produced (libpng then only drains the stream)"""
    d = zlib.decompressobj()
    out = b""
    for i in range(len(z)):
        try:
            out += d.decompress(z[i:i + 1])
        except zlib.error:
            return out[:need] if len(out) > need else None
        if d.eof:
            break
    if not d.eof or len(out) < need:
        return None
    return out[:need]


def _unfilter(buf, rows, rb, bpp):
    out = np.zeros((rows, rb - 1), np.uint8)
    prev = np.zeros(rb - 1, np.int64)
    for y in range(rows):
        f = buf[y * rb]
        c = np.frombuffer(buf[y * rb + 1:(y + 1) * rb], np.uint8).astype(np.int64).copy()
        if f > 4:
            return None
        if f == 2:
            c = (c + prev) & 255
        elif f in (1, 3, 4):
            for i in range(len(c)):
                a = c[i - bpp] if i >= bpp else 0
                ul = prev[i - bpp] if i >= bpp else 0
                if f == 1:
                    p = a
                elif f == 3:
                    p = (a + prev[i]) >> 1
                else:
                    pp = a + prev[i] - ul
                    pa, pb, pc = abs(pp - a), abs(pp - prev[i]), abs(pp - ul)
                    p = a if pa <= pb and pa <= pc else prev[i] if pb <= pc else ul
                c[i] = (c[i] + p) & 255
        out[y] = c
        prev = c
    return out


def _samples(rows, w, spp, depth):
    if depth == 16:
        return rows.view(">u2").reshape(rows.shape[0], -1)[:, :w * spp].reshape(rows.shape[0], w, spp).astype(np.int64)
    if depth == 8:
        return rows[:, :w * spp].reshape(rows.shape[0], w, spp).astype(np.int64)
    bits = np.unpackbits(rows, axis=1)[:, :w * depth].reshape(rows.shape[0], w, depth)
    return (bits.astype(np.int64) << np.arange(depth - 1, -1, -1)).sum(-1)[..., None]


def decode(stream):
    ch = _chunks(bytes(stream))
    if ch is None or ch[0][0] != b"IHDR" or not ch[0][2]:
        return None
    w, h, depth, ct, _, _, il = struct.unpack(">IIBBBBB", ch[0][1])
    if w > 1000000 or h > 1000000:
        return None                          # libpng's limit per side
    spp = SPP[ct]
    pal = np.zeros((256, 3), np.int64)
    idat, orientation, state = b"", 1, 0
    for t, d, ok in ch[1:]:
        if t == b"IDAT":
            if state == 2:
                return None
            state = 1
            if not ok:
                return None
            idat += d
            continue
        state = 2 if state == 1 else state
        if t == b"PLTE":
            if not ok:
                return None
            if ct == 3:
                pal[:len(d) // 3] = np.frombuffer(d[:len(d) // 3 * 3], np.uint8).reshape(-1, 3)
        elif t == b"eXIf" and ok:
            orientation = _exif_orientation(d)
        elif not t[0] & 0x20 and t not in (b"IEND",):
            return None
    passes = ADAM7 if il else [(0, 0, 1, 1)]
    geo = []
    for x0, y0, dx, dy in passes:
        pw, ph = max(0, (w - x0 + dx - 1) // dx), max(0, (h - y0 + dy - 1) // dy)
        geo.append((x0, y0, dx, dy, pw, ph, 1 + (pw * spp * depth + 7) // 8 if pw and ph else 0))
    need = sum(g[5] * g[6] for g in geo)
    raw = _inflate(idat, need)
    if raw is None:
        return None
    full = np.zeros((h, w, spp), np.int64)
    o = 0
    bpp = max(1, spp * depth // 8)
    for x0, y0, dx, dy, pw, ph, rb in geo:
        if not rb:
            continue
        rows = _unfilter(raw[o:o + ph * rb], ph, rb, bpp)
        if rows is None:
            return None
        full[y0::dy, x0::dx] = _samples(rows, pw, spp, depth)
        o += ph * rb
    if ct == 3:
        c = pal[full[..., 0]]
        rgb, gray = c, (GRAY8[0] * c[..., 0] + GRAY8[1] * c[..., 1] + GRAY8[2] * c[..., 2]) >> 15
    elif ct in (2, 6):
        c = full[..., :3]
        if depth == 16:
            rgb = c >> 8
            gray = ((GRAY8[0] * c[..., 0] + GRAY8[1] * c[..., 1] + GRAY8[2] * c[..., 2] + 16384) >> 15) >> 8
        else:
            rgb = c
            gray = (GRAY8[0] * c[..., 0] + GRAY8[1] * c[..., 1] + GRAY8[2] * c[..., 2]) >> 15
    else:
        g = full[..., 0]
        g = g >> 8 if depth == 16 else g * (255 // ((1 << depth) - 1)) if depth < 8 else g
        rgb, gray = np.stack([g] * 3, -1), g
    return rgb.astype(np.uint8), gray.astype(np.uint8), orientation


def orient(img, o):
    """EXIF orientation o applied to an (H, W[, C]) image, as cv2 and decoders.image(adjust_orientation=True) do"""
    if o in (5, 6, 7, 8):
        img = np.swapaxes(img, 0, 1)
    return {1: img, 2: img[:, ::-1], 3: img[::-1, ::-1], 4: img[::-1], 5: img, 6: img[:, ::-1], 7: img[::-1, ::-1],
            8: img[::-1]}[o]
