"""Seeded BMP / PNM corpus for the decoder tests: cv2- and Pillow-written files, and streams of a small hand encoder (BMP file + info
headers of every size cv2 reads, palettes, RLE4 / RLE8 with runs, absolute mode, delta, end-of-line and end-of-bitmap, bitfields,
top-down rows; PNM P1 - P6 with comments, odd separators and every maxval range), plus one crafted stream per corruption class.
Nothing is downloaded: every stream is generated here from a seed."""
import io
import struct

import numpy as np

try:
    import cv2
except ImportError:  # pragma: no cover
    cv2 = None
try:
    from PIL import Image
except ImportError:  # pragma: no cover
    Image = None

UNSUPPORTED, BAD_DATA = 2, 4


def image(h, w, seed, ch=3):
    """A smooth gradient plus noise, so that every colour conversion sees varied values."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([(x * 255 // max(w - 1, 1)), (y * 255 // max(h - 1, 1)), ((x + y) * 7) % 256], -1)[..., :ch]
    return np.clip(base + rng.integers(-20, 21, base.shape), 0, 255).astype(np.uint8)


# ---- BMP
def bmp(w, h, bpp, pixels, comp=0, palette=b"", header=40, clrused=0, masks=b"", offset=None,
        header_masks=(0xFF0000, 0xFF00, 0xFF, 0xFF000000)):
    """A BMP stream: 14-byte file header, info header of `header` bytes (12: OS/2 core header), masks, palette, pixel data.  h < 0 is
    top-down.  `palette` is the raw entry bytes (4 per entry, 3 for OS/2).  A header of more than 40 bytes holds `header_masks`
    (R, G, B, A)."""
    if header == 12:
        info = struct.pack("<IHHHH", 12, w, h, 1, bpp)
    else:
        info = struct.pack("<IiiHHIIiiII", header, w, h, 1, bpp, comp, len(pixels), 2835, 2835, clrused, 0)
        if header > 40:                           # V2 - V5: masks, colour space, ... (cv2 skips them)
            extra = struct.pack("<IIII", *header_masks) + b"sRGB"
            info += (extra + bytes(header))[:header - 40]
        info = info[:header]
    off = 14 + len(info) + len(masks) + len(palette) if offset is None else offset
    return b"BM" + struct.pack("<IHHi", (off + len(pixels)) & 0xFFFFFFFF, 0, 0, off) + info + masks + palette + pixels


def palette(n, seed, gray=False, entry=4):
    rng = np.random.default_rng(seed)
    c = rng.integers(0, 256, (n, 3)).astype(np.uint8)
    if gray:
        c[:, 1] = c[:, 2] = c[:, 0]
    return b"".join(bytes(e) + (b"\0" if entry == 4 else b"") for e in c)


def rows(a, bpp, top_down=False):
    """Pixel array of `a` (H x W indices for bpp <= 8; H x W uint16 for 16; H x W x 3 / 4 B, G, R(, A) bytes for 24 / 32), each row
    padded to 4 bytes, bottom row first unless top_down."""
    h, w = a.shape[:2]
    out = []
    for r in (range(h) if top_down else range(h - 1, -1, -1)):
        row = a[r]
        if bpp < 8:
            per = 8 // bpp
            v = np.zeros((w + per - 1) // per * per, np.uint8)
            v[:w] = row
            v = v.reshape(-1, per)
            b = np.zeros(len(v), np.uint8)
            for k in range(per):
                b |= (v[:, k] << (8 - bpp * (k + 1))).astype(np.uint8)
            data = b.tobytes()
        elif bpp == 16:
            data = row.astype("<u2").tobytes()
        else:
            data = row.astype(np.uint8).tobytes()
        out.append(data + b"\0" * (-len(data) % 4))
    return b"".join(out)


def rle(w, h, bits, seed, skips=True, eob=True):
    """RLE8 (bits 8) or RLE4 (bits 4) data for a w x h image, a random mix of runs, absolute runs (odd and even lengths), and with
    `skips`, end-of-line and delta codes.  The encoder tracks the position as cv2 reads it: an RLE8 run that fills its row moves to the
    next one, an RLE4 run does not; an RLE8 delta skips dx + dy * w pixels, an RLE4 delta dx pixels."""
    rng = np.random.default_rng(seed)
    top = 16 if bits == 4 else 256
    out = bytearray()
    x = y = 0
    while y < h:
        if x == w:                               # row full without a wrap: end of line
            out += b"\0\0"; x = 0; y += 1
            continue
        room = w - x
        k = int(rng.integers(0, 10 if skips else 6))
        if k < 3:                                # run
            n = int(rng.integers(1, min(room, 255) + 1))
            out += bytes([n, int(rng.integers(0, top)) if bits == 8 else int(rng.integers(0, 256))])
            x += n
            if bits == 8 and x == w:
                x = 0; y += 1
        elif k < 6 and room >= 3:                # absolute run
            n = int(rng.integers(3, min(room, 255) + 1))
            vals = rng.integers(0, top, n)
            if bits == 8:
                data = bytes(vals.astype(np.uint8)) + b"\0" * (n & 1)
            else:
                v = np.zeros(n + (n & 1), np.uint8); v[:n] = vals
                data = bytes((v[0::2] << 4) | v[1::2])
                data += b"\0" * (len(data) & 1)
            out += bytes([0, n]) + data
            x += n
        elif k < 8 and x > 0:                    # end of line
            out += b"\0\0"; x = 0; y += 1
        elif k < 10 and room > 1:                # delta
            dx = int(rng.integers(0, min(room - 1, 255) + 1))
            dy = int(rng.integers(0, 2)) if y + 1 < h else 0
            out += bytes([0, 2, dx, dy])
            x += dx
            if bits == 8:
                y += dy
    if eob:
        out += b"\0\1"
    return bytes(out)


def rle_bmp(w, h, bits, seed, **kw):
    return bmp(w, h, bits, rle(w, h, bits, seed, **kw), comp=1 if bits == 8 else 2, palette=palette(1 << bits, seed))


# ---- PNM
def pnm(kind, a, maxval=None, sep=b" ", row_sep=b"\n", header=None):
    """P1 - P6 of `a` (H x W, or H x W x 3 for P3 / P6; P1 / P4: 1 = black).  ASCII samples are joined by `sep`, rows by `row_sep`;
    `header` replaces the default 'Pk W H [maxval]\\n' header."""
    h, w = a.shape[:2]
    if header is None:
        header = b"P%d\n%d %d\n" % (kind, w, h) + (b"%d\n" % maxval if kind not in (1, 4) else b"")
    if kind == 1:
        return header + row_sep.join(sep.join(b"%d" % v for v in r) for r in a) + b"\n"
    if kind in (2, 3):
        return header + row_sep.join(sep.join(b"%d" % v for v in r.reshape(-1)) for r in a) + b"\n"
    if kind == 4:
        return header + b"".join(np.packbits(r.astype(np.uint8)).tobytes() for r in a)
    return header + a.astype(">u2" if maxval > 255 else np.uint8).tobytes()


def _cv2(ext, a, params=()):
    return cv2.imencode(ext, a, list(params))[1].tobytes()


def _pil(a, mode, fmt):
    buf = io.BytesIO()
    Image.fromarray(a).convert(mode).save(buf, format=fmt)
    return buf.getvalue()


def corpus():
    """[(name, stream)]: every stream decodes in cv2."""
    out = []
    for k, (h, w) in enumerate([(1, 1), (2, 3), (7, 5), (16, 16), (33, 17), (61, 97)]):
        bgr = image(h, w, k)
        out += [(f"cv2_bmp24_{h}x{w}", _cv2(".bmp", bgr)), (f"cv2_bmp8_{h}x{w}", _cv2(".bmp", bgr[..., 0])),
                (f"cv2_ppm_{h}x{w}", _cv2(".ppm", bgr)), (f"cv2_pgm_{h}x{w}", _cv2(".pgm", bgr[..., 1])),
                (f"cv2_pbm_{h}x{w}", _cv2(".pbm", bgr[..., 2])),
                (f"cv2_ppm_ascii_{h}x{w}", _cv2(".ppm", bgr, (cv2.IMWRITE_PXM_BINARY, 0))),
                (f"cv2_pgm_ascii_{h}x{w}", _cv2(".pgm", bgr[..., 1], (cv2.IMWRITE_PXM_BINARY, 0))),
                (f"cv2_pbm_ascii_{h}x{w}", _cv2(".pbm", bgr[..., 2], (cv2.IMWRITE_PXM_BINARY, 0))),
                (f"cv2_pgm16_{h}x{w}", _cv2(".pgm", (bgr[..., 0].astype(np.uint16) * 257 + k)))]
        if Image is not None:
            rgb = bgr[..., ::-1].copy()
            rgba = np.concatenate([rgb, image(h, w, k + 50, 1)], -1)
            out += [(f"pil_bmp1_{h}x{w}", _pil(rgb, "1", "BMP")), (f"pil_bmp8_{h}x{w}", _pil(rgb, "P", "BMP")),
                    (f"pil_bmp8l_{h}x{w}", _pil(rgb, "L", "BMP")), (f"pil_bmp24_{h}x{w}", _pil(rgb, "RGB", "BMP")),
                    (f"pil_bmp32_{h}x{w}", _pil(rgba, "RGBA", "BMP")), (f"pil_ppm_{h}x{w}", _pil(rgb, "RGB", "PPM")),
                    (f"pil_pgm_{h}x{w}", _pil(rgb, "L", "PPM")), (f"pil_pbm_{h}x{w}", _pil(rgb, "1", "PPM"))]
        # hand encoder: palettes, bitfields, headers, top-down, RLE
        idx8 = image(h, w, k + 1, 1)[..., 0]
        idx4, idx1 = idx8 >> 4, idx8 >> 7
        for td in (False, True):
            s = -h if td else h
            t = "td" if td else "bu"
            out += [(f"bmp1_{t}_{h}x{w}", bmp(w, s, 1, rows(idx1, 1, td), palette=palette(2, k))),
                    (f"bmp4_{t}_{h}x{w}", bmp(w, s, 4, rows(idx4, 4, td), palette=palette(16, k))),
                    (f"bmp8_{t}_{h}x{w}", bmp(w, s, 8, rows(idx8, 8, td), palette=palette(256, k))),
                    (f"bmp24_{t}_{h}x{w}", bmp(w, s, 24, rows(bgr, 24, td))),
                    (f"bmp32_{t}_{h}x{w}", bmp(w, s, 32, rows(np.concatenate([bgr, idx8[..., None]], -1), 32, td)))]
        v16 = image(h, w, k + 2, 2).astype(np.uint16)
        v16 = (v16[..., 0] << 8) | v16[..., 1]
        out += [(f"bmp16_555_rgb_{h}x{w}", bmp(w, h, 16, rows(v16 & 0x7FFF, 16))),
                (f"bmp16_555_bf_{h}x{w}", bmp(w, h, 16, rows(v16, 16), comp=3, masks=struct.pack("<III", 0x7C00, 0x3E0, 0x1F))),
                (f"bmp16_565_bf_{h}x{w}", bmp(w, -h, 16, rows(v16, 16, True), comp=3, masks=struct.pack("<III", 0xF800, 0x7E0, 0x1F))),
                (f"bmp32_bf_{h}x{w}", bmp(w, h, 32, rows(np.concatenate([bgr, idx8[..., None]], -1), 32), comp=3,
                                          masks=struct.pack("<III", 0xFF0000, 0xFF00, 0xFF))),
                (f"bmp32_bf_hdr56_{h}x{w}", bmp(w, h, 32, rows(np.concatenate([bgr, idx8[..., None]], -1), 32), comp=3, header=56)),
                (f"bmp32_bf_hdr108_{h}x{w}", bmp(w, -h, 32, rows(np.concatenate([bgr, idx8[..., None]], -1), 32, True), comp=3,
                                                 header=108, header_masks=(0xFF0000, 0xFF00, 0xFF, 0))),
                (f"bmp32_bf_hdr124_{h}x{w}", bmp(w, h, 32, rows(np.concatenate([bgr, idx8[..., None]], -1), 32), comp=3, header=124)),
                (f"bmp32_bf_hdr108_partial_{h}x{w}", bmp(w, h, 32, rows(np.concatenate([bgr, idx8[..., None]], -1), 32), comp=3,
                                                         header=108, header_masks=(0xFF, 0xFF00, 0, 0xFF000000))),
                (f"bmp8_clrused_{h}x{w}", bmp(w, h, 8, rows(idx8, 8), palette=palette(37, k), clrused=37)),
                (f"bmp8_graypal_{h}x{w}", bmp(w, h, 8, rows(idx8, 8), palette=palette(256, k, gray=True))),
                (f"bmp4_clrused_{h}x{w}", bmp(w, h, 4, rows(idx4, 4), palette=palette(5, k), clrused=5)),
                (f"os2_bmp8_{h}x{w}", bmp(w, h, 8, rows(idx8, 8), palette=palette(256, k, entry=3), header=12)),
                (f"os2_bmp1_{h}x{w}", bmp(w, h, 1, rows(idx1, 1), palette=palette(2, k, entry=3), header=12)),
                (f"os2_bmp24_{h}x{w}", bmp(w, h, 24, rows(bgr, 24), header=12))]
        for hs in (52, 56, 64, 108, 124):
            out.append((f"bmp24_hdr{hs}_{h}x{w}", bmp(w, h, 24, rows(bgr, 24), header=hs)))
        out.append((f"bmp8_hdr124_{h}x{w}", bmp(w, h, 8, rows(idx8, 8), header=124, palette=palette(256, k))))
        for j in range(3):
            out += [(f"rle8_{j}_{h}x{w}", rle_bmp(w, h, 8, 100 * k + j, skips=j > 0)),
                    (f"rle4_{j}_{h}x{w}", rle_bmp(w, h, 4, 100 * k + j + 50, skips=j > 0))]
        # PNM: maxval ranges, ASCII with comments and odd separators
        g8, c8 = bgr[..., 0], bgr
        out += [(f"p5_max100_{h}x{w}", pnm(5, g8 % 101, 100)), (f"p2_max100_{h}x{w}", pnm(2, g8, 100)),
                (f"p3_max255_{h}x{w}", pnm(3, c8.astype(np.int64) * 2, 255)),
                (f"p5_max1000_{h}x{w}", pnm(5, g8.astype(np.uint16) * 4, 1000)),
                (f"p2_max1000_{h}x{w}", pnm(2, g8.astype(np.int64) * 5, 1000, sep=b"\t", row_sep=b"\r\n")),
                (f"p6_max65535_{h}x{w}", pnm(6, c8.astype(np.uint16) * 257 + 3, 65535)),
                (f"p3_max4095_{h}x{w}", pnm(3, c8.astype(np.int64) * 16, 4095, sep=b" \n", row_sep=b"\n# row\n")),
                (f"p6_max7_{h}x{w}", pnm(6, c8 >> 5, 7)),
                (f"p1_nows_{h}x{w}", pnm(1, idx1, sep=b"", row_sep=b"\n")),
                (f"p4_{h}x{w}", pnm(4, idx1)),
                (f"p2_comments_{h}x{w}", pnm(2, g8, 255, sep=b" #c\n", header=b"P2 #a\n%d #b\n%d\n#c\r255\n" % (w, h)))]
    big = image(1080, 1920, 99)
    out += [("cv2_bmp24_1080p", _cv2(".bmp", big)), ("cv2_ppm_1080p", _cv2(".ppm", big)),
            ("rle8_1080p", rle_bmp(1920, 1080, 8, 7)), ("p2_gray_200x300", pnm(2, big[:200, :300, 0], 255))]
    # deltas past the image, end-of-bitmap on an early row
    out += [("rle8_delta_past_end", bmp(8, 4, 8, bytes([3, 5, 0, 2, 2, 9]), comp=1, palette=palette(256, 1))),
            ("rle8_early_eob", bmp(8, 4, 8, bytes([3, 5, 0, 1]), comp=1, palette=palette(256, 2))),
            ("rle4_eob_mid_rows", bmp(8, 3, 4, bytes([3, 0x5A, 0, 1, 8, 0x12, 0, 0, 2, 0x34, 0, 1]), comp=2, palette=palette(16, 3))),
            ("rle4_delta_dy_ignored", bmp(8, 2, 4, bytes([2, 0x11, 0, 2, 3, 1, 3, 0x22, 0, 0, 0, 3, 0x12, 0x30, 0, 1]), comp=2,
                                          palette=palette(16, 4)))]
    return out


def plan_corrupt():
    """[(name, stream, status)]: streams the plan set-up refuses, with the status it gives."""
    px = rows(image(4, 4, 1), 24)
    ok = bmp(4, 4, 24, px)
    return [
        ("bmp_truncated_header", ok[:30], BAD_DATA),
        ("bmp_info_size_16", ok[:14] + struct.pack("<I", 16) + ok[18:], BAD_DATA),
        ("bmp_info_size_0", ok[:14] + struct.pack("<I", 0) + ok[18:], BAD_DATA),
        ("bmp_2bit", bmp(4, 4, 2, bytes(16), palette=palette(4, 1)), UNSUPPORTED),
        ("bmp_rle24", bmp(4, 4, 24, bytes(16), comp=4), UNSUPPORTED),
        ("bmp_jpeg", bmp(4, 4, 0, b"\xff\xd8\xff\xd9", comp=4), UNSUPPORTED),
        ("bmp_png", bmp(4, 4, 0, b"\x89PNG\r\n\x1a\n", comp=5), UNSUPPORTED),
        ("bmp_alpha_bitfields", bmp(4, 4, 32, bytes(64), comp=6, masks=bytes(16)), UNSUPPORTED),
        ("bmp_rle8_with_4bit", bmp(4, 4, 4, b"\0\1", comp=1, palette=palette(16, 1)), UNSUPPORTED),
        ("bmp_bitfields_8bit", bmp(4, 4, 8, bytes(16), comp=3, palette=palette(256, 1)), UNSUPPORTED),
        ("bmp_16_masks_444", bmp(4, 4, 16, bytes(32), comp=3, masks=struct.pack("<III", 0xF00, 0xF0, 0xF)), UNSUPPORTED),
        ("bmp_16_masks_bgr565", bmp(4, 4, 16, bytes(32), comp=3, masks=struct.pack("<III", 0x1F, 0x7E0, 0xF800)), UNSUPPORTED),
        ("bmp_os2_16bit", bmp(4, 4, 16, bytes(32), header=12), UNSUPPORTED),
        ("bmp_clrused_300", bmp(4, 4, 8, bytes(16), palette=bytes(1200), clrused=300), BAD_DATA),
        ("bmp_palette_truncated", bmp(4, 4, 8, b"", palette=bytes(40)), BAD_DATA),
        ("bmp_zero_height", bmp(4, 0, 24, px), BAD_DATA),
        ("bmp_negative_width", bmp(-4, 4, 24, px), BAD_DATA),
        ("bmp_offset_past_end", bmp(4, 4, 24, px, offset=10000), BAD_DATA),
        ("bmp_negative_offset", bmp(4, 4, 24, px, offset=-5), BAD_DATA),
        ("bmp_pixels_truncated", ok[:-1], BAD_DATA),
        ("bmp_16_masks_truncated", bmp(4, 4, 16, b"", comp=3, masks=b"\0\xf8"), BAD_DATA),
        ("bmp_too_wide", bmp((1 << 20) + 1, 1, 8, b"", palette=palette(256, 1)), UNSUPPORTED),
        ("bmp_too_many_pixels", bmp(40000, 30000, 1, b"", palette=palette(2, 1)), UNSUPPORTED),
        ("bmp_color_limit", bmp(20000, 20000, 1, b"", palette=palette(2, 1)), UNSUPPORTED),
        ("pnm_maxval_70000", b"P5 1 1 70000\n\xff\xff", UNSUPPORTED),
        ("pnm_maxval_0", b"P5 1 1 0\n\x00", BAD_DATA),
        ("pnm_zero_width", b"P5 0 1 255\n\x00", BAD_DATA),
        ("pnm_bad_header_char", b"P5 1 x1 255\n\x00", BAD_DATA),
        ("pnm_width_overflow", b"P5 3000000000 1 255\n\x00", BAD_DATA),
        ("pnm_truncated_header", b"P6 4 4", BAD_DATA),
        ("pnm_p5_truncated", pnm(5, image(4, 4, 2)[..., 0], 255)[:-1], BAD_DATA),
        ("pnm_p6_16_truncated", pnm(6, image(4, 4, 2).astype(np.uint16) * 300, 65535)[:-1], BAD_DATA),
        ("pnm_p4_truncated", pnm(4, image(4, 9, 2)[..., 0] >> 7)[:-1], BAD_DATA),
        ("pnm_too_wide", b"P5 1048577 1 255\n" + bytes(16), UNSUPPORTED),
        ("pnm_too_many_pixels", b"P4 40000 30000\n" + bytes(16), UNSUPPORTED),
        ("bmp32_v4_masks_truncated", bmp(1, 1, 32, b"", comp=3, header=108, offset=54)[:62], BAD_DATA),
    ]


def refused_here_only():
    """[(name, stream, status)]: streams cv2 decodes and the plan set-up refuses (DESIGN section 2): 32-bit BITFIELDS in a V3 - V5
    header whose three colour masks are set but are not the standard 0xFF0000 / 0xFF00 / 0xFF (cv2's mask extraction is not
    restated)."""
    a = image(4, 5, 6, 3)
    px = rows(np.concatenate([a, a[..., :1]], -1), 32)
    return [("bmp32_v4_masks_swapped", bmp(5, 4, 32, px, comp=3, header=108, header_masks=(0xFF, 0xFF00, 0xFF0000, 0xFF000000)),
             UNSUPPORTED),
            ("bmp32_v3_masks_10bit", bmp(5, 4, 32, px, comp=3, header=56, header_masks=(0x3FF00000, 0xFFC00, 0x3FF, 0xC0000000)),
             UNSUPPORTED)]


def data_corrupt():
    """[(name, stream)]: streams that plan, and whose RLE or ASCII data the device stage refuses (sets the sample's status)."""
    pal = palette(256, 5)
    good = rle(6, 3, 8, 11)
    return [
        ("rle8_no_eob", bmp(6, 3, 8, bytes([6, 1, 6, 2]), comp=1, palette=pal)),
        ("rle8_truncated_mid_code", bmp(6, 3, 8, good[:-3], comp=1, palette=pal)),
        ("rle8_run_past_row", bmp(6, 3, 8, bytes([7, 1, 0, 1]), comp=1, palette=pal)),
        ("rle8_absolute_past_row", bmp(6, 3, 8, bytes([0, 8]) + bytes(8) + b"\0\1", comp=1, palette=pal)),
        ("rle8_absolute_truncated", bmp(6, 3, 8, bytes([0, 5, 1, 2]), comp=1, palette=pal)),
        ("rle8_delta_truncated", bmp(6, 3, 8, bytes([2, 1, 0, 2, 1]), comp=1, palette=pal)),
        ("rle8_run_after_full_absolute_row", bmp(6, 3, 8, bytes([0, 6, 1, 2, 3, 4, 5, 6, 2, 1, 0, 1]), comp=1, palette=pal)),
        ("rle4_no_eob", bmp(6, 3, 4, bytes([6, 0x12, 0, 0]), comp=2, palette=palette(16, 5))),
        ("rle4_run_past_row", bmp(6, 3, 4, bytes([7, 0x12, 0, 1]), comp=2, palette=palette(16, 5))),
        ("rle4_absolute_truncated", bmp(6, 3, 4, bytes([0, 5, 0x12]), comp=2, palette=palette(16, 5))),
        ("p2_bad_char", b"P2 2 1 255\n10 x20\n"),
        ("p2_ends_in_last_number", b"P2 2 1 255\n10 20"),
        ("p2_value_overflow", b"P2 2 1 255\n10 99999999999\n"),
        ("p3_truncated", b"P3 2 1 255\n1 2 3 4 5\n"),
        ("p1_truncated", b"P1 3 2\n1 0 1\n0 1\n"),
        ("p2_comment_to_eof", b"P2 2 1 255\n10 # no end"),
        ("p2_two_commas", b"P2 2 1 255\n10,,20\n"),
    ]


def kinds(s):
    """The variant tags of a stream, from its headers (what the corpus is checked to cover)."""
    tags = set()
    if s[:2] == b"BM":
        size = struct.unpack_from("<I", s, 14)[0]
        tags.add("os2" if size == 12 else f"hdr{size}")
        if size == 12:
            h, bpp, comp = struct.unpack_from("<H", s, 20)[0], struct.unpack_from("<H", s, 24)[0], 0
        else:
            h, bpp, comp = struct.unpack_from("<i", s, 22)[0], struct.unpack_from("<H", s, 28)[0], struct.unpack_from("<I", s, 30)[0]
            clrused = struct.unpack_from("<I", s, 46)[0]
            if bpp <= 8 and 0 < clrused < (1 << bpp):
                tags.add("clrused")
            if comp == 3 and bpp == 16:
                m = struct.unpack_from("<I", s, 14 + size + 4)[0]
                tags.add("bf565" if m == 0x7E0 else "bf555")
            if comp == 3 and bpp == 32 and size >= 56:
                m = struct.unpack_from("<III", s, 54)
                tags.add("bf32_header_masks" if all(m) else "bf32_header_partial_masks")
        tags.add(f"bmp{bpp}_c{comp}")
        tags.add("top_down" if h < 0 else "bottom_up")
        if comp in (1, 2):
            data = s[struct.unpack_from("<I", s, 10)[0]:]
            for i in range(0, len(data) - 1, 2):        # coarse: escape codes anywhere in the data
                if data[i] == 0 and data[i + 1] in (0, 2):
                    tags.add("rle_eol" if data[i + 1] == 0 else "rle_delta")
                if data[i] == 0 and data[i + 1] > 2 and data[i + 1] % 2:
                    tags.add("rle_odd_absolute")
    else:
        tags.add(s[:2].decode())
        if b"#" in s[:64]:
            tags.add("pnm_comment")
    return tags
