"""Seeded lossy WebP corpus for the tests: streams written by cv2 (qualities 1 to 100), by Pillow (methods 0-6, alpha, EXIF
orientations, an ICC profile) and by libwebp's advanced encoder API through ctypes (Pillow's bundled libwebp), which sweeps what cv2
and Pillow do not expose: segments, simple / normal loop filter, filter strength and sharpness, token partitions, spatial noise
shaping, sharp YUV.  Sizes from 1x1 to one 1080p image.  Plus one crafted stream per corruption class.

There is no VP8 decoder in numpy: cv2.imdecode is the oracle, used directly (decode())."""
import ctypes as C
import glob
import io
import os
import struct

import cv2
import numpy as np


def image(h, w, seed, noise=10.0):
    """a smooth random field plus noise, (h, w, 3) uint8 BGR"""
    rng = np.random.default_rng(seed)
    lo = rng.uniform(0, 255, (max(2, h // 16), max(2, w // 16), 3)).astype(np.float32)
    img = cv2.resize(lo, (w, h), interpolation=cv2.INTER_CUBIC) + rng.normal(0, noise, (h, w, 3))
    return np.clip(img, 0, 255).astype(np.uint8)


def cv2_webp(img, q):
    return cv2.imencode(".webp", img, [cv2.IMWRITE_WEBP_QUALITY, q])[1].tobytes()


def pil_webp(img_rgb, **kw):
    from PIL import Image
    b = io.BytesIO()
    Image.fromarray(img_rgb).save(b, "WEBP", **kw)
    return b.getvalue()


def exif_orientation(o):
    """a little-endian TIFF block holding one Orientation tag"""
    return b"II*\0" + struct.pack("<IHHHIHH", 8, 1, 0x0112, 3, 1, o, 0) + b"\0\0\0\0"


def decode(s, flags=cv2.IMREAD_COLOR):
    """cv2.imdecode of a stream (None when cv2 refuses it)"""
    return cv2.imdecode(np.frombuffer(s, np.uint8), flags)


# ---- libwebp's advanced encoder through ctypes ---------------------------------------------------------------------------------------
_LIB = None


def libwebp():
    """Pillow's bundled libwebp (libsharpyuv first, with RTLD_GLOBAL), or None"""
    global _LIB
    if _LIB is None:
        import PIL
        d = os.path.join(os.path.dirname(PIL.__file__), "..", "pillow.libs")
        sy, wp = glob.glob(os.path.join(d, "libsharpyuv-*")), glob.glob(os.path.join(d, "libwebp-*"))
        if not sy or not wp:
            _LIB = False
        else:
            C.CDLL(sy[0], mode=C.RTLD_GLOBAL)
            _LIB = C.CDLL(wp[0])
    return _LIB or None


# WebPConfig: every field is 4 bytes, in this order (src/webp/encode.h)
_CFG = ["lossless", "quality", "method", "image_hint", "target_size", "target_PSNR", "segments", "sns_strength", "filter_strength",
        "filter_sharpness", "filter_type", "autofilter", "alpha_compression", "alpha_filtering", "alpha_quality", "pass",
        "show_compressed", "preprocessing", "partitions", "partition_limit", "emulate_jpeg_size", "thread_level", "low_memory",
        "near_lossless", "exact", "use_delta_palette", "use_sharp_yuv"]
_FLOAT = {"quality", "target_PSNR"}


def libwebp_encode(img_bgr, quality=75.0, **settings):
    """WebPEncode with WebPConfig fields set by name (partitions: log2 of the count)"""
    lib = libwebp()
    cfg = (C.c_uint8 * 512)()
    assert lib.WebPConfigInitInternal(cfg, 0, C.c_float(quality), 0x0200)
    for k, v in settings.items():
        i = _CFG.index(k)
        struct.pack_into("<f" if k in _FLOAT else "<i", cfg, 4 * i, v)
    assert lib.WebPValidateConfig(cfg), settings
    pic = (C.c_uint8 * 1024)()
    assert lib.WebPPictureInitInternal(pic, 0x0200)
    h, w = img_bgr.shape[:2]
    struct.pack_into("<iiii", pic, 0, 0, 0, w, h)         # use_argb, colorspace (YUV420), width, height
    rgb = np.ascontiguousarray(img_bgr[..., ::-1])
    assert lib.WebPPictureImportRGB(pic, rgb.ctypes.data_as(C.c_void_p), w * 3)
    writer = (C.c_uint8 * 64)()
    lib.WebPMemoryWriterInit(writer)
    struct.pack_into("<QQ", pic, 96, C.cast(lib.WebPMemoryWrite, C.c_void_p).value, C.addressof(writer))   # writer, custom_ptr
    ok = lib.WebPEncode(cfg, pic)
    mem, size = struct.unpack_from("<QQ", writer, 0)
    out = C.string_at(mem, size) if ok else None
    lib.WebPPictureFree(pic)
    lib.WebPMemoryWriterClear(writer)
    assert ok, settings
    return out


# ---- the corpus ----------------------------------------------------------------------------------------------------------------------
SWEEP = ([dict(segments=s) for s in (1, 2, 3, 4)] +
         [dict(filter_type=t, filter_strength=fs) for t in (0, 1) for fs in (0, 100)] +
         [dict(filter_sharpness=k, filter_strength=60) for k in range(8)] +
         [dict(partitions=p, method=2) for p in (0, 1, 2, 3)] +
         [dict(sns_strength=v) for v in (0, 100)] +
         [dict(use_sharp_yuv=1), dict(segments=4, filter_type=0, filter_strength=40, partitions=3, method=1, quality=30.0),
          dict(autofilter=1, method=6)])


def corpus(big=False):
    """[(name, bytes)] of decodable streams"""
    out = []
    sizes = [(1, 1), (1, 37), (29, 1), (16, 16), (17, 33), (63, 80), (97, 131), (128, 200)]
    for k, (h, w) in enumerate(sizes):
        img = image(h, w, 10 + k, noise=[4.0, 25.0][k % 2])
        for q in (1, 10, 50, 75, 90, 100):
            out.append((f"cv2_{h}x{w}_q{q}", cv2_webp(img, q)))
    flat = np.full((256, 256, 3), (200, 120, 40), np.uint8)            # mostly skipped macroblocks: methods 0-2 code the skip
    flat[30:50, 40:70] = image(20, 30, 9, noise=40.0)                  # probability
    out += [(f"pil_flat_method{m}", pil_webp(flat, quality=50, method=m)) for m in (0, 2)]
    rgb = image(70, 90, 3)[..., ::-1]
    for m in range(7):
        out.append((f"pil_method{m}", pil_webp(rgb, quality=60, method=m)))
    rgba = np.dstack([rgb, (np.arange(70 * 90) % 251).reshape(70, 90).astype(np.uint8)])
    out.append(("pil_alpha", pil_webp(rgba, quality=80)))
    for o in range(1, 9):
        out.append((f"pil_exif{o}", pil_webp(image(37, 53, 70 + o)[..., ::-1], quality=70, exif=exif_orientation(o))))
    out.append(("pil_icc", pil_webp(rgb, quality=70, icc_profile=b"\0" * 64 + b"icc profile bytes")))
    if libwebp():
        img = image(96, 144, 5, noise=18.0)
        for s in SWEEP:
            s = dict(s)
            q = s.pop("quality", 75.0)
            name = "enc_" + "_".join(f"{k}{v}" for k, v in s.items())
            out.append((name, libwebp_encode(img, q, **s)))
    out += edge_decodable()
    if big:
        out.append(("cv2_1080p_q90", cv2_webp(image(1080, 1920, 99), 90)))
    return out


def simple_format(streams):
    """the [(name, bytes)] whose VP8 chunk holds the whole frame (the edge_ streams run past it): what tests/vp8_rewrite.py rewrites"""
    return [(n, s) for n, s in streams if s[8:16] == b"WEBPVP8 " and not n.startswith("edge_")]


def _opt(rng, p, draw):
    return draw() if rng.random() < p else None


def _i(rng, lo, hi):
    """an int in [lo, hi]"""
    return int(rng.integers(lo, hi + 1))


def _cycle_modes(f, v):
    """every macroblock's modes from its position and v: across v = 0..9 each 4x4 block takes every 4x4 mode, and across v = 0..3
    each macroblock every 16x16 and chroma mode"""
    for i, m in enumerate(f["mbs"]):
        y, x = divmod(i, f["mb_w"])
        m["uvmode"] = (v + x + 2 * y) % 4
        if m["i4"]:
            m["bmodes"] = [(v + 4 * x + (k & 3) + 3 * (4 * y + (k >> 2))) % 10 for k in range(16)]
        else:
            m["ymode"] = (v + 3 * x + y) % 4


def _random_modes(f, rng):
    for m in f["mbs"]:
        m["uvmode"] = _i(rng, 0, 3)
        if m["i4"]:
            m["bmodes"] = [_i(rng, 0, 9) for _ in range(16)]
        else:
            m["ymode"] = _i(rng, 0, 3)


def _segments(f, rng, q=None, strength=None, absolute=1, update_map=1, update_data=1, seg_proba=None):
    h = f["hdr"]
    h.update(use_segment=1, update_map=update_map, update_data=update_data, absolute_delta=absolute)
    h["quantizer"] = q if q is not None else [_opt(rng, 0.8, lambda: _i(rng, -127, 127)) for _ in range(4)]
    h["filter_strength"] = strength if strength is not None else [_opt(rng, 0.8, lambda: _i(rng, -63, 63)) for _ in range(4)]
    h["seg_proba"] = seg_proba if seg_proba is not None else [_opt(rng, 0.8, lambda: _i(rng, 1, 255)) for _ in range(3)]
    for m in f["mbs"]:
        m["segment"] = _i(rng, 0, 3) if update_map else 0


def rewritten(seed=0):
    """[(name, bytes, base)]: corpus streams (`base`) whose partition 0 tests/vp8_rewrite.py rewrote into header and mode values the
    encoders never write.  The name's first word is the family: segrel (relative segment deltas past both quantizer ends and the
    filter level's top), segnomap / segnodata (segmentation without a map or without data), segmap (random maps, each tree probability
    absent, 1 or 254), lfdelta (ref and mode filter deltas of both signs, unused deltas set, or no update), level0 (frame level 0 with
    segment strengths), level63 (every sharpness, both filters), quant (every quantizer delta at base index 0 and 127), q127 (cv2
    quality 90 / 100 streams at index 127), colorspace, modes (every mode at every edge position), skip (skip_p, use_skip 0 -> 1),
    scale (frame-tag scale bits, also inside VP8X) and mix (everything at random)."""
    import vp8_rewrite as vr
    rng = np.random.default_rng(seed)
    bases = dict(simple_format(corpus()))
    out = []

    def emit(name, f, base):
        out.append((name, vr.write(f), bases[base]))

    def frame(base):
        return vr.parse(bases[base])
    # both 16x16 and 4x4 macroblocks, sizes not multiples of 16
    mixed = ["cv2_63x80_q50", "cv2_97x131_q75", "cv2_128x200_q90", "pil_method4", "enc_segments4", "cv2_17x33_q100"]
    for k, b in enumerate(mixed):
        f = frame(b)
        h = f["hdr"]
        h["base_q0"], h["level"] = _i(rng, 20, 100), _i(rng, 20, 50)
        q0, lv = h["base_q0"], h["level"]
        _segments(f, rng, absolute=0,
                  q=[-(q0 + _i(rng, 1, 20)), 127 - q0 + _i(rng, 1, 20), _i(rng, -20, -1), None],
                  strength=[63 - lv + _i(rng, 1, 10), -(lv + _i(rng, 1, 10)), _i(rng, -10, -1), None])
        h["simple"] = k & 1
        emit(f"segrel_{b}", f, b)
        f = frame(b)
        _segments(f, rng, absolute=k & 1, update_map=0)
        f["hdr"]["level"] = _i(rng, 10, 40)
        emit(f"segnomap_{b}", f, b)
        f = frame(b)
        _segments(f, rng, update_data=0)
        f["hdr"]["level"] = _i(rng, 10, 40)
        f["hdr"].update(use_lf_delta=1, update_lf_delta=1, ref_lf_delta=[_i(rng, 5, 20), None, None, None],
                        mode_lf_delta=[_i(rng, 5, 20), None, None, None])
        emit(f"segnodata_{b}", f, b)
        for v in range(3):
            f = frame(b)
            _segments(f, rng, absolute=v & 1, seg_proba=[[None, 1, 254][(v + i) % 3] for i in range(3)])
            emit(f"segmap{v}_{b}", f, b)
        for v, (rs, ms) in enumerate([(1, 1), (1, -1), (-1, 1), (-1, -1)]):
            f = frame(b)
            h = f["hdr"]
            h.update(use_lf_delta=1, update_lf_delta=1, level=_i(rng, 15, 45), simple=(v + k) & 1, sharpness=_i(rng, 0, 7))
            h["ref_lf_delta"] = [rs * _i(rng, 4, 25)] + [_i(rng, -63, 63) for _ in range(3)]
            h["mode_lf_delta"] = [ms * _i(rng, 4, 25)] + [_i(rng, -63, 63) for _ in range(3)]
            if v == 3:
                _segments(f, rng)
            emit(f"lfdelta{v}_{b}", f, b)
        f = frame(b)
        f["hdr"].update(use_lf_delta=1, update_lf_delta=0, level=_i(rng, 15, 45))
        emit(f"lfdeltanoupdate_{b}", f, b)
        f = frame(b)
        _segments(f, rng, absolute=k & 1, strength=[_i(rng, 10, 63) for _ in range(4)])
        f["hdr"]["level"] = 0
        emit(f"level0_{b}", f, b)
        for ct in range(3):
            f = frame(b)
            f["hdr"]["color_space"], f["hdr"]["clamp_type"] = (ct + 1) & 1, (ct + 1) >> 1
            emit(f"colorspace{ct}_{b}", f, b)
    for sharp in range(8):
        for simple in (0, 1):
            b = mixed[(sharp + simple) % len(mixed)]
            f = frame(b)
            f["hdr"].update(level=63, sharpness=sharp, simple=simple)
            emit(f"level63_sharp{sharp}_simple{simple}_{b}", f, b)
    for d in range(5):
        for q0 in (0, 127):
            for sign in (-1, 1):
                b = mixed[(d + q0 + sign) % len(mixed)]
                f = frame(b)
                f["hdr"].update(use_segment=0, update_map=0, base_q0=q0)
                f["hdr"]["dq"] = [sign * _i(rng, 8, 15) if j == d else None for j in range(5)]
                emit(f"quant_dq{d}_q{q0}_{'neg' if sign < 0 else 'pos'}_{b}", f, b)
    for b in bases:
        if b.startswith("cv2_") and (b.endswith("_q90") or b.endswith("_q100")):
            f = frame(b)
            f["hdr"].update(use_segment=0, update_map=0, base_q0=127, dq=[None] * 5)
            emit(f"q127_{b}", f, b)
    for b in ("cv2_17x33_q100", "cv2_29x1_q90", "cv2_1x37_q90", "cv2_63x80_q10", "cv2_97x131_q100", "cv2_128x200_q50",
              "pil_method0", "pil_flat_method2"):
        for v in range(10):
            f = frame(b)
            _cycle_modes(f, v)
            emit(f"modes{v}_{b}", f, b)
    for b in bases:
        f = frame(b)
        h = f["hdr"]
        if h["use_skip"]:
            h["skip_p"] = [1, 254, _i(rng, 2, 253)][len(out) % 3]
            emit(f"skip_p_{b}", f, b)
        elif b.startswith("cv2_") or b.startswith("enc_"):
            h["use_skip"], h["skip_p"] = 1, _i(rng, 1, 255)
            emit(f"skip_on_{b}", f, b)
    for k, b in enumerate(["cv2_63x80_q75", "cv2_97x131_q50", "cv2_1x1_q90", "pil_method6"]):
        f = frame(b)
        _random_modes(f, rng)
        s = vr.set_scale_bits(vr.write(f), 1 + k % 3, 3 - k % 3)
        out.append((f"scale_{b}", s, bases[b]))
        out.append((f"scale_vp8x_{b}", vr.to_vp8x(s), bases[b]))
    names = sorted(bases)
    for k in range(40):
        b = names[_i(rng, 0, len(names) - 1)]
        f = frame(b)
        h = f["hdr"]
        if rng.random() < 0.6:
            _segments(f, rng, absolute=_i(rng, 0, 1), update_map=_i(rng, 0, 1), update_data=int(rng.random() < 0.85))
        if rng.random() < 0.6:
            h.update(use_lf_delta=1, update_lf_delta=int(rng.random() < 0.9))
            h["ref_lf_delta"] = [_opt(rng, 0.7, lambda: _i(rng, -63, 63)) for _ in range(4)]
            h["mode_lf_delta"] = [_opt(rng, 0.7, lambda: _i(rng, -63, 63)) for _ in range(4)]
        if rng.random() < 0.6:
            h["base_q0"] = _i(rng, 0, 127)
            h["dq"] = [_opt(rng, 0.7, lambda: _i(rng, -15, 15)) for _ in range(5)]
        h.update(simple=_i(rng, 0, 1), level=_i(rng, 0, 63), sharpness=_i(rng, 0, 7))
        _random_modes(f, rng)
        emit(f"mix{k}_{b}", f, b)
    return out


def _chunks(s):
    """[(tag, payload)] of the chunks of a well-formed stream"""
    out, pos = [], 12
    while pos + 8 <= len(s):
        n = struct.unpack_from("<I", s, pos + 4)[0]
        out.append((s[pos:pos + 4], s[pos + 8:pos + 8 + n]))
        pos += 8 + n + (n & 1)
    return out


def _set_p0(pay, p0):
    bits = (pay[0] | (pay[1] << 8) | (pay[2] << 16)) & 31 | (p0 << 5)
    return bytes([bits & 255, (bits >> 8) & 255, bits >> 16]) + bytes(pay[3:])


def edge_decodable():
    """[(name, bytes)]: streams whose VP8 data runs past the VP8 chunk, and which cv2 decodes: libwebp's VP8 decoder reads from the
    frame header to the end of the input, whatever the chunk and RIFF sizes say"""
    out = []
    img = image(64, 96, 4, noise=30.0)
    # VP8X with EXIF behind the frame (Pillow's layout), the VP8 payload cut, every size consistent: the last token partition runs
    # on into the EXIF chunk
    cs = _chunks(pil_webp(img[..., ::-1].copy(), quality=90, exif=exif_orientation(1)))
    for k in (5, 20):
        out.append((f"edge_vp8x_payload_cut{k}", _riff([_chunk(t, d[:len(d) - k] if t == b"VP8 " else d) for t, d in cs])))
    s = cv2_webp(img, 90)
    pay = _vp8_payload(s)
    p0 = (pay[0] | (pay[1] << 8) | (pay[2] << 16)) >> 5
    # the VP8 chunk cut to an even size, the rest of the payload behind the RIFF
    c = (len(pay) * 2 // 3) & ~1
    out.append(("edge_payload_behind_riff", _riff([_chunk(b"VP8 ", pay[:c])]) + pay[c:]))
    # the first partition runs past the chunk's end (but not past the chunk size, VP8GetInfo's check), into the bytes behind the RIFF
    c = (p0 + 2) & ~1
    out.append(("edge_p0_past_chunk", _riff([_chunk(b"VP8 ", pay[:c])]) + pay[c:]))
    # a token partition cut short, with zero bytes behind the RIFF: libwebp reads them as partition data
    out.append(("edge_partition_cut_zeros_behind", _partition_cut(s) + bytes(64)))
    return out


def orientation_cases():
    """[(name, bytes)]: VP8X streams with EXIF orientation 6 whose chunk structure varies; cv2 applies the orientation only when VP8X
    flags EXIF and every chunk inside the RIFF is complete"""
    s = pil_webp(image(37, 53, 7)[..., ::-1].copy(), quality=70, exif=exif_orientation(6))

    def fix(b):
        return b[:4] + struct.pack("<I", len(b) - 8) + b[8:]
    i = s.index(b"VP8 ")
    n = struct.unpack_from("<I", s, i + 4)[0]
    vp8 = s[i:i + 8 + n + (n & 1)]
    ex = s[s.index(b"EXIF"):]
    before = fix(s[:i] + ex + vp8)
    big = bytearray(s)
    struct.pack_into("<I", big, s.index(b"EXIF") + 4, 1 << 20)
    noflag = bytearray(s)
    noflag[20] &= ~0x08
    return [("exif_behind", s), ("exif_before_frame", before),
            ("exif_size_overruns_riff", bytes(big)),
            ("junk_chunk_overruns_riff", fix(s + b"XMP " + struct.pack("<I", 1 << 20) + b"ab")),
            ("partial_chunk_header", fix(s + b"XM")),
            ("complete_chunk_behind", fix(s + _chunk(b"XMP ", b"abc"))),
            ("bytes_behind_riff", s + b"XMP " + struct.pack("<I", 1 << 20)),
            ("exif_before_junk_behind", fix(before + b"XMP " + struct.pack("<I", 1 << 20))),
            ("exif_flag_clear", bytes(noflag)),
            ("two_exif_first_wins", fix(s + _chunk(b"EXIF", exif_orientation(3))))]


# ---- corruptions ---------------------------------------------------------------------------------------------------------------------
def _riff(chunks):
    body = b"WEBP" + b"".join(chunks)
    return b"RIFF" + struct.pack("<I", len(body)) + body


def _chunk(tag, data):
    return tag + struct.pack("<I", len(data)) + data + (b"\0" if len(data) & 1 else b"")


def _vp8_payload(s):
    """the payload of the VP8 chunk of a simple-format stream"""
    assert s[12:16] == b"VP8 "
    n = struct.unpack_from("<I", s, 16)[0]
    return s[20:20 + n]


def _partition_cut(s):
    """a stream whose last token partition is cut short, with every size field consistent"""
    pay = _vp8_payload(s)
    return _riff([_chunk(b"VP8 ", pay[:len(pay) - max(1, len(pay) // 8)])])


def _p0_cut(s):
    """partition 0 ends inside the macroblock headers (sizes consistent): its first-partition size is cut and the bytes behind it
    become token data"""
    pay = bytearray(_vp8_payload(s))
    bits = pay[0] | (pay[1] << 8) | (pay[2] << 16)
    p0 = bits >> 5
    nb = (bits & 31) | ((p0 * 2 // 3) << 5)
    pay[0:3] = bytes([nb & 255, (nb >> 8) & 255, nb >> 16])
    return _riff([_chunk(b"VP8 ", bytes(pay))])


def plan_corrupt():
    """[(name, bytes, status)]: streams that fail plan set-up (status: DALIB200_ERROR_BAD_DATA = 4 or UNSUPPORTED = 2, see
    include/dali_b200.h)"""
    s = cv2_webp(image(40, 56, 1), 80)
    pay = _vp8_payload(s)
    alpha = pil_webp(np.dstack([image(20, 30, 2), np.full((20, 30), 9, np.uint8)]), quality=70)
    out = [("truncated_10", s[:-10]), ("truncated_half", s[:len(s) // 2]), ("truncated_60", s[:60])]
    out.append(("bad_start_code", s[:23] + b"\x9d\x01\x2b" + s[26:]))
    b = bytearray(s); b[20] = (b[20] & ~0x0E) | (5 << 1); out.append(("profile_5", bytes(b)))
    b = bytearray(s); b[20] |= 1; out.append(("inter_frame", bytes(b)))
    vp8x = _chunk(b"VP8X", struct.pack("<I", 0) + (63).to_bytes(3, "little") + (39).to_bytes(3, "little"))
    out.append(("canvas_mismatch", _riff([vp8x, _chunk(b"VP8 ", pay)])))
    vp8x_ok = _chunk(b"VP8X", struct.pack("<I", 0) + (55).to_bytes(3, "little") + (39).to_bytes(3, "little"))
    over = _riff([vp8x_ok, b"XMP " + struct.pack("<I", 1 << 20) + b"abcd", _chunk(b"VP8 ", pay)])
    out.append(("chunk_overrun", over))
    b = bytearray(s); struct.pack_into("<I", b, 16, len(pay) + 1000); out.append(("vp8_chunk_overrun", bytes(b)))
    # VP8X: an odd-sized frame chunk ending at the RIFF's end without its padding byte (libwebp counts the padded size)
    odd = pay if len(pay) & 1 else pay + b"\0"
    s_odd = _riff([vp8x_ok, _chunk(b"VP8 ", odd)])[:-1]
    out.append(("odd_frame_chunk_unpadded", s_odd[:4] + struct.pack("<I", len(s_odd) - 8) + s_odd[8:]))
    out.append(("riff_too_small", s[:4] + struct.pack("<I", 8) + s[8:]))
    return [(n, x, 4) for n, x in out] + [
        ("vp8l", pil_webp(image(20, 30, 3)[..., ::-1], lossless=True), 2),
        ("animation_flag", alpha[:20] + bytes([alpha[20] | 0x02]) + alpha[21:], 2),
    ]


def data_corrupt():
    """[(name, bytes)]: streams whose headers plan but whose data is bad: the device sets the sample's status"""
    s = cv2_webp(image(64, 96, 4, noise=30.0), 90)
    return [("token_partition_cut", _partition_cut(s)), ("partition0_cut", _p0_cut(s))]


def alph_corrupt():
    """a stream whose ALPH data is corrupt: cv2 refuses it, the colour decode here does not read ALPH (DESIGN.md section 2)"""
    rgba = np.dstack([image(20, 30, 5)[..., ::-1], np.arange(600, dtype=np.uint8).reshape(20, 30)])
    s = bytearray(pil_webp(rgba, quality=70))
    i = s.index(b"ALPH")
    n = struct.unpack_from("<I", s, i + 4)[0]
    for k in range(i + 9, i + 8 + n):
        s[k] = 0xFF
    return bytes(s)
