"""Seeded WAV and FLAC streams for decoders.audio, written without the decoder's code.

The FLAC encoder follows RFC 9639 (frame header section 9.1, subframes 9.2, residual coding 9.2.7, metadata 8): every subframe type
(CONSTANT, VERBATIM, FIXED 0-4, LPC 1-32 with several precisions and shifts), Rice and Rice2 partitions with escape codes, partition
orders 0-8, the four channel assignments, wasted bits, fixed and variable block size, every block-size and sample-rate code, 8 / 16 / 24
bits, an ID3v2 tag and extra metadata blocks.  Its CRC-8 / CRC-16 are computed here from the polynomials.  A lossless stream defines its
samples uniquely, so the decode is checked against the samples the encoder was given.

WAV streams are written by the stdlib `wave` module (PCM) or by hand (IEEE float, WAVE_FORMAT_EXTENSIBLE); scipy.io.wavfile reads them
back independently.  refused() and corrupt() hold one stream per refusal and per corruption class.
"""
import io
import struct
import wave

import numpy as np

UNSUPPORTED, BAD_DATA = 2, 4


# ---------------------------------------------------------------------------------------------------------------- CRCs (RFC 9639 9.1.8, 9.3)
def _crc_table(poly, width):
    top, mask = 1 << (width - 1), (1 << width) - 1
    t = []
    for i in range(256):
        c = i << (width - 8)
        for _ in range(8):
            c = ((c << 1) ^ poly) & mask if c & top else (c << 1) & mask
        t.append(c)
    return t


_CRC8 = _crc_table(0x07, 8)
_CRC16 = np.array(_crc_table(0x8005, 16), np.uint32)


def crc8(b):
    c = 0
    for x in b:
        c = _CRC8[c ^ x]
    return c


def crc16_many(frames):
    """CRC-16 of each byte string, all at once: zero bytes in front do not change a CRC that starts at 0, so the frames are left-padded
    to one length and the table is applied column by column."""
    if not frames:
        return []
    m = max(len(f) for f in frames)
    a = np.zeros((len(frames), m), np.uint8)
    for i, f in enumerate(frames):
        a[i, m - len(f):] = np.frombuffer(f, np.uint8)
    c = np.zeros(len(frames), np.uint32)
    for j in range(m):
        c = ((c << 8) & 0xFFFF) ^ _CRC16[((c >> 8) ^ a[:, j]) & 0xFF]
    return [int(v) for v in c]


class Bits:
    def __init__(self):
        self.parts = []
        self.n = 0

    def put(self, v, n):
        if n:
            self.parts.append(format(v & ((1 << n) - 1), f"0{n}b"))
            self.n += n

    def sput(self, v, n):
        assert -(1 << (n - 1)) <= v < (1 << (n - 1)) if n else v == 0, (v, n)
        self.put(v, n)

    def unary(self, q):
        self.parts.append("0" * q + "1")
        self.n += q + 1

    def align(self):
        self.put(0, (-self.n) % 8)

    def bytes(self):
        s = "".join(self.parts)
        return int(s, 2).to_bytes(len(s) // 8, "big") if s else b""


def utf8_number(v):
    if v < 0x80:
        return bytes([v])
    for n in range(2, 8):
        if v < (1 << (5 * n + 1)) or n == 7:
            out = []
            for _ in range(n - 1):
                out.append(0x80 | (v & 0x3F))
                v >>= 6
            lead = (0xFF00 >> n) & 0xFF
            return bytes([lead | v] + out[::-1])


# ---------------------------------------------------------------------------------------------------------------- FLAC encoder
_RATE_CODES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}
_BS_CODES = {192: 1, 576: 2, 1152: 3, 2304: 4, 4608: 5, **{1 << k: k for k in range(8, 16)}}
_BITS_CODES = {8: 1, 16: 4, 24: 6}


def _rice_bits(u, k):
    return int(np.sum(u >> k)) + len(u) * (k + 1)


def _residual(bw, r, order, bs, method, porder, escape_parts=()):
    """residual section (RFC 9639 9.2.7): partition p of 2^porder holds bs >> porder samples, the first minus the predictor order"""
    bw.put(method, 2)
    bw.put(porder, 4)
    pbits, esc = (5, 31) if method else (4, 15)
    ps = bs >> porder
    pos = 0
    for p in range(1 << porder):
        cnt = ps - order if p == 0 else ps
        seg = np.asarray(r[pos:pos + cnt], np.int64)
        pos += cnt
        u = np.where(seg >= 0, 2 * seg, -2 * seg - 1)
        kmax = esc - 1
        if p in escape_parts or (len(u) and int(u.max()) >> kmax > 64):
            width = max([int(v).bit_length() + 1 for v in seg if v] or [0])
            assert width <= 31
            bw.put(esc, pbits)
            bw.put(width, 5)
            for v in seg:
                bw.sput(int(v), width)
            continue
        best = min(range(0, kmax + 1), key=lambda k: _rice_bits(u, k)) if len(u) else 0
        bw.put(best, pbits)
        for v in u:
            v = int(v)
            bw.unary(v >> best)
            bw.put(v & ((1 << best) - 1), best)
    assert pos == bs - order


def _lpc_coefs(x, order, precision, rng):
    """quantised predictor coefficients: a least-squares fit where the block allows one, else seeded values (any coefficients are
    lossless: the residual absorbs the prediction)"""
    x = np.asarray(x, np.float64)
    n = len(x)
    lim = (1 << (precision - 1)) - 1
    if n > 2 * order + 4:
        a = np.stack([x[order - 1 - i:n - 1 - i] for i in range(order)], 1)
        c, *_ = np.linalg.lstsq(a, x[order:], rcond=None)
    else:
        c = rng.uniform(-0.5, 0.5, order)
    m = float(np.max(np.abs(c))) or 1.0
    shift = int(np.clip(np.floor(np.log2(lim / m)), 0, 15))
    q = np.clip(np.round(c * (1 << shift)), -lim - 1, lim).astype(np.int64)
    return q, shift


def _predict(x, coefs, shift):
    order = len(coefs)
    pred = np.zeros(len(x) - order, np.int64)
    for i, c in enumerate(coefs):
        pred += int(c) * x[order - 1 - i:len(x) - 1 - i]
    return x[order:] - (pred >> shift if shift >= 0 else pred << -shift)


_FIXED = {0: [], 1: [1], 2: [2, -1], 3: [3, -3, 1], 4: [4, -6, 4, -1]}


def subframe(bw, x, sb, spec, rng):
    """one subframe of the int64 samples x (sb bits) by spec = (kind, params...) with optional 'wasted' / 'method' / 'porder' / 'escape'"""
    kind = spec["kind"]
    wasted = spec.get("wasted", 0)
    bw.put(0, 1)
    x = np.asarray(x, np.int64)
    if wasted:
        assert not np.any(x & ((1 << wasted) - 1))
        x = x >> wasted
        sb -= wasted
    code = {"constant": 0, "verbatim": 1}.get(kind)
    if kind == "fixed":
        code = 8 + spec["order"]
    elif kind == "lpc":
        code = 31 + spec["order"]
    bw.put(code, 6)
    if wasted:
        bw.put(1, 1)
        bw.unary(wasted - 1)
    else:
        bw.put(0, 1)
    if kind == "constant":
        assert np.all(x == x[0])
        bw.sput(int(x[0]), sb)
        return
    if kind == "verbatim":
        for v in x:
            bw.sput(int(v), sb)
        return
    order = spec["order"]
    for v in x[:order]:
        bw.sput(int(v), sb)
    if kind == "fixed":
        c = np.array(_FIXED[order], np.int64)
        r = _predict(x, c, 0) if order else x
    else:
        prec = spec.get("precision", 12)
        coefs, shift = _lpc_coefs(x, order, prec, rng)
        shift = spec.get("shift", shift)
        bw.put(prec - 1, 4)
        bw.sput(shift, 5)
        for c in coefs:
            bw.sput(int(c), prec)
        r = _predict(x, coefs, shift)
    _residual(bw, r, order, len(x), spec.get("method", 0), spec.get("porder", 0), spec.get("escape", ()))


def frame(x, bits, rate, number, variable, assign, specs, rng, bs_code=None, rate_code=None, bits_code=None):
    """one frame of the [bs, C] block x; returns its bytes (header, subframes, padding, CRC-16)"""
    bs, C = x.shape
    if bs_code is None:
        bs_code = _BS_CODES.get(bs, 6 if bs <= 256 else 7)
    if rate_code is None:
        rate_code = _RATE_CODES.get(rate, 0)
    if bits_code is None:
        bits_code = _BITS_CODES[bits]
    h = bytearray([0xFF, 0xF8 | int(variable), (bs_code << 4) | rate_code, (assign << 4) | (bits_code << 1)])
    h += utf8_number(number)
    if bs_code == 6:
        h.append(bs - 1)
    elif bs_code == 7:
        h += struct.pack(">H", bs - 1)
    if rate_code == 12:
        h.append(rate // 1000)
    elif rate_code == 13:
        h += struct.pack(">H", rate)
    elif rate_code == 14:
        h += struct.pack(">H", rate // 10)
    h.append(crc8(h))
    x = np.asarray(x, np.int64)
    chans = [x[:, c] for c in range(C)]
    if assign == 8:
        chans = [x[:, 0], x[:, 0] - x[:, 1]]
    elif assign == 9:
        chans = [x[:, 0] - x[:, 1], x[:, 1]]
    elif assign == 10:
        chans = [(x[:, 0] + x[:, 1]) >> 1, x[:, 0] - x[:, 1]]
    bw = Bits()
    for c, ch in enumerate(chans):
        side = (assign == 8 and c == 1) or (assign == 9 and c == 0) or (assign == 10 and c == 1)
        subframe(bw, ch, bits + side, specs[c], rng)
    bw.align()
    return bytes(h) + bw.bytes()


def streaminfo(min_bs, max_bs, rate, C, bits, total, min_fs=0, max_fs=0):
    v = (rate << 44) | ((C - 1) << 41) | ((bits - 1) << 36) | total
    return struct.pack(">HH", min_bs, max_bs) + min_fs.to_bytes(3, "big") + max_fs.to_bytes(3, "big") + v.to_bytes(8, "big") + bytes(16)


def meta_block(t, body, last):
    return bytes([(0x80 if last else 0) | t]) + len(body).to_bytes(3, "big") + body


def id3_tag(size=37):
    s = size
    return b"ID3\x04\x00\x00" + bytes([(s >> 21) & 127, (s >> 14) & 127, (s >> 7) & 127, s & 127]) + bytes(size)


def flac(x, bits, rate, blocks, *, variable=False, assign=None, spec=None, rng=None, id3=False, extra=False, si_min=None, si_max=None,
         total=None, codes=None, frames_out=None):
    """x: [T, C] int samples; blocks: the block sizes in order (sum = T); spec(frame index, channel, block) -> subframe spec; assign(frame
    index) -> channel assignment.  codes(frame index) -> (bs_code, rate_code, bits_code) overrides."""
    rng = rng or np.random.default_rng(0)
    x = np.asarray(x, np.int64)
    T, C = x.shape
    assert sum(blocks) == T
    raw = []
    pos = 0
    for k, bs in enumerate(blocks):
        blk = x[pos:pos + bs]
        a = assign(k) if assign else C - 1
        specs = [spec(k, c, blk) if spec else {"kind": "fixed", "order": 2} for c in range(C)]
        bc, rc, sc = codes(k) if codes else (None, None, None)
        raw.append(frame(blk, bits, rate, pos if variable else k, variable, a, specs, rng, bc, rc, sc))
        pos += bs
    crcs = crc16_many(raw)
    frames = [f + struct.pack(">H", c) for f, c in zip(raw, crcs)]
    if frames_out is not None:
        frames_out.extend(frames)
    body = blocks[:-1] or blocks
    mn = si_min if si_min is not None else max(16, min(body))
    mx = si_max if si_max is not None else max(blocks)
    out = b"fLaC"
    si = streaminfo(mn, mx, rate, C, bits, T if total is None else total)
    if extra:
        out += meta_block(0, si, False) + meta_block(4, b"\x05\x00\x00\x00test" + bytes(4), False) + meta_block(1, bytes(100), True)
    else:
        out += meta_block(0, si, True)
    out = out + b"".join(frames)
    return (id3_tag() if id3 else b"") + out


def signal(T, C, bits, rng, wasted=0, kind="music"):
    """seeded test signal [T, C] in the signed range of `bits` (low `wasted` bits zero)"""
    t = np.arange(T)[:, None]
    amp = (1 << (bits - 1)) - 1
    if kind == "music":
        f = rng.uniform(0.001, 0.05, (3, C))
        s = sum(np.sin(2 * np.pi * f[i] * t + rng.uniform(0, 6, C)) * rng.uniform(0.1, 0.3) for i in range(3))
        s = s + rng.normal(0, 0.02, (T, C))
    else:
        s = rng.uniform(-1, 1, (T, C))
    v = np.clip(np.round(s * amp), -amp - 1, amp).astype(np.int64)
    if wasted:
        v = (v >> wasted) << wasted
    return v


# ---------------------------------------------------------------------------------------------------------------- WAV
def wav_pcm(x, bits, rate):
    """PCM WAV through the stdlib writer; x: [T, C] signed ints of `bits` (8-bit: stored as u + 128)"""
    x = np.asarray(x, np.int64)
    T, C = x.shape
    if bits == 8:
        data = (x + 128).astype(np.uint8).tobytes()
    elif bits == 24:
        u = (x & 0xFFFFFF).astype(np.uint32)
        data = np.stack([u & 255, (u >> 8) & 255, (u >> 16) & 255], -1).astype(np.uint8).tobytes()
    else:
        data = x.astype({16: "<i2", 32: "<i4"}[bits]).tobytes()
    b = io.BytesIO()
    with wave.open(b, "wb") as w:
        w.setnchannels(C)
        w.setsampwidth(bits // 8)
        w.setframerate(rate)
        w.writeframes(data)
    return b.getvalue()


def wav_raw(fmt_body, data, extra_chunks=b"", data_size=None):
    """hand-written RIFF/WAVE: fmt chunk body, any chunks between fmt and data, the data chunk (size field overridable)"""
    def chunk(cid, body, size=None):
        return cid + struct.pack("<I", len(body) if size is None else size) + body + (b"\0" if len(body) & 1 else b"")
    body = b"WAVE" + chunk(b"fmt ", fmt_body) + extra_chunks + chunk(b"data", data, data_size)
    return b"RIFF" + struct.pack("<I", len(body)) + body


def fmt(tag, C, rate, bits, align=None):
    align = C * bits // 8 if align is None else align
    return struct.pack("<HHIIHH", tag, C, rate, rate * align, align, bits)


_GUID_TAIL = bytes([0x00, 0x00, 0x00, 0x00, 0x10, 0x00, 0x80, 0x00, 0x00, 0xAA, 0x00, 0x38, 0x9B, 0x71])


def fmt_ext(sub, C, rate, bits):
    return fmt(0xFFFE, C, rate, bits) + struct.pack("<HHI", 22, bits, (1 << C) - 1) + struct.pack("<H", sub) + _GUID_TAIL


def wav_float(xf, rate, extensible=False):
    xf = np.asarray(xf, np.float32)
    C = xf.shape[1]
    f = fmt_ext(3, C, rate, 32) if extensible else fmt(3, C, rate, 32)
    return wav_raw(f, xf.astype("<f4").tobytes())


# ---------------------------------------------------------------------------------------------------------------- corpus
def _spec_cycle(k, c, blk, rng):
    """a spread of subframe kinds over the frames and channels"""
    kinds = [{"kind": "verbatim"}] + [{"kind": "fixed", "order": o, "porder": p} for o, p in ((0, 0), (1, 2), (2, 3), (3, 1), (4, 4))] + \
        [{"kind": "lpc", "order": o, "precision": pr, "porder": p, "method": m}
         for o, pr, p, m in ((1, 5, 0, 0), (2, 8, 1, 1), (8, 12, 2, 0), (12, 15, 5, 1), (16, 14, 6, 0), (24, 13, 7, 1), (32, 15, 8, 0))]
    s = dict(kinds[(3 * k + c) % len(kinds)])
    bs = len(blk)
    while s.get("porder", 0) and (bs % (1 << s["porder"]) or (bs >> s["porder"]) < s.get("order", 0)):
        s["porder"] -= 1
    if s["kind"] in ("fixed", "lpc") and s["order"] > bs:
        s = {"kind": "verbatim"}
    if (k + c) % 5 == 4:
        s["escape"] = (0,)
    return s


def corpus():
    """[(name, stream bytes, expected int samples [T, C], bits, rate, format)]"""
    rng = np.random.default_rng(2024)
    out = []
    # FLAC: every subframe kind and partition setting across frames, fixed block sizes, every stereo mode
    for bits in (8, 16, 24):
        for C, assigns in ((1, [0]), (2, [1, 8, 9, 10]), (3, [2]), (6, [5]), (8, [7])):
            bs = {8: 192, 16: 576, 24: 1152}[bits]
            T = bs * 3 + 100
            x = signal(T, C, bits, rng)
            blocks = [bs] * 3 + [100]
            s = flac(x, bits, 44100 if C > 1 else 16000, blocks, assign=lambda k, a=assigns: a[k % len(a)],
                     spec=lambda k, c, blk: _spec_cycle(k, c, blk, rng), rng=rng)
            out.append((f"flac_b{bits}_c{C}", s, x, bits))
    # LPC orders 1..32, precisions 2..15, Rice2 and partition orders across them
    x = signal(32 * 256, 1, 16, rng)
    s = flac(x, 16, 16000, [256] * 32, spec=lambda k, c, blk: {"kind": "lpc", "order": k + 1, "precision": 2 + k % 14, "method": k % 2,
                                                               "porder": k % 4})
    out.append(("flac_lpc_orders", s, x, 16))
    # the highest partition orders
    x = signal(2 * 4096, 1, 16, rng)
    s = flac(x, 16, 16000, [4096] * 2, spec=lambda k, c, blk: {"kind": "fixed", "order": 2, "porder": 7 + k, "method": k, "escape": (3,)})
    out.append(("flac_partitions", s, x, 16))
    # constant subframes and wasted bits
    x = signal(1024, 2, 16, rng, wasted=3)
    x[:300, 1] = 40
    s = flac(x, 16, 48000, [256, 256, 512], variable=True, assign=lambda k: 1,
             spec=lambda k, c, blk: {"kind": "constant"} if np.all(blk[:, c] == blk[0, c]) else
             {"kind": ["fixed", "lpc", "verbatim"][k % 3], "order": 2, "wasted": 3})
    out.append(("flac_wasted_constant", s, x, 16))
    # variable block size, every block-size code, ID3v2 and extra metadata
    blocks = [192, 576, 1152, 2304, 4608, 256, 512, 1024, 2048, 4096, 8192, 16384, 32768, 17, 200, 300, 1000, 4000, 65535 - 1, 53]
    T = sum(blocks)
    x = signal(T, 1, 16, rng)
    s = flac(x, 16, 22050, blocks, variable=True, spec=lambda k, c, blk: {"kind": "fixed", "order": 2, "porder": 0},
             codes=lambda k: (6 if blocks[k] <= 256 and blocks[k] in (17, 200) else None, None, None), id3=True, extra=True, si_min=16)
    out.append(("flac_variable_codes", s, x, 16))
    # every sample-rate code (the header's own rate, or 0 = STREAMINFO's), bits code 0
    for rate, rc in ((88200, 1), (176400, 2), (192000, 3), (8000, 4), (16000, 5), (22050, 6), (24000, 7), (32000, 8), (44100, 9),
                     (48000, 10), (96000, 11), (37000, 12), (12345, 13), (101230, 14), (44100, 0)):
        x = signal(600, 1, 8, rng)
        s = flac(x, 8, rate, [300, 300], codes=lambda k, r=rc: (None, r, 0 if k else None),
                 spec=lambda k, c, blk: {"kind": "lpc", "order": 3, "precision": 9, "shift": 7 + k})
        out.append((f"flac_rate_{rate}_{rc}", s, x, 8))
    # WAV: PCM 8 / 16 / 24 / 32 through `wave`, float and EXTENSIBLE by hand
    for bits in (8, 16, 24, 32):
        for C in (1, 2, 5):
            x = signal(777, C, bits, rng, kind="noise")
            out.append((f"wav_pcm{bits}_c{C}", wav_pcm(x, bits, 16000), x, bits))
    x = signal(500, 3, 24, rng)
    out.append(("wav_ext_pcm24", wav_raw(fmt_ext(1, 3, 44100, 24), wav_pcm(x, 24, 44100)[44:], extra_chunks=b"LIST\x03\x00\x00\x00abc\x00"), x, 24))
    xf = rng.uniform(-1.5, 1.5, (400, 2)).astype(np.float32)
    out.append(("wav_float", wav_float(xf, 48000), xf, 32))
    out.append(("wav_ext_float", wav_float(xf, 48000, extensible=True), xf, 32))
    return out


def refused():
    """[(name, stream, code, why)]"""
    rng = np.random.default_rng(7)
    x = signal(400, 2, 16, rng)
    good = flac(x, 16, 16000, [200, 200])
    si_off = 8                                  # STREAMINFO body inside `good`
    def patch_si(fn):
        si = bytearray(good[si_off:si_off + 34])
        fn(si)
        return good[:si_off] + bytes(si) + good[si_off + 34:]
    def set_bits(si, b):
        si[12] = (si[12] & 0xFE) | ((b - 1) >> 4)
        si[13] = (si[13] & 0x0F) | (((b - 1) & 15) << 4)
    pcm16 = wav_pcm(x, 16, 16000)
    out = [
        ("ogg", b"OggS" + bytes(60), UNSUPPORTED, "Ogg container"),
        ("garbage", bytes(range(64)), UNSUPPORTED, "neither WAV nor FLAC"),
        ("wav_adpcm", wav_raw(fmt(2, 1, 8000, 4, align=1), bytes(100)), UNSUPPORTED, "ADPCM"),
        ("wav_mulaw", wav_raw(fmt(7, 1, 8000, 8), bytes(100)), UNSUPPORTED, "mu-law"),
        ("wav_alaw", wav_raw(fmt(6, 1, 8000, 8), bytes(100)), UNSUPPORTED, "A-law"),
        ("wav_float64", wav_raw(fmt(3, 1, 8000, 64), bytes(80)), UNSUPPORTED, "float64"),
        ("wav_pcm12", wav_raw(fmt(1, 1, 8000, 12, align=2), bytes(80)), UNSUPPORTED, "12-bit PCM"),
        ("wav_ext_unknown", wav_raw(fmt_ext(2, 1, 8000, 16)[:24] + b"\x07\x00" + bytes(14), bytes(80)), UNSUPPORTED, "unknown sub-format"),
        ("wav_9ch", wav_raw(fmt(1, 9, 8000, 16), bytes(18 * 10)), UNSUPPORTED, "9 channels"),
        ("flac_12bit", patch_si(lambda si: set_bits(si, 12)), UNSUPPORTED, "12-bit FLAC"),
        ("flac_20bit", patch_si(lambda si: set_bits(si, 20)), UNSUPPORTED, "20-bit FLAC"),
        ("flac_unknown_total", patch_si(lambda si: si.__setitem__(slice(13, 18), bytes([si[13] & 0xF0, 0, 0, 0, 0]))), UNSUPPORTED, "total 0"),
        ("ogg_flac", b"OggS\x00\x02" + bytes(20) + b"\x7fFLAC" + good[4:], UNSUPPORTED, "Ogg FLAC"),
        ("wav_truncated_riff", b"RIFF\x10\x00\x00\x00WAV", BAD_DATA, "truncated RIFF"),
        ("wav_truncated_fmt", wav_raw(fmt(1, 1, 8000, 16), b"")[:30], BAD_DATA, "truncated fmt"),
        ("wav_bad_align", wav_raw(fmt(1, 2, 8000, 16, align=3), bytes(60)), BAD_DATA, "block_align != C * bytes"),
        ("wav_no_data", pcm16[:36], BAD_DATA, "no data chunk"),
        ("wav_rate0", wav_raw(fmt(1, 1, 0, 16), bytes(20)), BAD_DATA, "sample rate 0"),
        ("wav_0ch", wav_raw(fmt(1, 0, 8000, 16, align=0), bytes(20)), BAD_DATA, "0 channels"),
        ("flac_no_streaminfo", b"fLaC" + meta_block(4, bytes(8), False) + good[4:], BAD_DATA, "STREAMINFO not first"),
        ("flac_truncated_meta", good[:20], BAD_DATA, "truncated STREAMINFO"),
        ("flac_small_block", patch_si(lambda si: si.__setitem__(slice(0, 4), b"\x00\x08\x00\x08")), BAD_DATA, "block size < 16"),
        ("flac_rate0", patch_si(lambda si: si.__setitem__(slice(10, 13), bytes([0, 0, si[12] & 0x0F]))), BAD_DATA, "sample rate 0"),
    ]
    return out


def corrupt():
    """[(name, stream)] whose headers plan but whose frames are damaged: the sample's status must be set"""
    rng = np.random.default_rng(11)
    x = signal(2000, 2, 16, rng)
    blocks = [512, 512, 512, 464]
    frames = []
    good = flac(x, 16, 16000, blocks, assign=lambda k: 10, spec=lambda k, c, blk: {"kind": "lpc", "order": 4, "precision": 12}, frames_out=frames)
    head = good[:len(good) - sum(len(f) for f in frames)]

    def join(fs):
        return head + b"".join(fs)

    def flip(f, i, bit=0x10):
        b = bytearray(f)
        b[i] ^= bit
        return bytes(b)

    def with_crc(body):
        return body + struct.pack(">H", crc16_many([body])[0])

    out = [
        ("bad_crc8", join([frames[0], flip(frames[1], 4), frames[2], frames[3]])),
        ("bad_crc16", join([frames[0], frames[1], flip(frames[2], len(frames[2]) - 1, 1), frames[3]])),
        ("bad_data_bit", join([frames[0], flip(frames[1], 40, 0x04), frames[2], frames[3]])),
        ("missing_frame", join([frames[0], frames[2], frames[3]])),
        ("extra_frame", join(frames + [frames[3]])),
        ("truncated", join(frames)[:-100]),
        ("short_total", join(frames[:3])),
    ]
    # sample numbers that do not add up: STREAMINFO claims more samples than the frames hold
    out.append(("total_mismatch", flac(x, 16, 16000, blocks, total=2500)))
    # reserved subframe type, residual method, LPC precision; negative shift; order above the block / partition
    def bad_sub(spec_fn, patch):
        y = signal(256, 1, 16, rng)
        fs = []
        flac(y, 16, 16000, [256], spec=spec_fn, frames_out=fs)
        h = bytearray(fs[0][:-2])
        patch(h)
        s = flac(y, 16, 16000, [256], spec=spec_fn)
        return s[:len(s) - len(fs[0])] + with_crc(bytes(h))
    hl = 6                                              # header bytes of these one-frame streams (number 0, codes in table)
    out += [
        ("reserved_subframe_type", bad_sub(lambda k, c, b: {"kind": "verbatim"}, lambda h: h.__setitem__(hl, 0x04))),   # type 000010
        ("reserved_residual_method", bad_sub(lambda k, c, b: {"kind": "fixed", "order": 0}, lambda h: h.__setitem__(hl + 1, h[hl + 1] | 0x80))),
        ("reserved_lpc_precision", bad_sub(lambda k, c, b: {"kind": "lpc", "order": 1, "precision": 8},
                                           lambda h: h.__setitem__(hl + 3, h[hl + 3] | 0xF0))),
        ("negative_lpc_shift", bad_sub(lambda k, c, b: {"kind": "lpc", "order": 1, "precision": 8, "shift": -3}, lambda h: None)),
        ("order_above_partition", bad_sub(lambda k, c, b: {"kind": "fixed", "order": 4, "porder": 0},
                                          lambda h: h.__setitem__(hl + 9, (h[hl + 9] & 0xC3) | (8 << 2)))),
    ]
    return out
