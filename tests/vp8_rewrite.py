"""A partition-0 rewriter for VP8 key frames (lossy WebP, simple format): parse() reads the frame header and every macroblock's segment
id, skip flag and intra modes in libwebp's order (src/dec/vp8_dec.c VP8GetHeaders, tree_dec.c ParseIntraMode; RFC 6386 sections 9,
11, 13 and 19.2); write() writes partition 0 back with any edits and keeps the partition-size table and the token partitions byte for
byte.

Token parsing depends only on the coefficient probabilities, each macroblock's skip flag and i4 flag (whether a Y2 block exists) and
the non-zero contexts.  So every header field may change except the partition count, the probability updates and use_skip; so may
the segment ids, skip_p, the 16x16 mode among its 4, each 4x4 mode among its 10 and the chroma mode among its 4.  write() refuses
edits outside that set.  use_skip may go from 0 to 1 when every skip flag is written as 0.

Modes use libwebp's numbering: DC 0, TM 1, VE 2, HE 3 (the 16x16 and chroma modes), then RD, VR, LD, VL, HD, HU.  The 4x4 mode
probabilities and the coefficient-update probabilities are read from the product's headers; a wrong entry there would show as a
stream cv2 decodes differently after a round trip (tests/test_webp_rewrite_cpu.py)."""
import os
import re
import struct

import numpy as np

_CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "dali_b200", "csrc")


def _table(header, name, n):
    """the first n integers of the initialiser of C array `name` in one of the product's headers"""
    with open(os.path.join(_CSRC, header)) as fh:
        text = fh.read()
    i = j = text.index("{", text.index(name))
    depth = 0
    while True:                                # to the brace that closes the initialiser
        depth += {"{": 1, "}": -1}.get(text[j], 0)
        if depth == 0:
            break
        j += 1
    vals = [int(v) for v in re.findall(r"\d+", text[i:j])]
    assert len(vals) == n, (header, name, len(vals))
    return vals


BMODES_PROBA = np.array(_table("webp_core.h", "webp_bmodes_proba[10][10][9]", 900)).reshape(10, 10, 9)   # [top][left][node]
COEFF_UPDATE_PROBA = _table("webp_plan.h", "kWebpCoeffsUpdateProba[4][8][3][11]", 1056)
# libwebp kYModesIntra4: node i reads probability i; a value <= 0 is the leaf -mode
_YMODES4_TREE = [0, 1, -1, 2, -2, 3, 4, 6, -3, 5, -4, -5, -6, 7, -7, 8, -8, -9]
# the 16x16 modes as (probability, bit) paths: 156 ? (128 ? TM : HE) : (163 ? VE : DC)
_YMODE16_PATH = {0: [(156, 0), (163, 0)], 2: [(156, 0), (163, 1)], 3: [(156, 1), (128, 0)], 1: [(156, 1), (128, 1)]}
# the chroma modes: 142 ? (114 ? (183 ? TM : HE) : VE) : DC
_UVMODE_PATH = {0: [(142, 0)], 2: [(142, 1), (114, 0)], 1: [(142, 1), (114, 1), (183, 1)], 3: [(142, 1), (114, 1), (183, 0)]}


def _ymode4_paths():
    paths = {}

    def walk(node, path):
        for bit in (0, 1):
            nxt = _YMODES4_TREE[2 * node + bit]
            step = path + [(node, bit)]
            if nxt > 0:
                walk(nxt, step)
            else:
                paths[-nxt] = step
    walk(0, [])
    assert sorted(paths) == list(range(10))
    return paths


_YMODE4_PATH = _ymode4_paths()


class BoolDecoder:
    """RFC 6386 section 7.3; past the end of the data it reads zero bytes and counts them in `overrun`"""

    def __init__(self, data):
        self.data, self.pos, self.overrun = data, 2, 0
        self.value = ((data[0] if data else 0) << 8) | (data[1] if len(data) > 1 else 0)
        self.range, self.count = 255, 0

    def bit(self, prob):
        split = 1 + (((self.range - 1) * prob) >> 8)
        big = split << 8
        if self.value >= big:
            bit, self.range, self.value = 1, self.range - split, self.value - big
        else:
            bit, self.range = 0, split
        while self.range < 128:
            self.value <<= 1
            self.range <<= 1
            self.count += 1
            if self.count == 8:
                self.count = 0
                if self.pos < len(self.data):
                    self.value |= self.data[self.pos]
                else:
                    self.overrun += 1
                self.pos += 1
        return bit

    def literal(self, n):
        v = 0
        for _ in range(n):
            v = (v << 1) | self.bit(128)
        return v

    def signed(self, n):                       # libwebp VP8GetSignedValue: magnitude, then sign
        v = self.literal(n)
        return -v if self.bit(128) else v

    def optional(self, read):                  # a flag bit, then the value when it is set; None when it is not
        return read() if self.bit(128) else None


class BoolEncoder:
    """RFC 6386 section 7.3, with the carry into bytes already written"""

    def __init__(self):
        self.out, self.low, self.range, self.count = bytearray(), 0, 255, 24
        self.carries = 0                       # carries into bytes already written, and how many of them crossed a 0xFF byte
        self.long_carries = 0

    def bit(self, prob, bit):
        split = 1 + (((self.range - 1) * prob) >> 8)
        if bit:
            self.low += split
            self.range -= split
        else:
            self.range = split
        while self.range < 128:
            self.range <<= 1
            if self.low & (1 << 31):
                k = len(self.out) - 1
                self.carries += 1
                self.long_carries += self.out[k] == 255
                while self.out[k] == 255:
                    self.out[k] = 0
                    k -= 1
                self.out[k] += 1
            self.low = (self.low << 1) & 0xFFFFFFFF
            self.count -= 1
            if self.count == 0:
                self.out.append(self.low >> 24)
                self.low &= 0xFFFFFF
                self.count = 8

    def literal(self, v, n):
        for i in range(n - 1, -1, -1):
            self.bit(128, (v >> i) & 1)

    def signed(self, v, n):
        self.literal(abs(v), n)
        self.bit(128, int(v < 0))

    def optional(self, v, write):
        self.bit(128, int(v is not None))
        if v is not None:
            write(v)

    def finish(self):
        """32 zero bits at probability 1/2 push every pending bit out and leave padding behind the last one, so that a decoder never
        reads past the partition's end (libwebp fails such a stream: "Premature end-of-partition0")"""
        for _ in range(32):
            self.bit(128, 0)
        return bytes(self.out)


def vp8_payload(stream):
    assert stream[:4] == b"RIFF" and stream[8:16] == b"WEBPVP8 ", "simple-format lossy WebP expected"
    return stream[20:20 + struct.unpack_from("<I", stream, 16)[0]]


def parse(stream):
    """the frame of a simple-format lossy WebP stream: a dict with the payload, sizes, `hdr` (the frame header, optional fields None
    when absent) and `mbs` (per macroblock: segment, skip, i4, ymode or bmodes[16], uvmode)"""
    pay = vp8_payload(stream)
    p0 = (pay[0] | pay[1] << 8 | pay[2] << 16) >> 5
    W, H = (pay[6] | pay[7] << 8) & 0x3FFF, (pay[8] | pay[9] << 8) & 0x3FFF
    r = BoolDecoder(pay[10:10 + p0])
    h = dict(color_space=r.bit(128), clamp_type=r.bit(128), use_segment=r.bit(128), update_map=0, update_data=0, absolute_delta=1,
             quantizer=[None] * 4, filter_strength=[None] * 4, seg_proba=[None] * 3)
    if h["use_segment"]:
        h["update_map"], h["update_data"] = r.bit(128), r.bit(128)
        if h["update_data"]:
            h["absolute_delta"] = r.bit(128)
            h["quantizer"] = [r.optional(lambda: r.signed(7)) for _ in range(4)]
            h["filter_strength"] = [r.optional(lambda: r.signed(6)) for _ in range(4)]
        if h["update_map"]:
            h["seg_proba"] = [r.optional(lambda: r.literal(8)) for _ in range(3)]
    h["simple"], h["level"], h["sharpness"] = r.bit(128), r.literal(6), r.literal(3)
    h["use_lf_delta"], h["update_lf_delta"] = r.bit(128), 0
    h["ref_lf_delta"], h["mode_lf_delta"] = [None] * 4, [None] * 4
    if h["use_lf_delta"]:
        h["update_lf_delta"] = r.bit(128)
        if h["update_lf_delta"]:
            h["ref_lf_delta"] = [r.optional(lambda: r.signed(6)) for _ in range(4)]
            h["mode_lf_delta"] = [r.optional(lambda: r.signed(6)) for _ in range(4)]
    h["log2_parts"], h["base_q0"] = r.literal(2), r.literal(7)
    h["dq"] = [r.optional(lambda: r.signed(4)) for _ in range(5)]          # Y1 DC, Y2 DC, Y2 AC, UV DC, UV AC
    h["refresh"] = r.bit(128)
    h["proba"] = [r.literal(8) if r.bit(p) else None for p in COEFF_UPDATE_PROBA]
    h["use_skip"] = r.bit(128)
    h["skip_p"] = r.literal(8) if h["use_skip"] else None
    mb_w, mb_h = (W + 15) >> 4, (H + 15) >> 4
    sp = [255 if v is None else v for v in h["seg_proba"]]
    mbs, top = [], [[0] * 4 for _ in range(mb_w)]
    for _ in range(mb_h):
        left = [0] * 4
        for x in range(mb_w):
            m = dict(segment=0, skip=0)
            if h["update_map"]:
                m["segment"] = r.bit(sp[1]) if not r.bit(sp[0]) else 2 + r.bit(sp[2])
            if h["use_skip"]:
                m["skip"] = r.bit(h["skip_p"])
            m["i4"] = 1 - r.bit(145)
            if not m["i4"]:
                m["ymode"] = (1 if r.bit(128) else 3) if r.bit(156) else (2 if r.bit(163) else 0)
                top[x], left = [m["ymode"]] * 4, [m["ymode"]] * 4
            else:
                modes = []
                for k in range(16):
                    yy, xx = divmod(k, 4)
                    prob = BMODES_PROBA[top[x][xx]][left[yy]]
                    i = _YMODES4_TREE[r.bit(prob[0])]
                    while i > 0:
                        i = _YMODES4_TREE[2 * i + r.bit(prob[i])]
                    modes.append(-i)
                    top[x][xx] = left[yy] = -i
                m["bmodes"] = modes
            m["uvmode"] = 0 if not r.bit(142) else 2 if not r.bit(114) else (1 if r.bit(183) else 3)
            mbs.append(m)
    assert r.overrun == 0, "partition 0 ends inside the macroblock headers"
    token = [(m["i4"], m["skip"] if h["use_skip"] else 0) for m in mbs]
    return dict(pay=pay, p0=p0, width=W, height=H, mb_w=mb_w, mb_h=mb_h, hdr=h, mbs=mbs,
                _fixed=(h["log2_parts"], list(h["proba"]), h["use_skip"], token))


def _check_token_safe(f):
    h, mbs = f["hdr"], f["mbs"]
    parts, proba, use_skip, token = f["_fixed"]
    assert h["log2_parts"] == parts, "the partition count is fixed by the partition-size table"
    assert h["proba"] == proba, "the probability updates decide how the tokens parse"
    assert h["use_skip"] in (use_skip, 1), "use_skip may only go from 0 to 1"
    for m, (i4, skip) in zip(mbs, token):
        assert m["i4"] == i4, "an i4 flag decides whether a Y2 block is parsed"
        assert (m["skip"] if h["use_skip"] else 0) == skip, "a skip flag decides whether tokens are parsed"
        assert (m["ymode"] in range(4)) if not i4 else (len(m["bmodes"]) == 16 and set(m["bmodes"]) <= set(range(10)))
        assert m["uvmode"] in range(4) and m["segment"] in range(4)


def write(f):
    """the simple-format stream of frame f: partition 0 rewritten, the first-partition size, VP8 chunk size and RIFF size patched"""
    _check_token_safe(f)
    h, w = f["hdr"], BoolEncoder()
    w.bit(128, h["color_space"])
    w.bit(128, h["clamp_type"])
    w.bit(128, h["use_segment"])
    if h["use_segment"]:
        w.bit(128, h["update_map"])
        w.bit(128, h["update_data"])
        if h["update_data"]:
            w.bit(128, h["absolute_delta"])
            for v in h["quantizer"]:
                w.optional(v, lambda v: w.signed(v, 7))
            for v in h["filter_strength"]:
                w.optional(v, lambda v: w.signed(v, 6))
        if h["update_map"]:
            for v in h["seg_proba"]:
                w.optional(v, lambda v: w.literal(v, 8))
    w.bit(128, h["simple"])
    w.literal(h["level"], 6)
    w.literal(h["sharpness"], 3)
    w.bit(128, h["use_lf_delta"])
    if h["use_lf_delta"]:
        w.bit(128, h["update_lf_delta"])
        if h["update_lf_delta"]:
            for v in h["ref_lf_delta"] + h["mode_lf_delta"]:
                w.optional(v, lambda v: w.signed(v, 6))
    w.literal(h["log2_parts"], 2)
    w.literal(h["base_q0"], 7)
    for v in h["dq"]:
        w.optional(v, lambda v: w.signed(v, 4))
    w.bit(128, h["refresh"])
    for p, v in zip(COEFF_UPDATE_PROBA, h["proba"]):
        w.bit(p, int(v is not None))
        if v is not None:
            w.literal(v, 8)
    w.bit(128, h["use_skip"])
    if h["use_skip"]:
        w.literal(h["skip_p"], 8)
    sp = [255 if v is None else v for v in h["seg_proba"]]
    top = [[0] * 4 for _ in range(f["mb_w"])]
    for y in range(f["mb_h"]):
        left = [0] * 4
        for x in range(f["mb_w"]):
            m = f["mbs"][y * f["mb_w"] + x]
            if h["use_segment"] and h["update_map"]:
                s = m["segment"]
                w.bit(sp[0], int(s >= 2))
                w.bit(sp[2] if s >= 2 else sp[1], s & 1)
            if h["use_skip"]:
                w.bit(h["skip_p"], m["skip"])
            w.bit(145, 1 - m["i4"])
            if not m["i4"]:
                for p, b in _YMODE16_PATH[m["ymode"]]:
                    w.bit(p, b)
                top[x], left = [m["ymode"]] * 4, [m["ymode"]] * 4
            else:
                for k, md in enumerate(m["bmodes"]):
                    yy, xx = divmod(k, 4)
                    prob = BMODES_PROBA[top[x][xx]][left[yy]]
                    for node, b in _YMODE4_PATH[md]:
                        w.bit(prob[node], b)
                    top[x][xx] = left[yy] = md
            for p, b in _UVMODE_PATH[m["uvmode"]]:
                w.bit(p, b)
    p0 = w.finish()
    assert len(p0) < 1 << 19, "the first-partition size has 19 bits"
    pay = f["pay"]
    tag = (pay[0] | pay[1] << 8 | pay[2] << 16) & 31 | len(p0) << 5
    npay = bytes([tag & 255, tag >> 8 & 255, tag >> 16]) + pay[3:10] + p0 + pay[10 + f["p0"]:]
    body = b"WEBPVP8 " + struct.pack("<I", len(npay)) + npay + b"\0" * (len(npay) & 1)
    return b"RIFF" + struct.pack("<I", len(body)) + body


def set_scale_bits(stream, xscale, yscale):
    """the frame tag's 2-bit horizontal and vertical scale fields (the top bits of the 16-bit width and height): a byte edit"""
    b = bytearray(stream)
    i = stream.index(b"VP8 ") + 8
    b[i + 7] = (b[i + 7] & 0x3F) | xscale << 6
    b[i + 9] = (b[i + 9] & 0x3F) | yscale << 6
    return bytes(b)


def to_vp8x(stream):
    """the simple-format stream inside a VP8X container whose canvas is the frame's size (scale bits masked off)"""
    pay = vp8_payload(stream)
    W, H = (pay[6] | pay[7] << 8) & 0x3FFF, (pay[8] | pay[9] << 8) & 0x3FFF
    vp8x = b"VP8X" + struct.pack("<I", 10) + bytes(4) + (W - 1).to_bytes(3, "little") + (H - 1).to_bytes(3, "little")
    body = b"WEBP" + vp8x + stream[12:]
    return b"RIFF" + struct.pack("<I", len(body)) + body


def scale_bits(stream):
    """(xscale, yscale) of the frame tag"""
    i = stream.index(b"VP8 ") + 8
    return stream[i + 7] >> 6, stream[i + 9] >> 6


def position_classes(mbx, mby, mb_w, mb_h):
    """the edge positions of macroblock (mbx, mby): top-left, first row, first column, last column, last row"""
    out = set()
    if mbx == 0 and mby == 0:
        out.add("top_left")
    if mby == 0 and mbx > 0:
        out.add("first_row")
    if mbx == 0 and mby > 0:
        out.add("first_col")
    if mbx == mb_w - 1:
        out.add("last_col")
    if mby == mb_h - 1:
        out.add("last_row")
    return out


def block_position_classes(mbx, mby, k, mb_w, mb_h):
    """the same classes for 4x4 block k (raster order) of macroblock (mbx, mby), at the image's 4x4-block grid: the top-left block,
    the blocks of the first block row and column, the last block column (whose top-right samples are replicated) and last row"""
    bx, by = 4 * mbx + (k & 3), 4 * mby + (k >> 2)
    out = set()
    if bx == 0 and by == 0:
        out.add("top_left")
    if by == 0 and bx > 0:
        out.add("first_row")
    if bx == 0 and by > 0:
        out.add("first_col")
    if bx == 4 * mb_w - 1:
        out.add("last_col")
    if by == 4 * mb_h - 1:
        out.add("last_row")
    return out


POSITIONS = ("top_left", "first_row", "first_col", "last_col", "last_row")


def mode_positions(f):
    """{(kind, mode, position)} of a parsed frame, kind 'y16', 'b4' or 'uv'"""
    out = set()
    for i, m in enumerate(f["mbs"]):
        y, x = divmod(i, f["mb_w"])
        pos = position_classes(x, y, f["mb_w"], f["mb_h"])
        out |= {("uv", m["uvmode"], p) for p in pos}
        if m["i4"]:
            for k, md in enumerate(m["bmodes"]):
                out |= {("b4", md, p) for p in block_position_classes(x, y, k, f["mb_w"], f["mb_h"])}
        else:
            out |= {("y16", m["ymode"], p) for p in pos}
    return out
