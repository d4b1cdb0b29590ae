"""Lossless JPEG (SOF3, ITU-T T.81 Annex H) hand encoder and seeded corpus for the decoder tests.

`encode` writes one interleaved Huffman-coded scan: sample precision P = 2..16, point transform Pt, predictors 1-7, 1 or 3 components
with Hi = Vi = 1, standard (T.81 K.3) or per-image optimised (K.2, codes up to 16 bits) DC tables, a distinct table per component,
restart intervals, 0xFF stuffing, and optional JFIF / Adobe markers.  `corpus()` is the seeded set of streams the tests decode,
`refused()` the streams the plan must refuse and `corrupt()` the streams whose entropy data is damaged.  Nothing is downloaded."""
import struct

import numpy as np

UNSUPPORTED, BAD_DATA = 2, 4

# T.81 K.3: DC luminance and chrominance tables (categories 0..11)
STD_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
STD_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
# every category 0..16 on code lengths 1..14 and three 16-bit codes (the all-ones code stays unused, as T.81 C requires), the most
# frequent categories on the LONGEST codes: the data of a smooth image is then almost all 12..16-bit codes, many of them across subsequence boundaries
DEEP = ([1] * 14 + [0, 3], [16, 15, 14, 13, 12, 11, 10, 9, 8, 7, 6, 5, 4, 3, 2, 1, 0])


def optimal_table(freq):
    """libjpeg's jpeg_gen_optimal_table (T.81 K.2): (bits[1..16], values) of a length-limited Huffman code for 17 categories."""
    freq = [int(f) for f in freq] + [0] * (257 - len(freq))
    freq[256] = 1                                       # reserves the all-ones code
    codesize, others = [0] * 257, [-1] * 257
    while True:
        c1, v = -1, None
        for i in range(257):
            if freq[i] and (v is None or freq[i] <= v):
                v, c1 = freq[i], i
        c2, v = -1, None
        for i in range(257):
            if freq[i] and (v is None or freq[i] <= v) and i != c1:
                v, c2 = freq[i], i
        if c2 < 0:
            break
        freq[c1] += freq[c2]
        freq[c2] = 0
        codesize[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            codesize[c1] += 1
        others[c1] = c2
        codesize[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            codesize[c2] += 1
    bits = [0] * 33
    for i in range(257):
        if codesize[i]:
            bits[codesize[i]] += 1
    for i in range(32, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    i = 16
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1
    vals = [s for n in range(1, 33) for s in range(256) if codesize[s] == n]
    return bits[1:17], vals


def codes_of(table):
    """Canonical codes (T.81 C.2): {symbol: (code, length)}."""
    bits, vals = table
    out, code, k = {}, 0, 0
    for n in range(1, 17):
        for _ in range(bits[n - 1]):
            out[vals[k]] = (code, n)
            code += 1
            k += 1
        code <<= 1
    return out


def predict(s, P, Pt, pred, restart_lines=0):
    """Per-sample prediction and difference (T.81 H.1.2.1, libjpeg-turbo jcpred.c / jdpred.c) of the H x W x C array s of shifted
    samples.  restart_lines: the rows at which a restart interval begins are predicted like the first row.  Returns the int32 differences
    (modulo 2^16, in [-32767, 32768])."""
    s = s.astype(np.int64)
    H, W, C = s.shape
    px = np.zeros_like(s)
    for y in range(H):
        first = y == 0 or (restart_lines and y % restart_lines == 0)
        for c in range(C):
            row, up = s[y, :, c], s[y - 1, :, c] if y else None
            p = np.empty(W, np.int64)
            if first:
                p[0] = 1 << max(P - Pt - 1, 0)
                p[1:] = row[:-1]
            else:
                Ra, Rb, Rc = row[:-1], up[1:], up[:-1]
                p[0] = up[0]
                p[1:] = {1: Ra, 2: Rb, 3: Rc, 4: Ra + Rb - Rc, 5: Ra + ((Rb - Rc) >> 1), 6: Rb + ((Ra - Rc) >> 1), 7: (Ra + Rb) >> 1}.get(pred, Ra)
            px[y, :, c] = p
    d = (s - px) & 0xFFFF
    return np.where(d > 32768, d - 65536, d)


def entropy_bytes(d, codes, tid):
    """The Huffman-coded, byte-stuffed data of the differences d (N x C, interleaved), padded with 1-bits to a whole byte (T.81 F.1.2.3)."""
    N, C = d.shape
    v = d.ravel().astype(np.int64)
    mag = np.abs(v)
    cat = np.where(v == 32768, 16, np.where(mag == 0, 0, np.floor(np.log2(np.maximum(mag, 1))).astype(np.int64) + 1))
    comp = np.tile(np.arange(C), N)
    code = np.zeros_like(v)
    clen = np.zeros_like(v)
    for c in range(C):
        for k, (cv, n) in codes[tid[c]].items():
            m = (comp == c) & (cat == k)
            code[m], clen[m] = cv, n
    assert np.all(clen > 0), "a category without a code"
    xlen = np.where((cat > 0) & (cat < 16), cat, 0)
    xbits = np.where(v > 0, v, v - 1 + (1 << xlen)) & ((1 << xlen) - 1)
    word = (code << xlen) | xbits                     # at most 31 bits
    wlen = clen + xlen
    shifts = np.arange(31, -1, -1)
    bits = ((word[:, None] >> shifts[None, :]) & 1).astype(np.uint8)
    keep = shifts[None, :] < wlen[:, None]
    flat = bits[keep]
    pad = (-flat.size) % 8
    flat = np.concatenate([flat, np.ones(pad, np.uint8)])
    by = np.packbits(flat)
    ff = np.flatnonzero(by == 0xFF)
    return np.insert(by, ff + 1, 0).tobytes()


def category(d):
    return 16 if d == 32768 else int(abs(int(d))).bit_length()


def encode(img, P=8, Pt=0, pred=1, restart=0, tables="std", jfif=False, adobe=None, ids=None, diffs=None, rst_seq=None):
    """A lossless JPEG stream of img (H x W or H x W x C integer samples < 2^P whose low Pt bits are dropped).

    tables: "std" (K.3 luma for component 0, chroma for the others), "opt" (one K.2 table per component from its own statistics),
    "deep" (DEEP for every component) or a list of (bits, values) per component.  restart: the restart interval in MCUs (0: none).
    diffs: the differences to code instead of the image's own (corrupt streams).  rst_seq: the RST numbers to write (bad sequences)."""
    a = np.asarray(img)
    if a.ndim == 2:
        a = a[..., None]
    H, W, C = a.shape
    s = a.astype(np.int64) >> Pt
    lines = restart // W if restart and restart % W == 0 else 0
    d = predict(s, P, Pt, pred, lines) if diffs is None else np.asarray(diffs).reshape(H, W, C)
    if tables == "std":
        tabs = [STD_LUMA] + [STD_CHROMA] * (C - 1)
    elif tables == "deep":
        tabs = [DEEP] * C
    elif tables == "opt":
        tabs = []
        for c in range(C):
            cats = np.vectorize(category)(d[..., c].ravel()) if d[..., c].size else np.zeros(0, int)
            tabs.append(optimal_table(np.bincount(cats, minlength=17)))
    else:
        tabs = list(tables)
    ntab = len({(tuple(t[0]), tuple(t[1])) for t in tabs})
    uniq = []
    for t in tabs:
        if t not in uniq:
            uniq.append(t)
    tid = [uniq.index(t) for t in tabs]
    assert len(uniq) <= 4 and ntab == len(uniq)
    codes = [codes_of(t) for t in uniq]
    ids = ids or ([1, 2, 3, 4][:C] if C != 3 else [1, 2, 3])
    seg = lambda m, body: struct.pack(">BBH", 0xFF, m, len(body) + 2) + body
    out = bytearray(b"\xFF\xD8")
    if jfif:
        out += seg(0xE0, b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0")
    if adobe is not None:
        out += seg(0xEE, b"Adobe" + struct.pack(">HHHB", 100, 0, 0, adobe))
    for k, (bits, vals) in enumerate(uniq):
        out += seg(0xC4, bytes([k]) + bytes(bits) + bytes(vals))
    if restart:
        out += seg(0xDD, struct.pack(">H", restart))
    out += seg(0xC3, struct.pack(">BHHB", P, H, W, C) + b"".join(bytes([ids[c], 0x11, 0]) for c in range(C)))
    out += seg(0xDA, bytes([C]) + b"".join(bytes([ids[c], tid[c] << 4]) for c in range(C)) + bytes([pred, 0, Pt]))
    flat = d.reshape(-1, C)
    per = restart if restart else H * W
    for k, m0 in enumerate(range(0, H * W, per)):
        if k:
            n = (k - 1) % 8 if rst_seq is None else rst_seq[(k - 1) % len(rst_seq)]
            out += bytes([0xFF, 0xD0 + n])
        out += entropy_bytes(flat[m0:m0 + per], codes, tid)
    return bytes(out + b"\xFF\xD9")


def image(h, w, c, P, seed, kind="smooth"):
    """Test samples < 2^P: a smooth gradient with noise, or uniform noise ("noise": long codes and every category)."""
    rng = np.random.default_rng(seed)
    top = (1 << P) - 1
    if kind == "noise":
        return rng.integers(0, top + 1, (h, w, c)).astype(np.uint8 if P <= 8 else np.uint16)
    y, x = np.mgrid[0:h, 0:w]
    base = np.stack([x * top // max(w - 1, 1), y * top // max(h - 1, 1), ((x + y) * 3) % (top + 1)], -1)[..., :c]
    return np.clip(base + rng.integers(-2, 3, base.shape), 0, top).astype(np.uint8 if P <= 8 else np.uint16)


def ff_image(h, w, c, seed):
    """8-bit samples whose differences (predictor 1) code to runs of 0xFF bytes under the DEEP table: stuffing everywhere."""
    rng = np.random.default_rng(seed)
    a = np.full((h, w, c), 128, np.uint8)
    a[rng.random((h, w, c)) < 0.02] = 255
    return a


def corpus(big=False):
    """[(name, stream, expected H x W x C samples after the point transform, params)].  big adds the 1080p and 4K images."""
    out = []

    def add(name, img, **kw):
        a = np.asarray(img)
        if a.ndim == 2:
            a = a[..., None]
        Pt = kw.get("Pt", 0)
        exp = (a.astype(np.int64) >> Pt) << Pt
        out.append((name, encode(a, **kw), exp.astype(np.uint8), dict(kw, shape=a.shape)))

    seed = 0
    for P in range(2, 9):
        for Pt in sorted({0, P - 1, P // 2}):
            for pred in range(1, 8):
                c = 3 if (pred + P) % 2 else 1
                seed += 1
                add(f"P{P}_Pt{Pt}_p{pred}_c{c}", image(13 + pred, 17 + 2 * P, c, P, seed), P=P, Pt=Pt, pred=pred)
    for c in (1, 3):
        for pred in (1, 4, 7):
            seed += 1
            add(f"opt_p{pred}_c{c}", image(40, 57, c, 8, seed, "noise" if pred == 4 else "smooth"), pred=pred, tables="opt")
            add(f"deep_p{pred}_c{c}", image(33, 70, c, 8, seed + 100), pred=pred, tables="deep")
            add(f"rst_p{pred}_c{c}", image(24, 31, c, 8, seed + 200), pred=pred, restart=31 * 3, tables="opt")
            add(f"rst1_p{pred}_c{c}", image(9, 20, c, 8, seed + 300), pred=pred, restart=20)
    add("distinct_tables", image(30, 40, 3, 8, 7), tables=[STD_LUMA, DEEP, STD_CHROMA])
    add("one_px_gray", np.array([[77]], np.uint8))
    add("one_px_rgb", np.array([[[1, 200, 255]]], np.uint8))
    add("one_sample_units", image(5, 1, 1, 8, 8), restart=1)
    add("row_1xN", image(1, 300, 3, 8, 9), pred=7)
    add("col_Nx1", image(300, 1, 1, 8, 10), pred=2)
    add("stuffing", ff_image(64, 128, 1, 11), tables="deep")
    add("stuffing_rgb", ff_image(40, 90, 3, 12), tables="deep", restart=90 * 4)
    add("noise_long_codes", image(64, 200, 1, 8, 13, "noise"), tables="deep", pred=5)
    add("adobe0_rgb", image(20, 30, 3, 8, 14), adobe=0)
    add("jfif_gray", image(20, 30, 1, 8, 15), jfif=True)
    add("wide", image(37, 1500, 1, 8, 16), pred=6, tables="opt")
    if big:
        add("1080p_gray_p1", image(1080, 1920, 1, 8, 20), pred=1, tables="opt")
        add("1080p_rgb_p7_rst", image(1080, 1920, 3, 8, 21), pred=7, restart=1920 * 8)
        add("4k_rgb_p4", image(2160, 3840, 3, 8, 22), pred=4, tables="opt")
    return out


def refused():
    """[(name, stream, status, reason)]: streams whose plan set-up must fail."""
    g = image(16, 16, 1, 8, 30)
    rgb = image(16, 16, 3, 8, 31)
    out = [
        ("P12", encode(image(8, 8, 1, 12, 32), P=12, tables="opt"), UNSUPPORTED, "P > 8"),
        ("P16", encode(image(8, 8, 1, 16, 33), P=16, tables="opt"), UNSUPPORTED, "P > 8"),
        ("jfif_rgb", encode(rgb, jfif=True), UNSUPPORTED, "3 components with JFIF"),
        ("adobe1_rgb", encode(rgb, adobe=1), UNSUPPORTED, "Adobe transform 1"),
        ("adobe2_rgb", encode(rgb, adobe=2), UNSUPPORTED, "Adobe transform 2"),
        ("rst_partial_line", encode(g, restart=24), UNSUPPORTED, "restart interval not a whole number of lines"),
        ("pred0", encode(g, pred=0), BAD_DATA, "predictor 0"),
        ("pred8", encode(g, pred=8), BAD_DATA, "predictor 8"),
        ("Pt_eq_P", encode(g, Pt=8), BAD_DATA, "Pt >= P"),
    ]
    two = encode(image(8, 8, 2, 8, 34))
    out.append(("two_components", two, UNSUPPORTED, "2 components"))
    four = encode(np.concatenate([image(8, 8, 3, 8, 35), image(8, 8, 1, 8, 36)], 2), ids=[1, 2, 3, 4])
    out.append(("four_components", four, UNSUPPORTED, "4 components"))
    s = bytearray(encode(rgb))
    k = s.index(b"\xFF\xC3") + 2 + 2 + 6
    s[k + 1] = 0x21                                    # component 0: H = 2
    out.append(("sampling_2x1", bytes(s), UNSUPPORTED, "sampling factors"))
    s3 = bytearray(encode(rgb))                        # the first scan of a 3-component frame codes one component
    k = s3.index(b"\xFF\xDA")
    sos1 = b"\xFF\xDA\x00\x08\x01\x01\x00\x01\x00\x00"
    out.append(("multi_scan", bytes(s3[:k]) + sos1 + b"\x00" * 16 + b"\xFF\xD9", UNSUPPORTED, "one scan per component"))
    s = bytearray(encode(g))
    k = s.index(b"\xFF\xC4") + 4 + 1 + 16
    s[k] = 17                                          # a category above 16 in the table
    out.append(("category17", bytes(s), BAD_DATA, "Huffman value above 16"))
    s = bytearray(encode(g))
    k = s.index(b"\xFF\xC4") + 4 + 1                   # the K.3 luma counts 0, 1, 5, ... become 3, 1, 3: three 1-bit codes
    s[k], s[k + 2] = 3, 3
    out.append(("dht_overflow", bytes(s), BAD_DATA, "more codes of a length than it holds"))
    s = bytearray(encode(rgb))
    k = s.index(b"\xFF\xDA") + 5                       # the SOS component entries: 1, 2, 3 -> 2, 1, 3
    s[k], s[k + 2] = s[k + 2], s[k]
    out.append(("scan_order", bytes(s), BAD_DATA, "scan components out of frame order"))
    s = bytearray(encode(rgb))
    s[k + 2] = s[k]                                    # 1, 1, 3
    out.append(("scan_repeat", bytes(s), BAD_DATA, "a scan component twice"))
    return out


def corrupt():
    """[(name, stream, kind)]: streams whose entropy data is damaged; the plan accepts them and the decode sets the sample's status."""
    g = image(32, 40, 1, 8, 40)
    rgb = image(24, 30, 3, 8, 41)
    full = encode(g, tables="opt")
    k = full.index(b"\xFF\xDA")
    body = full[k:]
    out = [("truncated", full[: k + len(body) // 2], "truncated"),
           ("truncated_rgb", encode(rgb)[: len(encode(rgb)) * 2 // 3], "truncated")]
    # an invalid code: 16 one-bits (never a code of a K.2 / K.3 table) in the middle of the data
    s = bytearray(encode(g))
    sos = s.index(b"\xFF\xDA")
    hdr = sos + 2 + struct.unpack(">H", bytes(s[sos + 2: sos + 4]))[0]
    mid = hdr + (len(s) - 2 - hdr) // 2
    s[mid: mid + 3] = b"\xFF\x00\xFF\x00\xFF\x00"[:3]
    s[mid: mid] = b""
    out.append(("bad_code", bytes(s[:mid]) + b"\xFF\x00\xFF\x00" + bytes(s[mid + 3:]), "bad_code"))
    out.append(("bad_rst_sequence", encode(rgb, restart=30 * 4, rst_seq=[0, 2, 1, 3, 4]), "bad_rst"))
    out.append(("missing_rst", encode(g, restart=40 * 8).replace(b"\xFF\xD1", b""), "bad_rst"))
    return out
