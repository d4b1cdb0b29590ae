"""Test-only builder of 4-component JPEG streams in the layout Photoshop writes for YCCK: Y 2x2, Cb 1x1, Cr 1x1, K 2x2 (10 blocks per
MCU, the T.81 limit), which Pillow cannot write.  The Y/Cb/Cr blocks are the oracle's coefficients of a cv2 4:2:0 YCbCr stream, the K
blocks those of a cv2 grayscale stream of the same size; a plain interleaved Huffman encoder (the cv2 stream's standard tables) codes
them behind an Adobe APP14 marker.  Needs only cv2, numpy and the oracle, so the GPU tests build these streams at run time and compare
the decoder with cv2.imdecode of the same bytes.  one_scan_per_component() re-codes any baseline stream, 4-component ones included, as
one scan per component."""
import numpy as np

import jpeg_cmyk_oracle as cmyk_oracle
from oracle import pyoracle as po

_ZZ = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
       35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]


def _segments(b):
    """marker -> list of segment payloads, up to the first SOS"""
    pos, segs = 2, {}
    while True:
        assert b[pos] == 0xFF
        m, L = b[pos + 1], (b[pos + 2] << 8) | b[pos + 3]
        segs.setdefault(m, []).append(b[pos + 4:pos + 2 + L])
        if m == 0xDA:
            return segs
        pos += 2 + L


def _huff_codes(dht):
    tables, o = {}, 0
    while o < len(dht):
        tc_th, bits = dht[o], dht[o + 1:o + 17]
        vals = dht[o + 17:o + 17 + sum(bits)]
        code, k, enc = 0, 0, {}
        for l in range(1, 17):
            for _ in range(bits[l - 1]):
                enc[vals[k]] = (code, l)
                code += 1
                k += 1
            code <<= 1
        tables[tc_th] = enc
        o += 17 + len(vals)
    return tables


class _BitWriter:
    """Huffman-coded blocks of one scan (T.81 F.1.2), with byte stuffing and restart markers."""

    def __init__(self):
        self.data, self.acc, self.nbits = bytearray(), 0, 0

    def put(self, v, n):
        self.acc = (self.acc << n) | (v & ((1 << n) - 1))
        self.nbits += n
        while self.nbits >= 8:
            byte = (self.acc >> (self.nbits - 8)) & 255
            self.data.append(byte)
            if byte == 0xFF:
                self.data.append(0)
            self.nbits -= 8
        self.acc &= (1 << self.nbits) - 1

    def flush(self):
        if self.nbits:
            self.put((1 << (8 - self.nbits)) - 1, 8 - self.nbits)

    def restart(self, k):
        self.flush()
        self.data.extend([0xFF, 0xD0 + (k & 7)])

    def finish(self):
        self.flush()
        return bytes(self.data)

    @staticmethod
    def _val(v):
        s = int(abs(v)).bit_length()
        return s, (v if v >= 0 else v + (1 << s) - 1)

    def block(self, blk, pred, dc_t, ac_t):
        """codes one block (natural order, absolute DC); returns the new DC predictor"""
        s, bits = self._val(int(blk[0]) - pred)
        self.put(*dc_t[s])
        if s:
            self.put(bits, s)
        run = 0
        for k in range(1, 64):
            val = int(blk[_ZZ[k]])
            if val == 0:
                run += 1
                continue
            while run > 15:
                self.put(*ac_t[0xF0])
                run -= 16
            s, bits = self._val(val)
            self.put(*ac_t[(run << 4) | s])
            self.put(bits, s)
            run = 0
        if run:
            self.put(*ac_t[0])
        return int(blk[0])


def _seg(marker, payload):
    return bytes([0xFF, marker, (len(payload) + 2) >> 8, (len(payload) + 2) & 255]) + bytes(payload)


def photoshop_ycck(h, w, seed, quality=90, rst=0, transform=2):
    """A 4-component baseline stream, Y 2x2 / Cb 1x1 / Cr 1x1 / K 2x2, with an Adobe APP14 marker of the given transform (2: YCCK,
    0: the same samples read as CMYK) and, with rst > 0, a restart interval of rst MCUs."""
    import cv2
    r = np.random.default_rng(seed)
    lo = r.uniform(0, 255, (max(2, h // 32), max(2, w // 32), 4)).astype(np.float32)
    img = np.stack([cv2.resize(lo[..., c], (w, h), interpolation=cv2.INTER_CUBIC) for c in range(4)], -1) + r.normal(0, 5, (h, w, 4))
    img = np.clip(img, 0, 255).astype(np.uint8)
    q = [cv2.IMWRITE_JPEG_QUALITY, quality]
    ycc = cv2.imencode(".jpg", np.ascontiguousarray(img[..., :3]), q + [cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                                                     cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])[1].tobytes()
    gray = cv2.imencode(".jpg", np.ascontiguousarray(img[..., 3]), q)[1].tobytes()
    cy, ccb, ccr = po.jpeg_coeffs(ycc)
    (ck_raw,) = po.jpeg_coeffs(gray)
    mcux, mcuy = (w + 15) // 16, (h + 15) // 16
    ck = np.zeros((2 * mcuy, 2 * mcux, 64), np.int16)                 # K at luma resolution; blocks past the gray stream's grid stay 0
    ck[:ck_raw.shape[0], :ck_raw.shape[1]] = ck_raw[:2 * mcuy, :2 * mcux]
    sy, sg = _segments(ycc), _segments(gray)
    qtab = {}                                                          # 8-bit tables (cv2 at quality >= 25)
    for seg in sy[0xDB]:
        for o in range(0, len(seg), 65):
            qtab[seg[o] & 15] = seg[o + 1:o + 65]
    qtab[2] = sg[0xDB][0][1:65]                                        # the grayscale stream's table 0, as table 2
    codes = _huff_codes(b"".join(sy[0xC4]))
    out = bytearray(b"\xff\xd8")
    out += _seg(0xEE, b"Adobe" + bytes([0, 100, 0, 0, 0, 0, transform]))
    out += _seg(0xDB, b"".join(bytes([t]) + qtab[t] for t in (0, 1, 2)))
    out += _seg(0xC0, bytes([8, h >> 8, h & 255, w >> 8, w & 255, 4, 1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1, 4, 0x22, 2]))
    out += b"".join(_seg(0xC4, s) for s in sy[0xC4])
    if rst:
        out += _seg(0xDD, bytes([rst >> 8, rst & 255]))
    # component: (coefficients, h, v, DC table, AC table); K codes with the luma tables
    comps = [(cy, 2, 2, 0x00, 0x10), (ccb, 1, 1, 0x01, 0x11), (ccr, 1, 1, 0x01, 0x11), (ck, 2, 2, 0x00, 0x10)]
    out += _seg(0xDA, bytes([4, 1, 0x00, 2, 0x11, 3, 0x11, 4, 0x00, 0, 63, 0]))
    bw, pred = _BitWriter(), [0, 0, 0, 0]
    for m in range(mcux * mcuy):
        if rst and m and m % rst == 0:
            bw.restart(m // rst - 1)
            pred = [0, 0, 0, 0]
        my, mx = divmod(m, mcux)
        for c, (cf, hs, vs, dct, act) in enumerate(comps):
            for v in range(vs):
                for hh in range(hs):
                    pred[c] = bw.block(cf[my * vs + v, mx * hs + hh], pred[c], codes[dct], codes[act])
    out += bw.finish() + b"\xff\xd9"
    return bytes(out)


def one_scan_per_component(stream, rst=0):
    """Re-codes the entropy data of an interleaved baseline stream (any component count, no restart interval) as one scan per component,
    legal in a sequential frame (T.81 A.2): same headers and Huffman tables, the oracle's coefficients.  Returns the stream and, per
    component, the blocks per column and row that such a scan codes (ceil(component extent / 8), not padded to whole MCUs)."""
    b = bytes(stream)
    info = po.jpeg_info(b)
    comps = cmyk_oracle.coeffs(b)
    ncomp, W, H = info["ncomp"], info["width"], info["height"]
    hmax, vmax = max(info["hs"][:ncomp]), max(info["vs"][:ncomp])
    segs = _segments(b)
    assert 0xDD not in segs
    sof = (segs.get(0xC0) or segs[0xC1])[0]
    cids = [sof[6 + 3 * c] for c in range(ncomp)]
    sos = segs[0xDA][0]
    tdta = {sos[1 + 2 * i]: sos[2 + 2 * i] for i in range(sos[0])}
    codes = _huff_codes(b"".join(segs[0xC4]))
    out = bytearray(b[:b.index(b"\xff\xda" + bytes([0, len(sos) + 2]) + sos)])
    if rst:
        out += _seg(0xDD, bytes([rst >> 8, rst & 255]))
    hblk = [((H * info["vs"][c] + vmax - 1) // vmax + 7) // 8 for c in range(ncomp)]
    wblk = [((W * info["hs"][c] + hmax - 1) // hmax + 7) // 8 for c in range(ncomp)]
    for c in range(ncomp):
        t = tdta[cids[c]]
        out += _seg(0xDA, bytes([1, cids[c], t, 0, 63, 0]))
        bw, pred, n = _BitWriter(), 0, 0
        for by in range(hblk[c]):
            for bx in range(wblk[c]):
                if rst and n and n % rst == 0:
                    bw.restart(n // rst - 1)
                    pred = 0
                n += 1
                pred = bw.block(comps[c][by, bx], pred, codes[t >> 4], codes[0x10 | (t & 15)])
        out += bw.finish()
    out += b"\xff\xd9"
    return bytes(out), hblk, wblk


def multiscan_expected(stream, hblk, wblk):
    """arena-order coefficients of the interleaved twin; the blocks a non-interleaved scan does not code (padding up to the MCU) stay 0"""
    comps, info = cmyk_oracle.coeffs(stream), po.jpeg_info(stream)
    for c in range(info["ncomp"]):
        comps[c][hblk[c]:] = 0
        comps[c][:, wblk[c]:] = 0
    hs, vs = info["hs"], info["vs"]
    return np.stack([comps[c][my * vs[c] + v, mx * hs[c] + h] for my in range(info["mcuy"]) for mx in range(info["mcux"])
                     for c in range(info["ncomp"]) for v in range(vs[c]) for h in range(hs[c])])
