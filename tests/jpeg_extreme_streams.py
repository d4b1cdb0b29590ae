"""Test-only builder of legal JPEG streams from arbitrary quantised coefficients, and the corpora built from it.

Natural streams keep every IDCT value in range; these do not.  baseline() codes coefficient planes as one interleaved scan (SOF0 with
8-bit DQT, or SOF1 with 16-bit DQT), with the standard Huffman tables (DC categories <= 11, AC sizes <= 10) or wide built tables
(every DC category 0..15, every AC run / size up to 15, codes of up to 16 bits), optionally with a restart interval and an Adobe APP14
marker for 4-component frames.  progressive() codes the same planes as a spectral-selection script (one DC scan, two AC bands per
component); jpeg_cmyk_streams.one_scan_per_component() re-codes a baseline one as one scan per component.  extreme_corpus() and
mutated() are the corpora of tests/test_jpeg_extreme_cpu.py and tests/test_gpu_jpeg_extreme.py, which compare them with
cv2.imdecode."""
import numpy as np

from jpeg_cmyk_streams import _ZZ, _BitWriter, _huff_codes, _seg, _segments

SAMPLINGS = {"gray": [(1, 1)], "444": [(1, 1)] * 3, "422": [(2, 1), (1, 1), (1, 1)], "440": [(1, 2), (1, 1), (1, 1)],
             "420": [(2, 2), (1, 1), (1, 1)], "cmyk": [(1, 1)] * 4, "ycck": [(2, 2), (1, 1), (1, 1), (2, 2)]}


def _dht(tc_th, bits, vals):
    counts = [0] * 16
    for l in bits:
        counts[l - 1] += 1
    order = sorted(range(len(vals)), key=lambda i: bits[i])
    return bytes([tc_th] + counts + [vals[i] for i in order])


_STD = None


def std_tables():
    """DHT payloads [DC0, AC0, DC1, AC1] of the T.81 K.3 tables, taken from a cv2 stream"""
    global _STD
    if _STD is None:
        import cv2
        s = cv2.imencode(".jpg", np.zeros((8, 8, 3), np.uint8))[1].tobytes()
        dht = b"".join(_segments(s)[0xC4])
        out, o = {}, 0
        while o < len(dht):
            n = 17 + sum(dht[o + 1:o + 17])
            out[dht[o]] = dht[o:o + n]
            o += n
        _STD = [out[0x00], out[0x10], out[0x01], out[0x11]]
    return _STD


def wide_tables():
    """DHT payloads [DC0, AC0, DC1, AC1]: every DC category 0..15 and every AC symbol of sizes 1..15 plus EOB and ZRL, canonical codes of
    2..16 bits (Kraft sum < 1, so invalid codes exist), the rarer symbols on codes longer than the decoder's first-level lookup"""
    dc_len = [2, 3, 3, 3, 4, 4, 4, 5, 5, 6, 6, 7, 8, 10, 12, 16]
    ac_syms = [0x00, 0xF0] + sorted(((r << 4) | s for r in range(16) for s in range(1, 16)), key=lambda v: (v & 15) + 2 * (v >> 4))
    counts = {2: 1, 3: 1, 4: 2, 5: 3, 6: 4, 7: 6, 8: 8, 9: 10, 10: 14, 11: 18, 12: 24, 13: 30, 14: 36, 15: 40, 16: 45}
    ac_len = [l for l in sorted(counts) for _ in range(counts[l])]
    assert len(ac_len) == len(ac_syms) == 242
    dc, ac = _dht(0x00, dc_len, list(range(16))), _dht(0x10, ac_len, ac_syms)
    return [dc, ac, bytes([0x01]) + dc[1:], bytes([0x11]) + ac[1:]]


def _dqt(tables, dqt16):
    out = b""
    for t, q in enumerate(tables):
        zz = [int(q[_ZZ[k]]) for k in range(64)]
        out += bytes([(16 if dqt16 else 0) | t]) + (b"".join(v.to_bytes(2, "big") for v in zz) if dqt16 else bytes(zz))
    return _seg(0xDB, out)


def _header(h, w, sampling, qtabs, dqt16, tables, rst, adobe, sof):
    ncomp = len(sampling)
    out = bytearray(b"\xff\xd8")
    if adobe is not None:
        out += _seg(0xEE, b"Adobe" + bytes([0, 100, 0, 0, 0, 0, adobe]))
    out += _dqt(qtabs, dqt16)
    comp = b"".join(bytes([c + 1, (hs << 4) | vs, c]) for c, (hs, vs) in enumerate(sampling))
    out += _seg(sof, bytes([8, h >> 8, h & 255, w >> 8, w & 255, ncomp]) + comp)
    out += b"".join(_seg(0xC4, t) for t in tables)
    if rst:
        out += _seg(0xDD, bytes([rst >> 8, rst & 255]))
    return out


def _tsel(c):
    return 0x00 if c == 0 else 0x11


def baseline(h, w, sampling, planes, qtabs, dqt16=False, wide=False, rst=0, adobe=None):
    """One interleaved scan.  planes[c]: [mcuy * vs, mcux * hs, 64] coefficients (natural order, absolute DC); qtabs[c]: the 64 quantisation
    values of component c (natural order), table c.  Components > 0 use Huffman tables 1."""
    tables = wide_tables() if wide else std_tables()
    out = _header(h, w, sampling, qtabs, dqt16, tables, rst, adobe, 0xC1 if dqt16 else 0xC0)
    codes = _huff_codes(b"".join(tables))
    hmax, vmax = max(s[0] for s in sampling), max(s[1] for s in sampling)
    mcux, mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    ncomp = len(sampling)
    out += _seg(0xDA, bytes([ncomp]) + b"".join(bytes([c + 1, _tsel(c)]) for c in range(ncomp)) + bytes([0, 63, 0]))
    bw, pred = _BitWriter(), [0] * ncomp
    for m in range(mcux * mcuy):
        if rst and m and m % rst == 0:
            bw.restart(m // rst - 1)
            pred = [0] * ncomp
        my, mx = divmod(m, mcux)
        for c, (hs, vs) in enumerate(sampling):
            t = _tsel(c)
            for v in range(vs):
                for hh in range(hs):
                    pred[c] = bw.block(planes[c][my * vs + v, mx * hs + hh], pred[c], codes[t >> 4], codes[0x10 | (t & 15)])
    return bytes(out + bw.finish() + b"\xff\xd9")


def _ac_band(bw, blk, ss, se, ac_t):
    """AC first scan of one block, Al = 0, every block ends with its own EOB (no EOB runs)"""
    run = 0
    for k in range(ss, se + 1):
        val = int(blk[_ZZ[k]])
        if val == 0:
            run += 1
            continue
        while run > 15:
            bw.put(*ac_t[0xF0])
            run -= 16
        s, bits = _BitWriter._val(val)
        bw.put(*ac_t[(run << 4) | s])
        bw.put(bits, s)
        run = 0
    if run:
        bw.put(*ac_t[0])


def progressive(h, w, sampling, planes, qtabs, dqt16=False, wide=False, rst=0, adobe=None, bands=((1, 5), (6, 63))):
    """SOF2: one DC scan over all components (interleaved when there are several), then one scan per component and band.  The image
    size must be a whole number of MCUs, so that the non-interleaved scans code every block of the planes."""
    tables = wide_tables() if wide else std_tables()
    out = _header(h, w, sampling, qtabs, dqt16, tables, rst, adobe, 0xC2)
    codes = _huff_codes(b"".join(tables))
    hmax, vmax = max(s[0] for s in sampling), max(s[1] for s in sampling)
    assert h % (8 * vmax) == 0 and w % (8 * hmax) == 0
    mcux, mcuy = w // (8 * hmax), h // (8 * vmax)
    ncomp = len(sampling)
    out += _seg(0xDA, bytes([ncomp]) + b"".join(bytes([c + 1, _tsel(c) & 0xF0]) for c in range(ncomp)) + bytes([0, 0, 0]))
    bw, pred = _BitWriter(), [0] * ncomp
    nmcu = mcux * mcuy if ncomp > 1 else planes[0].shape[0] * planes[0].shape[1]
    for m in range(nmcu):
        if rst and m and m % rst == 0:
            bw.restart(m // rst - 1)
            pred = [0] * ncomp
        if ncomp == 1:
            by, bx = divmod(m, planes[0].shape[1])
            blk = planes[0][by, bx]
            s, bits = _BitWriter._val(int(blk[0]) - pred[0])
            bw.put(*codes[0x00][s])
            bw.put(bits, s)
            pred[0] = int(blk[0])
            continue
        my, mx = divmod(m, mcux)
        for c, (hs, vs) in enumerate(sampling):
            dct = codes[_tsel(c) >> 4]
            for v in range(vs):
                for hh in range(hs):
                    blk = planes[c][my * vs + v, mx * hs + hh]
                    s, bits = _BitWriter._val(int(blk[0]) - pred[c])
                    bw.put(*dct[s])
                    bw.put(bits, s)
                    pred[c] = int(blk[0])
    out += bw.finish()
    for c in range(ncomp):
        act = codes[0x10 | (_tsel(c) & 15)]
        for ss, se in bands:
            out += _seg(0xDA, bytes([1, c + 1, _tsel(c) & 0x0F, ss, se, 0]))
            bw, (bh, bwid) = _BitWriter(), planes[c].shape[:2]
            for n in range(bh * bwid):
                if rst and n and n % rst == 0:
                    bw.restart(n // rst - 1)
                by, bx = divmod(n, bwid)
                _ac_band(bw, planes[c][by, bx], ss, se, act)
            out += bw.finish()
    return bytes(out + b"\xff\xd9")


# ---- random extreme content ------------------------------------------------------------------------------------------------------
def extreme_blocks(rng, n, amax=1023, dmax=1023):
    """n blocks [n, 64] (natural order): absolute DC in [-dmax, dmax], a few AC coefficients up to +-amax, biased to low frequencies; a
    quarter keep rows 1..7 zero (pass-1 shortcut of the SIMD IDCT), a tenth are DC only"""
    blk = np.zeros((n, 64), np.int64)
    blk[:, 0] = rng.integers(-dmax, dmax + 1, n)
    kind = rng.random(n)
    for i in range(n):
        if kind[i] < 0.1:
            continue
        cnt = int(rng.integers(1, 7))
        if kind[i] < 0.35:
            pos = rng.integers(1, 8, cnt)                                             # row 0 only
        else:
            pos = np.minimum(rng.geometric(0.15, cnt), 63)
            pos = np.array([_ZZ[p] for p in pos])
        mag = np.where(rng.random(cnt) < 0.5, rng.integers(1, amax + 1, cnt), rng.integers(1, 64, cnt))
        blk[i, pos] = mag * rng.choice([-1, 1], cnt)
    return blk


def extreme_qtab(rng, dqt16=False):
    """a random table per entry, a flat one, or (16-bit) one with large entries"""
    k = rng.integers(0, 3)
    top = 65535 if dqt16 else 255
    if k == 0:
        return rng.integers(1, 256, 64)
    if k == 1:
        return np.full(64, int(rng.integers(1, 256)))
    return rng.integers(1, top + 1, 64)


def planes_for(rng, h, w, sampling, amax=1023, dmax=1023):
    hmax, vmax = max(s[0] for s in sampling), max(s[1] for s in sampling)
    mcux, mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    out = []
    for hs, vs in sampling:
        bh, bw = mcuy * vs, mcux * hs
        out.append(extreme_blocks(rng, bh * bw, amax, dmax).reshape(bh, bw, 64))
    return out


def extreme_stream(seed, h, w, layout, dqt16=False, wide=False, rst=0, kind="baseline"):
    """one random extreme stream; returns (stream, planes, qtabs).  Wide tables allow AC up to +-32767 and DC up to +-16383."""
    rng = np.random.default_rng(seed)
    sampling = SAMPLINGS[layout]
    amax, dmax = (32767, 16383) if wide else (1023, 1023)
    planes = planes_for(rng, h, w, sampling, amax, dmax)
    qtabs = [extreme_qtab(rng, dqt16) for _ in sampling]
    adobe = {"cmyk": 0, "ycck": 2}.get(layout)
    build = progressive if kind == "progressive" else baseline
    return build(h, w, sampling, planes, qtabs, dqt16, wide, rst, adobe), planes, qtabs


# ---- damaged natural streams -----------------------------------------------------------------------------------------------------
def entropy_span(b):
    """[begin, end) of the entropy-coded bytes behind the first SOS"""
    i = b.index(b"\xff\xda")
    return i + 2 + ((b[i + 2] << 8) | b[i + 3]), b.rindex(b"\xff\xd9")


def mutate(stream, rng, nbytes, span=None):
    """replaces nbytes entropy-coded bytes (inside span, default: the first scan to EOI) by random ones; never writes 0xFF and never
    touches a 0xFF, a stuffed 00 or a marker code, so every marker of the stream stays where it was"""
    b = bytearray(stream)
    lo, hi = span or entropy_span(b)
    for _ in range(nbytes):
        for _ in range(100):
            p = int(rng.integers(lo, hi))
            if b[p] != 0xFF and b[p - 1] != 0xFF:
                b[p] = int(rng.integers(0, 255))
                break
    return bytes(b)


def natural_image(rng, h, w, ch):
    import cv2
    lo = rng.uniform(0, 255, (max(2, h // 16), max(2, w // 16), ch)).astype(np.float32)
    img = cv2.resize(lo, (w, h), interpolation=cv2.INTER_CUBIC).reshape(h, w, ch) + rng.normal(0, 12, (h, w, ch))
    return np.clip(img, 0, 255).astype(np.uint8)


def mutated(seed, n, color=False, progressive=False):
    """n cv2-encoded streams (quality 20..100, restart intervals 0 / 1 / 3, colour at 4:2:0 / 4:4:4 / 4:2:2) with 1..3 entropy bytes
    replaced; progressive streams get the damage in one of their scans"""
    import cv2
    rng = np.random.default_rng(seed)
    sub = [cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422]
    out = []
    for i in range(n):
        h, w = int(rng.integers(8, 72)), int(rng.integers(8, 72))
        img = natural_image(rng, h, w, 3 if color else 1)
        p = [cv2.IMWRITE_JPEG_QUALITY, int(rng.integers(20, 101)), cv2.IMWRITE_JPEG_RST_INTERVAL, int(rng.choice([0, 1, 3]))]
        if color:
            p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, int(sub[i % 3])]
        if progressive:
            p += [cv2.IMWRITE_JPEG_PROGRESSIVE, 1]
        s = cv2.imencode(".jpg", img if color else img[..., 0], p)[1].tobytes()
        span = None
        if progressive:                                                                # damage one scan, chosen at random
            starts = [k for k in range(len(s) - 1) if s[k] == 0xFF and s[k + 1] == 0xDA]
            k = starts[int(rng.integers(0, len(starts)))]
            lo = k + 2 + ((s[k + 2] << 8) | s[k + 3])
            hi = next(j for j in range(lo, len(s) - 1) if s[j] == 0xFF and s[j + 1] != 0 and not 0xD0 <= s[j + 1] <= 0xD7)
            span = (lo, hi)
        out.append(mutate(s, rng, int(rng.integers(1, 4)), span))
    return out
