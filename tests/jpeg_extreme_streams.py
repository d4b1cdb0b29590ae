"""Test-only builder of legal JPEG streams from arbitrary quantised coefficients, and the corpora built from it.

Natural streams keep every IDCT value in range; these do not.  baseline() codes coefficient planes as one interleaved scan (SOF0 with
8-bit DQT, or SOF1 with 16-bit DQT), with the standard Huffman tables (DC categories <= 11, AC sizes <= 10) or wide built tables
(every DC category 0..15, every AC run / size up to 15, codes of up to 16 bits), optionally with a restart interval and an Adobe APP14
marker for 4-component frames.  progressive() codes the same planes under any scan script (T.81 G.1.2: successive approximation,
EOB runs, refinement, restart intervals, tables and DQT placed between scans), expected() and waves() state what the decoder's arena
holds after any prefix of a script and how many launches its planner makes, and the catalogue below names the scripts encoders
write; jpeg_cmyk_streams.one_scan_per_component() re-codes a baseline stream as one scan per component.  extreme_corpus() and
mutated() are the corpora of tests/test_jpeg_extreme_cpu.py and tests/test_gpu_jpeg_extreme.py, which compare them with
cv2.imdecode."""
from collections import Counter, namedtuple

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
    """tables: a list (ids 0, 1, ...) or {id: values}, natural order"""
    out = b""
    for t, q in (tables.items() if isinstance(tables, dict) else enumerate(tables)):
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


# ---- progressive scripts (T.81 G.1.2; the coding decisions follow libjpeg's jcphuff.c) --------------------------------------------
Scan = namedtuple("Scan", "comps ss se ah al rst slot dqt", defaults=(None, 0, None))
Scan.__doc__ = """One SOS of a script: the component indices it codes, the band Ss..Se and the successive approximation Ah / Al.  rst: a DRI
segment in front of the scan (0 switches restarts off; None keeps the interval in force).  slot: the Huffman table slot of the scan's
tables (component i of a DC scan takes slot + i, mod 4).  dqt: {table id: 64 values, natural order}, a DQT segment in front of the scan."""

_EOB_FLUSH_BITS = 1000 - 64 + 1        # jcphuff.c MAX_CORR_BITS - DCTSIZE2 + 1: more buffered correction bits end the EOB run


def _geometry(h, w, sampling):
    """(mcux, mcuy, [(blocks per column, blocks per row)] of each component in a non-interleaved scan: ceil(component extent / 8))"""
    hmax, vmax = max(s[0] for s in sampling), max(s[1] for s in sampling)
    blk = [((-(-h * vs // vmax) + 7) // 8, (-(-w * hs // hmax) + 7) // 8) for hs, vs in sampling]
    return -(-w // (8 * hmax)), -(-h // (8 * vmax)), blk


def _optimal_dht(tc_th, counts, skew=False):
    """DHT payload of a table built from symbol counts by jchuff.c jpeg_gen_optimal_table (a reserved all-ones code, then no code longer
    than 16 bits).  skew: the counts are replaced by weights that halve with each rank, so that the rarer symbols get 9..16-bit codes."""
    freq = [0] * 257
    ranked = sorted(counts, key=lambda s: (-counts[s], s))
    for rank, s in enumerate(ranked):
        freq[s] = 1 << max(0, 40 - rank) if skew else counts[s]
    freq[256] = 1
    codesize, others = [0] * 257, [-1] * 257
    active = [i for i in range(257) if freq[i]]
    while len(active) > 1:
        c1 = min(active, key=lambda i: (freq[i], -i))             # the smallest count, on a tie the largest symbol (jchuff.c)
        c2 = min((i for i in active if i != c1), key=lambda i: (freq[i], -i))
        freq[c1] += freq[c2]
        active.remove(c2)
        codesize[c1] += 1
        while others[c1] >= 0:
            c1 = others[c1]
            codesize[c1] += 1
        others[c1] = c2
        codesize[c2] += 1
        while others[c2] >= 0:
            c2 = others[c2]
            codesize[c2] += 1
    maxl = max(codesize)
    bits = [0] * (max(maxl, 16) + 1)
    for i in range(257):
        if codesize[i]:
            bits[codesize[i]] += 1
    for i in range(maxl, 16, -1):
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
    bits[i] -= 1                                                  # drop the reserved code
    vals = [s for l in range(1, maxl + 1) for s in range(256) if codesize[s] == l]
    return bytes([tc_th] + bits[1:17] + vals)


class _ScanCoder:
    """The symbols, raw bits and restart markers of one scan in stream order; the tables are built from the symbols afterwards."""

    def __init__(self, overlong):
        self.ev, self.eobrun, self.pend, self.overlong = [], 0, [], overlong

    def sym(self, key, s):
        self.ev.append((0, key, s))

    def bits(self, v, n):
        if n:
            self.ev.append((1, v, n))

    def flush_eobrun(self, key):                                  # jcphuff.c emit_eobrun: the run, then the bits buffered behind it
        if self.eobrun:
            n = self.eobrun.bit_length() - 1
            self.sym(key, n << 4)
            self.bits(self.eobrun, n)
            for b in self.pend:
                self.bits(b, 1)
            self.eobrun, self.pend = 0, []

    def end_block(self, key, pend):
        self.eobrun += 1
        self.pend += pend
        if self.eobrun == 0x7FFF or len(self.pend) > _EOB_FLUSH_BITS:
            self.flush_eobrun(key)

    def ac_first(self, key, a, sgn, al):                           # encode_mcu_AC_first; a: |coefficients| >> Al of the band
        nk, prev = len(a), -1
        for p in np.flatnonzero(a):
            r = p - prev - 1
            prev = p
            self.flush_eobrun(key)
            while r > 15:
                self.sym(key, 0xF0)
                r -= 16
            v = int(a[p])
            s = v.bit_length()
            self.sym(key, (r << 4) | s)
            self.bits(v if sgn[p] else ~v, s)
        if prev < nk - 1:
            self.end_block(key, [])

    def ac_refine(self, key, a, sgn):                              # encode_mcu_AC_refine
        nz = np.flatnonzero(a)
        eob = max((p for p in nz if a[p] == 1), default=-1)       # the last coefficient that becomes nonzero in this pass
        r, br, prev = 0, [], -1
        for p in nz:
            r += p - prev - 1
            prev = p
            while r > 15 and p <= eob:
                self.flush_eobrun(key)
                self.sym(key, 0xF0)
                r -= 16
                for b in br:
                    self.bits(b, 1)
                br = []
            if a[p] > 1:
                br.append(int(a[p]) & 1)                          # a correction bit of an already nonzero coefficient
                continue
            self.flush_eobrun(key)
            self.sym(key, (r << 4) | 1)
            self.bits(int(sgn[p]), 1)
            for b in br:
                self.bits(b, 1)
            br, r = [], 0
        r += len(a) - 1 - prev
        if r > 0 or br:
            self.end_block(key, br)

    def block(self, dkey, akey, blk, pred):                       # one block of a sequential scan
        s, b = _BitWriter._val(int(blk[0]) - pred)
        self.sym(dkey, s)
        self.bits(b, s)
        z = np.asarray(blk, np.int64)[_ZZ]
        prev = 0
        for p in np.flatnonzero(z[1:]) + 1:
            r = p - prev - 1
            prev = p
            while r > 15:
                self.sym(akey, 0xF0)
                r -= 16
            s, b = _BitWriter._val(int(z[p]))
            self.sym(akey, (r << 4) | s)
            self.bits(b, s)
        if prev < 63:
            self.sym(akey, 0)
        return int(blk[0])

    def code(self, skew):
        """(DHT payload, entropy-coded bytes)"""
        counts = {}
        for e in self.ev:
            if e[0] == 0:
                counts.setdefault(e[1], Counter())[e[2]] += 1
        dht = b"".join(_optimal_dht((tc << 4) | th, counts[(tc, th)], skew) for tc, th in sorted(counts))
        codes = _huff_codes(dht)
        bw = _BitWriter()
        for kind, x, y in self.ev:
            if kind == 0:
                bw.put(*codes[(x[0] << 4) | x[1]][y])
            elif kind == 1:
                bw.put(x, y)
            else:
                bw.restart(x)
        return dht, bw.finish()


def _scan_data(sc, planes, sampling, geo, dri, sequential, skew, overlong):
    """(SOS payload, DHT payload, entropy-coded bytes) of one scan"""
    mcux, mcuy, blk = geo
    comps, single = sc.comps, len(sc.comps) == 1
    if single:
        c = comps[0]
        units = [[(0, c, by, bx)] for by in range(blk[c][0]) for bx in range(blk[c][1])]
    else:
        units = [[(i, c, my * sampling[c][1] + v, mx * sampling[c][0] + hh) for i, c in enumerate(comps)
                  for v in range(sampling[c][1]) for hh in range(sampling[c][0])] for my in range(mcuy) for mx in range(mcux)]
    dc_slot = [(sc.slot + i) % 4 for i in range(len(comps))]
    akey = (1, sc.slot)
    if sequential:
        sel = [(t << 4) | t for t in dc_slot]
    elif sc.ss == 0:
        sel = [t << 4 if sc.ah == 0 else 0 for t in dc_slot]
    else:
        sel = [sc.slot]
    sos = bytes([len(comps)]) + b"".join(bytes([c + 1, t]) for c, t in zip(comps, sel)) + bytes([sc.ss, sc.se, (sc.ah << 4) | sc.al])
    e = _ScanCoder(overlong)
    if sc.ss > 0:                                                 # the band of every block, |v| >> Al, and the signs
        c = comps[0]
        band = planes[c][:blk[c][0], :blk[c][1]].reshape(-1, 64)[:, [_ZZ[k] for k in range(sc.ss, sc.se + 1)]].astype(np.int64)
        mag, pos = np.abs(band) >> sc.al, band >= 0
        any_ = mag.any(1)
    pred = [0] * 4
    for u, unit in enumerate(units):
        if dri and u and u % dri == 0:
            if e.eobrun and e.overlong:
                e.eobrun = min(e.eobrun + 5, 0x7FFF)              # a run that claims blocks past the marker
            e.flush_eobrun(akey)
            e.ev.append((2, (u // dri - 1) & 7, None))
            pred = [0] * 4
        if sequential:
            for i, c, by, bx in unit:
                t = dc_slot[i]
                pred[i] = e.block((0, t), (1, t), planes[c][by, bx], pred[i])
        elif sc.ss == 0:
            for i, c, by, bx in unit:
                v = int(planes[c][by, bx, 0]) >> sc.al
                if sc.ah:
                    e.bits(v & 1, 1)                              # encode_mcu_DC_refine
                else:
                    s, b = _BitWriter._val(v - pred[i])           # encode_mcu_DC_first: the point transform is an arithmetic shift
                    pred[i] = v
                    e.sym((0, dc_slot[i]), s)
                    e.bits(b, s)
        elif not any_[u]:
            e.end_block(akey, [])                                 # nothing in the band at this bit position: the block joins the run
        elif sc.ah == 0:
            e.ac_first(akey, mag[u], pos[u], sc.al)
        else:
            e.ac_refine(akey, mag[u], pos[u])
    e.flush_eobrun(akey)
    return sos, *e.code(skew)


def progressive(h, w, sampling, planes, qtabs, dqt16=False, wide=False, rst=0, adobe=None, script=None, sof=0xC2, qhead=None,
                overlong_runs=False):
    """Codes planes[c] ([mcuy * vs, mcux * hs, 64] coefficients, natural order, absolute DC) as the scans of `script` (a list of Scan;
    default spectral(): one DC scan, then the bands 1..5 and 6..63 of each component).  Non-interleaved scans code ceil(component
    extent / 8) blocks per axis, interleaved ones whole MCUs, so any image size works.  Each scan gets Huffman tables built from its own
    symbol counts, defined in front of it; wide=True skews them so that the rarer symbols sit on 9..16-bit codes.  Component c uses
    quantisation table c, qtabs[c]; the frame header defines the tables of qhead ({id: values}, default all of them), the script's dqt
    the others.  rst: the restart interval in force from the start.  sof 0xC0 / 0xC1: a sequential frame, every scan 0..63, Ah = Al = 0,
    coding whole blocks of its components.  overlong_runs: an EOB run in front of a restart marker claims 5 more blocks than the interval
    has left; a decoder must end every run at a marker (jdphuff.c process_restart), as libjpeg does."""
    script = spectral(len(sampling)) if script is None else script
    out = _header(h, w, sampling, dict(enumerate(qtabs)) if qhead is None else qhead, dqt16, [], rst, adobe, sof)
    geo = _geometry(h, w, sampling)
    dri = rst
    for sc in script:
        if sc.dqt:
            out += _dqt(sc.dqt, dqt16)
        if sc.rst is not None:
            dri = sc.rst
            out += _seg(0xDD, bytes([dri >> 8, dri & 255]))
        sos, dht, data = _scan_data(sc, planes, sampling, geo, dri, sof != 0xC2, wide, overlong_runs)
        if dht:
            out += _seg(0xC4, dht)
        out += _seg(0xDA, sos) + data
    return bytes(out + b"\xff\xd9")


def segments(stream):
    """(offset, marker, payload) of every marker segment of a stream, in order: a marker walk that skips entropy-coded data"""
    b, pos, out = bytes(stream), 2, []
    while pos + 4 <= len(b) and b[pos + 1] != 0xD9:
        m, L = b[pos + 1], (b[pos + 2] << 8) | b[pos + 3]
        out.append((pos, m, b[pos + 4:pos + 2 + L]))
        pos += 2 + L
        while m == 0xDA and not (b[pos] == 0xFF and b[pos + 1] != 0 and not 0xD0 <= b[pos + 1] <= 0xD7):
            pos += 1
    return out


def scan_starts(stream):
    return [pos for pos, m, _ in segments(stream) if m == 0xDA]


def prefix(stream, k):
    """the stream cut in front of its scan k (k scans kept), with EOI appended"""
    starts = scan_starts(stream)
    return stream if k >= len(starts) else bytes(stream[:starts[k]]) + b"\xff\xd9"


def arena(planes, sampling):
    """per-component planes -> the decoder's coefficient arena: MCU by MCU, in each the blocks of every component, v-major"""
    parts = []
    for p, (hs, vs) in zip(planes, sampling):
        my, mx = p.shape[0] // vs, p.shape[1] // hs
        parts.append(p.reshape(my, vs, mx, hs, 64).transpose(0, 2, 1, 3, 4).reshape(my, mx, vs * hs, 64))
    return np.concatenate(parts, 2).reshape(-1, 64)


def expected(h, w, sampling, planes, script, upto=None):
    """The decoder's arena after the first `upto` scans of script (all by default), absolute DC in slot 0.  A DC first scan leaves the
    value shifted right by Al ARITHMETICALLY (toward -inf) and back, a refinement ORs in the next bit; an AC coefficient last sent with
    point transform Al holds sign * (|v| >> Al << Al), its MAGNITUDE shifted (toward 0).  A coefficient no scan sent is 0: an
    interleaved scan codes whole MCUs, a non-interleaved one ceil(component extent / 8) blocks per axis."""
    _, _, blk = _geometry(h, w, sampling)
    out = []
    for c, p in enumerate(planes):
        v = p.astype(np.int64)
        al = np.full(p.shape[:2] + (64,), -1, np.int64)
        dc = np.zeros(p.shape[:2], np.int64)
        for sc in script[:upto]:
            if c not in sc.comps:
                continue
            bh, bw = p.shape[:2] if len(sc.comps) > 1 else blk[c]
            al[:bh, :bw, [_ZZ[k] for k in range(sc.ss, sc.se + 1)]] = sc.al
            if sc.ss == 0:
                dc[:bh, :bw] = ((v[:bh, :bw, 0] >> sc.al) << sc.al) if sc.ah == 0 else dc[:bh, :bw] | ((v[:bh, :bw, 0] >> sc.al & 1) << sc.al)
        a = np.maximum(al, 0)
        q = np.where(al >= 0, np.sign(v) * ((np.abs(v) >> a) << a), 0)
        q[..., 0] = dc
        out.append(q.astype(np.int16))
    return arena(out, sampling)


def waves(script):
    """the planner's launch count: a scan runs one wave after the latest earlier scan that shares a component AND a coefficient"""
    w = []
    for i, b in enumerate(script):
        w.append(max((w[k] + 1 for k, a in enumerate(script[:i]) if not (a.se < b.ss or b.se < a.ss) and set(a.comps) & set(b.comps)),
                     default=0))
    return max(w) + 1


def complete(script, ncomp, upto=None):
    """every coefficient of every component has received its last bit (Al = 0) within the first `upto` scans"""
    al = np.full((ncomp, 64), -1)
    for sc in script[:upto]:
        for c in sc.comps:
            al[c, sc.ss:sc.se + 1] = sc.al
    return bool((al == 0).all())


# The catalogue.  Each function returns the script for `n` components (frame order 0..n-1).
def spectral(n):
    """spectral selection only: one DC scan, then the bands 1..5 and 6..63 of each component"""
    return [Scan(tuple(range(n)), 0, 0, 0, 0)] + [Scan((c,), ss, se, 0, 0) for c in range(n) for ss, se in ((1, 5), (6, 63))]


def simple(n):
    """libjpeg's jpeg_simple_progression (jcparam.c), the script cv2 writes"""
    a = tuple(range(n))
    if n == 3:
        return [Scan(a, 0, 0, 0, 1), Scan((0,), 1, 5, 0, 2), Scan((2,), 1, 63, 0, 1), Scan((1,), 1, 63, 0, 1), Scan((0,), 6, 63, 0, 2),
                Scan((0,), 1, 63, 2, 1), Scan(a, 0, 0, 1, 0), Scan((2,), 1, 63, 1, 0), Scan((1,), 1, 63, 1, 0), Scan((0,), 1, 63, 1, 0)]
    return ([Scan(a, 0, 0, 0, 1)] + [Scan((c,), ss, se, 0, 2) for c in a for ss, se in ((1, 5), (6, 63))]
            + [Scan((c,), 1, 63, 2, 1) for c in a] + [Scan(a, 0, 0, 1, 0)] + [Scan((c,), 1, 63, 1, 0) for c in a])


def deep(n, al=3):
    """full bands at point transform al, then al refinements of every one: DC interleaved, AC per component"""
    a = tuple(range(n))
    out = [Scan(a, 0, 0, 0, al)] + [Scan((c,), 1, 63, 0, al) for c in a]
    for t in range(al, 0, -1):
        out += [Scan(a, 0, 0, t, t - 1)] + [Scan((c,), 1, 63, t, t - 1) for c in a]
    return out


def per_component_dc(n):
    """one DC scan per component with its own refinements (mozjpeg's shape)"""
    a = range(n)
    return ([Scan((c,), 0, 0, 0, 2) for c in a] + [Scan((c,), 1, 63, 0, 1) for c in a] + [Scan((c,), 0, 0, 2, 1) for c in a]
            + [Scan((c,), 0, 0, 1, 0) for c in a] + [Scan((c,), 1, 63, 1, 0) for c in a])


def subset_dc(n):
    """DC scans that interleave some of the components: Y alone then the chroma together, refined as Y + Cb, then the rest (n >= 3)"""
    return ([Scan((0,), 0, 0, 0, 1), Scan(tuple(range(1, n)), 0, 0, 0, 1)] + [Scan((c,), 1, 63, 0, 1) for c in range(n)]
            + [Scan((0, 1), 0, 0, 1, 0), Scan(tuple(range(2, n)), 0, 0, 1, 0)] + [Scan((c,), 1, 63, 1, 0) for c in range(n)])


def sequential_subset(n):
    """a SEQUENTIAL frame (progressive(..., sof=0xC0)) coded as Y + Cb in one scan and the rest in another (n >= 3)"""
    return [Scan((0, 1), 0, 63, 0, 0), Scan(tuple(range(2, n)), 0, 63, 0, 0)]


def single_coefficient(n):
    """Ss = Se = k for every k from 1 to 63: after the DC scan, one wide wave"""
    return [Scan(tuple(range(n)), 0, 0, 0, 0)] + [Scan((c,), k, k, 0, 0) for c in range(n) for k in range(1, 64)]


def reordered(n):
    """the last component first, bands high to low, the last component's refinement between the first component's first scans, the
    DC refinement last"""
    last, out = n - 1, [Scan((c,), 0, 0, 0, 1) for c in reversed(range(n))]
    for c in reversed(range(n)):
        for i, (ss, se) in enumerate(((33, 63), (6, 32), (1, 5))):
            out.append(Scan((c,), ss, se, 0, 1))
            if c == 0 and i == 0 and n > 1:
                out.append(Scan((last,), 1, 63, 1, 0))
    out += [Scan((c,), 1, 63, 1, 0) for c in reversed(range(n)) if c != last or n == 1]
    return out + [Scan(tuple(range(n)), 0, 0, 1, 0)]


def restarts(n):
    """simple() with restart intervals of 1, 2 and 7 blocks / MCUs, changed between scans and switched off (DRI 0) in the middle"""
    pattern = [1, 2, None, 7, 0, 3, None, 1, 0, 2]
    return [sc._replace(rst=pattern[i % len(pattern)]) for i, sc in enumerate(simple(n))]


def repeated_dc_refinement(n):
    """simple() with its DC refinement sent twice: libjpeg warns of a bogus progression and ORs the same bit in again"""
    sc = simple(n)
    k = next(i for i, x in enumerate(sc) if x.ss == 0 and x.ah)
    return sc[:k + 1] + sc[k:]


def table_slots(n):
    """simple() with its tables in slots 2 and 3 (a DC scan's components take slot, slot + 1, ... mod 4)"""
    return [sc._replace(slot=2 + i % 2) for i, sc in enumerate(simple(n))]


def scan_limit(total, n=3):
    """exactly `total` scans (up to 14 * n + 882 n / 3): each component's DC at Al = 13 with 13 refinements, then single-coefficient
    bands, each sent at some Al and refined down to 0"""
    out = [Scan((c,), 0, 0, 0, 13) for c in range(n)] + [Scan((c,), 0, 0, t, t - 1) for t in range(13, 0, -1) for c in range(n)]
    pairs = [(c, k) for c in range(n) for k in range(1, 64)]
    base, extra = divmod(total - len(out), len(pairs))
    assert 1 <= base and base + (extra > 0) <= 14
    for i, (c, k) in enumerate(pairs):
        al = base + (i < extra) - 1
        out += [Scan((c,), k, k, 0, al)] + [Scan((c,), k, k, t, t - 1) for t in range(al, 0, -1)]
    return out


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
