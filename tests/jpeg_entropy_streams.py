"""Test-only baseline JPEG streams built bit by bit for the entropy stage of jpeg.cu, and a plain model of its synchronisation.

Builder.  Stream() takes chosen DHT tables (code length and symbol per code) and a Huffman table selector per component, and writes
blocks as symbol lists, so that every block has a known bit length: filler blocks move a byte, a block start or a unit end to a chosen
bit.  It controls restart intervals, the pad bits in front of each marker, 0xFF fill bytes before RSTn / EOI and bytes after EOI.

Model.  units() splits a stream into entropy-coded units and un-stuffs them exactly as the decoder's plan and U1 - U3 do.  Unit.walk()
decodes a unit sequentially as every pass of the decoder does (one symbol per step; an invalid code takes 17 bits and symbol 0; a block
ends at z >= 64) and keeps the state (pos, c, z) at every symbol start.  From it:
  * exits(S): the true exit state and completed-block count of every subsequence of S bits (what H2 leaves in each record);
  * spec_exit(o, S): the exit state of the speculative decoder that H1 starts at subsequence o from (c, z) = (0, 0);
  * sync(o, S): the first subsequence whose exit the decoder started at o shares with the true decoder;
  * chain(S): the subsequence at which the true chain of the unit stops, min over o >= 1 of sync(o): the number of subsequences it
    decodes behind its origin.
coefficients() decodes the blocks of a whole stream in MCU order (natural order in each block, absolute DC), as the decoder's arena
holds them after D1.

The decoder's constants are read from its sources, so a change of them moves the cases with it."""
import os
import re
from bisect import bisect_left

import numpy as np

from jpeg_cmyk_streams import _ZZ, _seg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _constant(path, name):
    with open(os.path.join(ROOT, "dali_b200", "csrc", path)) as f:
        return int(re.search(rf"constexpr (?:int|uint32_t) {name} = (\d+);", f.read()).group(1))


SYNC_THREADS = _constant("jpeg.cu", "kSyncThreads")
WRITE_THREADS = _constant("jpeg.cu", "kWriteThreads")
MAX_CHAIN_LEN = _constant("jpeg.cu", "kMaxChainLen")
CHUNK_BYTES = _constant("jpeg_recon.h", "kChunkBytes")
CLEAN_PAD = _constant("jpeg_recon.h", "kCleanPad")
TAIL_COL_WORDS = _constant("jpeg.cu", "kTailColWords")
MAX_LOG2_SUB = _constant("jpeg.cu", "kMaxLog2Sub")
SUB_BYTES = (32, 64, 128)


# ---- tables ------------------------------------------------------------------------------------------------------------------------
def dht(tc_th, codes):
    """DHT payload of [(code length, symbol), ...]: the codes are canonical, so the first listed code of the shortest length is all
    zeros and codes of one length follow the listed order"""
    codes = sorted(codes, key=lambda lv: lv[0])                   # stable: the listed order within a length
    counts = [0] * 16
    for l, _ in codes:
        counts[l - 1] += 1
    return bytes([tc_th] + counts + [v for _, v in codes])


class Table:
    """A Huffman table as the encoder writes it (symbol -> (code, length)) and as the decoder reads it (16-bit window -> length,
    symbol; 17 bits and symbol 0 where no code matches, as libjpeg and the device tables)"""

    def __init__(self, codes):
        self.codes, self.enc = list(codes), {}
        self.lut = np.full(1 << 16, 17 << 8, np.int32)
        code, prev = 0, None
        for l, v in sorted(self.codes, key=lambda lv: lv[0]):
            if prev is not None:
                code = (code + 1) << (l - prev)
            prev = l
            self.enc[v] = (code, l)
            self.lut[code << (16 - l):(code + 1) << (16 - l)] = (l << 8) | v
        self.lut = self.lut.tolist()


# ---- builder -----------------------------------------------------------------------------------------------------------------------
class Stream:
    """One interleaved baseline scan.  sampling[c] = (hs, vs); sel[c] = (DC table, AC table) of component c; tables =
    {0x00: DC0 codes, 0x01: DC1, 0x10: AC0, 0x11: AC1} (lists of (code length, symbol)).  A block is a list of symbols
    [(symbol, magnitude bits)], DC first; add() appends one block of the MCU order and counts its bits."""

    def __init__(self, h, w, sampling, tables, sel, rst=0, fills=None):
        self.h, self.w, self.sampling, self.sel, self.rst = h, w, sampling, sel, rst
        self.fills = fills or {}         # unit -> 0xFF fill bytes in front of the RSTn that ends it
        self.dht = {k: v for k, v in tables.items()}
        self.tab = {k: Table(v) for k, v in tables.items()}
        hmax, vmax = max(s[0] for s in sampling), max(s[1] for s in sampling)
        self.mcux, self.mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
        self.blk_comp = [c for c, (hs, vs) in enumerate(sampling) for _ in range(hs * vs)]
        self.bpm = len(self.blk_comp)
        self.nblocks = self.mcux * self.mcuy * self.bpm
        self.raw, self.acc, self.nbits = bytearray(), 0, 0
        self.bits = 0                    # clean bits written into the current unit
        self.blocks = 0                  # blocks written
        self.unit = 0
        self.unit_raw0 = 0               # offset of the current unit's first byte in `raw`

    # -- bits
    def _put(self, v, n):
        self.bits += n
        self.acc = (self.acc << n) | (v & ((1 << n) - 1))
        self.nbits += n
        while self.nbits >= 8:
            b = (self.acc >> (self.nbits - 8)) & 255
            self.raw.append(b)
            if b == 0xFF:
                self.raw.append(0)
            self.nbits -= 8
        self.acc &= (1 << self.nbits) - 1

    def tables_of(self, k):
        """(DC table, AC table) of block k of the scan"""
        c = self.blk_comp[k % self.bpm]
        return self.tab[self.sel[c][0]], self.tab[0x10 | self.sel[c][1]]

    def add(self, block):
        """block = [(symbol, magnitude bits as a string of '0' / '1'), ...], DC first"""
        assert self.blocks < self.nblocks, "more blocks than the frame has"
        dt, at = self.tables_of(self.blocks)
        for i, (sym, mag) in enumerate(block):
            code, l = (dt if i == 0 else at).enc[sym]
            self._put(code, l)
            if mag:
                self._put(int(mag, 2), len(mag))
        self.blocks += 1
        if self.rst and self.blocks % (self.rst * self.bpm) == 0 and self.blocks < self.nblocks:
            self.end_unit(self.fills.get(self.unit, 0))

    def end_unit(self, fill=0):
        """pad with 1-bits, fill bytes, RSTn"""
        if self.nbits:
            self._put((1 << (8 - self.nbits)) - 1, 8 - self.nbits)
        self.raw += b"\xff" * fill
        self.raw += bytes([0xFF, 0xD0 + (self.unit & 7)])
        self.unit += 1
        self.unit_raw0 = len(self.raw)
        self.bits = 0

    def finish(self, fill_eoi=0, tail=b"", eoi=True, qtab=None):
        assert self.blocks == self.nblocks, f"{self.blocks} of {self.nblocks} blocks written"
        if self.nbits:
            self._put((1 << (8 - self.nbits)) - 1, 8 - self.nbits)
        ncomp = len(self.sampling)
        q = np.ones(64, np.int64) if qtab is None else qtab
        out = bytearray(b"\xff\xd8")
        out += _seg(0xDB, b"".join(bytes([t]) + bytes(int(q[_ZZ[k]]) for k in range(64)) for t in range(min(ncomp, 2))))
        comp = b"".join(bytes([c + 1, (hs << 4) | vs, min(c, 1)]) for c, (hs, vs) in enumerate(self.sampling))
        out += _seg(0xC0, bytes([8, self.h >> 8, self.h & 255, self.w >> 8, self.w & 255, ncomp]) + comp)
        for k in sorted(self.dht):
            out += _seg(0xC4, dht(k, self.dht[k]))
        if self.rst:
            out += _seg(0xDD, bytes([self.rst >> 8, self.rst & 255]))
        out += _seg(0xDA, bytes([ncomp]) + b"".join(bytes([c + 1, (d << 4) | a]) for c, (d, a) in enumerate(self.sel)) + bytes([0, 63, 0]))
        return bytes(out + self.raw + b"\xff" * fill_eoi + (b"\xff\xd9" if eoi else b"") + tail)


# ---- model -------------------------------------------------------------------------------------------------------------------------
def _parse(stream):
    """(DC / AC tables by id, [(DC id, AC id)] per block of the MCU, blocks per frame, restart interval, scan start)"""
    pos, tabs, rst, comps = 2, {}, 0, None
    while True:
        m, L = stream[pos + 1], (stream[pos + 2] << 8) | stream[pos + 3]
        p = stream[pos + 4:pos + 2 + L]
        if m == 0xC4:
            o = 0
            while o < len(p):
                counts = p[o + 1:o + 17]
                vals = p[o + 17:o + 17 + sum(counts)]
                lens = [l + 1 for l in range(16) for _ in range(counts[l])]
                tabs[p[o]] = Table(list(zip(lens, vals)))
                o += 17 + len(vals)
        elif m == 0xC0:
            h, w, n = (p[1] << 8) | p[2], (p[3] << 8) | p[4], p[5]
            comps = [(p[7 + 3 * i] >> 4, p[7 + 3 * i] & 15) for i in range(n)]
        elif m == 0xDD:
            rst = (p[0] << 8) | p[1]
        elif m == 0xDA:
            sel = [(p[2 + 2 * i] >> 4, p[2 + 2 * i] & 15) for i in range(p[0])]
            break
        pos += 2 + L
    blk = [(tabs[sel[c][0]], tabs[0x10 | sel[c][1]], c) for c, (hs, vs) in enumerate(comps) for _ in range(hs * vs)]
    hmax, vmax = max(c[0] for c in comps), max(c[1] for c in comps)
    mcux, mcuy = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    return blk, mcux * mcuy, rst, pos + 2 + L, comps, mcux


class Unit:
    """One entropy-coded unit: `raw` (its staged bytes), `clean` (un-stuffed), `raw_off` (offset of its first byte behind the scan
    start, the staged offset modulo 16), `nblocks` (blocks it codes) and the per-block tables of the MCU"""

    def __init__(self, raw, raw_off, blk, nblocks):
        self.raw, self.raw_off, self.blk, self.nblocks = raw, raw_off, blk, nblocks
        keep = [i for i in range(len(raw)) if not (raw[i] == 0 and i > 0 and raw[i - 1] == 0xFF)]
        self.clean = bytes(raw[i] for i in keep)
        self.clean_bits = 8 * len(self.clean)
        self._buf = self.clean + bytes(8)
        self._walk = None

    def _step(self, pos, c, z):
        """one symbol: (bits, zig-zag advance, magnitude size, symbol code length)"""
        b = pos >> 3
        if b + 4 <= len(self._buf):
            win = (int.from_bytes(self._buf[b:b + 4], "big") << (pos & 7) >> 16) & 0xFFFF
        else:
            win = 0
        dt, at, _ = self.blk[c]
        e = (dt if z == 0 else at).lut[win]
        l, sym = e >> 8, e & 255
        s = sym & 15
        if z == 0:
            adv = 1
        else:
            r = sym >> 4
            adv = (16 if r == 15 else 64) if s == 0 else r + 1
        return l + s, adv, s, l

    def _bits(self, pos, n):
        v = 0
        for k in range(n):
            p = pos + k
            v = (v << 1) | ((self._buf[p >> 3] >> (7 - (p & 7))) & 1 if (p >> 3) < len(self._buf) else 0)
        return v

    def walk(self):
        """the true decoder's state at every symbol start, through the whole clean stream: arrays pos, c, z, and `ends` (1 where the
        symbol starting there is the last of its block)"""
        if self._walk is None:
            bpm = len(self.blk)
            P, Cs, Zs, E = [], [], [], []
            pos = c = z = 0
            while pos < self.clean_bits:
                bits, adv, _, _ = self._step(pos, c, z)
                P.append(pos); Cs.append(c); Zs.append(z)
                pos += bits
                z += adv
                E.append(1 if z >= 64 else 0)
                if z >= 64:
                    z, c = 0, (c + 1) % bpm
            P.append(pos); Cs.append(c); Zs.append(z); E.append(0)
            self._walk = (np.array(P, np.int64), np.array(Cs), np.array(Zs), np.array(E, np.int64))
        return self._walk

    def nsub(self, S):
        return -(-self.clean_bits // S)

    def exits(self, S):
        """per subsequence of S bits: (exit pos, c, z, completed blocks), as the records hold them once synchronised"""
        P, Cs, Zs, E = self.walk()
        ce = np.concatenate([[0], np.cumsum(E)])
        n = self.nsub(S)
        ends = np.minimum((np.arange(n) + 1) * S, self.clean_bits)
        idx = np.searchsorted(P, ends)                              # first symbol start >= the end
        prev = np.concatenate([[0], idx[:-1]])
        return P[idx], Cs[idx], Zs[idx], ce[idx] - ce[prev]

    def pad_bits(self):
        """clean bits behind the end of the unit's last block"""
        P, Cs, Zs, _ = self.walk()
        starts = P[:-1][Zs[:-1] == 0]
        return self.clean_bits - int(starts[self.nblocks]) if len(starts) > self.nblocks else 0

    def extra_symbols(self):
        """symbols the passes decode behind the unit's last block (pad bits, fill bytes, bytes after EOI)"""
        P, Cs, Zs, _ = self.walk()
        starts = P[:-1][Zs[:-1] == 0]
        return 0 if len(starts) <= self.nblocks else int((P[:-1] >= starts[self.nblocks]).sum())

    def spec(self, o, S, bound=None):
        """the decoder H1 starts at subsequence o from (c, z) = (0, 0): (its exit state at subsequence o, the subsequence from which on
        it shares every exit with the true decoder, or None if that is not within `bound` subsequences)"""
        P, Cs, Zs, _ = self.walk()
        true_at = dict(zip(P.tolist(), zip(Cs.tolist(), Zs.tolist())))
        bpm = len(self.blk)
        pos, c, z, prev = o * S, 0, 0, None
        own_end = min((o + 1) * S, self.clean_bits)
        own = None
        limit = self.clean_bits if bound is None else min(self.clean_bits, (o + bound + 1) * S)
        x = None
        while True:
            if own is None and pos >= own_end:
                own = (pos, c, z)
            if true_at.get(pos) == (c, z):
                x = o if prev is None else max(o, prev // S)
                break
            if pos >= limit:
                break
            bits, adv, _, _ = self._step(pos, c, z)
            prev = pos
            pos += bits
            z += adv
            if z >= 64:
                z, c = 0, (c + 1) % bpm
        if own is None:                                             # synchronised inside its own subsequence
            i = bisect_left(P.tolist(), own_end)
            own = (int(P[i]), int(Cs[i]), int(Zs[i]))
        return own, x

    def spec_exit(self, o, S):
        return self.spec(o, S, bound=0)[0]

    def sync(self, o, S, bound=None):
        return self.spec(o, S, bound)[1]

    def chain(self, S, bound=None):
        """the subsequence at which the true chain stops: the first one whose record some speculative decoder (origin >= 1) already
        filled with the true state; None if there is none within `bound`"""
        best = None
        o = 1
        while o < self.nsub(S) and (best is None or o < best):
            b = None if best is None and bound is None else (bound if best is None else best - o)
            x = self.sync(o, S, b)
            if x is not None and (best is None or x < best):
                best = x
            o += 1
        return best


def units(stream):
    """the entropy-coded units of a baseline stream, split and staged as the decoder's plan does (trimmed at a final EOI, split at
    every FF Dn with n in 0..7 found by a byte search)"""
    blk, nmcu, rst, sb, comps, mcux = _parse(stream)
    se = len(stream)
    if se >= sb + 2 and stream[se - 2] == 0xFF and stream[se - 1] == 0xD9:
        se -= 2
    bpm = len(blk)
    out = []
    if rst == 0:
        return [Unit(stream[sb:se], 0, blk, nmcu * bpm)]
    b, q, mcu0 = sb, sb, 0
    while True:
        f = stream.find(b"\xff", q, se)
        if f < 0 or f + 1 >= se:
            break
        if 0xD0 <= stream[f + 1] <= 0xD7:
            mcus = min(rst, nmcu - mcu0)
            if mcus > 0:
                out.append(Unit(stream[b:f], b - sb, blk, mcus * bpm))
            mcu0 += mcus
            b = q = f + 2
        else:
            q = f + 1
    if mcu0 < nmcu:
        out.append(Unit(stream[b:se], b - sb, blk, min(rst, nmcu - mcu0) * bpm))
    return out


def planner_sub_bytes(lengths):
    """the subsequence size the decoder's plan picks for a batch of streams of these lengths when none is pinned (the rule and its
    threshold read from jpeg.cu): the largest size that still gives the batch enough subsequences, 32 bytes at least"""
    with open(os.path.join(ROOT, "dali_b200", "csrc", "jpeg.cu")) as f:
        want = int(re.search(r"\(total_len >> log2_bytes\) < (\d+)\)", f.read()).group(1))
    log2_bytes, total = MAX_LOG2_SUB - 3, sum(lengths)
    while log2_bytes > 5 and (total >> log2_bytes) < want:
        log2_bytes -= 1
    return 1 << log2_bytes


def table_key(stream):
    """the Huffman tables a sequential (SOF0 / SOF1) stream has at its scan (DHT payload per class and id), as the plan keys its table
    sets; "progressive" for a progressive stream (the plan gives those one zeroed set); None for a stream without a set"""
    if stream[:2] != b"\xff\xd8":
        return None
    pos, key, sof = 2, {}, None
    while pos + 4 <= len(stream):
        m, L = stream[pos + 1], (stream[pos + 2] << 8) | stream[pos + 3]
        p = stream[pos + 4:pos + 2 + L]
        if 0xC0 <= m <= 0xCF and m not in (0xC4, 0xC8, 0xCC):
            sof = m
        elif m == 0xC4:
            o = 0
            while o < len(p):
                n = 17 + sum(p[o + 1:o + 17])
                key[p[o]] = bytes(p[o:o + n])
                o += n
        elif m == 0xDA:
            break
        pos += 2 + L
    if sof == 0xC2:
        return "progressive"
    return tuple(key.get(k) for k in (0x00, 0x01, 0x10, 0x11)) if sof in (0xC0, 0xC1) else None


def walk_paths(batch):
    """per sample of a batch: 'shared' when the chain walk reads its tables from the copy in shared memory (the sample's table set is
    sample 0's; a sample without a set of its own, such as a PNG, points at set 0), 'global' when it reads them from global memory,
    None for a sample without baseline units"""
    keys = [table_key(s) for s in batch]
    sets = {}
    for k in keys:
        if k is not None:
            sets.setdefault(k, len(sets))
    lead = 0 if keys[0] is None else sets[keys[0]]
    return [None if k is None or k == "progressive" else ("shared" if sets[k] == lead else "global") for k in keys]


def coefficients(stream):
    """the quantised blocks of a stream in MCU order, natural order, absolute DC (the decoder's arena after D1), decoded from the
    units by the model"""
    us = units(stream)
    blk = us[0].blk
    ncomp = max(b[2] for b in blk) + 1
    out = []
    for u in us:
        pred = [0] * ncomp
        pos = 0
        for k in range(u.nblocks):
            c = k % len(blk)
            b = np.zeros(64, np.int16)
            z = 0
            while z < 64:
                bits, adv, s, l = u._step(pos, c, z)
                v = u._bits(pos + l, s)
                if s and v < (1 << (s - 1)):
                    v -= (1 << s) - 1
                if z == 0:
                    pred[blk[c][2]] += v if s else 0
                    b[0] = np.int16(((pred[blk[c][2]] + 32768) & 0xFFFF) - 32768)
                elif s:
                    b[_ZZ[min(z + adv - 1, 63)]] = v
                pos += bits
                z += adv
            out.append(b)
    return np.stack(out)


def mcu_order(stream):
    """po.jpeg_coeffs of a stream in MCU order (the oracle)"""
    from oracle import pyoracle as po
    comps = po.jpeg_coeffs(stream)
    info = po.jpeg_info(stream)
    hs, vs = info["hs"], info["vs"]
    blocks = []
    for my in range(info["mcuy"]):
        for mx in range(info["mcux"]):
            for c in range(info["ncomp"]):
                for v in range(vs[c]):
                    for h in range(hs[c]):
                        blocks.append(comps[c][my * vs[c] + v, mx * hs[c] + h])
    return np.stack(blocks)


# ---- cases -------------------------------------------------------------------------------------------------------------------------
# Placement tables (gray, table 0).  DC: '0' category 0, '10' category 1.  AC: '00' EOB, '01' (0, 9), '10' (0, 8), '110' (0, 7).  No
# table has an all-ones code (libjpeg refuses such tables).  Every block ends with the EOB '00', so pad bits never complete a 0xFF byte;
# a (0, 8) symbol with an all-ones magnitude makes a 0xFF byte where it is placed; pad bits (ones) followed by the zeros behind a unit
# decode into extra symbols ('10': a category-1 DC).  WIDE adds 16-bit codes (DC category 11, AC (0, 10)) for the longest block.
PLACE = {0x00: [(1, 0), (2, 1)], 0x10: [(2, 0x00), (2, 0x09), (2, 0x08), (3, 0x07)]}
WIDE = {0x00: [(1, 0), (2, 1), (16, 11)], 0x10: [(2, 0x00), (2, 0x09), (3, 0x07), (16, 0x0A)]}
GRAY, SEL0 = [(1, 1)], [(0, 0)]


def _extras(l9, l7):
    """extra bits over the 3-bit empty block -> (a (0, 9) symbols, b (0, 7) symbols, category-1 DC)"""
    ex = {}
    for a in range(63):
        for b in range(63 - a):
            for d in (0, 1):
                ex.setdefault(l9 * a + l7 * b + 2 * d, (a, b, d))
    t0 = 1 + max(x for x in range(200) if x not in ex)           # every extra from t0 to top has a block
    top = t0
    while top + 1 in ex:
        top += 1
    ex = {e: v for e, v in ex.items() if e <= top}
    small = sorted(e for e in ex if e < 2 * t0)
    return ex, top, {a + b for a in small for b in small}, t0


class Placer:
    """fills a Stream (PLACE or WIDE tables, gray) with blocks of chosen lengths; the DC differences alternate +1 / -1"""

    def __init__(self, st):
        self.st, self.sign = st, 0
        self.ex, self.top, self.ex2, self.t0 = _extras(st.tab[0x10].enc[0x09][1] + 9, st.tab[0x10].enc[0x07][1] + 7)

    def block(self, extra):
        a, b, d = self.ex[extra]
        blk = [(1, "01"[self.sign]) if d else (0, "")]
        self.sign ^= d
        blk += [(0x09, "100000000")] * a + [(0x07, "1000000")] * b
        self.st.add(blk + [(0x00, "")])

    def fill(self, nblk, bits):
        """nblk blocks of `bits` clean bits in all (planned first: nothing is written when they cannot be had)"""
        rest, plan = bits - 3 * nblk, []
        for k in range(nblk, 0, -1):
            e = min(max(rest, 0), self.top)
            while e > 0 and (e not in self.ex or not self._feasible(rest - e, k - 1)):
                e -= 1
            plan.append(e)
            rest -= e
        assert rest == 0, (nblk, bits)
        for e in plan:
            self.block(e)

    def _feasible(self, r, m):
        if m == 0 or r > m * self.top:
            return r == 0
        return r in self.ex if m == 1 else (r in self.ex2 or r >= 2 * self.t0)

    def to_bit(self, bit, nblk):
        """nblk blocks that end exactly at clean bit `bit` of the current unit"""
        self.fill(nblk, bit - self.st.bits)

    def ones(self, n):
        """a block of n (0, 8) symbols with all-ones magnitudes (PLACE): its bits [3, 11) are ones, and so are [10 k + 3, 10 k + 11)"""
        self.st.add([(0, "")] + [(0x08, "11111111")] * n + [(0x00, "")])

    def widest(self):
        """the longest block (WIDE): a 16-bit DC code + 11 bits, 63 x ((0, 10) 16-bit code + 10 bits) = 1665 bits"""
        self.st.add([(11, "10000000001")] + [(0x0A, "1000000001")] * 63)


def unit_bytes(nbytes, nblk, st, pl):
    """nblk more blocks, so that the current unit's raw length is nbytes (no 0xFF inside: a pad of 0..7 ones)"""
    for pad in range(8):
        bits = 8 * nbytes - pad - st.bits
        if bits >= 3 * nblk:
            try:
                pl.fill(nblk, bits)
                return
            except AssertionError:
                continue
    raise AssertionError("no fill")


def stuffing_stream():
    """U1 - U3.  A gray image with a restart interval of 128 blocks, one unit per case:
      units 0-5: a 0xFF 0x00 pair whose 0xFF is raw byte 4093 .. 4098 of the unit (around the first chunk boundary);
      unit 6: stuffed pairs at raw bytes 4093 .. 4094 and 4096 .. 4097, on both sides of the boundary;  unit 7: 0xFF at raw byte 8191 (second chunk boundary);
      units 8-12: raw lengths 4095, 4096, 4097, 8191, 8193 bytes;  unit 13: two thirds of its raw bytes are stuffed pairs;
      unit 14: the rest.  Returns (stream, {unit: (what, where)})."""
    R, per_row = 128, 8
    st = Stream(8 * (R * 15 // per_row), 8 * per_row, GRAY, PLACE, SEL0, rst=R)
    pl = Placer(st)
    notes = {}

    def ff_at(raw_off, nblk=100):
        # block start p so that its bits [p + 3, p + 11) are clean byte q
        q = raw_off - st.raw[st.unit_raw0:].count(b"\xff\x00")
        pl.to_bit(8 * q - 3, nblk)
        pl.ones(1)

    for u, off in enumerate(range(4093, 4099)):
        ff_at(off)
        notes[u] = ("ff", off)
        pl.fill(R - 101, 8 * 5000 - st.bits)
    ff_at(4093)
    ff_at(4096, 1)
    notes[6] = ("ff2", 4093)
    pl.fill(R - 103, 8 * 5000 - st.bits)
    ff_at(8191)
    notes[7] = ("ff", 8191)
    pl.fill(R - 101, 8 * 8500 - st.bits)
    for u, n in zip(range(8, 13), (4095, 4096, 4097, 8191, 8193)):
        unit_bytes(n, R, st, pl)
        notes[u] = ("len", n)
    pl.to_bit(8 * 16 - 3, 2)
    for _ in range((R - 2) // 2):               # 13 + 3 bits: every second clean byte is 0xFF
        pl.ones(1)
        pl.block(0)
    notes[13] = ("stuffed", None)
    pl.fill(st.nblocks - st.blocks, 8 * 1000)
    return st.finish(), notes


def small_units_stream(nunits=48, fill=0):
    """U1 - U3: units of 1 .. 8 raw bytes (two blocks each), so that their staged offsets take every residue mod 16; fill: 0xFF fill
    bytes in front of every RSTn and of the EOI"""
    st = Stream(8, 8 * 2 * nunits, GRAY, PLACE, SEL0, rst=2, fills={u: fill for u in range(nunits)})
    pl = Placer(st)
    sizes = [1 + (k * 5) % 8 for k in range(nunits)]
    for n in sizes:
        unit_bytes(n, 2, st, pl)
    return st.finish(fill_eoi=fill), sizes


def subseq_stream(nsub, sub_bytes, width=64):
    """H1: one unit of exactly nsub subsequences of sub_bytes (its clean length nsub * sub_bytes, a multiple of 16)"""
    bits = 8 * nsub * sub_bytes
    per_row = width // 8
    nblk = (-(-bits // 600) // per_row + 1) * per_row
    st = Stream(8 * (nblk // per_row), width, GRAY, PLACE, SEL0)
    Placer(st).fill(nblk, bits)
    return st.finish()


def sync_edge_stream(sub_bytes, nunits=10):
    """H1 / H3 (WIDE tables): a restart interval of 128 blocks; units 0-4 are 51 subsequences long each, so that unit 5 begins in the
    last column of sync block 0 (image subsequence 255), whose decoder is the last one of its CTA.  In that column the widest block
    (1665 bits) starts 8 bits before its end: H1's thread 255 decodes its first symbols from the first look-ahead column staged behind
    the sync block, and H3 completes it 208 bytes into sync block 1 from global memory.  The following units are 60 subsequences long."""
    S, R = 8 * sub_bytes, 128
    st = Stream(8 * (R * nunits // 8), 64, GRAY, WIDE, SEL0, rst=R)
    pl = Placer(st)
    for _ in range(5):
        unit_bytes(51 * sub_bytes, R, st, pl)
    pl.to_bit(S - 8, 10)
    pl.widest()
    unit_bytes(60 * sub_bytes, R - 11, st, pl)
    while st.blocks < st.nblocks:
        unit_bytes(60 * sub_bytes, min(R, st.nblocks - st.blocks), st, pl)
    return st.finish()


def write_edge_stream(sub_bytes):
    """H2b / H3 (WIDE tables, one unit): the widest block starts 8 bits before the end of image subsequence WRITE_THREADS - 1 and of
    2 WRITE_THREADS - 1, the last subsequences of write blocks 0 and 1, and spans the next 1665 bits: up to 8 subsequences, all but
    the first without a block start of their own"""
    S = 8 * sub_bytes
    ends = [(k * WRITE_THREADS - 1) * S + S - 8 for k in (1, 2)]
    per_row, top = 8, 600
    nblk = [-(-(ends[0]) // top), -(-(ends[1] - ends[0] - 1665) // top)]
    tail = per_row - (nblk[0] + nblk[1] + 2) % per_row + per_row
    st = Stream(8 * ((nblk[0] + nblk[1] + 2 + tail) // per_row), 8 * per_row, GRAY, WIDE, SEL0)
    pl = Placer(st)
    for e, n in zip(ends, nblk):
        pl.to_bit(e, n)
        pl.widest()
    pl.fill(tail, 400 * tail)
    return st.finish()


def pad_stream():
    """H2b / H3: a restart interval of 2 blocks and units of 8 clean bytes whose last block ends 1 .. 7 bits before the unit's end:
    pad bits of every length, which decode into extra symbols ('1' then the zeros behind the unit: a category-1 DC)"""
    st = Stream(8, 8 * 2 * 8, GRAY, PLACE, SEL0, rst=2)
    pl = Placer(st)
    for pad in (1, 2, 3, 4, 5, 6, 7, 0):
        pl.fill(2, 64 - pad)
    return st.finish()


# Long chains.  A segment whose bits are all zero, under tables that hold one code each (DC: category 0; AC: (0, s)), is decoded alike
# from every bit: each decoder parses it as the true decoder does, shifted by its start.  A decoder started at an MCU phase other than 0
# never meets the true one, so the speculative decoder of subsequence o synchronises at once when o * S = 0 (mod P), P the MCU's bits,
# and never otherwise: the true chain stops at the first such o.  P = q 2^a with q odd gives o = q 2^max(0, a - log2 S).
def zero_chain(P, S):
    """the subsequence (of S bits) at which the true chain of an all-zero segment of P-bit MCUs stops"""
    o = 1
    while (o * S) % P:
        o += 1
    return o


def zero_layout(P):
    """(sampling, selectors, {table: codes}) of an MCU of exactly P bits under one-code tables: gray (P = d + 63 a) or 4:2:0 with Y and
    Cr on tables 0 and Cb on tables 1 (P = 5 (d0 + 63 a0) + d1 + 63 a1); d = DC code length 1..16, a = AC code length + size, 2..26"""
    for d in range(1, 17):
        if (P - d) % 63 == 0 and 2 <= (P - d) // 63 <= 26:
            a = (P - d) // 63
            al = max(1, a - 10)
            return GRAY, SEL0, {0x00: [(d, 0)], 0x10: [(al, a - al)]}
    for a0 in range(26, 1, -1):
        for d0 in range(16, 0, -1):
            r = P - 5 * (d0 + 63 * a0)
            for d1 in range(1, 17):
                if r - d1 > 0 and (r - d1) % 63 == 0 and 2 <= (r - d1) // 63 <= 26:
                    a1 = (r - d1) // 63
                    l0, l1 = max(1, a0 - 10), max(1, a1 - 10)
                    tabs = {0x00: [(d0, 0)], 0x01: [(d1, 0)], 0x10: [(l0, a0 - l0)], 0x11: [(l1, a1 - l1)]}
                    return [(2, 2), (1, 1), (1, 1)], [(0, 0), (1, 1), (0, 0)], tabs
    raise ValueError(P)


def zero_stream(P, nmcu_min):
    """an all-zero entropy-coded segment of P-bit MCUs, at least nmcu_min of them"""
    sampling, sel, tabs = zero_layout(P)
    m = 8 * max(s[0] for s in sampling)
    mx = 16 if nmcu_min >= 256 else max(1, min(nmcu_min, 8))
    my = -(-nmcu_min // mx)
    st = Stream(m * my, m * mx, sampling, tabs, sel)
    for k in range(st.nblocks):
        dt, at = st.tables_of(k)
        (s_ac,) = at.enc
        st.add([(0, "")] + [(s_ac, "0" * (s_ac & 15))] * 63)
    return st.finish()
