"""CPU tests of the progressive-JPEG entropy stage: the PRODUCT's planner and scan decoder (dali_b200/csrc/jpeg_prog_plan.h +
jpeg_prog_core.h -- the body of the CUDA kernels) compiled for the host by tools/emul/jpeg_prog_emul.cc.  A progressive stream and the
baseline stream of the same image, quality and sampling hold the same quantised coefficients (same DCT + quantisation, different entropy
coding), so the coefficients decoded here must equal those the oracle decodes from the baseline twin -- bit for bit, for every sampling,
with and without restart intervals.  No GPU and no device code runs here."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from oracle import pyoracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emul") / "libjpegprog.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-I/usr/local/cuda/include",
                        os.path.join(ROOT, "tools", "emul", "jpeg_prog_emul.cc"), "-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return C.CDLL(out)


def decode(lib, stream):
    b = np.frombuffer(bytes(stream), np.uint8)
    info = (C.c_int * 8)()
    rc = lib.emul_jpeg_progressive(b.ctypes.data_as(C.c_void_p), C.c_size_t(b.size), None, info)
    if rc:
        return rc, None, None
    coef = np.zeros((info[1] * info[2] * info[3], 64), np.int16)
    rc = lib.emul_jpeg_progressive(b.ctypes.data_as(C.c_void_p), C.c_size_t(b.size), coef.ctypes.data_as(C.c_void_p), info)
    return rc, coef, dict(ncomp=info[0], mcux=info[1], mcuy=info[2], bpm=info[3], nscans=info[4], nwaves=info[5], truncated=info[6])


def mcu_order(stream):
    """the oracle's per-component coefficient planes of a BASELINE stream, rearranged into the decoder's arena order"""
    comps, info = po.jpeg_coeffs(stream), po.jpeg_info(stream)
    hs, vs = info["hs"], info["vs"]
    blocks = []
    for my in range(info["mcuy"]):
        for mx in range(info["mcux"]):
            for c in range(info["ncomp"]):
                for v in range(vs[c]):
                    for h in range(hs[c]):
                        blocks.append(comps[c][my * vs[c] + v, mx * hs[c] + h])
    return np.stack(blocks)


def twins(img, quality, sampling=None, rst=0):
    import cv2
    p = [cv2.IMWRITE_JPEG_QUALITY, quality]
    if sampling is not None:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sampling]
    if rst:
        p += [cv2.IMWRITE_JPEG_RST_INTERVAL, rst]
    base = cv2.imencode(".jpg", img, p)[1].tobytes()
    prog = cv2.imencode(".jpg", img, p + [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    assert b"\xff\xc2" in prog and b"\xff\xc2" not in base[:600]
    return base, prog


def synth(h, w, seed):
    import cv2
    r = np.random.default_rng(seed)
    lo = r.uniform(0, 255, (max(2, h // 32), max(2, w // 32), 3)).astype(np.float32)
    return np.clip(cv2.resize(lo, (w, h), interpolation=cv2.INTER_CUBIC) + r.normal(0, 5, (h, w, 3)), 0, 255).astype(np.uint8)


def test_coefficients_equal_the_baseline_twin(emul):
    import cv2
    ss = [cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422,
          cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_411]
    k = 0
    for (h, w) in [(48, 64), (33, 47), (97, 61), (136, 200), (17, 23), (8, 8), (1, 1)]:
        for s in ss:
            for q in (30, 90):
                for rst in (0, 3):
                    k += 1
                    base, prog = twins(synth(h, w, k), q, s, rst)
                    rc, got, info = decode(emul, prog)
                    assert rc == 0 and info["truncated"] == 0, (h, w, s, q, rst, rc, info)
                    assert info["nscans"] == 10 and info["nwaves"] == 3, info        # libjpeg's jpeg_simple_progression script
                    assert np.array_equal(got, mcu_order(base)), (h, w, s, q, rst)
    for (h, w) in [(20, 20), (65, 130)]:                                              # single component: six scans
        base, prog = twins(synth(h, w, 99)[..., 0], 85)
        rc, got, info = decode(emul, prog)
        assert rc == 0 and info["ncomp"] == 1 and info["nscans"] == 6 and np.array_equal(got, mcu_order(base))


def test_large_image_and_decoded_pixels_equal_libjpeg(emul):
    """1080p 4:2:0: coefficients equal the twin's, hence the shared stages (pinned elsewhere) produce libjpeg's pixels; checked here
    end to end through the oracle's IDCT + upsampling + colour stages against cv2.imdecode of the PROGRESSIVE stream."""
    import cv2
    base, prog = twins(synth(1080, 1920, 5), 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420)
    rc, got, info = decode(emul, prog)
    assert rc == 0 and np.array_equal(got, mcu_order(base))
    want = cv2.imdecode(np.frombuffer(prog, np.uint8), cv2.IMREAD_COLOR)[..., ::-1]
    assert np.array_equal(po.jpeg_decode(base), want)


def test_truncated_and_malformed_streams_return_a_status(emul):
    import cv2
    base, prog = twins(synth(64, 80, 7), 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420)
    full = mcu_order(base)
    last = prog.rfind(b"\xff\xda")
    rc, got, info = decode(emul, prog[: (last + len(prog)) // 2])                   # cut inside the last scan (Y, last bit)
    assert rc == 0 and info["truncated"] == 1 and not np.array_equal(got, full)
    assert np.array_equal(got >> 1, full >> 1) or np.array_equal((got + (got < 0)) >> 1, (full + (full < 0)) >> 1)
    rc, got, info = decode(emul, prog[: last - 3])                                # cut between two scans: the progression is incomplete
    assert rc == 0 and info["truncated"] == 1
    assert decode(emul, b"\xff\xd8\xff\xd9")[0] != 0
    bad = bytearray(prog)
    i = bad.find(b"\xff\xda")
    bad[i + 4 + 2 * bad[i + 4] + 1] = 70                                           # Ss = 70
    assert decode(emul, bytes(bad))[0] == 4


def test_dc_scan_interleaving_a_subset_of_the_components_decodes(emul):
    """the DC scan split into Y + Cb interleaved and Cr alone (T.81 G.1.1.1 allows a scan to interleave a subset of the components):
    the twin's coefficients"""
    import cv2
    import jpeg_extreme_streams as xs
    base, _ = twins(synth(64, 80, 7), 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420)
    full = mcu_order(base)
    planes, info = po.jpeg_coeffs(base), po.jpeg_info(base)
    sampling = [(info["hs"][c], info["vs"][c]) for c in range(3)]
    script = [xs.Scan((0, 1), 0, 0, 0, 0), xs.Scan((2,), 0, 0, 0, 0)] + [xs.Scan((c,), 1, 63, 0, 0) for c in range(3)]
    two = xs.progressive(64, 80, sampling, planes, [np.ones(64, np.int64)] * 3, script=script)
    rc, got, info = decode(emul, two)
    assert rc == 0 and info["truncated"] == 0 and np.array_equal(got, full)


# ---- sequential frames coded in several scans (one per component) -----------------------------------------------------------------
def to_multiscan_baseline(stream, rst=0):
    """Re-codes the entropy data of an interleaved baseline stream as one scan per component (legal in a sequential frame, T.81 A.2):
    same headers and Huffman tables, the coefficients the oracle decodes, a plain Huffman encoder.  Test-only."""
    b = bytes(stream)
    info = po.jpeg_info(b)
    comps = po.jpeg_coeffs(b)
    ncomp, W, H = info["ncomp"], info["width"], info["height"]
    hmax, vmax = max(info["hs"][:ncomp]), max(info["vs"][:ncomp])
    zz = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
          35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]
    # marker walk: tables, component ids, the scan header
    pos, tables, cids, sos = 2, {}, [], None
    while True:
        assert b[pos] == 0xFF
        m, L = b[pos + 1], (b[pos + 2] << 8) | b[pos + 3]
        seg = b[pos + 4:pos + 2 + L]
        if m == 0xC4:
            o = 0
            while o < len(seg):
                tc_th, bits = seg[o], seg[o + 1:o + 17]
                vals = seg[o + 17:o + 17 + sum(bits)]
                code, k, enc = 0, 0, {}
                for l in range(1, 17):
                    for _ in range(bits[l - 1]):
                        enc[vals[k]] = (code, l)
                        code += 1
                        k += 1
                    code <<= 1
                tables[tc_th] = enc
                o += 17 + len(vals)
        elif m == 0xC0:
            cids = [seg[6 + 3 * c] for c in range(ncomp)]
        elif m == 0xDA:
            sos = seg
            head = b[:pos]
            break
        pos += 2 + L
    tdta = {sos[1 + 2 * i]: sos[2 + 2 * i] for i in range(sos[0])}
    out = bytearray(head)
    if rst:
        out += bytes([0xFF, 0xDD, 0, 4, rst >> 8, rst & 255])
    for c in range(ncomp):
        cw, ch = (W * info["hs"][c] + hmax - 1) // hmax, (H * info["vs"][c] + vmax - 1) // vmax
        wb, hb = (cw + 7) // 8, (ch + 7) // 8
        dc_t, ac_t = tables[tdta[cids[c]] >> 4], tables[0x10 | (tdta[cids[c]] & 15)]
        out += bytes([0xFF, 0xDA, 0, 8, 1, cids[c], tdta[cids[c]], 0, 63, 0])
        acc, nb, pred, data, count = 0, 0, 0, bytearray(), 0

        def put(v, n):
            nonlocal acc, nb
            acc = (acc << n) | (v & ((1 << n) - 1))
            nb += n
            while nb >= 8:
                byte = (acc >> (nb - 8)) & 255
                data.append(byte)
                if byte == 0xFF:
                    data.append(0)
                nb -= 8

        def put_val(v):
            s = int(abs(v)).bit_length()
            return s, (v if v >= 0 else v + (1 << s) - 1)
        for by in range(hb):
            for bx in range(wb):
                if rst and count and count % rst == 0:
                    if nb:
                        put((1 << (8 - nb)) - 1, 8 - nb)
                    data += bytes([0xFF, 0xD0 + ((count // rst - 1) & 7)])
                    pred = 0
                count += 1
                blk = comps[c][by, bx]
                d = int(blk[0]) - pred
                pred = int(blk[0])
                s, bits_ = put_val(d)
                put(*dc_t[s])
                if s:
                    put(bits_, s)
                run = 0
                for k in range(1, 64):
                    v = int(blk[zz[k]])
                    if v == 0:
                        run += 1
                        continue
                    while run > 15:
                        put(*ac_t[0xF0])
                        run -= 16
                    s, bits_ = put_val(v)
                    put(*ac_t[(run << 4) | s])
                    put(bits_, s)
                    run = 0
                if run:
                    put(*ac_t[0])
        if nb:
            put((1 << (8 - nb)) - 1, 8 - nb)
        out += data
    out += b"\xff\xd9"
    return bytes(out), [((H * info["vs"][c] + vmax - 1) // vmax + 7) // 8 for c in range(ncomp)], [((W * info["hs"][c] + hmax - 1) // hmax + 7) // 8 for c in range(ncomp)]


def multiscan_expected(stream, hblk, wblk):
    """arena-order coefficients of the twin; the blocks a non-interleaved scan does not code (padding up to the MCU) stay zero"""
    comps, info = po.jpeg_coeffs(stream), po.jpeg_info(stream)
    for c in range(info["ncomp"]):
        comps[c] = comps[c].copy()
        comps[c][hblk[c]:] = 0
        comps[c][:, wblk[c]:] = 0
    hs, vs = info["hs"], info["vs"]
    return np.stack([comps[c][my * vs[c] + v, mx * hs[c] + h] for my in range(info["mcuy"]) for mx in range(info["mcux"])
                     for c in range(info["ncomp"]) for v in range(vs[c]) for h in range(hs[c])])


def test_sequential_frames_in_several_scans(emul):
    import cv2
    k = 0
    for (h, w) in [(48, 64), (33, 47), (97, 61), (17, 23)]:
        for s in (cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_422):
            for rst in (0, 5):
                k += 1
                base, _ = twins(synth(h, w, 500 + k), 85, s)
                multi, hblk, wblk = to_multiscan_baseline(base, rst)
                # libjpeg-turbo accepts the re-coded stream and decodes the same picture: the test encoder is sound
                assert np.array_equal(cv2.imdecode(np.frombuffer(multi, np.uint8), cv2.IMREAD_COLOR), cv2.imdecode(np.frombuffer(base, np.uint8), cv2.IMREAD_COLOR))
                rc, got, info = decode(emul, multi)
                assert rc == 0 and info["truncated"] == 0 and info["nscans"] == 3 and info["nwaves"] == 1, (h, w, s, rst, rc, info)
                assert np.array_equal(got, multiscan_expected(base, hblk, wblk)), (h, w, s, rst)
