"""CPU tests of the lossy WebP decode on frame headers and intra modes the encoders never write: tests/vp8_rewrite.py rewrites
partition 0 of corpus streams (ws.rewritten()), and the PRODUCT's planner and decode bodies (webp_plan.h + webp_core.h, compiled for
the host by tools/emul/webp_emul.cc) must equal cv2.imdecode on every rewritten stream in RGB, BGR and GRAY.  The rewriter itself is
pinned by a round trip through cv2, and what the rewritten corpus covers is read back from the written streams."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import webp_streams as ws  # noqa: E402
import vp8_rewrite as vr  # noqa: E402

cv2 = pytest.importorskip("cv2")
EMUL = os.path.join(ROOT, "tools", "emul", "webp_emul.cc")
RGB, BGR, GRAY = 0, 1, 2
NOORIENT = cv2.IMREAD_IGNORE_ORIENTATION


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp_path_factory.mktemp("webp_emul") / "libwebpemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-shared", "-fPIC", "-I/usr/local/cuda/include", "-O2", EMUL, "-o", out],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(out)
    lib.emul_webp_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _decode(lib, s, out_type):
    info = np.zeros(4, np.int32)
    rc = lib.emul_webp_decode(s, len(s), out_type, None, info.ctypes.data)
    if rc:
        return rc, None
    out = np.zeros((info[1], info[0], 1 if out_type == GRAY else 3), np.uint8)
    return lib.emul_webp_decode(s, len(s), out_type, out.ctypes.data, info.ctypes.data), out


@pytest.fixture(scope="module")
def rewritten():
    return ws.rewritten()


def test_bool_coder_round_trip_with_carries():
    """random bits, and runs that keep the coding interval across a multiple of 256 of its low end until the low end's pending bytes
    are 0xFF: the bit after such a run carries into bytes already written"""
    rng = np.random.default_rng(5)
    w = vr.BoolEncoder()
    probs, bits = [], []

    def put(p, b):
        probs.append(p)
        bits.append(b)
        w.bit(p, b)
    for _ in range(200):
        for _ in range(int(rng.integers(0, 20))):
            put(int(rng.integers(1, 256)), int(rng.integers(0, 2)))
        for _ in range(int(rng.integers(4, 60))):
            boundary, p = (w.low | 0xFF) + 1, int(rng.integers(2, 255))
            put(p, int(w.low + 1 + (((w.range - 1) * p) >> 8) <= boundary - 1))
        put(int(rng.integers(1, 256)), 1)
    data = w.finish()
    assert w.carries > 0 and w.long_carries > 0, "the sequence should carry into written bytes, across 0xFF bytes too"
    r = vr.BoolDecoder(data)
    assert [r.bit(p) for p in probs] == bits and r.overrun == 0


def test_round_trip_keeps_every_corpus_stream():
    """parse then write with no edit: cv2 decodes every simple-format stream of the corpus as before"""
    streams = ws.simple_format(ws.corpus(big=True))
    assert len(streams) >= 80
    for name, s in streams:
        f = vr.parse(s)
        out = vr.write(f)
        again = vr.parse(out)
        assert again["pay"][10 + again["p0"]:] == f["pay"][10 + f["p0"]:], name        # the token partitions, byte for byte
        assert again["hdr"] == f["hdr"] and again["mbs"] == f["mbs"], name
        assert np.array_equal(ws.decode(out, cv2.IMREAD_COLOR | NOORIENT), ws.decode(s, cv2.IMREAD_COLOR | NOORIENT)), name


def test_writer_refuses_edits_that_change_token_parsing():
    f = vr.parse(dict(ws.simple_format(ws.corpus()))["cv2_63x80_q50"])
    for edit in (lambda f: f["mbs"][3].update(i4=1 - f["mbs"][3]["i4"], bmodes=[0] * 16, ymode=0),
                 lambda f: f["hdr"].update(log2_parts=(f["hdr"]["log2_parts"] + 1) & 3),
                 lambda f: f["hdr"]["proba"].__setitem__(40, 7 if f["hdr"]["proba"][40] is None else None)):
        g = vr.parse(vr.write(f))
        edit(g)
        with pytest.raises(AssertionError):
            vr.write(g)


def test_host_build_equals_cv2_on_the_rewritten_corpus(emul, rewritten):
    for name, s, _ in rewritten:
        bgr = ws.decode(s, cv2.IMREAD_COLOR | NOORIENT)
        gray = ws.decode(s, cv2.IMREAD_GRAYSCALE | NOORIENT)
        if bgr is None:                                            # a stream cv2 refuses must fail here too
            assert _decode(emul, s, RGB)[0] != 0, name
            continue
        for ot, want in ((RGB, bgr[..., ::-1]), (BGR, bgr), (GRAY, gray[..., None])):
            rc, out = _decode(emul, s, ot)
            assert rc == 0, (name, ot, rc)
            assert np.array_equal(out, want), (name, ot, int((out != want).sum()))


def test_q127_requantised_streams(emul, rewritten):
    """cv2 quality 90 / 100 streams re-quantised at index 127: dequantised coefficients near the int16 limit, where libwebp's full
    inverse DCT wraps in int16 lanes (webp_core.h webp_idct_add)"""
    d = {n: s for n, s, _ in rewritten}
    names = [n for n in d if n.startswith("q127_")]
    assert {"q127_cv2_16x16_q100", "q127_cv2_63x80_q100", "q127_cv2_128x200_q100"} <= set(names) and len(names) == 16
    for n in names:
        rc, out = _decode(emul, d[n], BGR)
        assert rc == 0 and np.array_equal(out, ws.decode(d[n], cv2.IMREAD_COLOR | NOORIENT)), n


def _features(name, s, base):
    """what one written stream holds, read back from its bytes"""
    out = set()
    if s[12:16] == b"VP8X":
        out.add("vp8x")
    if vr.scale_bits(s) != (0, 0):
        out.add("scale_bits")
    if s[12:16] != b"VP8 ":
        return out
    f, fb = vr.parse(s), vr.parse(base)
    h, hb = f["hdr"], fb["hdr"]
    mbs = f["mbs"]
    used = {m["segment"] for m in mbs}
    has_i4, has_i16 = any(m["i4"] for m in mbs), any(not m["i4"] for m in mbs)
    if f["width"] % 16 and f["height"] % 16:
        out.add("size_not_multiple_of_16")
    if h["use_segment"]:
        out.add("seg_nomap" if not h["update_map"] else "seg_map")
        if not h["update_data"]:
            out.add("seg_nodata")
        if h["update_map"] and len(used) > 1:
            for i, p in enumerate(h["seg_proba"]):
                out.add(f"seg_proba{i}_{'absent' if p is None else p}")
        if h["update_data"] and not h["absolute_delta"]:
            q = [h["base_q0"] + (v or 0) for v in h["quantizer"]]
            lv = [h["level"] + (v or 0) for v in h["filter_strength"]]
            out |= {"rel_q_below_0"} if min(q) < 0 else set()
            out |= {"rel_q_above_127"} if max(q) > 127 else set()
            out |= {"rel_level_above_63"} if max(lv) > 63 and h["level"] else set()
            out |= {"rel_negative_delta"} if min(v or 0 for v in h["quantizer"] + h["filter_strength"]) < 0 else set()
        if h["level"] == 0 and h["update_data"] and any(h["filter_strength"]):
            out.add("level0_segment_strengths")
    if h["use_lf_delta"] and h["level"]:
        if not h["update_lf_delta"]:
            out.add("lf_delta_no_update")
        r0, m0 = h["ref_lf_delta"][0] or 0, h["mode_lf_delta"][0] or 0
        if r0 and has_i16:
            out.add(f"lf_ref0_{'pos' if r0 > 0 else 'neg'}_16x16")
        if m0 and has_i4:
            out.add(f"lf_mode0_{'pos' if m0 > 0 else 'neg'}_4x4")
        if any(v is not None for v in h["ref_lf_delta"][1:] + h["mode_lf_delta"][1:]):
            out.add("lf_unused_deltas_set")
    if h["level"] == 63:
        out.add(f"level63_sharpness{h['sharpness']}_{'simple' if h['simple'] else 'normal'}")
    if not h["use_segment"]:
        for d, v in enumerate(h["dq"]):
            if v and h["base_q0"] in (0, 127):
                out.add(f"dq{d}_q{h['base_q0']}")
        q = h["base_q0"]
        if q + (h["dq"][3] or 0) > 117:
            out.add("uv_dc_clip_117")
        if min(127, max(0, q + (h["dq"][2] or 0))) <= 1:              # AC steps 4 and 5: x * 155 / 100 < 8
            out.add("y2_ac_floor_8")
        if q == 127 and not any(h["dq"]) and name.startswith("q127_cv2_"):
            out.add("q127_cv2_stream")
    if h["color_space"]:
        out.add("color_space_bit")
    if h["clamp_type"]:
        out.add("clamp_type_bit")
    if h["use_skip"] and hb["use_skip"] and h["skip_p"] != hb["skip_p"]:
        out.add("skip_p_changed")
    if h["use_skip"] and not hb["use_skip"]:
        out.add("use_skip_0_to_1")
    return out | {("mode",) + t for t in vr.mode_positions(f)}


def test_rewritten_corpus_covers_every_family(rewritten):
    """read from the written streams, not from the settings that made them"""
    seen = set()
    for name, s, base in rewritten:
        seen |= _features(name, s, base)
    want = {"seg_nomap", "seg_nodata", "seg_map", "rel_q_below_0", "rel_q_above_127", "rel_level_above_63", "rel_negative_delta",
            "lf_ref0_pos_16x16", "lf_ref0_neg_16x16", "lf_mode0_pos_4x4", "lf_mode0_neg_4x4", "lf_unused_deltas_set",
            "lf_delta_no_update", "level0_segment_strengths", "uv_dc_clip_117", "y2_ac_floor_8", "q127_cv2_stream",
            "color_space_bit", "clamp_type_bit", "skip_p_changed", "use_skip_0_to_1", "scale_bits", "vp8x",
            "size_not_multiple_of_16"}
    want |= {f"seg_proba{i}_{v}" for i in range(3) for v in ("absent", 1, 254)}
    want |= {f"level63_sharpness{k}_{t}" for k in range(8) for t in ("simple", "normal")}
    want |= {f"dq{d}_q{q}" for d in range(5) for q in (0, 127)}
    want |= {("mode", kind, m, p) for kind, n in (("y16", 4), ("b4", 10), ("uv", 4)) for m in range(n) for p in vr.POSITIONS}
    missing = want - seen
    assert not missing, sorted(map(str, missing))
