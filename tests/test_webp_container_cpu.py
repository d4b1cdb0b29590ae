"""CPU tests of how the WebP planner bounds the VP8 data and reads the container, pinned against cv2.imdecode: the VP8 decoder reads
from the frame header to the end of the input (chunks and bytes behind the frame included), a damaged chunk behind the frame does
not fail the stream, the EXIF orientation is applied only when cv2 applies it, and every chunk up to the frame must fit in the RIFF
with its padding.  The planner and decode bodies run on the host through tools/emul/webp_emul.cc."""
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

cv2 = pytest.importorskip("cv2")
NOORIENT = cv2.IMREAD_IGNORE_ORIENTATION


@pytest.fixture(scope="module")
def emul(tmp_path_factory):
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    out = str(tmp_path_factory.mktemp("webp_emul") / "libwebpemul.so")
    r = subprocess.run(["g++", "-std=c++17", "-O2", "-shared", "-fPIC", "-I/usr/local/cuda/include",
                        os.path.join(ROOT, "tools", "emul", "webp_emul.cc"), "-o", out], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    lib = C.CDLL(out)
    lib.emul_webp_decode.argtypes = [C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p]
    return lib


def _decode(lib, s):
    info = np.zeros(4, np.int32)
    rc = lib.emul_webp_decode(s, len(s), 1, None, info.ctypes.data)
    if rc:
        return rc, None, info
    out = np.zeros((info[1], info[0], 3), np.uint8)
    return lib.emul_webp_decode(s, len(s), 1, out.ctypes.data, info.ctypes.data), out, info


def _orient(a, o):
    """EXIF orientation o applied to an image (as cv2 applies it)"""
    a = a[:, ::-1] if o in (2, 7) else a[::-1] if o == 4 else a[::-1, ::-1] if o == 3 else a
    if o in (5, 6, 7, 8):
        a = np.swapaxes(a, 0, 1)
        a = a[:, ::-1] if o in (6, 7) else a[::-1] if o == 8 else a
    return np.ascontiguousarray(a)


def test_vp8_data_runs_to_the_end_of_the_input(emul):
    """payloads cut inside the chunk with data behind it, a first partition past the chunk, zeros behind a cut partition: cv2 decodes
    them all, and so does the planner, bit for bit"""
    edge = ws.edge_decodable()
    assert len(edge) == 5
    for name, s in edge:
        want = ws.decode(s, cv2.IMREAD_COLOR | NOORIENT)
        assert want is not None, name
        rc, out, _ = _decode(emul, s)
        assert rc == 0 and np.array_equal(out, want), (name, rc)


def test_orientation_as_cv2_applies_it(emul):
    for name, s in ws.orientation_cases():
        raw = ws.decode(s, cv2.IMREAD_COLOR | NOORIENT)
        rc, out, info = _decode(emul, s)
        assert rc == 0 and np.array_equal(out, raw), name
        assert np.array_equal(_orient(raw, int(info[3])), ws.decode(s)), (name, int(info[3]))
    o = {name: _decode(emul, s)[2][3] for name, s in ws.orientation_cases()}
    assert o["exif_behind"] == 6 and o["exif_before_frame"] == 6 and o["two_exif_first_wins"] == 6
    assert o["exif_size_overruns_riff"] == 1 and o["junk_chunk_overruns_riff"] == 1 and o["exif_flag_clear"] == 1


def test_unpadded_odd_frame_chunk_is_refused(emul):
    s = dict((n, x) for n, x, _ in ws.plan_corrupt())["odd_frame_chunk_unpadded"]
    assert ws.decode(s) is None
    assert _decode(emul, s)[0] == 4                      # DALIB200_ERROR_BAD_DATA
