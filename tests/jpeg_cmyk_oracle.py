"""ctypes bindings of tests/jpeg_cmyk_oracle.c: the oracle's decode of 4-component (CMYK / YCCK) JPEG, built on first use with gcc into a
temporary directory (oracle/jpeg_oracle.c, which it includes, stays as it is).  Also decodes 1- and 3-component streams by the same rules
as oracle/pyoracle.py, and gives cv2's GRAYSCALE output of every stream."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

from oracle import pyoracle as po

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.dirname(_HERE)
_lib = None


def lib():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="jpeg_cmyk_oracle_"), "libjpegcmykoracle.so")
        subprocess.run(["gcc", "-O2", "-fPIC", "-ffp-contract=off", "-Wall", "-Wno-unused-function", "-shared",
                        "-I" + os.path.join(_ROOT, "oracle"), os.path.join(_HERE, "jpeg_cmyk_oracle.c"), "-o", out], check=True)
        _lib = C.CDLL(out)
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def coeffs(buf):
    """Quantised DCT coefficients per component, natural order: list of [bh, bw, 64] int16."""
    b = np.frombuffer(bytes(buf), np.uint8)
    i = po.jpeg_info(buf)
    outs = [np.zeros((i["mcuy"] * i["vs"][c], i["mcux"] * i["hs"][c], 64), np.int16) if c < i["ncomp"] else None for c in range(4)]
    rc = lib().cmyk_oracle_coeffs(_p(b), C.c_size_t(b.size), *[_p(o) for o in outs])
    if rc != 0:
        raise ValueError(f"cmyk_oracle_coeffs rc={rc}")
    return [o for o in outs if o is not None]


def mcu_order(buf):
    """coeffs() rearranged into the decoder's arena order: [MCU][component][v][h] blocks"""
    comps, info = coeffs(buf), po.jpeg_info(buf)
    hs, vs = info["hs"], info["vs"]
    return np.stack([comps[c][my * vs[c] + v, mx * hs[c] + h] for my in range(info["mcuy"]) for mx in range(info["mcux"])
                     for c in range(info["ncomp"]) for v in range(vs[c]) for h in range(hs[c])])


def _decode(buf, fancy, gray):
    b = np.frombuffer(bytes(buf), np.uint8)
    i = po.jpeg_info(buf)
    out = np.empty((i["height"], i["width"]) if gray else (i["height"], i["width"], 3), np.uint8)
    rc = lib().cmyk_oracle_decode(_p(b), C.c_size_t(b.size), _p(out), int(bool(fancy)), int(bool(gray)))
    if rc != 0:
        raise ValueError(f"cmyk_oracle_decode rc={rc}")
    return out


def decode(buf, fancy=True):
    """[H, W, 3] RGB u8 as cv2.imdecode(..., IMREAD_COLOR)[..., ::-1] returns it."""
    return _decode(buf, fancy, False)


def decode_gray(buf, fancy=True):
    """[H, W] u8 as cv2.imdecode(..., IMREAD_GRAYSCALE) returns it (Y plane, rgb_gray for RGB frames, CMYK -> gray for 4 components)."""
    return _decode(buf, fancy, True)
