"""Generates tests/golden/jpeg_cmyk.npz -- 4-component (CMYK / YCCK) JPEG streams written by Pillow (libjpeg-turbo) and their
cv2.imdecode decodes (OpenCV 4.13 / libjpeg-turbo), the parity target of every decoder output.  Pillow is only needed to run this
script; the tests read the committed file.

Streams, for every size x subsampling x (baseline, progressive):
  cmyk    Pillow's CMYK stream (Adobe APP14 marker, transform 0)
  ycck    the same bytes with the APP14 transform set to 2: components 0..2 are then read as YCbCr (a valid YCCK stream)
  noadobe the same bytes without the APP14 segment: CMYK by default
Pillow's `subsampling` 1 / 2 subsamples the other components against the first (h2v1 / h2v2 on component 0).
Keys: enc_i (stream bytes), color_i (cv2 IMREAD_COLOR, BGR), gray_i (cv2 IMREAD_GRAYSCALE), name_i.
Usage:  python tests/golden/make_cmyk_golden.py
"""
import io
import os

import cv2
import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = [(1, 1), (17, 9), (250, 3), (61, 77)]          # (height, width)


def synth_cmyk(h, w, seed):
    r = np.random.default_rng(seed)
    lo = r.uniform(0, 255, (max(2, h // 16), max(2, w // 16), 4)).astype(np.float32)
    img = np.stack([cv2.resize(lo[..., c], (w, h), interpolation=cv2.INTER_CUBIC) for c in range(4)], -1) + r.normal(0, 5, (h, w, 4))
    return np.clip(img, 0, 255).astype(np.uint8)


def app14(stream):
    """offset of the Adobe APP14 segment's marker, or -1"""
    pos = 2
    while pos + 4 <= len(stream) and stream[pos] == 0xFF:
        m, L = stream[pos + 1], (stream[pos + 2] << 8) | stream[pos + 3]
        if m == 0xEE and stream[pos + 4:pos + 9] == b"Adobe":
            return pos
        if m == 0xDA:
            break
        pos += 2 + L
    return -1


def variants(stream):
    p = app14(stream)
    assert p > 0 and stream[p + 4 + 11] == 0, "Pillow writes CMYK with an Adobe marker, transform 0"
    ycck = bytearray(stream)
    ycck[p + 4 + 11] = 2
    L = (stream[p + 2] << 8) | stream[p + 3]
    return {"cmyk": stream, "ycck": bytes(ycck), "noadobe": stream[:p] + stream[p + 2 + L:]}


def main():
    out, k, seed = {}, 0, 0
    for (h, w) in SIZES:
        for sub in (0, 1, 2):
            seed += 1
            for prog in (False, True):                   # the baseline and progressive twins code the same image
                buf = io.BytesIO()
                Image.fromarray(synth_cmyk(h, w, seed), "CMYK").save(buf, "JPEG", quality=90, subsampling=sub, progressive=prog)
                for kind, s in variants(buf.getvalue()).items():
                    a = np.frombuffer(s, np.uint8)
                    color = cv2.imdecode(a, cv2.IMREAD_COLOR)
                    gray = cv2.imdecode(a, cv2.IMREAD_GRAYSCALE)
                    assert color is not None and gray is not None and color.shape[:2] == (h, w)
                    out[f"enc_{k}"] = a
                    out[f"color_{k}"] = color
                    out[f"gray_{k}"] = gray
                    out[f"name_{k}"] = np.array(f"{kind}_s{sub}_{'prog' if prog else 'base'}_{h}x{w}")
                    k += 1
    np.savez_compressed(os.path.join(HERE, "jpeg_cmyk.npz"), **out)
    print(k, "streams")


if __name__ == "__main__":
    main()
