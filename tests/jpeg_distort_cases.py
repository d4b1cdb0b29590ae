"""Inputs and the cv2 reference of fn.jpeg_compression_distortion, shared by the CPU and GPU tests: seeded noise, smooth and saturated
RGB images over sizes that cover every MCU edge case (1 pixel, odd and even block counts, partial MCUs, widths 1..4 where the decoder's
chroma upsampling is box replication), the quality range with its scaling breakpoints, and cv2's encode + decode."""
import numpy as np

SIZES = [(1, 1), (1, 37), (29, 1), (2, 2), (3, 5), (9, 9), (17, 33), (63, 80), (97, 131), (200, 37), (224, 224)]
QUALITIES = [1, 2, 3, 10, 25, 49, 50, 51, 75, 90, 97, 99, 100]
KINDS = ["noise", "smooth", "saturated"]


def image(h, w, kind, seed):
    rng = np.random.default_rng(seed)
    if kind == "noise":
        return rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "smooth":
        y, x = np.mgrid[0:h, 0:w].astype(np.float64)
        ph = rng.uniform(0, 6.3, 3)
        img = np.stack([127.5 + 110 * np.sin(x / (7 + 5 * c) + y / (11 + 3 * c) + ph[c]) for c in range(3)], -1)
        return np.clip(img + rng.normal(0, 2, img.shape), 0, 255).astype(np.uint8)
    # saturated: 4x4 tiles of pure primaries / black / white, which drive the colour conversion and the IDCT to their clamps
    tiles = rng.integers(0, 2, ((h + 3) // 4, (w + 3) // 4, 3), dtype=np.uint8) * 255
    return np.ascontiguousarray(np.repeat(np.repeat(tiles, 4, 0), 4, 1)[:h, :w])


def encode(rgb, q):
    import cv2
    ok, enc = cv2.imencode(".jpg", np.ascontiguousarray(rgb[..., ::-1]), [cv2.IMWRITE_JPEG_QUALITY, int(q)])
    assert ok
    return enc.tobytes()


def reference(rgb, q):
    """what the operator must produce: cv2's decode of cv2's encode, as RGB"""
    import cv2
    return cv2.imdecode(np.frombuffer(encode(rgb, q), np.uint8), cv2.IMREAD_COLOR)[..., ::-1]


def mcu_coefficients(stream):
    """the stream's quantised coefficients in the operator's layout: MCU order, blocks Y00 Y01 Y10 Y11 Cb Cr, natural order"""
    from oracle import pyoracle as po
    comps, info = po.jpeg_coeffs(stream), po.jpeg_info(stream)
    hs, vs = info["hs"], info["vs"]
    assert info["ncomp"] == 3 and (hs[0], vs[0], hs[1], vs[1], hs[2], vs[2]) == (2, 2, 1, 1, 1, 1)
    blocks = []
    for my in range(info["mcuy"]):
        for mx in range(info["mcux"]):
            for c in range(3):
                for v in range(vs[c]):
                    for h in range(hs[c]):
                        blocks.append(comps[c][my * vs[c] + v, mx * hs[c] + h])
    return np.stack(blocks).reshape(-1)


_ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
           35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63]


def dqt_tables(stream):
    """{table id: 64 values in natural order} from the stream's DQT segments (8-bit precision)"""
    b, i, out = stream, 2, {}
    while i + 4 <= len(b) and b[i] == 0xFF and b[i + 1] != 0xDA:
        seg_len = (b[i + 2] << 8) | b[i + 3]
        if b[i + 1] == 0xDB:
            j = i + 4
            while j < i + 2 + seg_len:
                pq, tq = b[j] >> 4, b[j] & 15
                assert pq == 0
                t = np.zeros(64, np.uint16)
                for k in range(64):
                    t[_ZIGZAG[k]] = b[j + 1 + k]
                out[tq] = t
                j += 65
        i += 2 + seg_len
    return out
