"""fn.experimental.equalize in numpy: cv2.equalizeHist's table for every (frame, channel) plane of a uint8 sample.

Per plane of `total` pixels: i = the first non-zero bin; if hist[i] == total the plane maps to itself; else lut[i] = 0 and, for k > i,
sum += hist[k], lut[k] = clamp(rint_half_even((float)sum * scale), 0, 255) with scale = 255.f / (float)(total - hist[i]), every
operation in correctly rounded fp32."""
import numpy as np

LAYOUTS = ("HW", "HWC", "CHW", "FHW", "FHWC", "FCHW")
BY_RANK = {2: "HW", 3: "HWC", 4: "FHWC"}


def plane_lut(plane):
    h = np.bincount(plane.ravel(), minlength=256)
    i = int(np.argmax(h > 0))
    total = plane.size
    if h[i] == total:
        return np.arange(256, dtype=np.uint8)
    scale = np.float32(255.0) / np.float32(total - h[i])
    s = np.cumsum(h) - h[i]
    v = np.rint(s.astype(np.float32) * scale)               # np.rint: half to even
    lut = np.clip(v, 0, 255).astype(np.uint8)
    lut[:i + 1] = 0
    return lut


def equalize_plane(plane):
    return plane_lut(plane)[plane] if plane.size else plane.copy()


def equalize(x, layout=""):
    """x equalized per (frame, channel) plane; layout "" is read by rank"""
    lay = layout or BY_RANK[x.ndim]
    y = np.moveaxis(x, [lay.index(a) for a in "HW"], [-2, -1]).copy() if x.size else x.copy()
    if not x.size:
        return y
    flat = y.reshape(-1, y.shape[-2], y.shape[-1])
    for k in range(flat.shape[0]):
        flat[k] = equalize_plane(flat[k])
    return np.moveaxis(flat.reshape(y.shape), [-2, -1], [lay.index(a) for a in "HW"])


def big_plane():
    """(plane, total - hist[i], sum at 1): one plane of 33 202 324 pixels, one 0, 21 288 547 ones and the rest twos.  The running sum
    at 1 is odd and above 2^24, so (float)sum rounds it, and that moves lut[1] from 163 (the exact sum times the fp32 scale) to 164"""
    d, s = 33202323, 21288547
    return np.concatenate([np.zeros(1, np.uint8), np.ones(s, np.uint8), np.full(d - s, 2, np.uint8)]).reshape(1, -1), d, s
