"""fn.multi_paste and fn.paste stated in numpy (DESIGN.md section 2).

multi_paste: output i starts as zeros of (H, W, C) in the output type; region k, in list order, takes the rectangle of its source at
the in-anchor (y, x) of extent (h, w), converts it with the arithmetic kernel's ConvertSat (tests/arith_ref.py) when the output type
differs, and assigns it at the out-anchor, so a later region lies on top of an earlier one.  Absolute coordinates are integers; a
relative one is llround(value * extent) in double (half away from zero, tests/erase_ref.py).  Defaults: anchors 0, extent the source
extent minus the in-anchor.

paste: on a canvas of H' = max(int(ratio * H), int(min_canvas_size)) rows and W' the same way, the float32 products truncated, filled
with fill_value per channel, the image is put at (int(paste_y * (H' - H)), int(paste_x * (W' - W))), again in float32.
Outputs are compared bit for bit."""
import numpy as np

import arith_ref as ar
from erase_ref import TYPES, llround

ARGS = ("in_anchors", "in_anchors_rel", "shapes", "shapes_rel", "out_anchors", "out_anchors_rel")


def _coord(v, ext, rel):
    return llround(float(v) * ext) if rel else int(v)


def regions(src_shapes, out_hw, args):
    """The pixel rectangles (src, iy, ix, h, w, oy, ox) of one output, zero-size ones included.  src_shapes: the (H, W, C) of each
    region's source, in region order; args: the given region arguments of this output by name, each K x 2 values."""
    out = []
    for k, (hs, ws, _) in enumerate(src_shapes):
        def pair(name, ext):
            for rel in (False, True):
                v = args.get(name + ("_rel" if rel else ""))
                if v is not None:
                    v = np.asarray(v, np.float64).reshape(-1, 2)[k]
                    return _coord(v[0], ext[0], rel), _coord(v[1], ext[1], rel)
            return None
        ia = pair("in_anchors", (hs, ws)) or (0, 0)
        sh = pair("shapes", (hs, ws)) or (hs - ia[0], ws - ia[1])
        oa = pair("out_anchors", out_hw) or (0, 0)
        out.append((k, ia[0], ia[1], sh[0], sh[1], oa[0], oa[1]))
    return out


def convert(x, dtype):
    x = np.asarray(x)
    dtype = np.dtype(dtype)
    if x.dtype == dtype:
        return x
    if x.dtype == np.float16 and dtype == np.float64:
        x = x.astype(np.float32)              # exact; a NaN is widened through float32 and quieted, as the kernel does
    out = np.asarray(ar.convert_sat(x, TYPES[x.dtype], TYPES[dtype]), dtype)
    if dtype == np.float16 and x.dtype in (np.float32, np.float64):
        # a NaN keeps its sign and the top 10 bits of its float32 payload, quieted (arith_core.h's arith_to_bits)
        b = x.astype(np.float32).view(np.uint32)
        nan = np.isnan(x)
        bits = ((b >> 16) & 0x8000) | 0x7C00 | 0x200 | ((b >> 13) & 0x3FF)
        out = out.copy()
        out.view(np.uint16)[nan] = bits[nan].astype(np.uint16)
    return out


def multi_paste_ref(sources, out_hw, args=None, dtype=None, channels=None):
    """One output.  sources: the source image of each region, in region order; args: the region arguments by name; channels: the
    inputs' channel count (needed when there is no region)."""
    args = args or {}
    c = channels if channels is not None else sources[0].shape[2]
    dtype = np.dtype(dtype or (sources[0].dtype if sources else np.uint8))
    out = np.zeros((out_hw[0], out_hw[1], c), dtype)
    for k, iy, ix, h, w, oy, ox in regions([s.shape for s in sources], out_hw, args):
        if h == 0 or w == 0:
            continue
        out[oy:oy + h, ox:ox + w] = convert(sources[k][iy:iy + h, ix:ix + w], dtype)
    return out


def paste_geometry(h, w, ratio, paste_x=0.5, paste_y=0.5, min_canvas_size=0.0):
    """(H', W', y, x) in float32 arithmetic, truncated as static_cast<int> does"""
    f = np.float32
    ho = max(int(f(ratio) * f(h)), int(f(min_canvas_size)))
    wo = max(int(f(ratio) * f(w)), int(f(min_canvas_size)))
    return ho, wo, int(f(paste_y) * f(ho - h)), int(f(paste_x) * f(wo - w))


def paste_ref(x, ratio, paste_x=0.5, paste_y=0.5, min_canvas_size=0.0, fill=(0,)):
    h, w, c = x.shape
    ho, wo, y, xo = paste_geometry(h, w, ratio, paste_x, paste_y, min_canvas_size)
    fv = np.asarray(ar.convert_sat(np.asarray(fill, np.float32).reshape(-1), ar.F32, TYPES[x.dtype]), x.dtype)
    out = np.empty((ho, wo, c), x.dtype)
    out[...] = fv if fv.size == c else fv[0]
    out[y:y + h, xo:xo + w] = x
    return out
