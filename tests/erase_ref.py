"""fn.erase stated in numpy (DESIGN.md section 2): per erased axis, in float64 from the float32 argument values,
  a = anchor, s = shape, each times the axis's extent when normalised; a -= s / 2 when the anchor is centred;
  begin = llround(a), end = llround(a + s) (half away from zero), clipped to [0, extent];
then out = x.copy() and one slice assignment of the fill per region.  The fill is one value, or one per channel of the C axis,
converted with the arithmetic kernel's ConvertSat (tests/arith_ref.py).  Outputs are compared bit for bit."""
import math

import numpy as np

import arith_ref as ar

TYPES = {np.dtype(v): k for k, v in ar.NP.items()}


def llround(x):
    """C's llround: to nearest, half away from zero, exact for every double"""
    m = abs(x)
    r = math.floor(m)
    if m - r >= 0.5:
        r += 1
    return int(r if x >= 0 else -r)


def boxes(shape, axes, anchor, shp, normalized_anchor=False, normalized_shape=False, centered=False):
    """the clipped [begin, end) of every region on every dimension (unerased dimensions whole); anchor, shp: flat value lists"""
    anchor = np.asarray(anchor, np.float32).reshape(-1)
    shp = np.asarray(shp, np.float32).reshape(-1)
    assert anchor.size == shp.size and anchor.size % len(axes) == 0
    out = []
    for r in range(anchor.size // len(axes)):
        b, e = [0] * len(shape), list(shape)
        for k, a in enumerate(axes):
            x, w = float(anchor[r * len(axes) + k]), float(shp[r * len(axes) + k])
            if normalized_anchor:
                x *= shape[a]
            if normalized_shape:
                w *= shape[a]
            if centered:
                x -= w / 2
            b[a] = min(max(llround(x), 0), shape[a])
            e[a] = min(max(llround(x + w), 0), shape[a])
        out.append((b, e))
    return out


def fill_values(fill, dtype):
    """fill_value converted to the data type with ConvertSat (from float32)"""
    f = np.asarray(fill, np.float32).reshape(-1)
    return np.asarray(ar.convert_sat(f, ar.F32, TYPES[np.dtype(dtype)]), dtype)


def erase_ref(x, axes, anchor, shp, fill=(0.0,), layout="", normalized_anchor=False, normalized_shape=False, centered=False):
    """axes: the erased dimensions, in the order of the anchor / shape values"""
    out = x.copy()
    fv = fill_values(fill, x.dtype)
    for b, e in boxes(x.shape, axes, anchor, shp, normalized_anchor, normalized_shape, centered):
        if any(hi <= lo for lo, hi in zip(b, e)):
            continue
        idx = tuple(slice(lo, hi) for lo, hi in zip(b, e))
        if fv.size == 1:
            out[idx] = fv[0]
        else:
            c = layout.index("C")
            view = np.moveaxis(out[idx], c, -1)
            view[...] = fv
    return out


def axes_of(layout, names):
    return [layout.index(c) for c in names]
