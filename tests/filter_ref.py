"""numpy statement of fn.experimental.filter (DESIGN.md section 2) in float64: each frame padded with np.pad by the border rule, the
filter slid over it (correlation: not flipped; channels independent), then ConvertSat to the output type (tests/arith_ref.py).  Also the
per-element error bound of a float32 fmaf chain over k taps, gamma_k * sum |f x|, and the check that an output lies within it.

tests/test_filter_cpu.py pins this statement to cv2.filter2D; the host build of the kernel bodies and the GPU are checked against it."""
import numpy as np

import arith_ref as ar

BORDERS = ("reflect_101", "reflect_1001", "wrap", "clamp", "constant")
PAD_MODE = {"reflect_101": "reflect", "reflect_1001": "symmetric", "wrap": "wrap", "clamp": "edge", "constant": "constant"}
LAYOUTS = ("HW", "HWC", "FHW", "FHWC")
BY_RANK = {2: "HW", 3: "HWC", 4: "FHWC"}
TYPES = {np.dtype(np.uint8): ar.U8, np.dtype(np.int8): ar.I8, np.dtype(np.uint16): ar.U16, np.dtype(np.int16): ar.I16,
         np.dtype(np.float16): ar.F16, np.dtype(np.float32): ar.F32}
NP_OF = {v: k.type for k, v in TYPES.items()}


def frames(x, layout):
    """x as F x H x W x C"""
    lay = layout or BY_RANK[x.ndim]
    y = x if lay[0] == "F" else x[None]
    return y if lay[-1] == "C" else y[..., None]


def unframes(y, layout, ndim):
    lay = layout or BY_RANK[ndim]
    y = y if lay[-1] == "C" else y[..., 0]
    return y if lay[0] == "F" else y[0]


def _pad(fr, f, anchor, border, mode, fill):
    fh, fw = f.shape
    if mode == "valid":
        return fr
    ar_, ac = (fh // 2 if anchor[0] < 0 else anchor[0]), (fw // 2 if anchor[1] < 0 else anchor[1])
    width = ((ar_, fh - 1 - ar_), (ac, fw - 1 - ac), (0, 0))
    if border == "constant":
        return np.pad(fr, width, "constant", constant_values=fill)
    out = fr
    for ax in (0, 1):                                         # reflect_101 of one element is that element: "edge"
        w = [(0, 0)] * 3
        w[ax] = width[ax]
        out = np.pad(out, w, "edge" if border == "reflect_101" and out.shape[ax] == 1 else PAD_MODE[border])
    return out


def correlate64(x, f, layout="", anchor=(-1, -1), border="reflect_101", mode="same", fill=None, absolute=False):
    """float64 sums, F x Ho x Wo x C; fill: None (0), a scalar or one value per frame.  absolute: sum |f| |x| instead."""
    fr = frames(x, layout).astype(np.float64)
    f = np.asarray(f, np.float64)
    if absolute:
        fr, f = np.abs(fr), np.abs(f)
    fh, fw = f.shape
    fills = np.zeros(fr.shape[0]) if fill is None else np.broadcast_to(np.asarray(fill, np.float64).reshape(-1), (fr.shape[0],))
    h, w = fr.shape[1:3]
    ho, wo = (h - fh + 1, w - fw + 1) if mode == "valid" else (h, w)
    outs = []
    for k in range(fr.shape[0]):
        if not fr[k].size:
            outs.append(np.zeros((ho, wo, fr.shape[3])))
            continue
        p = _pad(fr[k], f, anchor, border, mode, abs(fills[k]) if absolute else fills[k])
        acc = np.zeros((ho, wo, fr.shape[3]))
        for r in range(fh):
            for s in range(fw):
                acc += f[r, s] * p[r:r + ho, s:s + wo]
        outs.append(acc)
    return np.stack(outs) if outs else np.zeros((0, ho, wo, fr.shape[3]))


def gamma(k):
    u = 2.0 ** -24
    return k * u / (1 - k * u)


def bound(x, f, layout="", anchor=(-1, -1), border="reflect_101", mode="same", fill=None):
    """gamma_k * sum |f x| per output element (F x Ho x Wo x C), k the filter's taps"""
    return gamma(np.asarray(f).size) * correlate64(x, f, layout, anchor, border, mode, fill, absolute=True)


def filter_ref(x, f, layout="", anchor=(-1, -1), border="reflect_101", mode="same", fill=None, dtype=None):
    """the output in its layout and type: convert_sat of the float64 sums"""
    to = TYPES[np.dtype(dtype or x.dtype)]
    y = correlate64(x, f, layout, anchor, border, mode, fill)
    return unframes(ar.convert_sat(y, ar.F64, to), layout, x.ndim)


def within(got, x, f, layout="", anchor=(-1, -1), border="reflect_101", mode="same", fill=None, dtype=None):
    """The elements of `got` outside [conv(rn32(v - b)), conv(rn32(v + b))], v the float64 sum and b its bound: ConvertSat is
    monotone, so a float32 chain within the bound converts into that range.  An integer output may thus take the other neighbour only
    where v lies within the bound of a .5 boundary.  Returns the count of elements outside."""
    to = TYPES[np.dtype(dtype or x.dtype)]
    v = correlate64(x, f, layout, anchor, border, mode, fill)
    b = bound(x, f, layout, anchor, border, mode, fill)
    lo = ar.convert_sat((v - b).astype(np.float32), ar.F32, to).astype(np.float64)
    hi = ar.convert_sat((v + b).astype(np.float32), ar.F32, to).astype(np.float64)
    g = frames(np.asarray(got), layout).astype(np.float64).reshape(v.shape)
    return int(np.count_nonzero((g < lo) | (g > hi)))
