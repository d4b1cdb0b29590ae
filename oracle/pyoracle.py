"""oracle/pyoracle.py -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

ctypes bindings for oracle/liboracle.so (plain-C restatement of the reference CPU path) and, when
present, oracle/_ref/libdali_ref_cpu.so (the reference's own CPU kernels compiled in place).
Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs may import this module.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "liboracle.so")
_REF = os.path.join(_HERE, "_ref", "libdali_ref_cpu.so")

F_NN, F_LINEAR, F_TRIANGULAR, F_GAUSSIAN, F_CUBIC, F_LANCZOS3 = range(6)
IT_RGB, IT_BGR, IT_GRAY, IT_YCBCR = range(4)


class FilterDesc(C.Structure):
    _fields_ = [("type", C.c_int), ("antialias", C.c_int), ("radius", C.c_float)]


def build(ref=True):
    """Compile the oracle (always) and the reference CPU library (only if /root/reference exists)."""
    subprocess.check_call(["make", "-s", "-C", _HERE, "liboracle.so"])
    if ref and os.path.isdir("/root/reference/dali"):
        subprocess.check_call(["make", "-s", "-C", _HERE, "ref"])


def _load(path):
    return C.CDLL(path) if os.path.exists(path) else None


_lib = None
_ref = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_LIB):
            build(ref=False)
        _lib = C.CDLL(_LIB)
        _lib.oracle_crop_anchor.restype = C.c_int64
        _lib.oracle_num_windows.restype = C.c_int64
        _lib.oracle_float2half.restype = C.c_uint16
    return _lib


def ref():
    """The compiled reference library or None (it cannot be built where /root/reference is absent
    unless the prebuilt .so travelled with the snapshot)."""
    global _ref
    if _ref is None and os.path.exists(_REF):
        _ref = C.CDLL(_REF)
        _ref.ref_float2half.restype = C.c_uint16
    return _ref


def have_ref():
    return ref() is not None


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _f32(v):
    return None if v is None else np.ascontiguousarray(v, dtype=np.float32)


# ------------------------------------------------------------------------------------------- JPEG
def jpeg_info(buf):
    b = np.frombuffer(bytes(buf), np.uint8)
    info = (C.c_int * 16)()
    rc = lib().jpeg_oracle_info(_p(b), C.c_size_t(b.size), info)
    if rc != 0:
        raise ValueError(f"jpeg_oracle_info rc={rc}")
    keys = ["width", "height", "ncomp"]
    d = {k: info[i] for i, k in enumerate(keys)}
    d["hs"] = [info[3 + c] for c in range(4)]
    d["vs"] = [info[7 + c] for c in range(4)]
    d["restart_interval"], d["progressive"], d["orientation"] = info[11], info[12], info[13]
    d["mcux"], d["mcuy"] = info[14], info[15]
    return d


def jpeg_decode(buf, fancy=True):
    b = np.frombuffer(bytes(buf), np.uint8)
    i = jpeg_info(buf)
    out = np.empty((i["height"], i["width"], 3), np.uint8)
    rc = lib().jpeg_oracle_decode_rgb(_p(b), C.c_size_t(b.size), _p(out), int(bool(fancy)))
    if rc != 0:
        raise ValueError(f"jpeg_oracle_decode_rgb rc={rc}")
    return out


def jpeg_coeffs(buf):
    """Quantised DCT coefficients per component, natural order: list of [bh, bw, 64] int16."""
    b = np.frombuffer(bytes(buf), np.uint8)
    i = jpeg_info(buf)
    hmax, vmax = max(i["hs"][: i["ncomp"]]), max(i["vs"][: i["ncomp"]])
    outs = []
    for c in range(3):
        if c < i["ncomp"]:
            outs.append(np.zeros((i["mcuy"] * i["vs"][c], i["mcux"] * i["hs"][c], 64), np.int16))
        else:
            outs.append(None)
    rc = lib().jpeg_oracle_coeffs(_p(b), C.c_size_t(b.size), _p(outs[0]), _p(outs[1]), _p(outs[2]))
    if rc != 0:
        raise ValueError(f"jpeg_oracle_coeffs rc={rc}")
    return [o for o in outs if o is not None]


def jpeg_overrun():
    """Whether the last JPEG entropy decode of the oracle (jpeg_decode, jpeg_coeffs) consumed padding bits behind a marker or the end of
    the data in some unit: that unit ran out of data, which the GPU decoder reports as status 1."""
    return bool(lib().jpeg_oracle_overrun())


# ------------------------------------------------------------------------------------------- resample
def _fd(t):
    if isinstance(t, FilterDesc):
        return t
    if isinstance(t, int):
        return FilterDesc(t, 1, 0.0)
    return FilterDesc(*t)


def _resample(fn, img, out_hw, min_filter, mag_filter, out_dtype, roi, want_order):
    img = np.ascontiguousarray(img)
    assert img.ndim == 3 and img.dtype in (np.uint8, np.float32)
    H, W, Cn = img.shape
    oh, ow = int(out_hw[0]), int(out_hw[1])
    out_dtype = np.dtype(out_dtype or img.dtype)
    out = np.empty((oh, ow, Cn), out_dtype)
    def pair(f):
        return [_fd(f[0]), _fd(f[1])] if isinstance(f, list) else [_fd(f), _fd(f)]
    minf = (FilterDesc * 2)(*pair(min_filter))
    magf = (FilterDesc * 2)(*pair(mag_filter))
    use = (C.c_int * 2)(0, 0)
    rs = (C.c_float * 2)(0, 0)
    re = (C.c_float * 2)(0, 0)
    if roi is not None:  # ((y0, x0), (y1, x1)) ; None entries = no ROI on that axis
        for d in range(2):
            if roi[0][d] is not None:
                use[d], rs[d], re[d] = 1, roi[0][d], roi[1][d]
    dt = lambda a: 0 if a.dtype == np.uint8 else 1
    order = C.c_int(-1)
    if fn.__name__.startswith("ref"):
        rc = fn(_p(img), dt(img), H, W, Cn, _p(out), dt(out), oh, ow, minf, magf, use, rs, re, C.byref(order))
    else:
        rc = fn(_p(img), dt(img), H, W, Cn, _p(out), dt(out), oh, ow, minf, magf, use, rs, re)
        if want_order:
            order.value = lib().oracle_resample_order(H, W, oh, ow, minf, magf, use, rs, re, None, None)
    if rc != 0:
        raise RuntimeError(f"resample rc={rc}")
    return (out, order.value) if want_order else out


def resample(img, out_hw, min_filter=(F_LINEAR, 1, 0.0), mag_filter=(F_LINEAR, 1, 0.0), out_dtype=None,
             roi=None, want_order=False):
    """Defaults = fn.resize defaults: linear with antialias (=> triangular when shrinking)."""
    return _resample(lib().oracle_resample_hwc, img, out_hw, min_filter, mag_filter, out_dtype, roi, want_order)


def ref_resample(img, out_hw, min_filter=(F_LINEAR, 1, 0.0), mag_filter=(F_LINEAR, 1, 0.0), out_dtype=None,
                 roi=None, want_order=False):
    return _resample(ref().ref_resample_hwc, img, out_hw, min_filter, mag_filter, out_dtype, roi, want_order)


def _resample3(fn, vol, out_dhw, min_filter, mag_filter, out_dtype, roi, want_order):
    vol = np.ascontiguousarray(vol)
    assert vol.ndim == 4 and vol.dtype in (np.uint8, np.float32)
    Cn = vol.shape[3]
    out_dtype = np.dtype(out_dtype or vol.dtype)
    out = np.empty(tuple(int(v) for v in out_dhw) + (Cn,), out_dtype)
    def triple(f):
        return [_fd(x) for x in f] if isinstance(f, list) else [_fd(f)] * 3
    minf = (FilterDesc * 3)(*triple(min_filter))
    magf = (FilterDesc * 3)(*triple(mag_filter))
    ish = (C.c_int * 3)(*vol.shape[:3])
    osh = (C.c_int * 3)(*[int(v) for v in out_dhw])
    use, rs, re = (C.c_int * 3)(0, 0, 0), (C.c_float * 3)(0, 0, 0), (C.c_float * 3)(0, 0, 0)
    if roi is not None:  # ((z0, y0, x0), (z1, y1, x1)); None entries = no ROI on that axis
        for d in range(3):
            if roi[0][d] is not None:
                use[d], rs[d], re[d] = 1, roi[0][d], roi[1][d]
    dt = lambda a: 0 if a.dtype == np.uint8 else 1
    order = (C.c_int * 3)(-1, -1, -1)
    rc = fn(_p(vol), dt(vol), ish, Cn, _p(out), dt(out), osh, minf, magf, use, rs, re, order)
    if rc != 0:
        raise RuntimeError(f"resample3d rc={rc}")
    return (out, list(order)) if want_order else out


def resample3d(vol, out_dhw, min_filter=(F_LINEAR, 1, 0.0), mag_filter=(F_LINEAR, 1, 0.0), out_dtype=None, roi=None,
               want_order=False):
    """DHWC volume, separable_cpu.h with spatial_ndim = 3 (oracle/imgproc_oracle.c: oracle_resample_dhwc)."""
    return _resample3(lib().oracle_resample_dhwc, vol, out_dhw, min_filter, mag_filter, out_dtype, roi, want_order)


def ref_resample3d(vol, out_dhw, min_filter=(F_LINEAR, 1, 0.0), mag_filter=(F_LINEAR, 1, 0.0), out_dtype=None, roi=None,
                   want_order=False):
    return _resample3(ref().ref_resample_dhwc, vol, out_dhw, min_filter, mag_filter, out_dtype, roi, want_order)


# ------------------------------------------------------------------------------------------- CMN
def float2half(x):
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty(x.shape, np.uint16)
    f = lib().oracle_float2half
    f.argtypes = [C.c_float]
    flat, o = x.ravel(), out.ravel()
    for i in range(flat.size):
        o[i] = f(float(flat[i]))
    return out.view(np.float16)


def ref_float2half(x):
    x = np.ascontiguousarray(x, np.float32)
    out = np.empty(x.shape, np.uint16)
    f = ref().ref_float2half
    f.argtypes = [C.c_float]
    flat, o = x.ravel(), out.ravel()
    for i in range(flat.size):
        o[i] = f(float(flat[i]))
    return out.view(np.float16)


def cmn_norm_args(mean, std, scale=1.0, shift=0.0, n=None):
    mean, std = _f32(np.atleast_1d(mean)), _f32(np.atleast_1d(std))
    n = n or max(mean.size, std.size)
    m, s = np.empty(n, np.float32), np.empty(n, np.float32)
    lib().oracle_cmn_norm_args(n, _p(mean), mean.size, _p(std), std.size, C.c_float(scale), C.c_float(shift), _p(m), _p(s))
    return m, s


def crop_anchor(pos_norm, in_extent, crop_extent, truncate=False):
    return int(lib().oracle_crop_anchor(C.c_float(pos_norm), C.c_int64(in_extent), C.c_int64(crop_extent), int(truncate)))


def _cmn(fn, img, anchor, crop, mirror, mean, inv_std, out_dtype, layout, pad_channels, fill):
    img = np.ascontiguousarray(img, np.uint8)
    H, W, Cn = img.shape
    ch, cw = crop if crop is not None else (H, W)
    ay, ax = anchor if anchor is not None else (0, 0)
    oc = pad_channels or Cn
    out_dtype = np.dtype(out_dtype)
    shape = (oc, ch, cw) if layout == "CHW" else (ch, cw, oc)
    out = np.empty(shape, out_dtype)
    mean = _f32(mean if mean is not None else np.zeros(Cn))
    inv_std = _f32(inv_std if inv_std is not None else np.ones(Cn))
    fillv = np.zeros(oc, np.float32)
    if fill is not None:
        f = np.atleast_1d(np.asarray(fill, np.float32))
        fillv[: f.size] = f if f.size > 1 else f[0]
        if f.size == 1:
            fillv[:] = f[0]
    rc = fn(_p(img), H, W, Cn, _p(out), 1 if out_dtype == np.float32 else 2, int(layout == "CHW"), oc,
            int(ay), int(ax), int(ch), int(cw), int(bool(mirror)), _p(mean), _p(inv_std), _p(fillv))
    if rc != 0:
        raise RuntimeError(f"cmn rc={rc}")
    return out


def cmn(img, anchor=None, crop=None, mirror=False, mean=None, inv_std=None, out_dtype=np.float32,
        layout="CHW", pad_channels=None, fill=None):
    return _cmn(lib().oracle_cmn, img, anchor, crop, mirror, mean, inv_std, out_dtype, layout, pad_channels, fill)


def ref_cmn(img, anchor=None, crop=None, mirror=False, mean=None, inv_std=None, out_dtype=np.float32,
            layout="CHW", pad_channels=None, fill=None):
    return _cmn(ref().ref_cmn, img, anchor, crop, mirror, mean, inv_std, out_dtype, layout, pad_channels, fill)


# ------------------------------------------------------------------------------------------- warp / colour
def _warp(fn, img, M, out_hw, interp, fill, out_dtype):
    img = np.ascontiguousarray(img, np.uint8)
    H, W, Cn = img.shape
    oh, ow = out_hw or (H, W)
    out = np.empty((oh, ow, Cn), np.dtype(out_dtype))
    M = _f32(np.asarray(M).reshape(6))
    border = 0 if fill is None else 1
    fl = np.full(Cn, 0.0 if fill is None else fill, np.float32)
    rc = fn(_p(img), H, W, Cn, _p(out), 0 if out.dtype == np.uint8 else 1, oh, ow, _p(M), int(interp), border, _p(fl))
    if rc != 0:
        raise RuntimeError(f"warp rc={rc}")
    return out


def warp_affine(img, M, out_hw=None, interp=1, fill=None, out_dtype=np.uint8):
    """M is the dst->src 2x3 matrix (fn.warp_affine's matrix with inverse_map=True)."""
    return _warp(lib().oracle_warp_affine, img, M, out_hw, interp, fill, out_dtype)


def ref_warp_affine(img, M, out_hw=None, interp=1, fill=None, out_dtype=np.uint8):
    return _warp(ref().ref_warp_affine, img, M, out_hw, interp, fill, out_dtype)


def affine_inv(M, use_ref=False):
    M = _f32(np.asarray(M).reshape(6))
    out = np.empty(6, np.float32)
    (ref().ref_affine_inv if use_ref else lib().oracle_affine_inv)(_p(M), _p(out))
    return out.reshape(2, 3)


def color_twist_matrix(hue=0.0, saturation=1.0, value=1.0, brightness=1.0, contrast=1.0, half_range=128.0, use_ref=False):
    M, T = np.empty(9, np.float32), np.empty(3, np.float32)
    fn = ref().ref_color_twist_matrix if use_ref else lib().oracle_color_twist_matrix
    fn(C.c_float(hue), C.c_float(saturation), C.c_float(value), C.c_float(brightness), C.c_float(contrast),
       C.c_float(half_range), _p(M), _p(T))
    return M.reshape(3, 3), T


def linear_transform(img, M, T, out_dtype=np.uint8, use_ref=False):
    img = np.ascontiguousarray(img, np.uint8)
    out = np.empty(img.shape, np.dtype(out_dtype))
    M, T = _f32(np.asarray(M).reshape(9)), _f32(np.asarray(T).reshape(3))
    npix = img.size // 3
    if use_ref:
        rc = ref().ref_linear_transform(_p(img), 1, npix, _p(out), 0 if out.dtype == np.uint8 else 1, _p(M), _p(T))
    else:
        rc = lib().oracle_linear_transform(_p(img), C.c_size_t(npix), _p(out), 0 if out.dtype == np.uint8 else 1, _p(M), _p(T))
    if rc != 0:
        raise RuntimeError(f"linear_transform rc={rc}")
    return out


def hsv(img, hue=0.0, saturation=1.0, value=1.0, out_dtype=np.uint8, use_ref=False):
    M, T = color_twist_matrix(hue, saturation, value, use_ref=use_ref)
    return linear_transform(img, M, T, out_dtype, use_ref=use_ref)


def csc(img, in_type, out_type, use_ref=False):
    img = np.ascontiguousarray(img, np.uint8)
    ic = 1 if in_type == IT_GRAY else 3
    oc = 1 if out_type == IT_GRAY else 3
    npix = img.size // ic
    out = np.empty(img.shape[:-1] + (oc,), np.uint8)
    if use_ref:
        rc = ref().ref_csc_bt601(_p(img), C.c_size_t(npix), _p(out), in_type, out_type)
    else:
        rc = lib().oracle_csc(_p(img), C.c_size_t(npix), _p(out), in_type, out_type)
    if rc != 0:
        raise RuntimeError(f"csc rc={rc}")
    return out


# ------------------------------------------------------------------------------------------- audio
def hann_window(n, use_ref=False):
    w = np.empty(n, np.float32)
    (ref().ref_hann_window if use_ref else lib().oracle_hann_window)(_p(w), n)
    return w


def num_windows(n, win_len, step, centered=True):
    return int(lib().oracle_num_windows(C.c_int64(n), win_len, step, int(centered)))


def extract_windows(sig, wfn, win_len, step, center=True, reflect=True, use_ref=False):
    sig, wfn = _f32(sig), _f32(wfn)
    nwin = num_windows(sig.size, win_len, step, center)
    out = np.empty((nwin, win_len), np.float32)
    pad = (2 if reflect else 1) if center else 0
    fn = ref().ref_extract_windows if use_ref else lib().oracle_extract_windows
    fn(_p(sig), C.c_int64(sig.size), _p(wfn), win_len, step, win_len // 2 if center else 0, pad, _p(out))
    return out


def spectrogram(sig, nfft=None, window_length=512, window_step=256, power=2, center=True, reflect=True,
                layout="ft", window_fn=None):
    sig = _f32(sig).ravel()
    nfft = nfft or window_length
    wfn = _f32(window_fn) if window_fn is not None else hann_window(window_length)
    nwin = num_windows(sig.size, window_length, window_step, center)
    nbin = nfft // 2 + 1
    out = np.empty((nbin, nwin) if layout == "ft" else (nwin, nbin), np.float32)
    rc = lib().oracle_spectrogram(_p(sig), C.c_int64(sig.size), _p(wfn), window_length, window_step, nfft, power,
                                  int(center), int(reflect), int(layout == "ft"), _p(out))
    if rc != 0:
        raise RuntimeError(f"spectrogram rc={rc}")
    return out


def mel_filter_bank(spec, nfilter=128, sample_rate=44100.0, freq_low=0.0, freq_high=0.0, mel_formula="slaney",
                    normalize=True, use_ref=False):
    spec = _f32(spec)
    nbin, nwin = spec.shape
    out = np.empty((nfilter, nwin), np.float32)
    if freq_high <= 0:
        freq_high = sample_rate / 2
    fn = ref().ref_mel_filter_bank_ft if use_ref else lib().oracle_mel_filter_bank_ft
    rc = fn(_p(spec), nbin, C.c_int64(nwin), _p(out), nfilter, C.c_float(sample_rate), C.c_float(freq_low),
            C.c_float(freq_high), int(mel_formula == "htk"), int(bool(normalize)))
    if rc != 0:
        raise RuntimeError(f"mel rc={rc}")
    return out


def mel_weights(nbin, nfilter=128, sample_rate=44100.0, freq_low=0.0, freq_high=0.0, mel_formula="slaney", normalize=True):
    W = np.empty((nfilter, nbin), np.float32)
    lib().oracle_mel_weights(_p(W), nbin, nfilter, C.c_float(sample_rate), C.c_float(freq_low), C.c_float(freq_high),
                             int(mel_formula == "htk"), int(bool(normalize)))
    return W


# ------------------------------------------------------------------------------------------- decoder post-conversion, random crops
def exif_transform(img, orientation):
    """The displayed (upright) image of a stored image with EXIF orientation 1..8 (TIFF/EXIF tag 0x0112)."""
    o = int(orientation)
    if o == 2:
        return img[:, ::-1]
    if o == 3:
        return img[::-1, ::-1]
    if o == 4:
        return img[::-1]
    if o == 5:
        return np.swapaxes(img, 0, 1)
    if o == 6:
        return np.swapaxes(img, 0, 1)[:, ::-1]
    if o == 7:
        return np.swapaxes(img, 0, 1)[::-1, ::-1]
    if o == 8:
        return np.swapaxes(img, 0, 1)[::-1]
    return img


def with_exif_orientation(jpeg_bytes, orientation):
    """Inserts a minimal APP1 / Exif segment carrying the orientation tag behind SOI."""
    tiff = b"II*\x00" + (8).to_bytes(4, "little") + (1).to_bytes(2, "little") + \
        (0x0112).to_bytes(2, "little") + (3).to_bytes(2, "little") + (1).to_bytes(4, "little") + int(orientation).to_bytes(2, "little") + b"\x00\x00" + \
        (0).to_bytes(4, "little")
    payload = b"Exif\x00\x00" + tiff
    seg = b"\xff\xe1" + (len(payload) + 2).to_bytes(2, "big") + payload
    b = bytes(jpeg_bytes)
    assert b[:2] == b"\xff\xd8"
    return b[:2] + seg + b[2:]


def ref_decoder_convert(img, out_type, out_float):
    """The reference's post-decode conversion (dali/operators/imgcodec/util/convert.h ConvertPixel functors) of a decoded RGB / GRAY
    u8 image: out_type IT_RGB / IT_BGR / IT_GRAY / IT_YCBCR, u8 or f32."""
    a = np.ascontiguousarray(img)
    in_c = 1 if a.ndim == 2 or a.shape[2] == 1 else 3
    npix = a.shape[0] * a.shape[1]
    oc = 1 if out_type == IT_GRAY else 3
    out = np.empty((a.shape[0], a.shape[1], oc), np.float32 if out_float else np.uint8)
    ref().ref_decoder_convert(_p(a), C.c_size_t(npix), in_c, int(out_type), int(bool(out_float)), _p(out))
    return out


def ref_random_crop(seed, sample_idx, H, W, aspect=(3 / 4, 4 / 3), area=(0.08, 1.0), num_attempts=10, ncalls=1):
    """[(anchor_y, anchor_x, h, w)] from the reference's RandomCropGenerator with RandomCropAttr's per-sample Philox state."""
    w = (C.c_int * (4 * ncalls))()
    ref().ref_random_crop(C.c_int64(seed), int(sample_idx), int(H), int(W), C.c_float(aspect[0]), C.c_float(aspect[1]),
                          C.c_float(area[0]), C.c_float(area[1]), int(num_attempts), int(ncalls), w)
    return [tuple(w[4 * k:4 * k + 4]) for k in range(ncalls)]


# ------------------------------------------------------------------------------------------- audio tail
def ref_to_decibels(x, multiplier=10.0, reference=None, cutoff_db=-200.0):
    """dali/kernels/signal/decibel/to_decibels_cpu.cc (compiled reference); reference=None -> per-sample maximum."""
    a = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(a)
    rc = ref().ref_to_decibels(_p(a), C.c_int64(a.size), _p(out), C.c_float(multiplier), C.c_float(reference if reference is not None else 1.0),
                               C.c_float(cutoff_db), int(reference is None))
    assert rc == 0
    return out


def to_decibels(x, multiplier=10.0, reference=None, cutoff_db=-200.0):
    """oracle/audio_oracle.c restatement of ToDecibels; reference=None -> per-sample maximum."""
    a = np.ascontiguousarray(x, np.float32)
    out = np.empty_like(a)
    lib().oracle_to_decibels(_p(a), C.c_int64(a.size), _p(out), C.c_float(multiplier), C.c_float(reference if reference is not None else 1.0),
                             C.c_float(cutoff_db), int(reference is None))
    return out


def mfcc(mel, n_mfcc=20, dct_type=2, normalize=False, lifter=0.0):
    """oracle/audio_oracle.c restatement of the DCT + liftering along axis 0 of [nfeat, ncols]."""
    a = np.ascontiguousarray(mel, np.float32)
    nfeat, ncols = a.shape
    out = np.empty((min(n_mfcc, nfeat), ncols), np.float32)
    rows = lib().oracle_mfcc(_p(a), nfeat, C.c_int64(ncols), _p(out), int(n_mfcc), int(dct_type), int(bool(normalize)), C.c_float(lifter))
    assert rows == out.shape[0], rows
    return out


def nonsilent_region(x, cutoff_db=-60.0, window_length=2048, reference_power=None, reset_interval=8192):
    """oracle/audio_oracle.c restatement of NonsilentRegion: (begin, length)."""
    a = np.ascontiguousarray(x, np.float32)
    b, l = C.c_int32(-1), C.c_int32(-1)
    lib().oracle_nonsilent_region(_p(a), C.c_int64(a.size), C.c_float(cutoff_db), C.c_float(reference_power or 0.0), int(reference_power is not None),
                                  int(window_length), int(reset_interval), C.byref(b), C.byref(l))
    return b.value, l.value


def audio_resample(x, in_rate, out_rate, quality=50.0, out_length=None):
    """oracle/audio_oracle.c restatement of AudioResample (float -> float); x: [n] or [n, channels]."""
    import math
    a = np.ascontiguousarray(x, np.float32)
    n_in, ch = a.shape[0], (a.shape[1] if a.ndim == 2 else 1)
    n_out = int(out_length) if out_length is not None else int(math.ceil(n_in * float(out_rate) / float(in_rate)))
    out = np.empty((n_out,) + a.shape[1:], np.float32)
    rc = lib().oracle_audio_resample(_p(a), C.c_int64(n_in), ch, C.c_double(in_rate), C.c_double(out_rate), C.c_int64(n_out), C.c_float(quality), _p(out))
    assert rc == 0
    return out


def ref_audio_resample(x, in_rate, out_rate, quality=50.0, out_length=None):
    """dali/kernels/signal/resampling_cpu.cc through ResamplerCPU (compiled reference); x: [n] or [n, channels] float32."""
    a = np.ascontiguousarray(x, np.float32)
    n_in, ch = a.shape[0], (a.shape[1] if a.ndim == 2 else 1)
    lib = ref()
    lib.ref_resampled_length.restype = C.c_int64
    n_out = int(out_length) if out_length is not None else int(lib.ref_resampled_length(C.c_int64(n_in), C.c_double(in_rate), C.c_double(out_rate)))
    out = np.empty((n_out,) + a.shape[1:], np.float32)
    rc = lib.ref_audio_resample(_p(a), C.c_int64(n_in), ch, C.c_double(in_rate), C.c_double(out_rate), C.c_int64(n_out), C.c_float(quality), _p(out))
    assert rc == 0
    return out


def ref_nonsilent_region(x, cutoff_db=-60.0, window_length=2048, reference_power=None, reset_interval=8192):
    """dali/operators/audio/nonsilence_op.h over the compiled reference kernels (moving mean square, dB -> magnitude): (begin, length)."""
    a = np.ascontiguousarray(x, np.float32)
    b, l = C.c_int32(-1), C.c_int32(-1)
    rc = ref().ref_nonsilent_region(_p(a), C.c_int64(a.size), C.c_float(cutoff_db), C.c_float(reference_power or 0.0), int(reference_power is not None),
                                    int(window_length), int(reset_interval), C.byref(b), C.byref(l))
    assert rc == 0
    return b.value, l.value


def ref_mfcc(mel, n_mfcc=20, dct_type=2, normalize=False, lifter=0.0):
    """dali/kernels/signal/dct/dct_cpu.cc along axis 0 of [nfeat, ncols] + the liftering of dali/operators/audio/mfcc."""
    a = np.ascontiguousarray(mel, np.float32)
    nfeat, ncols = a.shape
    out = np.empty((min(n_mfcc, nfeat), ncols), np.float32)
    rows = ref().ref_mfcc(_p(a), nfeat, C.c_int64(ncols), _p(out), int(n_mfcc), int(dct_type), int(bool(normalize)), C.c_float(lifter))
    assert rows == out.shape[0], rows
    return out


# ------------------------------------------------------------------------------------------- f4 operators
def ref_rotate_params(angle_deg, in_h, in_w, keep_size=False, size=None):
    """(out_h, out_w), 2x3 destination->source matrix of fn.rotate (rotate_params.h, built from the reference's transform.h)."""
    hw = (C.c_int * 2)()
    M = np.empty(6, np.float32)
    sz = None if size is None else (C.c_float * 2)(float(size[0]), float(size[1]))
    ref().ref_rotate_params(C.c_float(angle_deg), int(in_h), int(in_w), int(bool(keep_size)), sz, hw, _p(M))
    return (hw[0], hw[1]), M.reshape(2, 3)


def ref_brightness_contrast(img, brightness=1.0, brightness_shift=0.0, contrast=1.0, contrast_center=128.0, out_float=False):
    a = np.ascontiguousarray(img, np.uint8)
    out = np.empty(a.shape, np.float32 if out_float else np.uint8)
    ref().ref_brightness_contrast(_p(a), C.c_size_t(a.size), int(bool(out_float)), C.c_float(brightness), C.c_float(brightness_shift),
                                  C.c_float(contrast), C.c_float(contrast_center), _p(out))
    return out


# ---- reference random number operators (oracle/ref_random_shim.cc); only with oracle/_ref
def ref_random_coin_flip(seed, iterations, batch, volume, probability, dtype=np.int32):
    code = {np.dtype(np.int32): 6, np.dtype(np.uint8): 0}[np.dtype(dtype)]
    out = np.empty((iterations, batch, volume), dtype)
    rc = ref().ref_random_coin_flip(C.c_int64(seed), iterations, batch, C.c_int64(volume), C.c_float(probability), code,
                                        out.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return out


def ref_random_uniform(seed, iterations, batch, volume, rng=(-1.0, 1.0), values=None, dtype=np.float32):
    code = {np.dtype(np.uint8): 0, np.dtype(np.int16): 5, np.dtype(np.int32): 6, np.dtype(np.int64): 7, np.dtype(np.float32): 9,
            np.dtype(np.float64): 10}[np.dtype(dtype)]
    out = np.empty((iterations, batch, volume), dtype)
    vals = None if values is None else np.ascontiguousarray(values, np.float32)
    rc = ref().ref_random_uniform(C.c_int64(seed), iterations, batch, C.c_int64(volume), C.c_float(rng[0]), C.c_float(rng[1]),
                                      None if vals is None else vals.ctypes.data_as(C.c_void_p), C.c_int64(0 if vals is None else vals.size),
                                      code, out.ctypes.data_as(C.c_void_p))
    assert rc == 0
    return out


def ref_philox(key, sequence, offset, n):
    out = np.empty(n, np.uint32)
    ref().ref_philox(C.c_uint64(key), C.c_uint64(sequence), C.c_uint64(offset), n, out.ctypes.data_as(C.c_void_p))
    return out
