"""Plain numpy references of the per-pixel conversions whose kernels have no compiled reference on a GPU machine: the image decoder's
post pass (output type / dtype, jpeg.cu jpeg_post_kernel) and fn.brightness_contrast (generic.cu multiply_add_kernel).

Each operation has two forms:
  * a float32 restatement in the reference's operation order.  numpy's float32 scalar / array operations round to nearest and are
    never fused, so a kernel that rounds the same steps in the same order agrees bit for bit;
  * a float64 statement of the formula, which catches a mistake the restatement could share with the kernel (a coefficient, a bias,
    a channel order, a range).
tests/test_pointwise_ref_cpu.py pins the two forms against each other and, where oracle/_ref exists, against the reference's code."""
import numpy as np

RGB, BGR, GRAY, YCBCR = 0, 1, 2, 3                     # the decoder's output types (capi.RGB ... / pyoracle.IT_RGB ...)

INV255 = np.float32(1.0 / 255)                        # ConvertSatNorm<float>(uint8_t): v * (1.0f / 255) (convert.h:263-275)
# kernels::color::itu_r_bt_601::rgb_to_ycbcr (color_space_conversion_impl.h:64-103): rows Y, Cb, Cr over (R, G, B)
YCBCR_COEFFS = ((0.25678823529, 0.50412941176, 0.09790588235),
                (-0.14822289945, -0.29099278682, 0.43921568627),
                (0.43921568627, -0.36778831435, -0.07142737192))


def round_sat_u8(x):
    """ConvertSat<uint8_t>(float): round half away from zero, then saturate.  Exact: a float32 plus 0.5 is exact in float64."""
    x = np.asarray(x, np.float64)
    return np.clip(np.floor(np.abs(x) + 0.5) * np.sign(x), 0, 255).astype(np.uint8)


def _rgb_planes(img):
    a = np.asarray(img)
    assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 3, (a.dtype, a.shape)
    return a[..., 0], a[..., 1], a[..., 2]


def decoder_convert(img, out_type, out_float):
    """float32 form of the post pass.  img: the u8 RGB decode (H, W, 3), or for GRAY the u8 Y plane (H, W, 1).  Grayscale streams
    decoded to YCbCr go through the RGB formula with R = G = B, as the kernel does (src_c is 1 only for GRAY output)."""
    a = np.asarray(img)
    if out_type == GRAY:
        assert a.dtype == np.uint8 and a.ndim == 3 and a.shape[2] == 1, (a.dtype, a.shape)
        return a.astype(np.float32) * INV255 if out_float else a.copy()
    r, g, b = _rgb_planes(a)
    if out_type in (RGB, BGR):
        out = np.stack((r, g, b) if out_type == RGB else (b, g, r), -1)
        return out.astype(np.float32) * INV255 if out_float else out
    assert out_type == YCBCR, out_type
    sf = INV255 if out_float else np.float32(1)        # vec3 * scale_factor<uint8_t, Out>(): a float product per coefficient
    bias = (np.float32(0.0625), np.float32(0.5)) if out_float else (np.float32(16), np.float32(128))
    fr, fg, fb = r.astype(np.float32), g.astype(np.float32), b.astype(np.float32)
    planes = []
    for k, (c0, c1, c2) in enumerate(YCBCR_COEFFS):
        k0, k1, k2 = np.float32(c0) * sf, np.float32(c1) * sf, np.float32(c2) * sf
        planes.append((k0 * fr + k1 * fg) + k2 * fb + bias[min(k, 1)])
    out = np.stack(planes, -1)
    return out if out_float else round_sat_u8(out)


def decoder_convert_f64(img, out_type, out_float):
    """float64 statement of the post pass: v / 255 for RGB / BGR / GRAY, BT.601 with biases 16 / 128 (u8) or 0.0625 / 0.5 (float)
    for YCbCr.  u8 results are the unrounded values (compare with assert_u8_matches_f64)."""
    a = np.asarray(img).astype(np.float64)
    scale = 1 / 255 if out_float else 1.0
    if out_type == GRAY:
        return a * scale
    r, g, b = a[..., 0], a[..., 1], a[..., 2]
    if out_type in (RGB, BGR):
        return np.stack((r, g, b) if out_type == RGB else (b, g, r), -1) * scale
    bias = (0.0625, 0.5) if out_float else (16.0, 128.0)
    return np.stack([(c0 * r + c1 * g + c2 * b) * scale + bias[min(k, 1)] for k, (c0, c1, c2) in enumerate(YCBCR_COEFFS)], -1)


def brightness_contrast_args(brightness, shift, contrast, center=128.0, out_float=False):
    """(multiplier, addend) of BrightnessContrast in float32, each step rounded in the reference's order (brightness_contrast.h:84-103):
    add = shift * range + brightness * (center - contrast * center), mul = brightness * contrast; range 255 (u8) or 1 (float)."""
    b, s, c, ctr = (np.float32(v) for v in (brightness, shift, contrast, center))
    rng = np.float32(1 if out_float else 255)
    return b * c, s * rng + b * (ctr - c * ctr)


def brightness_contrast(img, brightness, shift, contrast, center=128.0, out_float=False):
    """float32 form: out = ConvertSat<Out>(in * mul + add), the product and the sum rounded separately."""
    a = np.asarray(img)
    assert a.dtype == np.uint8, a.dtype
    mul, add = brightness_contrast_args(brightness, shift, contrast, center, out_float)
    v = a.astype(np.float32) * mul + add
    return v if out_float else round_sat_u8(v)


def brightness_contrast_f64(img, brightness, shift, contrast, center=128.0, out_float=False):
    """float64 statement: shift * range + brightness * (center + contrast * (in - center)), of the float32 arguments the operator
    receives; u8 results are the unrounded values."""
    b, s, c, ctr = (float(np.float32(v)) for v in (brightness, shift, contrast, center))
    return s * (1.0 if out_float else 255.0) + b * (ctr + c * (np.asarray(img).astype(np.float64) - ctr))


def assert_u8_matches_f64(got, ref64, tie_eps=1e-4, what=""):
    """got == round-half-away-and-saturate(ref64) everywhere, except that where ref64 lies within tie_eps of a half the other neighbour
    is accepted too (the float32 computation may land on either side of such a tie).  Returns the number of elements that needed
    this guard; callers assert it stays small, so that the guard cannot hide a systematic error."""
    got, ref64 = np.asarray(got), np.asarray(ref64, np.float64)
    assert got.shape == ref64.shape and got.dtype == np.uint8, (what, got.shape, got.dtype, ref64.shape)
    lo = np.floor(ref64)
    tie = np.abs(ref64 - lo - 0.5) < tie_eps
    g = got.astype(np.float64)
    exact = g == np.clip(np.floor(ref64 + 0.5), 0, 255)
    ok = exact | (tie & ((g == np.clip(lo, 0, 255)) | (g == np.clip(lo + 1, 0, 255))))
    if not ok.all():
        bad = np.argwhere(~ok)[:5]
        raise AssertionError(f"{what}: {int((~ok).sum())} elements differ from the float64 form, first at "
                             f"{[(tuple(int(v) for v in i), int(got[tuple(i)]), float(ref64[tuple(i)])) for i in bad]}")
    return int((~exact).sum())


def assert_f32_close(got, ref64, atol, what=""):
    got, ref64 = np.asarray(got), np.asarray(ref64, np.float64)
    assert got.shape == ref64.shape and got.dtype == np.float32, (what, got.shape, got.dtype, ref64.shape)
    err = np.abs(got.astype(np.float64) - ref64)
    assert np.all(err <= atol), (what, float(err.max()), atol)


def check_decoder_output(got, src, out_type, out_float, what=""):
    """A decoder output against both forms: bit-exact with the float32 form; float outputs also within 1e-6 of the float64 form, u8
    YCbCr also rounded from it (the float32 form is pinned to it over every input by tests/test_pointwise_ref_cpu.py)."""
    want = decoder_convert(src, out_type, out_float)
    got = np.asarray(got)
    assert got.shape == want.shape and got.dtype == want.dtype, (what, got.shape, got.dtype, want.shape, want.dtype)
    if out_float:
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (what, "float32 form")
        assert_f32_close(got, decoder_convert_f64(src, out_type, True), 1e-6, what)
    else:
        assert np.array_equal(got, want), (what, "float32 form")
