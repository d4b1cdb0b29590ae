"""Two integer statements of libjpeg's "islow" IDCT (Loeffler-Ligtenberg-Moschytz, CONST_BITS 13, PASS1_BITS 2), vectorised over blocks.

idct16() is the dataflow of libjpeg-turbo's x86 SIMD kernels (jidctint-sse2 / -avx2), which is what cv2.imdecode runs:
  - dequantisation keeps the low 16 bits of coef * q (pmullw);
  - i0 +- i4, i7 + i3 and i5 + i1 wrap to 16 bits (paddw / psubw);
  - the multiply-adds are exact in 32 bits (pmaddwd) and every later sum wraps to 32 bits (paddd);
  - each pass's output saturates to int16 (packssdw), the result to [-128, 127] (packsswb) before 128 is added;
  - a block whose COEFFICIENTS in rows 1..7 are all zero skips pass 1: every row of the workspace is row 0 of the dequantised block
    shifted left by PASS1_BITS in 16 bits (psllw).
idct_c() is libjpeg's C jidctint: 32-bit dequantisation and arithmetic, range_limit[(x + 128) & 1023].

On every block of a natural (encoder-made) stream the two agree; they part only where coefficients are far out of range.
Blocks are [..., 64] int arrays in natural order (row = vertical frequency); q broadcasts against them.  Both return [..., 8, 8] uint8."""
import numpy as np


def w16(x):
    return ((x + 32768) & 0xFFFF) - 32768


def i32(x):
    return ((x + (1 << 31)) & 0xFFFFFFFF) - (1 << 31)


def _pass16(v, shift):
    """one 1-D pass along the last axis of int64 v [..., 8] holding int16 values; returns the saturated int16 outputs [..., 8]"""
    i0, i1, i2, i3, i4, i5, i6, i7 = (v[..., k] for k in range(8))
    tmp3 = i2 * 10703 + i6 * 4433
    tmp2 = i2 * 4433 - i6 * 10704
    tmp0 = i32(w16(i0 + i4) << 13)
    tmp1 = i32(w16(i0 - i4) << 13)
    t10, t13, t11, t12 = i32(tmp0 + tmp3), i32(tmp0 - tmp3), i32(tmp1 + tmp2), i32(tmp1 - tmp2)
    z3, z4 = w16(i7 + i3), w16(i5 + i1)
    Z3 = z3 * -6436 + z4 * 9633
    Z4 = z3 * 9633 + z4 * 6437
    o0 = i32(i7 * -4927 + i1 * -7373 + Z3)
    o3 = i32(i7 * -7373 + i1 * 4926 + Z4)
    o1 = i32(i5 * -4176 + i3 * -20995 + Z4)
    o2 = i32(i5 * -20995 + i3 * 4177 + Z3)
    outs = [t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3]
    return np.stack([np.clip(i32(i32(x) + (1 << (shift - 1))) >> shift, -32768, 32767) for x in outs], -1)


def idct16(coef, q):
    coef = np.asarray(coef, np.int64)
    d = w16(coef * np.asarray(q, np.int64)).reshape(coef.shape[:-1] + (8, 8))
    skip = ~np.asarray(coef, np.int64).reshape(d.shape)[..., 1:, :].any(axis=(-2, -1))
    ws = np.swapaxes(_pass16(np.swapaxes(d, -1, -2), 11), -1, -2)          # pass 1 along the columns
    ws = np.where(skip[..., None, None], w16(d[..., :1, :] << 2), ws)
    return (np.clip(_pass16(ws, 18), -128, 127) + 128).astype(np.uint8)


def _pass_c(v, shift):
    """jidctint.c's 1-D pass (32-bit C arithmetic) along the last axis of int64 v [..., 8]"""
    z2, z3 = v[..., 2], v[..., 6]
    z1 = i32((z2 + z3) * 4433)
    tmp2 = i32(z1 + z3 * -15137)
    tmp3 = i32(z1 + z2 * 6270)
    tmp0 = i32((v[..., 0] + v[..., 4]) << 13)
    tmp1 = i32((v[..., 0] - v[..., 4]) << 13)
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    a0, a1, a2, a3 = v[..., 7], v[..., 5], v[..., 3], v[..., 1]
    z1, z2, z3, z4 = a0 + a3, a1 + a2, a0 + a2, a1 + a3
    z5 = i32((z3 + z4) * 9633)
    a0, a1, a2, a3 = i32(a0 * 2446), i32(a1 * 16819), i32(a2 * 25172), i32(a3 * 12299)
    z1, z2 = i32(z1 * -7373), i32(z2 * -20995)
    z3, z4 = i32(z3 * -16069 + z5), i32(z4 * -3196 + z5)
    a0, a1, a2, a3 = i32(a0 + z1 + z3), i32(a1 + z2 + z4), i32(a2 + z2 + z3), i32(a3 + z1 + z4)
    outs = [t10 + a3, t11 + a2, t12 + a1, t13 + a0, t13 - a0, t12 - a1, t11 - a2, t10 - a3]
    return np.stack([i32(i32(x) + (1 << (shift - 1))) >> shift for x in outs], -1)


def idct_c(coef, q):
    coef = np.asarray(coef, np.int64)
    d = i32(coef * np.asarray(q, np.int64)).reshape(coef.shape[:-1] + (8, 8))
    ws = np.swapaxes(_pass_c(np.swapaxes(d, -1, -2), 11), -1, -2)
    y = (_pass_c(ws, 18) + 128) & 1023
    return np.where(y < 256, y, np.where(y < 640, 255, 0)).astype(np.uint8)
