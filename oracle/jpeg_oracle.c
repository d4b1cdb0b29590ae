/*
 * oracle/jpeg_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the baseline-JPEG decode arithmetic that the reference reaches through
 * nvImageCodec's libjpeg-turbo CPU extension (reference call sites:
 * dali/operators/imgcodec/image_decoder.h:265-281 (extension list), :473-499 (ParseSample),
 * :767-816 (decode); CPU backend always uses fancy upsampling, image_decoder.h:297-304,468-470).
 * The arithmetic itself is NOT in /root/reference (un-vendored dependency: nvimgcodec >=0.9,<0.10,
 * cmake/Dependencies.common.cmake:310-311 -> libjpeg-turbo).  It is restated here from the
 * published algorithms:
 *   - ITU-T T.81 Annex B (markers), C (Huffman table generation), F.2.2 (sequential decode),
 *   - libjpeg "islow" integer IDCT (Loeffler-Ligtenberg-Moschytz, CONST_BITS=13, PASS1_BITS=2) in the 16-bit dataflow of
 *     libjpeg-turbo's x86 SIMD kernels (see jo_idct_block),
 *   - libjpeg "fancy" (triangle) h2v1 / h2v2 chroma upsampling,
 *   - libjpeg fixed-point (SCALEBITS=16) YCbCr->RGB.
 * Pinned (tests/test_oracle_jpeg.py, tests/golden/) against cv2.imdecode (OpenCV 4.13 bundling
 * libjpeg-turbo 3.1.2 -- the same codec family/defaults the reference's CPU decoder uses);
 * the pin is bit-exact, which is tighter than the reference's own decoder tests
 * (dali/test/python/decoder/test_image.py:308-321, mean abs err <= 4).
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg may call this.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>

#define JO_OK 0
#define JO_ERR_FORMAT -1
#define JO_ERR_UNSUPPORTED -2

typedef struct {
  int width, height;
  int ncomp;
  int hs[4], vs[4], tq[4], cid[4];
  int hmax, vmax;
  int mcux, mcuy;          /* MCUs per row / column */
  int restart_interval;
  int progressive;
  int precision;
  int adobe_transform;     /* -1: no Adobe marker */
  int jfif;
  int orientation;         /* EXIF orientation (1 if absent) */
  /* per component padded block grid */
  int bw[4], bh[4];        /* blocks per row / col (padded to whole MCUs) */
} jo_info;

typedef struct {
  uint8_t bits[17];
  uint8_t vals[256];
  int present;
  /* derived */
  int mincode[17], maxcode[18], valptr[17];
} jo_huff;

typedef struct {
  const uint8_t *data;
  size_t len;
  jo_info info;
  uint16_t qt[4][64];      /* natural order */
  int qt_present[4];
  jo_huff dc[4], ac[4];
  int td[4], ta[4];        /* per scan component */
  size_t scan_begin;       /* offset of entropy-coded data */
  int scan_ncomp;
  int scan_comp[4];
} jo_dec;

static const uint8_t jo_zigzag[64] = {
   0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5,
  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
  58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };

static int rd16(const uint8_t *p) { return (p[0] << 8) | p[1]; }

/* T.81 Annex C: generate code tables */
static void jo_build_huff(jo_huff *h) {
  int code = 0, k = 0;
  for (int l = 1; l <= 16; l++) {
    h->valptr[l] = k;
    h->mincode[l] = code;
    k += h->bits[l];
    code += h->bits[l];
    h->maxcode[l] = h->bits[l] ? code - 1 : -1;
    code <<= 1;
  }
  h->maxcode[17] = 0x7fffffff;
}

static int jo_parse_exif_orientation(const uint8_t *p, int len) {
  /* p points after "Exif\0\0" */
  if (len < 8) return 1;
  int le;
  if (p[0] == 'I' && p[1] == 'I') le = 1; else if (p[0] == 'M' && p[1] == 'M') le = 0; else return 1;
#define R16(o) (le ? (p[o] | (p[(o)+1] << 8)) : ((p[o] << 8) | p[(o)+1]))
#define R32(o) (le ? (p[o] | (p[(o)+1] << 8) | (p[(o)+2] << 16) | ((unsigned)p[(o)+3] << 24)) \
                   : (((unsigned)p[o] << 24) | (p[(o)+1] << 16) | (p[(o)+2] << 8) | p[(o)+3]))
  unsigned ifd = R32(4);
  if (ifd + 2 > (unsigned)len) return 1;
  int n = R16(ifd);
  for (int i = 0; i < n; i++) {
    unsigned e = ifd + 2 + 12 * i;
    if (e + 12 > (unsigned)len) return 1;
    if (R16(e) == 0x0112) {
      int v = R16(e + 8);
      return (v >= 1 && v <= 8) ? v : 1;
    }
  }
#undef R16
#undef R32
  return 1;
}

static int jo_parse(jo_dec *d) {
  const uint8_t *p = d->data;
  size_t n = d->len, pos = 2;
  jo_info *in = &d->info;
  memset(in, 0, sizeof(*in));
  in->adobe_transform = -1;
  in->orientation = 1;
  if (n < 4 || p[0] != 0xFF || p[1] != 0xD8) return JO_ERR_FORMAT;
  int got_sof = 0;
  while (pos + 4 <= n) {
    if (p[pos] != 0xFF) return JO_ERR_FORMAT;
    while (pos < n && p[pos] == 0xFF) pos++;     /* fill bytes */
    if (pos >= n) return JO_ERR_FORMAT;
    int m = p[pos++];
    if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;
    if (m == 0xD9) return JO_ERR_FORMAT;         /* EOI before SOS */
    if (pos + 2 > n) return JO_ERR_FORMAT;
    int L = rd16(p + pos);
    if (L < 2 || pos + L > n) return JO_ERR_FORMAT;
    const uint8_t *s = p + pos + 2;
    int sl = L - 2;
    if (m == 0xDB) {                             /* DQT */
      int o = 0;
      while (o < sl) {
        int pq = s[o] >> 4, tq = s[o] & 15; o++;
        if (tq > 3) return JO_ERR_FORMAT;
        for (int i = 0; i < 64; i++) {
          int v;
          if (pq) { v = rd16(s + o); o += 2; } else { v = s[o++]; }
          d->qt[tq][jo_zigzag[i]] = (uint16_t)v;
        }
        d->qt_present[tq] = 1;
      }
    } else if (m == 0xC4) {                      /* DHT */
      int o = 0;
      while (o < sl) {
        int tc = s[o] >> 4, th = s[o] & 15; o++;
        if (th > 3 || tc > 1) return JO_ERR_FORMAT;
        jo_huff *h = tc ? &d->ac[th] : &d->dc[th];
        int cnt = 0;
        h->bits[0] = 0;
        for (int i = 1; i <= 16; i++) { h->bits[i] = s[o++]; cnt += h->bits[i]; }
        if (cnt > 256 || o + cnt > sl) return JO_ERR_FORMAT;
        memcpy(h->vals, s + o, cnt); o += cnt;
        h->present = 1;
        jo_build_huff(h);
      }
    } else if (m == 0xC0 || m == 0xC1 || m == 0xC2) {   /* SOF0/1/2 */
      in->progressive = (m == 0xC2);
      in->precision = s[0];
      in->height = rd16(s + 1);
      in->width = rd16(s + 3);
      in->ncomp = s[5];
      if (in->ncomp < 1 || in->ncomp > 4 || sl < 6 + 3 * in->ncomp) return JO_ERR_FORMAT;
      for (int c = 0; c < in->ncomp; c++) {
        in->cid[c] = s[6 + 3 * c];
        in->hs[c] = s[7 + 3 * c] >> 4;
        in->vs[c] = s[7 + 3 * c] & 15;
        in->tq[c] = s[8 + 3 * c];
        if (in->hs[c] < 1 || in->hs[c] > 4 || in->vs[c] < 1 || in->vs[c] > 4 || in->tq[c] > 3)
          return JO_ERR_FORMAT;
        if (in->hs[c] > in->hmax) in->hmax = in->hs[c];
        if (in->vs[c] > in->vmax) in->vmax = in->vs[c];
      }
      got_sof = 1;
    } else if (m >= 0xC3 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      return JO_ERR_UNSUPPORTED;                 /* lossless / arithmetic / hierarchical */
    } else if (m == 0xDD) {                      /* DRI */
      in->restart_interval = rd16(s);
    } else if (m == 0xE0) {
      if (sl >= 5 && !memcmp(s, "JFIF\0", 5)) in->jfif = 1;
    } else if (m == 0xE1) {
      if (sl >= 6 && !memcmp(s, "Exif\0\0", 6))
        in->orientation = jo_parse_exif_orientation(s + 6, sl - 6);
    } else if (m == 0xEE) {
      if (sl >= 12 && !memcmp(s, "Adobe", 5)) in->adobe_transform = s[11];
    } else if (m == 0xDA) {                      /* SOS */
      if (!got_sof) return JO_ERR_FORMAT;
      d->scan_ncomp = s[0];
      if (d->scan_ncomp < 1 || d->scan_ncomp > 4) return JO_ERR_FORMAT;
      for (int i = 0; i < d->scan_ncomp; i++) {
        int cs = s[1 + 2 * i], ci = -1;
        for (int c = 0; c < in->ncomp; c++) if (in->cid[c] == cs) ci = c;
        if (ci < 0) return JO_ERR_FORMAT;
        d->scan_comp[i] = ci;
        d->td[i] = s[2 + 2 * i] >> 4;
        d->ta[i] = s[2 + 2 * i] & 15;
      }
      d->scan_begin = pos + L;
      break;
    }
    pos += L;
  }
  if (!got_sof || !d->scan_begin) return JO_ERR_FORMAT;
  if (in->width == 0 || in->height == 0) return JO_ERR_FORMAT;
  in->mcux = (in->width + 8 * in->hmax - 1) / (8 * in->hmax);
  in->mcuy = (in->height + 8 * in->vmax - 1) / (8 * in->vmax);
  for (int c = 0; c < in->ncomp; c++) {
    in->bw[c] = in->mcux * in->hs[c];
    in->bh[c] = in->mcuy * in->vs[c];
  }
  return JO_OK;
}

/* ---------------------------------------------------------------- entropy decode (T.81 F.2.2) */
typedef struct {
  const uint8_t *p;
  size_t pos, end;
  uint32_t acc;
  int nbits;
  int marker;       /* pending marker seen (stops feeding real bits) */
  int pad;          /* the last `pad` bits of the window are zero padding supplied behind a marker or the end of the data */
  int overrun;      /* padding bits have been CONSUMED (decoded as data) */
} jo_bits;

static void jo_fill(jo_bits *b) {
  while (b->nbits <= 24) {
    int byte = 0, real = 0;
    if (!b->marker && b->pos < b->end) {
      byte = b->p[b->pos];
      if (byte == 0xFF) {
        int nx = b->pos + 1 < b->end ? b->p[b->pos + 1] : 0xD9;
        if (nx == 0x00) { b->pos += 2; real = 1; }
        else { b->marker = nx; byte = 0; }      /* do not consume the marker */
      } else {
        b->pos++; real = 1;
      }
    }
    if (!real) b->pad += 8;
    b->acc |= (uint32_t)byte << (24 - b->nbits);
    b->nbits += 8;
  }
}
static inline void jo_drop(jo_bits *b, int n) {
  b->acc <<= n; b->nbits -= n;
  if (b->nbits < b->pad) { b->overrun = 1; b->pad = b->nbits; }
}
static inline int jo_getbits(jo_bits *b, int n) {
  if (n == 0) return 0;
  if (b->nbits < n) jo_fill(b);
  int v = (int)(b->acc >> (32 - n));
  jo_drop(b, n);
  return v;
}
/* libjpeg jdhuff.c jpeg_huff_decode: a code that matches no length up to 16 consumes 17 bits and yields symbol 0.  The macros below
 * exist so that tests/test_jpeg_extreme_cpu.py can build variants with planted mistakes and show that its comparisons catch them. */
#ifndef JO_BAD_CODE_BITS
#define JO_BAD_CODE_BITS 17
#endif
static int jo_decode_sym(jo_bits *b, const jo_huff *h) {
  if (b->nbits < 17) jo_fill(b);
  int code = 0;
  for (int l = 1; l <= 16; l++) {
    code = (int)(b->acc >> (32 - l));
    if (h->maxcode[l] >= 0 && code <= h->maxcode[l] && code >= h->mincode[l]) {
      jo_drop(b, l);
      return h->vals[h->valptr[l] + code - h->mincode[l]];
    }
  }
  jo_drop(b, JO_BAD_CODE_BITS);
  return 0;   /* corrupt stream: libjpeg warns and substitutes 0 */
}
static inline int jo_extend(int v, int s) { return (s && v < (1 << (s - 1))) ? v - (1 << s) + 1 : v; }

/* Whether the last jo_entropy() decoded padding bits supplied behind a marker (or the end of the data) in any unit (restart interval or
 * whole scan): the unit ran out of data, which libjpeg answers with zeros and the GPU decoder with status 1. */
static int jo_overrun;
int jpeg_oracle_overrun(void) { return jo_overrun; }

/* Decode all blocks of the (single, interleaved or 1-component) scan.
 * coef[c]: int16 [bh*bw][64] natural order, quantized (NOT dequantized). */
static int jo_entropy(jo_dec *d, int16_t *coef[4]) {
  jo_info *in = &d->info;
  jo_overrun = 0;
  if (in->progressive) return JO_ERR_UNSUPPORTED;
  if (in->precision != 8) return JO_ERR_UNSUPPORTED;
  if (d->scan_ncomp != in->ncomp) return JO_ERR_UNSUPPORTED;   /* multi-scan baseline */
  for (int i = 0; i < d->scan_ncomp; i++)
    if (!d->dc[d->td[i]].present || !d->ac[d->ta[i]].present) return JO_ERR_FORMAT;
  jo_bits b = { d->data, d->scan_begin, d->len, 0, 0, 0, 0, 0 };
  int pred[4] = {0, 0, 0, 0};
  int nmcu = in->mcux * in->mcuy;
  int rst_left = in->restart_interval;
  for (int m = 0; m < nmcu; m++) {
    if (in->restart_interval && rst_left == 0) {
      /* byte align, expect RSTn */
      b.acc = 0; b.nbits = 0; b.pad = 0;
      /* 0xFF fill bytes in front of the marker (T.81 B.1.1.2), which libjpeg's next_marker skips */
      if (b.marker == 0xFF)
        while (b.pos + 1 < b.end && b.p[b.pos] == 0xFF && b.p[b.pos + 1] == 0xFF) b.pos++;
      if (!b.marker) {
        /* skip to next marker */
        while (b.pos + 1 < b.end && !(b.p[b.pos] == 0xFF && b.p[b.pos + 1] >= 0xD0 && b.p[b.pos + 1] <= 0xD7)) b.pos++;
      }
      if (b.pos + 1 < b.end && b.p[b.pos] == 0xFF && b.p[b.pos + 1] >= 0xD0 && b.p[b.pos + 1] <= 0xD7) b.pos += 2;
      b.marker = 0;
      pred[0] = pred[1] = pred[2] = pred[3] = 0;
      rst_left = in->restart_interval;
    }
    int mx = m % in->mcux, my = m / in->mcux;
    for (int i = 0; i < d->scan_ncomp; i++) {
      int c = d->scan_comp[i];
      const jo_huff *hd = &d->dc[d->td[i]], *ha = &d->ac[d->ta[i]];
      for (int v = 0; v < in->vs[c]; v++)
        for (int h = 0; h < in->hs[c]; h++) {
          int bx = mx * in->hs[c] + h, by = my * in->vs[c] + v;
          int16_t *blk = coef[c] + ((size_t)by * in->bw[c] + bx) * 64;
          int s = jo_decode_sym(&b, hd);
          int diff = s ? jo_extend(jo_getbits(&b, s), s) : 0;
          pred[c] += diff;
          blk[0] = (int16_t)pred[c];
          for (int k = 1; k < 64; ) {
            int rs = jo_decode_sym(&b, ha);
            int r = rs >> 4, ss = rs & 15;
            if (ss == 0) {
              if (r == 15) { k += 16; continue; }
              break;                              /* EOB */
            }
            k += r;                               /* a run past 63 (corrupt) lands on 63: jpeg_natural_order's guard entries */
#ifdef JO_RUN_PAST_63_BREAKS
            if (k > 63) break;
#endif
            blk[jo_zigzag[k > 63 ? 63 : k]] = (int16_t)jo_extend(jo_getbits(&b, ss), ss);
            k++;
          }
        }
    }
    if (in->restart_interval) rst_left--;
  }
  jo_overrun = b.overrun;
  return JO_OK;
}

/* ---------------------------------------------------------------- islow IDCT, as libjpeg-turbo's x86 SIMD kernels compute it
 * The islow algorithm of libjpeg's jidctint.c (Loeffler-Ligtenberg-Moschytz, CONST_BITS 13, PASS1_BITS 2) in the 16-bit dataflow of
 * jidctint-sse2 / -avx2, the IDCT cv2.imdecode runs.  On natural streams it equals the C code; they part where coefficients are far out
 * of range (a damaged stream, a hostile encoder, 16-bit DQT):
 *   - dequantisation keeps the low 16 bits of coef * q (pmullw);
 *   - i0 +- i4, i7 + i3 and i5 + i1 wrap to 16 bits (paddw / psubw); the products and their sums are exact in 32 bits (pmaddwd);
 *   - each pass's output saturates to int16 (packssdw), the result to [-128, 127] before 128 is added (packsswb);
 *   - a block whose coefficients in rows 1..7 are all zero skips pass 1: the workspace rows are row 0 of the dequantised block shifted
 *     left by PASS1_BITS in 16 bits (psllw), so they wrap instead of saturating.
 * tests/jpeg_idct16.py states the same in numpy; tests/test_jpeg_extreme_cpu.py pins both against cv2. */
static inline int jo_w16(int x) { return (int16_t)(uint16_t)(unsigned)x; }
static inline int jo_sat16(int x) { return x < -32768 ? -32768 : x > 32767 ? 32767 : x; }

/* in[0..7]: int16 values; out: the descaled 32-bit results (the caller saturates).  No sum below leaves 32 bits for int16 inputs. */
static void jo_idct_1d(const int in[8], int out[8], int shift) {
  const int tmp3 = in[2] * 10703 + in[6] * 4433, tmp2 = in[2] * 4433 - in[6] * 10704;
  const int tmp0 = jo_w16(in[0] + in[4]) * 8192, tmp1 = jo_w16(in[0] - in[4]) * 8192;
  const int t10 = tmp0 + tmp3, t13 = tmp0 - tmp3, t11 = tmp1 + tmp2, t12 = tmp1 - tmp2;
  const int z3 = jo_w16(in[7] + in[3]), z4 = jo_w16(in[5] + in[1]);
  const int Z3 = z3 * -6436 + z4 * 9633, Z4 = z3 * 9633 + z4 * 6437;
  const int o0 = in[7] * -4927 + in[1] * -7373 + Z3, o3 = in[7] * -7373 + in[1] * 4926 + Z4;
  const int o1 = in[5] * -4176 + in[3] * -20995 + Z4, o2 = in[5] * -20995 + in[3] * 4177 + Z3;
  const int r = 1 << (shift - 1);
  out[0] = (t10 + o3 + r) >> shift; out[7] = (t10 - o3 + r) >> shift;
  out[1] = (t11 + o2 + r) >> shift; out[6] = (t11 - o2 + r) >> shift;
  out[2] = (t12 + o1 + r) >> shift; out[5] = (t12 - o1 + r) >> shift;
  out[3] = (t13 + o0 + r) >> shift; out[4] = (t13 - o0 + r) >> shift;
}

static void jo_idct_block(const int16_t *coef, const uint16_t *q, uint8_t *out, int stride) {
  int ws[64], skip = 1;
  for (int i = 8; i < 64; i++) skip &= coef[i] == 0;
  for (int x = 0; x < 8; x++) {               /* pass 1: columns */
    int in[8], o[8];
    for (int y = 0; y < 8; y++) in[y] = jo_w16(coef[y * 8 + x] * (int)q[y * 8 + x]);
    jo_idct_1d(in, o, 11);
    for (int y = 0; y < 8; y++) ws[y * 8 + x] = skip ? jo_w16(in[0] * 4) : jo_sat16(o[y]);
  }
  for (int y = 0; y < 8; y++) {               /* pass 2: rows */
    int o[8];
    jo_idct_1d(ws + y * 8, o, 18);
    for (int x = 0; x < 8; x++) out[y * stride + x] = (uint8_t)((o[x] < -128 ? -128 : o[x] > 127 ? 127 : o[x]) + 128);
  }
}

/* ---------------------------------------------------------------- upsampling + colour */
/* plane: component samples, pw x ph (padded); dw x dh = "downsampled" real size.
 * out: full-resolution plane W x H (W = image width, H = image height). */
static void jo_upsample(const uint8_t *pl, int pw, int dw, int dh, int hexp, int vexp, int fancy,
                        uint8_t *out, int W, int H) {
  if (hexp == 1 && vexp == 1) {
    for (int y = 0; y < H; y++) memcpy(out + (size_t)y * W, pl + (size_t)y * pw, W);
    return;
  }
  if (fancy && hexp == 2 && vexp == 1 && dw > 2) {          /* h2v1 fancy */
    for (int y = 0; y < H; y++) {
      const uint8_t *r = pl + (size_t)y * pw;
      uint8_t *o = out + (size_t)y * W;
      for (int x = 0; x < W; x++) {
        int i = x >> 1, v;
        if (x & 1) v = (i == dw - 1) ? r[i] : (r[i] * 3 + r[i + 1] + 2) >> 2;
        else       v = (i == 0) ? r[i] : (r[i] * 3 + r[i - 1] + 1) >> 2;
        o[x] = (uint8_t)v;
      }
    }
    return;
  }
  if (fancy && hexp == 2 && vexp == 2 && dw > 2) {          /* h2v2 fancy (triangle) */
    for (int y = 0; y < H; y++) {
      int i0 = y >> 1;
      int i1 = (y & 1) ? i0 + 1 : i0 - 1;
      if (i1 < 0) i1 = 0;
      if (i1 > dh - 1) i1 = dh - 1;
      const uint8_t *r0 = pl + (size_t)i0 * pw, *r1 = pl + (size_t)i1 * pw;
      uint8_t *o = out + (size_t)y * W;
      for (int x = 0; x < W; x++) {
        int i = x >> 1;
        int cur = r0[i] * 3 + r1[i], v;
        if (x & 1) {
          if (i == dw - 1) v = (cur * 4 + 7) >> 4;
          else v = (cur * 3 + (r0[i + 1] * 3 + r1[i + 1]) + 7) >> 4;
        } else {
          if (i == 0) v = (cur * 4 + 8) >> 4;
          else v = (cur * 3 + (r0[i - 1] * 3 + r1[i - 1]) + 8) >> 4;
        }
        o[x] = (uint8_t)v;
      }
    }
    return;
  }
  if (fancy && hexp == 1 && vexp == 2) {                    /* h1v2 fancy (libjpeg-turbo >= 2.0) */
    for (int y = 0; y < H; y++) {
      int i0 = y >> 1;
      int i1 = (y & 1) ? i0 + 1 : i0 - 1;
      if (i1 < 0) i1 = 0;
      if (i1 > dh - 1) i1 = dh - 1;
      int bias = (y & 1) ? 2 : 1;
      const uint8_t *r0 = pl + (size_t)i0 * pw, *r1 = pl + (size_t)i1 * pw;
      uint8_t *o = out + (size_t)y * W;
      for (int x = 0; x < W; x++) o[x] = (uint8_t)((r0[x] * 3 + r1[x] + bias) >> 2);
    }
    return;
  }
  /* box replication (libjpeg int_upsample / h2v1_upsample / h2v2_upsample) */
  for (int y = 0; y < H; y++) {
    const uint8_t *r = pl + (size_t)(y / vexp) * pw;
    uint8_t *o = out + (size_t)y * W;
    for (int x = 0; x < W; x++) o[x] = r[x / hexp];
  }
}

#define FIXC(x) ((int)((x) * 65536.0 + 0.5))
static inline void jo_ycc_rgb(int y, int cb, int cr, uint8_t *rgb) {
  cb -= 128; cr -= 128;
  int r = y + ((FIXC(1.40200) * cr + 32768) >> 16);
  int g = y + ((-FIXC(0.34414) * cb + 32768 - FIXC(0.71414) * cr) >> 16);
  int b = y + ((FIXC(1.77200) * cb + 32768) >> 16);
  rgb[0] = (uint8_t)(r < 0 ? 0 : r > 255 ? 255 : r);
  rgb[1] = (uint8_t)(g < 0 ? 0 : g > 255 ? 255 : g);
  rgb[2] = (uint8_t)(b < 0 ? 0 : b > 255 ? 255 : b);
}

/* ---------------------------------------------------------------- public API */
int jpeg_oracle_info(const uint8_t *data, size_t len, int *out /* [16] */) {
  jo_dec *d = (jo_dec *)calloc(1, sizeof(jo_dec));
  d->data = data; d->len = len;
  int rc = jo_parse(d);
  if (rc == JO_OK) {
    jo_info *in = &d->info;
    out[0] = in->width; out[1] = in->height; out[2] = in->ncomp;
    for (int c = 0; c < 4; c++) { out[3 + c] = in->hs[c]; out[7 + c] = in->vs[c]; }
    out[11] = in->restart_interval; out[12] = in->progressive; out[13] = in->orientation;
    out[14] = in->mcux; out[15] = in->mcuy;
  }
  free(d);
  return rc;
}

/* Quantized coefficients, natural order. coef_out[c] must hold bw[c]*bh[c]*64 int16. */
int jpeg_oracle_coeffs(const uint8_t *data, size_t len, int16_t *c0, int16_t *c1, int16_t *c2) {
  jo_dec *d = (jo_dec *)calloc(1, sizeof(jo_dec));
  d->data = data; d->len = len;
  int rc = jo_parse(d);
  if (rc == JO_OK) {
    int16_t *coef[4] = { c0, c1, c2, NULL };
    if (d->info.ncomp > 3) rc = JO_ERR_UNSUPPORTED;
    else {
      for (int c = 0; c < d->info.ncomp; c++)
        memset(coef[c], 0, (size_t)d->info.bw[c] * d->info.bh[c] * 64 * sizeof(int16_t));
      rc = jo_entropy(d, coef);
    }
  }
  free(d);
  return rc;
}

/* Full decode to interleaved RGB u8 [H][W][3] (gray JPEG -> replicated).
 * fancy != 0 -> libjpeg fancy upsampling (the reference's CPU behaviour). */
int jpeg_oracle_decode_rgb(const uint8_t *data, size_t len, uint8_t *out, int fancy) {
  jo_dec *d = (jo_dec *)calloc(1, sizeof(jo_dec));
  d->data = data; d->len = len;
  int rc = jo_parse(d);
  if (rc != JO_OK) { free(d); return rc; }
  jo_info *in = &d->info;
  if (in->ncomp != 1 && in->ncomp != 3) { free(d); return JO_ERR_UNSUPPORTED; }
  int16_t *coef[4] = {0};
  uint8_t *plane[4] = {0}, *full[4] = {0};
  for (int c = 0; c < in->ncomp; c++) {
    if (!d->qt_present[in->tq[c]]) { rc = JO_ERR_FORMAT; goto done; }
    coef[c] = (int16_t *)calloc((size_t)in->bw[c] * in->bh[c] * 64, sizeof(int16_t));
  }
  rc = jo_entropy(d, coef);
  if (rc != JO_OK) goto done;
  int W = in->width, H = in->height;
  for (int c = 0; c < in->ncomp; c++) {
    int pw = in->bw[c] * 8, ph = in->bh[c] * 8;
    plane[c] = (uint8_t *)malloc((size_t)pw * ph);
    for (int by = 0; by < in->bh[c]; by++)
      for (int bx = 0; bx < in->bw[c]; bx++)
        jo_idct_block(coef[c] + ((size_t)by * in->bw[c] + bx) * 64, d->qt[in->tq[c]],
                      plane[c] + (size_t)by * 8 * pw + bx * 8, pw);
    int hexp = in->hmax / in->hs[c], vexp = in->vmax / in->vs[c];
    if (in->hmax % in->hs[c] || in->vmax % in->vs[c]) { rc = JO_ERR_UNSUPPORTED; goto done; }
    int dw = (W * in->hs[c] + in->hmax - 1) / in->hmax;
    int dh = (H * in->vs[c] + in->vmax - 1) / in->vmax;
    full[c] = (uint8_t *)malloc((size_t)W * H);
    jo_upsample(plane[c], pw, dw, dh, hexp, vexp, fancy, full[c], W, H);
  }
  if (in->ncomp == 1) {
    for (size_t i = 0; i < (size_t)W * H; i++) { out[3 * i] = out[3 * i + 1] = out[3 * i + 2] = full[0][i]; }
  } else {
    int is_rgb = (in->adobe_transform == 0) ||
                 (in->adobe_transform < 0 && !in->jfif && in->cid[0] == 'R' && in->cid[1] == 'G' && in->cid[2] == 'B');
    for (size_t i = 0; i < (size_t)W * H; i++) {
      if (is_rgb) { out[3 * i] = full[0][i]; out[3 * i + 1] = full[1][i]; out[3 * i + 2] = full[2][i]; }
      else jo_ycc_rgb(full[0][i], full[1][i], full[2][i], out + 3 * i);
    }
  }
done:
  for (int c = 0; c < 4; c++) { free(coef[c]); free(plane[c]); free(full[c]); }
  free(d);
  return rc;
}
