/*
 * tests/jpeg_cmyk_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * The oracle's decode of 4-component (CMYK / YCCK) JPEG.  It includes oracle/jpeg_oracle.c unchanged -- its marker parser, baseline
 * entropy decoder, islow IDCT and fancy / box upsampling already handle four components -- and adds what that file's public entry
 * points leave out: the coefficients of a fourth component, the colour rules of 4-component frames, and cv2's GRAYSCALE output.
 * Built by tests/jpeg_cmyk_oracle.py into a temporary directory; pinned against cv2.imdecode by tests/test_jpeg_cmyk_cpu.py.
 */
#include "jpeg_oracle.c"

/* Quantized coefficients, natural order: coef_out[c] must hold bw[c]*bh[c]*64 int16 for every component of the frame. */
int cmyk_oracle_coeffs(const uint8_t *data, size_t len, int16_t *c0, int16_t *c1, int16_t *c2, int16_t *c3) {
  jo_dec *d = (jo_dec *)calloc(1, sizeof(jo_dec));
  d->data = data; d->len = len;
  int rc = jo_parse(d);
  if (rc == JO_OK) {
    int16_t *coef[4] = { c0, c1, c2, c3 };
    for (int c = 0; c < d->info.ncomp; c++)
      memset(coef[c], 0, (size_t)d->info.bw[c] * d->info.bh[c] * 64 * sizeof(int16_t));
    rc = jo_entropy(d, coef);
  }
  free(d);
  return rc;
}

/* Colour space of the frame (libjpeg default_decompress_parms) */
enum { JO_GRAY, JO_YCC, JO_RGB, JO_CMYK, JO_YCCK };
static int jo_color(const jo_info *in) {
  if (in->ncomp == 1) return JO_GRAY;
  if (in->ncomp == 4) return in->adobe_transform > 0 ? JO_YCCK : JO_CMYK;
  int is_rgb = (in->adobe_transform == 0) ||
               (in->adobe_transform < 0 && !in->jfif && in->cid[0] == 'R' && in->cid[1] == 'G' && in->cid[2] == 'B');
  return is_rgb ? JO_RGB : JO_YCC;
}

/* 4-component frames -> RGB: C, M, Y, K as libjpeg delivers them (YCCK: C = 255 - R of the YCbCr->RGB of components 0..2, ...), then
 * OpenCV's icvCvt_CMYK2BGR, which reads them as inverted (Adobe) samples: R = K - ((255 - C) * K >> 8). */
static void jo_cmyk_rgb(int color, int c0, int c1, int c2, int k, uint8_t *rgb) {
  int cmy[3] = { c0, c1, c2 };
  if (color == JO_YCCK) {
    uint8_t t[3];
    jo_ycc_rgb(c0, c1, c2, t);
    for (int i = 0; i < 3; i++) cmy[i] = 255 - t[i];
  }
  for (int i = 0; i < 3; i++) rgb[i] = (uint8_t)(k - (((255 - cmy[i]) * k) >> 8));
}

/* Full decode.  gray == 0: interleaved RGB u8 [H][W][3] (gray JPEG -> replicated); gray != 0: [H][W] as cv2.IMREAD_GRAYSCALE returns it
 * (the Y plane for YCbCr and 1-component frames, libjpeg's rgb_gray for RGB frames, OpenCV's icvCvt_CMYK2Gray for CMYK / YCCK).
 * fancy != 0 -> libjpeg fancy upsampling (the reference's CPU behaviour). */
int cmyk_oracle_decode(const uint8_t *data, size_t len, uint8_t *out, int fancy, int gray) {
  jo_dec *d = (jo_dec *)calloc(1, sizeof(jo_dec));
  d->data = data; d->len = len;
  int rc = jo_parse(d);
  if (rc != JO_OK) { free(d); return rc; }
  jo_info *in = &d->info;
  if (in->ncomp != 1 && in->ncomp != 3 && in->ncomp != 4) { free(d); return JO_ERR_UNSUPPORTED; }
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
  int color = jo_color(in);
  for (size_t i = 0; i < (size_t)W * H; i++) {
    uint8_t rgb[3];
    if (color == JO_GRAY || (gray && color == JO_YCC)) { rgb[0] = rgb[1] = rgb[2] = full[0][i]; }
    else if (color == JO_RGB) { rgb[0] = full[0][i]; rgb[1] = full[1][i]; rgb[2] = full[2][i]; }
    else if (color == JO_YCC) jo_ycc_rgb(full[0][i], full[1][i], full[2][i], rgb);
    else jo_cmyk_rgb(color, full[0][i], full[1][i], full[2][i], full[3][i], rgb);
    if (!gray) { out[3 * i] = rgb[0]; out[3 * i + 1] = rgb[1]; out[3 * i + 2] = rgb[2]; }
    else if (color == JO_RGB) out[i] = (uint8_t)((rgb[0] * 19595 + rgb[1] * 38470 + rgb[2] * 7471 + 32768) >> 16);
    else if (color >= JO_CMYK) out[i] = (uint8_t)((rgb[2] * 1868 + rgb[1] * 9617 + rgb[0] * 4899 + 8192) >> 14);
    else out[i] = rgb[0];
  }
done:
  for (int c = 0; c < 4; c++) { free(coef[c]); free(plane[c]); free(full[c]); }
  free(d);
  return rc;
}

