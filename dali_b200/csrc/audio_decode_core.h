// dali_b200/csrc/audio_decode_core.h -- decoders.audio written once for device and host: the descriptors the kernels of
// audio_decode.cu read, the FLAC frame header and frame parser (RFC 9639 sections 9 - 11), and the per-element conversion.
//
// A FLAC frame is found by its header alone: 15 sync bits, the header fields, a CRC-8 over them.  Nothing indexes the frames, so the
// device tries every byte (flac_header), parses every candidate to its end (flac_frame<false>: subframes, residuals, zero padding,
// CRC-16), walks the chain of real frames from the first byte of the audio region, and decodes only the frames of that chain
// (flac_frame<true>).  A false sync inside frame data can thus never reach the output.
#ifndef DALI_B200_CSRC_AUDIO_DECODE_CORE_H_
#define DALI_B200_CSRC_AUDIO_DECODE_CORE_H_
#include <stdint.h>
#include <cstring>
#include "../../include/dali_b200.h"
#include "host_device.h"

namespace dalib200 {

// One sample of the batch, as audio_convert reads it.
struct AudioDesc {
  int32_t sample;                // batch index
  int32_t format;                // kAudioWav | kAudioFlac (audio_decode_plan.h)
  int32_t channels, bits, is_float;
  int32_t dtype;                 // DALIB200_FLOAT | DALIB200_INT16 | DALIB200_INT32
  int32_t out_channels;          // 1 with downmix, else channels
  int64_t length;                // T
  int64_t first_elem;            // first element of the sample in the flat index space of audio_convert (T * out_channels each)
  int64_t raw_off;               // WAV: byte offset of the data chunk's frames in the staged bytes
  int64_t pcm_off;               // FLAC: int32 offset of the decoded [T][C] samples in the pcm scratch
  void *out;                     // dtype output [T][out_channels], or the float input of the resampler
  float *rate_out;               // the sample's sample_rate output (device float scalar)
  float rate;
  float weight;                  // downmix weight 1 / channels (rounded once, on the host)
};

// One FLAC stream, as the frame kernels read it.  The candidate and frame slots are sized from the plan (stream bytes, T, STREAMINFO
// block sizes), never from a value a frame header carries.
struct FlacDesc {
  int32_t sample, channels, bits, rate;
  int32_t min_block, max_block;
  int64_t length;                // STREAMINFO total samples
  int64_t raw_off, raw_len;      // the audio region in the staged bytes (its offsets index fend too)
  int64_t first_byte;            // first byte of the region in the flat index space of flac_sync
  int64_t cand_base, frame_base; // first candidate / frame slot
  int32_t cand_cap, frame_cap;
  int64_t pcm_off;               // int32 offset of the stream's [T][C] samples in the pcm scratch
};

struct FlacFrame { uint32_t off, nsamp; int64_t start; };

// What the kernels of audio_decode.cu read and write (passed by value).
struct AudioLaunch {
  const AudioDesc *descs;
  const FlacDesc *flac;
  const uint8_t *raw;
  uint32_t *fend, *cand, *ccount, *nframes;
  FlacFrame *frames;
  int32_t *pcm, *status;
  int64_t flac_bytes, cand_slots, frame_slots, total_elems;
  int n, nf;
};

struct FlacHeader {
  int32_t blocksize, assign, variable, len;   // assign: 0..7 independent, 8 left/side, 9 right/side, 10 mid/side; len: header bytes
  uint64_t number;                            // frame number (fixed block size) or first sample number (variable)
};

// Frames the stream may hold: every frame but the last has at least STREAMINFO's minimum block size, and every frame at least 9 + C bytes
// (a 6-byte header, C subframes of at least 9 bits each, the CRC-16), so that a STREAMINFO total alone cannot raise the cap.
DB_HD int64_t flac_frame_cap(int64_t length, int32_t min_block, int64_t raw_len, int32_t channels) {
  const int64_t by_length = (length + min_block - 1) / min_block + 1, by_bytes = raw_len / (8 + channels) + 1;
  return by_length < by_bytes ? by_length : by_bytes;
}
// Candidate headers the parser follows: twice the frames plus a margin for false syncs; more fails the sample.
DB_HD int64_t flac_cand_cap(int64_t frame_cap) { return 2 * frame_cap + 64; }
// Longest frame of `block` samples followed: the header, per channel an LPC-32 subframe header and 5 bytes per sample (a 31-bit escape
// code with its partition overhead stays below that), the CRC-16.  Longer frames are corrupt here.
DB_HD int64_t flac_frame_bound(int32_t channels, int32_t block) { return 18 + (int64_t)channels * (160 + 5 * (int64_t)block); }

DB_HD uint32_t flac_crc8(const uint8_t *p, int n) {       // x^8 + x^2 + x + 1
  uint32_t c = 0;
  for (int i = 0; i < n; i++) {
    c ^= p[i];
    for (int b = 0; b < 8; b++) c = (c & 0x80) ? ((c << 1) ^ 0x07) & 0xFF : (c << 1) & 0xFF;
  }
  return c;
}

DB_HD uint32_t flac_crc16(const uint8_t *p, int64_t n) {  // x^16 + x^15 + x^2 + 1
  uint32_t c = 0;
  for (int64_t i = 0; i < n; i++) {
    c ^= (uint32_t)p[i] << 8;
    for (int b = 0; b < 8; b++) c = (c & 0x8000) ? ((c << 1) ^ 0x8005) & 0xFFFF : (c << 1) & 0xFFFF;
  }
  return c;
}

// Parses the frame header at p (avail bytes readable) and checks it against STREAMINFO: channel count, bits per sample and sample rate
// where the header gives them, block size at most STREAMINFO's maximum.  False for anything else.
DB_HD bool flac_header(const uint8_t *p, int64_t avail, const FlacDesc &d, FlacHeader *h) {
  if (avail < 6 || p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return false;
  const int bs_code = p[2] >> 4, rate_code = p[2] & 15, ch = p[3] >> 4, ss = (p[3] >> 1) & 7;
  if (bs_code == 0 || rate_code == 15 || ch > 10 || ss == 3 || (p[3] & 1)) return false;
  h->variable = p[1] & 1;
  // the coded number: UTF-8-like, 1 to 6 bytes (frame number, 31 bits) or 1 to 7 (sample number, 36 bits)
  int pos = 4;
  const uint32_t x = p[pos++];
  int extra;
  uint64_t v;
  if (x < 0x80) { extra = 0; v = x; }
  else if (x >= 0xC0 && x < 0xE0) { extra = 1; v = x & 0x1F; }
  else if (x >= 0xE0 && x < 0xF0) { extra = 2; v = x & 0x0F; }
  else if (x >= 0xF0 && x < 0xF8) { extra = 3; v = x & 0x07; }
  else if (x >= 0xF8 && x < 0xFC) { extra = 4; v = x & 0x03; }
  else if (x >= 0xFC && x < 0xFE) { extra = 5; v = x & 0x01; }
  else if (x == 0xFE && h->variable) { extra = 6; v = 0; }
  else return false;
  if (avail < pos + extra + 5) return false;
  for (int i = 0; i < extra; i++) {
    const uint32_t c = p[pos++];
    if ((c & 0xC0) != 0x80) return false;
    v = (v << 6) | (c & 0x3F);
  }
  h->number = v;
  int bs;
  if (bs_code == 1) bs = 192;
  else if (bs_code <= 5) bs = 144 << bs_code;
  else if (bs_code == 6) bs = p[pos++] + 1;
  else if (bs_code == 7) { bs = ((p[pos] << 8) | p[pos + 1]) + 1; pos += 2; }
  else bs = 1 << bs_code;
  int32_t rate = 0;
  switch (rate_code) {
    case 1: rate = 88200; break;
    case 2: rate = 176400; break;
    case 3: rate = 192000; break;
    case 4: rate = 8000; break;
    case 5: rate = 16000; break;
    case 6: rate = 22050; break;
    case 7: rate = 24000; break;
    case 8: rate = 32000; break;
    case 9: rate = 44100; break;
    case 10: rate = 48000; break;
    case 11: rate = 96000; break;
    case 12: rate = p[pos++] * 1000; break;
    case 13: rate = (p[pos] << 8) | p[pos + 1]; pos += 2; break;
    case 14: rate = ((p[pos] << 8) | p[pos + 1]) * 10; pos += 2; break;
    default: break;
  }
  if (flac_crc8(p, pos) != p[pos]) return false;
  h->len = pos + 1;
  h->blocksize = bs;
  h->assign = ch;
  const int bits = ss == 1 ? 8 : ss == 2 ? 12 : ss == 4 ? 16 : ss == 5 ? 20 : ss == 6 ? 24 : 32;
  const int nch = ch < 8 ? ch + 1 : 2;
  if (nch != d.channels || (ss != 0 && bits != d.bits) || (rate_code != 0 && rate != d.rate) || bs > d.max_block) return false;
  return true;
}

// MSB-first bit reader over [p, p + end); bytes past the end read as 0 and are caught by past_end() and by the unary reader.
struct FlacBits {
  const uint8_t *p;
  int64_t pos, end;              // next byte to load, end of the readable bytes
  uint64_t cache;                // left-aligned; the bits below the `n` valid ones are 0
  int n;
  DB_HD void init(const uint8_t *q, int64_t start, int64_t e) { p = q; pos = start; end = e; cache = 0; n = 0; }
  DB_HD void refill() {
    while (n <= 56) {
      const uint64_t b = pos < end ? p[pos] : 0u;
      cache |= b << (56 - n);
      n += 8;
      pos++;
    }
  }
  DB_HD int64_t tell() const { return pos * 8 - n; }
  DB_HD bool past_end() const { return tell() > end * 8; }
  DB_HD uint32_t get(int k) {                             // k <= 32
    refill();
    if (k == 0) return 0;
    const uint32_t v = (uint32_t)(cache >> (64 - k));
    cache <<= k;
    n -= k;
    return v;
  }
  DB_HD int32_t sget(int k) {                             // k <= 32 bits, two's complement
    if (k == 0) return 0;
    const uint32_t v = get(k);
    return (int32_t)(v << (32 - k)) >> (32 - k);
  }
  // number of 0 bits before the next 1 (consumed), or -1 past the end
  DB_HD int64_t unary() {
    int64_t q = 0;
    for (;;) {
      refill();
      if (cache) {
#if defined(__CUDA_ARCH__)
        const int z = __clzll((long long)cache);
#else
        const int z = __builtin_clzll(cache);
#endif
        cache <<= z;
        cache <<= 1;
        n -= z + 1;
        return q + z;
      }
      q += n;
      n = 0;
      if (past_end()) return -1;
    }
  }
};

// Subframe samples go to out[t * stride] (write mode).  Returns false on a reserved code, a bad parameter or data past the end.
template <bool kWrite>
DB_HD bool flac_subframe(FlacBits &br, int bs, int sb, int32_t *out, int stride) {
  if (br.get(1)) return false;                               // the zero bit in front of the subframe type
  const uint32_t type = br.get(6);
  int wasted = 0;
  if (br.get(1)) {
    const int64_t z = br.unary();
    if (z < 0 || z + 1 >= sb) return false;
    wasted = (int)z + 1;
    sb -= wasted;
  }
  int order;
  bool lpc = false;
  if (type == 0) {                                           // CONSTANT
    const int32_t v = br.sget(sb);
    if (kWrite) for (int t = 0; t < bs; t++) out[(int64_t)t * stride] = (int32_t)((uint32_t)v << wasted);
    return !br.past_end();
  } else if (type == 1) {                                    // VERBATIM
    for (int t = 0; t < bs; t++) {
      const int32_t v = br.sget(sb);
      if (kWrite) out[(int64_t)t * stride] = (int32_t)((uint32_t)v << wasted);
      if (((t & 255) == 255) && br.past_end()) return false;
    }
    return !br.past_end();
  } else if (type >= 8 && type <= 12) {                      // FIXED, order 0..4
    order = (int)type - 8;
  } else if (type >= 32) {                                   // LPC, order 1..32
    order = (int)type - 31;
    lpc = true;
  } else {
    return false;
  }
  if (order > bs) return false;
  for (int t = 0; t < order; t++) {
    const int32_t v = br.sget(sb);
    if (kWrite) out[(int64_t)t * stride] = v;
  }
  int32_t coef[32];
  int shift = 0;
  if (lpc) {
    const int prec = (int)br.get(4) + 1;
    if (prec == 16) return false;                            // 0b1111 is reserved
    shift = br.sget(5);
    if (shift < 0) return false;                             // a negative shift is not allowed (RFC 9639 section 9.2.6)
    for (int i = 0; i < order; i++) coef[i] = br.sget(prec);
  }
  // residual (RFC 9639 section 9.2.7)
  const uint32_t method = br.get(2);
  if (method > 1) return false;
  const int pbits = method ? 5 : 4;
  const uint32_t escape = method ? 31u : 15u;
  const int porder = (int)br.get(4);
  const int parts = 1 << porder;
  if (bs & (parts - 1)) return false;
  const int psize = bs >> porder;
  if (psize < order) return false;
  int t = order;
  for (int part = 0; part < parts; part++) {
    const int cnt = part == 0 ? psize - order : psize;
    const uint32_t k = br.get(pbits);
    if (k == escape) {
      const int eb = (int)br.get(5);
      for (int i = 0; i < cnt; i++, t++) {
        const int32_t r = br.sget(eb);
        if (kWrite) out[(int64_t)t * stride] = r;
      }
    } else {
      for (int i = 0; i < cnt; i++, t++) {
        const int64_t q = br.unary();
        if (q < 0 || q > (int64_t)(0xFFFFFFFFu >> k)) return false;
        const uint32_t u = ((uint32_t)q << k) | br.get((int)k);
        const int32_t r = (int32_t)(u >> 1) ^ -(int32_t)(u & 1);
        if (kWrite) out[(int64_t)t * stride] = r;
      }
    }
    if (br.past_end()) return false;
  }
  if (kWrite) {
    // restore in place: out[t] holds the residual, out[t - 1 .. t - order] the restored history; 64-bit accumulation
    if (lpc) {
      for (int s = order; s < bs; s++) {
        uint64_t acc = 0;
        for (int i = 0; i < order; i++) acc += (uint64_t)((int64_t)coef[i] * out[(int64_t)(s - 1 - i) * stride]);
        out[(int64_t)s * stride] = (int32_t)(uint32_t)((uint64_t)out[(int64_t)s * stride] + (uint64_t)((int64_t)acc >> shift));
      }
    } else if (order > 0) {
      for (int s = order; s < bs; s++) {
        const int64_t x1 = out[(int64_t)(s - 1) * stride];
        const int64_t x2 = order >= 2 ? out[(int64_t)(s - 2) * stride] : 0;
        const int64_t x3 = order >= 3 ? out[(int64_t)(s - 3) * stride] : 0;
        const int64_t x4 = order >= 4 ? out[(int64_t)(s - 4) * stride] : 0;
        const int64_t pred = order == 1 ? x1 : order == 2 ? 2 * x1 - x2 : order == 3 ? 3 * x1 - 3 * x2 + x3 : 4 * x1 - 6 * x2 + 4 * x3 - x4;
        out[(int64_t)s * stride] = (int32_t)(uint32_t)((uint64_t)out[(int64_t)s * stride] + (uint64_t)pred);
      }
    }
    if (wasted)
      for (int s = 0; s < bs; s++) out[(int64_t)s * stride] = (int32_t)((uint32_t)out[(int64_t)s * stride] << wasted);
  }
  return true;
}

// Parses (kWrite = false) or decodes (kWrite = true) the frame whose header h starts at p, with `avail` bytes readable.  Parse mode
// checks the zero padding and the CRC-16 and returns the frame's length in bytes, 0 when it is not a valid frame.  Decode mode writes
// the decorrelated samples to pcm[t * channels + c] and returns the length, or 0 on an error.
template <bool kWrite>
DB_HD int64_t flac_frame(const uint8_t *p, int64_t avail, const FlacDesc &d, const FlacHeader &h, int32_t *pcm) {
  FlacBits br;
  br.init(p, h.len, avail);
  const int C = d.channels, bs = h.blocksize;
  for (int c = 0; c < C; c++) {
    const bool side = (h.assign == 8 && c == 1) || (h.assign == 9 && c == 0) || (h.assign == 10 && c == 1);
    if (!flac_subframe<kWrite>(br, bs, d.bits + (side ? 1 : 0), pcm + c, C)) return 0;
  }
  const int pad = br.n & 7;                                  // to the byte boundary: zero bits
  if (br.get(pad) != 0) return 0;
  const int64_t body = br.tell() >> 3;
  if (body + 2 > avail) return 0;
  if (!kWrite) {
    if (flac_crc16(p, body) != ((uint32_t)p[body] << 8 | p[body + 1])) return 0;
  } else if (h.assign >= 8) {
    for (int t = 0; t < bs; t++) {
      int32_t *s = pcm + (int64_t)t * 2;
      const int64_t a = s[0], b = s[1];
      if (h.assign == 8) s[1] = (int32_t)(a - b);                          // left, side: right = left - side
      else if (h.assign == 9) s[0] = (int32_t)(a + b);                     // side, right: left = side + right
      else {                                                               // mid, side
        const int64_t mid = (int64_t)((uint64_t)a << 1) | (b & 1);
        s[0] = (int32_t)((mid + b) >> 1);
        s[1] = (int32_t)((mid - b) >> 1);
      }
    }
  }
  return body + 2;
}

// ---- audio_convert: one output element
DB_HD int32_t wav_sample(const uint8_t *q, int bits) {  // q: the sample's bytes, little-endian
  if (bits == 8) return (int32_t)q[0] - 128;
  if (bits == 16) return (int32_t)(int16_t)(uint16_t)(q[0] | q[1] << 8);
  if (bits == 24) return (int32_t)((uint32_t)q[0] << 8 | (uint32_t)q[1] << 16 | (uint32_t)q[2] << 24) >> 8;
  return (int32_t)((uint32_t)q[0] | (uint32_t)q[1] << 8 | (uint32_t)q[2] << 16 | (uint32_t)q[3] << 24);
}

// the source sample (t, c) as libsndfile's float read gives it: x / 2^(b-1) (exact for b <= 24; 32-bit: RN(float(x)) * 2^-31), a float
// WAV sample as stored.  mul: the host / device multiplication without contraction.
template <typename Mul>
DB_HD float audio_float(const AudioDesc &a, const uint8_t *raw, const int32_t *pcm, int64_t t, int c, Mul mul) {
  const int64_t i = t * a.channels + c;
  if (a.format == 2) return mul((float)pcm[a.pcm_off + i], 1.0f / (float)(1u << (a.bits - 1)));
  const uint8_t *q = raw + a.raw_off + i * (a.bits >> 3);
  if (a.is_float) {
    const uint32_t u = (uint32_t)q[0] | (uint32_t)q[1] << 8 | (uint32_t)q[2] << 16 | (uint32_t)q[3] << 24;
    float f;
    memcpy(&f, &u, 4);
    return f;
  }
  return mul((float)wav_sample(q, a.bits), 1.0f / (float)(1u << (a.bits - 1)));
}

// the integer read: x shifted to 16 / 32 bits (left to widen, arithmetic right to narrow)
DB_HD int32_t audio_int(const AudioDesc &a, const uint8_t *raw, const int32_t *pcm, int64_t t, int c, int out_bits) {
  const int64_t i = t * a.channels + c;
  const int32_t x = a.format == 2 ? pcm[a.pcm_off + i] : wav_sample(raw + a.raw_off + i * (a.bits >> 3), a.bits);
  const int s = out_bits - a.bits;
  return s >= 0 ? (int32_t)((uint32_t)x << s) : x >> -s;
}

// Element le of sample a's output.  Downmix: w = 1 / C, sum = x0 * w, then sum = sum + xc * w, every product and sum rounded on its own.
template <typename Mul, typename Add>
DB_HD void audio_convert(const AudioDesc &a, const uint8_t *raw, const int32_t *pcm, int64_t le, Mul mul, Add add) {
  const float w = a.weight;
  const int64_t t = le / a.out_channels;
  const int c = (int)(le - t * a.out_channels);
  if (a.dtype == DALIB200_INT16) {
    static_cast<int16_t *>(a.out)[le] = (int16_t)audio_int(a, raw, pcm, t, c, 16);
  } else if (a.dtype == DALIB200_INT32) {
    static_cast<int32_t *>(a.out)[le] = audio_int(a, raw, pcm, t, c, 32);
  } else if (a.out_channels == a.channels) {
    static_cast<float *>(a.out)[le] = audio_float(a, raw, pcm, t, c, mul);
  } else {
    float sum = mul(audio_float(a, raw, pcm, t, 0, mul), w);
    for (int k = 1; k < a.channels; k++) sum = add(sum, mul(audio_float(a, raw, pcm, t, k, mul), w));
    static_cast<float *>(a.out)[le] = sum;
  }
}

// ---- the per-thread bodies of the FLAC kernels
// flac_sync: byte pos of stream f.  Clears its end record and keeps the offset as a candidate when a header that agrees with STREAMINFO
// starts there.  add: atomic add returning the old value.
template <typename Add>
DB_HD void flac_sync_at(const FlacDesc &d, int f, const uint8_t *raw, int64_t pos, uint32_t *fend, uint32_t *cand, uint32_t *ccount, Add add) {
  fend[d.first_byte + pos] = 0;
  const uint8_t *p = raw + d.raw_off + pos;
  if (pos + 1 >= d.raw_len || p[0] != 0xFF || (p[1] & 0xFE) != 0xF8) return;
  FlacHeader h;
  if (!flac_header(p, d.raw_len - pos, d, &h)) return;
  const uint32_t k = add(ccount + f, 1u);
  if (k < (uint32_t)d.cand_cap) cand[d.cand_base + k] = (uint32_t)pos;
}

// flac_frame (parse): candidate k of stream f.  Records the frame's length at its offset when it parses to a valid CRC-16.
DB_HD void flac_candidate(const FlacDesc &d, int f, const uint8_t *raw, int64_t k, const uint32_t *cand, const uint32_t *ccount,
                             uint32_t *fend) {
  if (k >= (int64_t)ccount[f] || k >= d.cand_cap) return;
  const int64_t pos = cand[d.cand_base + k];
  const uint8_t *p = raw + d.raw_off + pos;
  FlacHeader h;
  if (!flac_header(p, d.raw_len - pos, d, &h)) return;
  const int64_t bound = flac_frame_bound(d.channels, h.blocksize);       // the parse follows no frame past its own block's bound
  const int64_t len = flac_frame<false>(p, d.raw_len - pos < bound ? d.raw_len - pos : bound, d, h, nullptr);
  if (len > 0) fend[d.first_byte + pos] = (uint32_t)len;
}

// flac_chain: stream f from the first byte of its audio region, each frame's end to the next start.  Keeps the frames of the chain and
// returns false when it breaks: too many candidates, a gap, a frame number or sample number out of sequence, a change of blocking
// strategy, more samples than STREAMINFO's total, fewer, or another frame behind the last.
DB_HD bool flac_chain(const FlacDesc &d, int f, const uint8_t *raw, const uint32_t *fend, const uint32_t *ccount, FlacFrame *frames,
                         uint32_t *nframes) {
  nframes[f] = 0;
  if (ccount[f] > (uint32_t)d.cand_cap) return false;
  int64_t pos = 0, total = 0;
  int64_t k = 0;
  int variable = -1, nominal = 0;
  while (total < d.length) {
    if (pos >= d.raw_len) return false;
    const uint32_t len = fend[d.first_byte + pos];
    if (len == 0) return false;
    FlacHeader h;
    if (!flac_header(raw + d.raw_off + pos, d.raw_len - pos, d, &h)) return false;
    if (variable < 0) { variable = h.variable; nominal = h.blocksize; }
    if (h.variable != variable) return false;
    if (variable ? h.number != (uint64_t)total : (h.number != (uint64_t)k || total != k * nominal || h.blocksize > nominal)) return false;
    if (total + h.blocksize > d.length || k >= d.frame_cap) return false;
    frames[d.frame_base + k] = FlacFrame{(uint32_t)pos, (uint32_t)h.blocksize, total};
    k++;
    total += h.blocksize;
    pos += len;
  }
  if (pos < d.raw_len && fend[d.first_byte + pos] != 0) return false;
  nframes[f] = (uint32_t)k;
  return true;
}

// flac_frame (decode): frame slot k of stream f, into the stream's [T][C] samples
DB_HD bool flac_decode(const FlacDesc &d, int f, const uint8_t *raw, int64_t k, const FlacFrame *frames, const uint32_t *nframes,
                          int32_t *pcm) {
  if (k >= (int64_t)nframes[f]) return true;
  const FlacFrame fr = frames[d.frame_base + k];
  const uint8_t *p = raw + d.raw_off + fr.off;
  const int64_t avail = d.raw_len - fr.off;
  FlacHeader h;
  if (!flac_header(p, avail, d, &h)) return false;
  return flac_frame<true>(p, avail, d, h, pcm + d.pcm_off + fr.start * d.channels) > 0;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_AUDIO_DECODE_CORE_H_
