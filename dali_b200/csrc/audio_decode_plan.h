// dali_b200/csrc/audio_decode_plan.h -- host-side container parse of decoders.audio (plain C++, no CUDA types).
//
// Detects the format from the bytes and reads only the container: the RIFF / fmt / data chunks of a WAV file, or the ID3v2 tag, the
// fLaC marker and the metadata blocks of a native FLAC stream (STREAMINFO first, every other block skipped).  The FLAC frames are never
// walked here: the device finds them (audio_decode.cu).  Refusals name DALIB200_ERROR_UNSUPPORTED for streams this decoder does not
// read (other codecs, depths, more than 8 channels, an unknown length) and DALIB200_ERROR_BAD_DATA for malformed headers.
#ifndef DALI_B200_CSRC_AUDIO_DECODE_PLAN_H_
#define DALI_B200_CSRC_AUDIO_DECODE_PLAN_H_

#include <stdint.h>
#include <algorithm>
#include <cstring>
#include <string>
#include "../../include/dali_b200.h"

namespace dalib200 {

enum { kAudioWav = 1, kAudioFlac = 2 };

struct AudioStream {
  int format = 0;                  // kAudioWav | kAudioFlac
  int channels = 0, bits = 0;      // bits: container bits of a WAV sample, bits per sample of FLAC
  int is_float = 0;                // WAV IEEE float (32-bit)
  int rate = 0;
  int64_t length = 0;              // T: samples per channel
  // the bytes the device reads: the whole frames of the WAV data chunk, or the FLAC audio region behind the metadata
  size_t data_off = 0, data_len = 0;
  int min_block = 0, max_block = 0;  // FLAC STREAMINFO block sizes
};

namespace audio_detail {
inline uint32_t le16(const uint8_t *p) { return p[0] | (uint32_t)p[1] << 8; }
inline uint32_t le32(const uint8_t *p) { return p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
inline uint32_t be24(const uint8_t *p) { return (uint32_t)p[0] << 16 | (uint32_t)p[1] << 8 | p[2]; }

inline int Fail(std::string *err, int code, const char *msg) { if (err) *err = msg; return code; }

inline int ParseWav(const uint8_t *p, size_t n, AudioStream *s, std::string *err) {
  if (n < 12) return Fail(err, DALIB200_ERROR_BAD_DATA, "truncated RIFF header");
  bool have_fmt = false;
  size_t pos = 12;
  for (;;) {
    if (pos + 8 > n) return Fail(err, DALIB200_ERROR_BAD_DATA, have_fmt ? "no data chunk" : "no fmt chunk");
    const uint8_t *c = p + pos;
    const uint64_t size = le32(c + 4);
    const size_t body = pos + 8;
    if (!memcmp(c, "fmt ", 4)) {
      if (size < 16 || body + size > n) return Fail(err, DALIB200_ERROR_BAD_DATA, "truncated fmt chunk");
      const uint8_t *f = p + body;
      int tag = (int)le16(f);
      s->channels = (int)le16(f + 2);
      s->rate = (int)le32(f + 4);
      const int align = (int)le16(f + 12);
      s->bits = (int)le16(f + 14);
      if (tag == 0xFFFE) {                                   // WAVE_FORMAT_EXTENSIBLE: the sub-format GUID names the codec
        static const uint8_t kGuidTail[14] = {0x00, 0x00, 0x00, 0x00, 0x10, 0x00, 0x80, 0x00, 0x00, 0xAA, 0x00, 0x38, 0x9B, 0x71};
        if (size < 40) return Fail(err, DALIB200_ERROR_BAD_DATA, "truncated WAVE_FORMAT_EXTENSIBLE fmt chunk");
        if (memcmp(f + 26, kGuidTail, 14)) return Fail(err, DALIB200_ERROR_UNSUPPORTED, "unknown WAVE_FORMAT_EXTENSIBLE sub-format");
        tag = (int)le16(f + 24);
      }
      if (tag == 1) {
        if (s->bits != 8 && s->bits != 16 && s->bits != 24 && s->bits != 32)
          return Fail(err, DALIB200_ERROR_UNSUPPORTED, "PCM WAV bit depth other than 8, 16, 24 or 32");
        s->is_float = 0;
      } else if (tag == 3) {
        if (s->bits != 32) return Fail(err, DALIB200_ERROR_UNSUPPORTED, "float WAV other than 32-bit");
        s->is_float = 1;
      } else {
        return Fail(err, DALIB200_ERROR_UNSUPPORTED, "WAV codec other than PCM or IEEE float");
      }
      if (s->channels == 0) return Fail(err, DALIB200_ERROR_BAD_DATA, "WAV with 0 channels");
      if (s->channels > 8) return Fail(err, DALIB200_ERROR_UNSUPPORTED, "more than 8 channels");
      if (s->rate == 0) return Fail(err, DALIB200_ERROR_BAD_DATA, "sample rate 0");
      if (align != s->channels * (s->bits / 8)) return Fail(err, DALIB200_ERROR_BAD_DATA, "block_align differs from channels x bytes per sample");
      have_fmt = true;
    } else if (!memcmp(c, "data", 4)) {
      if (!have_fmt) return Fail(err, DALIB200_ERROR_BAD_DATA, "data chunk before the fmt chunk");
      // a data chunk that claims more than the file holds decodes the whole frames present (libsndfile's reading)
      const uint64_t avail = std::min<uint64_t>(size, n - body);
      const uint64_t frame = (uint64_t)s->channels * (s->bits / 8);
      s->length = (int64_t)(avail / frame);
      s->data_off = body;
      s->data_len = (size_t)(s->length * frame);
      return DALIB200_SUCCESS;
    }
    if (size > n - body) return Fail(err, DALIB200_ERROR_BAD_DATA, have_fmt ? "no data chunk" : "truncated chunk");
    pos = body + (size_t)size + (size & 1);                 // odd-sized chunks carry a pad byte
  }
}

inline int ParseFlac(const uint8_t *p, size_t n, size_t pos, AudioStream *s, std::string *err) {
  pos += 4;                                                  // "fLaC"
  bool first = true, last = false;
  while (!last) {
    if (pos + 4 > n) return Fail(err, DALIB200_ERROR_BAD_DATA, "truncated FLAC metadata");
    const int type = p[pos] & 0x7F;
    last = (p[pos] & 0x80) != 0;
    const size_t len = be24(p + pos + 1);
    const size_t body = pos + 4;
    if (len > n - body) return Fail(err, DALIB200_ERROR_BAD_DATA, "truncated FLAC metadata block");
    if (type == 127) return Fail(err, DALIB200_ERROR_BAD_DATA, "invalid FLAC metadata block type");
    if (first != (type == 0)) return Fail(err, DALIB200_ERROR_BAD_DATA, "STREAMINFO missing or not the first metadata block");
    if (type == 0) {
      if (len != 34) return Fail(err, DALIB200_ERROR_BAD_DATA, "STREAMINFO of the wrong length");
      const uint8_t *q = p + body;
      s->min_block = (q[0] << 8) | q[1];
      s->max_block = (q[2] << 8) | q[3];
      s->rate = (int)((uint32_t)q[10] << 12 | (uint32_t)q[11] << 4 | q[12] >> 4);
      s->channels = ((q[12] >> 1) & 7) + 1;
      s->bits = (((q[12] & 1) << 4) | (q[13] >> 4)) + 1;
      s->length = (int64_t)(q[13] & 15) << 32 | (int64_t)q[14] << 24 | (int64_t)q[15] << 16 | (int64_t)q[16] << 8 | q[17];
      if (s->min_block < 16 || s->max_block < s->min_block) return Fail(err, DALIB200_ERROR_BAD_DATA, "STREAMINFO block size below 16");
      if (s->rate == 0) return Fail(err, DALIB200_ERROR_BAD_DATA, "sample rate 0");
      if (s->bits != 8 && s->bits != 16 && s->bits != 24) return Fail(err, DALIB200_ERROR_UNSUPPORTED, "FLAC bits per sample other than 8, 16 or 24");
      if (s->length == 0) return Fail(err, DALIB200_ERROR_UNSUPPORTED, "FLAC with an unknown total sample count");
    }
    first = false;
    pos = body + len;
  }
  s->data_off = pos;
  s->data_len = n - pos;
  return DALIB200_SUCCESS;
}
}  // namespace audio_detail

// Parses the container of one stream.  Returns DALIB200_SUCCESS or a refusal code (with a message in *err).
inline int ParseAudioStream(const uint8_t *p, size_t n, AudioStream *s, std::string *err) {
  using namespace audio_detail;
  *s = AudioStream();
  if (n >= 4 && !memcmp(p, "RIFF", 4) && (n < 12 || !memcmp(p + 8, "WAVE", 4))) {
    s->format = kAudioWav;
    return ParseWav(p, n, s, err);
  }
  size_t pos = 0;
  if (n >= 10 && !memcmp(p, "ID3", 3)) {                       // ID3v2 tag in front of the stream: syncsafe size, optional footer
    if ((p[6] | p[7] | p[8] | p[9]) & 0x80) return Fail(err, DALIB200_ERROR_BAD_DATA, "malformed ID3v2 tag");
    pos = 10 + ((size_t)p[6] << 21 | (size_t)p[7] << 14 | (size_t)p[8] << 7 | p[9]) + ((p[5] & 0x10) ? 10 : 0);
    if (pos > n) return Fail(err, DALIB200_ERROR_BAD_DATA, "truncated ID3v2 tag");
  }
  if (n >= pos + 4 && !memcmp(p + pos, "fLaC", 4)) {
    s->format = kAudioFlac;
    const int rc = ParseFlac(p, n, pos, s, err);
    if (rc) return rc;
  } else if (n >= 4 && !memcmp(p, "OggS", 4)) {
    return Fail(err, DALIB200_ERROR_UNSUPPORTED, "Ogg streams (Vorbis, Opus, Ogg FLAC) are not supported");
  } else {
    return Fail(err, DALIB200_ERROR_UNSUPPORTED, "neither a WAV nor a native FLAC stream");
  }
  return DALIB200_SUCCESS;
}

// Checks every limit that does not depend on the requested output: T * C < 2^31.
inline int CheckAudioLimits(const AudioStream &s, std::string *err) {
  if (s.length * s.channels >= ((int64_t)1 << 31)) return audio_detail::Fail(err, DALIB200_ERROR_UNSUPPORTED, "T x C reaches 2^31 samples");
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_AUDIO_DECODE_PLAN_H_
