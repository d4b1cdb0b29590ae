// tools/emul/audio_decode_emul.cc -- TEST INFRASTRUCTURE.  Runs the WAV / FLAC decode of the product on the host.
//
// The planner (dali_b200/csrc/audio_decode_plan.h) is plain C++ and the kernels of audio_decode.cu are thin wrappers around the
// host/device bodies of audio_decode_core.h.  This file compiles them with the host compiler and runs them the way a launch does, so that
// tests/test_audio_decode_cpu.py can compare the decode with the encoder's samples on a machine without a GPU, and run mutated streams
// under ASan + UBSan.  The staged bytes sit in a heap buffer of exactly their size: any read past them is a sanitizer report.  Every
// pass takes its threads in REVERSE order, so that a result that depended on the order in which the device runs them would show up here.
//   g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC -I/usr/local/cuda/include tools/emul/audio_decode_emul.cc
#include <cstdlib>
#include <string>
#include <vector>
#include "../../dali_b200/csrc/audio_decode_plan.h"
#include "../../dali_b200/csrc/audio_decode_core.h"

using namespace dalib200;

// info: { format, rate, channels, bits, T }.  out ([T][downmix ? 1 : C] of dtype) may be NULL: plan only.  Returns the planner's
// DALIB200 status (non-zero: refused at plan set-up), or -1 when the device stages set the sample's status.
extern "C" int emul_audio_decode(const uint8_t *data, size_t len, int downmix, int dtype, void *out, int64_t *info) {
  AudioStream s;
  std::string err;
  int rc = ParseAudioStream(data, len, &s, &err);
  if (!rc) rc = CheckAudioLimits(s, &err);
  if (!rc && dtype != DALIB200_FLOAT && (s.is_float || downmix)) rc = DALIB200_ERROR_UNSUPPORTED;
  if (rc) return rc;
  info[0] = s.format; info[1] = s.rate; info[2] = s.channels; info[3] = s.bits; info[4] = s.length;
  if (!out) return 0;
  uint8_t *raw = static_cast<uint8_t *>(malloc(s.data_len ? s.data_len : 1));
  memcpy(raw, data + s.data_off, s.data_len);
  AudioDesc d;
  memset(&d, 0, sizeof(d));
  d.format = s.format; d.channels = s.channels; d.bits = s.bits; d.is_float = s.is_float; d.dtype = dtype;
  d.out_channels = downmix ? 1 : s.channels; d.length = s.length; d.weight = 1.0f / (float)s.channels; d.out = out;
  std::vector<int32_t> pcm;
  int status = 0;
  if (s.format == kAudioFlac) {
    FlacDesc f;
    memset(&f, 0, sizeof(f));
    f.channels = s.channels; f.bits = s.bits; f.rate = s.rate; f.min_block = s.min_block; f.max_block = s.max_block; f.length = s.length;
    f.raw_len = (int64_t)s.data_len;
    const int64_t fc = flac_frame_cap(s.length, s.min_block, f.raw_len, s.channels);
    f.frame_cap = (int32_t)fc; f.cand_cap = (int32_t)flac_cand_cap(fc);
    std::vector<uint32_t> fend(s.data_len + 1, 0xA5A5A5A5u), cand(f.cand_cap), ccount(1, 0), nframes(1, 0);
    std::vector<FlacFrame> frames(f.frame_cap);
    pcm.assign((size_t)(s.length * s.channels), (int32_t)0xA5A5A5A5);
    auto add = [](uint32_t *p, uint32_t v) { const uint32_t o = *p; *p = o + v; return o; };
    for (int64_t pos = f.raw_len - 1; pos >= 0; pos--) flac_sync_at(f, 0, raw, pos, fend.data(), cand.data(), ccount.data(), add);
    for (int64_t k = f.cand_cap - 1; k >= 0; k--) flac_candidate(f, 0, raw, k, cand.data(), ccount.data(), fend.data());
    if (!flac_chain(f, 0, raw, fend.data(), ccount.data(), frames.data(), nframes.data())) status = -1;
    for (int64_t k = f.frame_cap - 1; k >= 0; k--)
      if (!flac_decode(f, 0, raw, k, frames.data(), nframes.data(), pcm.data())) status = -1;
    if (status) { free(raw); return status; }
  }
  const int64_t total = s.length * d.out_channels;
  for (int64_t e = total - 1; e >= 0; e--)
    audio_convert(d, raw, pcm.data(), e, [](float x, float y) { return x * y; }, [](float x, float y) { return x + y; });
  free(raw);
  return status;
}
