// dali_b200/csrc/audio_decode.cu -- decoders.audio: WAV and FLAC decoding, downmix and resampling on the device.
//
// The planner (audio_decode_plan.h) parses the containers on the host; the staged bytes are the WAV frames and the FLAC audio regions,
// uploaded with the descriptors in one copy.  On the caller's stream:
//   flac_sync     one thread per byte of every FLAC audio region: clears the byte's end record and keeps it as a candidate when a frame
//                 header that agrees with STREAMINFO starts there (CRC-8 included)
//   flac_frame    one lane per candidate slot: parses the candidate frame to its end (subframes, residuals, padding, CRC-16) and records
//                 the end at its offset
//   flac_chain    one thread per FLAC stream: from the first byte of the region, each end to the next start; keeps the frames of the
//                 chain or sets the sample's status
//   flac_decode   one lane per kept frame: decodes it into the stream's int32 [T][C] samples
//   audio_convert one thread per output element over the whole batch: reads the WAV bytes or the FLAC samples, converts, downmixes, and
//                 writes the output -- or the float input of the resampler, which then runs as AudioResample does (audio_tail.cu)
// The per-thread bodies are in audio_decode_core.h.
#include "common.cuh"
#include "audio_decode_core.h"
#include "audio_decode_plan.h"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace dalib200 {

__global__ void __launch_bounds__(256) flac_sync_kernel(AudioLaunch a) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < a.flac_bytes; g += step) {
    const int f = last_at_most(a.flac, 0, a.nf - 1, g, [](const FlacDesc &d) { return d.first_byte; });
    flac_sync_at(a.flac[f], f, a.raw, g - a.flac[f].first_byte, a.fend, a.cand, a.ccount,
                 [](uint32_t *p, uint32_t v) { return atomicAdd(p, v); });
  }
}

__global__ void __launch_bounds__(32) flac_frame_kernel(AudioLaunch a, int lanes) {
  if ((int)threadIdx.x >= lanes) return;
  for (int64_t k = (int64_t)blockIdx.x * lanes + threadIdx.x; k < a.cand_slots; k += (int64_t)gridDim.x * lanes) {
    const int f = last_at_most(a.flac, 0, a.nf - 1, k, [](const FlacDesc &d) { return d.cand_base; });
    flac_candidate(a.flac[f], f, a.raw, k - a.flac[f].cand_base, a.cand, a.ccount, a.fend);
  }
}

__global__ void __launch_bounds__(128) flac_chain_kernel(AudioLaunch a) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= a.nf) return;
  if (!flac_chain(a.flac[f], f, a.raw, a.fend, a.ccount, a.frames, a.nframes)) a.status[a.flac[f].sample] = 1;
}

__global__ void __launch_bounds__(32) flac_decode_kernel(AudioLaunch a, int lanes) {
  if ((int)threadIdx.x >= lanes) return;
  for (int64_t k = (int64_t)blockIdx.x * lanes + threadIdx.x; k < a.frame_slots; k += (int64_t)gridDim.x * lanes) {
    const int f = last_at_most(a.flac, 0, a.nf - 1, k, [](const FlacDesc &d) { return d.frame_base; });
    if (!flac_decode(a.flac[f], f, a.raw, k - a.flac[f].frame_base, a.frames, a.nframes, a.pcm)) a.status[a.flac[f].sample] = 1;
  }
}

__global__ void __launch_bounds__(256) audio_convert_kernel(AudioLaunch a) {
  const int64_t g0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g0 < a.n) *a.descs[g0].rate_out = a.descs[g0].rate;
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = g0; e < a.total_elems; e += step) {
    const AudioDesc &d = a.descs[last_at_most(a.descs, 0, a.n - 1, e, [](const AudioDesc &p) { return p.first_elem; })];
    audio_convert(d, a.raw, a.pcm, e - d.first_elem, [](float x, float y) { return mul_rn(x, y); }, [](float x, float y) { return add_rn(x, y); });
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200AudioPlan {
  int max_batch = 0, n = 0, nf = 0;
  std::vector<const uint8_t *> src;                     // borrowed until the launch
  std::vector<AudioStream> streams;
  std::vector<AudioDesc> descs;
  std::vector<FlacDesc> flac;
  std::vector<int64_t> out_len;
  std::vector<int32_t> out_ndim;
  std::vector<int> resampled;                           // batch index of each resampled sample
  std::vector<int64_t> resamp_off;                      // float offset of its input in the resampler scratch
  int64_t raw_bytes = 0, flac_bytes = 0, cand_slots = 0, frame_slots = 0, pcm_elems = 0, resamp_elems = 0, total_elems = 0;
  DescArena arena;                                      // descriptors and staged bytes: one copy per launch
  uint8_t *d_scratch = nullptr; size_t scratch_cap = 0;
  int32_t *h_status = nullptr;                          // pinned, max_batch words
  int32_t *d_status = nullptr;
  dalib200SignalPlan *resampler = nullptr;
};

namespace {
size_t Align16(size_t v) { return (v + 15) & ~(size_t)15; }
}  // namespace

extern "C" {

int dalib200AudioGetInfo(const uint8_t *data, size_t len, dalib200AudioInfo *info) try {
  DB_CHECK_ARG(data && info, "AudioGetInfo: bad arguments");
  AudioStream s;
  std::string err;
  int rc = ParseAudioStream(data, len, &s, &err);
  if (!rc) rc = CheckAudioLimits(s, &err);
  if (rc) { SetLastError("%s", err.c_str()); return rc; }
  info->format = s.format; info->sample_rate = s.rate; info->channels = s.channels; info->bits = s.bits; info->is_float = s.is_float;
  info->length = s.length;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200AudioPlanCreate(dalib200AudioPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "AudioPlanCreate: bad arguments");
  auto *p = new dalib200AudioPlan();
  p->max_batch = max_batch;
  int rc = dalib200SignalPlanCreate(&p->resampler, max_batch);
  if (!rc) { cudaError_t e = cudaMallocHost(reinterpret_cast<void **>(&p->h_status), sizeof(int32_t) * max_batch); if (e) { rc = DALIB200_ERROR_CUDA; SetLastError("cudaMallocHost failed"); } }
  if (rc) { dalib200AudioPlanDestroy(p); return rc; }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200AudioPlanDestroy(dalib200AudioPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  if (p->d_scratch) cudaFree(p->d_scratch);
  if (p->h_status) cudaFreeHost(p->h_status);
  dalib200SignalPlanDestroy(p->resampler);
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200AudioPlanSetup(dalib200AudioPlan *p, int n, const uint8_t *const *streams, const size_t *lengths,
                           const dalib200AudioParams *params) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_batch && (n == 0 || (streams && lengths && params)), "AudioPlanSetup: bad arguments");
  p->n = p->nf = 0;                                     // a set-up that fails leaves an empty batch behind, never a partial one
  p->src.assign(streams, streams + n);
  p->streams.assign(n, AudioStream());
  p->descs.assign(n, AudioDesc());
  p->flac.clear();
  p->out_len.assign(n, 0); p->out_ndim.assign(n, 2);
  p->resampled.clear(); p->resamp_off.clear();
  p->raw_bytes = p->flac_bytes = p->cand_slots = p->frame_slots = p->pcm_elems = p->resamp_elems = p->total_elems = 0;
  std::vector<dalib200AudioResampleSample> rs;
  float quality = -1;
  for (int i = 0; i < n; i++) {
    const dalib200AudioParams &a = params[i];
    AudioStream &s = p->streams[i];
    std::string err;
    DB_CHECK_ARG(a.dtype == DALIB200_FLOAT || a.dtype == DALIB200_INT16 || a.dtype == DALIB200_INT32,
                 "decoders.audio: sample %d: dtype must be FLOAT, INT16 or INT32", i);
    DB_CHECK_ARG(a.out_rate >= 0 && std::isfinite(a.out_rate), "decoders.audio: sample %d: the sample rate must be positive (0: keep)", i);
    int rc = ParseAudioStream(streams[i], lengths[i], &s, &err);
    if (!rc) rc = CheckAudioLimits(s, &err);
    if (!rc && s.data_len >= 0xFFFFFFFFull) { rc = DALIB200_ERROR_UNSUPPORTED; err = "audio data of 4 GiB or more"; }
    if (!rc && a.dtype != DALIB200_FLOAT && (s.is_float || a.downmix || a.out_rate > 0)) {
      rc = DALIB200_ERROR_UNSUPPORTED;
      err = "integer output is available for integer sources without downmix and resampling";
    }
    if (rc) { SetLastError("decoders.audio: sample %d: %s", i, err.c_str()); return rc; }
    AudioDesc &d = p->descs[i];
    memset(&d, 0, sizeof(d));
    d.sample = i; d.format = s.format; d.channels = s.channels; d.bits = s.bits; d.is_float = s.is_float; d.dtype = a.dtype;
    d.out_channels = a.downmix ? 1 : s.channels;
    d.length = s.length;
    d.weight = 1.0f / (float)s.channels;
    d.first_elem = p->total_elems;
    p->total_elems += s.length * d.out_channels;
    const bool resample = a.out_rate > 0 && (double)a.out_rate != (double)s.rate;
    d.rate = a.out_rate > 0 ? a.out_rate : (float)s.rate;
    p->out_ndim[i] = a.downmix ? 1 : 2;
    p->out_len[i] = s.length;
    if (resample) {
      DB_CHECK_ARG(a.quality >= 0 && a.quality <= 100, "``quality`` out of range: %g\nValid range is [0..100].", (double)a.quality);
      DB_CHECK_ARG(quality < 0 || quality == a.quality, "decoders.audio: the resampled samples of a batch share one quality");
      quality = a.quality;
      dalib200AudioResampleSample r;
      r.in_rate = s.rate; r.out_rate = a.out_rate;
      r.in_length = s.length;
      r.out_length = static_cast<int64_t>(std::ceil(s.length * r.out_rate / r.in_rate));   // the AudioResample operator's length
      r.channels = d.out_channels;
      rs.push_back(r);
      p->out_len[i] = r.out_length;
      p->resampled.push_back(i);
      p->resamp_off.push_back(p->resamp_elems);
      p->resamp_elems += (int64_t)Align16(s.length * d.out_channels);
    }
    d.raw_off = p->raw_bytes;
    if (s.format == kAudioFlac) {
      FlacDesc f;
      memset(&f, 0, sizeof(f));
      f.sample = i; f.channels = s.channels; f.bits = s.bits; f.rate = s.rate; f.min_block = s.min_block; f.max_block = s.max_block;
      f.length = s.length;
      f.raw_off = p->raw_bytes; f.raw_len = (int64_t)s.data_len;
      f.first_byte = p->flac_bytes;
      const int64_t fc = flac_frame_cap(s.length, s.min_block, (int64_t)s.data_len, s.channels);
      f.frame_cap = (int32_t)std::min<int64_t>(fc, INT32_MAX / 4);
      f.cand_cap = (int32_t)std::min<int64_t>(flac_cand_cap(fc), INT32_MAX / 4);
      f.cand_base = p->cand_slots; f.frame_base = p->frame_slots;
      f.pcm_off = p->pcm_elems;
      d.pcm_off = p->pcm_elems;
      p->flac_bytes += f.raw_len;
      p->cand_slots += f.cand_cap;
      p->frame_slots += f.frame_cap;
      p->pcm_elems += (int64_t)Align16(s.length * s.channels);
      p->flac.push_back(f);
    }
    p->raw_bytes += (int64_t)Align16(s.data_len);
  }
  if (!rs.empty()) {
    const int rc = dalib200AudioResampleSetup(p->resampler, (int)rs.size(), rs.data(), quality);
    if (rc) return rc;
  }
  p->n = n;
  p->nf = (int)p->flac.size();
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200AudioPlanGetOutputShape(const dalib200AudioPlan *p, int sample, int64_t *shape, int32_t *ndim, float *rate) try {
  DB_CHECK_ARG(p && shape && ndim && rate && sample >= 0 && sample < p->n, "AudioPlanGetOutputShape: bad arguments");
  shape[0] = p->out_len[sample];
  shape[1] = p->descs[sample].out_channels;
  *ndim = p->out_ndim[sample];
  *rate = p->descs[sample].rate;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200AudioLaunch(dalib200AudioPlan *p, void *const *out_ptrs, void *const *rate_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && (p->n == 0 || (out_ptrs && rate_ptrs)), "AudioLaunch: bad arguments");
  if (p->n == 0) return DALIB200_SUCCESS;
  const int n = p->n, nf = p->nf;
  // scratch: status | ccount | nframes | fend | cand | frames | pcm | resampler input
  const size_t o_status = 0, o_ccount = Align16(sizeof(int32_t) * n), o_nframes = o_ccount + Align16(sizeof(uint32_t) * nf);
  const size_t o_fend = o_nframes + Align16(sizeof(uint32_t) * nf);
  const size_t o_cand = o_fend + Align16(sizeof(uint32_t) * p->flac_bytes);
  const size_t o_frames = o_cand + Align16(sizeof(uint32_t) * p->cand_slots);
  const size_t o_pcm = o_frames + Align16(sizeof(FlacFrame) * p->frame_slots);
  const size_t o_res = o_pcm + Align16(sizeof(int32_t) * p->pcm_elems);
  const size_t total = o_res + sizeof(float) * p->resamp_elems;
  int rc = GrowDevice(p->d_scratch, p->scratch_cap, total);
  if (rc) return rc;
  uint8_t *s = p->d_scratch;
  p->d_status = reinterpret_cast<int32_t *>(s + o_status);
  float *res_in = reinterpret_cast<float *>(s + o_res);
  // descriptors and staged bytes, one upload
  const size_t o_descs = 0, o_flac = Align16(sizeof(AudioDesc) * n), o_raw = o_flac + Align16(sizeof(FlacDesc) * std::max(nf, 1));
  uint8_t *h;
  if ((rc = p->arena.Stage(o_raw + p->raw_bytes, &h))) return rc;
  AudioDesc *hd = reinterpret_cast<AudioDesc *>(h + o_descs);
  size_t r = 0;
  for (int i = 0; i < n; i++) {
    hd[i] = p->descs[i];
    hd[i].out = out_ptrs[i];
    hd[i].rate_out = static_cast<float *>(rate_ptrs[i]);
    if (r < p->resampled.size() && p->resampled[r] == i) { hd[i].out = res_in + p->resamp_off[r]; r++; }
    memcpy(h + o_raw + p->descs[i].raw_off, p->src[i] + p->streams[i].data_off, p->streams[i].data_len);
  }
  if (nf) memcpy(h + o_flac, p->flac.data(), sizeof(FlacDesc) * nf);
  if ((rc = p->arena.Upload(o_raw + p->raw_bytes, stream))) return rc;
  DB_CUDA(cudaMemsetAsync(s, 0, o_fend, stream));                 // status, candidate and frame counters
  AudioLaunch a;
  a.descs = reinterpret_cast<const AudioDesc *>(p->arena.dev + o_descs);
  a.flac = reinterpret_cast<const FlacDesc *>(p->arena.dev + o_flac);
  a.raw = p->arena.dev + o_raw;
  a.ccount = reinterpret_cast<uint32_t *>(s + o_ccount);
  a.nframes = reinterpret_cast<uint32_t *>(s + o_nframes);
  a.fend = reinterpret_cast<uint32_t *>(s + o_fend);
  a.cand = reinterpret_cast<uint32_t *>(s + o_cand);
  a.frames = reinterpret_cast<FlacFrame *>(s + o_frames);
  a.pcm = reinterpret_cast<int32_t *>(s + o_pcm);
  a.status = p->d_status;
  a.flac_bytes = p->flac_bytes; a.cand_slots = p->cand_slots; a.frame_slots = p->frame_slots; a.total_elems = p->total_elems;
  a.n = n; a.nf = nf;
  const int sms = NumSMs();
  auto grid_of = [&](int64_t m) { return (int)std::max<int64_t>(1, std::min<int64_t>((m + 255) / 256, (int64_t)sms * 16)); };
  if (nf && p->flac_bytes > 0) {
    Launch("flac_sync", flac_sync_kernel, grid_of(p->flac_bytes), 256, 0, stream, a);
    const SerialLanes g = SerialLaneGeometry((int)std::min<int64_t>(p->cand_slots, INT32_MAX), INT32_MAX);
    Launch("flac_frame", flac_frame_kernel, g.warps, 32, 0, stream, a, g.lanes);
  }
  if (nf) {
    Launch("flac_chain", flac_chain_kernel, (nf + 127) / 128, 128, 0, stream, a);
    const SerialLanes g = SerialLaneGeometry((int)std::min<int64_t>(p->frame_slots, INT32_MAX), INT32_MAX);
    Launch("flac_decode", flac_decode_kernel, g.warps, 32, 0, stream, a, g.lanes);
  }
  Launch("audio_convert", audio_convert_kernel, grid_of(std::max<int64_t>(p->total_elems, n)), 256, 0, stream, a);
  DB_CUDA(cudaGetLastError());
  if (!p->resampled.empty()) {
    std::vector<const void *> in(p->resampled.size());
    std::vector<void *> out(p->resampled.size());
    for (size_t k = 0; k < p->resampled.size(); k++) { in[k] = res_in + p->resamp_off[k]; out[k] = out_ptrs[p->resampled[k]]; }
    if ((rc = dalib200SignalLaunch(p->resampler, in.data(), out.data(), stream))) return rc;
  }
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200AudioStatusAsync(dalib200AudioPlan *p, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->d_status, "AudioStatusAsync: launch the plan first");
  DB_CUDA(cudaMemcpyAsync(p->h_status, p->d_status, sizeof(int32_t) * p->n, cudaMemcpyDeviceToHost, stream));
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200AudioStatusFetch(const dalib200AudioPlan *p, int32_t *status_out, int n) try {
  DB_CHECK_ARG(p && status_out && n >= 0 && n <= p->n, "AudioStatusFetch: bad arguments");
  memcpy(status_out, p->h_status, sizeof(int32_t) * n);
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
