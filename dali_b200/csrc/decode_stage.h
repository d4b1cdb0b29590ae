// dali_b200/csrc/decode_stage.h -- the decode stages that dalib200JpegLaunch runs beside its baseline JPEG kernels (host only).
#ifndef DALI_B200_CSRC_DECODE_STAGE_H_
#define DALI_B200_CSRC_DECODE_STAGE_H_
#include <string>
#include <vector>
#include "common.cuh"
#include "jpeg_recon.h"
#include "stream_info.h"

namespace dalib200 {

// What dalib200JpegLaunch hands every stage.
struct StageInputs {
  const JpegImage *images;                   // the batch's records with this launch's output pointers (the decode windows)
  const uint8_t *d_raw;                      // the plan's staged bytes
  int32_t *d_status;
  int16_t *d_coef, *d_dc;                    // coefficient and DC arenas (the progressive stage writes its samples' ranges)
  const uint8_t *d_clean;                    // the clean streams of U1 - U3 and their lengths per JpegUnit (the lossless stage reads them)
  const uint32_t *d_unit_clean_len;
};

// A decode stage beside the baseline JPEG kernels (progressive JPEG, PNG, TIFF, WebP, BMP / PNM, lossless JPEG), for samples whose
// decode is a serial chain per image or needs no JPEG kernel: it runs on a stream of its own, so that its work overlaps the JPEG
// kernels.  It writes only its samples' decode windows (the progressive stage: their coefficient and DC ranges), its scratch and their
// status words.  Its order on the caller's stream s:
//   Run(s)    after the status clear: fork (s -> stage stream); the stage uploads its descriptors and launches its kernels there, then
//             records the join;
//   Join(s)   s waits on the join in front of the first kernel that reads the stage's result (dc_scan for the progressive stage,
//             jpeg_post for the others).
// A stage with no sample in the batch is not touched: no stream is created, no event recorded.
struct SideStage {
  virtual ~SideStage() = default;
  virtual bool Empty() const = 0;            // no sample of the batch is the stage's
  virtual void Clear() = 0;                  // forgets the samples of the last set-up

  bool Create() {
    return cudaEventCreateWithFlags(&fork, cudaEventDisableTiming) == cudaSuccess &&
           cudaEventCreateWithFlags(&join, cudaEventDisableTiming) == cudaSuccess;
  }
  // Waits for the stage's work, then frees its stream, events and arena; a stage with device scratch frees it too.
  virtual void Destroy() {
    if (stream) { cudaStreamSynchronize(stream); cudaStreamDestroy(stream); }
    if (fork) cudaEventDestroy(fork);
    if (join) cudaEventDestroy(join);
    arena.Free();
  }
  int Run(const StageInputs &in, cudaStream_t s) {
    if (Empty()) return DALIB200_SUCCESS;
    int rc;
    if ((rc = Reserve())) return rc;
    if (!stream) DB_CUDA(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    DB_CUDA(cudaEventRecord(fork, s));
    DB_CUDA(cudaStreamWaitEvent(stream, fork, 0));
    if ((rc = Enqueue(in, stream))) return rc;
    DB_CUDA(cudaEventRecord(join, stream));
    return DALIB200_SUCCESS;
  }
  int Join(cudaStream_t s) {
    if (!Empty()) DB_CUDA(cudaStreamWaitEvent(s, join, 0));
    return DALIB200_SUCCESS;
  }

 protected:
  virtual int Reserve() { return DALIB200_SUCCESS; }                  // grows the stage's device scratch for the batch (before the fork)
  virtual int Enqueue(const StageInputs &in, cudaStream_t s) = 0;    // uploads the descriptors and launches the kernels on s
  DescArena arena;

 private:
  cudaStream_t stream = nullptr;             // created at the first launch that has samples for the stage
  cudaEvent_t fork = nullptr, join = nullptr;
};

// The stage of a format with a container of its own (PNG, TIFF, WebP, BMP / PNM): a sample is planned from its stream alone.
struct StreamStage : SideStage {
  // Appends the descriptors of the stream `data` (sample `sample`, whose staged bytes go to `raw_off` of the raw staging area) and
  // fills *info.  Returns a DALIB200 status; *err says why on failure.
  virtual int Plan(const uint8_t *data, size_t len, int sample, int64_t raw_off, StreamInfo *info, std::string *err) = 0;
};

// The decode window and output pointer of every image of a stage, from its sample's JpegImage as patched for this launch (`hi`).
// Returns the pixel total; each image's first_px is its prefix, by which the colour kernel finds the image of a pixel.
template <typename Image>
int64_t FillWindows(std::vector<Image> &images, const JpegImage *hi) {
  int64_t px = 0;
  for (Image &d : images) {
    const JpegImage &im = hi[d.sample];
    d.out = im.out; d.out_type = im.out_type;
    d.win_x0 = im.win_x0; d.win_y0 = im.win_y0; d.win_w = im.win_w; d.win_h = im.win_h;
    d.first_px = px;
    px += (int64_t)im.win_w * im.win_h;
  }
  return px;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_DECODE_STAGE_H_
