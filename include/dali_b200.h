/*
 * include/dali_b200.h -- the thin C-ABI under the reference's operator boundary.
 *
 * Every hot-path kernel family is exposed as   plan create -> plan setup (host, per batch: shapes and
 * per-sample arguments) -> launch (enqueue on a caller stream, no host sync) -> plan destroy.
 * POD arguments only, caller owns every data buffer, the callee owns the plan and its pinned /
 * device descriptor arena.  Non-zero return = error; dalib200GetLastError() returns a thread-local
 * message (conventions follow the reference's C API: include/dali/dali.h:43-164).
 *
 * The reference has no such ABI (its kernels are C++ templates: Setup()/Run(ctx,out,in,args),
 * dali/kernels/kernel.h); each entry point below names the reference interface it replaces.
 * The C++ operators in dali_b200/host (Operator<GPUBackend>::SetupImpl / RunImpl, reference
 * dali/pipeline/operator/operator.h:117-123) call PlanSetup from SetupImpl and Launch from RunImpl.
 */
#ifndef DALI_B200_H_
#define DALI_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st *dalib200Stream_t;   /* == cudaStream_t */

/* Data type ids equal the reference's DALIDataType (include/dali/core/dali_data_type.h:44-57). */
enum { DALIB200_UINT8 = 0, DALIB200_INT16 = 5, DALIB200_INT32 = 6, DALIB200_FLOAT16 = 8, DALIB200_FLOAT = 9 };
/* Image types equal DALIImageType (include/dali/core/common.h:156-162). */
enum { DALIB200_RGB = 0, DALIB200_BGR = 1, DALIB200_GRAY = 2, DALIB200_YCbCr = 3 };
/* Resampling filters equal kernels::ResamplingFilterType (dali/kernels/imgproc/resample/params.h:27-34). */
enum { DALIB200_FILTER_NN = 0, DALIB200_FILTER_LINEAR = 1, DALIB200_FILTER_TRIANGULAR = 2,
       DALIB200_FILTER_GAUSSIAN = 3, DALIB200_FILTER_CUBIC = 4, DALIB200_FILTER_LANCZOS3 = 5 };
enum { DALIB200_LAYOUT_HWC = 0, DALIB200_LAYOUT_CHW = 1 };

enum {
  DALIB200_SUCCESS = 0,
  DALIB200_ERROR_INVALID_ARGUMENT = 1,
  DALIB200_ERROR_UNSUPPORTED = 2,
  DALIB200_ERROR_CUDA = 3,
  DALIB200_ERROR_BAD_DATA = 4,
  DALIB200_ERROR_INTERNAL = 5
};

const char *dalib200GetLastError(void);
int dalib200GetVersion(void);
/* number of kernels this library has launched from the calling process, one per launch (bench.py's gpu_launches) */
uint64_t dalib200GetLaunchCount(void);
/* Per-launch device timing with CUDA events on the launching stream (off by default).  Collect synchronises,
 * returns the records in launch order and clears the log. */
int dalib200ProfilingEnable(int on);
int dalib200ProfilingCollect(char *names, int name_stride, float *ms, int max, int *count);

/* ------------------------------------------------------------------------------------------------
 * Image decode.  JPEG (Huffman + dequant + IDCT + chroma upsampling + YCbCr->RGB): baseline sequential (self-synchronising parallel
 * entropy decode) and progressive (SOF2: scans in dependency waves, one warp per scan; spectral selection + successive approximation).
 * PNG (detected by its signature; IDAT CRCs, inflate + unfilter, colour conversion, bit-exact with cv2.imdecode).
 * TIFF (detected by its header; first IFD, strips or tiles, LZW / Deflate / PackBits / none, one GPU lane per segment, colour
 * conversion, bit-exact with cv2.imdecode; unsupported layouts fail with DALIB200_ERROR_UNSUPPORTED).
 * Lossy WebP (detected by its RIFF header; VP8 key frame: one GPU lane per image for the entropy decode, macroblock-wavefront
 * reconstruction and loop filter, fancy upsampling, bit-exact with cv2.imdecode; lossless and animated WebP fail with
 * DALIB200_ERROR_UNSUPPORTED).  Lossless JPEG (SOF3: precision 2..8, predictors 1..7, 1 or 3 components at 1x1 sampling, restart
 * intervals of whole lines; self-synchronising parallel Huffman decode and a diagonal-wavefront prediction, bit-exact with cv2.imdecode;
 * precision above 8 bits fails with DALIB200_ERROR_UNSUPPORTED).  All formats may be mixed in one batch of a plan.
 * Replaces: imgcodec::ImageDecoder<MixedBackend>::RunImplImpl -> nvimgcodecDecoderDecode
 *           (dali/operators/imgcodec/image_decoder.h:613-882) and ParseSample (:473-499).
 * Host work: marker / table / chunk-header parse only.  Device work: everything arithmetic. */
typedef struct dalib200JpegPlan dalib200JpegPlan;

typedef struct {
  int32_t width, height;        /* decoded image size */
  int32_t components;           /* JPEG: 1, 3 or 4; PNG, TIFF: channels of the file (palette: 3); WebP: 3, 4 with alpha */
  int32_t subsampling;          /* (hmax<<4)|vmax of the luma sampling factors, e.g. 0x22 = 4:2:0 (WebP: always 0x22) */
  int32_t restart_interval;
  int32_t orientation;          /* EXIF orientation, 1 = none */
} dalib200JpegInfo;

/* header-only parse of a JPEG, PNG, TIFF or WebP stream: the analogue of nvimgcodecCodeStreamGetImageInfo (image_decoder.h:482) */
int dalib200JpegGetInfo(const uint8_t *data, size_t len, dalib200JpegInfo *info);

int dalib200JpegPlanCreate(dalib200JpegPlan **plan, int max_batch);
int dalib200JpegPlanDestroy(dalib200JpegPlan *plan);
/* Parses n encoded streams (host pointers) and builds the per-sample descriptors.  The streams are BORROWED until
 * dalib200JpegUpload returns (it packs the entropy-coded segments / IDAT runs into the plan's pinned staging buffer, in groups, and
 * issues the H2D copy of each group as soon as it is packed).  Output shapes via ...GetInfo().
 * fancy_upsampling != 0 selects libjpeg "fancy" (triangle) chroma upsampling -- the reference CPU
 * backend's behaviour; 0 = box replication. */
int dalib200JpegPlanSetup(dalib200JpegPlan *plan, int n, const uint8_t *const *streams, const size_t *lengths,
                          int output_type /* DALIB200_RGB | BGR | GRAY */, int fancy_upsampling);
int dalib200JpegPlanGetInfo(const dalib200JpegPlan *plan, int sample, dalib200JpegInfo *info);
/* Full argument surface of the decoder operators (decoders.image / image_crop / image_random_crop / image_slice):
 *   output_type          DALIB200_RGB | BGR | GRAY | YCbCr   (decoder_schema.cc:21-60; YCbCr = BT.601 of the decoded RGB,
 *                        dali/operators/imgcodec/util/convert.h:150-160)
 *   dtype                DALIB200_UINT8 | DALIB200_FLOAT     (ConvertSatNorm: u8 * (1 / 255), convert.h:118-128)
 *   adjust_orientation   apply the EXIF orientation (image_decoder.h:211,678-679,806)
 *   rois[i]              region of interest of sample i in OUTPUT (oriented) pixel coordinates, [x0, x1) x [y0, y1)
 *                        (imgcodec.h:26-44, image_decoder.h:681-716); only the MCUs (PNG, TIFF: pixels) under the region are
 *                        transformed.
 * The result equals the full decode followed by orientation, crop and conversion, bit for bit. */
typedef struct { int32_t output_type, fancy_upsampling, dtype, adjust_orientation; } dalib200JpegParams;
typedef struct {
  int32_t use_roi, x0, y0, x1, y1;
  int32_t planes_only;        /* skip upsampling + colour conversion for this sample: the caller reads the component planes
                                 (dalib200JpegPlanGetPlanes -> dalib200ResampleLaunchPlanar); 4:2:0 YCbCr JPEG streams only */
} dalib200JpegRoi;
/* The decoder's planar output of a sample: 8-bit planes, Cb / Cr at half resolution (4:2:0), rows padded to a multiple of 16 bytes.
 * Only the MCUs under the sample's region of interest hold data.  crop_x / crop_y: filled by the caller (window the resampler treats
 * as its input image). */
typedef struct {
  const uint8_t *y, *cb, *cr;
  int32_t pitch_y, pitch_c;
  int32_t width, height;
  int32_t crop_x, crop_y;
} dalib200PlanarImage;
/* Alternative to the planes_only flags of SetupEx, for callers that learn only after the setup which samples they can consume as
 * planes: want[i] != 0 asks for sample i, granted[i] tells whether the stream qualifies (3 components, 4:2:0, YCbCr, fancy upsampling,
 * no orientation, RGB u8 request).  Call between JpegPlanSetupEx and JpegUpload. */
int dalib200JpegPlanSetPlanesOnly(dalib200JpegPlan *plan, const uint8_t *want, uint8_t *granted);
/* valid after dalib200JpegLaunch of the batch (the plane arena may grow there) until the next launch */
int dalib200JpegPlanGetPlanes(const dalib200JpegPlan *plan, int sample, dalib200PlanarImage *out);
int dalib200JpegPlanSetupEx(dalib200JpegPlan *plan, int n, const uint8_t *const *streams, const size_t *lengths,
                            const dalib200JpegParams *params, const dalib200JpegRoi *rois_or_null);
/* (H, W, C) of the sample the launch will write (after orientation and region of interest) */
int dalib200JpegPlanGetOutputShape(const dalib200JpegPlan *plan, int sample, int32_t *hwc);
/* Bytes of packed entropy-coded data + tables staged for the batch (the H2D payload). */
size_t dalib200JpegPlanStagedBytes(const dalib200JpegPlan *plan);
/* Pinned staging + H2D copy of the batch (async on stream, host work overlapped with the transfer).  Split from Launch
 * so that a caller can time the device-resident decode separately from the transfer. */
int dalib200JpegUpload(dalib200JpegPlan *plan, dalib200Stream_t stream);
/* stable != 0: the caller guarantees that the encoded streams passed to the next JpegPlanSetup calls stay valid and unmodified
 * until the launch that consumes them has completed -- the contract of the reference's external_source(no_copy=True)
 * (dali/python/nvidia/dali/external_source.py, `no_copy`) and of its readers' own buffers.  JpegUpload then copies samples that
 * live in page-locked memory straight from the caller's buffers (one DMA per sample, no host repack); anything else still goes
 * through the pinned staging buffer.  JpegPlanLastUploadDirect: 0 = staged, 1 = direct (one cudaMemcpyAsync per
 * sample), 2 = direct as one cudaMemcpyBatchAsync submission. */
int dalib200JpegPlanSetSourceStable(dalib200JpegPlan *plan, int stable);
int dalib200JpegPlanLastUploadDirect(const dalib200JpegPlan *plan);
/* Test hook: exhaustive (2^32 inputs) check of the kernels' float -> float16 conversion against the integer restatement of the
 * reference's half_float rounding (include/dali/util/half.hpp, ties away from zero).  *mismatches == 0 on success. */
int dalib200DebugCheckHalfConversion(uint64_t *mismatches);
/* Page-locked host memory for callers that want the direct path (cudaHostAlloc / cudaFreeHost behind the C ABI). */
int dalib200HostAlloc(void **ptr, size_t bytes);
/* The same from a thread whose current device is not the consumer's: allocated with `device` current (no context appears on another
 * GPU as a side effect), page-locked for every context (cudaHostAllocPortable); the thread's current device is restored. */
int dalib200HostAllocOnDevice(void **ptr, size_t bytes, int device);
int dalib200HostFree(void *ptr);
/* Enqueues the decode of the uploaded batch; out_ptrs[i] -> device buffer H*W*C of dtype (HWC, see ...GetOutputShape). */
int dalib200JpegLaunch(dalib200JpegPlan *plan, void *const *out_ptrs, dalib200Stream_t stream);
/* Per-sample device status after a launch (0 ok, 1 = entropy-coded data ended early).  Synchronises. */
int dalib200JpegGetStatus(dalib200JpegPlan *plan, int32_t *status_out);
/* Non-blocking status: ...Async enqueues the D2H copy of the status words on `stream` into the plan's pinned buffer, ...Fetch reads
 * them once the caller has synchronised the stream (the operator does it where the executor waits for the outputs, so a truncated
 * stream raises from Pipeline.run() without an extra synchronisation). */
int dalib200JpegStatusAsync(dalib200JpegPlan *plan, dalib200Stream_t stream);
int dalib200JpegStatusFetch(const dalib200JpegPlan *plan, int32_t *status_out, int n);
/* Test accessor: quantised coefficients of one sample (MCU order, natural order per block).  Synchronises. */
int dalib200JpegDebugGetCoefficients(dalib200JpegPlan *plan, int sample, int16_t *out, size_t count);

/* ------------------------------------------------------------------------------------------------
 * JPEG compression distortion (fn.jpeg_compression_distortion): every RGB u8 image is JPEG-compressed at its quality and decoded
 * again, bit-exact with cv2.imdecode(cv2.imencode(".jpg", img, {IMWRITE_JPEG_QUALITY, quality}), IMREAD_COLOR) (libjpeg-turbo
 * defaults: 4:2:0, islow DCT, the Annex K tables scaled by the quality, fancy upsampling).  No entropy-coded stream is written: the
 * quantised coefficients go straight to the decoder's reconstruct kernels.
 * Replaces: JpegCompressionDistortion (dali/operators/image/distortion/jpeg_compression_distortion_op*.{h,cc}). */
typedef struct dalib200JpegDistortPlan dalib200JpegDistortPlan;
typedef struct { int32_t height, width, quality; } dalib200JpegDistortSample;

int dalib200JpegDistortPlanCreate(dalib200JpegDistortPlan **plan, int max_batch);
int dalib200JpegDistortPlanDestroy(dalib200JpegDistortPlan *plan);
/* quality in [1, 100]; each side in [1, 65500] (libjpeg's limit); otherwise DALIB200_ERROR_INVALID_ARGUMENT */
int dalib200JpegDistortPlanSetup(dalib200JpegDistortPlan *plan, int n, const dalib200JpegDistortSample *samples);
/* in_ptrs[i] / out_ptrs[i]: device HWC RGB u8 [height][width][3]; in and out must not overlap */
int dalib200JpegDistortLaunch(dalib200JpegDistortPlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);
/* Test accessor: the quantised coefficients of one sample after a launch (MCU order Y00 Y01 Y10 Y11 Cb Cr, natural order per block,
 * absolute DC), as the JPEG stream cv2.imencode writes would hold them.  Synchronises. */
int dalib200JpegDistortDebugGetCoefficients(dalib200JpegDistortPlan *plan, int sample, int16_t *out, size_t count);

/* ------------------------------------------------------------------------------------------------
 * Separable resampling (fused two-pass).  Replaces kernels::ResampleGPU / SeparableResamplingGPUImpl::Run
 * (dali/kernels/imgproc/resample/separable_impl.h:110-203) and BatchResamplingSetup::SetupBatch
 * (resampling_setup.cc:347-418); numerics follow the CPU kernel SeparableResampleCPU
 * (separable_cpu.h:124-249) -- the parity target. */
typedef struct dalib200ResamplePlan dalib200ResamplePlan;

typedef struct { int32_t type; int32_t antialias; float radius; } dalib200FilterDesc;

typedef struct {
  int32_t in_h, in_w, channels;
  int32_t out_h, out_w;
  /* index [0] = vertical (y), [1] = horizontal (x): the reference's ResamplingParams2D order */
  int32_t use_roi[2];
  float roi_start[2], roi_end[2];
  dalib200FilterDesc min_filter[2], mag_filter[2];
} dalib200ResampleSample;

int dalib200ResamplePlanCreate(dalib200ResamplePlan **plan, int max_batch);
int dalib200ResamplePlanDestroy(dalib200ResamplePlan *plan);
int dalib200ResamplePlanSetup(dalib200ResamplePlan *plan, int n, const dalib200ResampleSample *samples,
                              int in_dtype /* UINT8 | FLOAT */, int out_dtype /* UINT8 | FLOAT */);
/* in_ptrs[i]: device HWC in_dtype; out_ptrs[i]: device HWC out_dtype [out_h][out_w][channels] */
int dalib200ResampleLaunch(dalib200ResamplePlan *plan, const void *const *in_ptrs, void *const *out_ptrs,
                           dalib200Stream_t stream);
/* Decode -> resize without the RGB image (SURVEY.md 8f rank 1: the reference's fused ROI decode + resize path,
 * image_decoder.h:699-716 + resize.cc): samples whose `planar_ok` is 1 after ...SetupPlanar are resampled straight from the decoder's
 * planes (fancy chroma upsampling + YCbCr->RGB happen inside the resampling kernel, bit-exact with decode-then-resize); sample i of
 * ...LaunchPlanar reads srcs[i] (window crop_x, crop_y, in_w x in_h of the setup) and is skipped when planar_ok[i] == 0. */
int dalib200ResamplePlanSetupPlanar(dalib200ResamplePlan *plan, int n, const dalib200ResampleSample *samples, uint8_t *planar_ok);
int dalib200ResampleLaunchPlanar(dalib200ResamplePlan *plan, const dalib200PlanarImage *srcs, void *const *out_ptrs,
                                 dalib200Stream_t stream);
/* introspection used by the tests: processing order chosen for a sample (0 = horizontal pass first) */
int dalib200ResamplePlanGetOrder(const dalib200ResamplePlan *plan, int sample);
/* 1 when the sample went through the streaming (TMA ring) kernel in the last launch, 0 = tile kernel, -1 = bad index. */
int dalib200ResamplePlanGetPath(const dalib200ResamplePlan *plan, int sample);
/* The streaming kernel's view of a sample after set-up (read-only): info[0] = 1 when the sample is eligible (the 16-byte alignment of its
 * input is checked at launch), info[1] = accumulator slots W of its row walk (0: no walk), info[2] = the most source rows one chunk of 8
 * output rows walks (the sample streams only up to 96), info[3] = its work items (column strips x 56-row segments). */
int dalib200ResamplePlanGetStreamInfo(const dalib200ResamplePlan *plan, int sample, int32_t info[4]);

/* ------------------------------------------------------------------------------------------------
 * Separable resampling of volumes (DHWC), three passes.  Replaces the spatial_ndim = 3 instances of kernels::ResampleGPU /
 * SeparableResamplingGPUImpl (dali/kernels/imgproc/resample/separable_impl.h:110-203, resampling_setup.cc:232-337) behind
 * ResizeBase<GPUBackend> (dali/operators/image/resize/resize_base.cc, resize_op_impl_gpu.h); numerics follow
 * SeparableResampleCPU<Out, In, 3> (separable_cpu.h:124-249) -- the parity target. */
typedef struct dalib200Resample3DPlan dalib200Resample3DPlan;

typedef struct {
  /* index [0] = depth (z), [1] = height (y), [2] = width (x): shape order = the reference's ResamplingParams3D order */
  int32_t in_shape[3], channels;
  int32_t out_shape[3];
  int32_t use_roi[3];
  float roi_start[3], roi_end[3];
  dalib200FilterDesc min_filter[3], mag_filter[3];
} dalib200Resample3DSample;

int dalib200Resample3DPlanCreate(dalib200Resample3DPlan **plan, int max_batch);
int dalib200Resample3DPlanDestroy(dalib200Resample3DPlan *plan);
int dalib200Resample3DPlanSetup(dalib200Resample3DPlan *plan, int n, const dalib200Resample3DSample *samples,
                                int in_dtype /* UINT8 | FLOAT */, int out_dtype /* UINT8 | FLOAT */);
/* in_ptrs[i]: device DHWC in_dtype; out_ptrs[i]: device DHWC out_dtype [out_shape][channels] */
int dalib200Resample3DLaunch(dalib200Resample3DPlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);
/* introspection used by the tests: the pass order chosen for a sample, axes numbered 0 = x (width), 1 = y, 2 = z (depth) */
int dalib200Resample3DPlanGetOrder(const dalib200Resample3DPlan *plan, int sample, int32_t order[3]);

/* ------------------------------------------------------------------------------------------------
 * CropMirrorNormalize.  Replaces kernels::SliceHwc2HwcChwNormalizeGPU::Run
 * (dali/kernels/slice/slice_hwc2chw_normalize_gpu.cu:863-1020) and the generic SliceFlipNormalize kernels;
 * numerics follow SliceFlipNormalizePermutePadCpu (slice_flip_normalize_permute_pad_cpu.h:37-46). */
typedef struct dalib200CmnPlan dalib200CmnPlan;

typedef struct {
  int32_t in_h, in_w, channels;              /* u8 HWC input */
  int32_t anchor_y, anchor_x, crop_h, crop_w;/* window in input coordinates; may leave the image (padding) */
  int32_t mirror;                            /* flip the cropped window horizontally */
  float mean[4], inv_std[4], fill[4];        /* per OUTPUT channel */
} dalib200CmnSample;

int dalib200CmnPlanCreate(dalib200CmnPlan **plan, int max_batch);
int dalib200CmnPlanDestroy(dalib200CmnPlan *plan);
int dalib200CmnPlanSetup(dalib200CmnPlan *plan, int n, const dalib200CmnSample *samples,
                         int out_dtype /* FLOAT | FLOAT16 */, int out_layout /* HWC | CHW */, int out_channels);
int dalib200CmnLaunch(dalib200CmnPlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * WarpAffine.  Replaces kernels::WarpGPU<AffineMapping2D,...> (dali/kernels/imgproc/warp_gpu.h,
 * warp/warp_variable_size_impl.cuh:31-42); numerics follow WarpCPU (warp_cpu.h:143-178) and
 * Sampler (sampler.h:122-330). */
typedef struct dalib200WarpPlan dalib200WarpPlan;

typedef struct {
  int32_t in_h, in_w, channels;
  int32_t out_h, out_w;
  float matrix[6];            /* 2x3 row-major DESTINATION -> SOURCE map (already inverted if needed) */
} dalib200WarpSample;

int dalib200WarpPlanCreate(dalib200WarpPlan **plan, int max_batch);
int dalib200WarpPlanDestroy(dalib200WarpPlan *plan);
int dalib200WarpPlanSetup(dalib200WarpPlan *plan, int n, const dalib200WarpSample *samples,
                          int interp /* NN | LINEAR */, int use_fill, float fill_value,
                          int out_dtype /* UINT8 | FLOAT */);
int dalib200WarpLaunch(dalib200WarpPlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);
/* Kernel taken by the last launch: 1 = band kernel with the source boxes staged by tiled TMA loads through a tensor map (bilinear
 * u8 -> u8 over 3-channel frames of one shape laid out at a constant 16-byte-aligned stride, e.g. the frames of an FHWC batch);
 * 2 = band kernel without a tensor map (bilinear u8 -> u8, 3 channels, any shapes); 0 = generic kernel (NN, float output, other
 * channel counts). */
int dalib200WarpPlanGetPath(const dalib200WarpPlan *plan);
/* host helper: include/dali/core/geom/transform.h:166-174 */
void dalib200AffineInverse(const float *m2x3, float *out2x3);

/* ------------------------------------------------------------------------------------------------
 * Per-pixel 3x3 linear colour transform (Hsv / ColorTwist) and colour-space conversion.
 * Replaces kernels::LinearTransformationGpu (pointwise/linear_transformation_gpu.h:47-79) and
 * ColorSpaceConvKernel (color_manipulation/color_space_conversion_kernel.cuh:139-211). */
typedef struct dalib200PointwisePlan dalib200PointwisePlan;

typedef struct {
  int64_t num_pixels;
  float matrix[9];          /* row-major 3x3 */
  float offset[3];
} dalib200ColorSample;

int dalib200PointwisePlanCreate(dalib200PointwisePlan **plan, int max_batch);
int dalib200PointwisePlanDestroy(dalib200PointwisePlan *plan);
int dalib200LinearTransformSetup(dalib200PointwisePlan *plan, int n, const dalib200ColorSample *samples,
                                 int out_dtype /* UINT8 | FLOAT */);
int dalib200ColorSpaceSetup(dalib200PointwisePlan *plan, int n, const int64_t *num_pixels, int in_type, int out_type);
int dalib200PointwiseLaunch(dalib200PointwisePlan *plan, const void *const *in_ptrs, void *const *out_ptrs,
                            dalib200Stream_t stream);
/* host helper: dali/operators/image/color/color_twist.h:50-83,156-170 */
void dalib200ColorTwistMatrix(float hue, float saturation, float value, float brightness, float contrast,
                              float half_range, float *m3x3, float *offset3);

/* ------------------------------------------------------------------------------------------------
 * Spectrogram (window extraction + FFT + |X|^p) and MelFilterBank.
 * Replaces kernels::signal::fft::StftGPU (dali/kernels/signal/fft/stft_gpu_impl.cu:200-294, cuFFT) and
 * kernels::audio::MelFilterBankGpu (audio/mel_scale/mel_filter_bank_gpu.cu:76-261). */
typedef struct dalib200SpectrogramPlan dalib200SpectrogramPlan;

typedef struct {
  int32_t nfft, window_length, window_step;
  int32_t power;             /* 1 = magnitude, 2 = power */
  int32_t center, reflect;   /* center_windows / reflect_padding */
  int32_t layout_ft;         /* 1: [freq][time] (default "ft"), 0: [time][freq] */
} dalib200SpectrogramArgs;

int dalib200SpectrogramPlanCreate(dalib200SpectrogramPlan **plan, int max_batch);
int dalib200SpectrogramPlanDestroy(dalib200SpectrogramPlan *plan);
/* window_fn: host pointer to window_length floats, or NULL for the reference's Hann window */
int dalib200SpectrogramPlanSetup(dalib200SpectrogramPlan *plan, const dalib200SpectrogramArgs *args,
                                 const float *window_fn, int n, const int64_t *lengths);
int64_t dalib200SpectrogramNumWindows(const dalib200SpectrogramPlan *plan, int sample);
int dalib200SpectrogramLaunch(dalib200SpectrogramPlan *plan, const void *const *in_ptrs, void *const *out_ptrs,
                              dalib200Stream_t stream);
void dalib200HannWindow(float *out, int n);
/* Pre-emphasis applied where the framing reads the signal (PreemphasisFilter -> Spectrogram in one kernel, the filtered signal
 * is never written): every launch then transforms y[t] = x[t] - coeffs[i] * x[t - 1] of the f32 input with the border rule of
 * dalib200PreemphasisSetup, and the spectrogram's padding applies to y.  coeffs: host pointer to one coefficient per sample of
 * the last dalib200SpectrogramPlanSetup, or NULL to switch pre-emphasis off.  dalib200SpectrogramPlanSetup switches it off:
 * call this after it. */
int dalib200SpectrogramPlanSetPreemphasis(dalib200SpectrogramPlan *plan, const float *coeffs, int border);

typedef struct dalib200MelPlan dalib200MelPlan;

typedef struct {
  int32_t nfilter;
  float sample_rate, freq_low, freq_high;
  int32_t htk;               /* mel_formula == "htk" */
  int32_t normalize;
} dalib200MelArgs;

int dalib200MelPlanCreate(dalib200MelPlan **plan, int max_batch);
int dalib200MelPlanDestroy(dalib200MelPlan *plan);
/* input spectrograms are [nbin][nwin[i]] f32 ("ft"); outputs [nfilter][nwin[i]] */
int dalib200MelPlanSetup(dalib200MelPlan *plan, const dalib200MelArgs *args, int nbin, int n, const int64_t *nwin);
/* enable != 0: run the filter bank as one dense GEMM on the tensor cores (mma.sync TF32, 3-term split, FP32 accumulate).
 * Tolerance path (summation order differs from the reference CPU kernel, ~1e-6 relative); the default (0) is the bit-exact
 * banded kernel. */
int dalib200MelPlanSetTensorCores(dalib200MelPlan *plan, int enable);
int dalib200MelLaunch(dalib200MelPlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);
/* Spectrogram -> MelFilterBank in ONE kernel (audio/mel_scale/mel_filter_bank.cc consuming signal/fft/spectrogram.cc): the
 * power spectrum of a frame pair stays in shared memory and only the nfilter x nwin mel output is written.  Available for
 * nfft = 1024 with the (f, t) layout and a mel plan set up for the same batch (dalib200SpectrogramMelSupported returns 1).
 * spec_out_ptrs may be NULL: the spectrogram is then not materialised at all. */
int dalib200SpectrogramMelSupported(const dalib200SpectrogramPlan *plan, const dalib200MelPlan *mel);
int dalib200SpectrogramMelLaunch(dalib200SpectrogramPlan *plan, dalib200MelPlan *mel, const void *const *in_ptrs,
                                 void *const *spec_out_ptrs, void *const *mel_out_ptrs, dalib200Stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Audio tail behind Spectrogram / MelFilterBank: ToDecibels, MFCC (DCT + liftering), Normalize.
 * Replaces kernels::signal::ToDecibelsGpu (dali/kernels/signal/decibel/to_decibels_gpu.cu), kernels::signal::dct::Dct1DGpu
 * (dali/kernels/signal/dct/dct_gpu.cu) + the liftering of dali/operators/audio/mfcc/mfcc.cu, and the 2-D float case of
 * kernels::NormalizeGPU (dali/kernels/normalize/normalize_gpu.cu); numerics follow the CPU kernels
 * (to_decibels_cpu.cc:47-72, dct_cpu.cc:76-115, mfcc.cc:52-72). */
typedef struct dalib200SignalPlan dalib200SignalPlan;
typedef struct {
  float multiplier, reference, cutoff_db;   /* dali/operators/signal/decibel/to_decibels_op.h:38-50 */
  int32_t ref_max;                          /* no `reference` given: the per-sample maximum is the reference */
} dalib200ToDecibelsArgs;
typedef struct { int32_t n_mfcc, dct_type, normalize; float lifter; } dalib200MfccArgs;
typedef struct {
  int32_t mode;                             /* 0: reduce both axes, 1: reduce axis 1 (per row), 2: reduce axis 0 (per column) */
  int32_t ddof;
  float scale, shift, epsilon;
} dalib200NormalizeArgs;

int dalib200SignalPlanCreate(dalib200SignalPlan **plan, int max_batch);
int dalib200SignalPlanDestroy(dalib200SignalPlan *plan);
int dalib200ToDecibelsSetup(dalib200SignalPlan *plan, const dalib200ToDecibelsArgs *args, int n, const int64_t *volumes);
/* shapes: n x 2 = (features, frames); the transform runs along axis 0; outputs are [min(n_mfcc, features)][frames] */
int dalib200MfccSetup(dalib200SignalPlan *plan, const dalib200MfccArgs *args, int n, const int64_t *shapes);
int dalib200SignalOutputRows(const dalib200SignalPlan *plan);
int dalib200NormalizeSetup(dalib200SignalPlan *plan, const dalib200NormalizeArgs *args, int n, const int64_t *shapes);
/* in_ptrs[i] / out_ptrs[i]: device f32 */
int dalib200SignalLaunch(dalib200SignalPlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);

/* AudioResample (dali/operators/audio/resample.{h,cc}, kernel dali/kernels/signal/resampling_cpu.cc): float in, float out, 1..8
 * interleaved channels; in_rate / out_rate as the operator derives them (scale: 1 / scale; out_length: in_length / out_length);
 * out_length = resampled_length() = ceil(in_length * out_rate / in_rate) unless given.  quality 0..100 selects the windowed-sinc
 * width (resampling_params.h).  Launched with dalib200SignalLaunch. */
typedef struct {
  double in_rate, out_rate;
  int64_t in_length, out_length;
  int32_t channels;
} dalib200AudioResampleSample;
int dalib200AudioResampleSetup(dalib200SignalPlan *plan, int n, const dalib200AudioResampleSample *samples, float quality);

/* NonsilentRegion (dali/operators/audio/nonsilence_op.{h,cc}; moving mean square: dali/kernels/signal/moving_mean_square.cc):
 * float input, two int32 scalars per sample (begin, length).  use_reference_power == 0: the reference is the maximum of the
 * moving mean square (the operator's default).  reset_interval: -1 or a multiple of window_length (float inputs: 8192). */
typedef struct {
  float cutoff_db;
  float reference_power;
  int32_t use_reference_power;
} dalib200NonsilentSample;
int dalib200NonsilentSetup(dalib200SignalPlan *plan, int n, const int64_t *lengths, const dalib200NonsilentSample *args,
                           int window_length, int reset_interval);
int dalib200NonsilentLaunch(dalib200SignalPlan *plan, const void *const *in_ptrs, void *const *begin_ptrs,
                            void *const *length_ptrs, dalib200Stream_t stream);

/* PreemphasisFilter (dali/operators/audio/preemphasis_filter_op*): y[t] = x[t] - coeff * x[t - 1] for t >= 1 and
 * y[0] = x[0] - coeff * x_border, x_border = 0 (ZERO), x[0] (CLAMP) or x[1] (REFLECT; x[0] for a one-element signal); the
 * product and the difference are rounded separately (no FMA), coeff == 0 copies.  in_dtype: FLOAT or INT16 (converted to float
 * exactly); the output is f32 of the same length.  coeffs: one per sample.  Launched with dalib200SignalLaunch. */
enum { DALIB200_BORDER_ZERO = 0, DALIB200_BORDER_CLAMP = 1, DALIB200_BORDER_REFLECT = 2 };
int dalib200PreemphasisSetup(dalib200SignalPlan *plan, int n, const int64_t *lengths, const float *coeffs, int border,
                             int in_dtype);

/* ------------------------------------------------------------------------------------------------
 * Small per-pixel / geometry helpers (SURVEY.md 8f rank 4) for interleaved u8 images:
 *   multiply-add   out = ConvertSat<Out>(in * multiplier + addend)   -- brightness_contrast
 *                  (kernels::MultiplyAddGpu, dali/kernels/imgproc/pointwise/multiply_add_gpu.h; CPU numerics multiply_add.h:47-60)
 *   window copy    crop / slice / flip with out-of-bounds fill        -- fn.crop, fn.slice, fn.flip
 *                  (kernels::SliceGPU / SliceFlipNormalizePermutePadGpu, dali/kernels/slice/) */
typedef struct dalib200GenericPlan dalib200GenericPlan;
typedef struct {
  int32_t in_h, in_w, channels;
  int32_t anchor_y, anchor_x, out_h, out_w;   /* window in input coordinates; may leave the image (filled) */
  int32_t flip_x, flip_y;                     /* mirror the window horizontally / vertically */
  uint8_t fill[4];                            /* per channel */
} dalib200WindowSample;
int dalib200GenericPlanCreate(dalib200GenericPlan **plan, int max_batch);
int dalib200GenericPlanDestroy(dalib200GenericPlan *plan);
int dalib200MultiplyAddSetup(dalib200GenericPlan *plan, int n, const int64_t *volumes, const float *multipliers,
                             const float *addends, int out_dtype /* UINT8 | FLOAT */);
int dalib200WindowCopySetup(dalib200GenericPlan *plan, int n, const dalib200WindowSample *samples);
/* Pad (dali/operators/generic/pad*): each sample's data copied to the start of a larger array of the same rank, the rest set to
 * the fill value.  in_shapes / out_shapes: n x ndim extents (out >= in on every axis, ndim 1..6); elem_size 1, 2 or 4 bytes;
 * fill_bytes: elem_size bytes, the fill element as stored in the output. */
int dalib200PadSetup(dalib200GenericPlan *plan, int n, int ndim, int elem_size, const int64_t *in_shapes,
                     const int64_t *out_shapes, const void *fill_bytes);
int dalib200GenericLaunch(dalib200GenericPlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Arithmetic expressions on DataNodes and fn.cast (the reference's ArithmeticGenericOp<GPUBackend>, Cast): one launch per
 * expression and batch, whatever its size.
 *   desc         the reference's prefix description, e.g. "fdiv(sub(&0 $0:float32) &1)": &k = input k, $k:type = constant k of
 *                int_consts (integer and bool types; two's complement bits, read as uint64 for UINT64) or real_consts (float16 /
 *                float32 / float64); cast_<type>(x) = ConvertSat<type>; an identical subexpression written twice is evaluated once
 *   in_types     DALIDataType of every input; in_scalar[k] != 0 (in_scalar may be NULL): input k holds one element per sample, read on
 *                the host at set-up (a CPU per-sample scalar), not a tensor operand
 * Type promotion, operator result types and the integer corner cases are DESIGN.md section 2's.  Limits (checked at compile /
 * set-up, DALIB200_ERROR_INVALID_ARGUMENT with a message): 16 inputs, 16 constants + scalar inputs, 64 instructions, 8 live values,
 * 6 dimensions, 64 levels of nesting; `//` and the bitwise operators refuse float operands.
 * Replaces: dali/operators/math/expressions/arithmetic.{h,cc} (ArithmeticGenericOp) and dali/operators/generic/cast.cc. */
typedef struct dalib200ArithPlan dalib200ArithPlan;
int dalib200ArithPlanCreate(dalib200ArithPlan **plan, int max_batch);
int dalib200ArithPlanDestroy(dalib200ArithPlan *plan);
int dalib200ArithCompile(dalib200ArithPlan *plan, const char *desc, int ninputs, const int32_t *in_types, const uint8_t *in_scalar,
                         const int64_t *int_consts, int nint, const double *real_consts, int nreal, int32_t *out_type);
/* ndims: per input (same for every sample); shapes: n x ninputs x 6 extents (first ndims[k] used); scalars: n x ninputs host
 * pointers, read at this call for the scalar inputs (may be NULL without any).  Output shapes: numpy broadcasting of the tensor
 * inputs (n x 6, *out_ndim used); a shape that does not broadcast fails naming the sample and both shapes. */
int dalib200ArithSetup(dalib200ArithPlan *plan, int n, const int32_t *ndims, const int64_t *shapes, const void *const *scalars,
                       int64_t *out_shapes, int32_t *out_ndim);
/* in_ptrs: n x ninputs device pointers (entries of scalar inputs are ignored); out_ptrs: n device buffers of the output type */
int dalib200ArithLaunch(dalib200ArithPlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * fn.transpose, fn.cat and fn.stack (the reference's Transpose, Cat, Stack): one batched N-D strided copy per operator and batch.
 * Every (sample, input) is one copy of a dense input into its place in the dense output; the planner collapses its dimensions and
 * picks a path from the shape alone (DESIGN.md section 5): whole rows when the run shared by both sides is 64 bytes or more, a
 * shared-memory tile of units between the input's and the output's fastest dimensions otherwise.  Elements of 1, 2, 4 or 8 bytes;
 * outputs of at most 6 dimensions; offsets are 64-bit.  Any byte alignment of the buffers is accepted.
 *   max_copies   samples (transpose) or samples x inputs (join) the plan takes
 *   TransposeSetup   in_shapes: n x ndim; perm: output dimension j is input dimension perm[j] (a permutation of 0..ndim-1);
 *                    out_shapes: n x ndim
 *   JoinSetup        in_shapes: n x ninputs x ndim; new_axis == 0: cat along `axis` in [0, ndim) (shapes equal except along it);
 *                    new_axis != 0: stack along a new axis inserted at `axis` in [0, ndim] (shapes equal);
 *                    out_shapes: n x (ndim + (new_axis != 0))
 * A shape, rank or argument that does not fit fails with DALIB200_ERROR_INVALID_ARGUMENT and a message naming the sample and input.
 * Launch: in_ptrs: n x ninputs device pointers (ninputs = 1 for transpose); out_ptrs: n device buffers. */
typedef struct dalib200PermutePlan dalib200PermutePlan;
int dalib200PermutePlanCreate(dalib200PermutePlan **plan, int max_copies);
int dalib200PermutePlanDestroy(dalib200PermutePlan *plan);
int dalib200TransposeSetup(dalib200PermutePlan *plan, int n, int ndim, int elem_size, const int64_t *in_shapes, const int32_t *perm,
                           int64_t *out_shapes);
int dalib200JoinSetup(dalib200PermutePlan *plan, int n, int ninputs, int ndim, int elem_size, const int64_t *in_shapes, int axis,
                      int new_axis, int64_t *out_shapes);
int dalib200PermuteLaunch(dalib200PermutePlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);
/* the path of every copy of the last setup: 0 rows, 1 tiled, 2 small, -1 nothing to copy (kinds: one entry per copy) */
int dalib200PermutePlanGetPaths(const dalib200PermutePlan *plan, int32_t *kinds, int cap);

/* ------------------------------------------------------------------------------------------------
 * fn.reductions.* (the reference's reductions.Min, Max, Sum, Mean, MeanSquare, RMS, StdDev, Variance): each sample is reduced over
 * a set of its axes on its own.  The planner drops unit axes, merges neighbouring axes of the same kind and reduces one group of
 * reduced axes per pass (at most 3 passes for 6 dimensions), innermost first; each pass is one launch for the batch, plus a combine
 * launch when a sample's reduction is cut into chunks (DESIGN.md section 5).  The order of every accumulation follows from the
 * sample's shape alone, so a result is bit-identical alone or in any batch.  Types and their rules: DESIGN.md section 2.
 *   op            DALIB200_REDUCE_*
 *   in_type       DALIDataType code of the data (the 11 numeric types; BOOL is refused)
 *   out_type      in: the dtype argument, or -1 for the default; out: the output type
 *   in_shapes     n x ndim; axis_mask: bit a set = axis a reduced; keep_dims: reduced axes stay as extent 1
 *   out_shapes    n x (ndim when keep_dims, else ndim minus the reduced axes)
 *   ddof          StdDev / Variance: the divisor is max(1, reduced elements - ddof)
 * A shape, type or argument that does not fit fails with DALIB200_ERROR_INVALID_ARGUMENT and a message naming the sample.
 * Launch: in_ptrs, out_ptrs: n device buffers; mean_ptrs (StdDev / Variance only, else NULL): n device buffers of FLOAT holding the
 * mean of every output element. */
enum {
  DALIB200_REDUCE_MIN = 0, DALIB200_REDUCE_MAX = 1, DALIB200_REDUCE_SUM = 2, DALIB200_REDUCE_MEAN = 3, DALIB200_REDUCE_MEAN_SQUARE = 4,
  DALIB200_REDUCE_RMS = 5, DALIB200_REDUCE_STD_DEV = 6, DALIB200_REDUCE_VARIANCE = 7
};
typedef struct dalib200ReducePlan dalib200ReducePlan;
int dalib200ReducePlanCreate(dalib200ReducePlan **plan, int max_samples);
int dalib200ReducePlanDestroy(dalib200ReducePlan *plan);
int dalib200ReduceSetup(dalib200ReducePlan *plan, int op, int in_type, int32_t *out_type, int n, int ndim, const int64_t *in_shapes,
                        uint32_t axis_mask, int keep_dims, int ddof, int64_t *out_shapes);
int dalib200ReduceLaunch(dalib200ReducePlan *plan, const void *const *in_ptrs, const void *const *mean_ptrs, void *const *out_ptrs,
                         dalib200Stream_t stream);
/* kinds: n x 3, the path of each (sample, pass) of the last setup: 0 columns, 1 inner, 2 split, -1 no such pass; depths (NULL or n):
 * the number of additions on the longest path of each sample's floating-point accumulation tree */
int dalib200ReducePlanGetPaths(const dalib200ReducePlan *plan, int32_t *kinds, int32_t *depths, int cap);

/* ------------------------------------------------------------------------------------------------
 * fn.experimental.equalize (the reference's experimental.Equalize): per-channel histogram equalization of UINT8 images and sequences.
 * Every (sample, frame, channel) plane is mapped through the table cv2.equalizeHist builds from that plane's histogram (DESIGN.md
 * section 2).  Two launches per batch, plus zeroing the histogram scratch: the histogram of every plane, then the tables and the
 * mapping (DESIGN.md section 5).  The histograms are integer, so the output is exact and the same alone or in any batch.
 *   in_type       DALIDataType code of the data: UINT8 only
 *   in_shapes     n x ndim; the output has the input's shape
 *   layout        HW, HWC, CHW, FHW, FHWC or FCHW; "" or NULL: HW, HWC or FHWC by rank (2, 3, 4)
 * At most 16 channels, and at most 2^31 - 1 pixels in one plane.  A type, layout or shape that does not fit fails with
 * DALIB200_ERROR_INVALID_ARGUMENT and a message naming the sample.  Launch: in_ptrs, out_ptrs: n device buffers, any byte offset. */
typedef struct dalib200EqualizePlan dalib200EqualizePlan;
int dalib200EqualizePlanCreate(dalib200EqualizePlan **plan, int max_samples);
int dalib200EqualizePlanDestroy(dalib200EqualizePlan *plan);
int dalib200EqualizeSetup(dalib200EqualizePlan *plan, int in_type, int n, int ndim, const int64_t *in_shapes, const char *layout);
int dalib200EqualizeLaunch(dalib200EqualizePlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * fn.experimental.filter (the reference's experimental.Filter): 2-D correlation of images and sequences with one float32 filter per
 * sample, out[y][x][c] = sum_r sum_s f[r][s] in[y + r - a_r][x + s - a_s][c], channels independent, every frame of a sequence with its
 * sample's filter (DESIGN.md section 2).  One launch per batch (DESIGN.md section 5).  Each output is one float32 fmaf chain in a fixed
 * order (filter rows outer), so it is the same alone or in any batch.
 *   in_type         DALIDataType code of the data: UINT8, INT8, UINT16, INT16, FLOAT16 or FLOAT
 *   out_type        the input's type or FLOAT; -1: the input's type.  ConvertSat: half away from zero, saturating, NaN -> 0
 *   in_shapes       n x ndim; out_shapes (n x ndim) receives the output shapes
 *   layout          HW, HWC, FHW or FHWC; "" or NULL: HW, HWC or FHWC by rank (2, 3, 4)
 *   filter_type / filter_ndim / filter_shapes   FLOAT, 2, n x 2: each extent 1 to 255
 *   anchors         NULL or n x 2 (row, column): -1 for extent / 2, else in [0, extent - 1]; ignored in DALIB200_FILTER_VALID
 *   border, mode    DALIB200_FILTER_BORDER_*, DALIB200_FILTER_SAME / VALID (each spatial extent n - f + 1)
 *   fill_type       -1 without fill values, else the input's type; fill_counts: n, 1 value or (sequences) one per frame; the fill
 *                   value is read only with DALIB200_FILTER_BORDER_CONSTANT (0 without fill values)
 * 1 to 64 channels, at most 2^31 - 1 elements in one frame.  A type, layout, shape or argument that does not fit fails with
 * DALIB200_ERROR_INVALID_ARGUMENT and a message naming the sample.  Launch: in_ptrs, out_ptrs: n device buffers aligned to their
 * element size (else DALIB200_ERROR_INVALID_ARGUMENT); filters, fills: n pointers, in device memory (read in place) when *_on_device, else in host memory (uploaded with the
 * descriptors); fills may be NULL when the set-up had no fill values. */
enum { DALIB200_FILTER_BORDER_REFLECT_101 = 0, DALIB200_FILTER_BORDER_REFLECT_1001 = 1, DALIB200_FILTER_BORDER_WRAP = 2,
       DALIB200_FILTER_BORDER_CLAMP = 3, DALIB200_FILTER_BORDER_CONSTANT = 4 };
enum { DALIB200_FILTER_SAME = 0, DALIB200_FILTER_VALID = 1 };
typedef struct dalib200FilterPlan dalib200FilterPlan;
int dalib200FilterPlanCreate(dalib200FilterPlan **plan, int max_samples);
int dalib200FilterPlanDestroy(dalib200FilterPlan *plan);
int dalib200FilterSetup(dalib200FilterPlan *plan, int in_type, int out_type, int n, int ndim, const int64_t *in_shapes, const char *layout,
                        int filter_type, int filter_ndim, const int64_t *filter_shapes, const int32_t *anchors, int border, int mode,
                        int fill_type, const int64_t *fill_counts, int64_t *out_shapes);
int dalib200FilterLaunch(dalib200FilterPlan *plan, const void *const *in_ptrs, const void *const *filters, int filters_on_device,
                         const void *const *fills, int fills_on_device, void *const *out_ptrs, dalib200Stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * fn.erase: rectangular regions of each sample filled with a value (or one value per channel), every other element copied bit for
 * bit; the output has the input's shape, type and layout (DESIGN.md section 2).  One launch per batch (DESIGN.md section 5).
 *   type            any of the 12 DALIDataType codes
 *   shapes          n x ndim, ndim 1 to 6; layout: ndim distinct characters, or "" / NULL
 *   axis_names      the erased axes as layout characters (needs a layout), or NULL to take axes: naxes dimension indices
 *   anchors, region_shapes   the region values of all samples back to back, anchor_counts / shape_counts of them per sample; a
 *                   sample's two counts are equal and a multiple of the number of erased axes (0: no region), laid out region by
 *                   region in the order of the erased axes
 *   normalized_anchor, normalized_shape   values are fractions of each axis's extent; centered_anchor: the anchor is the centre
 *   fill, nfill     one value, or one per channel of a C axis that is not erased; converted with ConvertSat
 * Per axis, in double precision: a, s scaled if normalised; a -= s / 2 if centred; [llround(a), llround(a + s)) clipped to the
 * extent.  A type, layout, axis, region or fill that does not fit fails with DALIB200_ERROR_INVALID_ARGUMENT and a message naming the
 * sample and the argument.  Launch: in_ptrs, out_ptrs: n device buffers aligned to their element size (else
 * DALIB200_ERROR_INVALID_ARGUMENT); no launch when the batch has no elements. */
typedef struct dalib200ErasePlan dalib200ErasePlan;
int dalib200ErasePlanCreate(dalib200ErasePlan **plan, int max_samples);
int dalib200ErasePlanDestroy(dalib200ErasePlan *plan);
int dalib200EraseSetup(dalib200ErasePlan *plan, int type, int n, int ndim, const int64_t *shapes, const char *layout, const char *axis_names,
                       const int32_t *axes, int naxes, const float *anchors, const int64_t *anchor_counts, const float *region_shapes,
                       const int64_t *shape_counts, int normalized_anchor, int normalized_shape, int centered_anchor, const float *fill,
                       int nfill);
int dalib200EraseLaunch(dalib200ErasePlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * fn.multi_paste and fn.paste: each output built from rectangles of input samples, later rectangles on top of earlier ones, every
 * element no rectangle covers a fill (DESIGN.md section 2).  HWC images only.  One launch per batch (DESIGN.md section 5).
 * Setup (multi_paste):
 *   in_type, out_type   DALIDataType codes; out_type -1: the input's type.  A converting paste applies ConvertSat.
 *   ninputs, n          1 to 64 inputs of n samples each (exactly 1 with in_ids); n outputs
 *   ndims, layouts      per input: the rank (3) and the layout ("HWC", "" or NULL); layouts may be NULL
 *   in_shapes           ninputs x n x (H, W, C), input-major; one channel count across all of them
 *   in_ids, in_id_counts  NULL for the multi-input form (region k of output i is sample i of input k), else in_id_counts[i] sample
 *                       indices per output, back to back
 *   region_args[6], region_counts[6]   in_anchors, in_anchors_rel, shapes, shapes_rel, out_anchors, out_anchors_rel: NULL when not
 *                       given, else region_counts[a][i] values per output ((y, x) per region, 2 K values for K regions), back to back.
 *                       Absolute values are integers; relative ones are llround(value * extent) in double.  Defaults: anchors 0,
 *                       shapes the source extent minus the in-anchor.
 *   output_sizes        NULL (every input sample has one shape, which the outputs take) or n x (H, W)
 *   fill, nfill         the value of uncovered elements: one, or one per channel (multi_paste passes 0)
 *   out_shapes          n x (H, W, C), written
 * CanvasSetup (paste): UINT8 input of n_channels channels; per sample ratio >= 1, paste_x, paste_y in [0, 1], min_canvas_size >= 0;
 *   H' = max(int(ratio * H), int(min_canvas_size)) (float product, truncated), W' the same way; the image at
 *   (int(paste_y * (H' - H)), int(paste_x * (W' - W))); fill: one value per channel, or one for all.
 * A type, layout, shape, region or fill that does not fit fails with DALIB200_ERROR_INVALID_ARGUMENT and a message naming the sample,
 * the region and the argument.  Launch: in_ptrs: ninputs x n device buffers, input-major (only those a region reads must be set),
 * out_ptrs: n; each aligned to its element size (else DALIB200_ERROR_INVALID_ARGUMENT); no launch when the batch has no elements. */
typedef struct dalib200PastePlan dalib200PastePlan;
int dalib200PastePlanCreate(dalib200PastePlan **plan, int max_samples);
int dalib200PastePlanDestroy(dalib200PastePlan *plan);
int dalib200PasteSetup(dalib200PastePlan *plan, int in_type, int out_type, int ninputs, int n, const int *ndims, const char *const *layouts,
                       const int64_t *in_shapes, const int32_t *in_ids, const int64_t *in_id_counts, const double *const *region_args,
                       const int64_t *const *region_counts, const int64_t *output_sizes, const float *fill, int nfill, int64_t *out_shapes);
int dalib200PasteCanvasSetup(dalib200PastePlan *plan, int in_type, int n, int ndim, const char *layout, const int64_t *in_shapes, int n_channels,
                             const float *ratio, const float *paste_x, const float *paste_y, const float *min_canvas_size, const float *fill,
                             int nfill, int64_t *out_shapes);
int dalib200PasteLaunch(dalib200PastePlan *plan, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Audio decode (fn.decoders.audio).  WAV (PCM 8 / 16 / 24 / 32-bit, IEEE float 32, WAVE_FORMAT_EXTENSIBLE with either) and native FLAC
 * (8 / 16 / 24 bits per sample, optional ID3v2 tag in front), detected from the bytes.  The host parses the container and STREAMINFO
 * only; the FLAC frames are found, checked (CRC-8, CRC-16, frame chain) and decoded on the device.  Samples read as libsndfile's
 * sf_readf_float / short / int give them; an optional downmix to mono and a resampling behind it (the AudioResample kernel).
 * Replaces: the reference's CPU AudioDecoder (dali/operators/decoder/audio/audio_decoder_op.cc, libsndfile). */
typedef struct dalib200AudioPlan dalib200AudioPlan;
enum { DALIB200_AUDIO_WAV = 1, DALIB200_AUDIO_FLAC = 2 };
typedef struct {
  int32_t format;               /* DALIB200_AUDIO_WAV | DALIB200_AUDIO_FLAC */
  int32_t sample_rate, channels;
  int32_t bits;                 /* bits per sample (WAV: of the container) */
  int32_t is_float;             /* IEEE float WAV */
  int64_t length;               /* samples per channel */
} dalib200AudioInfo;
/* per-sample decode arguments: out_rate 0 keeps the file's rate; quality 0..100 as AudioResample (one value for the batch's resampled
 * samples); dtype DALIB200_FLOAT | INT16 | INT32 (integer output: no downmix, no resampling, integer sources) */
typedef struct { int32_t downmix; float out_rate; float quality; int32_t dtype; } dalib200AudioParams;

/* header-only parse of one stream; DALIB200_ERROR_UNSUPPORTED / BAD_DATA as at plan set-up */
int dalib200AudioGetInfo(const uint8_t *data, size_t len, dalib200AudioInfo *info);
int dalib200AudioPlanCreate(dalib200AudioPlan **plan, int max_batch);
int dalib200AudioPlanDestroy(dalib200AudioPlan *plan);
/* Parses n streams (host pointers, BORROWED until dalib200AudioLaunch returns) and plans the batch.  A refused stream fails the call
 * with its code and a message naming the sample. */
int dalib200AudioPlanSetup(dalib200AudioPlan *plan, int n, const uint8_t *const *streams, const size_t *lengths,
                           const dalib200AudioParams *params);
/* shape of sample i's audio output: shape[0] = T, shape[1] = C; *ndim = 1 with downmix ([T]), 2 otherwise ([T, C]);
 * *rate: the sample_rate output (the target rate when resampling, else the file's) */
int dalib200AudioPlanGetOutputShape(const dalib200AudioPlan *plan, int sample, int64_t *shape, int32_t *ndim, float *rate);
/* out_ptrs[i]: device buffer of the shape above in the sample's dtype; rate_ptrs[i]: device float scalar */
int dalib200AudioLaunch(dalib200AudioPlan *plan, void *const *out_ptrs, void *const *rate_ptrs, dalib200Stream_t stream);
/* per-sample status of the last launch (0 ok, 1 = the FLAC frame chain is broken or a frame is corrupt): ...Async enqueues the copy,
 * ...Fetch reads it after the caller synchronised the stream */
int dalib200AudioStatusAsync(dalib200AudioPlan *plan, dalib200Stream_t stream);
int dalib200AudioStatusFetch(const dalib200AudioPlan *plan, int32_t *status_out, int n);

#ifdef __cplusplus
}
#endif
#endif  /* DALI_B200_H_ */
