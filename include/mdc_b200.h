/*
 * mdc_b200.h — C ABI of the H100-native frame-preparation library (libmdc_b200.so).
 *
 * The reference (tum-vision/mono_dataset_code) has no FFI/plugin layer: its boundary
 * is the C++ class surface of four headers (SURVEY.md §8b).  This ABI is what those
 * classes are re-implemented on (the headers under include/compat) and what any other host
 * language binds (INTEGRATION.md).  Each entry point names the reference interface it
 * replaces; paths are relative to the reference's src/ directory.
 *
 * Conventions: plain pointers and sizes only; every function returns an int status
 * (MDC_OK = 0) and never throws; mdc_last_error() gives a thread-local message.  The
 * reference's "print + early return + validity flag" error style (SURVEY.md §5) is
 * reproduced by the compat classes on top of these statuses.  There is NO CPU
 * fallback: per-frame work always runs in the sm_90a kernels of this library and
 * fails with MDC_ERR_CUDA when no device is usable.
 */
#ifndef MDC_B200_H
#define MDC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- status codes ---------------------------------------------------------------- */
#define MDC_OK 0
#define MDC_ERR_INVALID_ARG 1   /* null pointer, bad size, wrong pixel count            */
#define MDC_ERR_IO 2            /* file missing / unreadable                            */
#define MDC_ERR_FORMAT 3        /* file present but not in the reference's format       */
#define MDC_ERR_INVALID_OBJECT 4 /* operating on an object the reference would flag !valid */
#define MDC_ERR_CUDA 5          /* CUDA runtime/driver failure (message has the detail) */
#define MDC_ERR_UNSUPPORTED 6

/* ---- per-frame mode flags (DatasetReader::getImage arguments, BenchmarkDatasetReader.h:188) */
#define MDC_RECTIFY 1u          /* rectify                                              */
#define MDC_REMOVE_GAMMA 2u     /* removeGamma     -> unMapImage undoGamma              */
#define MDC_REMOVE_VIGNETTE 4u  /* removeVignette  -> unMapImage undoVignette           */
#define MDC_NAN_OVEREXPOSED 8u  /* nanOverexposed  -> unMapImage killOverexposed        */

/* output-camera modes of camera.txt line 3 (FOVUndistorter.cpp:86-110) */
#define MDC_FOV_CROP (-1)
#define MDC_FOV_FULL (-2)
#define MDC_FOV_EXPLICIT 0

#define MDC_MAX_PYR_LEVELS 8

/* Element type of prepared levels (the out_type of the mdc_*_ex calls).  Every level is computed in fp32 exactly as for
 * MDC_OUT_F32 and converted when it is stored; no level is ever computed from a converted one:
 *   MDC_OUT_F32  float, the getImage result itself
 *   MDC_OUT_F16  IEEE binary16, round to nearest even (__float2half_rn; numpy astype(float16), torch .to(float16)): NaN stays NaN,
 *                a value above 65504 after rounding becomes +-inf
 *   MDC_OUT_U8   uint8 as cv::Mat::convertTo(CV_8U) (saturate_cast<uchar>(float)) does it on x86-64: round half to even, NaN,
 *                +-inf and values outside int32 become 0, anything else is clamped to [0, 255] */
#define MDC_OUT_F32 0
#define MDC_OUT_F16 1
#define MDC_OUT_U8 2

typedef struct mdc_fov mdc_fov;     /* host-side FOV rectifier model  (UndistorterFOV state)          */
typedef struct mdc_photo mdc_photo; /* host-side photometric model    (PhotometricUndistorter state)  */
typedef struct mdc_ctx mdc_ctx;     /* device context: tables resident in HBM + tile plan + streams   */
typedef void* mdc_stream;           /* cudaStream_t (NULL = the context's own stream, synchronous API) */

const char* mdc_last_error(void);
const char* mdc_version(void);

/* =====================================================================================
 * FOV rectifier model — replaces UndistorterFOV's constructor and getters
 * (FOVUndistorter.h:40-83, FOVUndistorter.cpp:48-269).  Tables are built on the HOST in
 * strict IEEE float so they are bit-identical to the reference's (SURVEY.md §7).
 * ===================================================================================== */

/* UndistorterFOV(const char* configFileName), FOVUndistorter.cpp:48.  Always returns an
 * object in *out (like the reference's constructor); status is MDC_OK only if the
 * object is valid.  float_math: 0 = unqualified tan()/sqrt() are the double functions
 * (canonical, SURVEY.md §8c), 1 = the float overloads. */
int mdc_fov_create(const char* camera_txt, mdc_fov** out);
int mdc_fov_create_ex(const char* camera_txt, int float_math, mdc_fov** out);
/* Same model from numbers instead of a file (lines 1-4 of camera.txt). */
int mdc_fov_create_from_params(const float in_calib[5], int in_w, int in_h, int mode,
                               const float out_calib[5], int out_w, int out_h, int float_math,
                               mdc_fov** out);
void mdc_fov_destroy(mdc_fov* f);
int mdc_fov_is_valid(const mdc_fov* f);                              /* isValid(),  FOVUndistorter.h:80 */
int mdc_fov_dims(const mdc_fov* f, int* in_w, int* in_h, int* out_w, int* out_h); /* getInputDims/getOutputDims, :71-78 */
int mdc_fov_get_K(const mdc_fov* f, float k_rect[9], float k_org[9]);/* getK_rect/getK_org (row-major 3x3), :49-56 */
float mdc_fov_omega(const mdc_fov* f);                               /* getOmega(), :57 */
int mdc_fov_original_calibration(const mdc_fov* f, float v[5]);      /* getOriginalCalibration(), :61-70 */
/* distortCoordinates(float*, float*, int), FOVUndistorter.cpp:280-319 (host, in place). */
int mdc_fov_distort_coordinates(const mdc_fov* f, float* x, float* y, int n);
/* The same function on the GPU, in place on DEVICE arrays of n points (n up to 2^63; vignetteCalib calls it with 10^6-point
 * grids per image, main_vignetteCalib.cpp:284).  Bit-identical to the host version: sqrtf and the divisions are IEEE
 * operations, and atanf is a restatement of glibc 2.39's algorithm that matches this platform's libm on every float
 * (csrc/mdc_atanf.h).  `device` = CUDA ordinal the arrays live on, `stream` as for mdc_prepare_batch. */
int mdc_fov_distort_coordinates_device(const mdc_fov* f, float* d_x, float* d_y, size_t n, int device, mdc_stream stream);
/* The restated atanf alone, so that a deployment can check it against ITS libm: out[i] = atanf(in[i]) evaluated on the host
 * (mdc_atanf_host) or on the GPU (mdc_atanf_device, device pointers). */
void mdc_atanf_host(const float* in, float* out, size_t n);
int mdc_atanf_device(const float* d_in, float* d_out, size_t n, int device, mdc_stream stream);
/* remapX / remapY (out_w*out_h floats each; NULL for an invalid object) — private in the
 * reference (FOVUndistorter.h:92-93); exposed for bit-compare and for NCCL broadcast. */
const float* mdc_fov_remap_x(const mdc_fov* f);
const float* mdc_fov_remap_y(const mdc_fov* f);

/* =====================================================================================
 * Photometric model — replaces PhotometricUndistorter's constructor and getters
 * (PhotometricUndistorter.h:40-45, PhotometricUndistorter.cpp:42-157).
 * ===================================================================================== */

/* PhotometricUndistorter(std::string file, std::string vignetteImage, int w, int h).
 * vignette: 8/16-bit greyscale PNG (non-interlaced) or binary PGM.  Always returns an
 * object; status MDC_OK only if both gamma and vignette loaded. */
int mdc_photo_create(const char* pcalib_txt, const char* vignette_image, int w, int h, mdc_photo** out);
/* Same model from arrays: raw 256-entry inverse response (NULL = none) and decoded
 * vignette pixels (depth 8 or 16; NULL = none; rows x cols must equal h x w). */
int mdc_photo_create_from_arrays(const float* ginv_raw256, const void* vignette_pixels, int depth,
                                 int rows, int cols, int w, int h, mdc_photo** out);
void mdc_photo_destroy(mdc_photo* p);
int mdc_photo_valid_gamma(const mdc_photo* p);
int mdc_photo_valid_vignette(const mdc_photo* p);
float* mdc_photo_ginv(mdc_photo* p);            /* getGInv(): NULL if !validGamma, PhotometricUndistorter.h:44 */
float* mdc_photo_g(mdc_photo* p);               /* getG(),    PhotometricUndistorter.h:45 */
const float* mdc_photo_vignette_map(const mdc_photo* p);     /* vignetteMap    (w*h) or NULL */
const float* mdc_photo_vignette_map_inv(const mdc_photo* p); /* vignetteMapInv (w*h) or NULL */

/* =====================================================================================
 * Device context — tables uploaded once, resident in HBM; tile plan + TMA descriptors.
 * One context per GPU (one process per GPU).  fov and/or photo may be NULL/invalid:
 * operations needing the missing half then fail with MDC_ERR_INVALID_OBJECT.
 * Concurrency: one context may be used from several streams, by one host thread at a time
 * (its host caches and pipeline buffers are not locked).  Different contexts, on the same
 * device or not, may be used from different host threads at once, and may be created at
 * the same time.  The responseCalib calls keep their own rule (see below).
 * ===================================================================================== */
int mdc_ctx_create(int device, const mdc_fov* fov, const mdc_photo* photo, mdc_ctx** out);
/* Multi-GPU init: rank 0 builds the host models, broadcasts the four tables over NCCL
 * (the host language's NCCL binding, e.g. torch.distributed) into DEVICE buffers the
 * caller owns, and every rank adopts them here.  Pointers may be NULL for a missing
 * half (d_remap_* NULL = no rectifier; d_ginv / d_vinv NULL = not loaded).  The buffers
 * must outlive the context.
 * Every remap entry (x, y) must lie where undistort reads inside the frame (FOVUndistorter.cpp:347-365):
 *   x < 0 (a black pixel; y may then be anything, NaN included), or
 *   0 <= x < in_w-1 and -1 < y < in_h-1, both finite (-0.0 counts as 0; a y in (-1, 0) truncates to row 0).
 * The tables UndistorterFOV builds always do.  Any other entry (x = in_w-1, y = in_h-1, y = -1, a NaN or infinite x, a NaN y
 * under a valid x) makes the call fail with MDC_ERR_INVALID_ARG before any kernel runs; mdc_last_error() names the first such
 * output pixel and its values.  The check reads the host copy of the tables that the tile plan is built from. */
int mdc_ctx_create_from_device_tables(int device, int in_w, int in_h, int out_w, int out_h,
                                      const float* d_remap_x, const float* d_remap_y,
                                      const float* d_ginv256, const float* d_vinv, mdc_ctx** out);
/* After this call the context frees (cudaFree) the tables it adopted in mdc_ctx_create_from_device_tables. */
int mdc_ctx_take_table_ownership(mdc_ctx* c);
void mdc_ctx_destroy(mdc_ctx* c);
int mdc_ctx_device_tables(const mdc_ctx* c, const float** d_remap_x, const float** d_remap_y,
                          const float** d_ginv256, const float** d_vinv);
/* Pyramid geometry: level l has (out_w >> l) x (out_h >> l) pixels (odd trailing row/column dropped). */
int mdc_ctx_level_dims(const mdc_ctx* c, int level, int* w, int* h);
/* Number of kernel launches issued through this context so far (bench bookkeeping). */
long long mdc_ctx_launch_count(const mdc_ctx* c);
/* Tuning knobs.  use_tma selects how the fused kernel K1 fetches the input taps: -1 = auto (the fastest loader usable for this
 * geometry), or one of MDC_LOADER_*; a loader that cannot describe the geometry / pointer makes the per-frame calls fail with
 * MDC_ERR_UNSUPPORTED (LDG always works).  ctas_per_sm: 0 keeps the default. */
#define MDC_LOADER_LDG 0   /* register-staged global loads into shared memory (any row pitch) */
#define MDC_LOADER_TMA 1   /* cp.async.bulk.tensor boxes into a shared-memory ring (row pitch multiple of 16 bytes) */
#define MDC_LOADER_TEX 2   /* texture gather (tld4) straight from the frames: taps on the TEX pipe, look-ups + stores on the LSU pipe
                              (row pitch multiple of the device's texture pitch alignment; enabled by a bit-exactness self-check
                              against the other loaders when the context is created) */
#define MDC_LOADER_HYBRID 3 /* TMA-staged and texture-gather kernels side by side on every SM, the batch split between them:
                              the LSU pipe and the TEX pipe each carry part of the tap traffic */
int mdc_ctx_configure(mdc_ctx* c, int use_tma, int ctas_per_sm);
/* 1 if `loader` (MDC_LOADER_*) can be used with this context's geometry on this device, else 0. */
int mdc_ctx_loader_usable(const mdc_ctx* c, int loader);
/* The MDC_LOADER_* that use_tma = -1 resolves to for this context. */
int mdc_ctx_auto_loader(const mdc_ctx* c);
/* The same two answers for frames whose rows are row_pitch_bytes apart (mdc_prepare_batch_pitched, and the padded rows that
 * mdc_prepare_batch_host copies to the device); the two calls above answer for tightly packed rows (row_pitch_bytes = in_w).
 * A pitch below in_w or above 2^30 is usable by no loader (and resolves to MDC_LOADER_LDG). */
int mdc_ctx_loader_usable_pitched(const mdc_ctx* c, int loader, size_t row_pitch_bytes);
int mdc_ctx_auto_loader_pitched(const mdc_ctx* c, size_t row_pitch_bytes);

/* -------------------------------------------------------------------------------------
 * Device-resident per-frame operators (all pointers are DEVICE pointers; `stream` is a
 * cudaStream_t, NULL = the context's stream followed by a synchronize).
 * ------------------------------------------------------------------------------------- */

/* PhotometricUndistorter::unMapImage, PhotometricUndistorter.cpp:165-212, batched:
 * in  [n_frames][n] u8, out [n_frames][n] f32; n must equal w*h of the photometric model.
 * flags: MDC_REMOVE_GAMMA | MDC_REMOVE_VIGNETTE | MDC_NAN_OVEREXPOSED (sanitised as in :173-189). */
int mdc_unmap_u8(mdc_ctx* c, const uint8_t* d_in, float* d_out, int n, int n_frames, unsigned flags, mdc_stream stream);

/* UndistorterFOV::undistort<unsigned char> / <float>, FOVUndistorter.cpp:322-370, batched.
 * Pixel-count mismatch leaves the output untouched and returns MDC_ERR_INVALID_ARG (the
 * reference prints and returns, :327-338); an invalid rectifier returns MDC_ERR_INVALID_OBJECT (:325). */
int mdc_undistort_u8(mdc_ctx* c, const uint8_t* d_in, float* d_out, int n_pix_in, int n_pix_out, int n_frames, mdc_stream stream);
int mdc_undistort_f32(mdc_ctx* c, const float* d_in, float* d_out, int n_pix_in, int n_pix_out, int n_frames, mdc_stream stream);

/* DatasetReader::getImage mode switch (BenchmarkDatasetReader.h:210-241) fused into one
 * pass, batched, plus the consumer-side box-filter pyramid (SURVEY.md §8a row P):
 *   d_frames      [n_frames][in_w*in_h] u8
 *   d_out_levels  array of `levels` device pointers; level l: [n_frames][w_l*h_l] f32.
 *                 Level 0 is the getImage result (out_w x out_h if MDC_RECTIFY else in_w x in_h).
 * levels = 1 gives exactly getImage.  This is the hot path (kernel K1).  One host thread may issue calls on one context to
 * several streams at once; each staged K1 launch takes one of 64 work counters in turn, so at most 64 of them may be in flight
 * per context. */
int mdc_prepare_batch(mdc_ctx* c, const uint8_t* d_frames, int n_frames, unsigned flags,
                      float* const* d_out_levels, int levels, mdc_stream stream);
/* Same with padded input rows: d_frames is [n_frames][in_h][row_pitch_bytes] (row_pitch_bytes >= in_w; rectifying mode only).
 * A pitch that is a multiple of 16 bytes keeps image widths that are NOT a multiple of 16 on the TMA loader (a tightly packed odd
 * width can only use the ~2x slower LDG loader); mdc_prepare_batch_host pads such rows itself during its host-to-device copy, in
 * rectifying mode, to the next multiple of 32 bytes (when the context's tile plan can use TMA at all). */
int mdc_prepare_batch_pitched(mdc_ctx* c, const uint8_t* d_frames, size_t row_pitch_bytes, int n_frames, unsigned flags,
                              float* const* d_out_levels, int levels, mdc_stream stream);

/* The same getImage + pyramid with the levels stored as out_type (MDC_OUT_F32 / MDC_OUT_F16 / MDC_OUT_U8): level l of type T is
 * conv_T of what the same call with MDC_OUT_F32 gives, pixel for pixel (see MDC_OUT_*); the conversion happens in the kernels' stores,
 * so the call launches exactly the kernels the fp32 call launches.  d_out_levels[l]: [n_frames][w_l*h_l] elements of out_type.
 * row_pitch_bytes = 0: tightly packed input rows (mdc_prepare_batch), else as mdc_prepare_batch_pitched.  Narrow types keep the levels
 * a K2 pass reads (level 2 when levels > 3; every level but the last in non-rectifying mode) in fp32 scratch that the call takes from a
 * memory pool of the context, stream-ordered on `stream`.  An unknown out_type returns MDC_ERR_INVALID_ARG before anything else is
 * looked at; every other argument rule is that of mdc_prepare_batch(_pitched).  mdc_prepare_batch(_pitched) is this call with
 * MDC_OUT_F32. */
int mdc_prepare_batch_ex(mdc_ctx* c, const uint8_t* d_frames, size_t row_pitch_bytes, int n_frames, unsigned flags, int out_type,
                         void* const* d_out_levels, int levels, mdc_stream stream);

/* Stand-alone pyramid level (kernel K2): dst[x,y] = 0.25f*(((a+b)+c)+d) over the 2x2 block. */
int mdc_pyr_down(mdc_ctx* c, const float* d_src, int src_w, int src_h, float* d_dst, int n_frames, mdc_stream stream);

/* =====================================================================================
 * Sequence reader + decode-ahead feed — the host side of DatasetReader (BenchmarkDatasetReader.h:83-147, :159-186, :247-345)
 * without OpenCV / libzip (SURVEY.md §8f N1).  Frames: 8/16-bit grey PNG, binary PGM and baseline JPEG (grey or colour, read as
 * grey), decoded by this library to the same bytes as cv::imread(..., CV_LOAD_IMAGE_GRAYSCALE).
 * ===================================================================================== */
typedef struct mdc_seq mdc_seq;
/* DatasetReader(folder), :85-140: the sorted entries of <folder>/images/, or, if there are none, of <folder>/images.zip (stored /
 * deflated entries, no zip64); <folder>/times.txt ("id timestamp [exposure]" per line; a count mismatch zeroes all, :322-329).
 * A missing / unreadable archive returns MDC_ERR_IO (the reference calls exit(1), :117-121). */
int mdc_seq_open(const char* folder, mdc_seq** out);
void mdc_seq_close(mdc_seq* s);
int mdc_seq_num_images(const mdc_seq* s);                 /* getNumImages(), :169 */
int mdc_seq_is_zipped(const mdc_seq* s);
const char* mdc_seq_name(const mdc_seq* s, int id);       /* path (folder) or entry name (zip); NULL if out of range */
double mdc_seq_timestamp(const mdc_seq* s, int id);       /* getTimestamp(), :171-177: 0 if out of range */
float mdc_seq_exposure(const mdc_seq* s, int id);         /* getExposure(), :179-186 */
/* getImageRaw_internal(id), :247-276, CV_LOAD_IMAGE_GRAYSCALE semantics: 8-bit grey pixels (a 16-bit PNG keeps its high byte, a
 * colour JPEG gives its luminance component).
 * out may be NULL to query the size only.  MDC_ERR_FORMAT if the frame cannot be decoded. */
int mdc_seq_read_gray8(const mdc_seq* s, int id, uint8_t* out, size_t capacity, int* w, int* h);
/* getImage(id, flags...) for id in [first, first+count) into HOST level buffers (level l: [count][(w>>l)*(h>>l)] floats, as for
 * mdc_prepare_batch_host): `threads` host threads (0 = all) decode the next chunk (two frames per decode thread, 16..256 frames) into
 * pinned memory while the current chunk goes through H2D -> fused kernel -> D2H.  A frame of the wrong size or an undecodable one stops the call with MDC_ERR_FORMAT
 * (the reference prints and returns 0 for that frame, :194-205); the chunks before the one holding that frame are complete, the
 * rows from that chunk on are not written.  first / count outside the sequence, levels outside 1..MDC_MAX_PYR_LEVELS or a NULL
 * level that has pixels (a level without pixels may be NULL) return MDC_ERR_INVALID_ARG before anything is decoded. */
int mdc_seq_prepare(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, float* const* h_out_levels, int levels, int threads);
/* mdc_seq_prepare with the levels stored as out_type (MDC_OUT_*, as for mdc_prepare_batch_ex); h_out_levels[l] holds count*w_l*h_l
 * elements of that type.  An unknown out_type returns MDC_ERR_INVALID_ARG before any other check; everything else as mdc_seq_prepare. */
int mdc_seq_prepare_ex(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, int out_type, void* const* h_out_levels,
                       int levels, int threads);
/* The same getImage for [first, first+count) into DEVICE level buffers (level l: [count][(w>>l)*(h>>l)] floats), with the JPEG frames
 * decoded on the GPU: `threads` host threads (0 = all) read the files, parse the JPEG headers and split the scans into restart intervals,
 * and the main thread packs the entropy-coded bytes of a chunk into pinned staging; each chunk then goes H2D -> entropy decode (J1) ->
 * inverse DCT (J2) -> fused kernel (K1) on `stream` (NULL = the context's stream).  A chunk holds min(512, max(16, 32 * threads))
 * frames; the host side of chunk k+1 overlaps the GPU side of chunk k.  PNG and PGM frames are decoded on the host and copied as
 * 8-bit pixels.  The result equals mdc_seq_prepare's bit for bit, and so do the argument checks, the wrong-size rule and the error
 * rule: a frame that cannot be decoded (on the host or on the GPU) stops the call with MDC_ERR_FORMAT, the chunks before its chunk
 * are complete, and nothing from its chunk on is written.  Returns when the work is done on the device. */
int mdc_seq_prepare_device(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, float* const* d_out_levels, int levels,
                           int threads, mdc_stream stream);
/* mdc_seq_prepare_device with the levels stored as out_type (as mdc_seq_prepare_ex); the same bytes as mdc_seq_prepare_ex. */
int mdc_seq_prepare_device_ex(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, int out_type, void* const* d_out_levels,
                              int levels, int threads, mdc_stream stream);
/* getImageRaw_internal(ids[k]) for k < n into DEVICE memory: frame k -> d_out + k*h*row_pitch (row_pitch >= w; a multiple of 16 keeps
 * mdc_prepare_batch_pitched on its TMA loader).  ids may be in any order and may repeat.  The same device feed as mdc_seq_prepare_device
 * (`threads` host threads, 0 = the default count; chunks of min(512, max(16, 32 * threads)) frames; JPEG frames decoded on the GPU,
 * PNG / PGM frames on the host; `stream` as for mdc_prepare_batch), without the fused kernel.  Per frame, the outcome of
 * mdc_seq_read_gray8(s, ids[k], ...): status_host[k] (n ints, may be NULL) is MDC_OK if the frame reads and is w x h, and its rows
 * then hold the host reader's bytes; MDC_ERR_FORMAT if the host reader fails on it; MDC_ERR_INVALID_ARG if it reads at another size.
 * sizes_host (2*n ints: w h per frame, may be NULL) gets the size the host reader reports, or 0 0 if it fails.  Rows of a frame that
 * is not MDC_OK, and the padding bytes of every row, are left untouched; the frames around a failed one are still written.
 * Returns MDC_ERR_INVALID_ARG before anything is read for n < 0, a NULL c, s, ids or d_out with n > 0, an id outside the sequence,
 * w or h < 1 or row_pitch < w (none of which needs a device; n = 0 is a no-op); otherwise MDC_OK if every frame is MDC_OK,
 * MDC_ERR_FORMAT with the first such frame's message if not, MDC_ERR_CUDA on a runtime failure.  Returns when the frames are on
 * the device. */
int mdc_seq_read_gray8_device(mdc_ctx* c, const mdc_seq* s, const int* ids, int n, int w, int h, uint8_t* d_out, size_t row_pitch,
                              int* status_host, int* sizes_host, int threads, mdc_stream stream);
/* Baseline JPEGs in HOST memory (files[i], sizes[i] bytes) -> 8-bit grey planes on the device, the same bytes as mdc_seq_read_gray8
 * (the host decoder): d_out is [n][h][row_pitch] (row_pitch >= w; a multiple of 16 keeps mdc_prepare_batch_pitched on its TMA
 * loader).  Headers are parsed on the host; a frame the parser rejects, or one that is not w x h, is never uploaded, and the frames
 * around it still decode.  status_host (n ints, may be NULL) gets MDC_OK or MDC_ERR_FORMAT per frame; the call returns
 * MDC_ERR_FORMAT if any frame failed, with the host decoder's message for the first one ("frame <i>: ..."), and leaves the rows of
 * failed frames untouched.  Uses the context's device; `stream` as for mdc_prepare_batch; returns when the frames are decoded. */
int mdc_jpeg_decode_device(mdc_ctx* c, const uint8_t* const* files, const size_t* sizes, int n, int w, int h, uint8_t* d_out,
                           size_t row_pitch, int* status_host, mdc_stream stream);
/* Bytes the file of a w x h frame can take at any quality 1..100 (header, worst-case code of every block, stuffing, EOI); 0 unless
 * 1 <= w, h <= 65535. */
size_t mdc_jpeg_encode_bound(int w, int h);
/* cv::imwrite(".jpg") of a single-channel 8-bit image with quality `quality` (OpenCV's default: 95): d_frames [n][h][row_pitch]
 * u8 on the device -> frame k's complete JFIF file at d_out + k*out_stride (DEVICE), its length in sizes_host[k].  The bytes are
 * libjpeg's baseline defaults for one component (standard Huffman tables, accurate integer DCT, no restart markers), the same on
 * every run.  Padding bytes of the input rows are never read; bytes of d_out past a frame's size are unspecified.
 * MDC_ERR_INVALID_ARG before any kernel runs for a NULL c, n < 0, quality outside 1..100, w or h outside 1..65535, row_pitch < w,
 * out_stride < mdc_jpeg_encode_bound(w, h), or a NULL d_frames, d_out or sizes_host with n > 0; n = 0 is a no-op.  Uses the context's
 * device; `stream` as for mdc_prepare_batch; returns when the files are on the device. */
int mdc_jpeg_encode_device(mdc_ctx* c, const uint8_t* d_frames, size_t row_pitch, int n, int w, int h, int quality,
                           uint8_t* d_out, size_t out_stride, size_t* sizes_host, mdc_stream stream);

/* =====================================================================================
 * vignetteCalib optimiser, main_vignetteCalib.cpp:395-585 (SURVEY.md §8f N4).  Everything is device-resident, contiguous:
 *   d_images [n][wI*hI] float (NaN = invalidated pixel, :300-310), d_p2x / d_p2y [n][gw*gh] float plane-to-image maps
 *   (NaN = plane point not visible; finite entries keep the four bilinear taps inside the image, :352-356),
 *   d_plane_color [gw*gh], d_vignette [wI*hI].  The homographies come from mdc_marker_detect and mdc_marker_homography below,
 *   the maps and images from mdc_vc_plane_maps and mdc_vc_prepare_images.
 * Unlike the reference, which reads planeColor uninitialised in its first pass (:381, :425), the caller provides it.
 * With n = 0, d_images, d_p2x and d_p2y may be null; the plane colour and the vignette then become NaN, as in the reference.
 * integer_abs: the reference's outlier test is `abs(residual) > oth2` on a double (:423, :481).  1 = the residual is truncated to
 *   int first, which is what that line does when only `int abs(int)` is visible to unqualified lookup (libstdc++ before GCC 6,
 *   i.e. the reference's era; also how the unmodified program builds against this repo's oracle headers); 0 = fabs(residual).
 * ===================================================================================== */
/* "optimize planeColor" (:400-446): d_plane_color is read (residual test) and overwritten with sum(color*fac)/sum(fac*fac),
 * NaN where sum(fac*fac) < 1.  Bit-identical to the reference.  stats_host = {E, R} (E: fp64 sum in a fixed order that is not the
 * reference's: rounding-level, but the same bits on every run). */
int mdc_vc_plane_step(mdc_ctx* c, const float* d_images, const float* d_p2x, const float* d_p2y, int n, int gw, int gh, int wI, int hI,
                      const float* d_vignette, float* d_plane_color, double outlier_th2, int integer_abs, double stats_host[2]);
/* "optimize vignette" (:458-523) including the normalisation to maximum factor 1: d_vignette is read and overwritten.
 * The reference adds the scattered fp32 terms one after the other in fp32; here the same terms are rounded to a multiple of 2^-s
 * (s from the largest colours and footprint count, DESIGN.md §4) and added exactly as 64-bit integers, so the result differs from
 * the reference by the rounding error of its own chain and that rounding (<= 2e-5 relative in the tests) and is the same bits on
 * every run.  Terms that are not finite are added in fp32, as the reference does. */
int mdc_vc_vignette_step(mdc_ctx* c, const float* d_images, const float* d_p2x, const float* d_p2y, int n, int gw, int gh, int wI, int hI,
                         const float* d_plane_color, float* d_vignette, double outlier_th2, int integer_abs, double stats_host[2]);
/* "dilate & smoothe" (:542-566): `iterations` rounds (the reference: 4) of the NaN-aware 3x3 mean.  Bit-identical. */
int mdc_vc_smooth(mdc_ctx* c, const float* d_vignette, int wI, int hI, int iterations, float* d_out);
/* The loop itself: max_iterations x {plane step, vignette step}, outlier threshold outlier_th^2 in the second half of the
 * iterations and 10000^2 before (:397-398); d_smoothed (may be NULL) receives the 4x smoothed result of the last iteration.
 * log_host (may be NULL): [max_iterations][4] = {E, R} of the plane step, {E, R} of the vignette step. */
int mdc_vignette_calib(mdc_ctx* c, const float* d_images, const float* d_p2x, const float* d_p2y, int n, int gw, int gh, int wI, int hI,
                       int max_iterations, int outlier_th, int integer_abs, float* d_plane_color, float* d_vignette, float* d_smoothed,
                       double* log_host);

/* The front end in front of that loop, on the device.
 *
 * mdc_vc_plane_maps replaces main_vignetteCalib.cpp:266-284 followed by :346-357: for each image i the gw x gh plane grid is
 * projected through H_i * K_p2idx^-1 (K_p2idx of :195-200 from gw, gh, facw, fach), distorted with the rectifier's
 * distortCoordinates and masked: a point whose `int(X + 0.5)`, `int(Y + 0.5)` is not strictly inside (1, wI-2) x (1, hI-2), with
 * wI x hI the rectifier's INPUT size, becomes NaN in both maps.  homographies: HOST doubles, [n][9] row-major as cv::findHomography
 * returns them; d_p2x / d_p2y: DEVICE [n][gw*gh].  The 3x3 products are computed on the host in float the way the stand-in Eigen
 * of the runnable reference program does them (inverse by adjugate / determinant); real Eigen may differ in the last bit there.
 * Everything after that is bit-identical to the reference.  One kernel; `device` and `stream` as for
 * mdc_fov_distort_coordinates_device.  MDC_ERR_INVALID_OBJECT (with the reference's message) for an invalid rectifier. */
int mdc_vc_plane_maps(const mdc_fov* fov, const double* homographies, int n, int gw, int gh, float facw, float fach, float* d_p2x,
                      float* d_p2y, int device, mdc_stream stream);
/* mdc_vc_prepare_images replaces :286-301: image = (mean_exposure * raw) / t in fp32 (an exposure t == 0 counts as 1, :286), then
 * the gradient invalidation: centres 2 <= x < wI-2, 2 <= y < hI-2 in raster order, neighbours deltax-major; |centre - neighbour|
 * > max_abs_grad (the reference: 255) sets both to NaN, in place.  Bit-identical to the reference, order dependence included.
 *   d_raw     DEVICE [n][wI*hI]: what getImage(i, false, true, false, false) gives, i.e. mdc_unmap_u8 with MDC_REMOVE_GAMMA
 *   d_images  DEVICE [n][wI*hI] output; d_images == d_raw is allowed
 *   exposures_host  HOST [n] exposure times of the images
 *   mean_exposure   the caller's, computed as at :222-227: the float sum of getExposure(i) over every skip-th frame i, divided
 *                   by getNumImages() (ALL frames, not the number summed), and 1 if that is 0.  Frames without a marker are not
 *                   prepared (:240) but still count in the sum.
 * Images narrower or lower than 5 pixels have no centres: normalisation only.  Any n; no host synchronisation per image.
 * `stream` NULL = the context's stream, synchronised before returning. */
int mdc_vc_prepare_images(mdc_ctx* c, const float* d_raw, int n, int wI, int hI, const float* exposures_host, float mean_exposure,
                          int max_abs_grad, float* d_images, mdc_stream stream);

/* =====================================================================================
 * vignetteCalib's marker detection and homography, main_vignetteCalib.cpp:231-253: aruco 1.3.0's MarkerDetector::detect with
 * its default settings (aruco-1.3.0/src/markerdetector.cpp:50-64: ADPT_THRES 7/7, LINES corners, 56-pixel warp,
 * FiducidalMarkers::detect) on the rectified frame rounded to 8 bits, then cv::findHomography from the unit square.  Paths
 * below are inside aruco-1.3.0/src/.  The per-pixel passes run on the GPU (mdc_marker_threshold); the contour logic runs on the
 * host, one frame per call, re-entrant (no shared state), so frames can go to as many host threads as there are.
 * ===================================================================================== */
typedef struct mdc_marker {
    int id;             /* FiducidalMarkers id, 0..1023 */
    float corners[8];   /* x0 y0 .. x3 y3 in rectified pixels, in the order aruco returns them (rotation applied) */
} mdc_marker;
/* main_vignetteCalib.cpp:235-236 (convertTo(CV_8U, 1, 0): round half to even, saturate; NaN -> 0) and markerdetector.cpp:437-458
 * (adaptiveThreshold(grey, 255, ADAPTIVE_THRESH_MEAN_C, THRESH_BINARY_INV, 7, 7): the 7x7 mean with replicated image borders,
 * rounded to 8 bits; mask = grey - mean <= -7 ? 255 : 0), batched and bit-identical to OpenCV for finite inputs below 2^31:
 *   d_rect [n][h][w] f32 (mdc_prepare_batch level 0 with MDC_RECTIFY only), d_grey, d_mask [n][h][w] u8 (DEVICE pointers).
 * Any 1 <= w, h with w*h <= 2^28; `stream` as for mdc_prepare_batch. */
int mdc_marker_threshold(mdc_ctx* c, const float* d_rect, int n, int w, int h, uint8_t* d_grey, uint8_t* d_mask, mdc_stream stream);
/* MarkerDetector::detect from there on (HOST pointers, w*h bytes each): detectRectangles (:287-430: findContours(CV_RETR_LIST,
 * CV_CHAIN_APPROX_NONE) with the outer rows and columns as background, contour length filter, approxPolyDP to convex quads with
 * sides > 10 px, anti-clockwise corners, too-near candidates), the id reader per candidate (:166-191, arucofidmarkers.cpp:290-465:
 * perspective warp to 56 x 56, Otsu, 7 x 7 cells, Hamming code in four rotations), LINES corner refinement (:779-928) and the
 * final filters (:218-253: one marker per id, the larger perimeter; none within 2.5 % of the image border).  *count = markers
 * found; at most `capacity` are written, sorted by id; more than `capacity` returns MDC_ERR_INVALID_ARG.  Ids, candidates and
 * warped patches are exact; the corners come from two least-squares solves done in double where aruco solves in fp32 by SVD,
 * so they agree to about 1e-3 px.  Masks with more than 2^22 contours or 2^14 candidates return MDC_ERR_UNSUPPORTED. */
int mdc_marker_detect(const uint8_t* grey, const uint8_t* mask, int w, int h, mdc_marker* out, int capacity, int* count);
/* main_vignetteCalib.cpp:242-253: the homography H (row-major, H[8] = 1) that maps the plane points (-0.5, 0.5), (0.5, 0.5),
 * (0.5, -0.5), (-0.5, -0.5) to corners 0..3, from the exact 8 x 8 system solved in double with partial pivoting (cv::findHomography
 * gives the same to ~1e-13 relative for four points).  A quad with three corners on a line, or with a non-finite corner,
 * returns MDC_ERR_INVALID_ARG. */
int mdc_marker_homography(const float corners[8], double H[9]);
/* The stages of mdc_marker_detect one by one, so that each can be checked against the OpenCV call it restates:
 *   mdc_marker_contours     findContours's output: *n_contours contours of lengths[i] points each, xy = x, y pairs of all of
 *                           them in findContours's order (last found first); capacities too small -> MDC_ERR_INVALID_ARG
 *   mdc_marker_approx_poly  approxPolyDP(xy[0..n), eps, closed = true) into out_xy (room for n points)
 *   mdc_marker_candidates   the candidates that detectRectangles returns (quads [count][8])
 *   mdc_marker_read_patch   the 56 x 56 warped patch of a quad (before Otsu), the Otsu threshold, id (-1 = none) and rotations */
int mdc_marker_contours(const uint8_t* mask, int w, int h, int* xy, size_t point_capacity, int* lengths, int contour_capacity,
                        int* n_contours, size_t* n_points);
int mdc_marker_approx_poly(const int* xy, int n, double eps, int* out_xy, int* n_out);
int mdc_marker_candidates(const uint8_t* mask, int w, int h, float* quads, int capacity, int* count);
int mdc_marker_read_patch(const uint8_t* grey, int w, int h, const float quad[8], uint8_t* patch, int* otsu_threshold, int* id,
                          int* rotations);

/* responseCalib E-step, main_responseCalib.cpp:317-346 (kernel K3):
 *   d_data [n][npix] u8 image-major, d_t [n] f64 exposure times, d_G [256] f64 -> d_E [npix] f64.
 * Bit-exact with the reference's loop (sequential fp64 accumulation per pixel, no FMA). */
int mdc_estep(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_G, double* d_E, mdc_stream stream);

/* responseCalib building blocks around the E-step (SURVEY.md §8f N2; all DEVICE pointers, data = [n][npix] u8
 * image-major, t = [n] f64 exposure times, G = [256] f64, E = [npix] f64):
 *   mdc_rc_leak_padding  3x3 dilation of saturated interior pixels, `iterations` rounds, in place   main_responseCalib.cpp:212-236  bit-exact
 *   mdc_rc_einit         E = per-pixel mean over the n images                                          :249-259                       bit-exact
 *   mdc_rc_gstep         G[b] = sum(E[k]*t[i]) / count over samples with value b != 255, gaps extrapolated  :286-304   rounding-level: the products are
 *                        rounded as in the reference and then summed EXACTLY (fixed point), where the reference has one fp64 chain;
 *                        order-independent, so the same bits on every run and for every launch geometry.  The fixed-point scale
 *                        2^s comes from the exponents of the largest finite |E| and |t|, so every finite product keeps 48 bits
 *                        below the largest one (and below 2^1024 when max|E| * max|t| overflows).  Non-finite products (an
 *                        overflowing E*t, a NaN or infinite E or t) are summed in fp64 on the side and poison their bins as in
 *                        the reference; a non-finite exposure time of a fully saturated frame changes nothing, as in the reference.
 *                        With n = 0, d_data and d_t may be null (also for mdc_estep, mdc_rc_einit and mdc_rc_rmse).  With npix = 0
 *                        (the empty slice of a pixel-sharded rank), mdc_estep, mdc_rc_einit and mdc_rc_rescale accept null d_data
 *                        and d_E and touch neither.
 *   mdc_rc_rescale       factor = 255/G[255]; E *= factor; G *= factor; *factor_host = factor           :350-355                       bit-exact
 *   mdc_rc_rmse          out_host = {1e5*sqrt(mean((G[b]-t*E)^2 * 1e-10)), count}                       :50-69                         rounding-level
 *                        (the reference sums in long double); residuals, finite test and count exact; same bits on every run.
 *                        The sums are fp64: where the sum of r^2 * 1e-10 passes 1.8e308 the result is inf, where the
 *                        reference's long double would still be finite.
 *   mdc_response_calib   the optimisation loop of main(): E := mean, then nits x {G-step, E-step, rescale}, rmse after
 *                        each half-step; log_host (may be NULL) receives nits x 4 doubles {rmse_G, rmse_E, rmse_rescaled, count}.
 * These calls share scratch memory of the context (the leak-padding buffer, the G-step and rmse accumulators): do not run them on one
 * context from several streams at once; give each stream its own context. */
int mdc_rc_leak_padding(mdc_ctx* c, uint8_t* d_data, int n, int w, int h, int iterations, mdc_stream stream);
int mdc_rc_einit(mdc_ctx* c, const uint8_t* d_data, int n, int npix, double* d_E, mdc_stream stream);
int mdc_rc_gstep(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_E, double* d_G, mdc_stream stream);
int mdc_rc_rescale(mdc_ctx* c, int npix, double* d_E, double* d_G, double* factor_host);
int mdc_rc_rmse(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_G, const double* d_E, double out_host[2]);
int mdc_response_calib(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, int nits, double* d_E, double* d_G, double* log_host);
/* mdc_response_calib with a per-step hook: step(iteration, which, d_E, d_G, user) is called after E-init (iteration 0,
 * MDC_RC_STEP_E), and in iteration it = 0..nits-1 after the G-step (it + 1, MDC_RC_STEP_G) and after the E-step, before the
 * rescale (it + 1, MDC_RC_STEP_E), each right after the rmse line of that step is printed: where the reference plots
 * (main_responseCalib.cpp:273, :309-310, :344-345).  The context's stream is idle during the call, so the hook may enqueue work on
 * the context (the plots below) but must not change d_E or d_G.  The loop writes d_E and d_G again on the context's stream as soon
 * as the hook returns, without waiting for other streams: work the hook puts on another stream that reads them (a copy, a plot
 * call with a non-NULL stream) must be finished before it returns.  step = NULL is mdc_response_calib; the hook changes no result. */
#define MDC_RC_STEP_E 0
#define MDC_RC_STEP_G 1
typedef void (*mdc_rc_step_fn)(int iteration, int which, const double* d_E, const double* d_G, void* user);
int mdc_response_calib_ex(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, int nits, double* d_E, double* d_G,
                          double* log_host, mdc_rc_step_fn step, void* user);

/* responseCalib's result images (main_responseCalib.cpp:72-146), the pixels the reference hands to cv::imwrite, bit for bit
 * (DEVICE pointers; log and exp are glibc's, csrc/mdc_libm.h):
 *   mdc_rc_plot_e_range  d_range4 = {min ln(E+20), max ln(E+20), min E, max E} over npix values, with the reference's starting values
 *                        1e10 / -1e10 and strict comparisons (NaN is skipped; all NaN or npix = 0 leaves the starting values).
 *                        Ties go to the lower pixel index, so a zero extreme has the sign the reference's scan gives it.  The
 *                        ranges of several slices of an image, taken in slice order, join into the range of the whole image
 *                        with the same rule: a later slice's value replaces an earlier one only when strictly smaller / larger.
 *   mdc_rc_plot_e_map    from a range in device memory: d_bgr [npix][3] u8, the colour map of ln(E+20) in cv::Mat's BGR order
 *                        (E-k.png), and d_e16 [npix] u16 = 65025 (E - Emin) / (Emax - Emin) (E-k16.png), converted through a
 *                        32-bit truncation as x86-64 converts (NaN and values of 2^31 or more give 0).  Slices concatenate.
 *   mdc_rc_plot_e        both passes on one stream.
 *   mdc_rc_plot_g        d_out [256][256] u8: plotG's image (G-k.png) as cv::imwrite converts GImg * 255 (round half to even,
 *                        saturate, NaN -> 0); minmax_host (may be NULL) = {min G, max G}, the values it prints. */
int mdc_rc_plot_e_range(mdc_ctx* c, const double* d_E, int npix, double* d_range4, mdc_stream stream);
int mdc_rc_plot_e_map(mdc_ctx* c, const double* d_E, int npix, const double* d_range4, uint8_t* d_bgr, uint16_t* d_e16, mdc_stream stream);
int mdc_rc_plot_e(mdc_ctx* c, const double* d_E, int npix, double* d_range4, uint8_t* d_bgr, uint16_t* d_e16, mdc_stream stream);
int mdc_rc_plot_g(mdc_ctx* c, const double* d_G, uint8_t* d_out, double* minmax_host, mdc_stream stream);

/* glibc's double exp and log as the plots evaluate them (csrc/mdc_libm.h), for checking against a deployment's libm:
 * out[i] = op(in[i]) on the host or on the GPU (device pointers). */
#define MDC_LIBM_EXP 0
#define MDC_LIBM_LOG 1
void mdc_libm_host(int op, const double* in, double* out, size_t n);
int mdc_libm_device(int op, const double* d_in, double* d_out, size_t n, int device, mdc_stream stream);

/* A PNG file of 8-bit or 16-bit samples, 1 (grey) or 3 channels, as cv::imwrite takes them: 3 channels in BGR order, 16-bit
 * samples in host byte order; rows row_bytes apart.  Decodes to the same pixels as cv::imwrite's file.  MDC_ERR_IO when the
 * file cannot be written. */
int mdc_png_write(const char* path, const void* pixels, int w, int h, size_t row_bytes, int depth, int channels);
/* The two global reductions of the loop as per-rank partials, for PIXEL-SHARDED runs (pixels are independent in every pass,
 * main_responseCalib.cpp:317-346; each rank holds its slice of every image as [n][npix_local]).  The accumulators stay on the device:
 *   mdc_rc_gstep_accumulate  d_gsum256[b] = sum E[k]*t[i], d_gnum256[b] = count over this rank's pixels (:290-299); reuse_counts != 0
 *                            keeps d_gnum256 (it depends on the images only) — all-reduce(sum) both arrays across ranks, then
 *   mdc_rc_gstep_finish      G = gsum/gnum with the reference's sequential gap extrapolation (:300-304), identically on every rank;
 *   mdc_rc_rmse_accumulate   d_acc2 = {sum (G[b]-t*E)^2 * 1e-10, count} over this rank's pixels (:50-69) — all-reduce(sum), then
 *                            rmse = 1e5*sqrt(acc[0]/acc[1]).
 * E-step, E-init and rescale need no collective (mdc_estep / mdc_rc_einit / mdc_rc_rescale on the local slice; G is replicated).
 * mdc_response_calib_sharded (include/mdc_b200_nccl.h) is the whole loop over NCCL. */
int mdc_rc_gstep_accumulate(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_E,
                            double* d_gsum256, unsigned long long* d_gnum256, int reuse_counts, mdc_stream stream);
int mdc_rc_gstep_finish(mdc_ctx* c, const double* d_gsum256, const unsigned long long* d_gnum256, double* d_G, mdc_stream stream);
int mdc_rc_rmse_accumulate(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_G, const double* d_E,
                           double* d_acc2, mdc_stream stream);
/* The G-step of a pixel-sharded run with sums that are exact ACROSS ranks, so that G (and therefore E) comes out bit-identical for
 * any number of ranks, 1 included (mdc_rc_gstep / mdc_response_calib compute the same bits).  The per-rank sums of
 * mdc_rc_gstep_accumulate are exact integers that are rounded to fp64 before the all-reduce; here they travel as integers:
 *   mdc_rc_gstep_scale             d_scale4 (4 x u64) = bit patterns of the largest finite |E|, |t| of this rank's pixels and a flag
 *                                  for non-finite exposure times — all-reduce(MAX) so that every rank scales alike, then
 *   mdc_rc_gstep_accumulate_exact  d_limbs768 (3 x 256 int64: each bin's 128-bit fixed-point sum as three 43-bit limbs),
 *                                  d_special256 (fp64 sums of non-finite products) and d_gnum256 as above — all-reduce(SUM) each, then
 *   mdc_rc_gstep_finish_exact      G from the summed limbs: limbs -> 128-bit integer -> fp64 -> / gnum, gaps extrapolated (:300-304). */
int mdc_rc_gstep_scale(mdc_ctx* c, const double* d_E, int npix, const double* d_t, int n, unsigned long long* d_scale4, mdc_stream stream);
int mdc_rc_gstep_accumulate_exact(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_E,
                                  const unsigned long long* d_scale4, long long* d_limbs768, double* d_special256,
                                  unsigned long long* d_gnum256, int reuse_counts, mdc_stream stream);
int mdc_rc_gstep_finish_exact(mdc_ctx* c, const unsigned long long* d_scale4, const long long* d_limbs768, const double* d_special256,
                              const unsigned long long* d_gnum256, double* d_G, mdc_stream stream);

/* -------------------------------------------------------------------------------------
 * Host-buffer entry points (what the compat classes call): H2D copy, kernels, D2H copy.
 * Host pointers may be pageable; pinned memory (mdc_host_alloc) makes the copies async.
 * ------------------------------------------------------------------------------------- */
int mdc_unmap_u8_host(mdc_ctx* c, const uint8_t* in, float* out, int n, unsigned flags);
int mdc_undistort_u8_host(mdc_ctx* c, const uint8_t* in, float* out, int n_pix_in, int n_pix_out);
int mdc_undistort_f32_host(mdc_ctx* c, const float* in, float* out, int n_pix_in, int n_pix_out);
/* getImage for n_frames host frames; out_levels[l] host buffers laid out as in mdc_prepare_batch (NULL only for a level without
 * pixels).  Internally chunked (MDC_HOST_CHUNK frames, default 16) on three streams so H2D, kernel and D2H overlap; returns
 * after the last copy into out_levels has landed. */
int mdc_prepare_batch_host(mdc_ctx* c, const uint8_t* frames, int n_frames, unsigned flags,
                           float* const* out_levels, int levels);
/* The same with the levels stored as out_type (MDC_OUT_*, as for mdc_prepare_batch_ex): the device buffers of the pipeline and the
 * copies back to out_levels move out_type elements, so F16 halves and U8 quarters the device-to-host bytes.  An unknown out_type
 * returns MDC_ERR_INVALID_ARG before anything else. */
int mdc_prepare_batch_host_ex(mdc_ctx* c, const uint8_t* frames, int n_frames, unsigned flags, int out_type, void* const* out_levels,
                              int levels);
/* Pinned host memory for the calling thread's current CUDA device, placed on the NUMA node that device is attached to
 * (MDC_NUMA_BIND=0 disables the placement). */
int mdc_host_alloc(void** p, size_t bytes);
void mdc_host_free(void* p);
/* NUMA node of a CUDA device (sysfs: PCI device -> numa_node), or -1 if unknown. */
int mdc_device_numa_node(int device);

#ifdef __cplusplus
}
#endif
#endif /* MDC_B200_H */
