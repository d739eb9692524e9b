// Device-side data structures and launch wrappers shared between mdc_kernels.cu and
// mdc_capi.cu.  sm_90a only.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "mdc_b200.h"

namespace mdc {

constexpr int kTile = 32;            // output tile edge (pixels); pyramid levels 0..4 close inside a tile
constexpr int kConsumers = 256;      // 8 consumer warps; warp w owns tile rows 4w..4w+3, lane = x
constexpr int kThreads = kConsumers;
constexpr int kInKernelLevels = 3;   // levels 0..2 come out of the fused kernel's (warp-local) epilogue; deeper levels use K2
constexpr int kMaxBoxWordsPerThread = 8;   // LDG loader: u32 words of the input box prefetched per thread
constexpr int kLdgStages = 2;         // LDG loader: double buffer
constexpr int kMaxStages = 8;
constexpr int kItemSlots = 4;          // work items in flight between the producer warp and the consumers
constexpr int kSmemHeaderBytes = 33024;   // lut 32768 + item ring 32 + 24 mbarriers 192, rounded up to 128
constexpr int kMaxClasses = 64;      // distinct TMA box shapes per plan (descriptors travel as kernel parameters)
constexpr int kMaxTex = 128;         // texture-gather loader: u8 pitch-2D texture objects per launch (one per chunk of frames)
constexpr int kTexThreads = 256;     // texture-gather loader: 8 independent warps per CTA, no producer warp

// How a tile's input pixels are fetched.
enum TileMode : int { TILE_EMPTY = 0, TILE_STAGED = 1, TILE_DIRECT = 2, TILE_HAS_BLACK = 0x10 /* flag */ };

// One output tile of the rectification plan (built once per context from the remap tables).
struct alignas(16) TileDesc {
    int x0, y0;        // origin of the input bounding box (x0 is a multiple of 16: TMA box origins must be 16-byte aligned)
    int bw_bh;         // box width (multiple of 16, also the smem pitch) | box height << 16
    int mode_map;      // TileMode (low nibble) | TILE_HAS_BLACK | (tensor-map class index << 8) | (TMA box height << 16)
};

// TMA descriptors of one launch: one 3-D u8 tensor map per box class, passed by value as a
// __grid_constant__ kernel parameter (no device-memory copy, no lifetime to manage).
struct TmaMaps {
    alignas(64) CUtensorMap m[kMaxClasses];
};

// Texture-gather loader: one u8 pitch-2D texture object per chunk of `chunk_frames` consecutive frames (stacked vertically:
// texture row = frame_in_chunk * in_h + y), passed by value like the TMA descriptors.
struct TexSet {
    unsigned long long tex[kMaxTex];
};

struct FusedParams {
    const uint8_t* frames;       // [n_frames][in_h][in_pitch]
    int n_frames;
    int in_w, in_h, out_w, out_h;
    int in_pitch;                // bytes from one input row to the next (>= in_w; the vignette / remap tables stay tightly packed)
    const float* remap_x;        // [out_w*out_h]
    const float* remap_y;
    const float* vinv;           // [in_w*in_h] or nullptr
    const float* ginv;           // [256] or nullptr
    const TileDesc* tiles;       // [tiles_x*tiles_y]
    int* work_counter;           // zeroed before the launch; item = gridDim.x + atomicAdd(work_counter, 1)
    int tiles_x, n_tiles;
    void* out[kInKernelLevels];  // levels 0..levels-1, elements of the launch's output type (MDC_OUT_*)
    float* level2_f32;           // narrow output types only: fp32 copy of level 2 for the K2 chain behind K1, or nullptr
    void* unused_[MDC_MAX_PYR_LEVELS - kInKernelLevels - 1];   // room for eight level pointers: the parameter offsets (and the fp32 code) stay
    int lw[MDC_MAX_PYR_LEVELS], lh[MDC_MAX_PYR_LEVELS];
    int levels;                  // 1..kInKernelLevels (levels written by K1 itself)
    unsigned lut_gamma, use_vig, kill;   // sanitised unMapImage flags
    int box_px_max;              // largest staged box (pixels) -> smem carve-up
    int chunk_frames;            // frames per schedule chunk (L2 residency of the inputs)
    int tma_stages;              // depth of the TMA stage ring (2..kMaxStages)
    int tiles_per_cta;           // texture-gather loader: consecutive tiles one CTA works through (grid.x = ceil(n_tiles / tiles_per_cta))
    int carveout;                // host side only: preferred shared-memory carve-out in percent for this launch, 0 = the driver's choice
};
static_assert(sizeof(FusedParams) == 256 && offsetof(FusedParams, lw) == 152, "FusedParams layout: the kernels' parameter offsets");

// Floor-study switches (scripts/k1_study.py): which of the three shared-memory/LSU consumers of the frame loop run.
// kStudyAll is the product; the others replace the disabled part by one or two ALU instructions so that the rest can be timed alone.
enum StudyBits : int { kStudyTaps = 1, kStudyLut = 2, kStudyStores = 4, kStudyAll = 7 };
// The K1 kernels' variant parameter: the study bits, and above them the output type (MDC_OUT_*) the levels are stored as.
constexpr int kOutShift = 8;
constexpr int k1_variant(int out_type, int study = kStudyAll) { return study | out_type << kOutShift; }

size_t fused_smem_bytes(int box_px_max, int stages);
int fused_tma_stages(int box_px_max, int ctas_per_sm);
// out_type (MDC_OUT_*): element type of p.out[]; every type computes the fp32 levels and converts them at the store
cudaError_t launch_fused(const FusedParams& p, const TmaMaps* maps, int grid, int min_ctas, int out_type, cudaStream_t stream);  // maps == nullptr: LDG loader
int fused_max_ctas_per_sm(int box_px_max, int stages, bool tma, bool vig, bool pyr, int min_ctas, int out_type);
cudaError_t launch_fused_study(const FusedParams& p, const TmaMaps* maps, int grid, int study, cudaStream_t stream);   // <tma, vig, no pyramid, 3 CTAs/SM> only
// texture-gather loader (taps through the TEX pipe, LUT + stores through the LSU pipe)
cudaError_t launch_fused_tex(const FusedParams& p, const TexSet& texs, int n_chunks, int min_ctas, bool prefetch, int study, int out_type,
                             cudaStream_t stream);
int fused_tex_max_ctas_per_sm(bool vig, bool pyr, int min_ctas, bool prefetch);
cudaError_t launch_count_mismatch(const void* a, const void* b, size_t n_words, unsigned long long* out, cudaStream_t stream);

// out: elements of out_type; out_f32 (narrow types only, may be nullptr): the same pixels as fp32, for a K2 pass that reads them
cudaError_t launch_unmap(const uint8_t* in, void* out, int out_type, float* out_f32, size_t n, int n_frames, const float* ginv,
                         const float* vinv, unsigned kill, cudaStream_t stream);
cudaError_t launch_undistort_f32(const float* in, float* out, int in_w, int n_in, int n_out, int n_frames,
                                 const float* remap_x, const float* remap_y, cudaStream_t stream);
// K2 reads fp32 levels and writes out_type; dst_f32 / d2_f32 (narrow types only, may be nullptr) get the fp32 result as well
cudaError_t launch_pyr_down(const float* src, int sw, int sh, void* dst, int out_type, float* dst_f32, int n_frames, cudaStream_t stream);
cudaError_t launch_pyr_down2(const float* src, int sw, int sh, void* d1, void* d2, int out_type, float* d2_f32, int n_frames,
                             cudaStream_t stream);
// per-calibration constants of distortCoordinates (same ten floats as mdc_distort_constants on the host side)
struct DistortConstants { float ocx, ocy, ofx, ofy, d2t, omega, fx, fy, cx, cy; };
cudaError_t launch_fov_distort(float* xs, float* ys, size_t n, const DistortConstants& k, cudaStream_t stream);
cudaError_t launch_atanf(const float* in, float* out, size_t n, cudaStream_t stream);
// vignetteCalib plane-to-image maps: hk [n][9] device floats (H * K_p2idx^-1 per image); xs/ys [n][gw*gh]
cudaError_t launch_vc_plane_maps(const float* hk, int n, int gw, int gh, int wI, int hI, const DistortConstants& k, float* xs, float* ys,
                                 cudaStream_t stream);
cudaError_t launch_estep(const uint8_t* data, int n, int npix, const double* t, const double* G, double* E,
                         cudaStream_t stream);

cudaError_t launch_rc_leak_padding(const uint8_t* in, uint8_t* out, int n, int w, int h, cudaStream_t s);
cudaError_t launch_rc_einit(const uint8_t* data, int n, int npix, double* E, cudaStream_t s);
// fx_scratch: kGstepFxScratchBytes of device memory for the fixed-point accumulators of one pass (zeroed by the call)
constexpr size_t kGstepFxScratchBytes = 64 + 3 * 256 * 8;
cudaError_t launch_rc_gstep(const uint8_t* data, int n, int npix, const double* t, const double* E, double* gsum, unsigned long long* gnum,
                            double* G, bool reuse_counts, void* fx_scratch, cudaStream_t s);
cudaError_t launch_rc_gstep_accum(const uint8_t* data, int n, int npix, const double* t, const double* E, double* gsum, unsigned long long* gnum,
                                  bool reuse_counts, void* fx_scratch, cudaStream_t s);
cudaError_t launch_rc_gstep_finish(const double* gsum, const unsigned long long* gnum, double* G, cudaStream_t s);
// the G-step of one rank of a pixel-sharded run, with sums that are exact across ranks: scale (four u64 words; all-reduce MAX) ->
// accumulate (limbs768: 3 x 256 int64, special256: 256 fp64, both all-reduce SUM) -> finish.  See mdc_kernels.cu.
cudaError_t launch_rc_gstep_scale(const double* E, int npix, const double* t, int n, void* scale4, cudaStream_t s);
cudaError_t launch_rc_gstep_accum_exact(const uint8_t* data, int n, int npix, const double* t, const double* E, const void* scale4, long long* limbs768,
                                        double* special256, unsigned long long* gnum, bool reuse_counts, void* fx_scratch, cudaStream_t s);
cudaError_t launch_rc_gstep_finish_exact(const void* scale4, const long long* limbs768, const double* special256, const unsigned long long* gnum,
                                         double* gsum_scratch, double* G, cudaStream_t s);
bool rc_counts_reusable(const uint8_t* data, int npix);      // reuse_counts is only available on the bulk-copy streaming path
cudaError_t launch_rc_rescale(int npix, double* E, double* G, double* factor, cudaStream_t s);
constexpr int kRmsePartialPairs = 2048;      // rmse: capacity of the per-CTA partial scratch ({error, count} pairs)
cudaError_t launch_rc_rmse(const uint8_t* data, int n, int npix, const double* t, const double* G, const double* E, double* acc2, double* partials,
                           cudaStream_t s);

}  // namespace mdc
