// C-ABI glue: device context (tables in HBM, tile plan, TMA descriptors), the getImage mode
// switch, and the host-buffer pipeline.  See include/mdc_b200.h for the contract of each entry.
#include <cuda.h>
#include <cuda_runtime.h>
#include <sys/syscall.h>
#include <unistd.h>

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <tuple>
#include <utility>
#include <vector>

#include "mdc_internal.h"
#include "mdc_kernels.cuh"

using namespace mdc;

#define CU_CHECK(expr)                                                                          \
    do {                                                                                        \
        cudaError_t e__ = (expr);                                                               \
        if (e__ != cudaSuccess) {                                                               \
            mdc_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return MDC_ERR_CUDA;                                                                \
        }                                                                                       \
    } while (0)

namespace {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// Looked up once per process; a function-local static is initialised once even when several threads create contexts at once.
EncodeTiledFn encode_tiled_fn() {
    static const EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        return cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess
                   ? reinterpret_cast<EncodeTiledFn>(p)
                   : nullptr;
    }();
    return fn;
}

constexpr int kHostPipeDepth = 3;   // host-buffer pipeline: chunks in flight
constexpr int kCounterRing = 64;
constexpr int kMaxStagedPx = 8192;  // largest staged box (pixels, height rounded to 8): 32 KB float tile

// Host cache of N sets of TMA descriptors or texture objects, keyed by what a set describes (frames pointer, frame count, row
// pitch, frames per texture object or 0) and refilled round-robin.  No call's frames are at address 0, so the default key marks a
// slot that holds nothing; a build clears the key first and sets it once the set is complete.
using FramesKey = std::tuple<const void*, int, int, int>;
template <class Set, int N>
struct HostCache {
    struct Slot { FramesKey key; Set set{}; };
    Slot slots[N];
    int next = 0;
    Set* find(const FramesKey& k) { for (Slot& s : slots) if (s.key == k) return &s.set; return nullptr; }
    Slot& take() { Slot& s = slots[next]; next = (next + 1) % N; return s; }    // the next slot; the caller releases what it held
};
using MapCache = HostCache<TmaMaps*, 8>;                           // 64-byte aligned host memory, reused across keys
using TexCache = HostCache<std::vector<cudaTextureObject_t>, 32>;   // one object per chunk of frames

}  // namespace

constexpr size_t kRcFxOffset = 256 + 256 + 1 + 2 + 2 * kRmsePartialPairs + 1;      // doubles before the fixed-point scratch in d_rc (8-byte units, 16-byte aligned start)
struct mdc_ctx {
    int device = 0, sm_count = 132;
    int in_w = 0, in_h = 0, out_w = 0, out_h = 0;
    bool have_fov = false, have_gamma = false, have_vig = false;
    // device tables (owned unless adopted)
    bool owns_tables = true;
    float *d_rx = nullptr, *d_ry = nullptr, *d_ginv = nullptr, *d_vinv = nullptr;
    // tile plan
    std::vector<TileDesc> tiles;
    std::vector<std::pair<int, int>> classes;   // (bw, bh rounded to 8) of every TMA box class
    int tiles_x = 0, tiles_y = 0, box_px_max = 128;
    bool plan_tma_ok = false;
    TileDesc* d_tiles = nullptr;
    int* d_counters = nullptr;   // ring of work counters (one per launch in flight)
    cudaEvent_t counter_free[kCounterRing] = {};   // recorded behind the launch that used the slot last; its next user waits on it
    unsigned counter_next = 0;
    MapCache map_cache;                  // TMA descriptor sets (descriptors are passed to the kernel by value)
    // texture-gather loader: device limits, self-check verdict, cache of texture-object sets
    int tex_max_rows = 0, tex_max_width = 0, tex_pitch_align = 32, tex_base_align = 512;
    bool tex_ok = false;                 // the context-creation self-check found the texture path bit-identical to the staged path
    TexCache tex_cache;
    // knobs (loader: -1 auto, 0 LDG, 1 TMA, 2 texture gather)
    int use_tma = -1, ctas_per_sm = 0, chunk_frames = 0, tma_stages = 0;
    int tex_tiles_per_cta = 2, tex_prefetch = 0, k1_study = kStudyAll;
    bool auto_hybrid = false;                    // "auto" prefers the hybrid loader (MDC_AUTO_HYBRID)
    int carveout = 0;                            // preferred shared-memory carve-out (%) of the K1 launches, 0 = driver's choice
    int hyb_tex_pct = 40, hyb_stg_ctas = 2;      // hybrid loader: share of the chunks given to the texture kernel, staged CTAs per SM
    cudaStream_t aux_stream = nullptr;           // hybrid loader: the texture kernel's stream + fork/join events
    cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
    // streams + host pipeline scratch
    cudaStream_t stream = nullptr;
    cudaStream_t pipe_stream[kHostPipeDepth] = {nullptr, nullptr, nullptr};
    uint8_t* pipe_in[kHostPipeDepth] = {nullptr, nullptr, nullptr};
    uint8_t* pipe_out[kHostPipeDepth] = {nullptr, nullptr, nullptr};   // the levels of a chunk (any output type), then its fp32 scratch
    size_t pipe_in_bytes = 0, pipe_out_bytes = 0;
    // scratch for the single-op host entry points
    void* scratch_a = nullptr; size_t scratch_a_bytes = 0;
    void* scratch_b = nullptr; size_t scratch_b_bytes = 0;
    cudaMemPool_t f32_pool = nullptr;   // narrow output types: fp32 copies of the levels K2 reads, allocated per call (stream-ordered)
    double* d_rc = nullptr;      // responseCalib scratch: gsum[256] gnum[256] factor[1] acc[2] partials[2*kRmsePartialPairs] | fixed-point G-step accumulators (kRcFxOffset)
    long long launches = 0;
};

namespace {

int ensure_bytes(void** p, size_t* have, size_t need) {
    if (*have >= need) return MDC_OK;
    if (*p) cudaFree(*p);
    *p = nullptr; *have = 0;
    CU_CHECK(cudaMalloc(p, need));
    *have = need;
    return MDC_OK;
}

// Every entry of the remap tables must lie in the domain inside which the reference's undistort reads only pixels of the frame
// (FOVUndistorter.cpp:347-365): x < 0 (black, whatever y holds), or 0 <= x < in_w-1 and -1 < y < in_h-1 (truncation toward zero
// makes the row of a y in (-1, 0) row 0).  NaN and infinite coordinates are outside it, except a y under a negative x.  The tile
// plan and the kernels rely on this: a box, tap or vignette index is never clamped.
int check_table_domain(const float* rx, const float* ry, int out_w, int out_h, int in_w, int in_h) {
    const size_t n = static_cast<size_t>(out_w) * out_h;
    for (size_t i = 0; i < n; ++i) {
        const float x = rx[i], y = ry[i];
        if (x < 0) continue;
        // compared in double: in_w-1 and in_h-1 are not always floats
        if (static_cast<double>(x) < in_w - 1.0 && static_cast<double>(y) > -1.0 && static_cast<double>(y) < in_h - 1.0) continue;
        mdc_set_error("remap table entry at output pixel (%zu, %zu) is (x %.9g, y %.9g): outside the domain x < 0, or 0 <= x < %d and -1 < y < %d, "
                      "in which undistort reads inside the %d x %d input frame", i % static_cast<size_t>(out_w), i / static_cast<size_t>(out_w),
                      static_cast<double>(x), static_cast<double>(y), in_w - 1, in_h - 1, in_w, in_h);
        return MDC_ERR_INVALID_ARG;
    }
    return MDC_OK;
}

// Input pixels one output tile's taps start from (xlo..xhi-1, ylo..yhi-1; xhi < 0: none), and whether it has black pixels (x < 0)
struct TileBounds { int xlo = 1 << 30, xhi = -1, ylo = 1 << 30, yhi = -1; bool black = false; };

// Rows of a staged box of pitch `bw` that one pass of the LDG loader covers (rows x words-per-row thread tiling).
int ldg_row_step(int bw) {
    int lg = 2;
    while ((4 << lg) < bw) ++lg;
    return std::max(1, kThreads >> lg);
}

// Box width = shared-memory pitch of the staged box of tile t (origin x0, ylo; bh rows, bh8 once rounded to the row granularity).
// The tap loads of a warp (32 lanes = one output row, 4 byte taps each) are a fixed, calibration-dependent access pattern, so their
// bank conflicts can be SIMULATED here, per candidate pitch, and traded against the extra bytes TMA has to write for a wider box.
// Returns the pitch with the fewest shared-memory wavefronts per frame, bw_min when no candidate fits.
int search_pitch(const mdc_ctx* c, const float* rx, const float* ry, int t, int x0, int ylo, int bh, int bh8, int bw_min) {
    const int OW = c->out_w, OH = c->out_h;
    const int tx0 = (t % c->tiles_x) * kTile, ty0 = (t / c->tiles_x) * kTile;
    int bw = bw_min;
    long best_cost = -1;
    for (int pitch = bw_min; pitch <= std::min(bw_min + 112, 256); pitch += 16) {
        if (pitch * bh8 > kMaxStagedPx) break;
        const int rs = ldg_row_step(pitch);
        if ((bh + rs - 1) / rs > kMaxBoxWordsPerThread) break;      // must stay loadable by the LDG loader as well
        long wavefronts = 0;
        for (int y = ty0; y < std::min(ty0 + kTile, OH); ++y) {
            int offs[kTile];
            int nl = 0;
            for (int x = tx0; x < std::min(tx0 + kTile, OW); ++x) {
                const float sx = rx[static_cast<size_t>(y) * OW + x], sy = ry[static_cast<size_t>(y) * OW + x];
                offs[nl++] = (sx < 0) ? 0 : (static_cast<int>(sy) - ylo) * pitch + (static_cast<int>(sx) - x0);
            }
            const int delta[4] = {0, 1, pitch, pitch + 1};
            for (int d = 0; d < 4; ++d) {
                int words[32][4], cnt[32];
                for (int b = 0; b < 32; ++b) cnt[b] = 0;
                int worst = 1;
                for (int l = 0; l < nl; ++l) {
                    const int w = (offs[l] + delta[d]) >> 2, b = w & 31;
                    bool seen = false;
                    for (int i = 0; i < cnt[b] && i < 4; ++i) seen |= (words[b][i] == w);
                    if (!seen) { if (cnt[b] < 4) words[b][cnt[b]] = w; ++cnt[b]; worst = std::max(worst, cnt[b]); }
                }
                wavefronts += worst;
            }
        }
        const long cost = wavefronts + pitch * bh8 / 128;   // + wavefronts TMA spends writing the box
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; bw = pitch; }
    }
    return bw;
}

// MDC_VERBOSE: the plan at row granularity `gran`
void print_plan(const mdc_ctx* c, int gran) {
    long staged_bytes = 0; int n_staged = 0, n_direct = 0, n_empty = 0, n_black = 0;
    for (const TileDesc& t : c->tiles) {
        const int mode = t.mode_map & 0x0f;
        if (mode == TILE_STAGED) { staged_bytes += (t.bw_bh & 0xffff) * (t.mode_map >> 16); ++n_staged; }
        n_direct += mode == TILE_DIRECT;
        n_empty += mode == TILE_EMPTY;
        n_black += (t.mode_map & TILE_HAS_BLACK) != 0;
    }
    fprintf(stderr, "[mdc] plan: %d tiles (%d staged, %d direct, %d empty, %d with black pixels), %zu TMA box classes at row granularity %d, "
            "largest box %d B, mean box %ld B\n", static_cast<int>(c->tiles.size()), n_staged, n_direct, n_empty, n_black, c->classes.size(),
            gran, c->box_px_max, n_staged ? staged_bytes / n_staged : 0);
}

// Build the tile plan from HOST copies of the remap tables (inside the domain of check_table_domain).
void build_plan(mdc_ctx* c, const float* rx, const float* ry) {
    const int OW = c->out_w, OH = c->out_h;
    c->tiles_x = (OW + kTile - 1) / kTile;
    c->tiles_y = (OH + kTile - 1) / kTile;
    const int n_tiles = c->tiles_x * c->tiles_y;
    c->tiles.assign(n_tiles, TileDesc{0, 0, 0, TILE_EMPTY});
    const char* e;
    const bool pitch_search = (e = getenv("MDC_PITCH_SEARCH")) ? atoi(e) != 0 : true;
    std::vector<TileBounds> bounds(n_tiles);
    for (int t = 0; t < n_tiles; ++t) {
        const int tx0 = (t % c->tiles_x) * kTile, ty0 = (t / c->tiles_x) * kTile;
        TileBounds& b = bounds[t];
        for (int y = ty0; y < std::min(ty0 + kTile, OH); ++y)
            for (int x = tx0; x < std::min(tx0 + kTile, OW); ++x) {
                const float sx = rx[static_cast<size_t>(y) * OW + x], sy = ry[static_cast<size_t>(y) * OW + x];
                if (sx < 0) { b.black = true; continue; }
                const int xi = static_cast<int>(sx), yi = static_cast<int>(sy);
                b.xlo = std::min(b.xlo, xi); b.xhi = std::max(b.xhi, xi + 1);
                b.ylo = std::min(b.ylo, yi); b.yhi = std::max(b.yhi, yi + 1);
            }
    }
    // TMA box classes: box heights are rounded up to `gran` rows; coarsen until the shapes fit kMaxClasses
    for (int gran = 8; gran <= 256; gran *= 2) {
        c->classes.clear();
        c->box_px_max = 128;
        std::map<std::pair<int, int>, int> class_index;
        for (int t = 0; t < n_tiles; ++t) {
            const TileBounds& b = bounds[t];
            TileDesc td{0, 0, 0, TILE_EMPTY};
            if (b.xhi >= 0) {
                // box origins are always 16-byte aligned (TMA faults on others): whether TMA can be used is decided per call from the ROW
                // PITCH of the frames (a width that is not a multiple of 16 is fine once the host pipeline pads the rows in its H2D copy)
                const int x0 = b.xlo & ~15;
                const int bh = b.yhi - b.ylo + 1, bh8 = (bh + gran - 1) / gran * gran;
                const int bw_min = ((b.xhi - x0 + 1) + 15) & ~15;
                const int bw = pitch_search ? search_pitch(c, rx, ry, t, x0, b.ylo, bh, bh8, bw_min) : bw_min;
                const int rstep = ldg_row_step(bw);
                td.x0 = x0; td.y0 = b.ylo; td.bw_bh = bw | (bh << 16);
                if (bw <= 256 && bh8 <= 256 && bw * bh8 <= kMaxStagedPx && (bh + rstep - 1) / rstep <= kMaxBoxWordsPerThread) {
                    const auto cls = class_index.emplace(std::make_pair(bw, bh8), static_cast<int>(c->classes.size()));
                    if (cls.second) c->classes.push_back(cls.first->first);
                    td.mode_map = TILE_STAGED | (cls.first->second << 8) | (bh8 << 16);
                    c->box_px_max = std::max(c->box_px_max, bw * bh8);
                } else {
                    td.mode_map = TILE_DIRECT;
                }
            }
            if (b.black) td.mode_map |= TILE_HAS_BLACK;
            c->tiles[t] = td;
        }
        if (getenv("MDC_VERBOSE")) print_plan(c, gran);
        if (static_cast<int>(c->classes.size()) <= kMaxClasses) break;
    }
    c->plan_tma_ok = !c->classes.empty() && static_cast<int>(c->classes.size()) <= kMaxClasses && encode_tiled_fn() != nullptr;
}

int upload_plan(mdc_ctx* c) {
    const size_t n = c->tiles.size();
    CU_CHECK(cudaMalloc(&c->d_tiles, std::max<size_t>(n, 1) * sizeof(TileDesc)));
    CU_CHECK(cudaMemcpy(c->d_tiles, c->tiles.data(), n * sizeof(TileDesc), cudaMemcpyHostToDevice));
    return MDC_OK;
}

int ctx_common_init(mdc_ctx* c, int device) {
    c->device = device;
    CU_CHECK(cudaSetDevice(device));
    int v = 0;
    CU_CHECK(cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device));
    c->sm_count = v;
    CU_CHECK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
    CU_CHECK(cudaMalloc(&c->d_counters, kCounterRing * sizeof(int)));
    for (cudaEvent_t& ev : c->counter_free) CU_CHECK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    CU_CHECK(cudaMalloc(&c->d_rc, kRcFxOffset * sizeof(double) + kGstepFxScratchBytes));
    const char* e = getenv("MDC_USE_TMA");
    if (e) c->use_tma = atoi(e);
    e = getenv("MDC_CTAS_PER_SM");
    if (e) c->ctas_per_sm = atoi(e);
    e = getenv("MDC_CHUNK_FRAMES");
    if (e) c->chunk_frames = atoi(e);
    e = getenv("MDC_TMA_STAGES");
    if (e) c->tma_stages = atoi(e);
    e = getenv("MDC_TEX_TILES");
    if (e) c->tex_tiles_per_cta = std::max(1, atoi(e));
    e = getenv("MDC_TEX_PREFETCH");
    if (e) c->tex_prefetch = atoi(e) != 0;
    e = getenv("MDC_K1_STUDY");
    if (e) c->k1_study = atoi(e) & kStudyAll;
    e = getenv("MDC_AUTO_HYBRID");
    if (e) c->auto_hybrid = atoi(e) != 0;
    e = getenv("MDC_K1_CARVEOUT");
    if (e) c->carveout = std::max(0, std::min(100, atoi(e)));
    e = getenv("MDC_HYB_TEX_PCT");
    if (e) c->hyb_tex_pct = std::max(0, std::min(100, atoi(e)));
    e = getenv("MDC_HYB_STG_CTAS");
    if (e) c->hyb_stg_ctas = std::max(1, atoi(e));
    cudaDeviceProp prop;
    CU_CHECK(cudaGetDeviceProperties(&prop, device));
    // texture gather has its own (smaller) size limit; pitch-2D linear textures have one too
    c->tex_max_width = std::min(prop.maxTexture2DGather[0], prop.maxTexture2DLinear[0]);
    c->tex_max_rows = std::min(prop.maxTexture2DGather[1], prop.maxTexture2DLinear[1]);
    e = getenv("MDC_TEX_MAX_ROWS");
    if (e) c->tex_max_rows = atoi(e);
    c->tex_pitch_align = static_cast<int>(prop.texturePitchAlignment);
    c->tex_base_align = static_cast<int>(prop.textureAlignment);
    return MDC_OK;
}

// TMA needs 16-byte aligned rows and frames (tensor-map strides), the LDG loader takes anything
bool tma_pitch_ok(const mdc_ctx* c, const uint8_t* frames, int pitch) {
    return c->plan_tma_ok && pitch % 16 == 0 && (static_cast<long long>(pitch) * c->in_h) % 16 == 0 && reinterpret_cast<uintptr_t>(frames) % 16 == 0;
}

// ---- texture-gather loader plumbing -------------------------------------------------------------------------------
bool tex_pitch_ok(const mdc_ctx* c, int pitch) { return pitch % c->tex_pitch_align == 0; }

// Frames per chunk (= per texture object) for `frames`: as many as the gather height limit allows (at most the schedule chunk of
// MDC_CHUNK_FRAMES), such that every chunk starts on a texture-aligned address.  0 = this geometry / pointer cannot use the texture path.
int tex_chunk_frames(const mdc_ctx* c, const uint8_t* frames, int pitch) {
    const int want = c->chunk_frames > 0 ? c->chunk_frames : 48;
    if (!tex_pitch_ok(c, pitch) || c->in_w > c->tex_max_width || c->in_h < 2) return 0;
    if (reinterpret_cast<uintptr_t>(frames) % static_cast<uintptr_t>(c->tex_base_align) != 0) return 0;
    const long long frame_bytes = static_cast<long long>(pitch) * c->in_h;
    for (int n = std::min(want, c->tex_max_rows / c->in_h); n >= 1; --n)
        if ((frame_bytes * n) % c->tex_base_align == 0) return n;
    return 0;
}

void tex_release(TexCache::Slot& s) {
    for (cudaTextureObject_t t : s.set) cudaDestroyTextureObject(t);
    s.set.clear();
    s.key = FramesKey();
}

// texture objects for `frames` ([n_frames][H][W] u8) cut into chunks of `chunk` frames; cached on the host
int get_textures(mdc_ctx* c, const uint8_t* frames, int pitch, int n_frames, int chunk, const std::vector<cudaTextureObject_t>** out) {
    const FramesKey key{frames, n_frames, pitch, chunk};
    if ((*out = c->tex_cache.find(key))) return MDC_OK;
    TexCache::Slot& s = c->tex_cache.take();
    if (!s.set.empty()) {              // evicting: a launch that still reads these objects may be in flight on any stream
        CU_CHECK(cudaDeviceSynchronize());
        tex_release(s);
    }
    const int n_chunks = (n_frames + chunk - 1) / chunk;
    const size_t frame_bytes = static_cast<size_t>(pitch) * c->in_h;
    for (int k = 0; k < n_chunks; ++k) {
        const int nf = std::min(chunk, n_frames - k * chunk);
        cudaResourceDesc rd = {};
        rd.resType = cudaResourceTypePitch2D;
        rd.res.pitch2D.devPtr = const_cast<uint8_t*>(frames) + static_cast<size_t>(k) * chunk * frame_bytes;
        rd.res.pitch2D.desc = cudaCreateChannelDesc(8, 0, 0, 0, cudaChannelFormatKindUnsigned);
        rd.res.pitch2D.width = static_cast<size_t>(c->in_w);
        rd.res.pitch2D.height = static_cast<size_t>(c->in_h) * nf;
        rd.res.pitch2D.pitchInBytes = static_cast<size_t>(pitch);
        cudaTextureDesc td = {};      // unnormalised coordinates
        td.addressMode[0] = td.addressMode[1] = td.addressMode[2] = cudaAddressModeClamp;
        td.filterMode = cudaFilterModePoint;
        td.readMode = cudaReadModeElementType;
        cudaTextureObject_t t = 0;
        cudaError_t err = cudaCreateTextureObject(&t, &rd, &td, nullptr);
        if (err != cudaSuccess) {
            mdc_set_error("cudaCreateTextureObject failed: %s (chunk %d, %d x %d rows)", cudaGetErrorString(err), k, c->in_w, c->in_h * nf);
            tex_release(s);
            return MDC_ERR_CUDA;
        }
        s.set.push_back(t);
    }
    s.key = key;
    *out = &s.set;
    return MDC_OK;
}

// descriptors for `frames` ([n_frames][H][W] u8): one per box class; encoded sets are cached on the host
int get_tensor_maps(mdc_ctx* c, const uint8_t* frames, int pitch, int n_frames, const TmaMaps** out) {
    const FramesKey key{frames, n_frames, pitch, 0};
    if (TmaMaps* const* hit = c->map_cache.find(key)) { *out = *hit; return MDC_OK; }
    EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) { mdc_set_error("cuTensorMapEncodeTiled unavailable"); return MDC_ERR_CUDA; }
    MapCache::Slot& s = c->map_cache.take();
    if (!s.set) {
        void* mem = nullptr;
        if (posix_memalign(&mem, 64, sizeof(TmaMaps)) != 0) { mdc_set_error("out of memory"); return MDC_ERR_CUDA; }
        memset(mem, 0, sizeof(TmaMaps));
        s.set = static_cast<TmaMaps*>(mem);
    }
    s.key = FramesKey();
    for (size_t i = 0; i < c->classes.size(); ++i) {
        const cuuint64_t dims[3] = {static_cast<cuuint64_t>(c->in_w), static_cast<cuuint64_t>(c->in_h), static_cast<cuuint64_t>(n_frames)};
        const cuuint64_t strides[2] = {static_cast<cuuint64_t>(pitch), static_cast<cuuint64_t>(pitch) * c->in_h};
        const cuuint32_t box[3] = {static_cast<cuuint32_t>(c->classes[i].first), static_cast<cuuint32_t>(c->classes[i].second), 1u};
        const cuuint32_t estr[3] = {1u, 1u, 1u};
        CUresult r = enc(&s.set->m[i], CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<uint8_t*>(frames), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) { mdc_set_error("cuTensorMapEncodeTiled failed (%d) for box %u x %u", (int)r, box[0], box[1]); return MDC_ERR_CUDA; }
    }
    s.key = key;
    *out = s.set;
    return MDC_OK;
}

struct UnmapFlags { bool gamma, vig, kill; };

// flag sanitising of unMapImage, PhotometricUndistorter.cpp:173-189
UnmapFlags sanitise(const mdc_ctx* c, unsigned flags) {
    UnmapFlags u{(flags & MDC_REMOVE_GAMMA) != 0, (flags & MDC_REMOVE_VIGNETTE) != 0, (flags & MDC_NAN_OVEREXPOSED) != 0};
    if (!c->have_gamma && u.gamma) {
        printf("Photometric Undistorter did not load Gamma correctly. correctly. Not undoing gamma!\n");
        u.gamma = false;
    }
    if (!c->have_vig && u.vig) {
        printf("Photometric Undistorter did not load Vignette correctly. correctly. Not undoing Vignette!\n");
        u.vig = false;
    }
    if (!u.gamma && u.vig) {
        printf("it doesn't make sense to undo vignette without undoing gamma! not doing neither.\n");
        u.vig = false; u.gamma = false;
    }
    return u;
}

// The level buffers of one call: the caller's, of element type `type` (MDC_OUT_*), and for a narrow type the fp32 copies of the
// levels a K2 pass reads (f32[l]; nullptr where no pass reads level l).  px[l] = pixels per frame of level l.
struct Outs {
    int type = MDC_OUT_F32;
    void* lv[MDC_MAX_PYR_LEVELS] = {};
    float* f32[MDC_MAX_PYR_LEVELS] = {};
    size_t px[MDC_MAX_PYR_LEVELS] = {};
    // fp32 source of a K2 pass that reads level l
    const float* src(int l) const { return type == MDC_OUT_F32 ? static_cast<const float*>(lv[l]) : f32[l]; }
    // the same levels from frame f0 on
    Outs from(size_t f0) const {
        Outs o = *this;
        for (int l = 0; l < MDC_MAX_PYR_LEVELS; ++l) {
            if (lv[l]) o.lv[l] = static_cast<uint8_t*>(lv[l]) + f0 * px[l] * mdc_out_elem_size(type);
            if (f32[l]) o.f32[l] = f32[l] + f0 * px[l];
        }
        return o;
    }
};
Outs f32_outs(float* const* levels, int n, const mdc_ctx* c) {       // rectified fp32 levels (context-internal callers)
    Outs o;
    for (int l = 0; l < n; ++l) { o.lv[l] = levels[l]; o.px[l] = static_cast<size_t>(c->out_w >> l) * (c->out_h >> l); }
    return o;
}

// Levels that a K2 pass reads (need[l] = 1), for `levels` levels of which the first `first_k2` come from K1 (rectifying mode: 3,
// or fewer) or from unmap_kernel (non-rectifying mode: 1).  The K2 chain behind K1 goes two levels per launch, from levels 2, 4, 6;
// in non-rectifying mode every level is read by the next one.
void k2_sources(bool rectify, int levels, bool need[MDC_MAX_PYR_LEVELS]) {
    for (int l = 0; l < MDC_MAX_PYR_LEVELS; ++l) need[l] = false;
    if (!rectify) {
        for (int l = 0; l + 1 < levels; ++l) need[l] = true;
        return;
    }
    for (int l = std::min(levels, kInKernelLevels); l < levels; l += 2) need[l - 1] = true;
}

// levels beyond the fused epilogue: stand-alone K2 chain, two levels per launch where possible
int run_deep_levels(mdc_ctx* c, int n_frames, const Outs& o, int in_kernel, int levels, cudaStream_t stream, long long& launches) {
    for (int l = in_kernel; l < levels;) {
        const int sw = c->out_w >> (l - 1), sh = c->out_h >> (l - 1);
        if (l + 1 < levels) {
            CU_CHECK(launch_pyr_down2(o.src(l - 1), sw, sh, o.lv[l], o.lv[l + 1], o.type, o.f32[l + 1], n_frames, stream));
            l += 2;
        } else {
            CU_CHECK(launch_pyr_down(o.src(l - 1), sw, sh, o.lv[l], o.type, nullptr, n_frames, stream));
            l += 1;
        }
        launches++;
    }
    return MDC_OK;
}

// The FusedParams fields of every K1 launch, for n_frames frames from `frames` into levels 0..in_kernel-1 of `outs`.  Everything
// else starts zeroed (unused_, lw / lh past in_kernel, the loader's own fields), so equal calls pass equal parameter bytes.
void fused_params(FusedParams& p, const mdc_ctx* c, const uint8_t* frames, int pitch, int n_frames, UnmapFlags u, const Outs& outs,
                  int in_kernel) {
    memset(&p, 0, sizeof p);
    p.frames = frames; p.n_frames = n_frames;
    p.in_w = c->in_w; p.in_h = c->in_h; p.out_w = c->out_w; p.out_h = c->out_h; p.in_pitch = pitch;
    p.remap_x = c->d_rx; p.remap_y = c->d_ry; p.vinv = c->d_vinv; p.ginv = c->d_ginv;
    p.tiles = c->d_tiles;
    p.tiles_x = c->tiles_x; p.n_tiles = static_cast<int>(c->tiles.size());
    p.levels = in_kernel;
    for (int l = 0; l < in_kernel; ++l) { p.out[l] = outs.lv[l]; p.lw[l] = c->out_w >> l; p.lh[l] = c->out_h >> l; }
    p.level2_f32 = outs.f32[2];
    p.lut_gamma = u.gamma; p.use_vig = u.vig; p.kill = u.kill;
    p.carveout = c->carveout;
}

// K1 through the texture-gather loader, levels 0..in_kernel-1.  One launch covers up to kMaxTex chunks (= texture objects).
int run_fused_tex(mdc_ctx* c, const uint8_t* d_frames, int pitch, int n_frames, int chunk, UnmapFlags u, const Outs& outs, int in_kernel,
                  int study, cudaStream_t stream, long long& launches) {
    const std::vector<cudaTextureObject_t>* objs = nullptr;
    int rc = get_textures(c, d_frames, pitch, n_frames, chunk, &objs);
    if (rc != MDC_OK) return rc;
    const int n_chunks = static_cast<int>(objs->size());
    const int min_ctas = c->ctas_per_sm > 0 ? std::min(std::max(c->ctas_per_sm, 2), 4) : 3;
    for (int c0 = 0; c0 < n_chunks; c0 += kMaxTex) {
        const int nc = std::min(kMaxTex, n_chunks - c0);
        const int f0 = c0 * chunk, nf = std::min(n_frames - f0, nc * chunk);
        FusedParams p;
        fused_params(p, c, d_frames + static_cast<size_t>(f0) * pitch * c->in_h, pitch, nf, u, outs.from(static_cast<size_t>(f0)), in_kernel);
        p.chunk_frames = chunk;
        p.tiles_per_cta = c->tex_tiles_per_cta;
        TexSet texs;
        memset(&texs, 0, sizeof texs);
        for (int k = 0; k < nc; ++k) texs.tex[k] = (*objs)[c0 + k];
        CU_CHECK(launch_fused_tex(p, texs, nc, min_ctas, c->tex_prefetch != 0, study, outs.type, stream));
        launches++;
    }
    return MDC_OK;
}

// What "auto" resolves to (order measured on H100 at 1280x1024: TMA ahead of hybrid and texture gather, DESIGN.md §7); a loader that turns out unusable for a particular
// frames pointer falls back to the next one.
int auto_loader(const mdc_ctx* c, const uint8_t* frames, int pitch) {
    const bool tma = tma_pitch_ok(c, frames, pitch);
    if (c->tex_ok && tma && c->auto_hybrid) return 3;
    if (tma) return 1;
    if (c->tex_ok) return 2;
    return 0;
}

// K1 through a staged loader, the TMA ring (tma) or the LDG double buffer, levels 0..in_kernel-1.  cap_per_sm > 0 bounds the
// persistent grid (hybrid mode leaves room for the texture kernel's CTAs on every SM).
int run_fused_staged(mdc_ctx* c, const uint8_t* d_frames, int pitch, int n_frames, UnmapFlags u, const Outs& outs, int in_kernel, bool tma,
                     int cap_per_sm, int study, cudaStream_t stream, long long& launches) {
    FusedParams p;
    fused_params(p, c, d_frames, pitch, n_frames, u, outs, in_kernel);
    // A counter is zeroed and then drawn from by the launch that takes it.  The launch that took the slot last may still run on
    // another caller stream, so the zeroing waits for it; on one stream that wait is already satisfied.
    const unsigned slot = c->counter_next++ % kCounterRing;
    p.work_counter = c->d_counters + slot;
    CU_CHECK(cudaStreamWaitEvent(stream, c->counter_free[slot], 0));
    CU_CHECK(cudaMemsetAsync(p.work_counter, 0, sizeof(int), stream));
    p.box_px_max = c->box_px_max;
    p.chunk_frames = c->chunk_frames > 0 ? c->chunk_frames : 48;
    const TmaMaps* maps = nullptr;
    if (tma) {
        int rc = get_tensor_maps(c, d_frames, pitch, n_frames, &maps);
        if (rc != MDC_OK) return rc;
    }
    // Register budget / residency the kernel variant was compiled for (H100, DESIGN.md §7): 3 CTAs/SM (72 registers, no spills)
    // for the plain variant, as fast as 2 within run-to-run spread; the pyramid variant spills at 3 CTAs/SM and is faster
    // spill-free at 2 CTAs/SM (96 registers) with a deeper ring.
    const int min_ctas = cap_per_sm > 0 ? 3 : c->ctas_per_sm > 0 ? (c->ctas_per_sm <= 2 ? 2 : 3) : (in_kernel > 1 ? 2 : 3);
    p.tma_stages = c->tma_stages > 0 ? std::min(std::max(c->tma_stages, 2), kMaxStages) : fused_tma_stages(p.box_px_max, min_ctas);
    int per_sm = fused_max_ctas_per_sm(p.box_px_max, tma ? p.tma_stages : kLdgStages, tma, u.vig, in_kernel > 1, min_ctas, outs.type);
    if (per_sm < 1) { mdc_set_error("fused kernel does not fit on an SM (box %d px)", p.box_px_max); return MDC_ERR_CUDA; }
    if (c->ctas_per_sm > 0) per_sm = std::min(per_sm, c->ctas_per_sm);
    if (cap_per_sm > 0) per_sm = std::min(per_sm, cap_per_sm);
    const long long items = static_cast<long long>(p.n_tiles) * ((n_frames + p.chunk_frames - 1) / p.chunk_frames);
    int grid = static_cast<int>(std::min<long long>(static_cast<long long>(per_sm) * c->sm_count, std::max<long long>(items, 1)));
    if (study != kStudyAll && tma && u.vig && in_kernel == 1 && min_ctas == 3 && outs.type == MDC_OUT_F32)
        CU_CHECK(launch_fused_study(p, maps, grid, study, stream));
    else CU_CHECK(launch_fused(p, maps, grid, min_ctas, outs.type, stream));
    CU_CHECK(cudaEventRecord(c->counter_free[slot], stream));
    launches++;
    return MDC_OK;
}

// Hybrid: the batch is split between the two kernels, which run CONCURRENTLY on every SM — the staged kernel (taps, look-ups and
// stores on the LSU / shared-memory pipe) with a reduced persistent grid, and the texture-gather kernel (taps on the TEX pipe) in
// the register / shared-memory space that is left.  The idea is that the two pipes add up; on H100 it is
// slower than the TMA kernel alone (DESIGN.md §7), so `auto` picks it only on request (MDC_AUTO_HYBRID).
// The leading n_tex frames go to the texture kernel, the rest to the TMA kernel; fork/join with events around an auxiliary stream.
int run_fused_hybrid(mdc_ctx* c, const uint8_t* d_frames, int pitch, int n_frames, int n_tex, int chunk, UnmapFlags u, const Outs& outs,
                     int in_kernel, int study, cudaStream_t stream, long long& launches) {
    if (!c->aux_stream) {
        CU_CHECK(cudaStreamCreateWithFlags(&c->aux_stream, cudaStreamNonBlocking));
        CU_CHECK(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
        CU_CHECK(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
    }
    CU_CHECK(cudaEventRecord(c->ev_fork, stream));
    CU_CHECK(cudaStreamWaitEvent(c->aux_stream, c->ev_fork, 0));
    // staged kernel first: its persistent CTAs take their slots on every SM, the texture kernel's short CTAs fill what is left
    int rc = run_fused_staged(c, d_frames + static_cast<size_t>(n_tex) * pitch * c->in_h, pitch, n_frames - n_tex, u,
                              outs.from(static_cast<size_t>(n_tex)), in_kernel, true, c->hyb_stg_ctas, study, stream, launches);
    if (rc != MDC_OK) return rc;
    rc = run_fused_tex(c, d_frames, pitch, n_tex, chunk, u, outs, in_kernel, study, c->aux_stream, launches);
    if (rc != MDC_OK) return rc;
    CU_CHECK(cudaEventRecord(c->ev_join, c->aux_stream));
    CU_CHECK(cudaStreamWaitEvent(stream, c->ev_join, 0));
    return MDC_OK;
}

// What one K1 call runs: `loader` (MDC_LOADER_*), for the texture and hybrid loaders the frames per texture object (`chunk`), and
// for the hybrid loader the leading frames the texture kernel takes (`n_tex`); or, where `refusal` is set, why the call cannot run.
struct K1Route { int loader, chunk, n_tex; const char* refusal; };

// The loader rule.  `loader` is the call's own request (only the self-check makes one), or -1 for the context's setting
// (mdc_ctx_configure / MDC_USE_TMA; -1 = auto_loader).  A texture or hybrid loader set on the context refuses a call it cannot
// serve; "auto" and the self-check fall back to TMA instead, or to LDG where TMA cannot describe the frames either.
K1Route route_k1(const mdc_ctx* c, const uint8_t* frames, int pitch, int n_frames, int loader) {
    const bool forced_tex = loader < 0 && c->use_tma >= 2;
    if (loader < 0) loader = c->use_tma;
    if (loader < 0) loader = auto_loader(c, frames, pitch);
    const bool tma = tma_pitch_ok(c, frames, pitch);
    const K1Route staged{tma ? MDC_LOADER_TMA : MDC_LOADER_LDG, 0, 0, nullptr};
    const auto refuse = [](const char* why) { return K1Route{MDC_LOADER_LDG, 0, 0, why}; };
    if (loader == MDC_LOADER_LDG) return K1Route{MDC_LOADER_LDG, 0, 0, nullptr};
    if (loader == MDC_LOADER_TMA && !tma) return refuse("TMA loader requested but unusable for this geometry/pointer");
    if (loader != MDC_LOADER_TEX && loader != MDC_LOADER_HYBRID) return staged;
    if (forced_tex && !c->tex_ok) return refuse("texture-gather loader requested, but its self-check did not pass on this device / geometry");
    const int chunk = tex_chunk_frames(c, frames, pitch);
    if (chunk == 0) return forced_tex ? refuse("texture-gather loader requested but unusable for this geometry/pointer") : staged;
    if (loader == MDC_LOADER_TEX) return K1Route{MDC_LOADER_TEX, chunk, 0, nullptr};
    // hybrid: the texture kernel takes the leading hyb_tex_pct percent of the chunks
    const int n_chunks = (n_frames + chunk - 1) / chunk;
    const int tex_chunks = std::max(0, std::min(static_cast<int>((static_cast<long long>(n_chunks) * c->hyb_tex_pct + 50) / 100), n_chunks));
    const int n_tex = std::min(n_frames, tex_chunks * chunk);
    if (n_tex == n_frames) return K1Route{MDC_LOADER_TEX, chunk, 0, nullptr};
    if (n_tex == 0 || !tma) return staged;
    return K1Route{MDC_LOADER_HYBRID, chunk, n_tex, nullptr};
}

// K1 and the K2 chain behind it, through the loader route_k1 picks for `loader` (-1 = the context's setting), with the floor-study
// bits `study`; every launch is counted in `launches`.  pitch = bytes between input rows (0 = tightly packed).
int run_fused(mdc_ctx* c, const uint8_t* d_frames, int pitch, int n_frames, UnmapFlags u, const Outs& outs, int levels, cudaStream_t stream,
              int loader, int study, long long& launches) {
    if (pitch <= 0) pitch = c->in_w;
    const K1Route r = route_k1(c, d_frames, pitch, n_frames, loader);
    if (r.refusal) { mdc_set_error("%s", r.refusal); return MDC_ERR_UNSUPPORTED; }
    const int in_kernel = std::min(levels, kInKernelLevels);
    const int rc =
        r.loader == MDC_LOADER_TEX    ? run_fused_tex(c, d_frames, pitch, n_frames, r.chunk, u, outs, in_kernel, study, stream, launches)
        : r.loader == MDC_LOADER_HYBRID ? run_fused_hybrid(c, d_frames, pitch, n_frames, r.n_tex, r.chunk, u, outs, in_kernel, study, stream, launches)
        : run_fused_staged(c, d_frames, pitch, n_frames, u, outs, in_kernel, r.loader == MDC_LOADER_TMA, 0, study, stream, launches);
    return rc != MDC_OK ? rc : run_deep_levels(c, n_frames, outs, in_kernel, levels, stream, launches);
}

// Self-check of the texture-gather loader, run once per context: K1 over three synthetic frames (all byte values, saturated
// pixels, NaN flag on) through the texture path and through the staged (TMA) or LDG path; the texture path is used by default
// only if the two outputs are bit-identical.  This pins the two things the CUDA documentation does not promise for this use —
// texture gather on pitch-linear memory and the order of the four returned texels — on the device the context lives on.
void tex_selfcheck(mdc_ctx* c) {
    c->tex_ok = false;
    const char* e = getenv("MDC_USE_TEX");
    const bool verbose = getenv("MDC_VERBOSE") != nullptr;
    if (e && atoi(e) == 0) return;
    if (!c->have_fov || c->tiles.empty()) return;
    const int nf = 3;
    const size_t n_in = static_cast<size_t>(c->in_w) * c->in_h, n_out = static_cast<size_t>(c->out_w) * c->out_h;
    uint8_t* raw = nullptr;
    float *out_a = nullptr, *out_b = nullptr;
    unsigned long long* d_bad = nullptr;
    auto cleanup = [&]() { cudaFree(raw); cudaFree(out_a); cudaFree(out_b); cudaFree(d_bad); cudaGetLastError(); };
    // rows padded to the texture pitch alignment when the width itself is not describable (the check is about the device's texture
    // gather semantics; whether a particular call can use the loader is decided from its own pointer and pitch)
    const int pitch = (c->in_w + c->tex_pitch_align - 1) / c->tex_pitch_align * c->tex_pitch_align;
    if (cudaMalloc(&raw, static_cast<size_t>(nf) * pitch * c->in_h + 1024) != cudaSuccess || cudaMalloc(&out_a, nf * n_out * 4) != cudaSuccess ||
        cudaMalloc(&out_b, nf * n_out * 4) != cudaSuccess || cudaMalloc(&d_bad, 8) != cudaSuccess) { cleanup(); return; }
    uint8_t* frames = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 511) & ~static_cast<uintptr_t>(511));
    const int chunk = tex_chunk_frames(c, frames, pitch);
    if (chunk < 1) { if (verbose) fprintf(stderr, "[mdc] texture-gather loader: geometry not describable (pitch %d, limit %d rows)\n", c->in_w, c->tex_max_rows); cleanup(); return; }
    std::vector<uint8_t> h(nf * n_in);
    uint32_t lcg = 12345u;
    for (size_t i = 0; i < h.size(); ++i) { lcg = lcg * 1664525u + 1013904223u; h[i] = static_cast<uint8_t>(lcg >> 24); }
    for (size_t i = 0; i < h.size(); i += 97) h[i] = 255;
    bool ok = cudaMemcpy2D(frames, static_cast<size_t>(pitch), h.data(), static_cast<size_t>(c->in_w), static_cast<size_t>(c->in_w),
                           static_cast<size_t>(c->in_h) * nf, cudaMemcpyHostToDevice) == cudaSuccess &&
              cudaMemset(out_a, 0xff, nf * n_out * 4) == cudaSuccess && cudaMemset(out_b, 0, nf * n_out * 4) == cudaSuccess &&
              cudaMemset(d_bad, 0, 8) == cudaSuccess;
    const UnmapFlags u{c->have_gamma, c->have_gamma && c->have_vig, true};
    // its own loader requests (MDC_USE_TMA=2/3 would refuse the texture loader while tex_ok is still false), all study bits (the
    // floor-study variants compute garbage by design), and its own launch count (the context's counts the caller's launches only)
    long long launches = 0;
    ok = ok && run_fused(c, frames, pitch, nf, u, f32_outs(&out_a, 1, c), 1, c->stream, MDC_LOADER_TEX, kStudyAll, launches) == MDC_OK;
    const bool tma_ref = tma_pitch_ok(c, frames, pitch);
    ok = ok && run_fused(c, frames, pitch, nf, u, f32_outs(&out_b, 1, c), 1, c->stream, tma_ref ? MDC_LOADER_TMA : MDC_LOADER_LDG, kStudyAll,
                         launches) == MDC_OK;
    ok = ok && launch_count_mismatch(out_a, out_b, nf * n_out, d_bad, c->stream) == cudaSuccess;
    unsigned long long bad = ~0ull;
    ok = ok && cudaMemcpyAsync(&bad, d_bad, 8, cudaMemcpyDeviceToHost, c->stream) == cudaSuccess && cudaStreamSynchronize(c->stream) == cudaSuccess;
    for (auto& s : c->tex_cache.slots) if (std::get<0>(s.key) == frames) tex_release(s);
    c->tex_ok = ok && bad == 0;
    if (verbose || (ok && bad != 0))
        fprintf(stderr, "[mdc] texture-gather loader self-check: %s (%llu of %zu output words differ from the %s loader; chunk = %d frames)\n",
                c->tex_ok ? "bit-identical, enabled" : "DISABLED", ok ? bad : 0ull, nf * n_out, tma_ref ? "TMA" : "LDG", chunk);
    cleanup();
}

int finish(mdc_ctx* c, mdc_stream user_stream, cudaStream_t s) {
    if (!user_stream) CU_CHECK(cudaStreamSynchronize(s));
    (void)c;
    return MDC_OK;
}

}  // namespace

// ------------------------------------------------------------------------------ context
extern "C" int mdc_ctx_create(int device, const mdc_fov* fov, const mdc_photo* photo, mdc_ctx** out) {
    if (!out) { mdc_set_error("mdc_ctx_create: out is NULL"); return MDC_ERR_INVALID_ARG; }
    *out = nullptr;
    mdc_ctx* c = new mdc_ctx();
    int rc = ctx_common_init(c, device);
    if (rc != MDC_OK) { delete c; return rc; }
    c->have_fov = fov && fov->valid;
    if (fov && fov->dims_known) { c->in_w = fov->in_w; c->in_h = fov->in_h; }
    if (c->have_fov) { c->out_w = fov->out_w; c->out_h = fov->out_h; }
    if (photo && (photo->valid_gamma || photo->valid_vignette)) {
        if (c->in_w == 0) { c->in_w = photo->w; c->in_h = photo->h; }
        if (photo->w != c->in_w || photo->h != c->in_h) {
            mdc_set_error("photometric model is %d x %d but the rectifier input is %d x %d", photo->w, photo->h, c->in_w, c->in_h);
            mdc_ctx_destroy(c);
            return MDC_ERR_INVALID_ARG;
        }
    } else if (photo && c->in_w == 0) { c->in_w = photo->w; c->in_h = photo->h; }
    c->have_gamma = photo && photo->valid_gamma;
    c->have_vig = photo && photo->valid_vignette;
    auto fail = [&](int code) { mdc_ctx_destroy(c); return code; };
#define CTX_CHECK(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { mdc_set_error("%s failed: %s", #expr, cudaGetErrorString(e__)); return fail(MDC_ERR_CUDA); } } while (0)
    if (c->have_fov) {
        const size_t nb = static_cast<size_t>(c->out_w) * c->out_h * sizeof(float);
        CTX_CHECK(cudaMalloc(&c->d_rx, nb));
        CTX_CHECK(cudaMalloc(&c->d_ry, nb));
        CTX_CHECK(cudaMemcpy(c->d_rx, fov->remap_x.data(), nb, cudaMemcpyHostToDevice));
        CTX_CHECK(cudaMemcpy(c->d_ry, fov->remap_y.data(), nb, cudaMemcpyHostToDevice));
        build_plan(c, fov->remap_x.data(), fov->remap_y.data());
        if ((rc = upload_plan(c)) != MDC_OK) return fail(rc);
    }
    if (c->have_gamma) {
        CTX_CHECK(cudaMalloc(&c->d_ginv, 256 * sizeof(float)));
        CTX_CHECK(cudaMemcpy(c->d_ginv, photo->GInv, 256 * sizeof(float), cudaMemcpyHostToDevice));
    }
    if (c->have_vig) {
        const size_t nb = static_cast<size_t>(c->in_w) * c->in_h * sizeof(float);
        CTX_CHECK(cudaMalloc(&c->d_vinv, nb));
        CTX_CHECK(cudaMemcpy(c->d_vinv, photo->vinv.data(), nb, cudaMemcpyHostToDevice));
    }
#undef CTX_CHECK
    tex_selfcheck(c);
    *out = c;
    return MDC_OK;
}

extern "C" int mdc_ctx_create_from_device_tables(int device, int in_w, int in_h, int out_w, int out_h,
                                                 const float* d_remap_x, const float* d_remap_y,
                                                 const float* d_ginv256, const float* d_vinv, mdc_ctx** out) {
    if (!out) { mdc_set_error("mdc_ctx_create_from_device_tables: out is NULL"); return MDC_ERR_INVALID_ARG; }
    *out = nullptr;
    if (in_w < 2 || in_h < 2) { mdc_set_error("bad input size"); return MDC_ERR_INVALID_ARG; }
    if (static_cast<long long>(in_w) * in_h > (1LL << 28) || (d_remap_x && (out_w < 1 || out_h < 1 || static_cast<long long>(out_w) * out_h > (1LL << 28)))) {
        mdc_set_error("image larger than 2^28 pixels");      // same limit as the table builders and the image decoders
        return MDC_ERR_INVALID_ARG;
    }
    if ((d_remap_x == nullptr) != (d_remap_y == nullptr)) { mdc_set_error("remap tables must come as a pair"); return MDC_ERR_INVALID_ARG; }
    mdc_ctx* c = new mdc_ctx();
    int rc = ctx_common_init(c, device);
    if (rc != MDC_OK) { delete c; return rc; }
    c->owns_tables = false;
    c->in_w = in_w; c->in_h = in_h;
    c->have_fov = d_remap_x != nullptr;
    c->have_gamma = d_ginv256 != nullptr;
    c->have_vig = d_vinv != nullptr;
    c->d_rx = const_cast<float*>(d_remap_x); c->d_ry = const_cast<float*>(d_remap_y);
    c->d_ginv = const_cast<float*>(d_ginv256); c->d_vinv = const_cast<float*>(d_vinv);
    if (c->have_fov) {
        if (out_w < 1 || out_h < 1) { mdc_set_error("bad output size"); mdc_ctx_destroy(c); return MDC_ERR_INVALID_ARG; }
        c->out_w = out_w; c->out_h = out_h;
        const size_t n = static_cast<size_t>(out_w) * out_h;
        std::vector<float> hx(n), hy(n);
        cudaError_t e = cudaMemcpy(hx.data(), d_remap_x, n * sizeof(float), cudaMemcpyDeviceToHost);
        if (e == cudaSuccess) e = cudaMemcpy(hy.data(), d_remap_y, n * sizeof(float), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) { mdc_set_error("reading back remap tables failed: %s", cudaGetErrorString(e)); mdc_ctx_destroy(c); return MDC_ERR_CUDA; }
        if ((rc = check_table_domain(hx.data(), hy.data(), out_w, out_h, in_w, in_h)) != MDC_OK) { mdc_ctx_destroy(c); return rc; }
        build_plan(c, hx.data(), hy.data());
        if ((rc = upload_plan(c)) != MDC_OK) { mdc_ctx_destroy(c); return rc; }
    }
    tex_selfcheck(c);
    *out = c;
    return MDC_OK;
}

extern "C" int mdc_ctx_take_table_ownership(mdc_ctx* c) {
    if (!c) return MDC_ERR_INVALID_ARG;
    c->owns_tables = true;
    return MDC_OK;
}

extern "C" void mdc_ctx_destroy(mdc_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    if (c->stream) cudaStreamSynchronize(c->stream);
    if (c->owns_tables) { cudaFree(c->d_rx); cudaFree(c->d_ry); cudaFree(c->d_ginv); cudaFree(c->d_vinv); }
    cudaFree(c->d_tiles); cudaFree(c->d_counters); cudaFree(c->d_rc);
    for (auto& s : c->map_cache.slots) free(s.set);
    cudaDeviceSynchronize();
    for (cudaEvent_t ev : c->counter_free) if (ev) cudaEventDestroy(ev);
    for (auto& s : c->tex_cache.slots) tex_release(s);
    if (c->aux_stream) { cudaStreamDestroy(c->aux_stream); cudaEventDestroy(c->ev_fork); cudaEventDestroy(c->ev_join); }
    for (int s = 0; s < kHostPipeDepth; ++s) {
        if (c->pipe_stream[s]) { cudaStreamSynchronize(c->pipe_stream[s]); cudaStreamDestroy(c->pipe_stream[s]); }
        cudaFree(c->pipe_in[s]); cudaFree(c->pipe_out[s]);
    }
    cudaFree(c->scratch_a); cudaFree(c->scratch_b);
    if (c->f32_pool) cudaMemPoolDestroy(c->f32_pool);
    if (c->stream) cudaStreamDestroy(c->stream);
    delete c;
}

extern "C" int mdc_ctx_device_tables(const mdc_ctx* c, const float** rx, const float** ry, const float** ginv, const float** vinv) {
    if (!c) return MDC_ERR_INVALID_ARG;
    if (rx) *rx = c->d_rx;
    if (ry) *ry = c->d_ry;
    if (ginv) *ginv = c->d_ginv;
    if (vinv) *vinv = c->d_vinv;
    return MDC_OK;
}

extern "C" int mdc_ctx_level_dims(const mdc_ctx* c, int level, int* w, int* h) {
    if (!c || level < 0 || level >= MDC_MAX_PYR_LEVELS) return MDC_ERR_INVALID_ARG;
    if (w) *w = c->out_w >> level;
    if (h) *h = c->out_h >> level;
    return MDC_OK;
}

extern "C" long long mdc_ctx_launch_count(const mdc_ctx* c) { return c ? c->launches : 0; }

extern "C" int mdc_ctx_configure(mdc_ctx* c, int use_tma, int ctas_per_sm) {
    if (!c || use_tma < -1 || use_tma > 3) return MDC_ERR_INVALID_ARG;
    c->use_tma = use_tma;
    c->ctas_per_sm = ctas_per_sm;
    return MDC_OK;
}

static bool pitch_valid(const mdc_ctx* c, size_t row_pitch_bytes) {
    return c && c->have_fov && row_pitch_bytes >= static_cast<size_t>(c->in_w) && row_pitch_bytes <= (1u << 30);
}

extern "C" int mdc_ctx_auto_loader_pitched(const mdc_ctx* c, size_t row_pitch_bytes) {
    return pitch_valid(c, row_pitch_bytes) ? auto_loader(c, nullptr, static_cast<int>(row_pitch_bytes)) : 0;
}
extern "C" int mdc_ctx_auto_loader(const mdc_ctx* c) { return c ? mdc_ctx_auto_loader_pitched(c, static_cast<size_t>(c->in_w)) : 0; }

extern "C" int mdc_ctx_loader_usable_pitched(const mdc_ctx* c, int loader, size_t row_pitch_bytes) {
    if (!pitch_valid(c, row_pitch_bytes)) return 0;
    const int pitch = static_cast<int>(row_pitch_bytes);
    switch (loader) {
        case MDC_LOADER_LDG: return 1;
        case MDC_LOADER_TMA: return tma_pitch_ok(c, nullptr, pitch) ? 1 : 0;
        case MDC_LOADER_TEX: return (c->tex_ok && tex_pitch_ok(c, pitch)) ? 1 : 0;
        case MDC_LOADER_HYBRID: return (c->tex_ok && tex_pitch_ok(c, pitch) && tma_pitch_ok(c, nullptr, pitch)) ? 1 : 0;
        default: return 0;
    }
}
extern "C" int mdc_ctx_loader_usable(const mdc_ctx* c, int loader) {      // for tightly packed frames
    return c ? mdc_ctx_loader_usable_pitched(c, loader, static_cast<size_t>(c->in_w)) : 0;
}

// --------------------------------------------------------------- device-resident operators
extern "C" int mdc_unmap_u8(mdc_ctx* c, const uint8_t* d_in, float* d_out, int n, int n_frames, unsigned flags, mdc_stream stream) {
    if (!c || !d_in || !d_out || n < 0 || n_frames < 0) { mdc_set_error("mdc_unmap_u8: bad argument"); return MDC_ERR_INVALID_ARG; }
    if (n != c->in_w * c->in_h) {   // the reference only asserts this (compiled out); refuse instead of reading the vignette out of bounds
        mdc_set_error("unMapImage: expected %d pixels, got %d", c->in_w * c->in_h, n);
        return MDC_ERR_INVALID_ARG;
    }
    CU_CHECK(cudaSetDevice(c->device));
    const UnmapFlags u = sanitise(c, flags);
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    CU_CHECK(launch_unmap(d_in, d_out, MDC_OUT_F32, nullptr, static_cast<size_t>(n), n_frames, u.gamma ? c->d_ginv : nullptr,
                          u.vig ? c->d_vinv : nullptr, u.kill, s));
    c->launches++;
    return finish(c, stream, s);
}

static int check_undistort_args(mdc_ctx* c, const void* in, const void* out, int n_pix_in, int n_pix_out, int n_frames) {
    if (!c || !in || !out || n_frames < 0) { mdc_set_error("undistort: bad argument"); return MDC_ERR_INVALID_ARG; }
    if (!c->have_fov) { mdc_set_error("undistort on an invalid rectifier"); return MDC_ERR_INVALID_OBJECT; }
    if (n_pix_in != c->in_w * c->in_h) {
        printf("ERROR: undistort called with wrong input image dismesions (expected %d pixel, got %d pixel)\n", c->in_w * c->in_h, n_pix_in);
        mdc_set_error("undistort: expected %d input pixels, got %d", c->in_w * c->in_h, n_pix_in);
        return MDC_ERR_INVALID_ARG;
    }
    if (n_pix_out != c->out_w * c->out_h) {
        printf("ERROR: undistort called with wrong output image dismesions (expected %d pixel, got %d pixel)\n", c->out_w * c->out_h, n_pix_out);
        mdc_set_error("undistort: expected %d output pixels, got %d", c->out_w * c->out_h, n_pix_out);
        return MDC_ERR_INVALID_ARG;
    }
    return MDC_OK;
}

extern "C" int mdc_undistort_u8(mdc_ctx* c, const uint8_t* d_in, float* d_out, int n_pix_in, int n_pix_out, int n_frames, mdc_stream stream) {
    int rc = check_undistort_args(c, d_in, d_out, n_pix_in, n_pix_out, n_frames);
    if (rc != MDC_OK) return rc;
    if (n_frames == 0) return MDC_OK;
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    rc = run_fused(c, d_in, 0, n_frames, UnmapFlags{false, false, false}, f32_outs(&d_out, 1, c), 1, s, -1, c->k1_study, c->launches);
    if (rc != MDC_OK) return rc;
    return finish(c, stream, s);
}

extern "C" int mdc_undistort_f32(mdc_ctx* c, const float* d_in, float* d_out, int n_pix_in, int n_pix_out, int n_frames, mdc_stream stream) {
    int rc = check_undistort_args(c, d_in, d_out, n_pix_in, n_pix_out, n_frames);
    if (rc != MDC_OK) return rc;
    if (n_frames == 0) return MDC_OK;
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    CU_CHECK(launch_undistort_f32(d_in, d_out, c->in_w, n_pix_in, n_pix_out, n_frames, c->d_rx, c->d_ry, s));
    c->launches++;
    return finish(c, stream, s);
}

extern "C" int mdc_pyr_down(mdc_ctx* c, const float* d_src, int src_w, int src_h, float* d_dst, int n_frames, mdc_stream stream) {
    if (!c || !d_src || !d_dst || src_w < 0 || src_h < 0 || n_frames < 0) { mdc_set_error("mdc_pyr_down: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    CU_CHECK(launch_pyr_down(d_src, src_w, src_h, d_dst, MDC_OUT_F32, nullptr, n_frames, s));
    c->launches++;
    return finish(c, stream, s);
}

// scratch: device memory for the fp32 copies of the levels a K2 pass reads (narrow output types only), at least
// prepare_f32_scratch_bytes(...) bytes, or nullptr to allocate it from the context's pool on the call's stream.
static int prepare_batch_impl(mdc_ctx* c, const uint8_t* d_frames, int pitch, int n_frames, unsigned flags, int out_type,
                              void* const* d_out_levels, int levels, mdc_stream stream, void* scratch = nullptr);

int mdc_check_out_type(int out_type, const char* where) {
    if (out_type == MDC_OUT_F32 || out_type == MDC_OUT_F16 || out_type == MDC_OUT_U8) return MDC_OK;
    mdc_set_error("%s: unknown output type %d", where, out_type);
    return MDC_ERR_INVALID_ARG;
}

extern "C" int mdc_prepare_batch(mdc_ctx* c, const uint8_t* d_frames, int n_frames, unsigned flags,
                                 float* const* d_out_levels, int levels, mdc_stream stream) {
    return prepare_batch_impl(c, d_frames, 0, n_frames, flags, MDC_OUT_F32, reinterpret_cast<void* const*>(d_out_levels), levels, stream);
}

extern "C" int mdc_prepare_batch_pitched(mdc_ctx* c, const uint8_t* d_frames, size_t row_pitch_bytes, int n_frames, unsigned flags,
                                         float* const* d_out_levels, int levels, mdc_stream stream) {
    if (c && (row_pitch_bytes < static_cast<size_t>(c->in_w) || row_pitch_bytes > (1u << 30))) {
        mdc_set_error("mdc_prepare_batch_pitched: row pitch %zu for %d-pixel rows", row_pitch_bytes, c->in_w);
        return MDC_ERR_INVALID_ARG;
    }
    return prepare_batch_impl(c, d_frames, static_cast<int>(row_pitch_bytes), n_frames, flags, MDC_OUT_F32,
                              reinterpret_cast<void* const*>(d_out_levels), levels, stream);
}

extern "C" int mdc_prepare_batch_ex(mdc_ctx* c, const uint8_t* d_frames, size_t row_pitch_bytes, int n_frames, unsigned flags, int out_type,
                                    void* const* d_out_levels, int levels, mdc_stream stream) {
    int rc = mdc_check_out_type(out_type, "mdc_prepare_batch_ex");
    if (rc != MDC_OK) return rc;
    if (c && row_pitch_bytes != 0 && (row_pitch_bytes < static_cast<size_t>(c->in_w) || row_pitch_bytes > (1u << 30))) {
        mdc_set_error("mdc_prepare_batch_ex: row pitch %zu for %d-pixel rows", row_pitch_bytes, c->in_w);
        return MDC_ERR_INVALID_ARG;
    }
    return prepare_batch_impl(c, d_frames, static_cast<int>(row_pitch_bytes), n_frames, flags, out_type, d_out_levels, levels, stream);
}

namespace {
// Bytes of fp32 scratch a narrow-type call needs per frame (0 for MDC_OUT_F32 and wherever no K2 pass runs).
size_t prepare_f32_scratch_bytes(const mdc_ctx* c, bool rectify, int out_type, int levels) {
    if (out_type == MDC_OUT_F32) return 0;
    bool need[MDC_MAX_PYR_LEVELS];
    k2_sources(rectify, levels, need);
    size_t b = 0;
    for (int l = 0; l < levels; ++l)
        if (need[l]) b += ((static_cast<size_t>((rectify ? c->out_w : c->in_w) >> l) * ((rectify ? c->out_h : c->in_h) >> l) * 4 + 15) & ~size_t(15));
    return b;
}
int f32_pool(mdc_ctx* c, cudaMemPool_t* out) {
    if (!c->f32_pool) {     // a pool of the context's own, kept warm between calls (the release threshold keeps its memory mapped)
        cudaMemPoolProps props = {};
        props.allocType = cudaMemAllocationTypePinned;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = c->device;
        CU_CHECK(cudaMemPoolCreate(&c->f32_pool, &props));
        uint64_t keep = ~0ull;
        CU_CHECK(cudaMemPoolSetAttribute(c->f32_pool, cudaMemPoolAttrReleaseThreshold, &keep));
    }
    *out = c->f32_pool;
    return MDC_OK;
}
}  // namespace

static int prepare_batch_impl(mdc_ctx* c, const uint8_t* d_frames, int pitch, int n_frames, unsigned flags, int out_type,
                              void* const* d_out_levels, int levels, mdc_stream stream, void* scratch) {
    if (!c || !d_frames || !d_out_levels || n_frames < 0 || levels < 1 || levels > MDC_MAX_PYR_LEVELS) {
        mdc_set_error("mdc_prepare_batch: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    if (c->in_w < 1) { mdc_set_error("mdc_prepare_batch: context has no image geometry"); return MDC_ERR_INVALID_OBJECT; }
    const bool rectify = (flags & MDC_RECTIFY) != 0;
    Outs o;
    o.type = out_type;
    for (int l = 0; l < levels; ++l) {   // a level that has no pixels (tiny images) may legitimately be a NULL buffer
        const int lw = (rectify ? c->out_w : c->in_w) >> l, lh = (rectify ? c->out_h : c->in_h) >> l;
        if (!d_out_levels[l] && lw > 0 && lh > 0) { mdc_set_error("mdc_prepare_batch: output level %d is NULL", l); return MDC_ERR_INVALID_ARG; }
        o.lv[l] = d_out_levels[l];
        o.px[l] = static_cast<size_t>(lw) * lh;
    }
    if (rectify && !c->have_fov) { mdc_set_error("getImage(rectify) on an invalid rectifier"); return MDC_ERR_INVALID_OBJECT; }
    if (n_frames == 0) return MDC_OK;
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    // narrow output types: the levels a K2 pass reads are also written in fp32, to scratch, and K2 reads those
    const size_t f32_bytes = prepare_f32_scratch_bytes(c, rectify, out_type, levels) * static_cast<size_t>(n_frames);
    void* pooled = nullptr;
    if (f32_bytes > 0) {
        if (!scratch) {
            cudaMemPool_t pool;
            int rc = f32_pool(c, &pool);
            if (rc != MDC_OK) return rc;
            CU_CHECK(cudaMallocFromPoolAsync(&pooled, f32_bytes, pool, s));
            scratch = pooled;
        }
        bool need[MDC_MAX_PYR_LEVELS];
        k2_sources(rectify, levels, need);
        uint8_t* at = static_cast<uint8_t*>(scratch);
        for (int l = 0; l < levels; ++l)
            if (need[l]) { o.f32[l] = reinterpret_cast<float*>(at); at += ((o.px[l] * 4 + 15) & ~size_t(15)) * n_frames; }
    }
    int rc = MDC_OK;
    // mode switch of DatasetReader::getImage, BenchmarkDatasetReader.h:210-241
    const bool photometric = (flags & (MDC_REMOVE_GAMMA | MDC_REMOVE_VIGNETTE | MDC_NAN_OVEREXPOSED)) != 0;
    UnmapFlags u{false, false, false};
    if (photometric) u = sanitise(c, flags);
    if (rectify) {
        rc = run_fused(c, d_frames, pitch, n_frames, u, o, levels, s, -1, c->k1_study, c->launches);
    } else if (pitch > 0 && pitch != c->in_w) {
        mdc_set_error("padded rows are supported in rectifying mode only");
        rc = MDC_ERR_UNSUPPORTED;
    } else {
        rc = [&]() -> int {
            const size_t n = static_cast<size_t>(c->in_w) * c->in_h;
            CU_CHECK(launch_unmap(d_frames, o.lv[0], o.type, o.f32[0], n, n_frames, u.gamma ? c->d_ginv : nullptr, u.vig ? c->d_vinv : nullptr,
                                  u.kill, s));
            c->launches++;
            for (int l = 1; l < levels; ++l) {
                CU_CHECK(launch_pyr_down(o.src(l - 1), c->in_w >> (l - 1), c->in_h >> (l - 1), o.lv[l], o.type, o.f32[l], n_frames, s));
                c->launches++;
            }
            return MDC_OK;
        }();
    }
    if (pooled) {
        const cudaError_t e = cudaFreeAsync(pooled, s);      // stream-ordered: after the launches above
        if (rc == MDC_OK && e != cudaSuccess) { mdc_set_error("cudaFreeAsync failed: %s", cudaGetErrorString(e)); rc = MDC_ERR_CUDA; }
    }
    return rc != MDC_OK ? rc : finish(c, stream, s);
}

extern "C" int mdc_fov_distort_coordinates_device(const mdc_fov* f, float* d_x, float* d_y, size_t n, int device, mdc_stream stream) {
    if (!f || (n && (!d_x || !d_y))) { mdc_set_error("mdc_fov_distort_coordinates_device: bad argument"); return MDC_ERR_INVALID_ARG; }
    if (!f->valid) {
        printf("ERROR: invalid UndistorterFOV!\n");          // FOVUndistorter.cpp:282-286
        mdc_set_error("distortCoordinates on an invalid rectifier");
        return MDC_ERR_INVALID_OBJECT;
    }
    CU_CHECK(cudaSetDevice(device));
    mdc_distort_constants h;
    mdc_fov_distort_constants(f, &h);
    const DistortConstants k{h.ocx, h.ocy, h.ofx, h.ofy, h.d2t, h.omega, h.fx, h.fy, h.cx, h.cy};
    CU_CHECK(launch_fov_distort(d_x, d_y, n, k, static_cast<cudaStream_t>(stream)));
    if (!stream) CU_CHECK(cudaStreamSynchronize(nullptr));
    return MDC_OK;
}

extern "C" int mdc_vc_plane_maps(const mdc_fov* fov, const double* homographies, int n, int gw, int gh, float facw, float fach, float* d_p2x,
                                 float* d_p2y, int device, mdc_stream stream) {
    if (!fov || n < 0 || gw < 0 || gh < 0 || (n && (!homographies || (static_cast<size_t>(gw) * gh && (!d_p2x || !d_p2y))))) {
        mdc_set_error("mdc_vc_plane_maps: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    if (!fov->valid) {
        printf("ERROR: invalid UndistorterFOV!\n");          // distortCoordinates, FOVUndistorter.cpp:282-286
        mdc_set_error("mdc_vc_plane_maps on an invalid rectifier");
        return MDC_ERR_INVALID_OBJECT;
    }
    if (n == 0 || static_cast<size_t>(gw) * gh == 0) return MDC_OK;
    std::vector<float> hk(static_cast<size_t>(9) * n);
    for (int i = 0; i < n; ++i) mdc_vc_plane_matrix(homographies + 9 * static_cast<size_t>(i), gw, gh, facw, fach, hk.data() + 9 * static_cast<size_t>(i));
    mdc_distort_constants h;
    mdc_fov_distort_constants(fov, &h);
    const DistortConstants k{h.ocx, h.ocy, h.ofx, h.ofy, h.d2t, h.omega, h.fx, h.fy, h.cx, h.cy};
    CU_CHECK(cudaSetDevice(device));
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    float* d_hk = nullptr;
    CU_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&d_hk), hk.size() * sizeof(float), s));
    cudaError_t e = cudaMemcpyAsync(d_hk, hk.data(), hk.size() * sizeof(float), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) e = launch_vc_plane_maps(d_hk, n, gw, gh, fov->in_w, fov->in_h, k, d_p2x, d_p2y, s);
    const cudaError_t f = cudaFreeAsync(d_hk, s);
    CU_CHECK(e);
    CU_CHECK(f);
    if (!stream) CU_CHECK(cudaStreamSynchronize(nullptr));
    return MDC_OK;
}

extern "C" int mdc_atanf_device(const float* d_in, float* d_out, size_t n, int device, mdc_stream stream) {
    if (n && (!d_in || !d_out)) { mdc_set_error("mdc_atanf_device: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(device));
    CU_CHECK(launch_atanf(d_in, d_out, n, static_cast<cudaStream_t>(stream)));
    if (!stream) CU_CHECK(cudaStreamSynchronize(nullptr));
    return MDC_OK;
}

int mdc_ctx_device_ordinal(const mdc_ctx* c) { return c->device; }
void* mdc_ctx_stream_handle(mdc_ctx* c) { return c->stream; }
void mdc_ctx_add_launches(mdc_ctx* c, int n) { c->launches += n; }
int mdc_ctx_scratch_pool(mdc_ctx* c, void** pool) {
    cudaMemPool_t p = nullptr;
    const int rc = f32_pool(c, &p);
    *pool = p;
    return rc;
}
void mdc_ctx_geometry(const mdc_ctx* c, int* in_w, int* in_h, int* out_w, int* out_h) { *in_w = c->in_w; *in_h = c->in_h; *out_w = c->out_w; *out_h = c->out_h; }

extern "C" int mdc_estep(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_G, double* d_E, mdc_stream stream) {
    // an empty pixel slice (npix = 0, e.g. a rank of a pixel-sharded run) reads no data and writes no E: both may be null
    if (!c || (n > 0 && ((npix > 0 && !d_data) || !d_t)) || !d_G || (npix > 0 && !d_E) || n < 0 || npix < 0) {
        mdc_set_error("mdc_estep: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    CU_CHECK(launch_estep(d_data, n, npix, d_t, d_G, d_E, s));
    c->launches++;
    return finish(c, stream, s);
}

// ------------------------------------------------------------------ responseCalib building blocks
extern "C" int mdc_rc_leak_padding(mdc_ctx* c, uint8_t* d_data, int n, int w, int h, int iterations, mdc_stream stream) {
    if (!c || !d_data || n < 0 || w < 1 || h < 1 || iterations < 0) { mdc_set_error("mdc_rc_leak_padding: bad argument"); return MDC_ERR_INVALID_ARG; }
    if (n == 0 || iterations == 0) return MDC_OK;
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    const size_t bytes = static_cast<size_t>(n) * w * h;
    int rc = ensure_bytes(&c->scratch_a, &c->scratch_a_bytes, bytes);
    if (rc != MDC_OK) return rc;
    uint8_t* tmp = static_cast<uint8_t*>(c->scratch_a);
    for (int it = 0; it < iterations; ++it) {      // ping-pong; an odd count ends in tmp and is copied back
        const uint8_t* src = (it & 1) ? tmp : d_data;
        uint8_t* dst = (it & 1) ? d_data : tmp;
        CU_CHECK(launch_rc_leak_padding(src, dst, n, w, h, s));
        c->launches++;
    }
    if (iterations & 1) CU_CHECK(cudaMemcpyAsync(d_data, tmp, bytes, cudaMemcpyDeviceToDevice, s));
    return finish(c, stream, s);
}

extern "C" int mdc_rc_einit(mdc_ctx* c, const uint8_t* d_data, int n, int npix, double* d_E, mdc_stream stream) {
    if (!c || (n > 0 && npix > 0 && !d_data) || (npix > 0 && !d_E) || n < 0 || npix < 0) { mdc_set_error("mdc_rc_einit: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    if (npix > 0) { CU_CHECK(launch_rc_einit(d_data, n, npix, d_E, s)); c->launches++; }
    return finish(c, stream, s);
}

// reuse_counts: GNum[] (the histogram of the unsaturated samples) is still in the context's scratch from the previous G-step over
// the SAME images, so only the sums are accumulated
static int rc_gstep_impl(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_E, double* d_G, bool reuse_counts,
                         mdc_stream stream) {
    if (!c || (n > 0 && (!d_data || !d_t)) || !d_E || !d_G || n < 0 || npix < 0) { mdc_set_error("mdc_rc_gstep: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    CU_CHECK(launch_rc_gstep(d_data, n, npix, d_t, d_E, c->d_rc, reinterpret_cast<unsigned long long*>(c->d_rc + 256), d_G, reuse_counts, c->d_rc + kRcFxOffset, s));
    c->launches += 4;      // scale, accumulate, convert, finish
    return finish(c, stream, s);
}
extern "C" int mdc_rc_gstep(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_E, double* d_G, mdc_stream stream) {
    return rc_gstep_impl(c, d_data, n, npix, d_t, d_E, d_G, false, stream);
}

// ---- the two reductions of the calibrator as partials, for pixel-sharded runs (SURVEY.md §8e row 2): every rank holds its
// slice of every image ([n][npix_local]); the accumulators stay on the device so the host language's collective (NCCL all-reduce:
// 256 doubles + 256 u64 for the G-step, 2 doubles for rmse) runs on them in place.
extern "C" int mdc_rc_gstep_accumulate(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_E,
                                       double* d_gsum256, unsigned long long* d_gnum256, int reuse_counts, mdc_stream stream) {
    if (!c || !d_t || !d_gsum256 || !d_gnum256 || n < 0 || npix < 0 || (npix > 0 && n > 0 && (!d_data || !d_E))) {
        mdc_set_error("mdc_rc_gstep_accumulate: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    if (reuse_counts && npix > 0 && !rc_counts_reusable(d_data, npix)) {
        mdc_set_error("mdc_rc_gstep_accumulate: reuse_counts needs a 16-byte aligned slice of a multiple of 16 pixels");
        return MDC_ERR_UNSUPPORTED;
    }
    CU_CHECK(launch_rc_gstep_accum(d_data, n, npix, d_t, d_E, d_gsum256, d_gnum256, reuse_counts != 0, c->d_rc + kRcFxOffset, s));
    c->launches += (npix > 0 && n > 0) ? 3 : 1;      // scale, accumulate, convert
    return finish(c, stream, s);
}
// ---- the same G-step with sums that are exact ACROSS ranks (include/mdc_b200.h)
extern "C" int mdc_rc_gstep_scale(mdc_ctx* c, const double* d_E, int npix, const double* d_t, int n, unsigned long long* d_scale4, mdc_stream stream) {
    if (!c || !d_scale4 || n < 0 || npix < 0 || (npix > 0 && n > 0 && (!d_E || !d_t))) { mdc_set_error("mdc_rc_gstep_scale: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    CU_CHECK(launch_rc_gstep_scale(d_E, npix, d_t, n, d_scale4, s));
    c->launches += (npix > 0 && n > 0) ? 1 : 0;
    return finish(c, stream, s);
}
extern "C" int mdc_rc_gstep_accumulate_exact(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_E,
                                             const unsigned long long* d_scale4, long long* d_limbs768, double* d_special256,
                                             unsigned long long* d_gnum256, int reuse_counts, mdc_stream stream) {
    if (!c || !d_t || !d_scale4 || !d_limbs768 || !d_special256 || !d_gnum256 || n < 0 || npix < 0 || (npix > 0 && n > 0 && (!d_data || !d_E))) {
        mdc_set_error("mdc_rc_gstep_accumulate_exact: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    if (reuse_counts && npix > 0 && n > 0 && !rc_counts_reusable(d_data, npix)) {
        mdc_set_error("mdc_rc_gstep_accumulate_exact: reuse_counts needs a 16-byte aligned slice of a multiple of 16 pixels");
        return MDC_ERR_UNSUPPORTED;
    }
    CU_CHECK(launch_rc_gstep_accum_exact(d_data, n, npix, d_t, d_E, d_scale4, d_limbs768, d_special256, d_gnum256, reuse_counts != 0, c->d_rc + kRcFxOffset, s));
    c->launches += (npix > 0 && n > 0) ? 2 : 1;      // histogram pass, split
    return finish(c, stream, s);
}
extern "C" int mdc_rc_gstep_finish_exact(mdc_ctx* c, const unsigned long long* d_scale4, const long long* d_limbs768, const double* d_special256,
                                         const unsigned long long* d_gnum256, double* d_G, mdc_stream stream) {
    if (!c || !d_scale4 || !d_limbs768 || !d_special256 || !d_gnum256 || !d_G) { mdc_set_error("mdc_rc_gstep_finish_exact: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    CU_CHECK(launch_rc_gstep_finish_exact(d_scale4, d_limbs768, d_special256, d_gnum256, c->d_rc, d_G, s));      // d_rc[0..255]: the joined sums
    c->launches += 2;
    return finish(c, stream, s);
}
extern "C" int mdc_rc_gstep_finish(mdc_ctx* c, const double* d_gsum256, const unsigned long long* d_gnum256, double* d_G, mdc_stream stream) {
    if (!c || !d_gsum256 || !d_gnum256 || !d_G) { mdc_set_error("mdc_rc_gstep_finish: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    CU_CHECK(launch_rc_gstep_finish(d_gsum256, d_gnum256, d_G, s));
    c->launches++;
    return finish(c, stream, s);
}
extern "C" int mdc_rc_rmse_accumulate(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_G, const double* d_E,
                                      double* d_acc2, mdc_stream stream) {
    if (!c || !d_t || !d_G || !d_acc2 || n < 0 || npix < 0 || (npix > 0 && n > 0 && (!d_data || !d_E))) {
        mdc_set_error("mdc_rc_rmse_accumulate: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    CU_CHECK(cudaSetDevice(c->device));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : c->stream;
    if (npix > 0 && n > 0) { CU_CHECK(launch_rc_rmse(d_data, n, npix, d_t, d_G, d_E, d_acc2, c->d_rc + 515, s)); c->launches += 2; }
    else CU_CHECK(cudaMemsetAsync(d_acc2, 0, 2 * sizeof(double), s));
    return finish(c, stream, s);
}

extern "C" int mdc_rc_rescale(mdc_ctx* c, int npix, double* d_E, double* d_G, double* factor_host) {
    if (!c || (npix > 0 && !d_E) || !d_G || npix < 0) { mdc_set_error("mdc_rc_rescale: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(c->device));
    CU_CHECK(launch_rc_rescale(npix, d_E, d_G, c->d_rc + 512, c->stream));      // with npix = 0 the E launch touches nothing
    c->launches += 3;
    if (factor_host) CU_CHECK(cudaMemcpyAsync(factor_host, c->d_rc + 512, sizeof(double), cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    return MDC_OK;
}

extern "C" int mdc_rc_rmse(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, const double* d_G, const double* d_E, double out_host[2]) {
    if (!c || (n > 0 && (!d_data || !d_t)) || !d_G || !d_E || !out_host || n < 0 || npix < 0) { mdc_set_error("mdc_rc_rmse: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(c->device));
    CU_CHECK(launch_rc_rmse(d_data, n, npix, d_t, d_G, d_E, c->d_rc + 513, c->d_rc + 515, c->stream));
    c->launches += 2;
    double acc[2];
    CU_CHECK(cudaMemcpyAsync(acc, c->d_rc + 513, sizeof acc, cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    out_host[0] = 1e5 * sqrt(acc[0] / acc[1]);
    out_host[1] = acc[1];
    return MDC_OK;
}

extern "C" int mdc_response_calib(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, int nits, double* d_E, double* d_G, double* log_host) {
    return mdc_response_calib_ex(c, d_data, n, npix, d_t, nits, d_E, d_G, log_host, nullptr, nullptr);
}

extern "C" int mdc_response_calib_ex(mdc_ctx* c, const uint8_t* d_data, int n, int npix, const double* d_t, int nits, double* d_E, double* d_G,
                                     double* log_host, mdc_rc_step_fn step, void* user) {
    if (!c || !d_data || !d_t || !d_E || !d_G || n < 1 || npix < 1 || nits < 0) { mdc_set_error("mdc_response_calib: bad argument"); return MDC_ERR_INVALID_ARG; }
    int rc = mdc_rc_einit(c, d_data, n, npix, d_E, c->stream);          // starting irradiance = mean of all images
    if (rc != MDC_OK) return rc;
    CU_CHECK(cudaMemsetAsync(d_G, 0, 256 * sizeof(double), c->stream));
    if (step) {
        CU_CHECK(cudaStreamSynchronize(c->stream));
        step(0, MDC_RC_STEP_E, d_E, d_G, user);
    }
    for (int it = 0; it < nits; ++it) {
        double r[2], row[4] = {0, 0, 0, 0};
        if ((rc = rc_gstep_impl(c, d_data, n, npix, d_t, d_E, d_G, /*reuse_counts=*/it > 0, c->stream)) != MDC_OK) return rc;
        if ((rc = mdc_rc_rmse(c, d_data, n, npix, d_t, d_G, d_E, r)) != MDC_OK) return rc;
        row[0] = r[0];
        printf("optG RMSE = %f! \t", r[0]);
        if (step) step(it + 1, MDC_RC_STEP_G, d_E, d_G, user);
        if ((rc = mdc_estep(c, d_data, n, npix, d_t, d_G, d_E, c->stream)) != MDC_OK) return rc;
        if ((rc = mdc_rc_rmse(c, d_data, n, npix, d_t, d_G, d_E, r)) != MDC_OK) return rc;
        row[1] = r[0];
        printf("OptE RMSE = %f!  \t", r[0]);
        if (step) step(it + 1, MDC_RC_STEP_E, d_E, d_G, user);
        double factor = 0;
        if ((rc = mdc_rc_rescale(c, npix, d_E, d_G, &factor)) != MDC_OK) return rc;
        if ((rc = mdc_rc_rmse(c, d_data, n, npix, d_t, d_G, d_E, r)) != MDC_OK) return rc;
        row[2] = r[0]; row[3] = r[1];
        printf("resc RMSE = %f!  \trescale with %f!\n", r[0], factor);
        if (log_host) memcpy(log_host + 4 * it, row, sizeof row);
    }
    return MDC_OK;
}

// ------------------------------------------------------------------ host-buffer entry points
// ---- NUMA placement of pinned host buffers.  On a two-socket box, a pinned buffer that lives on the other socket than the
// GPU it feeds sends every DMA across the inter-socket link.  The node of a GPU comes from sysfs (PCI device -> numa_node); the buffer is allocated while the calling thread's
// memory policy prefers that node (raw set_mempolicy syscall: the image has no libnuma), then the policy is restored.
extern "C" int mdc_device_numa_node(int device) {
    char bus[32] = {0};
    if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return -1; }
    for (char* q = bus; *q; ++q) *q = static_cast<char>(tolower(*q));
    char path[128];
    snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
    FILE* f = fopen(path, "r");
    if (!f) return -1;
    int node = -1;
    if (fscanf(f, "%d", &node) != 1) node = -1;
    fclose(f);
    return node;
}

namespace {
constexpr int kMpolDefault = 0, kMpolPreferred = 1;
long set_mempolicy_raw(int mode, const unsigned long* mask, unsigned long maxnode) {
#ifdef SYS_set_mempolicy
    return syscall(SYS_set_mempolicy, mode, mask, maxnode);
#else
    (void)mode; (void)mask; (void)maxnode;
    return -1;
#endif
}
}  // namespace

extern "C" int mdc_host_alloc(void** p, size_t bytes) {
    if (!p) return MDC_ERR_INVALID_ARG;
    int device = 0;
    const bool have_dev = cudaGetDevice(&device) == cudaSuccess;
    const char* e = getenv("MDC_NUMA_BIND");
    const int node = (have_dev && !(e && atoi(e) == 0)) ? mdc_device_numa_node(device) : -1;
    bool bound = false;
    if (node >= 0 && node < 64) {
        const unsigned long mask = 1ul << node;
        bound = set_mempolicy_raw(kMpolPreferred, &mask, 65) == 0;
    }
    const cudaError_t err = cudaMallocHost(p, bytes);
    if (bound) set_mempolicy_raw(kMpolDefault, nullptr, 0);
    if (err != cudaSuccess) { mdc_set_error("cudaMallocHost(%zu) failed: %s", bytes, cudaGetErrorString(err)); return MDC_ERR_CUDA; }
    return MDC_OK;
}
extern "C" void mdc_host_free(void* p) { if (p) cudaFreeHost(p); }

extern "C" int mdc_unmap_u8_host(mdc_ctx* c, const uint8_t* in, float* out, int n, unsigned flags) {
    if (!c || !in || !out) { mdc_set_error("mdc_unmap_u8_host: bad argument"); return MDC_ERR_INVALID_ARG; }
    if (n != c->in_w * c->in_h) { mdc_set_error("unMapImage: expected %d pixels, got %d", c->in_w * c->in_h, n); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(c->device));
    int rc;
    if ((rc = ensure_bytes(&c->scratch_a, &c->scratch_a_bytes, static_cast<size_t>(n))) != MDC_OK) return rc;
    if ((rc = ensure_bytes(&c->scratch_b, &c->scratch_b_bytes, static_cast<size_t>(n) * 4)) != MDC_OK) return rc;
    CU_CHECK(cudaMemcpyAsync(c->scratch_a, in, static_cast<size_t>(n), cudaMemcpyHostToDevice, c->stream));
    if ((rc = mdc_unmap_u8(c, static_cast<const uint8_t*>(c->scratch_a), static_cast<float*>(c->scratch_b), n, 1, flags, c->stream)) != MDC_OK) return rc;
    CU_CHECK(cudaMemcpyAsync(out, c->scratch_b, static_cast<size_t>(n) * 4, cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    return MDC_OK;
}

template <typename T>
static int undistort_host(mdc_ctx* c, const T* in, float* out, int n_pix_in, int n_pix_out) {
    int rc = check_undistort_args(c, in, out, n_pix_in, n_pix_out, 1);
    if (rc != MDC_OK) return rc;
    CU_CHECK(cudaSetDevice(c->device));
    if ((rc = ensure_bytes(&c->scratch_a, &c->scratch_a_bytes, static_cast<size_t>(n_pix_in) * sizeof(T))) != MDC_OK) return rc;
    if ((rc = ensure_bytes(&c->scratch_b, &c->scratch_b_bytes, static_cast<size_t>(n_pix_out) * 4)) != MDC_OK) return rc;
    CU_CHECK(cudaMemcpyAsync(c->scratch_a, in, static_cast<size_t>(n_pix_in) * sizeof(T), cudaMemcpyHostToDevice, c->stream));
    if (sizeof(T) == 1) rc = mdc_undistort_u8(c, static_cast<const uint8_t*>(c->scratch_a), static_cast<float*>(c->scratch_b), n_pix_in, n_pix_out, 1, c->stream);
    else rc = mdc_undistort_f32(c, static_cast<const float*>(c->scratch_a), static_cast<float*>(c->scratch_b), n_pix_in, n_pix_out, 1, c->stream);
    if (rc != MDC_OK) return rc;
    CU_CHECK(cudaMemcpyAsync(out, c->scratch_b, static_cast<size_t>(n_pix_out) * 4, cudaMemcpyDeviceToHost, c->stream));
    CU_CHECK(cudaStreamSynchronize(c->stream));
    return MDC_OK;
}
extern "C" int mdc_undistort_u8_host(mdc_ctx* c, const uint8_t* in, float* out, int n_pix_in, int n_pix_out) {
    return undistort_host<uint8_t>(c, in, out, n_pix_in, n_pix_out);
}
extern "C" int mdc_undistort_f32_host(mdc_ctx* c, const float* in, float* out, int n_pix_in, int n_pix_out) {
    return undistort_host<float>(c, in, out, n_pix_in, n_pix_out);
}

extern "C" int mdc_prepare_batch_host(mdc_ctx* c, const uint8_t* frames, int n_frames, unsigned flags,
                                      float* const* out_levels, int levels) {
    return mdc_prepare_batch_host_ex(c, frames, n_frames, flags, MDC_OUT_F32, reinterpret_cast<void* const*>(out_levels), levels);
}

extern "C" int mdc_seq_prepare_ex(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, int out_type, void* const* h_out_levels,
                                  int levels, int threads) {
    const int rc = mdc_check_out_type(out_type, "mdc_seq_prepare");
    if (rc != MDC_OK) return rc;
    return mdc_seq_prepare_feed(c, s, first, count, flags, out_type, h_out_levels, levels, threads, mdc_prepare_batch_host_ex);
}

extern "C" int mdc_prepare_batch_host_ex(mdc_ctx* c, const uint8_t* frames, int n_frames, unsigned flags, int out_type,
                                         void* const* out_levels, int levels) {
    int rc0 = mdc_check_out_type(out_type, "mdc_prepare_batch_host_ex");
    if (rc0 != MDC_OK) return rc0;
    if (!c || !frames || !out_levels || n_frames < 0 || levels < 1 || levels > MDC_MAX_PYR_LEVELS) {
        mdc_set_error("mdc_prepare_batch_host: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    if (c->in_w < 1) { mdc_set_error("mdc_prepare_batch_host: context has no image geometry"); return MDC_ERR_INVALID_OBJECT; }
    const bool rectify = (flags & MDC_RECTIFY) != 0;
    const int w0 = rectify ? c->out_w : c->in_w, h0 = rectify ? c->out_h : c->in_h;
    size_t lvl_px[MDC_MAX_PYR_LEVELS], px_per_frame = 0;
    for (int l = 0; l < levels; ++l) {
        lvl_px[l] = static_cast<size_t>(w0 >> l) * (h0 >> l);
        px_per_frame += lvl_px[l];
        // checked before any copy: a NULL host level that has pixels would otherwise reach cudaMemcpyAsync after earlier chunks ran
        if (!out_levels[l] && lvl_px[l] > 0) { mdc_set_error("mdc_prepare_batch_host: output level %d is NULL", l); return MDC_ERR_INVALID_ARG; }
    }
    if (rectify && !c->have_fov) { mdc_set_error("getImage(rectify) on an invalid rectifier"); return MDC_ERR_INVALID_OBJECT; }
    if (n_frames == 0) return MDC_OK;
    CU_CHECK(cudaSetDevice(c->device));
    const size_t n_in = static_cast<size_t>(c->in_w) * c->in_h;
    // chunking: enough frames per kernel to fill the machine, small enough to overlap copy and compute
    const char* e = getenv("MDC_HOST_CHUNK");
    int chunk = e ? atoi(e) : 16;
    chunk = std::max(1, std::min(chunk, n_frames));
    // Rows that are not a multiple of 16 bytes cannot be described to TMA — but the H2D copy can pad them for free (2-D copy into a
    // device buffer with a 32-byte multiple pitch), which keeps such widths on the fast loaders instead of the 2x slower LDG one.
    const int pitch = (rectify && c->in_w % 16 != 0 && c->plan_tma_ok) ? ((c->in_w + 31) & ~31) : c->in_w;
    // pipe buffers and D2H copies in the output type's element size; a narrow type's fp32 scratch (levels K2 reads) follows the levels
    const size_t esize = mdc_out_elem_size(out_type);
    const size_t lv_bytes = (static_cast<size_t>(chunk) * px_per_frame * esize + 255) & ~size_t(255);
    const size_t in_bytes = static_cast<size_t>(chunk) * pitch * c->in_h,
                 out_bytes = lv_bytes + static_cast<size_t>(chunk) * prepare_f32_scratch_bytes(c, rectify, out_type, levels);
    if (c->pipe_in_bytes < in_bytes || c->pipe_out_bytes < out_bytes) {
        for (int s = 0; s < kHostPipeDepth; ++s) {
            if (c->pipe_stream[s]) cudaStreamSynchronize(c->pipe_stream[s]);
            cudaFree(c->pipe_in[s]); cudaFree(c->pipe_out[s]);
            c->pipe_in[s] = nullptr; c->pipe_out[s] = nullptr;
        }
        c->pipe_in_bytes = c->pipe_out_bytes = 0;
        for (int s = 0; s < kHostPipeDepth; ++s) {
            if (!c->pipe_stream[s]) CU_CHECK(cudaStreamCreateWithFlags(&c->pipe_stream[s], cudaStreamNonBlocking));
            CU_CHECK(cudaMalloc(&c->pipe_in[s], in_bytes));
            CU_CHECK(cudaMalloc(&c->pipe_out[s], out_bytes));
        }
        c->pipe_in_bytes = in_bytes; c->pipe_out_bytes = out_bytes;
    }
    // On any failure the copies of earlier chunks into the caller's buffers may still be in flight on the other pipe streams:
    // drain all of them before returning, so the caller can free or reuse its buffers.
    auto drain = [&]() {
        cudaError_t first = cudaSuccess;
        for (int s = 0; s < kHostPipeDepth; ++s)
            if (c->pipe_stream[s]) { const cudaError_t e = cudaStreamSynchronize(c->pipe_stream[s]); if (first == cudaSuccess) first = e; }
        return first;
    };
    int k = 0, rc = MDC_OK;
    for (int f0 = 0; f0 < n_frames && rc == MDC_OK; f0 += chunk, ++k) {
        const int nf = std::min(chunk, n_frames - f0);
        const int s = k % kHostPipeDepth;
        cudaStream_t st = c->pipe_stream[s];
        cudaError_t ce = pitch == c->in_w
            ? cudaMemcpyAsync(c->pipe_in[s], frames + static_cast<size_t>(f0) * n_in, static_cast<size_t>(nf) * n_in, cudaMemcpyHostToDevice, st)
            : cudaMemcpy2DAsync(c->pipe_in[s], static_cast<size_t>(pitch), frames + static_cast<size_t>(f0) * n_in, static_cast<size_t>(c->in_w),
                                static_cast<size_t>(c->in_w), static_cast<size_t>(c->in_h) * nf, cudaMemcpyHostToDevice, st);
        void* lv[MDC_MAX_PYR_LEVELS];
        size_t off = 0;
        for (int l = 0; l < levels; ++l) { lv[l] = c->pipe_out[s] + off; off += static_cast<size_t>(nf) * lvl_px[l] * esize; }
        if (ce == cudaSuccess)
            rc = prepare_batch_impl(c, c->pipe_in[s], pitch == c->in_w ? 0 : pitch, nf, flags, out_type, lv, levels, st, c->pipe_out[s] + lv_bytes);
        for (int l = 0; l < levels && rc == MDC_OK && ce == cudaSuccess; ++l)
            ce = cudaMemcpyAsync(static_cast<uint8_t*>(out_levels[l]) + static_cast<size_t>(f0) * lvl_px[l] * esize, lv[l],
                                 static_cast<size_t>(nf) * lvl_px[l] * esize, cudaMemcpyDeviceToHost, st);
        if (ce != cudaSuccess) { mdc_set_error("mdc_prepare_batch_host: copy failed: %s", cudaGetErrorString(ce)); rc = MDC_ERR_CUDA; }
    }
    const cudaError_t drained = drain();
    if (rc == MDC_OK && drained != cudaSuccess) { mdc_set_error("mdc_prepare_batch_host: %s", cudaGetErrorString(drained)); rc = MDC_ERR_CUDA; }
    return rc;
}
