// Hand-written sm_90a kernels of the frame-preparation hot path.
//
//   K1  fused_prepare_kernel   unMapImage (PhotometricUndistorter.cpp:193-211) composed with
//                              undistort<T> (FOVUndistorter.cpp:341-367) as DatasetReader::getImage
//                              does (BenchmarkDatasetReader.h:210-241), plus pyramid levels 1..4 in
//                              the epilogue (SURVEY.md §8a row P).  Batched over frames.
//   K1a unmap_kernel           unMapImage alone (photo-only mode, BenchmarkDatasetReader.h:216)
//   K1b undistort_f32_kernel   undistort<float> alone (API parity, FOVUndistorter.cpp:369)
//   K2  pyr_down_kernel        one stand-alone pyramid level
//   K3  estep_kernel           responseCalib E-step (main_responseCalib.cpp:324-338)
//
// Arithmetic policy: every floating-point operation of the reference's loops is issued with an
// explicit round-to-nearest intrinsic (__fmul_rn/__fadd_rn/__fsub_rn, __dmul_rn/__dadd_rn/__ddiv_rn)
// in the reference's evaluation order, so nvcc cannot contract them into FMAs and the results are
// bit-identical to the reference's non-FMA x86-64 build (only NaN payloads may differ).
//
// All of this is HBM-bound byte/float streaming; there is no GEMM-shaped work, so no tcgen05.
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>
#include <stdlib.h>

#include <algorithm>
#include <mutex>
#include <type_traits>

#include "mdc_atanf.h"
#include "mdc_kernels.cuh"

namespace mdc {

// Grid of a grid-stride kernel whose result does not depend on the grid: `per_sm` CTAs of 256 threads per SM of the current device.
static size_t grid_cap(size_t per_sm) {
    int dev = 0, sms = 132;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    return static_cast<size_t>(sms) * per_sm;
}

// =====================================================================================
// small PTX helpers: shared-memory access by 32-bit address, mbarrier, TMA, streaming stores
// =====================================================================================
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// volatile: the staged bytes change every frame (TMA / other warps write them), so these loads must
// neither be hoisted out of the frame loop nor merged across iterations.
__device__ __forceinline__ uint32_t lds_u8(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t lds_u8_1(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1+1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ float lds_f32(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) {
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// evict-first store: the rectified images are written once and never re-read by this kernel; keep L2
// for the input frames of the current chunk and for the calibration tables.
__device__ __forceinline__ void stg_cs(float* p, float v) { asm volatile("st.global.cs.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory"); }

// ---- output types (MDC_OUT_*): every level is computed in fp32 and converted only where it is stored
template <int kOut> struct OutElem { using T = float; };
template <> struct OutElem<MDC_OUT_F16> { using T = __half; };
template <> struct OutElem<MDC_OUT_U8> { using T = uint8_t; };
// cv::saturate_cast<uchar>(float), i.e. convertTo(CV_8U), as OpenCV computes it on x86-64: cvRound is cvtss2si (round half to even;
// NaN, +-inf and values outside int32 give INT_MIN), then the clamp to [0, 255].  cvt.rni saturates instead (NaN -> 0, large -> INT_MAX),
// so what x86 turns into INT_MIN at the top end is mapped to 0 explicitly.
__device__ __forceinline__ uint32_t conv_u8(float v) {
    int r = __float2int_rn(v);
    if (!(v < 2147483648.0f)) r = 0;              // NaN, +inf, >= 2^31
    return static_cast<uint32_t>(min(max(r, 0), 255));
}
__device__ __forceinline__ void stg_cs(__half* p, float v) {
    asm volatile("st.global.cs.b16 [%0], %1;" ::"l"(p), "h"(__half_as_ushort(__float2half_rn(v))) : "memory");
}
__device__ __forceinline__ void stg_cs(uint8_t* p, float v) { asm volatile("st.global.cs.u8 [%0], %1;" ::"l"(p), "r"(conv_u8(v)) : "memory"); }
// plain stores of one / four converted pixels (streaming kernels)
__device__ __forceinline__ void put(float* p, float v) { *p = v; }
__device__ __forceinline__ void put(__half* p, float v) { *p = __float2half_rn(v); }
__device__ __forceinline__ void put(uint8_t* p, float v) { *p = static_cast<uint8_t>(conv_u8(v)); }
__device__ __forceinline__ void put4(__half* p, float4 o) {
    const __half2 a = __floats2half2_rn(o.x, o.y), b = __floats2half2_rn(o.z, o.w);
    *reinterpret_cast<uint2*>(p) = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
}
__device__ __forceinline__ void put4(uint8_t* p, float4 o) {
    *reinterpret_cast<uint32_t*>(p) = conv_u8(o.x) | conv_u8(o.y) << 8 | conv_u8(o.z) << 16 | conv_u8(o.w) << 24;
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
// Producer-side wait: the producer is always up to `tma_stages` frames ahead, so it polls politely
// (a spinning lane would steal issue slots from the consumer warps of its scheduler).
__device__ __forceinline__ void mbar_wait_backoff(uint32_t bar, uint32_t parity) {
    uint32_t done;
    for (;;) {
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n"
            : "=r"(done)
            : "r"(bar), "r"(parity), "r"(2000u)
            : "memory");
        if (done) break;
        __nanosleep(400);
    }
}
// 3-D tiled TMA load: box (bw, bh, 1) of the u8 frame stack at (x, y, frame) -> shared memory.
__device__ __forceinline__ void tma_load_box(uint32_t dst, const CUtensorMap* map, uint32_t bar, int x, int y, int frame) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(x), "r"(y), "r"(frame), "r"(bar)
        : "memory");
}
// Pixel pairs ride in the two halves of a 64-bit register pair.  Hopper has no packed FP32 multiply, so mul2 is two IEEE
// round-to-nearest multiplies (__fmul_rn: never contracted into an FMA, which would break bit-exactness).
__device__ __forceinline__ uint64_t pack2(float lo, float hi) { uint64_t r; asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi)); return r; }
__device__ __forceinline__ void unpack2(uint64_t v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
__device__ __forceinline__ uint64_t mul2(uint64_t a, uint64_t b) {
    float a0, a1, b0, b1;
    unpack2(a, a0, a1);
    unpack2(b, b0, b1);
    return pack2(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}

__device__ __forceinline__ void consumer_barrier() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory"); }

// =====================================================================================
// K1: fused photometric un-map + FOV rectification (+ pyramid epilogue)
// =====================================================================================
//
// Work decomposition.  The output image is cut into 32x32 tiles; a tile's bilinear taps fall into a
// compact bounding box of the input image (host-precomputed, TileDesc).  The unit of work is
// (tile, frame).  Frames are grouped into chunks of `chunk_frames`; a work ITEM is (chunk, tile) — one
// tile over the consecutive frames of one chunk — and items are numbered chunk-major, tile-minor.
// Persistent CTAs pull items from a global atomic counter (first item = blockIdx.x), so the load
// balances itself whatever the per-tile cost, and, chip-wide, all CTAs are inside the same chunk at
// the same time, so the overlapping parts of the input that neighbouring tiles re-read are still in
// L2 (50 MB) when they are read again.  48-frame chunks: on H100, 32-96 frames are equally fast within run-to-run spread
// and 16 is slower (DESIGN.md §7, scripts/k1_sweep.py).
//
// Everything that depends only on the calibration — the remap entry of each of the thread's 4 pixels
// (turned into 4 bilinear weights and a box-local byte offset) and the 4 vignette reciprocals under
// the taps — is loaded ONCE per (tile, chunk) into registers and reused for every frame of the run,
// which removes the 15.7 MB/frame of table traffic a naive fused kernel would add to the
// 6.5 MB/frame of unavoidable image traffic (SURVEY.md §7 "hard parts").
//
// Per frame the u8 input box is staged in shared memory:
//   * TMA loader: a dedicated producer warp issues one 3-D cp.async.bulk.tensor per (tile, frame)
//     into a 3-stage ring; full/empty mbarriers connect it to the 8 consumer warps, so in steady state
//     there is no CTA-wide barrier at all and the producer runs ahead across tile boundaries;
//   * LDG loader (image widths TMA cannot describe): every consumer prefetches its share of the next
//     frame's box into registers during the gather and stores it to the other stage afterwards.
// A consumer warp owns 4 output rows of the tile; lane = x.  For each of its 4 pixels a thread reads
// the 4 tap bytes (LDS.U8; 32 lanes along one output row touch ~24 different words, so the access is
// nearly conflict-free), pushes them through the response LUT — lane-replicated in shared memory,
// `lut[v*32+lane]`, so the data-dependent lookup is bank-conflict-free —, multiplies by the cached
// vignette reciprocals and blends with the cached weights in the reference's exact operation order.
// `killOverexposed` is folded into the LUT (lut[255]=NaN) and the no-gamma modes use an identity LUT,
// so one kernel covers all flag combinations as well as undistort<unsigned char>.

__device__ __forceinline__ float lut_value(const FusedParams& p, int v) {
    float r = p.lut_gamma ? __ldg(p.ginv + v) : static_cast<float>(v);
    if (p.kill && v == 255) r = __int_as_float(0x7fc00000);  // NAN
    return r;
}

// kStudy = the floor-study bits | the output type << kOutShift (see k1_variant).  Only the stores depend on the output type; a narrow
// type also writes the fp32 level 2 to p.level2_f32 when the K2 chain needs it.  The fp32 kernels must keep their machine code, so
// the output type rides in kStudy (the fp32 instantiations keep their names and template arguments) and is spelled out where it is
// used: a kernel-local constant here (the frame-loop lambda sees it) changes the fp32 code (scripts/sass_compare.py checks this).
template <bool kTma, bool kVig, bool kPyr, int kMinCtas, int kStudy = kStudyAll>
__global__ void __launch_bounds__(kTma ? kConsumers + 32 : kConsumers, kMinCtas)
fused_prepare_kernel(const __grid_constant__ FusedParams p, const __grid_constant__ TmaMaps maps) {
    using TOut = typename OutElem<(kStudy >> kOutShift)>::T;
    const int kNs = kTma ? p.tma_stages : kLdgStages;   // ring depth (runtime: as many stages as fit next to 3 CTAs/SM)
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // ---- shared-memory carve-up (see fused_smem_bytes)
    float* lut = reinterpret_cast<float*>(smem_raw);                    // [256][32] lane-replicated response LUT
    volatile int* s_item = reinterpret_cast<volatile int*>(lut + 256 * 32);   // [kItemSlots] work items handed from the producer to the consumers
    uint64_t* s_bar = reinterpret_cast<uint64_t*>(lut + 256 * 32 + 8);        // full[kMaxStages] empty[kMaxStages] item_full[kItemSlots] item_empty[kItemSlots]
    const uint32_t stage_bytes = (static_cast<uint32_t>(p.box_px_max) + 127u) & ~127u;
    const uint32_t stage0 = smem_u32(smem_raw) + kSmemHeaderBytes;
    const uint32_t bar_full = smem_u32(s_bar), bar_empty = bar_full + 8u * kMaxStages;
    const uint32_t bar_item_full = bar_empty + 8u * kMaxStages, bar_item_empty = bar_item_full + 8u * kItemSlots;
    const int n_items = ((p.n_frames + p.chunk_frames - 1) / p.chunk_frames) * p.n_tiles;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    // ---- one-time per CTA: LUT, barriers, work range
    for (int i = tid; i < 256 * 32; i += blockDim.x) lut[i] = lut_value(p, i >> 5);
    if (tid == 0 && kTma) {
        for (int i = 0; i < kNs; ++i) { mbar_init(bar_full + 8u * i, 1); mbar_init(bar_empty + 8u * i, kConsumers / 32); }
        for (int i = 0; i < kItemSlots; ++i) { mbar_init(bar_item_full + 8u * i, 1); mbar_init(bar_item_empty + 8u * i, kConsumers / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    int tile, f_begin, f_end;

    // ================================================================ producer warp (TMA loader only)
    if (kTma && warp == kConsumers / 32) {
        if (lane == 0) {
            uint32_t st = 0, round = 0;        // stage ring position of the next frame to issue
            uint32_t islot = 0, iround = 0;    // item ring position
            int item = blockIdx.x;
            for (;;) {
                if (iround > 0) mbar_wait_backoff(bar_item_empty + 8u * islot, (iround - 1u) & 1u);
                s_item[islot] = item;
                mbar_arrive(bar_item_full + 8u * islot);      // release: the item id is visible to whoever sees this phase complete
                if (++islot == static_cast<uint32_t>(kItemSlots)) { islot = 0; ++iround; }
                if (item >= n_items) break;
                tile = item % p.n_tiles;
                f_begin = (item / p.n_tiles) * p.chunk_frames;
                f_end = min(f_begin + p.chunk_frames, p.n_frames);
                const TileDesc td = p.tiles[tile];
                if ((td.mode_map & 0x0f) == TILE_STAGED) {
                    const CUtensorMap* tmap = &maps.m[(td.mode_map >> 8) & 0xff];
                    const uint32_t bytes = static_cast<uint32_t>(td.bw_bh & 0xffff) * static_cast<uint32_t>(td.mode_map >> 16);
                    for (int f = f_begin; f < f_end; ++f) {
                        if (round > 0) mbar_wait_backoff(bar_empty + 8u * st, (round - 1u) & 1u);   // consumers released this slot
                        mbar_expect_tx(bar_full + 8u * st, bytes);
                        tma_load_box(stage0 + st * stage_bytes, tmap, bar_full + 8u * st, td.x0, td.y0, f);
                        if (++st == static_cast<uint32_t>(kNs)) { st = 0; ++round; }
                    }
                }
                item = static_cast<int>(gridDim.x) + atomicAdd(p.work_counter, 1);
            }
        }
        return;
    }

    // ================================================================ consumer warps
    const size_t n_in = static_cast<size_t>(p.in_pitch) * p.in_h;      // bytes from one frame to the next (rows may be padded)
    const uint32_t lut_lane = smem_u32(lut) + 4u * lane;
    uint32_t st = 0, phase = 0;   // ring position / parity of the next staged frame to consume
    uint32_t st_addr = stage0;    // = stage0 + st * stage_bytes
    uint32_t islot = 0, iphase = 0;
    int item = blockIdx.x;

    for (;;) {
        if (kTma) {          // next item from the producer warp
            mbar_wait(bar_item_full + 8u * islot, iphase);
            item = s_item[islot];
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_item_empty + 8u * islot);
            if (++islot == static_cast<uint32_t>(kItemSlots)) { islot = 0; iphase ^= 1u; }
        }
        if (item >= n_items) break;
        tile = item % p.n_tiles;
        f_begin = (item / p.n_tiles) * p.chunk_frames;
        f_end = min(f_begin + p.chunk_frames, p.n_frames);
        // ------------------------------------------------------------ per-(tile, run) prologue
        const TileDesc td = p.tiles[tile];
        const int mode = td.mode_map & 0x0f;
        const bool staged = mode == TILE_STAGED;
        const int bw = td.bw_bh & 0xffff, bh = td.bw_bh >> 16;
        const int tx0 = (tile % p.tiles_x) * kTile, ty0 = (tile / p.tiles_x) * kTile;
        const int ox = tx0 + lane, oy0 = ty0 + 4 * warp;
        const int pitch = staged ? bw : p.in_pitch;   // distance between the two tap rows

        float w[4][4], vi[4][4];
        uint32_t off[4];
        unsigned valid = 0;
        const bool has_black = (td.mode_map & TILE_HAS_BLACK) != 0;   // some in-image pixel of the tile has no source
        const bool full_tile = tx0 + kTile <= p.out_w && ty0 + kTile <= p.out_h;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int oy = oy0 + q;
            float sx = -1.0f, sy = -1.0f;
            if (ox < p.out_w && oy < p.out_h) {
                const size_t o = static_cast<size_t>(oy) * p.out_w + ox;
                sx = __ldg(p.remap_x + o);
                sy = __ldg(p.remap_y + o);
            }
            off[q] = 0;
#pragma unroll
            for (int k = 0; k < 4; ++k) { w[q][k] = 0.0f; vi[q][k] = 1.0f; }
            if (!(sx < 0)) {  // the reference tests only remapX (FOVUndistorter.cpp:347)
                valid |= 1u << q;
                const int xi = static_cast<int>(sx), yi = static_cast<int>(sy);   // truncation, :352-353
                const float fx = __fsub_rn(sx, static_cast<float>(xi));
                const float fy = __fsub_rn(sy, static_cast<float>(yi));
                const float fxy = __fmul_rn(fx, fy);
                w[q][3] = fxy;
                w[q][2] = __fsub_rn(fy, fxy);
                w[q][1] = __fsub_rn(fx, fxy);
                w[q][0] = __fadd_rn(__fsub_rn(__fsub_rn(1.0f, fx), fy), fxy);
                const int g = yi * p.in_w + xi;               // index into the (tightly packed) vignette table
                off[q] = static_cast<uint32_t>(staged ? (yi - td.y0) * bw + (xi - td.x0) : yi * p.in_pitch + xi);
                if (kVig) {
                    vi[q][0] = __ldg(p.vinv + g);
                    vi[q][1] = __ldg(p.vinv + g + 1);
                    vi[q][2] = __ldg(p.vinv + g + p.in_w);
                    vi[q][3] = __ldg(p.vinv + g + p.in_w + 1);
                }
            }
        }

        // LDG loader geometry: threads tiled (rows x words-per-row) with a power-of-two row length
        int lg = 2;
        while ((4 << lg) < bw) ++lg;
        const int ld_col = tid & ((1 << lg) - 1), ld_row = tid >> lg, ld_rstep = kConsumers >> lg;
        const int ld_pass = (staged && !kTma) ? (bh + ld_rstep - 1) / ld_rstep : 0;
        const bool ld_col_ok = (ld_col * 4) < bw;
        const bool ld_fast = ((p.in_pitch & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.frames) & 3) == 0);
        uint32_t pre[kMaxBoxWordsPerThread];
        auto ldg_box = [&](int frame) {   // issue the global loads of `frame`'s box into registers
            const uint8_t* src = p.frames + static_cast<size_t>(frame) * n_in;
#pragma unroll
            for (int k = 0; k < kMaxBoxWordsPerThread; ++k) {
                uint32_t v = 0;
                if (k < ld_pass) {
                    const int row = ld_row + k * ld_rstep, gy = td.y0 + row, gx = td.x0 + ld_col * 4;
                    if (ld_col_ok && row < bh && gy < p.in_h && gx < p.in_w) {
                        const uint8_t* a = src + static_cast<size_t>(gy) * p.in_pitch + gx;
                        if (ld_fast) v = __ldg(reinterpret_cast<const uint32_t*>(a));
                        else {
                            v = __ldg(a);
                            if (gx + 1 < p.in_w) v |= static_cast<uint32_t>(__ldg(a + 1)) << 8;
                            if (gx + 2 < p.in_w) v |= static_cast<uint32_t>(__ldg(a + 2)) << 16;
                            if (gx + 3 < p.in_w) v |= static_cast<uint32_t>(__ldg(a + 3)) << 24;
                        }
                    }
                }
                pre[k] = v;
            }
        };
        auto sts_box = [&](uint32_t stage) {
#pragma unroll
            for (int k = 0; k < kMaxBoxWordsPerThread; ++k) {
                const int row = ld_row + k * ld_rstep;
                if (k < ld_pass && ld_col_ok && row < bh) sts_u32(stage + static_cast<uint32_t>(row * bw + ld_col * 4), pre[k]);
            }
        };
        if (!kTma && staged) {   // first frame of the run: load + publish before anybody gathers
            ldg_box(f_begin);        // (the barrier closing the previous run's last frame already freed both stages)
            sts_box(st_addr);
            consumer_barrier();
        }
        // packed (pixel q, pixel q+1) weights / vignette reciprocals for mul2
        uint64_t w2[2][4], vi2[2][4];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                w2[h][k] = pack2(w[2 * h][k], w[2 * h + 1][k]);
                vi2[h][k] = pack2(vi[2 * h][k], vi[2 * h + 1][k]);
            }

        TOut* o0 = static_cast<TOut*>(p.out[0]) + static_cast<size_t>(f_begin) * p.lw[0] * p.lh[0] + static_cast<size_t>(oy0) * p.out_w + ox;
        const size_t o0_step = static_cast<size_t>(p.lw[0]) * p.lh[0];
        const bool x_ok = ox < p.out_w;
        // pyramid levels 1-2: per-item output pointers and store predicates (advanced by one image per frame)
        TOut *o1 = nullptr, *o2 = nullptr;
        float* o2f = nullptr;                // narrow types: fp32 level 2 for the K2 chain
        uint32_t o1_step = 0, o2_step = 0;   // elements per image of level 1 / 2 (< 2^31)
        bool st1 = false, st2 = false, st2f = false;
        if (kPyr) {
            const int X1 = (tx0 >> 1) + (lane >> 1), Y1 = (ty0 >> 1) + 2 * warp + (lane & 1);   // even lane: upper block, odd lane: lower block
            st1 = X1 < p.lw[1] && Y1 < p.lh[1];
            o1_step = static_cast<uint32_t>(p.lw[1]) * static_cast<uint32_t>(p.lh[1]);
            o1 = static_cast<TOut*>(p.out[1]) + static_cast<size_t>(f_begin) * o1_step + static_cast<size_t>(Y1) * p.lw[1] + X1;
            if (p.levels > 2) {
                const int X2 = (tx0 >> 2) + (lane >> 2), Y2 = (ty0 >> 2) + warp;
                st2 = (lane & 3) == 0 && X2 < p.lw[2] && Y2 < p.lh[2];
                o2_step = static_cast<uint32_t>(p.lw[2]) * static_cast<uint32_t>(p.lh[2]);
                o2 = static_cast<TOut*>(p.out[2]) + static_cast<size_t>(f_begin) * o2_step + static_cast<size_t>(Y2) * p.lw[2] + X2;
                if constexpr ((kStudy >> kOutShift) != MDC_OUT_F32) {
                    if (p.level2_f32) {
                        o2f = p.level2_f32 + static_cast<size_t>(f_begin) * o2_step + static_cast<size_t>(Y2) * p.lw[2] + X2;
                        st2f = st2;
                    }
                }
            }
        }

        uint32_t study_acc = 0;
        // ------------------------------------------------------------ frame loop, specialised on how the taps are fetched
        auto run_frames = [&](auto staged_c, auto black_c) {
        constexpr bool kStaged = decltype(staged_c)::value;
        constexpr bool kBlack = decltype(black_c)::value;
        for (int f = f_begin; f < f_end; ++f) {
            float px[4];
            uint32_t base = 0;
            const uint8_t* frame = nullptr;
            if (kStaged) {
                if (kTma) mbar_wait(bar_full + 8u * st, phase);
                else if (f + 1 < f_end) ldg_box(f + 1);          // in flight during the gather below
                base = st_addr;
            } else {
                frame = p.frames + static_cast<size_t>(f) * n_in;
            }
            // two halves of two pixels each: keeps the live temporaries (tap bytes, LUT values) at 8 registers
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                uint32_t b[2][4];
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const int q = 2 * h + j;
                    if (!(kStudy & kStudyTaps)) {      // floor study: tap bytes from the ALU instead of the staged box
#pragma unroll
                        for (int k = 0; k < 4; ++k) b[j][k] = (off[q] + static_cast<uint32_t>(f + 37 * k)) & 0xffu;
                    } else if (kStaged) {
                        const uint32_t a0 = base + off[q], a1 = a0 + static_cast<uint32_t>(pitch);
                        b[j][0] = lds_u8(a0); b[j][1] = lds_u8_1(a0);
                        b[j][2] = lds_u8(a1); b[j][3] = lds_u8_1(a1);
                    } else {
                        const uint8_t* s = frame + off[q];
                        b[j][0] = __ldg(s); b[j][1] = __ldg(s + 1);
                        b[j][2] = __ldg(s + pitch); b[j][3] = __ldg(s + pitch + 1);
                    }
                }
                float g[2][4];
#pragma unroll
                for (int j = 0; j < 2; ++j)
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        g[j][k] = (kStudy & kStudyLut) ? lds_f32(lut_lane + (b[j][k] << 7)) : __uint_as_float(0x3f800000u | b[j][k]);
                if (kStaged && h == 1) {
                    if (kTma) {          // all tap bytes of this warp are in registers: hand the stage back to the producer
                        __syncwarp();
                        if (lane == 0) mbar_arrive(bar_empty + 8u * st);
                    }
                    st_addr += stage_bytes;
                    if (++st == static_cast<uint32_t>(kNs)) { st = 0; st_addr = stage0; phase ^= 1u; }
                }
                // unMapImage multiply + bilinear blend, reference order (PhotometricUndistorter.cpp:205, FOVUndistorter.cpp:362-365);
                // pixels 2h and 2h+1 ride in the two halves of packed registers
                float t_lo[4], t_hi[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    uint64_t v = pack2(g[0][k], g[1][k]);
                    if (kVig) v = mul2(v, vi2[h][k]);
                    v = mul2(w2[h][k], v);
                    unpack2(v, t_lo[k], t_hi[k]);
                }
                px[2 * h] = __fadd_rn(__fadd_rn(__fadd_rn(t_lo[3], t_lo[2]), t_lo[1]), t_lo[0]);
                px[2 * h + 1] = __fadd_rn(__fadd_rn(__fadd_rn(t_hi[3], t_hi[2]), t_hi[1]), t_hi[0]);
            }
            if (kBlack) {
#pragma unroll
                for (int q = 0; q < 4; ++q) px[q] = ((valid >> q) & 1u) ? px[q] : 0.0f;
            }

            // ---- level 0: one full 128-byte row segment per warp store
            if (!(kStudy & kStudyStores)) {      // floor study: fold the pixels into a register instead of storing them
                study_acc ^= __float_as_uint(px[0]) ^ __float_as_uint(px[1]);
                study_acc ^= __float_as_uint(px[2]) ^ __float_as_uint(px[3]);
            } else if (full_tile) {
#pragma unroll
                for (int q = 0; q < 4; ++q) stg_cs(o0 + static_cast<size_t>(q) * p.out_w, px[q]);
            } else if (x_ok) {
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if (oy0 + q < p.out_h) stg_cs(o0 + static_cast<size_t>(q) * p.out_w, px[q]);
            }
            o0 += o0_step;

            // ---- pyramid epilogue: dst = 0.25f*(((a+b)+c)+d), a=(2x,2y) b=(2x+1,2y) c=(2x,2y+1) d=(2x+1,2y+1).
            // A lane pair (x even / x odd) owns two 2x2 blocks (rows 0-1 and rows 2-3); the even lane finishes the upper
            // one, the odd lane the lower one, so each lane sends exactly the two values its partner lacks: 2 shuffles
            // and ONE store instruction for level 1 (instead of 4 and 2).
            if (kPyr) {
                const bool odd = (lane & 1) != 0;
                const float r1 = __shfl_xor_sync(0xffffffffu, odd ? px[0] : px[2], 1);
                const float r2 = __shfl_xor_sync(0xffffffffu, odd ? px[1] : px[3], 1);
                const float pa = odd ? r1 : px[0], pb = odd ? px[2] : r1, pc = odd ? r2 : px[1], pd = odd ? px[3] : r2;
                const float l1 = __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(pa, pb), pc), pd));
                if (st1) stg_cs(o1, l1);
                o1 += o1_step;
                if (p.levels > 2) {
                    // level-2 pixel of lanes 4m..4m+3: a = lane 4m (upper, X even), c = lane 4m+1 (lower, X even),
                    // b = lane 4m+2 (upper, X odd), d = lane 4m+3 (lower, X odd)
                    const float c2 = __shfl_down_sync(0xffffffffu, l1, 1);
                    const float b2 = __shfl_down_sync(0xffffffffu, l1, 2);
                    const float d2 = __shfl_down_sync(0xffffffffu, l1, 3);
                    const float l2 = __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(l1, b2), c2), d2));   // lanes = 0 mod 4
                    if (st2) stg_cs(o2, l2);
                    o2 += o2_step;
                    if constexpr ((kStudy >> kOutShift) != MDC_OUT_F32) {
                        if (st2f) stg_cs(o2f, l2);
                        o2f += o2_step;
                    }
                }
            }
            if (!kTma && kStaged) {
                if (f + 1 < f_end) sts_box(st_addr);   // st_addr already points at the next frame's stage
                consumer_barrier();     // next stage published; everybody done reading the current one
            }
        }
        };
        if (staged) { if (has_black) run_frames(std::true_type{}, std::true_type{}); else run_frames(std::true_type{}, std::false_type{}); }
        else run_frames(std::false_type{}, std::true_type{});
        if (!(kStudy & kStudyStores) && study_acc == 0x9e3779b9u && x_ok) stg_cs(static_cast<TOut*>(p.out[0]), 0.0f);   // keeps the folded pixels alive
        if (!kTma) {         // LDG loader: thread 0 pulls the next item for the whole CTA
            consumer_barrier();
            if (tid == 0) s_item[0] = static_cast<int>(gridDim.x) + atomicAdd(p.work_counter, 1);
            consumer_barrier();
            item = s_item[0];
        }
    }
}

// smem layout (bytes): lut 32768 | items 32 | barriers 8*(2*kMaxStages+2*kItemSlots) | pad -> kSmemHeaderBytes | stages
size_t fused_smem_bytes(int box_px_max, int stages) {
    const size_t stage = (static_cast<size_t>(box_px_max) + 127u) & ~static_cast<size_t>(127u);
    return kSmemHeaderBytes + static_cast<size_t>(stages) * stage;
}

// Deepest TMA ring (2..kMaxStages) that still lets `ctas_per_sm` CTAs share an SM's 228 KB (1 KB reserved per CTA).
int fused_tma_stages(int box_px_max, int ctas_per_sm) {
    const size_t stage = (static_cast<size_t>(box_px_max) + 127u) & ~static_cast<size_t>(127u);
    const size_t per_cta = (228u * 1024u) / static_cast<size_t>(ctas_per_sm) - 1024u;
    int s = per_cta > kSmemHeaderBytes ? static_cast<int>((per_cta - kSmemHeaderBytes) / stage) : 2;
    if (s > kMaxStages) s = kMaxStages;
    if (s < 2) s = 2;
    return s;
}

typedef void (*FusedKernelFn)(const FusedParams, const TmaMaps);
template <int kMinCtas, int kV = kStudyAll>
static FusedKernelFn fused_variant_t(bool tma, bool vig, bool pyr) {
    if (tma) {
        if (vig) return pyr ? fused_prepare_kernel<true, true, true, kMinCtas, kV> : fused_prepare_kernel<true, true, false, kMinCtas, kV>;
        return pyr ? fused_prepare_kernel<true, false, true, kMinCtas, kV> : fused_prepare_kernel<true, false, false, kMinCtas, kV>;
    }
    if (vig) return pyr ? fused_prepare_kernel<false, true, true, kMinCtas, kV> : fused_prepare_kernel<false, true, false, kMinCtas, kV>;
    return pyr ? fused_prepare_kernel<false, false, true, kMinCtas, kV> : fused_prepare_kernel<false, false, false, kMinCtas, kV>;
}
static FusedKernelFn fused_variant(bool tma, bool vig, bool pyr, int min_ctas, int out_type) {
    constexpr int kF16 = k1_variant(MDC_OUT_F16), kU8 = k1_variant(MDC_OUT_U8);
    if (out_type == MDC_OUT_F32) return min_ctas <= 2 ? fused_variant_t<2>(tma, vig, pyr) : fused_variant_t<3>(tma, vig, pyr);
    if (out_type == MDC_OUT_F16) return min_ctas <= 2 ? fused_variant_t<2, kF16>(tma, vig, pyr) : fused_variant_t<3, kF16>(tma, vig, pyr);
    return min_ctas <= 2 ? fused_variant_t<2, kU8>(tma, vig, pyr) : fused_variant_t<3, kU8>(tma, vig, pyr);
}

int fused_max_ctas_per_sm(int box_px_max, int stages, bool tma, bool vig, bool pyr, int min_ctas, int out_type) {
    int n = 0;
    const int smem = static_cast<int>(fused_smem_bytes(box_px_max, stages));
    FusedKernelFn fn = fused_variant(tma, vig, pyr, min_ctas, out_type);
    // the opt-in limit must be raised before the occupancy query, or it reports 0 for > 48 KB
    if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, tma ? kConsumers + 32 : kConsumers, smem) != cudaSuccess) return 0;
    return n;
}

cudaError_t launch_fused(const FusedParams& p, const TmaMaps* maps, int grid, int min_ctas, int out_type, cudaStream_t stream) {
    const bool tma = maps != nullptr;
    const size_t smem = fused_smem_bytes(p.box_px_max, tma ? p.tma_stages : kLdgStages);
    FusedKernelFn fn = fused_variant(tma, p.use_vig != 0, p.levels > 1, min_ctas, out_type);
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    if (p.carveout > 0 && (e = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, p.carveout)) != cudaSuccess) return e;
    static const TmaMaps none = {};
    fn<<<grid, tma ? kConsumers + 32 : kConsumers, smem, stream>>>(p, tma ? *maps : none);
    return cudaGetLastError();
}

// Floor-study launches of the shipped TMA variant <tma, vignette, no pyramid, 3 CTAs/SM> with parts of the frame loop disabled.
cudaError_t launch_fused_study(const FusedParams& p, const TmaMaps* maps, int grid, int study, cudaStream_t stream) {
    if (!maps || p.levels > 1) return cudaErrorInvalidValue;
    FusedKernelFn fn = nullptr;
    switch (study & kStudyAll) {
        case 0: fn = fused_prepare_kernel<true, true, false, 3, 0>; break;
        case 1: fn = fused_prepare_kernel<true, true, false, 3, 1>; break;
        case 2: fn = fused_prepare_kernel<true, true, false, 3, 2>; break;
        case 3: fn = fused_prepare_kernel<true, true, false, 3, 3>; break;
        case 4: fn = fused_prepare_kernel<true, true, false, 3, 4>; break;
        case 5: fn = fused_prepare_kernel<true, true, false, 3, 5>; break;
        case 6: fn = fused_prepare_kernel<true, true, false, 3, 6>; break;
        default: fn = fused_prepare_kernel<true, true, false, 3, 7>; break;
    }
    const size_t smem = fused_smem_bytes(p.box_px_max, p.tma_stages);
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    fn<<<grid, kConsumers + 32, smem, stream>>>(p, *maps);
    return cudaGetLastError();
}

// =====================================================================================
// K1, texture-gather loader.  Same arithmetic, different plumbing: the four tap bytes of an output pixel are exactly the
// 2x2 footprint a texture unit fetches for bilinear filtering, so ONE `tld4` (texture gather, point-addressed at the integer
// source position) returns them — through the TEX pipe, straight from the u8 frames in global memory (L2 -> L1), with no
// shared-memory staging at all.  That takes the tap traffic (16 LDS.U8 per warp and frame of the TMA-staged kernel) off
// the LSU data pipe, which is left with the response-LUT look-ups and the stores;
// the two pipes then run side by side:
//     TEX  4 tld4 per warp-frame (4 lanes/clock/SM)          LSU  16 LUT + ~7 store wavefronts per warp-frame
// There is no producer warp, no mbarrier and no CTA-wide barrier in the frame loop: a warp owns a STRIP (4 output rows x
// 32 columns) of its CTA's tile over the frames of one chunk and never talks to another warp.
//
// Frames are addressed as u8 pitch-2D texture objects over the caller's frame stack (no copy): the frames of a chunk are
// stacked vertically in one object (row = frame_in_chunk*in_h + y; texture gather limits the height, so the chunk length
// follows from it, see run_fused), point sampling, unnormalised coordinates.  tld4 at (xi+1, yi+1) selects texels floor(u-0.5) = xi, xi+1 / yi, yi+1 — both
// half-integers are exact in the TEX unit's fixed-point coordinates — and returns them as
//     .x = (xi, yi+1)   .y = (xi+1, yi+1)   .z = (xi+1, yi)   .w = (xi, yi)          (checked at context creation).
// =====================================================================================
__device__ __forceinline__ void tld4_u8(unsigned long long tex, float u, float v, uint32_t& x, uint32_t& y, uint32_t& z, uint32_t& w) {
    asm volatile("tld4.r.2d.v4.u32.f32 {%0, %1, %2, %3}, [%4, {%5, %6}];" : "=r"(x), "=r"(y), "=r"(z), "=r"(w) : "l"(tex), "f"(u), "f"(v));
}

// kStudy: floor-study bits | output type << kOutShift, as for the staged kernel
template <bool kVig, bool kPyr, int kMinCtas, bool kPrefetch, int kStudy>
__global__ void __launch_bounds__(kTexThreads, kMinCtas)
fused_tex_kernel(const __grid_constant__ FusedParams p, const __grid_constant__ TexSet texs) {
    constexpr int kOut = kStudy >> kOutShift;
    using TOut = typename OutElem<kOut>::T;     // only the stores depend on it
    constexpr bool kNarrow = kOut != MDC_OUT_F32;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    float* lut = reinterpret_cast<float*>(smem_raw);                    // [256][32] lane-replicated response LUT
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < 256 * 32; i += blockDim.x) lut[i] = lut_value(p, i >> 5);
    __syncthreads();

    const uint32_t lut_lane = smem_u32(lut) + 4u * lane;
    const float frame_rows = static_cast<float>(p.in_h);               // texture rows per frame (exact: < 2^24)

    // grid = (tile groups, chunks).  Everything that selects the texture object and bounds the loops below depends on
    // blockIdx and kernel parameters only, i.e. is CTA-uniform by construction, so ptxas keeps the handle in a uniform
    // register (with a dynamically scheduled work loop it wraps every TLD4 in a 7-instruction divergence loop instead).
    // Load balance is left to the hardware CTA scheduler: CTAs are short (tiles_per_cta tiles x one chunk of frames) and
    // are issued chunk-major, so chip-wide everybody is inside the same chunk or the next.
    const int chunk = blockIdx.y;
    const int f_begin = chunk * p.chunk_frames, f_end = min(f_begin + p.chunk_frames, p.n_frames);
    const unsigned long long tex = texs.tex[chunk];                     // one texture object per chunk (frames stacked vertically)
    const int wrow = warp;                                              // strip of the tile: output rows 4*warp .. 4*warp+3
    for (int t = 0; t < p.tiles_per_cta; ++t) {
        const int tile = static_cast<int>(blockIdx.x) * p.tiles_per_cta + t;
        if (tile >= p.n_tiles) break;
        {
        const int tx0 = (tile % p.tiles_x) * kTile, ty0 = (tile / p.tiles_x) * kTile;
        const int ox = tx0 + lane, oy0 = ty0 + 4 * wrow;

        // ------------------------------------------------------------ per-(strip, chunk) prologue: weights, vignette taps, coordinates
        float w[4][4], vi[4][4], tu[4], tv[4];
        unsigned valid = 0, inside = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const int oy = oy0 + q;
            float sx = -1.0f, sy = -1.0f;
            if (ox < p.out_w && oy < p.out_h) {
                inside |= 1u << q;
                const size_t o = static_cast<size_t>(oy) * p.out_w + ox;
                sx = __ldg(p.remap_x + o);
                sy = __ldg(p.remap_y + o);
            }
            tu[q] = 1.0f; tv[q] = 1.0f;
#pragma unroll
            for (int k = 0; k < 4; ++k) { w[q][k] = 0.0f; vi[q][k] = 1.0f; }
            if (!(sx < 0)) {  // the reference tests only remapX (FOVUndistorter.cpp:347)
                valid |= 1u << q;
                const int xi = static_cast<int>(sx), yi = static_cast<int>(sy);   // truncation, :352-353
                const float fx = __fsub_rn(sx, static_cast<float>(xi));
                const float fy = __fsub_rn(sy, static_cast<float>(yi));
                const float fxy = __fmul_rn(fx, fy);
                w[q][3] = fxy;
                w[q][2] = __fsub_rn(fy, fxy);
                w[q][1] = __fsub_rn(fx, fxy);
                w[q][0] = __fadd_rn(__fsub_rn(__fsub_rn(1.0f, fx), fy), fxy);
                tu[q] = static_cast<float>(xi + 1);
                tv[q] = static_cast<float>(yi + 1);
                if (kVig) {
                    const int g = yi * p.in_w + xi;
                    vi[q][0] = __ldg(p.vinv + g);
                    vi[q][1] = __ldg(p.vinv + g + 1);
                    vi[q][2] = __ldg(p.vinv + g + p.in_w);
                    vi[q][3] = __ldg(p.vinv + g + p.in_w + 1);
                }
            }
        }
        const bool any_black = valid != inside;                         // some in-image pixel of this thread has no source
        uint64_t w2[2][4], vi2[2][4];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                w2[h][k] = pack2(w[2 * h][k], w[2 * h + 1][k]);
                vi2[h][k] = pack2(vi[2 * h][k], vi[2 * h + 1][k]);
            }

        TOut* o0 = static_cast<TOut*>(p.out[0]) + static_cast<size_t>(f_begin) * p.lw[0] * p.lh[0] + static_cast<size_t>(oy0) * p.out_w + ox;
        const size_t o0_step = static_cast<size_t>(p.lw[0]) * p.lh[0];
        const bool full_strip = inside == 0xfu;
        TOut *o1 = nullptr, *o2 = nullptr;
        float* o2f = nullptr;
        uint32_t o1_step = 0, o2_step = 0;
        bool st1 = false, st2 = false, st2f = false;
        if (kPyr) {
            const int X1 = (tx0 >> 1) + (lane >> 1), Y1 = (ty0 >> 1) + 2 * wrow + (lane & 1);   // even lane: upper block, odd lane: lower block
            st1 = X1 < p.lw[1] && Y1 < p.lh[1];
            o1_step = static_cast<uint32_t>(p.lw[1]) * static_cast<uint32_t>(p.lh[1]);
            o1 = static_cast<TOut*>(p.out[1]) + static_cast<size_t>(f_begin) * o1_step + static_cast<size_t>(Y1) * p.lw[1] + X1;
            if (p.levels > 2) {
                const int X2 = (tx0 >> 2) + (lane >> 2), Y2 = (ty0 >> 2) + wrow;
                st2 = (lane & 3) == 0 && X2 < p.lw[2] && Y2 < p.lh[2];
                o2_step = static_cast<uint32_t>(p.lw[2]) * static_cast<uint32_t>(p.lh[2]);
                o2 = static_cast<TOut*>(p.out[2]) + static_cast<size_t>(f_begin) * o2_step + static_cast<size_t>(Y2) * p.lw[2] + X2;
                if constexpr (kNarrow) {
                    if (p.level2_f32) {
                        o2f = p.level2_f32 + static_cast<size_t>(f_begin) * o2_step + static_cast<size_t>(Y2) * p.lw[2] + X2;
                        st2f = st2;
                    }
                }
            }
        }
        uint32_t study_acc = 0;

        // taps of one frame: b[q] = {(xi,yi), (xi+1,yi), (xi,yi+1), (xi+1,yi+1)} = reference order src[0], src[1], src[in_w], src[1+in_w]
        auto fetch = [&](uint32_t (&b)[4][4], int f) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                if (kStudy & kStudyTaps) tld4_u8(tex, tu[q], tv[q], b[q][2], b[q][3], b[q][1], b[q][0]);
                else {
#pragma unroll
                    for (int k = 0; k < 4; ++k) b[q][k] = (__float_as_uint(tu[q]) + static_cast<uint32_t>(f + 37 * k)) & 0xffu;
                }
            }
            // advance the coordinates to the next frame of the stack
#pragma unroll
            for (int q = 0; q < 4; ++q) tv[q] = __fadd_rn(tv[q], frame_rows);
        };

        uint32_t bn[4][4];
        if (kPrefetch) fetch(bn, f_begin);
        for (int f = f_begin; f < f_end; ++f) {
            uint32_t b[4][4];
            if (kPrefetch) {
#pragma unroll
                for (int q = 0; q < 4; ++q)
#pragma unroll
                    for (int k = 0; k < 4; ++k) b[q][k] = bn[q][k];
                if (f + 1 < f_end) fetch(bn, f + 1);        // next frame's taps are in flight during this frame's arithmetic
            } else {
                fetch(b, f);
            }
            float px[4];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float g[2][4];
#pragma unroll
                for (int j = 0; j < 2; ++j)
#pragma unroll
                    for (int k = 0; k < 4; ++k)
                        g[j][k] = (kStudy & kStudyLut) ? lds_f32(lut_lane + (b[2 * h + j][k] << 7)) : __uint_as_float(0x3f800000u | b[2 * h + j][k]);
                // unMapImage multiply + bilinear blend, reference order (PhotometricUndistorter.cpp:205, FOVUndistorter.cpp:362-365)
                float t_lo[4], t_hi[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    uint64_t v = pack2(g[0][k], g[1][k]);
                    if (kVig) v = mul2(v, vi2[h][k]);
                    v = mul2(w2[h][k], v);
                    unpack2(v, t_lo[k], t_hi[k]);
                }
                px[2 * h] = __fadd_rn(__fadd_rn(__fadd_rn(t_lo[3], t_lo[2]), t_lo[1]), t_lo[0]);
                px[2 * h + 1] = __fadd_rn(__fadd_rn(__fadd_rn(t_hi[3], t_hi[2]), t_hi[1]), t_hi[0]);
            }
            if (any_black) {
#pragma unroll
                for (int q = 0; q < 4; ++q) px[q] = ((valid >> q) & 1u) ? px[q] : 0.0f;
            }
            // ---- level 0: one full 128-byte row segment per warp store
            if (!(kStudy & kStudyStores)) {
                study_acc ^= __float_as_uint(px[0]) ^ __float_as_uint(px[1]);
                study_acc ^= __float_as_uint(px[2]) ^ __float_as_uint(px[3]);
            } else if (full_strip) {
#pragma unroll
                for (int q = 0; q < 4; ++q) stg_cs(o0 + static_cast<size_t>(q) * p.out_w, px[q]);
            } else {
#pragma unroll
                for (int q = 0; q < 4; ++q)
                    if ((inside >> q) & 1u) stg_cs(o0 + static_cast<size_t>(q) * p.out_w, px[q]);
            }
            o0 += o0_step;
            // ---- pyramid epilogue (same lane roles as the staged kernel): dst = 0.25f*(((a+b)+c)+d)
            if (kPyr) {
                const bool odd = (lane & 1) != 0;
                const float r1 = __shfl_xor_sync(0xffffffffu, odd ? px[0] : px[2], 1);
                const float r2 = __shfl_xor_sync(0xffffffffu, odd ? px[1] : px[3], 1);
                const float pa = odd ? r1 : px[0], pb = odd ? px[2] : r1, pc = odd ? r2 : px[1], pd = odd ? px[3] : r2;
                const float l1 = __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(pa, pb), pc), pd));
                if (st1) stg_cs(o1, l1);
                o1 += o1_step;
                if (p.levels > 2) {
                    const float c2 = __shfl_down_sync(0xffffffffu, l1, 1);
                    const float b2 = __shfl_down_sync(0xffffffffu, l1, 2);
                    const float d2 = __shfl_down_sync(0xffffffffu, l1, 3);
                    const float l2 = __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(l1, b2), c2), d2));   // lanes = 0 mod 4
                    if (st2) stg_cs(o2, l2);
                    o2 += o2_step;
                    if constexpr (kNarrow) {
                        if (st2f) stg_cs(o2f, l2);
                        o2f += o2_step;
                    }
                }
            }
        }
        if (!(kStudy & kStudyStores) && study_acc == 0x9e3779b9u && (inside & 1u)) stg_cs(static_cast<TOut*>(p.out[0]), 0.0f);   // keeps the folded pixels alive
        }
    }
}

typedef void (*FusedTexFn)(const FusedParams, const TexSet);
template <int kMinCtas, bool kPrefetch, int kOut>
static FusedTexFn fused_tex_variant_t(bool vig, bool pyr) {
    constexpr int V = k1_variant(kOut);
    if (vig) return pyr ? fused_tex_kernel<true, true, kMinCtas, kPrefetch, V> : fused_tex_kernel<true, false, kMinCtas, kPrefetch, V>;
    return pyr ? fused_tex_kernel<false, true, kMinCtas, kPrefetch, V> : fused_tex_kernel<false, false, kMinCtas, kPrefetch, V>;
}
template <int kOut>
static FusedTexFn fused_tex_variant_o(bool vig, bool pyr, int min_ctas, bool prefetch) {
    if (prefetch) {
        if (min_ctas <= 2) return fused_tex_variant_t<2, true, kOut>(vig, pyr);
        return min_ctas == 3 ? fused_tex_variant_t<3, true, kOut>(vig, pyr) : fused_tex_variant_t<4, true, kOut>(vig, pyr);
    }
    if (min_ctas <= 2) return fused_tex_variant_t<2, false, kOut>(vig, pyr);
    return min_ctas == 3 ? fused_tex_variant_t<3, false, kOut>(vig, pyr) : fused_tex_variant_t<4, false, kOut>(vig, pyr);
}
// study: floor-study variants (fp32 only); out_type: MDC_OUT_*
static FusedTexFn fused_tex_variant(bool vig, bool pyr, int min_ctas, bool prefetch, int study, int out_type) {
    if (out_type == MDC_OUT_F16) return fused_tex_variant_o<MDC_OUT_F16>(vig, pyr, min_ctas, prefetch);
    if (out_type == MDC_OUT_U8) return fused_tex_variant_o<MDC_OUT_U8>(vig, pyr, min_ctas, prefetch);
    if (study != kStudyAll && vig && !pyr) {      // floor study: <vignette, no pyramid, 3 CTAs/SM, no prefetch> with parts disabled
        switch (study & kStudyAll) {
            case 0: return fused_tex_kernel<true, false, 3, false, 0>;
            case 1: return fused_tex_kernel<true, false, 3, false, 1>;
            case 2: return fused_tex_kernel<true, false, 3, false, 2>;
            case 3: return fused_tex_kernel<true, false, 3, false, 3>;
            case 4: return fused_tex_kernel<true, false, 3, false, 4>;
            case 5: return fused_tex_kernel<true, false, 3, false, 5>;
            case 6: return fused_tex_kernel<true, false, 3, false, 6>;
            default: break;
        }
    }
    return fused_tex_variant_o<MDC_OUT_F32>(vig, pyr, min_ctas, prefetch);
}
constexpr int kTexSmemBytes = 256 * 32 * 4;

int fused_tex_max_ctas_per_sm(bool vig, bool pyr, int min_ctas, bool prefetch) {
    int n = 0;
    FusedTexFn fn = fused_tex_variant(vig, pyr, min_ctas, prefetch, kStudyAll, MDC_OUT_F32);
    if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kTexSmemBytes) != cudaSuccess) return 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fn, kTexThreads, kTexSmemBytes) != cudaSuccess) return 0;
    return n;
}

cudaError_t launch_fused_tex(const FusedParams& p, const TexSet& texs, int n_chunks, int min_ctas, bool prefetch, int study, int out_type,
                             cudaStream_t stream) {
    if (n_chunks < 1 || n_chunks > kMaxTex || p.tiles_per_cta < 1) return cudaErrorInvalidValue;
    FusedTexFn fn = fused_tex_variant(p.use_vig != 0, p.levels > 1, min_ctas, prefetch, study, out_type);
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kTexSmemBytes);
    if (e != cudaSuccess) return e;
    if (p.carveout > 0 && (e = cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, p.carveout)) != cudaSuccess) return e;
    const dim3 grid(static_cast<unsigned>((p.n_tiles + p.tiles_per_cta - 1) / p.tiles_per_cta), static_cast<unsigned>(n_chunks));
    fn<<<grid, kTexThreads, kTexSmemBytes, stream>>>(p, texs);
    return cudaGetLastError();
}

// bit-wise comparison of two device buffers (self-check of the texture-gather loader at context creation)
__global__ void __launch_bounds__(256) count_mismatch_kernel(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, size_t n,
                                                             unsigned long long* __restrict__ out) {
    unsigned long long bad = 0;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) bad += a[i] != b[i];
    if (bad) atomicAdd(out, bad);
}
cudaError_t launch_count_mismatch(const void* a, const void* b, size_t n_words, unsigned long long* out, cudaStream_t stream) {
    if (n_words == 0) return cudaSuccess;
    size_t blocks = (n_words + 255) / 256;
    blocks = std::min(blocks, grid_cap(8));
    count_mismatch_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(static_cast<const uint32_t*>(a), static_cast<const uint32_t*>(b), n_words, out);
    return cudaGetLastError();
}

// =====================================================================================
// K1a: unMapImage alone (streaming; 1 B in, 4 B out, 4 B vignette per pixel).  T = output element; a narrow T converts at the
// store and, where a K2 pass reads this level, also writes the fp32 pixels to out_f32 (a trailing parameter, so that the float
// instantiation keeps the parameter offsets and the code of the fp32-only kernel).
// =====================================================================================
template <typename T>
__global__ void __launch_bounds__(256) unmap_kernel(const uint8_t* __restrict__ in, T* __restrict__ out, size_t n,
                                                    int n_frames, const float* __restrict__ ginv,
                                                    const float* __restrict__ vinv, unsigned kill, float* __restrict__ out_f32) {
    constexpr bool kNarrow = !std::is_same<T, float>::value;
    __shared__ float lut[256];
    {
        float v = ginv ? ginv[threadIdx.x] : static_cast<float>(threadIdx.x);
        if (kill && threadIdx.x == 255) v = __int_as_float(0x7fc00000);
        lut[threadIdx.x] = v;
    }
    __syncthreads();
    const size_t total = n * static_cast<size_t>(n_frames);
    bool vec = ((n & 3) == 0) && ((reinterpret_cast<uintptr_t>(in) & 3) == 0) && ((reinterpret_cast<uintptr_t>(out) & (4 * sizeof(T) - 1)) == 0) &&
               (!vinv || (reinterpret_cast<uintptr_t>(vinv) & 15) == 0);
    if constexpr (kNarrow) vec = vec && (reinterpret_cast<uintptr_t>(out_f32) & 15) == 0;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    if (vec) {
        const size_t words = total >> 2, nw = n >> 2;
        for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < words; i += stride) {
            const uint32_t v = __ldg(reinterpret_cast<const uint32_t*>(in) + i);
            float4 o = make_float4(lut[v & 0xff], lut[(v >> 8) & 0xff], lut[(v >> 16) & 0xff], lut[v >> 24]);
            if (vinv) {
                const float4 m = __ldg(reinterpret_cast<const float4*>(vinv) + (i % nw));
                o.x = __fmul_rn(o.x, m.x); o.y = __fmul_rn(o.y, m.y); o.z = __fmul_rn(o.z, m.z); o.w = __fmul_rn(o.w, m.w);
            }
            if constexpr (kNarrow) {
                put4(out + 4 * i, o);
                if (out_f32) reinterpret_cast<float4*>(out_f32)[i] = o;
            } else {
                reinterpret_cast<float4*>(out)[i] = o;
            }
        }
    } else {
        for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
            float o = lut[in[i]];
            if (vinv) o = __fmul_rn(o, __ldg(vinv + (i % n)));
            put(out + i, o);
            if constexpr (kNarrow) if (out_f32) out_f32[i] = o;
        }
    }
}

cudaError_t launch_unmap(const uint8_t* in, void* out, int out_type, float* out_f32, size_t n, int n_frames, const float* ginv,
                         const float* vinv, unsigned kill, cudaStream_t stream) {
    const size_t total = n * static_cast<size_t>(n_frames);
    if (total == 0) return cudaSuccess;
    size_t blocks = (total / 4 + 255) / 256;
    blocks = std::min(blocks, grid_cap(16));
    if (blocks < 1) blocks = 1;
    const unsigned g = static_cast<unsigned>(blocks);
    if (out_type == MDC_OUT_F16) unmap_kernel<<<g, 256, 0, stream>>>(in, static_cast<__half*>(out), n, n_frames, ginv, vinv, kill, out_f32);
    else if (out_type == MDC_OUT_U8) unmap_kernel<<<g, 256, 0, stream>>>(in, static_cast<uint8_t*>(out), n, n_frames, ginv, vinv, kill, out_f32);
    else unmap_kernel<<<g, 256, 0, stream>>>(in, static_cast<float*>(out), n, n_frames, ginv, vinv, kill, nullptr);
    return cudaGetLastError();
}

// =====================================================================================
// K1b: undistort<float> alone — float image in, tables from L2, one thread per output pixel
// =====================================================================================
__global__ void __launch_bounds__(256) undistort_f32_kernel(const float* __restrict__ in, float* __restrict__ out, int in_w,
                                                            size_t n_in, size_t n_out, int n_frames,
                                                            const float* __restrict__ remap_x, const float* __restrict__ remap_y) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < n_out; idx += stride) {
        const float sx = __ldg(remap_x + idx), sy = __ldg(remap_y + idx);
        if (sx < 0) {
            for (int f = 0; f < n_frames; ++f) out[static_cast<size_t>(f) * n_out + idx] = 0.0f;
            continue;
        }
        const int xi = static_cast<int>(sx), yi = static_cast<int>(sy);
        const float fx = __fsub_rn(sx, static_cast<float>(xi)), fy = __fsub_rn(sy, static_cast<float>(yi));
        const float fxy = __fmul_rn(fx, fy);
        const float w3 = fxy, w2 = __fsub_rn(fy, fxy), w1 = __fsub_rn(fx, fxy);
        const float w0 = __fadd_rn(__fsub_rn(__fsub_rn(1.0f, fx), fy), fxy);
        const size_t g = static_cast<size_t>(yi) * in_w + xi;
        for (int f = 0; f < n_frames; ++f) {
            const float* s = in + static_cast<size_t>(f) * n_in + g;
            const float v = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(w3, __ldg(s + in_w + 1)), __fmul_rn(w2, __ldg(s + in_w))),
                                                __fmul_rn(w1, __ldg(s + 1))),
                                      __fmul_rn(w0, __ldg(s)));
            out[static_cast<size_t>(f) * n_out + idx] = v;
        }
    }
}

cudaError_t launch_undistort_f32(const float* in, float* out, int in_w, int n_in, int n_out, int n_frames,
                                 const float* remap_x, const float* remap_y, cudaStream_t stream) {
    if (n_out == 0 || n_frames == 0) return cudaSuccess;
    int blocks = (n_out + 255) / 256;
    blocks = static_cast<int>(std::min(static_cast<size_t>(blocks), grid_cap(16)));
    undistort_f32_kernel<<<blocks, 256, 0, stream>>>(in, out, in_w, static_cast<size_t>(n_in), static_cast<size_t>(n_out), n_frames,
                                                     remap_x, remap_y);
    return cudaGetLastError();
}

// =====================================================================================
// K2: stand-alone pyramid level (used for levels beyond the fused epilogue and for API parity).  The source is always fp32; T is
// the destination element, and a narrow T also writes the fp32 level to dst_f32 when a later pass reads it (trailing parameter,
// as for unmap_kernel).
// =====================================================================================
template <typename T>
__global__ void __launch_bounds__(256) pyr_down_kernel(const float* __restrict__ src, int sw, int sh, T* __restrict__ dst,
                                                       int n_frames, float* __restrict__ dst_f32) {
    const int dw = sw >> 1, dh = sh >> 1;
    const size_t per = static_cast<size_t>(dw) * dh, total = per * n_frames;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const size_t f = i / per, r = i - f * per;
        const int y = static_cast<int>(r / dw), x = static_cast<int>(r - static_cast<size_t>(y) * dw);
        const float* s = src + f * static_cast<size_t>(sw) * sh + static_cast<size_t>(2 * y) * sw + 2 * x;
        const float v = __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(__ldg(s), __ldg(s + 1)), __ldg(s + sw)), __ldg(s + sw + 1)));
        put(dst + i, v);
        if constexpr (!std::is_same<T, float>::value) if (dst_f32) dst_f32[i] = v;
    }
}

// Two levels in one pass (used for levels 3+4 behind the fused kernel): each thread owns one 2x2 block of the first
// destination level — i.e. a 4x4 block of the source — writes those up to 4 pixels and, if complete, the pixel of the
// second destination level.  Same arithmetic as two pyr_down_kernel passes (the intermediate values are identical): the first
// level's pixels stay fp32 in registers whatever T is, and a narrow T writes the second level's fp32 pixels to d2_f32 as well.
template <typename T>
__global__ void __launch_bounds__(256) pyr_down2_kernel(const float* __restrict__ src, int sw, int sh, T* __restrict__ d1,
                                                        T* __restrict__ d2, int n_frames, float* __restrict__ d2_f32) {
    const int w1 = sw >> 1, h1 = sh >> 1, w2 = w1 >> 1, h2 = h1 >> 1;
    const int bw = (w1 + 1) >> 1, bh = (h1 + 1) >> 1;
    const size_t per = static_cast<size_t>(bw) * bh, total = per * n_frames;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const size_t f = i / per, r = i - f * per;
        const int by = static_cast<int>(r / bw), bx = static_cast<int>(r - static_cast<size_t>(by) * bw);
        const float* s = src + f * static_cast<size_t>(sw) * sh;
        float v[2][2] = {{0.f, 0.f}, {0.f, 0.f}};
#pragma unroll
        for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
                const int x = 2 * bx + dx, y = 2 * by + dy;
                if (x < w1 && y < h1) {
                    const float* q = s + static_cast<size_t>(2 * y) * sw + 2 * x;
                    v[dy][dx] = __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(__ldg(q), __ldg(q + 1)), __ldg(q + sw)), __ldg(q + sw + 1)));
                    put(d1 + (f * static_cast<size_t>(w1) * h1 + static_cast<size_t>(y) * w1 + x), v[dy][dx]);
                }
            }
        if (bx < w2 && by < h2) {
            const size_t o = f * static_cast<size_t>(w2) * h2 + static_cast<size_t>(by) * w2 + bx;
            const float v2 = __fmul_rn(0.25f, __fadd_rn(__fadd_rn(__fadd_rn(v[0][0], v[0][1]), v[1][0]), v[1][1]));
            put(d2 + o, v2);
            if constexpr (!std::is_same<T, float>::value) if (d2_f32) d2_f32[o] = v2;
        }
    }
}

cudaError_t launch_pyr_down2(const float* src, int sw, int sh, void* d1, void* d2, int out_type, float* d2_f32, int n_frames,
                             cudaStream_t stream) {
    const size_t total = static_cast<size_t>(((sw >> 1) + 1) >> 1) * (((sh >> 1) + 1) >> 1) * n_frames;
    if (total == 0) return cudaSuccess;
    size_t blocks = (total + 255) / 256;
    blocks = std::min(blocks, grid_cap(16));
    const unsigned g = static_cast<unsigned>(blocks);
    if (out_type == MDC_OUT_F16)
        pyr_down2_kernel<<<g, 256, 0, stream>>>(src, sw, sh, static_cast<__half*>(d1), static_cast<__half*>(d2), n_frames, d2_f32);
    else if (out_type == MDC_OUT_U8)
        pyr_down2_kernel<<<g, 256, 0, stream>>>(src, sw, sh, static_cast<uint8_t*>(d1), static_cast<uint8_t*>(d2), n_frames, d2_f32);
    else
        pyr_down2_kernel<<<g, 256, 0, stream>>>(src, sw, sh, static_cast<float*>(d1), static_cast<float*>(d2), n_frames, nullptr);
    return cudaGetLastError();
}

cudaError_t launch_pyr_down(const float* src, int sw, int sh, void* dst, int out_type, float* dst_f32, int n_frames, cudaStream_t stream) {
    const size_t total = static_cast<size_t>(sw >> 1) * (sh >> 1) * n_frames;
    if (total == 0) return cudaSuccess;
    size_t blocks = (total + 255) / 256;
    blocks = std::min(blocks, grid_cap(16));
    const unsigned g = static_cast<unsigned>(blocks);
    if (out_type == MDC_OUT_F16) pyr_down_kernel<<<g, 256, 0, stream>>>(src, sw, sh, static_cast<__half*>(dst), n_frames, dst_f32);
    else if (out_type == MDC_OUT_U8) pyr_down_kernel<<<g, 256, 0, stream>>>(src, sw, sh, static_cast<uint8_t*>(dst), n_frames, dst_f32);
    else pyr_down_kernel<<<g, 256, 0, stream>>>(src, sw, sh, static_cast<float*>(dst), n_frames, nullptr);
    return cudaGetLastError();
}

// =====================================================================================
// distortCoordinates on the device (FOVUndistorter.cpp:280-319), in place, bit-identical to the host: explicit IEEE
// operations in the reference's order, atanf restated from glibc (mdc_atanf.h).
// =====================================================================================
__device__ __forceinline__ void fov_distort_point(float& x, float& y, const DistortConstants& k) {
    const float nx = __fdiv_rn(__fsub_rn(x, k.ocx), k.ofx);
    const float ny = __fdiv_rn(__fsub_rn(y, k.ocy), k.ofy);
    const float rad = __fsqrt_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)));
    float scale = 1.0f;
    if (!(rad == 0.0f || k.omega == 0.0f)) scale = __fdiv_rn(mdc_atanf(__fmul_rn(rad, k.d2t)), __fmul_rn(k.omega, rad));
    x = __fadd_rn(__fmul_rn(__fmul_rn(k.fx, scale), nx), k.cx);
    y = __fadd_rn(__fmul_rn(__fmul_rn(k.fy, scale), ny), k.cy);
}
__global__ void __launch_bounds__(256) fov_distort_kernel(float* __restrict__ xs, float* __restrict__ ys, size_t n, DistortConstants k) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        float x = xs[i], y = ys[i];
        fov_distort_point(x, y, k);
        xs[i] = x;
        ys[i] = y;
    }
}

// vignetteCalib's plane-to-image maps (main_vignetteCalib.cpp:266-284 and :346-357) in one pass: grid point (x, y) of image img is
// projected through hk[img] = H * K_p2idx^-1 (9 floats, row-major, built on the host), distorted, and masked.  pp[r] =
// HK[r,0]*x + HK[r,1]*y + HK[r,2]*1 left to right, then pp[0]/pp[2], pp[1]/pp[2], as the stand-in Eigen product the reference
// program builds against evaluates it.  The mask is `int u_d = X + 0.5` (a double add, then truncation): x86 converts NaN and
// out-of-range values to INT_MIN, __double2int_rz saturates and turns NaN into 0; both fail `u_d > 1 && u_d < wI-2`, so the same
// points are rejected.
__global__ void __launch_bounds__(256) vc_plane_maps_kernel(const float* __restrict__ hk, int gw, size_t gwgh, size_t total, int wI, int hI,
                                                            DistortConstants k, float* __restrict__ xs, float* __restrict__ ys) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const size_t img = i / gwgh, pt = i - img * gwgh;
        const int gy = static_cast<int>(pt / gw), gx = static_cast<int>(pt - static_cast<size_t>(gy) * gw);
        const float* m = hk + 9 * img;
        const float fx = static_cast<float>(gx), fy = static_cast<float>(gy);
        float pp[3];
#pragma unroll
        for (int r = 0; r < 3; ++r)
            pp[r] = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(m + 3 * r), fx), __fmul_rn(__ldg(m + 3 * r + 1), fy)), __fmul_rn(__ldg(m + 3 * r + 2), 1.0f));
        float x = __fdiv_rn(pp[0], pp[2]), y = __fdiv_rn(pp[1], pp[2]);
        fov_distort_point(x, y, k);
        const int u_d = __double2int_rz(__dadd_rn(static_cast<double>(x), 0.5));
        const int v_d = __double2int_rz(__dadd_rn(static_cast<double>(y), 0.5));
        if (!(u_d > 1 && v_d > 1 && u_d < wI - 2 && v_d < hI - 2)) x = y = __int_as_float(0x7fc00000);
        xs[i] = x;
        ys[i] = y;
    }
}
__global__ void __launch_bounds__(256) atanf_kernel(const float* __restrict__ in, float* __restrict__ out, size_t n) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = mdc_atanf(in[i]);
}
static unsigned stream_blocks(size_t n) {
    size_t b = (n + 255) / 256;
    b = std::min(b, grid_cap(16));
    return static_cast<unsigned>(b < 1 ? 1 : b);
}
cudaError_t launch_fov_distort(float* xs, float* ys, size_t n, const DistortConstants& k, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    fov_distort_kernel<<<stream_blocks(n), 256, 0, stream>>>(xs, ys, n, k);
    return cudaGetLastError();
}
cudaError_t launch_vc_plane_maps(const float* hk, int n, int gw, int gh, int wI, int hI, const DistortConstants& k, float* xs, float* ys,
                                 cudaStream_t stream) {
    const size_t gwgh = static_cast<size_t>(gw) * gh, total = gwgh * n;
    if (total == 0) return cudaSuccess;
    vc_plane_maps_kernel<<<stream_blocks(total), 256, 0, stream>>>(hk, gw, gwgh, total, wI, hI, k, xs, ys);
    return cudaGetLastError();
}
cudaError_t launch_atanf(const float* in, float* out, size_t n, cudaStream_t stream) {
    if (n == 0) return cudaSuccess;
    atanf_kernel<<<stream_blocks(n), 256, 0, stream>>>(in, out, n);
    return cudaGetLastError();
}

// =====================================================================================
// K3: responseCalib E-step.  One lane per 4 adjacent pixels (one 32-bit load per exposure), sequential over the n
// exposures in the reference's order, fp64 with explicit non-fused multiplies/adds  ->  bit-identical to
// main_responseCalib.cpp:324-338.
//
// Layout of the work: a warp-task is 128 contiguous pixels; persistent warps take tasks round-robin.  Loads are
// software-pipelined with two register buffers of 8 exposures: while one group is accumulated, the next is in flight.
// Per sample the inner loop is six instructions:
//   PRMT   a = (byte << 8) | lane*8         one byte-permute builds the whole table address (the table row of a value is
//                                           256 bytes = 32 lane slots of one double, so every lookup is conflict-free)
//   LDS.64 g = G[byte]   ·  DMUL prod = g*t  ·  ISETP p = a < 0xff00 (byte != 255, main_responseCalib.cpp:329)
//   @p DADD ENum += t*t  ·  @p DADD ESum += prod        (predicated, so saturated samples are skipped like the reference's `continue`)
// The exposure times sit in shared memory next to the table (one broadcast 64-bit load + one DMUL for t*t per exposure).
// =====================================================================================
constexpr int kEstepGroup = 8;        // exposures per software-pipeline stage
constexpr int kEstepMaxN = 4096;      // exposure times cached in shared memory up to this n; beyond, read through L1
constexpr int kEstepThreads = 384;    // 12 warps; two CTAs per SM share 2 x 96 KB of shared memory
constexpr int kEstepTableBytes = 256 * 256;

// one sample: `a` = table byte offset built by PRMT; both sums only move when the sample is not saturated
__device__ __forceinline__ void estep_sample(uint32_t table, uint32_t a, double ti, double tt, double& esum, double& enumr) {
    asm("{\n\t"
        ".reg .pred p;\n\t"
        ".reg .f64 g, pr;\n\t"
        ".reg .u32 ad;\n\t"
        "add.u32 ad, %2, %3;\n\t"
        "ld.shared.f64 g, [ad];\n\t"
        "mul.rn.f64 pr, g, %4;\n\t"
        "setp.lt.u32 p, %3, 0xff00;\n\t"
        "@!p bra SKIP;\n\t"
        "add.rn.f64 %1, %1, %5;\n\t"
        "add.rn.f64 %0, %0, pr;\n\t"
        "SKIP:\n\t"
        "}"
        : "+d"(esum), "+d"(enumr)
        : "r"(table), "r"(a), "d"(ti), "d"(tt));
}

template <bool kVec>
__device__ __forceinline__ void estep_word(uint32_t v, double ti, double tt, uint32_t table, uint32_t lane8, double esum[4],
                                           double enumr[4], int npx) {
    // PRMT selectors: result byte 0 = lane8 (lane*8 < 256), byte 1 = byte j of v, bytes 2..3 = 0 (upper bytes of lane8)
    estep_sample(table, __byte_perm(v, lane8, 0x5504), ti, tt, esum[0], enumr[0]);
    if (kVec || npx > 1) estep_sample(table, __byte_perm(v, lane8, 0x5514), ti, tt, esum[1], enumr[1]);
    if (kVec || npx > 2) estep_sample(table, __byte_perm(v, lane8, 0x5524), ti, tt, esum[2], enumr[2]);
    if (kVec || npx > 3) estep_sample(table, __byte_perm(v, lane8, 0x5534), ti, tt, esum[3], enumr[3]);
}

template <bool kVec, bool kTimesInSmem>
__device__ __forceinline__ void estep_task(const uint8_t* __restrict__ col, int n, uint32_t npix, int npx, const double* __restrict__ t,
                                           const double* sT, uint32_t table, uint32_t lane8, double* __restrict__ Eout) {
    double esum[4] = {0.0, 0.0, 0.0, 0.0}, enumr[4] = {0.0, 0.0, 0.0, 0.0};
    const uint8_t* next = col;          // the loads walk down the column of this lane's 4 pixels, one exposure per step
    auto load = [&]() -> uint32_t {
        const uint8_t* a = next;
        next += npix;
        if (kVec) return __ldg(reinterpret_cast<const uint32_t*>(a));
        uint32_t v = __ldg(a);
        if (npx > 1) v |= static_cast<uint32_t>(__ldg(a + 1)) << 8;
        if (npx > 2) v |= static_cast<uint32_t>(__ldg(a + 2)) << 16;
        if (npx > 3) v |= static_cast<uint32_t>(__ldg(a + 3)) << 24;
        return v;
    };
    auto acc = [&](uint32_t v, int i) {
        const double ti = kTimesInSmem ? sT[i] : __ldg(t + i);
        estep_word<kVec>(v, ti, __dmul_rn(ti, ti), table, lane8, esum, enumr, npx);
    };
    auto acc8 = [&](const uint32_t (&buf)[kEstepGroup], int base) {
#pragma unroll
        for (int j = 0; j < kEstepGroup; ++j) acc(buf[j], base + j);
    };
    auto load8 = [&](uint32_t (&buf)[kEstepGroup]) {
#pragma unroll
        for (int j = 0; j < kEstepGroup; ++j) buf[j] = load();
    };
    uint32_t a[kEstepGroup], b[kEstepGroup];
    int i0 = 0;
    if (n >= kEstepGroup) load8(a);
    // invariant at the loop head: `a` holds exposures [i0, i0+8), `next` points at exposure i0+8
    for (; i0 + 2 * kEstepGroup <= n; i0 += 2 * kEstepGroup) {
        load8(b);
        acc8(a, i0);
        if (i0 + 3 * kEstepGroup <= n) load8(a);
        acc8(b, i0 + kEstepGroup);
    }
    if (i0 + kEstepGroup <= n) { acc8(a, i0); i0 += kEstepGroup; }
    for (; i0 < n; ++i0) acc(load(), i0);
    for (int j = 0; j < npx; ++j) {
        double e = __ddiv_rn(esum[j], enumr[j]);
        if (e < 0) e = 0;          // 0/0 = NaN survives the clamp, as in the reference
        Eout[j] = e;
    }
}

__global__ void __launch_bounds__(kEstepThreads, 2) estep_kernel(const uint8_t* __restrict__ data, int n, size_t npix,
                                                                const double* __restrict__ t, const double* __restrict__ G,
                                                                double* __restrict__ E, int vec_ok) {
    extern __shared__ __align__(16) double smem_d[];
    // G[256], one 256-byte row per value holding 32 copies (slot = lane): a 64-bit shared load is served per half-warp
    // and every lane reads its own slot, so the data-dependent lookup is bank-conflict-free
    double* sG = smem_d;                                                      // [256][32]
    double* sT = smem_d + kEstepTableBytes / 8;                               // [min(n, kEstepMaxN)] exposure times
    const bool times_in_smem = n <= kEstepMaxN;
    if (times_in_smem)
        for (int i = threadIdx.x; i < n; i += blockDim.x) sT[i] = t[i];
    for (int i = threadIdx.x; i < 256 * 32; i += blockDim.x) sG[i] = G[i >> 5];
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const uint32_t table = static_cast<uint32_t>(__cvta_generic_to_shared(sG));
    const uint32_t lane8 = static_cast<uint32_t>(lane) * 8u;
    const uint32_t npix32 = static_cast<uint32_t>(npix);                     // launch_estep takes an int
    const size_t n_tasks = (npix + 127) / 128;
    const size_t warps_total = static_cast<size_t>(gridDim.x) * (blockDim.x >> 5);
    for (size_t task = static_cast<size_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); task < n_tasks; task += warps_total) {
        const size_t k0 = task * 128 + static_cast<size_t>(lane) * 4;
        if (k0 >= npix) continue;
        const int npx = static_cast<int>(npix - k0 < 4 ? npix - k0 : 4);      // ragged tail of the image
        const uint8_t* col = data + k0;
        if (vec_ok && npx == 4) {
            if (times_in_smem) estep_task<true, true>(col, n, npix32, 4, t, sT, table, lane8, E + k0);
            else estep_task<true, false>(col, n, npix32, 4, t, sT, table, lane8, E + k0);
        } else {
            estep_task<false, false>(col, n, npix32, npx, t, sT, table, lane8, E + k0);
        }
    }
}

// ---- K3, bulk-copy loader (image sizes that are a multiple of 16 pixels): the same arithmetic, but the u8 planes come in
// through the async proxy.  A CTA owns a tile of kEbWarps x 128 pixels; a producer warp streams it plane by plane with 1-D
// cp.async.bulk copies (1536 contiguous bytes each, 8 planes per stage) into a shared-memory ring, full/empty mbarriers
// connect it to the kEbWarps consumer warps (warp = 128 pixels, lane = 4 pixels, one LDS.32 per exposure).  The ring keeps
// 24 planes x 1.5 KB per CTA in flight without holding a register, runs ahead across tile boundaries, and DRAM sees
// 1.5 KB bursts instead of independent 128-byte requests.
//
// The streaming skeleton is shared by the three passes of the calibrator that walk the whole image stack (E-step,
// G-step, rmse); what happens to a word of 4 samples is the `Op`.
constexpr int kEbWarps = 14;                     // consumer warps of the table ops (E-step, rmse: 2 CTAs per SM)
constexpr int kEbPlanes = 8;                     // exposures per stage
constexpr int kEbStages = 3;
constexpr int kEbMaxN = 1024;                    // exposure times served from constant memory up to this n
// Shape of a streaming kernel, fixed by its Op: Op::kWarps consumer warps (+1 producer warp), a tile of kWarps x 128 pixels,
// Op::kRegionBytes of shared memory for the op (lookup table / histograms) in front of the ring, Op::kCtasPerSm resident CTAs.
template <class Op> struct StreamShape {
    static constexpr int kWarps = Op::kWarps;
    static constexpr int kThreads = (kWarps + 1) * 32;
    static constexpr int kTile = kWarps * 128;                       // pixels (= bytes) of one plane per stage row
    static constexpr int kStageBytes = kEbPlanes * kTile;
    static constexpr int kRegionBytes = Op::kRegionBytes;
    static constexpr int kSmemBytes = kRegionBytes + kEbStages * kStageBytes + 2 * kEbStages * 8;
};

// warps: consumer warps that take part (1..Op::kWarps); a tile is warps x 128 pixels (chosen per launch, see launch_stream).
struct StreamArgs { const uint8_t* data; int n; uint32_t npix; const double* t; int warps; };

// Exposure times of the current pass in CONSTANT memory (n <= kEbMaxN): every lane of a warp needs the same t[i], so a shared-memory
// copy costs one (broadcast) LDS.64 wavefront per warp and exposure on the pipe that bounds these kernels — 1 of 10 for the E-step —
// while the constant cache serves it for free (LDC with a warp-uniform index).  The symbol is refilled device-to-device on the
// launching stream before every pass; an event keeps a refill (from any stream of this device) behind the last pass that read it.
__constant__ double c_exposure_t[kEbMaxN];

__device__ __forceinline__ void bulk_load_1d(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ void stream_consumer_barrier(int warps) { asm volatile("bar.sync 1, %0;" ::"r"(warps * 32) : "memory"); }

// producer lane: streams this CTA's tiles, plane group by plane group, as far ahead as the ring allows
template <class Shape>
__device__ __forceinline__ void stream_produce(const StreamArgs& a, uint32_t n_tiles, uint32_t stages, uint32_t bar_full, uint32_t bar_empty) {
    const int n_groups = (a.n + kEbPlanes - 1) / kEbPlanes;
    uint32_t s = 0, ph = 0, it = 0;
    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const uint32_t tile_px = static_cast<uint32_t>(a.warps) * 128u;
        const uint32_t k0 = tile * tile_px;
        const uint32_t bytes = a.npix - k0 < tile_px ? a.npix - k0 : tile_px;      // multiple of 16 (npix is)
        const uint8_t* src = a.data + k0;
        for (int g = 0; g < n_groups; ++g, ++it) {
            if (it >= kEbStages) {
                mbar_wait_backoff(bar_empty + 8u * s, ph ^ 1u);
                // the consumers read this stage through the generic proxy, the copy below writes it through the async proxy
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            }
            const int planes = a.n - g * kEbPlanes < kEbPlanes ? a.n - g * kEbPlanes : kEbPlanes;
            mbar_expect_tx(bar_full + 8u * s, static_cast<uint32_t>(planes) * bytes);
            const uint32_t dst = stages + s * static_cast<uint32_t>(Shape::kStageBytes);
            for (int p = 0; p < planes; ++p) {
                bulk_load_1d(dst + static_cast<uint32_t>(p) * Shape::kTile, src, bytes, bar_full + 8u * s);
                src += a.npix;
            }
            if (++s == kEbStages) { s = 0; ph ^= 1u; }
        }
    }
}

template <class Op, bool kTimesInConst>
__device__ __forceinline__ void stream_consume(const StreamArgs& a, uint32_t n_tiles, uint32_t stages, uint32_t bar_full,
                                               uint32_t bar_empty, Op& op) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t mine = stages + warp * 128u + lane * 4u;
    const int n_groups = (a.n + kEbPlanes - 1) / kEbPlanes;
    uint32_t s = 0, ph = 0;
    for (uint32_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const size_t k0 = static_cast<size_t>(tile) * (static_cast<uint32_t>(a.warps) * 128u) + warp * 128u + lane * 4u;
        op.begin_tile(k0, k0 < a.npix);
        for (int g = 0; g < n_groups; ++g) {
            mbar_wait(bar_full + 8u * s, ph);
            const uint32_t src = mine + s * static_cast<uint32_t>(StreamShape<Op>::kStageBytes);
            const int i0 = g * kEbPlanes;
            auto plane = [&](int p) {
                uint32_t v;
                asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(src + static_cast<uint32_t>(p) * StreamShape<Op>::kTile));
                op.word(v, kTimesInConst ? c_exposure_t[i0 + p] : __ldg(a.t + i0 + p));
            };
            if (i0 + kEbPlanes <= a.n) {
                if (Op::kUnroll) {
#pragma unroll
                    for (int p = 0; p < kEbPlanes; ++p) plane(p);
                } else {
#pragma unroll 1
                    for (int p = 0; p < kEbPlanes; ++p) plane(p);
                }
            } else {
                for (int p = 0; i0 + p < a.n; ++p) plane(p);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(bar_empty + 8u * s);
            if (++s == kEbStages) { s = 0; ph ^= 1u; }
            op.after_group();
        }
        op.end_tile(k0, k0 < a.npix);
    }
}

template <class Op>
__global__ void __launch_bounds__(StreamShape<Op>::kThreads, Op::kCtasPerSm) rc_stream_kernel(StreamArgs a, typename Op::Params prm) {
    using Shape = StreamShape<Op>;
    extern __shared__ __align__(128) uint8_t smem_b[];
    const uint32_t stages = smem_u32(smem_b + Shape::kRegionBytes);                   // [kEbStages][kEbPlanes][kTile]
    const uint32_t bar_full = stages + kEbStages * Shape::kStageBytes, bar_empty = bar_full + 8u * kEbStages;
    const bool times_in_const = a.n <= kEbMaxN;                                        // launch_stream filled c_exposure_t
    if (threadIdx.x == 0) {
        for (int i = 0; i < kEbStages; ++i) { mbar_init(bar_full + 8u * i, 1); mbar_init(bar_empty + 8u * i, static_cast<uint32_t>(a.warps)); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    Op::prologue(smem_b, prm);
    __syncthreads();
    const uint32_t tile_px = static_cast<uint32_t>(a.warps) * 128u;
    const uint32_t n_tiles = (a.npix + tile_px - 1) / tile_px;
    if ((threadIdx.x >> 5) >= a.warps && (threadIdx.x >> 5) != Shape::kWarps) return;  // consumer warps beyond the tile width sit this launch out
    if ((threadIdx.x >> 5) == Shape::kWarps) {
        if ((threadIdx.x & 31) == 0) stream_produce<Shape>(a, n_tiles, stages, bar_full, bar_empty);
        return;
    }
    Op op(smem_b, prm);
    op.warps = a.warps;
    if (times_in_const) stream_consume<Op, true>(a, n_tiles, stages, bar_full, bar_empty, op);
    else stream_consume<Op, false>(a, n_tiles, stages, bar_full, bar_empty, op);
    op.epilogue(smem_b, prm);
}

// G[256] -> one 256-byte row per value holding 32 copies (see estep_kernel)
__device__ __forceinline__ void fill_lane_table(uint8_t* region, const double* __restrict__ G) {
    double* sG = reinterpret_cast<double*>(region);
    for (int i = threadIdx.x; i < 256 * 32; i += blockDim.x) sG[i] = G[i >> 5];
}

// E-step (main_responseCalib.cpp:324-338)
struct EstepOp {
    struct Params { const double* G; double* E; };
    static constexpr bool kUnroll = true;
    static constexpr int kWarps = kEbWarps, kRegionBytes = kEstepTableBytes, kCtasPerSm = 2;
    static __device__ __forceinline__ void prologue(uint8_t* region, const Params& p) { fill_lane_table(region, p.G); }
    uint32_t table, lane8;
    int warps = kEbWarps;         // active consumer warps of this launch (set by the kernel)
    double* E;
    double esum[4], enumr[4];
    __device__ __forceinline__ EstepOp(uint8_t* region, const Params& p) : table(smem_u32(region)), lane8((threadIdx.x & 31) * 8u), E(p.E) {}
    __device__ __forceinline__ void begin_tile(size_t, bool) {
#pragma unroll
        for (int j = 0; j < 4; ++j) { esum[j] = 0.0; enumr[j] = 0.0; }
    }
    __device__ __forceinline__ void word(uint32_t v, double ti) { estep_word<true>(v, ti, __dmul_rn(ti, ti), table, lane8, esum, enumr, 4); }
    __device__ __forceinline__ void end_tile(size_t k0, bool active) {
        if (!active) return;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            double e = __ddiv_rn(esum[j], enumr[j]);
            if (e < 0) e = 0;          // 0/0 = NaN survives the clamp, as in the reference
            E[k0 + j] = e;
        }
    }
    __device__ __forceinline__ void after_group() {}
    __device__ __forceinline__ void epilogue(uint8_t*, const Params&) {}
};

// ---- G-step sums in fixed point.  GSum[b] (main_responseCalib.cpp:295) is one sequential fp64 chain over 10^9 samples in the
// reference; no parallel order reproduces its roundings, and fp64 atomics make the result depend on the order in which threads
// happen to arrive.  So every product E[k]*t[i] — rounded to fp64 exactly as the reference rounds it — is turned into an integer
// multiple of 2^-s and summed in integer arithmetic, which is associative: the bits of G do not depend on the launch
// geometry, on the timing of the atomics or on how often the pass is repeated.  s is chosen from the data (GstepScale: the
// largest finite |E| and |t| of the pass) such that every product is below 2^48 units; the conversion is one DADD with
// 1.5 * 2^52 (round to nearest even), so a sample is off by at most 2^-48 of the largest product — the sum of 4 * 10^6 samples
// of a bin is closer to the exact sum than the reference's own chain is.  Non-finite products (E = NaN of an all-saturated
// pixel meeting t = 0, a NaN exposure time, a product that overflows ...) go to a separate fp64 accumulator so that they poison
// G as they do in the reference; they do not change the scale, so every finite product keeps its 2^-48 resolution.
//
// Integer sums are also what makes the histogram cheap: shared memory has native 32-bit integer atomics (ATOMS.ADD, one
// wavefront per conflict-free warp instruction) but only a compare-and-swap loop for 64-bit ones (LDS.64 + ATOMS.CAS.64, a
// load, a compare and a retry per update; scripts/probes/smem_atomic_probe.cu times the two).
// A sample is therefore split into three limbs — bits 0-15, bits 16-31 and the signed rest, which are one LOP, one SHF and one
// IADD away from the two words of the DADD's result — that are added to three u32 histograms, and the histograms are folded
// into 64-bit totals long before a limb can overflow.
constexpr double kFxMagic = 6755399441055744.0;      // 1.5 * 2^52
constexpr double kFxLimit = 281474976710656.0;       // 2^48: scaled products stay below it
// bit patterns of max finite |E[k]|, |t[i]| (non-negative doubles order like integers); bad_t != 0: a non-finite exposure time exists.
// Four u64 words, so that the ranks of a pixel-sharded run can agree on one scale with a single all-reduce(MAX).
struct GstepScale { unsigned long long max_e_bits, max_t_bits, bad_t, reserved; };

// s with |E*t| * 2^s < 2^48 for every FINITE product E*t of the pass: s = 47 - ilogb(max|E| * max|t|), the exponent of that product
// taken from the two exponents and the product of the two mantissas, so that it exists where the product itself would overflow or
// underflow.  A product that overflows is not finite and goes to the fp64 side sums; every finite one is below 2^1024, so s need not
// go below 48 - 1024.  The range is wide (up to 47 + 2 * 1074), so 2^s is applied with scalbn, or as a multiply where it is a double.
constexpr int kFxMinScale = 48 - 1024;
__device__ __forceinline__ int gstep_scale_exponent(const GstepScale& sc) {
    const double e = __longlong_as_double(static_cast<long long>(sc.max_e_bits)), t = __longlong_as_double(static_cast<long long>(sc.max_t_bits));
    if (!(e > 0.0) || !(t > 0.0)) return 0;
    const int ee = ilogb(e), et = ilogb(t);
    const int s = 47 - (ee + et + ilogb(__dmul_rn(scalbn(e, -ee), scalbn(t, -et))));
    return s < kFxMinScale ? kFxMinScale : s;
}
// The fast path forms (E * 2^s) * t, which is the reference's E * t times 2^s exactly when E * 2^s is exact (checked per lane) and
// neither E * t nor the scaled product can leave the normal range in a way that changes an integer: for s in [-975, 1020] every
// product is below 2^1023 and a product that underflows is worth less than 2^-2 units.  Outside that range, and in a pass with a
// non-finite exposure time, every sample goes through the checked path.
__device__ __forceinline__ bool gstep_fast_pass(const GstepScale& sc, int s) { return !sc.bad_t && s > kFxMinScale && s <= 1020; }
// x (|x| < 2^48, already scaled) -> the integer nearest to it, as three limbs: value = l0 + l1 * 2^16 + l2 * 2^32, 0 <= l0, l1 < 2^16,
// -2^16 <= l2 < 2^16.  bits(x + 1.5 * 2^52) = 0x4338000000000000 + value, so the limbs are bit fields of the sum.
struct FxLimbs { uint32_t l0, l1; int l2; };
__device__ __forceinline__ FxLimbs fx_limbs(double x) {
    const double y = __dadd_rn(x, kFxMagic);
    const uint32_t lo = static_cast<uint32_t>(__double2loint(y));
    FxLimbs r;
    r.l0 = lo & 0xffffu;
    r.l1 = lo >> 16;
    r.l2 = __double2hiint(y) - 0x43380000;
    return r;
}
__device__ __forceinline__ bool fx_in_range(double x) { return fabs(x) < kFxLimit; }      // false for NaN
// 128-bit two's complement accumulators in global memory: {lo, hi} += {lo_part, hi_part} (order-independent: modular arithmetic)
__device__ __forceinline__ void fx_flush(unsigned long long* g_lo, unsigned long long* g_hi, unsigned long long lo_part, long long hi_part) {
    const unsigned long long old = atomicAdd(g_lo, lo_part);
    const unsigned long long carry = old + lo_part < old ? 1ull : 0ull;
    const unsigned long long h = static_cast<unsigned long long>(hi_part) + carry;
    if (h) atomicAdd(g_hi, h);
}
__device__ __forceinline__ void fx_flush_limb_totals(unsigned long long* g_lo, unsigned long long* g_hi, long long t0, long long t1, long long t2) {
    const __int128 v = static_cast<__int128>(t0) + (static_cast<__int128>(t1) << 16) + (static_cast<__int128>(t2) << 32);
    const unsigned long long lo = static_cast<unsigned long long>(v);
    const long long hi = static_cast<long long>(v >> 64);
    if (lo | static_cast<unsigned long long>(hi)) fx_flush(g_lo, g_hi, lo, hi);
}
// device scratch of one G-step pass (all zeroed by launch_rc_gstep_accum before the pass)
struct GstepFx {
    GstepScale* scale;
    unsigned long long* lo;      // [256]
    unsigned long long* hi;      // [256]
    double* special;             // [256] fp64 sums of the samples fixed point cannot hold
};

// G-step accumulation (main_responseCalib.cpp:290-299): GSum[b] += E[k]*t[i], GNum[b]++ for b != 255.  One CTA per SM with 28
// consumer warps keeps the histograms in shared memory as planes of [256 values][32 slots] u32 (slot = lane, 128 bytes per value:
// every warp-wide ATOMS.ADD is bank-conflict-free, and two threads only collide when the same lane of two warps meets the same
// value at the same moment): three limb planes and, in the first pass, a count plane (kCount = false: the caller already holds
// GNum — it depends on the images only, so the optimisation loop computes it once).  One PRMT + one LEA build each address.
// A slot receives at most 4 x 28 adds per exposure, i.e. a limb could overflow after 2^15 / 112 = 292 exposures; every 160
// exposures each warp therefore folds its share of the (plane, value) rows into 64-bit totals: it takes a slot's value with an
// atomic exchange against zero — the adds of the other warps go on around it, so no barrier is needed — and sums the 32 slots
// with REDUX.  The ring lets warps drift apart by at most 24 exposures, so a slot sees at most 4 x 28 x (160 + 48) = 23 296 adds
// between folds.  At the end the three totals of a bin are combined into one 128-bit number and added to the global accumulators.
constexpr int kGstepWarps = 28;
constexpr int kGstepPlaneBytes = 256 * 128;
constexpr int kGstepDrainGroups = 20;      // plane groups (of kEbPlanes exposures) between two folds
__device__ __forceinline__ void gstep_add(uint8_t* hist, uint32_t a, const FxLimbs& v, bool count) {
    uint8_t* p = hist + (a >> 1);
    atomicAdd(reinterpret_cast<unsigned*>(p), v.l0);
    atomicAdd(reinterpret_cast<unsigned*>(p + kGstepPlaneBytes), v.l1);
    atomicAdd(reinterpret_cast<int*>(p + 2 * kGstepPlaneBytes), v.l2);
    if (count) atomicAdd(reinterpret_cast<unsigned*>(p + 3 * kGstepPlaneBytes), 1u);
}
// one word with every sample range-checked (E * 2^s not exact for one of the lane's pixels, or no fast path in this pass): the
// reference's product E * t, then scaled by 2^s; a free function with everything passed by value so that the op's state stays in
// registers.  e0..e3 are the unscaled E.
template <bool kCount>
static __device__ __noinline__ void gstep_word_checked(uint8_t* hist, double* special, uint32_t lane8, int s, uint32_t v, double ti,
                                                       double e0, double e1, double e2, double e3) {
#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
        const uint32_t a = ((v >> (8 * j)) & 0xffu) << 8 | lane8;
        if (a >= 0xff00u) continue;      // saturated, :293
        const double p = __dmul_rn(j == 0 ? e0 : (j == 1 ? e1 : (j == 2 ? e2 : e3)), ti);      // :295
        const double x = scalbn(p, s);   // exact, or (below 2^-1022) worth nothing after rounding to an integer
        if (fx_in_range(x)) {
            gstep_add(hist, a, fx_limbs(x), kCount);
        } else {                         // only a non-finite product
            atomicAdd(special + (a >> 8), p);
            if (kCount) atomicAdd(reinterpret_cast<unsigned*>(hist + (a >> 1) + 3 * kGstepPlaneBytes), 1u);
        }
    }
}
template <bool kCount>
struct GstepOp {
    struct Params { const double* E; GstepFx fx; unsigned long long* gnum; };
    static constexpr bool kUnroll = true;
    static constexpr int kPlanes = kCount ? 4 : 3;
    static constexpr int kWarps = kGstepWarps, kCtasPerSm = 1;
    static constexpr int kRegionBytes = kPlanes * (kGstepPlaneBytes + 256 * 8);      // the planes, then long long totals[kPlanes][256]
    static_assert(4 * kGstepWarps * (kGstepDrainGroups * kEbPlanes + 2 * kEbStages * kEbPlanes) < (1 << 15), "a limb slot could overflow between two folds");
    static __device__ __forceinline__ void prologue(uint8_t* region, const Params&) {
        uint32_t* z = reinterpret_cast<uint32_t*>(region);
        for (int i = threadIdx.x; i < kRegionBytes / 4; i += blockDim.x) z[i] = 0u;
    }
    uint8_t* hist;
    int warps = kWarps;               // active consumer warps of this launch (set by the kernel)
    uint32_t lane8;
    int groups_since_fold;
    const double* E;
    double* special;
    double scale;                     // 2^s, or 0 if this pass has no fast path (gstep_fast_pass)
    double e[4];                      // E * 2^s (fast path) or E (checked path)
    uint32_t mode;                    // 0: fast path; 1: every sample range-checked (E * 2^s not exact for one of this lane's pixels, or no fast path); 2: no pixels
    int s;
    __device__ __forceinline__ GstepOp(uint8_t* region, const Params& p)
        : hist(region), lane8((threadIdx.x & 31) * 8u), groups_since_fold(0), E(p.E), special(p.fx.special), mode(2u) {
        s = gstep_scale_exponent(*p.fx.scale);
        scale = gstep_fast_pass(*p.fx.scale, s) ? scalbn(1.0, s) : 0.0;
    }
    __device__ __forceinline__ void begin_tile(size_t k0, bool act) {
        mode = !act ? 2u : (scale == 0.0 ? 1u : 0u);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const double ek = act ? E[k0 + j] : 0.0;
            const double sk = __dmul_rn(ek, scale);
            // exact unless it overflowed (or E is not finite) or lost bits below 2^-1022; then (E * 2^s) * t != (E * t) * 2^s
            if (!(fabs(sk) <= DBL_MAX) || (fabs(sk) < DBL_MIN && ek != 0.0)) mode |= 1u;
            e[j] = sk;
        }
        if (mode == 1u) {
#pragma unroll
            for (int j = 0; j < 4; ++j) e[j] = E[k0 + j];
        }
    }
    // a: (value << 8) | lane * 8, i.e. twice the byte offset of this lane's slot in a plane.  Saturated samples (:293) are not skipped:
    // they land in the rows of value 255, which nobody reads — cheaper than a predicate or a branch around the atomics.
    __device__ __forceinline__ void add(uint32_t a, const FxLimbs& v) { gstep_add(hist, a, v, kCount); }
    __device__ __forceinline__ void word(uint32_t v, double ti) {
        if (mode) {
            if (mode == 1u) gstep_word_checked<kCount>(hist, special, lane8, s, v, ti, e[0], e[1], e[2], e[3]);
            return;
        }
        add(__byte_perm(v, lane8, 0x5504), fx_limbs(__dmul_rn(e[0], ti)));
        add(__byte_perm(v, lane8, 0x5514), fx_limbs(__dmul_rn(e[1], ti)));
        add(__byte_perm(v, lane8, 0x5524), fx_limbs(__dmul_rn(e[2], ti)));
        add(__byte_perm(v, lane8, 0x5534), fx_limbs(__dmul_rn(e[3], ti)));
    }
    // this warp's share of the (plane, value) rows -> totals; safe while other warps keep adding (see above)
    __device__ __forceinline__ void fold() {
        const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        long long* totals = reinterpret_cast<long long*>(hist + kPlanes * kGstepPlaneBytes);
#pragma unroll 2
        for (int r = warp; r < kPlanes * 256; r += warps) {
            unsigned* slot = reinterpret_cast<unsigned*>(hist + r * 128) + lane;
            const unsigned cur = atomicExch(slot, 0u);      // read and clear in one atomic: nothing another warp adds can be lost
            long long sum;
            if ((r >> 8) == 2) {            // the signed limb
                const int c = static_cast<int>(cur);
                sum = static_cast<long long>(__reduce_add_sync(0xffffffffu, c & 0xffff)) + (static_cast<long long>(__reduce_add_sync(0xffffffffu, c >> 16)) << 16);
            } else {
                sum = static_cast<long long>(__reduce_add_sync(0xffffffffu, cur & 0xffffu)) + (static_cast<long long>(__reduce_add_sync(0xffffffffu, cur >> 16)) << 16);
            }
            if (lane == 0 && sum) totals[r] += sum;
        }
    }
    __device__ __forceinline__ void after_group() {
        if (++groups_since_fold == kGstepDrainGroups) { groups_since_fold = 0; fold(); }
    }
    __device__ __forceinline__ void end_tile(size_t, bool) {}
    __device__ __forceinline__ void epilogue(uint8_t* region, const Params& p) {
        stream_consumer_barrier(warps);      // all adds of all warps are in
        fold();
        stream_consumer_barrier(warps);
        const long long* totals = reinterpret_cast<const long long*>(region + kPlanes * kGstepPlaneBytes);
        for (int b = threadIdx.x; b < 255; b += warps * 32) {
            fx_flush_limb_totals(p.fx.lo + b, p.fx.hi + b, totals[b], totals[256 + b], totals[512 + b]);
            if (kCount && totals[768 + b]) atomicAdd(p.gnum + b, static_cast<unsigned long long>(totals[768 + b]));
        }
    }
};

// rmse() (main_responseCalib.cpp:50-69): e = sum (G[b] - t*E)^2 * 1e-10 over finite residuals of unsaturated samples, num = count.
// The reference keeps e in a long double, so its bits are out of reach anyway; what is kept exact is every residual r (one DMUL,
// one DADD, as the reference rounds it), the finite test on it and the count.  The squares of a word's four samples are summed
// with DFMA (saturated ones predicated off) and the factor 1e-10 is applied once at the end; a word whose partial sum is not finite
// — some r is NaN / inf, or a square overflowed — or is 2^900 or more is redone sample by sample in the reference's own form
// (r*r*1e-10).  The bound keeps the unscaled sum finite over up to 2^34 words per thread (2^934 < 2^1024), so squares of residuals
// near 1e153, each finite, cannot add up to inf where the reference's scaled sum does not.  Five instructions per sample instead of
// twelve; saturated samples are predicated off.
constexpr uint32_t kRmseFastBelow = 0x78300000u;      // high word of 2^900 (biased exponent 1023 + 900)
struct RmseChecked { double err; unsigned dropped; };
// one word, sample by sample, in the reference's own form; a free function with everything passed by value so that the op's state
// stays in registers
static __device__ __noinline__ RmseChecked rmse_word_checked(uint32_t table, uint32_t lane8, uint32_t v, double ti, double e0, double e1, double e2, double e3) {
    RmseChecked out{0.0, 0u};
#pragma unroll 1
    for (int j = 0; j < 4; ++j) {
        const uint32_t a = ((v >> (8 * j)) & 0xffu) << 8 | lane8;
        if (a >= 0xff00u) continue;                                    // :56 (not counted by the caller either)
        const double ek = j == 0 ? e0 : (j == 1 ? e1 : (j == 2 ? e2 : e3));
        double g;
        asm("ld.shared.f64 %0, [%1];" : "=d"(g) : "r"(table + a));
        const double r = __dsub_rn(g, __dmul_rn(ti, ek));              // :57
        if ((static_cast<uint32_t>(__double2hiint(r)) & 0x7ff00000u) == 0x7ff00000u) { ++out.dropped; continue; }      // :58
        out.err = __dadd_rn(out.err, __dmul_rn(__dmul_rn(r, r), 1e-10));      // :59
    }
    return out;
}
struct RmseOp {
    struct Params { const double* G; const double* E; double* partials; };      // partials[2*cta] = {error, count} of one CTA
    static constexpr bool kUnroll = true;
    static constexpr int kWarps = kEbWarps, kRegionBytes = kEstepTableBytes, kCtasPerSm = 2;
    static __device__ __forceinline__ void prologue(uint8_t* region, const Params& p) { fill_lane_table(region, p.G); }
    uint32_t table, lane8;
    int warps = kEbWarps;             // active consumer warps of this launch (set by the kernel)
    const double* E;
    double e[4];
    double sq, err_checked;           // sum of r^2 (fast path), sum of r^2 * 1e-10 (words redone sample by sample)
    unsigned cnt;
    unsigned long long cnt_total;
    bool active;
    __device__ __forceinline__ RmseOp(uint8_t* region, const Params& p)
        : table(smem_u32(region)), lane8((threadIdx.x & 31) * 8u), E(p.E), sq(0.0), err_checked(0.0), cnt(0u), cnt_total(0ull), active(false) {}
    __device__ __forceinline__ void begin_tile(size_t k0, bool act) {
        active = act;
#pragma unroll
        for (int j = 0; j < 4; ++j) e[j] = act ? E[k0 + j] : 0.0;
    }
    __device__ __forceinline__ double residual(uint32_t a, double ek, double ti) const {
        double g;
        asm("ld.shared.f64 %0, [%1];" : "=d"(g) : "r"(table + a));
        return __dsub_rn(g, __dmul_rn(ti, ek));      // :57
    }
    // w += r^2 and cnt += 1 unless the sample is saturated (a = (value << 8) | lane * 8).  No branch (random data has a saturated byte
    // in 40 % of the warp-words) and no 64-bit select: clearing the HIGH word of r leaves a subnormal number whose square is +0.
    __device__ __forceinline__ void square(uint32_t a, double r, double& w) {
        int hi;
        asm("{\n\t.reg .pred p;\n\tsetp.lt.u32 p, %3, 0xff00;\n\t@p add.u32 %0, %0, 1;\n\tselp.b32 %1, %2, 0, p;\n\t}" : "+r"(cnt), "=r"(hi) : "r"(__double2hiint(r)), "r"(a));
        const double rr = __hiloint2double(hi, __double2loint(r));
        w = fma(rr, rr, w);
    }
    __device__ __forceinline__ void word(uint32_t v, double ti) {
        if (!active) return;
        const uint32_t a0 = __byte_perm(v, lane8, 0x5504), a1 = __byte_perm(v, lane8, 0x5514), a2 = __byte_perm(v, lane8, 0x5524), a3 = __byte_perm(v, lane8, 0x5534);
        const double r0 = residual(a0, e[0], ti), r1 = residual(a1, e[1], ti), r2 = residual(a2, e[2], ti), r3 = residual(a3, e[3], ti);
        double w01 = 0.0, w23 = 0.0;
        square(a0, r0, w01); square(a2, r2, w23); square(a1, r1, w01); square(a3, r3, w23);
        const double w = w01 + w23;
        if ((static_cast<uint32_t>(__double2hiint(w)) & 0x7ff00000u) < kRmseFastBelow) {      // finite and below 2^900: four finite residuals (or saturated samples)
            sq += w;
        } else {
            const RmseChecked c = rmse_word_checked(table, lane8, v, ti, e[0], e[1], e[2], e[3]);
            err_checked = __dadd_rn(err_checked, c.err);
            cnt -= c.dropped;
        }
    }
    __device__ __forceinline__ void after_group() {}
    __device__ __forceinline__ void end_tile(size_t, bool) { cnt_total += cnt; cnt = 0u; }
    __device__ __forceinline__ void epilogue(uint8_t* region, const Params& p) {
        double err = __dadd_rn(__dmul_rn(sq, 1e-10), err_checked);
        double c = static_cast<double>(cnt_total);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            err = __dadd_rn(err, __shfl_xor_sync(0xffffffffu, err, o));
            c = __dadd_rn(c, __shfl_xor_sync(0xffffffffu, c, o));
        }
        stream_consumer_barrier(warps);                 // every warp is done with the lookup table: reuse its first bytes
        double* part = reinterpret_cast<double*>(region);
        if ((threadIdx.x & 31) == 0) { part[2 * (threadIdx.x >> 5)] = err; part[2 * (threadIdx.x >> 5) + 1] = c; }
        stream_consumer_barrier(warps);
        if (threadIdx.x == 0) {
            double se = 0.0, sc = 0.0;
            for (int w = 0; w < warps; ++w) { se = __dadd_rn(se, part[2 * w]); sc = __dadd_rn(sc, part[2 * w + 1]); }
            p.partials[2 * blockIdx.x] = se;            // no atomics: the CTA partials are folded in CTA order by rc_fold_pairs_kernel,
            p.partials[2 * blockIdx.x + 1] = sc;        // so two runs over the same data give the same bits
        }
    }
};

static cudaEvent_t g_exposure_reader[64] = {};      // per device: recorded behind the last pass that read c_exposure_t
static std::mutex g_exposure_mutex;                 // held from the wait on that event through its record (and over its creation)
template <class Op>
static cudaError_t launch_stream(const StreamArgs& a, const typename Op::Params& prm, cudaStream_t stream, int* grid_out = nullptr) {
    int dev = 0, sms = 132, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    using Shape = StreamShape<Op>;
    constexpr int kW = Shape::kWarps;
    cudaError_t e = cudaFuncSetAttribute(rc_stream_kernel<Op>, cudaFuncAttributeMaxDynamicSharedMemorySize, Shape::kSmemBytes);
    if (e != cudaSuccess) return e;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rc_stream_kernel<Op>, Shape::kThreads, Shape::kSmemBytes);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) per_sm = 1;
    // Tile width (consumer warps per CTA).  A CTA works through its tiles one after the other, and per-tile time is modelled as
    // growing like (2.6 + warps) for the 14-warp ops (a model from the project's earlier target, not re-measured on H100;
    // scripts/stream_warps_sweep.py measures it), so the width that minimises rounds x (2.6 + warps) fills the persistent CTAs best.
    // On H100 (132 SMs x 2 CTAs) 1 MP runs as 782 tiles of 10 warps in 3 rounds (14 warps: 559 tiles, also 3 rounds, the last one
    // short), and a slice of 125 k pixels (1 MP pixel-sharded over 8 GPUs) as 245 tiles of 4 warps on all SMs instead of 70
    // full-width tiles on about a quarter of them.  Ties go to the wider tile (fewer, longer bulk copies).
    const long long slots = static_cast<long long>(sms) * per_sm;
    int best_w = kW;
    double best_cost = -1.0;
    for (int w = kW; w >= 1; --w) {
        const long long tiles_w = (static_cast<long long>(a.npix) + w * 128 - 1) / (w * 128);
        const double cost = static_cast<double>((tiles_w + slots - 1) / slots) * (2.6 * kW / 14.0 + w);
        if (best_cost < 0 || cost < best_cost) { best_cost = cost; best_w = w; }
    }
    if (const char* ov = getenv("MDC_STREAM_WARPS")) {      // measurement knob
        const int w = atoi(ov);
        if (w >= 1 && w <= kW) best_w = w;
    }
    StreamArgs args = a;
    args.warps = best_w;
    const long long tiles = (static_cast<long long>(a.npix) + best_w * 128 - 1) / (best_w * 128);
    long long grid = slots;
    if (grid > tiles) grid = tiles;
    if (grid_out) *grid_out = static_cast<int>(grid);
    // exposure times -> constant memory (device-to-device, on this stream), behind the last pass that read the symbol
    cudaEvent_t* last_reader = g_exposure_reader;      // one event per device, shared by the three ops (they share the symbol)
    const bool use_const = a.n > 0 && a.n <= kEbMaxN && dev >= 0 && dev < 64;      // (no frames: nothing to copy, t may be null)
    // The symbol is shared by every context and host thread: a pass that waited on the event before another one recorded it would
    // overwrite the times that one's kernel still reads, so wait, copy, launch and record happen under one lock.
    std::unique_lock<std::mutex> lock(g_exposure_mutex, std::defer_lock);
    if (use_const) {
        lock.lock();
        if (!last_reader[dev] && (e = cudaEventCreateWithFlags(&last_reader[dev], cudaEventDisableTiming)) != cudaSuccess) return e;
        else if ((e = cudaStreamWaitEvent(stream, last_reader[dev], 0)) != cudaSuccess) return e;
        if ((e = cudaMemcpyToSymbolAsync(c_exposure_t, a.t, static_cast<size_t>(a.n) * sizeof(double), 0, cudaMemcpyDeviceToDevice, stream)) != cudaSuccess) return e;
    }
    rc_stream_kernel<Op><<<static_cast<unsigned>(grid), Shape::kThreads, Shape::kSmemBytes, stream>>>(args, prm);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    return use_const ? cudaEventRecord(last_reader[dev], stream) : cudaSuccess;
}
// the bulk-copy loader needs 16-byte aligned rows
static bool stream_ok(const uint8_t* data, int npix) {
    static const bool allow = [] { const char* e = getenv("MDC_ESTEP_BULK"); return !(e && e[0] == '0'); }();      // A/B knob
    return allow && npix % 16 == 0 && (reinterpret_cast<uintptr_t>(data) & 15) == 0;
}

cudaError_t launch_estep(const uint8_t* data, int n, int npix, const double* t, const double* G, double* E, cudaStream_t stream) {
    if (npix <= 0) return cudaSuccess;
    int dev = 0, sms = 132, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (stream_ok(data, npix))
        return launch_stream<EstepOp>(StreamArgs{data, n, static_cast<uint32_t>(npix), t, kEbWarps}, EstepOp::Params{G, E}, stream);
    const int vec_ok = (npix % 4 == 0) && ((reinterpret_cast<uintptr_t>(data) & 3) == 0);
    const size_t smem = kEstepTableBytes + static_cast<size_t>(kEstepMaxN) * sizeof(double);      // 96 KB
    cudaError_t e = cudaFuncSetAttribute(estep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, estep_kernel, kEstepThreads, smem);
    if (e != cudaSuccess) return e;
    if (per_sm < 1) per_sm = 1;
    const int warps = kEstepThreads / 32;
    const long long tasks = (static_cast<long long>(npix) + 127) / 128;
    long long grid = static_cast<long long>(sms) * per_sm;
    if (grid * warps > tasks) grid = (tasks + warps - 1) / warps;
    estep_kernel<<<static_cast<unsigned>(grid), kEstepThreads, smem, stream>>>(data, n, static_cast<size_t>(npix), t, G, E, vec_ok);
    return cudaGetLastError();
}

// =====================================================================================
// responseCalib building blocks around the E-step (SURVEY.md §8f N2): saturation leak padding, initial irradiance,
// G-step, rescale, rmse.  Integer / per-element work is bit-exact; the two global reductions (G-step bins, rmse)
// are order-dependent in the reference (one long sequential fp64 / long-double sum), so they match to rounding only.
// =====================================================================================

// 3x3 dilation of the value 255 around INTERIOR saturated pixels, main_responseCalib.cpp:212-236 (one iteration).
__global__ void __launch_bounds__(256) rc_leak_padding_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int n, int w, int h) {
    const size_t per = static_cast<size_t>(w) * h, total = per * n;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const size_t f = i / per, r = i - f * per;
        const int y = static_cast<int>(r / w), x = static_cast<int>(r - static_cast<size_t>(y) * w);
        const uint8_t* img = in + f * per;
        uint8_t v = img[r];
        if (v != 255) {
            // a neighbour c spreads onto (x,y) only if c itself lies in the interior [1,w-2] x [1,h-2]
            for (int dy = -1; dy <= 1 && v != 255; ++dy)
                for (int dx = -1; dx <= 1; ++dx) {
                    const int cx = x + dx, cy = y + dy;
                    if (cx >= 1 && cx <= w - 2 && cy >= 1 && cy <= h - 2 && img[static_cast<size_t>(cy) * w + cx] == 255) { v = 255; break; }
                }
        }
        out[i] = v;
    }
}

// E[k] = (sum_i data[i][k]) / n, main_responseCalib.cpp:249-259 (integer-valued sums: exact in any order).
__global__ void __launch_bounds__(256) rc_einit_kernel(const uint8_t* __restrict__ data, int n, size_t npix, double* __restrict__ E) {
    const size_t k = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (k >= npix) return;
    double s = 0.0, c = 0.0;
    for (int i = 0; i < n; ++i) { s = __dadd_rn(s, static_cast<double>(data[static_cast<size_t>(i) * npix + k])); c = __dadd_rn(c, 1.0); }
    E[k] = __ddiv_rn(s, c);
}

// largest finite |E[k]| and |t[i]| of a pass (bit patterns, see GstepScale); scale must be zeroed before the launch
__global__ void __launch_bounds__(256) rc_gstep_scale_kernel(const double* __restrict__ E, size_t npix, const double* __restrict__ t, int n, GstepScale* __restrict__ scale) {
    unsigned long long me = 0ull, mt = 0ull;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t k = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; k < npix; k += stride) {
        const unsigned long long v = static_cast<unsigned long long>(__double_as_longlong(E[k])) & 0x7fffffffffffffffull;
        if (v < 0x7ff0000000000000ull && v > me) me = v;
    }
    if (blockIdx.x == 0)
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const unsigned long long v = static_cast<unsigned long long>(__double_as_longlong(t[i])) & 0x7fffffffffffffffull;
            if (v >= 0x7ff0000000000000ull) scale->bad_t = 1ull;
            else if (v > mt) mt = v;
        }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long oe = __shfl_xor_sync(0xffffffffu, me, o), ot = __shfl_xor_sync(0xffffffffu, mt, o);
        me = oe > me ? oe : me;
        mt = ot > mt ? ot : mt;
    }
    if ((threadIdx.x & 31) == 0) {
        if (me) atomicMax(&scale->max_e_bits, me);
        if (mt) atomicMax(&scale->max_t_bits, mt);
    }
}

// G-step accumulation for image sizes the streaming kernels do not take, main_responseCalib.cpp:290-299: GSum[b] += E[k]*t[i],
// GNum[b]++ for b != 255.  Per-CTA shared-memory sums in the same fixed-point form (here one 64-bit word + a carry word per bin,
// updated with the compare-and-swap atomics: this kernel is the fallback, not the fast path), one 128-bit global add per bin per CTA.
__global__ void __launch_bounds__(256) rc_gstep_accum_kernel(const uint8_t* __restrict__ data, int n, size_t npix, const double* __restrict__ t,
                                                             const double* __restrict__ E, GstepFx fx, unsigned long long* __restrict__ gnum) {
    __shared__ unsigned long long s_lo[256], s_num[256];
    __shared__ int s_hi[256];
    s_lo[threadIdx.x] = 0ull; s_hi[threadIdx.x] = 0; s_num[threadIdx.x] = 0ull;
    __syncthreads();
    const int se = gstep_scale_exponent(*fx.scale);
    const bool mul = se >= -1022 && se <= 1023;      // 2^s is a double: p * 2^s and scalbn(p, s) are the same correctly rounded value
    const double scale = mul ? scalbn(1.0, se) : 1.0;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t k = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; k < npix; k += stride) {
        const double e = E[k];
        for (int i = 0; i < n; ++i) {
            const unsigned b = data[static_cast<size_t>(i) * npix + k];
            if (b == 255u) continue;
            atomicAdd(&s_num[b], 1ull);
            const double p = __dmul_rn(e, __ldg(t + i));      // :295
            const double x = mul ? __dmul_rn(p, scale) : scalbn(p, se);
            if (!fx_in_range(x)) { atomicAdd(fx.special + b, p); continue; }      // only a non-finite product
            const long long v = __double_as_longlong(__dadd_rn(x, kFxMagic)) - __double_as_longlong(kFxMagic);
            const unsigned long long uv = static_cast<unsigned long long>(v);
            const unsigned long long old = atomicAdd(&s_lo[b], uv);
            const int delta = static_cast<int>(old + uv < old) - static_cast<int>(v < 0);      // carry out of the low word, sign extension of v
            if (delta) atomicAdd(&s_hi[b], delta);
        }
    }
    __syncthreads();
    if (s_lo[threadIdx.x] | static_cast<unsigned long long>(static_cast<long long>(s_hi[threadIdx.x])))
        fx_flush(fx.lo + threadIdx.x, fx.hi + threadIdx.x, s_lo[threadIdx.x], s_hi[threadIdx.x]);
    atomicAdd(&gnum[threadIdx.x], s_num[threadIdx.x]);
}

// gsum[b] = (hi * 2^64 + lo) * 2^-s + special[b]: the 128-bit sums back in fp64 (two roundings at most, the same on every run)
__device__ __forceinline__ double fx_to_double(unsigned long long lo, unsigned long long hi, const GstepScale& scale, double special) {
    const int s = gstep_scale_exponent(scale);
    const double h = __dmul_rn(static_cast<double>(static_cast<long long>(hi)), 18446744073709551616.0);
    return __dadd_rn(scalbn(__dadd_rn(h, static_cast<double>(lo)), -s), special);
}
__global__ void __launch_bounds__(256) rc_gstep_convert_kernel(GstepFx fx, double* __restrict__ gsum) {
    const int b = threadIdx.x;
    gsum[b] = fx_to_double(fx.lo[b], fx.hi[b], *fx.scale, fx.special[b]);
}
// Pixel-sharded runs add the ranks' sums as integers, so that G does not depend on the number of ranks: each 128-bit sum travels as
// three signed limbs of 43 bits (limbs[b], limbs[256 + b], limbs[512 + b]), which an all-reduce(SUM) over any realistic number of
// ranks cannot overflow, and is put together again afterwards.
constexpr int kFxLimbBits = 43;
__global__ void __launch_bounds__(256) rc_gstep_split_kernel(const unsigned long long* __restrict__ lo, const unsigned long long* __restrict__ hi,
                                                             long long* __restrict__ limbs) {
    const int b = threadIdx.x;
    const __int128 v = (static_cast<__int128>(static_cast<long long>(hi[b])) << 64) | static_cast<__int128>(lo[b]);
    const long long mask = (1ll << kFxLimbBits) - 1;
    limbs[b] = static_cast<long long>(v) & mask;
    limbs[256 + b] = static_cast<long long>(v >> kFxLimbBits) & mask;
    limbs[512 + b] = static_cast<long long>(v >> (2 * kFxLimbBits));      // arithmetic shift: carries the sign
}
__global__ void __launch_bounds__(256) rc_gstep_join_kernel(const long long* __restrict__ limbs, const double* __restrict__ special,
                                                            const GstepScale* __restrict__ scale, double* __restrict__ gsum) {
    const int b = threadIdx.x;
    const __int128 v = static_cast<__int128>(limbs[b]) + (static_cast<__int128>(limbs[256 + b]) << kFxLimbBits) + (static_cast<__int128>(limbs[512 + b]) << (2 * kFxLimbBits));
    gsum[b] = fx_to_double(static_cast<unsigned long long>(v), static_cast<unsigned long long>(static_cast<long long>(v >> 64)), *scale, special[b]);
}

// G[i] = GSum[i]/GNum[i]; non-finite entries (empty bins) with i > 1 are extrapolated linearly from the two entries below, :300-304.
// The divisions run in parallel (one thread per bin, launch with 256 threads); the extrapolation is sequential in i like the
// reference's loop (an extrapolated entry feeds the next one) and is done by one thread in shared memory.
__global__ void __launch_bounds__(256) rc_gstep_finish_kernel(const double* __restrict__ gsum, const unsigned long long* __restrict__ gnum, double* __restrict__ G) {
    __shared__ double g[256];
    __shared__ int any_gap;
    const int i = threadIdx.x;
    if (i == 0) any_gap = 0;
    __syncthreads();
    const double v = __ddiv_rn(gsum[i], static_cast<double>(gnum[i]));
    g[i] = v;
    if (!isfinite(v) && i > 1) any_gap = 1;
    __syncthreads();
    if (i == 0 && any_gap)
        for (int k = 2; k < 256; ++k)
            if (!isfinite(g[k])) g[k] = __dadd_rn(g[k - 1], __dsub_rn(g[k - 1], g[k - 2]));
    __syncthreads();
    G[i] = g[i];
}

// Rescale so that G[255] = 255, :350-355.  `factor` is 255.0 / G[255] evaluated BEFORE G is touched.
__global__ void rc_factor_kernel(const double* __restrict__ G, double* __restrict__ factor) { if (threadIdx.x == 0 && blockIdx.x == 0) *factor = __ddiv_rn(255.0, G[255]); }
__global__ void __launch_bounds__(256) rc_scale_kernel(double* __restrict__ v, size_t n, const double* __restrict__ factor) {
    const double f = *factor;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) v[i] = __dmul_rn(v[i], f);
}

// rmse(), :50-69: e = sum (G[b] - t*E)^2 * 1e-10 over finite residuals of unsaturated samples, num = their count.
__global__ void __launch_bounds__(256) rc_rmse_kernel(const uint8_t* __restrict__ data, int n, size_t npix, const double* __restrict__ t,
                                                      const double* __restrict__ G, const double* __restrict__ E, double* __restrict__ acc /*[2]*/) {
    __shared__ double sG[256];
    __shared__ double s_e[256], s_n[256];
    sG[threadIdx.x] = G[threadIdx.x];
    __syncthreads();
    double e = 0.0, cnt = 0.0;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t k = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; k < npix; k += stride) {
        const double ek = E[k];
        for (int i = 0; i < n; ++i) {
            const unsigned b = data[static_cast<size_t>(i) * npix + k];
            if (b == 255u) continue;
            const double r = __dsub_rn(sG[b], __dmul_rn(__ldg(t + i), ek));
            if (!isfinite(r)) continue;
            e = __dadd_rn(e, __dmul_rn(__dmul_rn(r, r), 1e-10));
            cnt = __dadd_rn(cnt, 1.0);
        }
    }
    s_e[threadIdx.x] = e; s_n[threadIdx.x] = cnt;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
        if (threadIdx.x < s) { s_e[threadIdx.x] += s_e[threadIdx.x + s]; s_n[threadIdx.x] += s_n[threadIdx.x + s]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { acc[2 * blockIdx.x] = s_e[0]; acc[2 * blockIdx.x + 1] = s_n[0]; }      // per-CTA partials, folded in order afterwards
}

// out[0..1] = the per-CTA {error, count} pairs summed in CTA order (fixed order => run-to-run identical bits)
__global__ void __launch_bounds__(256) rc_fold_pairs_kernel(const double* __restrict__ partials, int n_pairs, double* __restrict__ out) {
    __shared__ double s[2 * kRmsePartialPairs];      // fetched by the whole block (one pass of coalesced loads), summed by one thread in order
    for (int i = threadIdx.x; i < 2 * n_pairs; i += blockDim.x) s[i] = partials[i];
    __syncthreads();
    if (threadIdx.x != 0) return;
    double a = 0.0, b = 0.0;
    for (int i = 0; i < n_pairs; ++i) { a = __dadd_rn(a, s[2 * i]); b = __dadd_rn(b, s[2 * i + 1]); }
    out[0] = a; out[1] = b;
}

static unsigned rc_blocks(size_t work) {
    size_t b = (work + 255) / 256;
    // a fixed cap (8 CTAs per H100 SM), not one read from the device: the rmse fallback folds per-CTA partials in CTA order, so
    // the grid fixes its bits, and they should not depend on which GPU runs it
    if (b > 132u * 8u) b = 132u * 8u;
    return static_cast<unsigned>(b < 1 ? 1 : b);
}
cudaError_t launch_rc_leak_padding(const uint8_t* in, uint8_t* out, int n, int w, int h, cudaStream_t s) {
    rc_leak_padding_kernel<<<rc_blocks(static_cast<size_t>(n) * w * h), 256, 0, s>>>(in, out, n, w, h);
    return cudaGetLastError();
}
cudaError_t launch_rc_einit(const uint8_t* data, int n, int npix, double* E, cudaStream_t s) {
    rc_einit_kernel<<<(npix + 255) / 256, 256, 0, s>>>(data, n, static_cast<size_t>(npix), E);
    return cudaGetLastError();
}
// G-step in two halves so that a pixel-sharded run (SURVEY.md §8e row 2) can all-reduce the 2 x 256 accumulators in between:
//   accumulate  gsum[b] = sum E[k]*t[i], gnum[b] = count over THIS pixel range (main_responseCalib.cpp:290-299); with reuse_counts the
//               caller's gnum (which depends on the images only) is kept and only the sums are rebuilt
//   finish      G = gsum/gnum + sequential gap extrapolation (:300-304)
// fx_scratch (kGstepFxScratchBytes): scale | lo[256] | hi[256] | special[256]
static GstepFx fx_of(void* fx_scratch) {
    GstepFx fx;
    fx.scale = static_cast<GstepScale*>(fx_scratch);
    fx.lo = reinterpret_cast<unsigned long long*>(static_cast<char*>(fx_scratch) + 64);
    fx.hi = fx.lo + 256;
    fx.special = reinterpret_cast<double*>(fx.hi + 256);
    return fx;
}
// largest finite |E|, |t| of this pixel range -> scale4 (GstepScale as four u64 words)
cudaError_t launch_rc_gstep_scale(const double* E, int npix, const double* t, int n, void* scale4, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(scale4, 0, sizeof(GstepScale), s);
    if (e != cudaSuccess || npix <= 0 || n <= 0) return e;
    rc_gstep_scale_kernel<<<rc_blocks(static_cast<size_t>(npix)), 256, 0, s>>>(E, static_cast<size_t>(npix), t, n, static_cast<GstepScale*>(scale4));
    return cudaGetLastError();
}
// the histogram pass itself: fx.scale must hold the scale (of this range, or agreed between ranks); lo / hi / special are rebuilt
static cudaError_t gstep_histogram(const uint8_t* data, int n, int npix, const double* t, const double* E, const GstepFx& fx, unsigned long long* gnum,
                                   bool reuse_counts, cudaStream_t s) {
    cudaError_t e = cudaMemsetAsync(fx.lo, 0, 2 * 256 * sizeof(unsigned long long), s);
    if (e == cudaSuccess) e = cudaMemsetAsync(fx.special, 0, 256 * sizeof(double), s);
    if (e == cudaSuccess && !reuse_counts) e = cudaMemsetAsync(gnum, 0, 256 * sizeof(unsigned long long), s);
    if (e != cudaSuccess || npix <= 0 || n <= 0) return e;
    const bool stream = stream_ok(data, npix);
    if (reuse_counts && !stream) return cudaErrorNotSupported;      // the generic kernel always counts (callers check rc_counts_reusable first)
    if (stream) {
        const StreamArgs a{data, n, static_cast<uint32_t>(npix), t, kEbWarps};
        return reuse_counts ? launch_stream<GstepOp<false>>(a, GstepOp<false>::Params{E, fx, gnum}, s)
                            : launch_stream<GstepOp<true>>(a, GstepOp<true>::Params{E, fx, gnum}, s);
    }
    rc_gstep_accum_kernel<<<rc_blocks(static_cast<size_t>(npix)), 256, 0, s>>>(data, n, static_cast<size_t>(npix), t, E, fx, gnum);
    return cudaGetLastError();
}
cudaError_t launch_rc_gstep_accum(const uint8_t* data, int n, int npix, const double* t, const double* E, double* gsum, unsigned long long* gnum,
                                  bool reuse_counts, void* fx_scratch, cudaStream_t s) {
    const GstepFx fx = fx_of(fx_scratch);
    cudaError_t e = launch_rc_gstep_scale(E, npix, t, n, fx.scale, s);
    if (e == cudaSuccess) e = gstep_histogram(data, n, npix, t, E, fx, gnum, reuse_counts, s);
    if (e != cudaSuccess) return e;
    rc_gstep_convert_kernel<<<1, 256, 0, s>>>(fx, gsum);
    return cudaGetLastError();
}
// the same pass for one rank of a pixel-sharded run: the scale comes from the caller (all-reduced MAX of launch_rc_gstep_scale's result),
// the sums leave as integer limbs (limbs768, all-reduce SUM) + special256 (fp64, all-reduce SUM) — see rc_gstep_split_kernel
cudaError_t launch_rc_gstep_accum_exact(const uint8_t* data, int n, int npix, const double* t, const double* E, const void* scale4, long long* limbs768,
                                        double* special256, unsigned long long* gnum, bool reuse_counts, void* fx_scratch, cudaStream_t s) {
    GstepFx fx = fx_of(fx_scratch);
    fx.scale = const_cast<GstepScale*>(static_cast<const GstepScale*>(scale4));
    fx.special = special256;
    cudaError_t e = gstep_histogram(data, n, npix, t, E, fx, gnum, reuse_counts, s);
    if (e != cudaSuccess) return e;
    rc_gstep_split_kernel<<<1, 256, 0, s>>>(fx.lo, fx.hi, limbs768);
    return cudaGetLastError();
}
cudaError_t launch_rc_gstep_finish_exact(const void* scale4, const long long* limbs768, const double* special256, const unsigned long long* gnum,
                                         double* gsum_scratch, double* G, cudaStream_t s) {
    rc_gstep_join_kernel<<<1, 256, 0, s>>>(limbs768, special256, static_cast<const GstepScale*>(scale4), gsum_scratch);
    rc_gstep_finish_kernel<<<1, 256, 0, s>>>(gsum_scratch, gnum, G);
    return cudaGetLastError();
}
cudaError_t launch_rc_gstep_finish(const double* gsum, const unsigned long long* gnum, double* G, cudaStream_t s) {
    rc_gstep_finish_kernel<<<1, 256, 0, s>>>(gsum, gnum, G);
    return cudaGetLastError();
}
bool rc_counts_reusable(const uint8_t* data, int npix) { return stream_ok(data, npix); }

cudaError_t launch_rc_gstep(const uint8_t* data, int n, int npix, const double* t, const double* E, double* gsum, unsigned long long* gnum, double* G,
                            bool reuse_counts, void* fx_scratch, cudaStream_t s) {
    cudaError_t e = launch_rc_gstep_accum(data, n, npix, t, E, gsum, gnum, reuse_counts && rc_counts_reusable(data, npix), fx_scratch, s);
    if (e != cudaSuccess) return e;
    return launch_rc_gstep_finish(gsum, gnum, G, s);
}
cudaError_t launch_rc_rescale(int npix, double* E, double* G, double* factor, cudaStream_t s) {
    rc_factor_kernel<<<1, 32, 0, s>>>(G, factor);
    rc_scale_kernel<<<rc_blocks(static_cast<size_t>(npix)), 256, 0, s>>>(E, static_cast<size_t>(npix), factor);
    rc_scale_kernel<<<1, 256, 0, s>>>(G, 256, factor);
    return cudaGetLastError();
}
// partials: scratch for one {error, count} pair per CTA (kRmsePartialPairs pairs)
cudaError_t launch_rc_rmse(const uint8_t* data, int n, int npix, const double* t, const double* G, const double* E, double* acc2, double* partials,
                           cudaStream_t s) {
    int grid = 0;
    cudaError_t e;
    if (stream_ok(data, npix)) {
        e = launch_stream<RmseOp>(StreamArgs{data, n, static_cast<uint32_t>(npix), t, kEbWarps}, RmseOp::Params{G, E, partials}, s, &grid);
        if (e != cudaSuccess) return e;
    } else {
        grid = static_cast<int>(rc_blocks(static_cast<size_t>(npix)));
        rc_rmse_kernel<<<grid, 256, 0, s>>>(data, n, static_cast<size_t>(npix), t, G, E, partials);
        if ((e = cudaGetLastError()) != cudaSuccess) return e;
    }
    if (grid > kRmsePartialPairs) return cudaErrorInvalidValue;
    rc_fold_pairs_kernel<<<1, 256, 0, s>>>(partials, grid, acc2);
    return cudaGetLastError();
}

}  // namespace mdc
