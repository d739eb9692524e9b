// vignetteCalib's alternating optimiser on the GPU (SURVEY.md §8f N4): main_vignetteCalib.cpp:395-585.
//
// State as the reference holds it when its loop starts (:395): n float images [wI*hI] (NaN = invalidated pixel), n
// plane-to-image maps p2x/p2y [gw*gh] (NaN = plane point not visible; finite entries keep all four bilinear taps inside the
// image, :352-356), planeColor [gw*gh], vignetteFactor [wI*hI].  Every array is device-resident, image-major, contiguous.
//
//   plane step (:400-446)     one thread per plane point, sequential over the images  ->  FF/FC accumulate in the reference's
//                             order, planeColor = FC/FF is BIT-IDENTICAL; E is a sum over 10^9 doubles (order-dependent).
//   vignette step (:458-533)  one thread per (image, plane point): bilinear scatter-add of 8 float terms into TT/CT.  The
//                             reference adds them in (image, point) order in fp32; no parallel order reproduces that chain,
//                             and fp32 atomics would make the result depend on thread timing.  The terms (each rounded
//                             exactly as the reference rounds it) are therefore added as 64-bit fixed-point integers:
//                             the sums are exact, so they are the same bits on every run, and they differ from the
//                             reference's chain only by the rounding error of that chain (compared to 2e-5 relative).
//                             Then CT/TT, the maximum, the division.
//   smoothing (:542-566)      NaN-aware 3x3 mean, ping-pong buffers, bit-identical.
//   front end (:286-301)      exposure normalisation, then the order-dependent gradient invalidation as a flag pass plus a
//                             skewed wavefront per image (see vc_grad_resolve_kernel), bit-identical.
//
// All float arithmetic is spelled out with round-to-nearest intrinsics in the reference's evaluation order (no FMA).
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "mdc_b200.h"
#include "mdc_internal.h"

#define VC_CHECK(expr)                                                                          \
    do {                                                                                        \
        cudaError_t e__ = (expr);                                                               \
        if (e__ != cudaSuccess) {                                                               \
            mdc_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return MDC_ERR_CUDA;                                                                \
        }                                                                                       \
    } while (0)

namespace {

struct Taps { float w00, w10, w01, w11; int base; };      // weights of bp[0], bp[1], bp[width], bp[1+width]

// the index/weight part of getInterpolatedElement (main_vignetteCalib.cpp:52-62)
__device__ __forceinline__ Taps vc_taps(float x, float y, int width) {
    const int ix = static_cast<int>(x), iy = static_cast<int>(y);
    const float dx = __fsub_rn(x, static_cast<float>(ix)), dy = __fsub_rn(y, static_cast<float>(iy));
    const float dxdy = __fmul_rn(dx, dy);
    Taps t;
    t.w11 = dxdy;
    t.w01 = __fsub_rn(dy, dxdy);
    t.w10 = __fsub_rn(dx, dxdy);
    t.w00 = __fadd_rn(__fsub_rn(__fsub_rn(1.0f, dx), dy), dxdy);
    t.base = ix + iy * width;
    return t;
}
// ... and its blend (:65-68): dxdy*bp[1+w] + (dy-dxdy)*bp[w] + (dx-dxdy)*bp[1] + (1-dx-dy+dxdy)*bp[0], left to right
__device__ __forceinline__ float vc_blend(const float* __restrict__ mat, const Taps& t, int width) {
    const float* bp = mat + t.base;
    float r = __fmul_rn(t.w11, __ldg(bp + 1 + width));
    r = __fadd_rn(r, __fmul_rn(t.w01, __ldg(bp + width)));
    r = __fadd_rn(r, __fmul_rn(t.w10, __ldg(bp + 1)));
    return __fadd_rn(r, __fmul_rn(t.w00, __ldg(bp)));
}

// CTA-wide reduction of (E, R) partials -> one pair per CTA in partials[]; vc_fold_stats_kernel adds the pairs in CTA order, so
// the statistics are the same bits on every run.  The cap is fixed (32 CTAs per H100 SM), not read from the device, because the
// grid fixes those bits and they should not depend on which GPU runs it.
constexpr int kVcMaxBlocks = 132 * 32;
__device__ __forceinline__ void vc_flush_stats(double e, double r, double* __restrict__ partials) {
    __shared__ double se[32], sr[32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        e += __shfl_xor_sync(0xffffffffu, e, o);
        r += __shfl_xor_sync(0xffffffffu, r, o);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = (blockDim.x + 31) >> 5;
    if (lane == 0) { se[warp] = e; sr[warp] = r; }
    __syncthreads();
    if (warp == 0) {
        e = lane < warps ? se[lane] : 0.0;
        r = lane < warps ? sr[lane] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            e += __shfl_xor_sync(0xffffffffu, e, o);
            r += __shfl_xor_sync(0xffffffffu, r, o);
        }
        if (lane == 0) { partials[2 * blockIdx.x] = e; partials[2 * blockIdx.x + 1] = r; }
    }
}
__global__ void __launch_bounds__(256) vc_fold_stats_kernel(const double* __restrict__ partials, int n_blocks, double* __restrict__ stats) {
    __shared__ double se[256], sr[256];
    const int chunk = (n_blocks + 255) / 256;      // thread i: pairs [i * chunk, (i + 1) * chunk) in order; thread 0: the 256 chunk sums in order
    double e = 0.0, r = 0.0;
    for (int i = threadIdx.x * chunk; i < (threadIdx.x + 1) * chunk && i < n_blocks; ++i) { e += partials[2 * i]; r += partials[2 * i + 1]; }
    se[threadIdx.x] = e; sr[threadIdx.x] = r;
    __syncthreads();
    if (threadIdx.x != 0) return;
    e = r = 0.0;
    for (int i = 0; i < 256; ++i) { e += se[i]; r += sr[i]; }
    stats[0] = e; stats[1] = r;
}

// The reference's outlier test `abs(residual) > oth2` (:423, :481) on a double residual: with only `int abs(int)` visible to
// unqualified lookup (libstdc++ before GCC 6 - the reference's era - and the oracle build) the residual is truncated to int first;
// with <cmath>'s overloads in the global namespace it is fabs.  integer_abs != 0 reproduces the former: residuals are squares
// (>= 0) or NaN, and an out-of-range / NaN conversion yields INT_MIN on x86, which is never an outlier.
__device__ __forceinline__ bool vc_outlier(double residual, double oth2, int integer_abs) {
    if (!integer_abs) return fabs(residual) > oth2;
    return residual < 2147483648.0 && static_cast<double>(__double2int_rz(residual)) > oth2;
}

constexpr int kVcBatch = 4;      // images whose maps and taps are fetched together (memory-level parallelism)

// ---- plane step: for each plane point the optimum is sum(color*fac) / sum(fac*fac) over the images that see it
__global__ void __launch_bounds__(256) vc_plane_kernel(const float* __restrict__ images, const float* __restrict__ p2x,
                                                       const float* __restrict__ p2y, int n, int gwgh, int wI, size_t npx,
                                                       const float* __restrict__ vignette, float* __restrict__ plane_color,
                                                       double oth2, int integer_abs, double* __restrict__ stats) {
    double e_sum = 0.0, r_cnt = 0.0;
    const int stride = gridDim.x * blockDim.x;
    for (int pi = blockIdx.x * blockDim.x + threadIdx.x; pi < gwgh; pi += stride) {
        const float pc = plane_color[pi];
        float ff = 0.0f, fc = 0.0f;
        // software pipeline: the maps of the NEXT batch of images are requested before the taps of the current batch are gathered,
        // so a batch costs one memory round trip instead of two dependent ones
        float mx[kVcBatch], my[kVcBatch];
        auto fetch_maps = [&](int img0, float (&x)[kVcBatch], float (&y)[kVcBatch]) {
#pragma unroll
            for (int j = 0; j < kVcBatch; ++j) {
                const int img = img0 + j;
                const bool in = img < n;
                x[j] = in ? __ldg(p2x + static_cast<size_t>(img) * gwgh + pi) : __int_as_float(0x7fc00000);
                y[j] = in ? __ldg(p2y + static_cast<size_t>(img) * gwgh + pi) : 0.0f;
            }
        };
        fetch_maps(0, mx, my);
        for (int img0 = 0; img0 < n; img0 += kVcBatch) {
            float nx[kVcBatch], ny[kVcBatch];
            fetch_maps(img0 + kVcBatch, nx, ny);
            float color[kVcBatch], fac[kVcBatch];
#pragma unroll
            for (int j = 0; j < kVcBatch; ++j) {
                color[j] = fac[j] = 0.0f;
                if (!isnan(mx[j])) {                                                       // :414
                    const Taps t = vc_taps(mx[j], my[j], wI);
                    color[j] = vc_blend(images + static_cast<size_t>(img0 + j) * npx, t, wI);
                    fac[j] = vc_blend(vignette, t, wI);
                }
            }
#pragma unroll
            for (int j = 0; j < kVcBatch; ++j) {
                if (isnan(mx[j]) || isnan(fac[j]) || isnan(color[j])) continue;            // :414, :420-421
                const float d = __fsub_rn(color[j], __fmul_rn(pc, fac[j]));
                const double residual = static_cast<double>(__fmul_rn(d, d));
                if (vc_outlier(residual, oth2, integer_abs)) { e_sum += oth2; r_cnt += 1.0; continue; }      // :424-429
                ff = __fadd_rn(ff, __fmul_rn(fac[j], fac[j]));
                fc = __fadd_rn(fc, __fmul_rn(color[j], fac[j]));
                if (isnan(pc)) continue;
                e_sum += residual;
                r_cnt += 1.0;
            }
#pragma unroll
            for (int j = 0; j < kVcBatch; ++j) { mx[j] = nx[j]; my[j] = ny[j]; }
        }
        plane_color[pi] = (ff < 1.0f) ? __int_as_float(0x7fc00000) : __fdiv_rn(fc, ff);    // :441-445
    }
    vc_flush_stats(e_sum, r_cnt, stats);
}

// ---- vignette step: bilinear scatter of the normal equations  TT += w*cP*cP,  CT += w*cI*cP, in 64-bit fixed point.
// Every term is computed in fp32 exactly as the reference computes it, then multiplied by 2^s (exact) and rounded to an integer
// (one DADD with 1.5 * 2^52); the integers are added with 64-bit global REDs.  s comes from three numbers measured on the
// device (VcFx): the largest finite |planeColor| and |image| bound every term, and the largest number of plane points whose
// bilinear footprint starts at one pixel bounds how many terms a pixel can receive (4 x that), so that neither a term (< 2^50)
// nor a sum (< 2^62) can overflow.  A term is off by at most 2^-(s+1), so a sum of K terms by at most K * 2^-(s+1), where
// 2^-s <= max(2^-49, (4 * max_count + 4) * 2^-61) * 1.001 * P * max(P, I).  That is not always below one fp32 ulp of a sum that
// passes the reference's TT >= 1 test: at 64 poses of 1000x1000 points in 1280x1024 images with values from 1 to 1e4 (max_count
// 1679, s = 22) the largest error at TT >= 1 is 1.6 ulps (1.2e-7 relative), at TT >= 1e6 3e-13 relative.  The sums do not depend
// on the order of the atomics.  tests/vc_fixed_point_spec.py states this arithmetic in numpy.
struct VcFx { unsigned max_plane_bits, max_image_bits, max_count, pad; };
constexpr double kVcMagic = 6755399441055744.0;      // 1.5 * 2^52
__device__ __forceinline__ int vc_scale_exponent(const VcFx& fx) {
    const double P = static_cast<double>(__uint_as_float(fx.max_plane_bits)), I = static_cast<double>(__uint_as_float(fx.max_image_bits));
    const double term = P * (P > I ? P : I) * 1.001;                  // |w*cP*cP|, |w*cI*cP| with w in [0,1], incl. the fp32 roundings
    if (!(term > 0.0)) return 0;
    const double total = term * (4.0 * static_cast<double>(fx.max_count) + 4.0);
    const int s_term = 50 - (ilogb(term) + 1), s_total = 62 - (ilogb(total) + 1);
    const int s = s_term < s_total ? s_term : s_total;
    return s < -1000 ? -1000 : (s > 1000 ? 1000 : s);
}
// largest finite |v[i]| as a float bit pattern (non-negative floats order like integers); *out must start at 0
__global__ void __launch_bounds__(256) vc_absmax_kernel(const float* __restrict__ v, size_t n, unsigned* __restrict__ out) {
    unsigned m = 0u;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const unsigned b = __float_as_uint(__ldg(v + i)) & 0x7fffffffu;
        if (b < 0x7f800000u && b > m) m = b;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const unsigned x = __shfl_xor_sync(0xffffffffu, m, o); m = x > m ? x : m; }
    if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}
// count[p] = number of (image, plane point) pairs whose footprint starts at pixel p; a pixel receives terms from the footprints
// starting at it, left of it, above it and above-left of it, i.e. at most 4 x max(count)
__global__ void __launch_bounds__(256) vc_count_kernel(const float* __restrict__ p2x, const float* __restrict__ p2y, size_t total, int wI,
                                                       unsigned* __restrict__ count) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const float x = __ldg(p2x + idx);
        if (isnan(x)) continue;
        atomicAdd(count + vc_taps(x, __ldg(p2y + idx), wI).base, 1u);
    }
}
__global__ void __launch_bounds__(256) vc_umax_kernel(const unsigned* __restrict__ v, size_t n, unsigned* __restrict__ out) {
    unsigned m = 0u;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) m = v[i] > m ? v[i] : m;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const unsigned x = __shfl_xor_sync(0xffffffffu, m, o); m = x > m ? x : m; }
    if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// A finite term goes to the fixed-point sum.  One that is not - from an infinite colour, or a product of finite colours beyond
// FLT_MAX, which the bounds do not cover - goes to the fp32 side sum, as the reference's fp32 chain would turn it into inf / NaN.
// The side sums thus only ever hold +-inf or NaN, whose sum does not depend on the order of the atomics either.
__device__ __forceinline__ void vc_add(long long* acc, float* special, float term, double scale) {
    if (!isfinite(term)) { atomicAdd(special, term); return; }
    const double y = __dadd_rn(__dmul_rn(static_cast<double>(term), scale), kVcMagic);
    atomicAdd(reinterpret_cast<unsigned long long*>(acc), static_cast<unsigned long long>(__double_as_longlong(y) - __double_as_longlong(kVcMagic)));
}
__global__ void __launch_bounds__(256) vc_vignette_kernel(const float* __restrict__ images, const float* __restrict__ p2x,
                                                          const float* __restrict__ p2y, size_t total, int gwgh, int wI, size_t npx,
                                                          const float* __restrict__ plane_color, const float* __restrict__ vignette,
                                                          long long* __restrict__ tt, long long* __restrict__ ct, float* __restrict__ tt_special,
                                                          float* __restrict__ ct_special, const VcFx* __restrict__ fx, double oth2, int integer_abs,
                                                          double* __restrict__ partials) {
    double e_sum = 0.0, r_cnt = 0.0;
    const double scale = scalbn(1.0, vc_scale_exponent(*fx));
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; idx < total; idx += stride) {
        const float x = __ldg(p2x + idx);
        if (isnan(x)) continue;                                                            // :469
        const float y = __ldg(p2y + idx);
        const size_t img = idx / static_cast<size_t>(gwgh);
        const int pi = static_cast<int>(idx - img * gwgh);
        const float cP = __ldg(plane_color + pi);
        if (isnan(cP)) continue;                                                           // :477
        const Taps t = vc_taps(x, y, wI);
        const float cI = vc_blend(images + img * npx, t, wI);
        if (isnan(cI)) continue;                                                           // :478
        const float fac = vc_blend(vignette, t, wI);
        const float d = __fsub_rn(cI, __fmul_rn(cP, fac));
        const double residual = static_cast<double>(__fmul_rn(d, d));
        if (vc_outlier(residual, oth2, integer_abs)) { e_sum += oth2; r_cnt += 1.0; continue; }              // :481-486
        const float a00 = __fmul_rn(__fmul_rn(t.w00, cP), cP), a10 = __fmul_rn(__fmul_rn(t.w10, cP), cP);
        const float a01 = __fmul_rn(__fmul_rn(t.w01, cP), cP), a11 = __fmul_rn(__fmul_rn(t.w11, cP), cP);
        const float b00 = __fmul_rn(__fmul_rn(t.w00, cI), cP), b10 = __fmul_rn(__fmul_rn(t.w10, cI), cP);
        const float b01 = __fmul_rn(__fmul_rn(t.w01, cI), cP), b11 = __fmul_rn(__fmul_rn(t.w11, cI), cP);
        long long* a = tt + t.base;
        long long* b = ct + t.base;
        float* as = tt_special + t.base;
        float* bs = ct_special + t.base;
        vc_add(a, as, a00, scale); vc_add(a + 1, as + 1, a10, scale); vc_add(a + wI, as + wI, a01, scale); vc_add(a + 1 + wI, as + 1 + wI, a11, scale);
        vc_add(b, bs, b00, scale); vc_add(b + 1, bs + 1, b10, scale); vc_add(b + wI, bs + wI, b01, scale); vc_add(b + 1 + wI, bs + 1 + wI, b11, scale);
        if (isnan(fac)) continue;
        e_sum += residual;
        r_cnt += 1.0;
    }
    vc_flush_stats(e_sum, r_cnt, partials);
}

// vignette = CT/TT where TT >= 1, NaN elsewhere; running maximum of the finite factors (:507-517)
__global__ void __launch_bounds__(256) vc_divide_kernel(const long long* __restrict__ tt, const long long* __restrict__ ct, const float* __restrict__ tt_special,
                                                        const float* __restrict__ ct_special, const VcFx* __restrict__ fx, size_t npx,
                                                        float* __restrict__ vignette, int* __restrict__ max_bits) {
    float m = 0.0f;
    const int s = vc_scale_exponent(*fx);
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < npx; i += stride) {
        const float t = __fadd_rn(static_cast<float>(scalbn(static_cast<double>(tt[i]), -s)), tt_special[i]);
        const float c = __fadd_rn(static_cast<float>(scalbn(static_cast<double>(ct[i]), -s)), ct_special[i]);
        float v = __int_as_float(0x7fc00000);
        if (!(t < 1.0f)) {
            v = __fdiv_rn(c, t);
            if (v > m) m = v;
        }
        vignette[i] = v;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    // m >= 0 and not NaN, so the integer order of the bit patterns is the float order
    if ((threadIdx.x & 31) == 0 && m > 0.0f) atomicMax(max_bits, __float_as_int(m));
}
// normalise to vignette max. factor 1 (:521-523)
__global__ void __launch_bounds__(256) vc_normalise_kernel(float* __restrict__ vignette, size_t npx, const int* __restrict__ max_bits) {
    const float m = __int_as_float(*max_bits);
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < npx; i += stride) vignette[i] = __fdiv_rn(vignette[i], m);
}

// one round of the NaN-aware 3x3 mean (:547-563), src -> dst
__global__ void __launch_bounds__(256) vc_smooth_kernel(const float* __restrict__ src, float* __restrict__ dst, int wI, int hI) {
    const size_t npx = static_cast<size_t>(wI) * hI;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < npx; i += stride) {
        const int y = static_cast<int>(i / wI), x = static_cast<int>(i - static_cast<size_t>(y) * wI);
        float sum = 0.0f, num = 0.0f;
        auto take = [&](bool inside, ptrdiff_t off) {
            if (!inside) return;
            const float v = src[static_cast<ptrdiff_t>(i) + off];
            if (!isnan(v)) { sum = __fadd_rn(sum, v); num = __fadd_rn(num, 1.0f); }
        };
        const bool r = x < wI - 1, l = x > 0, d = y < hI - 1, u = y > 0;
        take(r && d, 1 + wI);
        take(r, 1);
        take(r && u, 1 - wI);
        take(d, wI);
        take(true, 0);
        take(u, -wI);
        take(d && l, -1 + wI);
        take(l, -1);
        take(u && l, -1 - wI);
        dst[i] = (num > 0.0f) ? __fdiv_rn(sum, num) : src[i];
    }
}

// ---- front end: the images the loop works on (:286-301)
// image = (meanExposure * raw) / exposure, elementwise (in place allowed); exposures[img] has 0 already replaced by 1 (:286)
__global__ void __launch_bounds__(256) vc_normalise_images_kernel(const float* raw, float* out, size_t npx, size_t total,
                                                                  const float* __restrict__ exposures, float mean_exposure) {
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride)
        out[i] = __fdiv_rn(__fmul_rn(mean_exposure, raw[i]), __ldg(exposures + i / npx));
}

// The gradient invalidation (:293-301) visits the centres 2 <= x < wI-2, 2 <= y < hI-2 in raster order and compares each with its
// 24 neighbours (deltax-major); a hit sets centre and neighbour to NaN, in place, so the result depends on the order.  Values only
// ever become NaN and a comparison with NaN is false, so a comparison can only fire if it fires on the normalised values as they
// are before the pass.  Pass 1 (vc_grad_flags_kernel) therefore marks, data-parallel, every centre that has at least one candidate
// hit: one bit per centre, 32 consecutive centres of a row per word.  Pass 2 (vc_grad_resolve_kernel) replays the reference's loop
// literally, on the current values, at the marked centres only, in an order that is equivalent to raster order: the centre at
// (x, y) runs at step x + 5y.  Two centres of one step are at least 5 columns apart, so their 5x5 windows are disjoint; a centre
// whose window overlaps that of an earlier centre in raster order (|dx| <= 4, |dy| <= 4) runs at a strictly earlier step.  Each
// step is one __syncthreads apart, and the pixels live in global memory (one CTA per image: the writes of a step are visible to
// the whole CTA after the barrier).
__device__ __forceinline__ bool vc_grad_hit(float c, float nb, float g) { return fabsf(__fsub_rn(c, nb)) > g; }

// one thread per centre column x of a 32-wide word (x = word*32 + lane); the words of row y: flags[img][y][0 .. words)
__global__ void __launch_bounds__(256) vc_grad_flags_kernel(const float* __restrict__ images, int wI, int hI, int words, size_t total,
                                                            float g, unsigned* __restrict__ flags) {
    const size_t npx = static_cast<size_t>(wI) * hI;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;      // total and stride are multiples of 32: whole warps
    for (size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < total; i += stride) {
        const size_t row = i >> 5;                          // img * hI + y
        const int word = static_cast<int>(row % words);
        const size_t img_y = row / words;
        const int y = static_cast<int>(img_y % hI);
        const size_t img = img_y / hI;
        const int x = word * 32 + static_cast<int>(i & 31);
        bool hit = false;
        if (x >= 2 && x < wI - 2 && y >= 2 && y < hI - 2) {
            const float* p = images + img * npx + static_cast<size_t>(y) * wI + x;
            const float c = __ldg(p);
            for (int dy = -2; dy <= 2 && !hit; ++dy)
                for (int dx = -2; dx <= 2; ++dx)
                    if (vc_grad_hit(c, __ldg(p + dy * wI + dx), g)) { hit = true; break; }
        }
        const unsigned bits = __ballot_sync(0xffffffffu, hit);
        if ((i & 31) == 0) flags[row] = bits;
    }
}

// one CTA per image of the chunk; at step t the centres x + 5y = t run, one per row, rows spread over the CTA's threads
__global__ void __launch_bounds__(256) vc_grad_resolve_kernel(float* images, int wI, int hI, int words, float g, const unsigned* __restrict__ flags) {
    float* im = images + static_cast<size_t>(blockIdx.x) * wI * hI;
    const unsigned* fl = flags + static_cast<size_t>(blockIdx.x) * hI * words;
    const int t_last = (wI - 3) + 5 * (hI - 3);
    for (int t = 2 + 5 * 2; t <= t_last; ++t) {
        // rows y with 2 <= x = t - 5y <= wI-3 and 2 <= y <= hI-3
        const int lo = max(2, (t - (wI - 3) + 4) / 5), hi = min(hI - 3, (t - 2) / 5);
        for (int y = lo + static_cast<int>(threadIdx.x); y <= hi; y += blockDim.x) {
            const int x = t - 5 * y;
            if (!((__ldg(fl + static_cast<size_t>(y) * words + (x >> 5)) >> (x & 31)) & 1u)) continue;
            float* p = im + static_cast<size_t>(y) * wI + x;
            // the reference's loop (:296-300) on the current values; once the centre is NaN no comparison can fire
            bool dead = false;
            for (int dx = -2; dx <= 2 && !dead; ++dx)
                for (int dy = -2; dy <= 2; ++dy) {
                    float* q = p + dx + dy * wI;
                    if (vc_grad_hit(*p, *q, g)) {
                        *p = __int_as_float(0x7fc00000);
                        *q = __int_as_float(0x7fc00000);
                        dead = true;
                        break;
                    }
                }
        }
        __syncthreads();
    }
}

unsigned vc_blocks(size_t work) {
    size_t b = (work + 255) / 256;
    if (b > static_cast<size_t>(kVcMaxBlocks)) b = kVcMaxBlocks;
    return static_cast<unsigned>(b < 1 ? 1 : b);
}

struct Problem { const float *images, *p2x, *p2y; int n, gwgh, wI, hI; };

int check_problem(const char* who, mdc_ctx* c, const Problem& p, const void* a, const void* b) {
    // with no images, nothing reads the images or the maps (an empty tensor's pointer may be null)
    if (!c || (p.n > 0 && (!p.images || !p.p2x || !p.p2y)) || !a || !b || p.n < 0 || p.gwgh < 1 || p.wI < 2 || p.hI < 2) {
        mdc_set_error("%s: bad argument", who);
        return MDC_ERR_INVALID_ARG;
    }
    return MDC_OK;
}

// scratch: a 64-byte head {stats[2], max word, VcFx}, the per-CTA statistics pairs, then per pixel: TT and CT (64-bit fixed point),
// their fp32 side accumulators, and the footprint counts
struct Scratch {
    long long *tt = nullptr, *ct = nullptr;
    float *tt_special = nullptr, *ct_special = nullptr;
    unsigned* count = nullptr;
    double *stats = nullptr, *partials = nullptr;
    int* max_bits = nullptr;
    VcFx* fx = nullptr;
    void* base = nullptr;
    size_t npx = 0;
};
constexpr size_t kVcHeadBytes = 64 + 2 * kVcMaxBlocks * sizeof(double);
int alloc_scratch(Scratch* s, size_t npx) {
    VC_CHECK(cudaMalloc(&s->base, kVcHeadBytes + npx * (2 * sizeof(long long) + 2 * sizeof(float) + sizeof(unsigned))));
    char* b = static_cast<char*>(s->base);
    s->stats = reinterpret_cast<double*>(b);
    s->max_bits = reinterpret_cast<int*>(b + 16);
    s->fx = reinterpret_cast<VcFx*>(b + 32);
    s->partials = reinterpret_cast<double*>(b + 64);
    s->tt = reinterpret_cast<long long*>(b + kVcHeadBytes);
    s->ct = s->tt + npx;
    s->tt_special = reinterpret_cast<float*>(s->ct + npx);
    s->ct_special = s->tt_special + npx;
    s->count = reinterpret_cast<unsigned*>(s->ct_special + npx);
    s->npx = npx;
    return MDC_OK;
}

// what the fixed-point scale needs and does not change between iterations: the largest |image| and the footprint counts
int measure_static_bounds(mdc_ctx* c, const Problem& p, const Scratch& sc, cudaStream_t s) {
    const size_t npx = static_cast<size_t>(p.wI) * p.hI, total = static_cast<size_t>(p.n) * p.gwgh;
    VC_CHECK(cudaMemsetAsync(sc.fx, 0, sizeof(VcFx), s));
    VC_CHECK(cudaMemsetAsync(sc.count, 0, npx * sizeof(unsigned), s));
    if (total) {
        vc_absmax_kernel<<<vc_blocks(static_cast<size_t>(p.n) * npx), 256, 0, s>>>(p.images, static_cast<size_t>(p.n) * npx, &sc.fx->max_image_bits);
        vc_count_kernel<<<vc_blocks(total), 256, 0, s>>>(p.p2x, p.p2y, total, p.wI, sc.count);
        vc_umax_kernel<<<vc_blocks(npx), 256, 0, s>>>(sc.count, npx, &sc.fx->max_count);
        VC_CHECK(cudaGetLastError());
        mdc_ctx_add_launches(c, 3);
    }
    return MDC_OK;
}

int plane_step(mdc_ctx* c, const Problem& p, const float* d_vignette, float* d_plane_color, double oth2, int integer_abs, double* d_partials, double* d_stats,
               cudaStream_t s) {
    const unsigned blocks = vc_blocks(static_cast<size_t>(p.gwgh));
    vc_plane_kernel<<<blocks, 256, 0, s>>>(p.images, p.p2x, p.p2y, p.n, p.gwgh, p.wI, static_cast<size_t>(p.wI) * p.hI, d_vignette, d_plane_color, oth2,
                                           integer_abs, d_partials);
    vc_fold_stats_kernel<<<1, 256, 0, s>>>(d_partials, static_cast<int>(blocks), d_stats);
    VC_CHECK(cudaGetLastError());
    mdc_ctx_add_launches(c, 2);
    return MDC_OK;
}

// sc.fx->max_image_bits / max_count must be current (measure_static_bounds)
int vignette_step(mdc_ctx* c, const Problem& p, const float* d_plane_color, float* d_vignette, double oth2, int integer_abs, const Scratch& sc, cudaStream_t s) {
    const size_t npx = static_cast<size_t>(p.wI) * p.hI, total = static_cast<size_t>(p.n) * p.gwgh;
    VC_CHECK(cudaMemsetAsync(sc.stats, 0, 2 * sizeof(double) + sizeof(int), s));
    VC_CHECK(cudaMemsetAsync(&sc.fx->max_plane_bits, 0, sizeof(unsigned), s));
    VC_CHECK(cudaMemsetAsync(sc.tt, 0, npx * (2 * sizeof(long long) + 2 * sizeof(float)), s));
    int launches = 3;
    if (total) {
        const unsigned blocks = vc_blocks(total);
        vc_absmax_kernel<<<vc_blocks(static_cast<size_t>(p.gwgh)), 256, 0, s>>>(d_plane_color, static_cast<size_t>(p.gwgh), &sc.fx->max_plane_bits);
        vc_vignette_kernel<<<blocks, 256, 0, s>>>(p.images, p.p2x, p.p2y, total, p.gwgh, p.wI, npx, d_plane_color, d_vignette, sc.tt, sc.ct, sc.tt_special,
                                                  sc.ct_special, sc.fx, oth2, integer_abs, sc.partials);
        vc_fold_stats_kernel<<<1, 256, 0, s>>>(sc.partials, static_cast<int>(blocks), sc.stats);
        VC_CHECK(cudaGetLastError());
        launches += 3;
    }
    vc_divide_kernel<<<vc_blocks(npx), 256, 0, s>>>(sc.tt, sc.ct, sc.tt_special, sc.ct_special, sc.fx, npx, d_vignette, sc.max_bits);
    vc_normalise_kernel<<<vc_blocks(npx), 256, 0, s>>>(d_vignette, npx, sc.max_bits);
    VC_CHECK(cudaGetLastError());
    mdc_ctx_add_launches(c, launches - 1);
    return MDC_OK;
}

int smooth(mdc_ctx* c, const float* d_vignette, int wI, int hI, int iterations, float* d_out, float* d_tmp, cudaStream_t s) {
    const size_t npx = static_cast<size_t>(wI) * hI;
    VC_CHECK(cudaMemcpyAsync(d_out, d_vignette, npx * sizeof(float), cudaMemcpyDeviceToDevice, s));
    for (int it = 0; it < iterations; ++it) {
        VC_CHECK(cudaMemcpyAsync(d_tmp, d_out, npx * sizeof(float), cudaMemcpyDeviceToDevice, s));
        vc_smooth_kernel<<<vc_blocks(npx), 256, 0, s>>>(d_tmp, d_out, wI, hI);
        VC_CHECK(cudaGetLastError());
        mdc_ctx_add_launches(c, 1);
    }
    return MDC_OK;
}

}  // namespace

extern "C" int mdc_vc_plane_step(mdc_ctx* c, const float* d_images, const float* d_p2x, const float* d_p2y, int n, int gw, int gh, int wI, int hI,
                                 const float* d_vignette, float* d_plane_color, double outlier_th2, int integer_abs, double stats_host[2]) {
    const Problem p{d_images, d_p2x, d_p2y, n, gw * gh, wI, hI};
    int rc = check_problem("mdc_vc_plane_step", c, p, d_vignette, d_plane_color);
    if (rc != MDC_OK) return rc;
    VC_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    cudaStream_t s = static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
    double* d_stats = nullptr;      // stats[2], then the per-CTA pairs
    VC_CHECK(cudaMalloc(&d_stats, (2 + 2 * kVcMaxBlocks) * sizeof(double)));
    rc = plane_step(c, p, d_vignette, d_plane_color, outlier_th2, integer_abs, d_stats + 2, d_stats, s);
    double st[2] = {0, 0};
    if (rc == MDC_OK && cudaMemcpyAsync(st, d_stats, sizeof st, cudaMemcpyDeviceToHost, s) != cudaSuccess) rc = MDC_ERR_CUDA;
    if (cudaStreamSynchronize(s) != cudaSuccess && rc == MDC_OK) { mdc_set_error("mdc_vc_plane_step: %s", cudaGetErrorString(cudaGetLastError())); rc = MDC_ERR_CUDA; }
    cudaFree(d_stats);
    if (stats_host) { stats_host[0] = st[0]; stats_host[1] = st[1]; }
    return rc;
}

extern "C" int mdc_vc_vignette_step(mdc_ctx* c, const float* d_images, const float* d_p2x, const float* d_p2y, int n, int gw, int gh, int wI, int hI,
                                    const float* d_plane_color, float* d_vignette, double outlier_th2, int integer_abs, double stats_host[2]) {
    const Problem p{d_images, d_p2x, d_p2y, n, gw * gh, wI, hI};
    int rc = check_problem("mdc_vc_vignette_step", c, p, d_plane_color, d_vignette);
    if (rc != MDC_OK) return rc;
    VC_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    cudaStream_t s = static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
    Scratch sc;
    if ((rc = alloc_scratch(&sc, static_cast<size_t>(wI) * hI)) != MDC_OK) return rc;
    rc = measure_static_bounds(c, p, sc, s);
    if (rc == MDC_OK) rc = vignette_step(c, p, d_plane_color, d_vignette, outlier_th2, integer_abs, sc, s);
    double st[2] = {0, 0};
    if (rc == MDC_OK && cudaMemcpyAsync(st, sc.stats, sizeof st, cudaMemcpyDeviceToHost, s) != cudaSuccess) rc = MDC_ERR_CUDA;
    if (cudaStreamSynchronize(s) != cudaSuccess && rc == MDC_OK) { mdc_set_error("mdc_vc_vignette_step: %s", cudaGetErrorString(cudaGetLastError())); rc = MDC_ERR_CUDA; }
    cudaFree(sc.base);
    if (stats_host) { stats_host[0] = st[0]; stats_host[1] = st[1]; }
    return rc;
}

// flags scratch of one chunk of images: at most this many bytes, and at most kVcPrepChunkImages images (one resolve CTA each)
constexpr size_t kVcPrepScratchBytes = size_t(64) << 20;
constexpr int kVcPrepChunkImages = 512;

extern "C" int mdc_vc_prepare_images(mdc_ctx* c, const float* d_raw, int n, int wI, int hI, const float* exposures_host, float mean_exposure,
                                     int max_abs_grad, float* d_images, mdc_stream stream) {
    if (!c || n < 0 || wI < 0 || hI < 0 || (n && wI && hI && (!d_raw || !d_images || !exposures_host))) {
        mdc_set_error("mdc_vc_prepare_images: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    const size_t npx = static_cast<size_t>(wI) * hI;
    if (n == 0 || npx == 0) return MDC_OK;
    VC_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
    std::vector<float> t(exposures_host, exposures_host + n);
    for (float& e : t)
        if (e == 0) e = 1;                                   // :286
    const bool has_centres = wI >= 5 && hI >= 5;
    const int words = (wI + 31) / 32;
    const size_t flag_bytes = static_cast<size_t>(hI) * words * sizeof(unsigned);
    size_t chunk = std::min<size_t>(std::max<size_t>(kVcPrepScratchBytes / flag_bytes, 1), kVcPrepChunkImages);
    chunk = std::min<size_t>(chunk, static_cast<size_t>(n));
    char* scratch = nullptr;      // exposures [n], then the flags of one chunk (256-byte aligned)
    const size_t expo_bytes = (static_cast<size_t>(n) * sizeof(float) + 255) / 256 * 256;
    VC_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&scratch), expo_bytes + (has_centres ? chunk * flag_bytes : 0), s));
    const float* d_expo = reinterpret_cast<const float*>(scratch);
    unsigned* d_flags = reinterpret_cast<unsigned*>(scratch + expo_bytes);
    int launches = 1;
    cudaError_t e = cudaMemcpyAsync(scratch, t.data(), static_cast<size_t>(n) * sizeof(float), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
        const size_t total = npx * n;
        vc_normalise_images_kernel<<<vc_blocks(total), 256, 0, s>>>(d_raw, d_images, npx, total, d_expo, mean_exposure);
        e = cudaGetLastError();
    }
    if (has_centres) {
        const float g = static_cast<float>(max_abs_grad);    // fabsf(...) > maxAbsGrad compares in float (:299)
        // threads per resolve CTA: enough for the rows one step touches (about (wI-4)/5), whole warps, at most 256
        const int rows = std::min((wI - 4 + 4) / 5, hI - 4);
        const int threads = std::min(256, std::max(32, (rows + 31) / 32 * 32));
        for (size_t first = 0; first < static_cast<size_t>(n) && e == cudaSuccess; first += chunk) {
            const size_t m = std::min(chunk, static_cast<size_t>(n) - first);
            float* im = d_images + first * npx;
            const size_t lanes = m * hI * words * 32;
            vc_grad_flags_kernel<<<vc_blocks(lanes), 256, 0, s>>>(im, wI, hI, words, lanes, g, d_flags);
            vc_grad_resolve_kernel<<<static_cast<unsigned>(m), threads, 0, s>>>(im, wI, hI, words, g, d_flags);
            e = cudaGetLastError();
            launches += 2;
        }
    }
    const cudaError_t f = cudaFreeAsync(scratch, s);
    mdc_ctx_add_launches(c, launches);
    VC_CHECK(e);
    VC_CHECK(f);
    if (!stream) VC_CHECK(cudaStreamSynchronize(s));
    return MDC_OK;
}

extern "C" int mdc_vc_smooth(mdc_ctx* c, const float* d_vignette, int wI, int hI, int iterations, float* d_out) {
    if (!c || !d_vignette || !d_out || wI < 1 || hI < 1 || iterations < 0) { mdc_set_error("mdc_vc_smooth: bad argument"); return MDC_ERR_INVALID_ARG; }
    VC_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    cudaStream_t s = static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
    float* tmp = nullptr;
    VC_CHECK(cudaMalloc(&tmp, static_cast<size_t>(wI) * hI * sizeof(float)));
    int rc = smooth(c, d_vignette, wI, hI, iterations, d_out, tmp, s);
    if (cudaStreamSynchronize(s) != cudaSuccess && rc == MDC_OK) { mdc_set_error("mdc_vc_smooth: %s", cudaGetErrorString(cudaGetLastError())); rc = MDC_ERR_CUDA; }
    cudaFree(tmp);
    return rc;
}

// The reference's loop (:395-585): per iteration plane step, vignette step (+ normalisation), smoothed copy for output.
// log_host, if given, receives [max_iterations][4] = {E_plane, R_plane, E_vignette, R_vignette}.
extern "C" int mdc_vignette_calib(mdc_ctx* c, const float* d_images, const float* d_p2x, const float* d_p2y, int n, int gw, int gh, int wI, int hI,
                                  int max_iterations, int outlier_th, int integer_abs, float* d_plane_color, float* d_vignette, float* d_smoothed,
                                  double* log_host) {
    const Problem p{d_images, d_p2x, d_p2y, n, gw * gh, wI, hI};
    int rc = check_problem("mdc_vignette_calib", c, p, d_plane_color, d_vignette);
    if (rc != MDC_OK) return rc;
    if (max_iterations < 0) { mdc_set_error("mdc_vignette_calib: bad argument"); return MDC_ERR_INVALID_ARG; }
    VC_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    cudaStream_t s = static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
    const size_t npx = static_cast<size_t>(wI) * hI;
    Scratch sc;
    if ((rc = alloc_scratch(&sc, npx)) != MDC_OK) return rc;
    double* d_pstats = nullptr;
    if (cudaMalloc(&d_pstats, 2 * sizeof(double)) != cudaSuccess) { cudaFree(sc.base); mdc_set_error("mdc_vignette_calib: out of device memory"); return MDC_ERR_CUDA; }
    rc = measure_static_bounds(c, p, sc, s);      // images and maps do not change inside the loop
    for (int it = 0; it < max_iterations && rc == MDC_OK; ++it) {
        double oth2 = static_cast<double>(outlier_th) * outlier_th;           // :397-398 (int arithmetic in the reference)
        if (it < max_iterations / 2) oth2 = 10000.0 * 10000.0;
        double ps[2] = {0, 0}, vs[2] = {0, 0};
        rc = plane_step(c, p, d_vignette, d_plane_color, oth2, integer_abs, sc.partials, d_pstats, s);
        if (rc == MDC_OK && cudaMemcpyAsync(ps, d_pstats, sizeof ps, cudaMemcpyDeviceToHost, s) != cudaSuccess) rc = MDC_ERR_CUDA;
        if (rc == MDC_OK) rc = vignette_step(c, p, d_plane_color, d_vignette, oth2, integer_abs, sc, s);
        if (rc == MDC_OK && cudaMemcpyAsync(vs, sc.stats, sizeof vs, cudaMemcpyDeviceToHost, s) != cudaSuccess) rc = MDC_ERR_CUDA;
        if (rc == MDC_OK && cudaStreamSynchronize(s) != cudaSuccess) { mdc_set_error("mdc_vignette_calib: %s", cudaGetErrorString(cudaGetLastError())); rc = MDC_ERR_CUDA; }
        if (rc != MDC_OK) break;
        printf("%f residual terms => %f\n", ps[1], sqrtf(static_cast<float>(ps[0] / ps[1])));      // :448
        printf("%f residual terms => %f\n", vs[1], sqrtf(static_cast<float>(vs[0] / vs[1])));      // :519
        if (log_host) { log_host[4 * it] = ps[0]; log_host[4 * it + 1] = ps[1]; log_host[4 * it + 2] = vs[0]; log_host[4 * it + 3] = vs[1]; }
    }
    if (rc == MDC_OK && d_smoothed) {
        rc = smooth(c, d_vignette, wI, hI, 4, d_smoothed, sc.tt_special, s);
        if (cudaStreamSynchronize(s) != cudaSuccess && rc == MDC_OK) { mdc_set_error("mdc_vignette_calib: %s", cudaGetErrorString(cudaGetLastError())); rc = MDC_ERR_CUDA; }
    }
    cudaFree(d_pstats);
    cudaFree(sc.base);
    return rc;
}
