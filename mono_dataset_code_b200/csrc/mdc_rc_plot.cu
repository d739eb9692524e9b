// responseCalib's result images on the GPU: plotE and plotG (main_responseCalib.cpp:72-146), to the pixels the reference hands to
// cv::imwrite, bit for bit.
//   P1  mdc_rc_plot_e_range  {min ln(E+20), max ln(E+20), min E, max E}: per-CTA partials, then one CTA joins them.  Starting values
//       1e10 / -1e10 and strict comparisons as in the reference, so NaN is skipped; ties go to the lower pixel index, so +0 and -0
//       come out as the reference's scan leaves them and the result does not depend on the order of the join.
//   P2  mdc_rc_plot_e_map    one pass over E: the colour-mapped BGR pixel and the 16-bit irradiance, from a range in device memory
//   P3  mdc_rc_plot_g        the 256 x 256 plot of G, converted to 8 bits as cv::imwrite converts a float image
// Every operation is an explicitly rounded IEEE operation, and log / exp are glibc's (mdc_libm.h).  The conversions are those x86-64
// makes at -O3: float or double to int through a 32-bit truncation (cvttss2si / cvttsd2si: NaN and out-of-range values give
// INT_MIN), whose low byte or low 16 bits are stored.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>

#include "mdc_internal.h"
#include "mdc_libm.h"

#define CU_CHECK(expr)                                                                          \
    do {                                                                                        \
        cudaError_t e__ = (expr);                                                               \
        if (e__ != cudaSuccess) {                                                               \
            mdc_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return MDC_ERR_CUDA;                                                                \
        }                                                                                       \
    } while (0)

namespace {

constexpr int kThreads = 256;
constexpr int kRangeCtas = 264;            // two per SM of an H100 SXM; the partials are joined by one CTA

__device__ __forceinline__ int cvtt_f32(float x) { return (x >= -2147483648.0f && x < 2147483648.0f) ? __float2int_rz(x) : INT_MIN; }
__device__ __forceinline__ int cvtt_f64(double x) { return (x > -2147483649.0 && x < 2147483648.0) ? __double2int_rz(x) : INT_MIN; }

// Each extreme keeps the index of the pixel it came from.  Values that compare equal are either the same bits or +0 and -0; the
// reference's strict scan keeps the one it meets first, so on a tie the lower index wins, whatever order the threads join in.
struct Range { double v[4]; int at[4]; };      // min ln(E+20), max ln(E+20), min E, max E

__device__ __forceinline__ Range start_range() { return Range{{1e10, -1e10, 1e10, -1e10}, {INT_MAX, INT_MAX, INT_MAX, INT_MAX}}; }

__device__ __forceinline__ void take(Range& a, int k, double v, int at) {
    const bool better = (k & 1) ? v > a.v[k] : v < a.v[k];
    if (better || (v == a.v[k] && at < a.at[k])) { a.v[k] = v; a.at[k] = at; }
}

__device__ __forceinline__ void join(Range& a, const Range& b) {
#pragma unroll
    for (int k = 0; k < 4; ++k) take(a, k, b.v[k], b.at[k]);
}

__device__ Range block_join(Range r) {
    __shared__ Range part[kThreads / 32];
    for (int o = 16; o > 0; o >>= 1) {
        Range b;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            b.v[k] = __shfl_down_sync(0xffffffffu, r.v[k], o);
            b.at[k] = __shfl_down_sync(0xffffffffu, r.at[k], o);
        }
        join(r, b);
    }
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = r;
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < kThreads / 32; ++w) join(r, part[w]);
    return r;
}

__global__ void __launch_bounds__(kThreads) rc_plot_e_partials(const double* __restrict__ E, int npix, Range* __restrict__ partials) {
    Range r = start_range();
    for (int i = blockIdx.x * kThreads + threadIdx.x; i < npix; i += gridDim.x * kThreads) {      // rising i: strict tests keep the first
        const double e = E[i];
        const double le = mdc_log(__dadd_rn(e, 20.0));
        if (le < r.v[0]) { r.v[0] = le; r.at[0] = i; }
        if (le > r.v[1]) { r.v[1] = le; r.at[1] = i; }
        if (e < r.v[2]) { r.v[2] = e; r.at[2] = i; }
        if (e > r.v[3]) { r.v[3] = e; r.at[3] = i; }
    }
    r = block_join(r);
    if (threadIdx.x == 0) partials[blockIdx.x] = r;
}

__global__ void __launch_bounds__(kThreads) rc_plot_e_join(const Range* __restrict__ partials, int n, double* __restrict__ range4) {
    Range r = start_range();
    for (int i = threadIdx.x; i < n; i += kThreads) join(r, partials[i]);
    r = block_join(r);
    if (threadIdx.x == 0)
        for (int k = 0; k < 4; ++k) range4[k] = r.v[k];
}

// main_responseCalib.cpp:94-109 for one pixel
__global__ void __launch_bounds__(kThreads) rc_plot_e_map(const double* __restrict__ E, int npix, const double* __restrict__ range4,
                                                          uint8_t* __restrict__ bgr, uint16_t* __restrict__ e16) {
    const int i = blockIdx.x * kThreads + threadIdx.x;
    if (i >= npix) return;
    const double lmin = range4[0], lmax = range4[1], emin = range4[2], emax = range4[3];
    const double e = E[i];
    const double le = mdc_log(__dadd_rn(e, 20.0));
    const double v = __ddiv_rn(__dmul_rn(3.0, __dsub_rn(mdc_exp(__ddiv_rn(__dsub_rn(le, lmin), __dsub_rn(lmax, lmin))), 1.0)), 1.7183);
    const float val = __double2float_rn(v);
    const int icP = cvtt_f32(val);
    const float ifP = __fsub_rn(val, __int2float_rn(icP));
    const uint8_t c = static_cast<uint8_t>(cvtt_f32(__fmul_rn(255.0f, ifP)));
    uint8_t b = 0, g = 0, r = 0;                  // cv::Vec3b(): black when icP % 3 is negative (NaN, val >= 2^31)
    switch (icP % 3) {
        case 0: r = c; break;
        case 1: g = c; r = 255; break;
        case 2: b = c; g = 255; r = 255; break;
        default: break;
    }
    bgr[3 * static_cast<size_t>(i)] = b;
    bgr[3 * static_cast<size_t>(i) + 1] = g;
    bgr[3 * static_cast<size_t>(i) + 2] = r;
    e16[i] = static_cast<uint16_t>(cvtt_f64(__ddiv_rn(__dmul_rn(65025.0, __dsub_rn(e, emin)), __dsub_rn(emax, emin))));
}

// main_responseCalib.cpp:120-146: thread i owns column i; min / max by the reference's sequential scan (256 values)
__global__ void __launch_bounds__(256) rc_plot_g(const double* __restrict__ G, uint8_t* __restrict__ out, double* __restrict__ minmax) {
    __shared__ double g[256];
    const int i = threadIdx.x;
    g[i] = G[i];
    __syncthreads();
    double mn = 1e10, mx = -1e10;
    for (int k = 0; k < 256; ++k) {
        if (g[k] < mn) mn = g[k];
        if (g[k] > mx) mx = g[k];
    }
    if (i == 0) { minmax[0] = mn; minmax[1] = mx; }
    const double val = __ddiv_rn(__dmul_rn(256.0, __dsub_rn(g[i], mn)), __dsub_rn(mx, mn));
    for (int k = 0; k < 256; ++k) {
        int q = 0;
        if (val < k) {
            // GImg * 255 in float, then saturate_cast<uchar>: round half to even, NaN and values outside int32 -> 0
            const float f = __fmul_rn(__double2float_rn(__dsub_rn(static_cast<double>(k), val)), 255.0f);
            q = (f >= -2147483648.0f && f < 2147483648.0f) ? __float2int_rn(f) : INT_MIN;
            q = q < 0 ? 0 : (q > 255 ? 255 : q);
        }
        out[k * 256 + i] = static_cast<uint8_t>(q);
    }
}

__global__ void libm_eval(int op, const double* __restrict__ in, double* __restrict__ out, size_t n) {
    for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += static_cast<size_t>(gridDim.x) * blockDim.x)
        out[i] = op == MDC_LIBM_EXP ? mdc_exp(in[i]) : mdc_log(in[i]);
}

cudaStream_t pick(mdc_ctx* c, mdc_stream stream) {
    return stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
}

int done(mdc_stream user_stream, cudaStream_t s, const char* who) {
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && !user_stream) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) { mdc_set_error("%s: %s", who, cudaGetErrorString(e)); return MDC_ERR_CUDA; }
    return MDC_OK;
}

}  // namespace

extern "C" int mdc_rc_plot_e_range(mdc_ctx* c, const double* d_E, int npix, double* d_range4, mdc_stream stream) {
    if (!c || npix < 0 || (npix > 0 && !d_E) || !d_range4) { mdc_set_error("mdc_rc_plot_e_range: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    const cudaStream_t s = pick(c, stream);
    const int ctas = npix == 0 ? 1 : static_cast<int>(std::min<long long>(kRangeCtas, (npix + kThreads - 1) / kThreads));
    void* pool = nullptr;
    int rc = mdc_ctx_scratch_pool(c, &pool);
    if (rc != MDC_OK) return rc;
    Range* partials = nullptr;
    CU_CHECK(cudaMallocFromPoolAsync(reinterpret_cast<void**>(&partials), sizeof(Range) * ctas, static_cast<cudaMemPool_t>(pool), s));
    rc_plot_e_partials<<<ctas, kThreads, 0, s>>>(d_E, npix, partials);
    rc_plot_e_join<<<1, kThreads, 0, s>>>(partials, ctas, d_range4);
    mdc_ctx_add_launches(c, 2);
    CU_CHECK(cudaFreeAsync(partials, s));
    return done(stream, s, "mdc_rc_plot_e_range");
}

extern "C" int mdc_rc_plot_e_map(mdc_ctx* c, const double* d_E, int npix, const double* d_range4, uint8_t* d_bgr, uint16_t* d_e16,
                                 mdc_stream stream) {
    if (!c || npix < 0 || !d_range4 || (npix > 0 && (!d_E || !d_bgr || !d_e16))) {
        mdc_set_error("mdc_rc_plot_e_map: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    CU_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    const cudaStream_t s = pick(c, stream);
    if (npix > 0) {
        rc_plot_e_map<<<(npix + kThreads - 1) / kThreads, kThreads, 0, s>>>(d_E, npix, d_range4, d_bgr, d_e16);
        mdc_ctx_add_launches(c, 1);
    }
    return done(stream, s, "mdc_rc_plot_e_map");
}

extern "C" int mdc_rc_plot_e(mdc_ctx* c, const double* d_E, int npix, double* d_range4, uint8_t* d_bgr, uint16_t* d_e16, mdc_stream stream) {
    if (!c || npix < 0 || !d_range4 || (npix > 0 && (!d_E || !d_bgr || !d_e16))) {
        mdc_set_error("mdc_rc_plot_e: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    const mdc_stream s = pick(c, stream);
    int rc = mdc_rc_plot_e_range(c, d_E, npix, d_range4, s);
    if (rc == MDC_OK) rc = mdc_rc_plot_e_map(c, d_E, npix, d_range4, d_bgr, d_e16, s);
    if (rc == MDC_OK && !stream) CU_CHECK(cudaStreamSynchronize(static_cast<cudaStream_t>(s)));
    return rc;
}

extern "C" int mdc_rc_plot_g(mdc_ctx* c, const double* d_G, uint8_t* d_out, double* minmax_host, mdc_stream stream) {
    if (!c || !d_G || !d_out) { mdc_set_error("mdc_rc_plot_g: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    const cudaStream_t s = pick(c, stream);
    void* pool = nullptr;
    int rc = mdc_ctx_scratch_pool(c, &pool);
    if (rc != MDC_OK) return rc;
    double* d_minmax = nullptr;
    CU_CHECK(cudaMallocFromPoolAsync(reinterpret_cast<void**>(&d_minmax), 2 * sizeof(double), static_cast<cudaMemPool_t>(pool), s));
    rc_plot_g<<<1, 256, 0, s>>>(d_G, d_out, d_minmax);
    mdc_ctx_add_launches(c, 1);
    double mm[2] = {0, 0};
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && minmax_host) e = cudaMemcpyAsync(mm, d_minmax, sizeof mm, cudaMemcpyDeviceToHost, s);
    const cudaError_t f = cudaFreeAsync(d_minmax, s);
    if (e == cudaSuccess) e = f;
    if (e == cudaSuccess && (minmax_host || !stream)) e = cudaStreamSynchronize(s);      // the minimum and maximum are read here
    if (e != cudaSuccess) { mdc_set_error("mdc_rc_plot_g: %s", cudaGetErrorString(e)); return MDC_ERR_CUDA; }
    if (minmax_host) { minmax_host[0] = mm[0]; minmax_host[1] = mm[1]; }
    return MDC_OK;
}

extern "C" void mdc_libm_host(int op, const double* in, double* out, size_t n) {
    for (size_t i = 0; i < n; ++i) out[i] = op == MDC_LIBM_EXP ? mdc_exp(in[i]) : mdc_log(in[i]);
}

extern "C" int mdc_libm_device(int op, const double* d_in, double* d_out, size_t n, int device, mdc_stream stream) {
    if ((op != MDC_LIBM_EXP && op != MDC_LIBM_LOG) || (n && (!d_in || !d_out))) { mdc_set_error("mdc_libm_device: bad argument"); return MDC_ERR_INVALID_ARG; }
    CU_CHECK(cudaSetDevice(device));
    const cudaStream_t s = static_cast<cudaStream_t>(stream);
    if (n) libm_eval<<<static_cast<unsigned>(std::min<size_t>((n + 255) / 256, 4096)), 256, 0, s>>>(op, d_in, d_out, n);
    CU_CHECK(cudaGetLastError());
    if (!stream) CU_CHECK(cudaStreamSynchronize(nullptr));
    return MDC_OK;
}
