// The per-pixel half of vignetteCalib's marker detection (main_vignetteCalib.cpp:235-238, aruco-1.3.0/src/markerdetector.cpp:437-458):
// the rectified float frame rounded to 8 bits (convertTo(CV_8U, 1, 0)) and aruco's adaptive threshold of it,
//   cv::adaptiveThreshold(grey, 255, ADAPTIVE_THRESH_MEAN_C, THRESH_BINARY_INV, 7, 7)
// i.e. mean = the 7x7 box mean of grey with replicated image borders, rounded to 8 bits, and mask = (grey - mean <= -7) ? 255 : 0.
// One CTA produces a 32 x 32 tile of one frame: it rounds the tile and its 3-pixel apron into shared memory, sums rows of 7, then
// columns of 7.  All sums are integers; a sum / 49 is never within 0.01 of a half, so the fp32 division rounds as OpenCV does.
#include <cuda_runtime.h>

#include <algorithm>

#include "mdc_internal.h"

namespace {

constexpr int kTile = 32;
constexpr int kApron = 3;
constexpr int kIn = kTile + 2 * kApron;

// saturate_cast<uchar>(float): round half to even, then clamp (NaN -> 0; OpenCV on x86 also gives 0 for values >= 2^31, which
// rectified 8-bit frames never have)
__device__ __forceinline__ int round_u8(float v) {
    return v != v ? 0 : min(max(__float2int_rn(v), 0), 255);
}

__global__ void __launch_bounds__(256) marker_threshold_kernel(const float* __restrict__ rect, int n, int w, int h,
                                                               uint8_t* __restrict__ grey, uint8_t* __restrict__ mask) {
    __shared__ int g[kIn][kIn];
    __shared__ int rows[kIn][kTile];
    const size_t npx = static_cast<size_t>(w) * h;
    const int tiles_x = (w + kTile - 1) / kTile;
    const int x0 = static_cast<int>(blockIdx.x % tiles_x) * kTile, y0 = static_cast<int>(blockIdx.x / tiles_x) * kTile;
    const int tid = threadIdx.y * blockDim.x + threadIdx.x, nthreads = blockDim.x * blockDim.y;
    for (int f = blockIdx.z; f < n; f += gridDim.z) {
        const float* src = rect + f * npx;
        for (int i = tid; i < kIn * kIn; i += nthreads) {
            const int yy = min(max(y0 + i / kIn - kApron, 0), h - 1), xx = min(max(x0 + i % kIn - kApron, 0), w - 1);   // BORDER_REPLICATE
            g[i / kIn][i % kIn] = round_u8(src[static_cast<size_t>(yy) * w + xx]);
        }
        __syncthreads();
        for (int i = tid; i < kIn * kTile; i += nthreads) {
            const int r = i / kTile, c = i % kTile;
            int s = 0;
#pragma unroll
            for (int k = 0; k < 7; ++k) s += g[r][c + k];
            rows[r][c] = s;
        }
        __syncthreads();
        for (int i = tid; i < kTile * kTile; i += nthreads) {
            const int r = i / kTile, c = i % kTile, y = y0 + r, x = x0 + c;
            if (y < h && x < w) {
                int s = 0;
#pragma unroll
                for (int k = 0; k < 7; ++k) s += rows[r + k][c];
                const int mean = min(max(__float2int_rn(__int2float_rn(s) / 49.0f), 0), 255);
                const int v = g[r + kApron][c + kApron];
                const size_t o = f * npx + static_cast<size_t>(y) * w + x;
                grey[o] = static_cast<uint8_t>(v);
                mask[o] = v - mean <= -7 ? 255 : 0;
            }
        }
        __syncthreads();
    }
}

}  // namespace

extern "C" int mdc_marker_threshold(mdc_ctx* c, const float* d_rect, int n, int w, int h, uint8_t* d_grey, uint8_t* d_mask, mdc_stream stream) {
    if (!c || n < 0 || w < 1 || h < 1 || (n > 0 && (!d_rect || !d_grey || !d_mask))) {
        mdc_set_error("mdc_marker_threshold: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    if (static_cast<long long>(w) * h > (1LL << 28)) {
        mdc_set_error("mdc_marker_threshold: image larger than 2^28 pixels");
        return MDC_ERR_INVALID_ARG;
    }
    if (n == 0) return MDC_OK;
    cudaError_t e = cudaSetDevice(mdc_ctx_device_ordinal(c));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
    if (e == cudaSuccess) {
        const dim3 grid(((w + kTile - 1) / kTile) * ((h + kTile - 1) / kTile), 1, std::min(n, 65535));   // tiles in x: up to 2^23 of them
        marker_threshold_kernel<<<grid, dim3(32, 8), 0, s>>>(d_rect, n, w, h, d_grey, d_mask);
        e = cudaGetLastError();
        mdc_ctx_add_launches(c, 1);
    }
    if (e == cudaSuccess && !stream) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
        mdc_set_error("mdc_marker_threshold: %s", cudaGetErrorString(e));
        return MDC_ERR_CUDA;
    }
    return MDC_OK;
}
