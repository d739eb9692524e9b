// Baseline-JPEG encoding on the GPU, to the bytes cv::imwrite(".jpg") writes for a single-channel 8-bit image (mdc_jpeg_encode.cuh
// holds the per-block code the host shares).  Every stage runs over all blocks (or all bytes) of all frames of a batch:
//   E1  forward DCT + quantisation: eight threads per 8x8 block (a row each, then a column each, through shared memory); int16
//       coefficients in zig-zag order
//   E2  bits of each block's code, one thread per block; the DC difference is taken from the previous block's quantised DC
//   E3  exclusive scan of the block bit counts, one CTA per frame; the frame's total, and its word buffer zeroed up to it
//   E4  each block ORs its code into the word buffer at its bit offset, one thread per block (bits of different blocks are disjoint,
//       so the result does not depend on the order of the atomics); the last block adds the 1-bit padding
//   E5  one CTA per frame: the header, then the scan's bytes scattered after it with a 0x00 behind every 0xFF (an exclusive scan of
//       the 0xFF count of each 16-byte chunk), then EOI
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <vector>

#include "mdc_internal.h"
#include "mdc_jpeg_encode.cuh"

#define CU_CHECK(expr)                                                                          \
    do {                                                                                        \
        cudaError_t e__ = (expr);                                                               \
        if (e__ != cudaSuccess) {                                                               \
            mdc_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return MDC_ERR_CUDA;                                                                \
        }                                                                                       \
    } while (0)

namespace {

constexpr int kE1BlocksPerCta = 32;          // 8 threads per block
constexpr int kBlockThreads = 256;           // E2, E4: one thread per block
constexpr int kScanThreads = 1024;           // E3, E5: one CTA per frame
constexpr size_t kScratchCap = size_t(1) << 30;       // scratch of one group of frames, at least one frame

__device__ const uint8_t kZigZagEnc[64] = MDC_JPEG_ZIGZAG;

struct Header { uint8_t b[mdcje::kHeaderBytes]; };

// Per-frame layout of the scratch of a group of frames
struct Layout {
    size_t blocks;               // 8x8 blocks per frame
    size_t words;                // 32-bit words of a frame's scan buffer: a multiple of 4 that holds the worst-case scan + padding
    int16_t* coef;               // [frame][block][64]
    uint32_t* bits;              // [frame][block]
    unsigned long long* off;     // [frame][block]
    uint32_t* scan;              // [frame][words]
    unsigned long long* totals;  // [frame][2]: scan bits, 0xFF bytes
};

// Exclusive scan over a CTA of kScanThreads threads; returns the thread's prefix, the CTA's sum in *total
__device__ unsigned long long cta_exclusive_scan(unsigned long long v, unsigned long long* total) {
    __shared__ unsigned long long warp_sum[kScanThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long x = v;
    for (int d = 1; d < 32; d <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, d);
        if (lane >= d) x += y;
    }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    if (warp == 0) {
        unsigned long long s = warp_sum[lane];
        for (int d = 1; d < 32; d <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, s, d);
            if (lane >= d) s += y;
        }
        warp_sum[lane] = s;                                          // inclusive over warps
    }
    __syncthreads();
    const unsigned long long before = (warp ? warp_sum[warp - 1] : 0ull) + x - v;
    *total = warp_sum[kScanThreads / 32 - 1];
    __syncthreads();                                                 // warp_sum is reused by the next call
    return before;
}

// E1: blockIdx.y = frame, 32 blocks per CTA, 8 threads per block
__global__ void __launch_bounds__(8 * kE1BlocksPerCta) e1_fdct_quant(const uint8_t* __restrict__ frames, size_t pitch, int w, int h,
                                                                     mdcje::EncTables tab, Layout L) {
    __shared__ int32_t sdiv[64];
    __shared__ uint8_t szz_of[64];
    __shared__ int32_t ws[kE1BlocksPerCta][64];
    __shared__ __align__(16) int16_t sq[kE1BlocksPerCta][64];
    if (threadIdx.x < 64) {
        sdiv[threadIdx.x] = tab.div[threadIdx.x];
        szz_of[kZigZagEnc[threadIdx.x]] = static_cast<uint8_t>(threadIdx.x);
    }
    const int g = threadIdx.x >> 3, t = threadIdx.x & 7;
    const size_t blk = static_cast<size_t>(blockIdx.x) * kE1BlocksPerCta + g;
    const bool live = blk < L.blocks;
    const int bw = (w + 7) / 8;
    const int by = live ? static_cast<int>(blk / bw) : 0, bx = live ? static_cast<int>(blk - static_cast<size_t>(by) * bw) : 0;
    const uint8_t* frame = frames + static_cast<size_t>(blockIdx.y) * h * pitch;
    int32_t d[8], o[8];
    if (live) {
        mdcje::load_row(frame, pitch, w, h, bx, by, t, d);
        mdcje::fdct_1d(d, o, true);
        for (int i = 0; i < 8; ++i) ws[g][8 * t + i] = o[i];
    }
    __syncthreads();
    if (live) {
        for (int r = 0; r < 8; ++r) d[r] = ws[g][8 * r + t];
        mdcje::fdct_1d(d, o, false);
        for (int r = 0; r < 8; ++r) sq[g][szz_of[8 * r + t]] = mdcje::quantise(o[r], sdiv[8 * r + t]);
    }
    __syncthreads();
    if (live) reinterpret_cast<uint4*>(L.coef + (static_cast<size_t>(blockIdx.y) * L.blocks + blk) * 64)[t] = reinterpret_cast<const uint4*>(sq[g])[t];
}

__device__ void load_tables(const mdcje::EncTables& tab, mdcje::EncTables* s) {
    const uint32_t* src = reinterpret_cast<const uint32_t*>(&tab);
    uint32_t* dst = reinterpret_cast<uint32_t*>(s);
    for (int i = threadIdx.x; i < static_cast<int>(sizeof(mdcje::EncTables) / 4); i += blockDim.x) dst[i] = src[i];
    __syncthreads();
}

// E2: blockIdx.y = frame, one thread per block
__global__ void __launch_bounds__(kBlockThreads) e2_block_bits(mdcje::EncTables tab, Layout L) {
    __shared__ mdcje::EncTables s;
    load_tables(tab, &s);
    const size_t blk = static_cast<size_t>(blockIdx.x) * kBlockThreads + threadIdx.x;
    if (blk >= L.blocks) return;
    const int16_t* zz = L.coef + (static_cast<size_t>(blockIdx.y) * L.blocks + blk) * 64;
    const int pred = blk ? zz[-64] : 0;
    L.bits[static_cast<size_t>(blockIdx.y) * L.blocks + blk] = mdcje::block_bits(zz, pred, s);
}

// E3: one CTA per frame, four consecutive blocks per thread and pass
__global__ void __launch_bounds__(kScanThreads) e3_scan_bits(Layout L) {
    const size_t f = blockIdx.x;
    const uint32_t* bits = L.bits + f * L.blocks;
    unsigned long long* off = L.off + f * L.blocks;
    unsigned long long carry = 0;
    for (size_t base = 0; base < L.blocks; base += 4 * kScanThreads) {
        const size_t i0 = base + 4 * static_cast<size_t>(threadIdx.x);
        uint32_t v[4];
        unsigned long long sum = 0;
        for (int j = 0; j < 4; ++j) { v[j] = i0 + j < L.blocks ? bits[i0 + j] : 0u; sum += v[j]; }
        unsigned long long total;
        unsigned long long at = carry + cta_exclusive_scan(sum, &total);
        for (int j = 0; j < 4; ++j)
            if (i0 + j < L.blocks) { off[i0 + j] = at; at += v[j]; }
        carry += total;
    }
    if (threadIdx.x == 0) L.totals[2 * f] = carry;
    // the words the scan and its padding occupy, rounded up to whole 16-byte chunks, start out zero for E4
    const size_t chunks = (carry + 127) / 128;
    uint4* w = reinterpret_cast<uint4*>(L.scan + f * L.words);
    for (size_t i = threadIdx.x; i < chunks; i += kScanThreads) w[i] = make_uint4(0, 0, 0, 0);
}

struct OrDevice {
    uint32_t* w;
    __device__ void operator()(uint64_t i, uint32_t v) { if (v) atomicOr(w + i, v); }
};

// E4: blockIdx.y = frame, one thread per block
__global__ void __launch_bounds__(kBlockThreads) e4_emit(mdcje::EncTables tab, Layout L) {
    __shared__ mdcje::EncTables s;
    load_tables(tab, &s);
    const size_t blk = static_cast<size_t>(blockIdx.x) * kBlockThreads + threadIdx.x;
    if (blk >= L.blocks) return;
    const size_t fb = static_cast<size_t>(blockIdx.y) * L.blocks + blk;
    const int16_t* zz = L.coef + fb * 64;
    const int pred = blk ? zz[-64] : 0;
    OrDevice sink{L.scan + static_cast<size_t>(blockIdx.y) * L.words};
    mdcje::emit_block(zz, pred, s, L.off[fb], sink);
    if (blk == L.blocks - 1) mdcje::emit_padding(L.totals[2 * static_cast<size_t>(blockIdx.y)], sink);
}

// E5: one CTA per frame, one 16-byte chunk of the scan per thread and pass
__global__ void __launch_bounds__(kScanThreads) e5_stuff(Header hdr, Layout L, uint8_t* __restrict__ out, size_t out_stride) {
    const size_t f = blockIdx.x;
    uint8_t* dst = out + f * out_stride;
    for (int i = threadIdx.x; i < mdcje::kHeaderBytes; i += kScanThreads) dst[i] = hdr.b[i];
    dst += mdcje::kHeaderBytes;
    const unsigned long long nbytes = (L.totals[2 * f] + 7) / 8;
    const uint4* chunks = reinterpret_cast<const uint4*>(L.scan + f * L.words);
    const size_t n_chunks = (nbytes + 15) / 16;
    unsigned long long carry = 0;
    for (size_t base = 0; base < n_chunks; base += kScanThreads) {
        const size_t c = base + threadIdx.x;
        uint8_t b[16];
        int ff = 0;
        if (c < n_chunks) {                // bytes past nbytes are zero (E3), never 0xFF
            const uint4 v = chunks[c];
            memcpy(b, &v, 16);
            for (int j = 0; j < 16; ++j) ff += b[j] == 0xff;
        }
        unsigned long long total;
        unsigned long long at = c * 16 + carry + cta_exclusive_scan(static_cast<unsigned long long>(ff), &total);
        if (c < n_chunks) {
            const int n = static_cast<int>(min(16ull, nbytes - static_cast<unsigned long long>(c) * 16));
            for (int j = 0; j < n; ++j) {
                dst[at++] = b[j];
                if (b[j] == 0xff) dst[at++] = 0x00;
            }
        }
        carry += total;
    }
    if (threadIdx.x == 0) {
        dst[nbytes + carry] = 0xff;
        dst[nbytes + carry + 1] = 0xd9;
        L.totals[2 * f + 1] = carry;
    }
}

}  // namespace

extern "C" size_t mdc_jpeg_encode_bound(int w, int h) {
    if (w < 1 || h < 1 || w > 65535 || h > 65535) return 0;
    return mdcje::encode_bound(w, h);
}

extern "C" int mdc_jpeg_encode_device(mdc_ctx* c, const uint8_t* d_frames, size_t row_pitch, int n, int w, int h, int quality,
                                      uint8_t* d_out, size_t out_stride, size_t* sizes_host, mdc_stream stream) {
    if (!c || n < 0 || quality < 1 || quality > 100 || w < 1 || h < 1 || w > 65535 || h > 65535 || row_pitch < static_cast<size_t>(w) ||
        out_stride < mdc_jpeg_encode_bound(w, h) || (n > 0 && (!d_frames || !d_out || !sizes_host))) {
        mdc_set_error("mdc_jpeg_encode_device: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    if (n == 0) return MDC_OK;
    CU_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
    mdcje::EncTables tab;
    mdcje::make_tables(quality, &tab);
    Header hdr;
    mdcje::write_header(w, h, quality, hdr.b);

    Layout L;
    L.blocks = mdcje::block_count(w, h);
    L.words = (L.blocks * mdcje::kMaxBlockBits + 8 + 127) / 128 * 4;
    const size_t per_frame = L.blocks * (64 * sizeof(int16_t) + sizeof(uint32_t) + sizeof(unsigned long long)) + L.words * 4 + 16;
    const int group = static_cast<int>(std::max<size_t>(1, std::min<size_t>(static_cast<size_t>(n), kScratchCap / per_frame)));
    void* pool = nullptr;
    int rc = mdc_ctx_scratch_pool(c, &pool);
    if (rc != MDC_OK) return rc;
    uint8_t* scratch = nullptr;
    CU_CHECK(cudaMallocFromPoolAsync(reinterpret_cast<void**>(&scratch), per_frame * group + 256, static_cast<cudaMemPool_t>(pool), s));
    std::vector<unsigned long long> totals_host(2 * static_cast<size_t>(n));      // a few bytes per frame: pageable, no pinning per call
    // scratch layout of a group: totals | off | scan | coef | bits, every part 16-byte aligned
    L.totals = reinterpret_cast<unsigned long long*>(scratch);
    L.off = reinterpret_cast<unsigned long long*>(scratch + 16 * group);
    L.scan = reinterpret_cast<uint32_t*>(L.off + L.blocks * group + (L.blocks * group & 1));
    L.coef = reinterpret_cast<int16_t*>(L.scan + L.words * group);
    L.bits = reinterpret_cast<uint32_t*>(L.coef + L.blocks * group * 64);
    for (int f0 = 0; f0 < n && rc == MDC_OK; f0 += group) {
        const int g = std::min(group, n - f0);
        const uint8_t* frames = d_frames + static_cast<size_t>(f0) * h * row_pitch;
        e1_fdct_quant<<<dim3(static_cast<unsigned>((L.blocks + kE1BlocksPerCta - 1) / kE1BlocksPerCta), g), 8 * kE1BlocksPerCta, 0, s>>>(
            frames, row_pitch, w, h, tab, L);
        const dim3 per_block(static_cast<unsigned>((L.blocks + kBlockThreads - 1) / kBlockThreads), g);
        e2_block_bits<<<per_block, kBlockThreads, 0, s>>>(tab, L);
        e3_scan_bits<<<g, kScanThreads, 0, s>>>(L);
        e4_emit<<<per_block, kBlockThreads, 0, s>>>(tab, L);
        e5_stuff<<<g, kScanThreads, 0, s>>>(hdr, L, d_out + static_cast<size_t>(f0) * out_stride, out_stride);
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) { mdc_set_error("mdc_jpeg_encode_device: %s", cudaGetErrorString(e)); rc = MDC_ERR_CUDA; break; }
        mdc_ctx_add_launches(c, 5);
        const cudaError_t m = cudaMemcpyAsync(totals_host.data() + 2 * static_cast<size_t>(f0), L.totals, 2 * sizeof(unsigned long long) * g,
                                              cudaMemcpyDeviceToHost, s);
        if (m != cudaSuccess) { mdc_set_error("mdc_jpeg_encode_device: %s", cudaGetErrorString(m)); rc = MDC_ERR_CUDA; }
    }
    const cudaError_t fr = cudaFreeAsync(scratch, s);
    const cudaError_t e = cudaStreamSynchronize(s);
    if (rc == MDC_OK && (fr != cudaSuccess || e != cudaSuccess)) {
        mdc_set_error("mdc_jpeg_encode_device: %s", cudaGetErrorString(fr != cudaSuccess ? fr : e));
        rc = MDC_ERR_CUDA;
    }
    if (rc == MDC_OK)
        for (int k = 0; k < n; ++k)
            sizes_host[k] = mdcje::kHeaderBytes + (totals_host[2 * k] + 7) / 8 + totals_host[2 * k + 1] + 2;
    return rc;
}
