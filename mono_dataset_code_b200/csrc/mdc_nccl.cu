// Native NCCL side of the multi-GPU paths (see include/mdc_b200_nccl.h): communicator helpers, broadcast of the calibration
// tables (frame-sharded K1), and the pixel-sharded responseCalib loop with its two all-reduces.
#include <cuda_runtime.h>
#include <nccl.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>

#include "mdc_b200.h"
#include "mdc_b200_nccl.h"

namespace {
// error text goes through stderr here: mdc_set_error lives in the other library and is not part of its ABI
#define NC_CHECK(expr, code)                                                                      \
    do {                                                                                          \
        if (!(expr)) { fprintf(stderr, "mdc_ctx_create_broadcast: %s failed (%s:%d)\n", #expr, __FILE__, __LINE__); return code; } \
    } while (0)
}  // namespace

extern "C" int mdc_ctx_create_broadcast(void* nccl_comm, int rank, int root, int device, const mdc_fov* fov, const mdc_photo* photo,
                                        mdc_ctx** out) {
    if (!nccl_comm || !out) return MDC_ERR_INVALID_ARG;
    *out = nullptr;
    ncclComm_t comm = static_cast<ncclComm_t>(nccl_comm);
    NC_CHECK(cudaSetDevice(device) == cudaSuccess, MDC_ERR_CUDA);
    cudaStream_t s;
    NC_CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess, MDC_ERR_CUDA);

    // geometry + which tables exist
    int meta_h[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (rank == root) {
        if (fov) mdc_fov_dims(fov, &meta_h[0], &meta_h[1], &meta_h[2], &meta_h[3]);
        meta_h[4] = fov && mdc_fov_is_valid(fov);
        meta_h[5] = photo && mdc_photo_valid_gamma(photo);
        meta_h[6] = photo && mdc_photo_valid_vignette(photo);
    }
    int* meta_d = nullptr;
    NC_CHECK(cudaMalloc(&meta_d, sizeof meta_h) == cudaSuccess, MDC_ERR_CUDA);
    NC_CHECK(cudaMemcpyAsync(meta_d, meta_h, sizeof meta_h, cudaMemcpyHostToDevice, s) == cudaSuccess, MDC_ERR_CUDA);
    NC_CHECK(ncclBroadcast(meta_d, meta_d, 8, ncclInt, root, comm, s) == ncclSuccess, MDC_ERR_CUDA);
    NC_CHECK(cudaMemcpyAsync(meta_h, meta_d, sizeof meta_h, cudaMemcpyDeviceToHost, s) == cudaSuccess, MDC_ERR_CUDA);
    NC_CHECK(cudaStreamSynchronize(s) == cudaSuccess, MDC_ERR_CUDA);
    cudaFree(meta_d);
    const int in_w = meta_h[0], in_h = meta_h[1], out_w = meta_h[2], out_h = meta_h[3];
    const bool has_fov = meta_h[4] != 0, has_g = meta_h[5] != 0, has_v = meta_h[6] != 0;

    auto bcast = [&](const float* host_src, size_t count, float** dev) -> bool {
        if (cudaMalloc(dev, count * sizeof(float)) != cudaSuccess) return false;
        if (rank == root && cudaMemcpyAsync(*dev, host_src, count * sizeof(float), cudaMemcpyHostToDevice, s) != cudaSuccess) return false;
        return ncclBroadcast(*dev, *dev, count, ncclFloat, root, comm, s) == ncclSuccess;
    };
    float *rx = nullptr, *ry = nullptr, *g = nullptr, *v = nullptr;
    const size_t n_out = static_cast<size_t>(out_w) * out_h, n_in = static_cast<size_t>(in_w) * in_h;
    if (has_fov) {
        NC_CHECK(bcast(rank == root ? mdc_fov_remap_x(fov) : nullptr, n_out, &rx), MDC_ERR_CUDA);
        NC_CHECK(bcast(rank == root ? mdc_fov_remap_y(fov) : nullptr, n_out, &ry), MDC_ERR_CUDA);
    }
    if (has_g) NC_CHECK(bcast(rank == root ? mdc_photo_ginv(const_cast<mdc_photo*>(photo)) : nullptr, 256, &g), MDC_ERR_CUDA);
    if (has_v) NC_CHECK(bcast(rank == root ? mdc_photo_vignette_map_inv(photo) : nullptr, n_in, &v), MDC_ERR_CUDA);
    NC_CHECK(cudaStreamSynchronize(s) == cudaSuccess, MDC_ERR_CUDA);
    cudaStreamDestroy(s);

    int rc = mdc_ctx_create_from_device_tables(device, in_w, in_h, out_w, out_h, rx, ry, g, v, out);
    if (rc != MDC_OK) { cudaFree(rx); cudaFree(ry); cudaFree(g); cudaFree(v); return rc; }
    return mdc_ctx_take_table_ownership(*out);   // the context now frees the four buffers
}


// ---------------------------------------------------------------- communicator helpers (so that hosts without an NCCL binding of
// their own — ctypes, a C++ program — can set one up: rank 0 makes the id, ships the 128 bytes to its peers by any means, all init)
extern "C" int mdc_nccl_unique_id(char id_out[128]) {
    if (!id_out) return MDC_ERR_INVALID_ARG;
    static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
    ncclUniqueId id;
    NC_CHECK(ncclGetUniqueId(&id) == ncclSuccess, MDC_ERR_CUDA);
    memcpy(id_out, &id, sizeof id);
    return MDC_OK;
}
extern "C" int mdc_nccl_comm_create(const char id[128], int world, int rank, int device, void** comm_out) {
    if (!id || !comm_out || world < 1 || rank < 0 || rank >= world) return MDC_ERR_INVALID_ARG;
    *comm_out = nullptr;
    NC_CHECK(cudaSetDevice(device) == cudaSuccess, MDC_ERR_CUDA);
    ncclUniqueId uid;
    memcpy(&uid, id, sizeof uid);
    ncclComm_t comm = nullptr;
    NC_CHECK(ncclCommInitRank(&comm, world, uid, rank) == ncclSuccess, MDC_ERR_CUDA);
    *comm_out = comm;
    return MDC_OK;
}
extern "C" void mdc_nccl_comm_destroy(void* comm) { if (comm) ncclCommDestroy(static_cast<ncclComm_t>(comm)); }
extern "C" int mdc_nccl_version(void) { int v = 0; ncclGetVersion(&v); return v; }

// ---------------------------------------------------------------- pixel-sharded responseCalib (SURVEY.md §8e row 2)
// main(), main_responseCalib.cpp:281-362, with the image stack split by pixel range: every pass is per-pixel work on the local
// slice; the G-step's sums (:290-299) are added across ranks as integers — one all-reduce(MAX) of the scale inputs, then
// all-reduce(SUM) of 768 int64 limbs, 256 fp64 side sums and, once, 256 counts — so that G and E are bit-identical for any number of
// ranks; rmse's {error, count} pair (:50-69) is summed as fp64.  All of it is latency-bound on NVLink (<= 6 KB per call).
extern "C" int mdc_response_calib_sharded(mdc_ctx* c, void* nccl_comm, int device, const uint8_t* d_data_local, int n, int npix_local,
                                          const double* d_t, int nits, double* d_E_local, double* d_G, double* log_host) {
    if (!c || !nccl_comm || !d_t || !d_G || n < 1 || npix_local < 0 || nits < 0) return MDC_ERR_INVALID_ARG;
    ncclComm_t comm = static_cast<ncclComm_t>(nccl_comm);
    NC_CHECK(cudaSetDevice(device) == cudaSuccess, MDC_ERR_CUDA);
    cudaStream_t s;
    NC_CHECK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) == cudaSuccess, MDC_ERR_CUDA);
    double* scratch = nullptr;                                   // special[256] | gnum[256] (u64) | acc[2] | scale[4] (u64) | limbs[768] (i64)
    NC_CHECK(cudaMalloc(&scratch, (256 + 256 + 2 + 4 + 768) * sizeof(double)) == cudaSuccess, MDC_ERR_CUDA);
    double* special = scratch;
    unsigned long long* gnum = reinterpret_cast<unsigned long long*>(scratch + 256);
    double* acc = scratch + 512;
    unsigned long long* scale = reinterpret_cast<unsigned long long*>(scratch + 514);
    long long* limbs = reinterpret_cast<long long*>(scratch + 518);
    int rc = MDC_OK;
    auto rmse = [&](double out[2]) -> int {
        int r = mdc_rc_rmse_accumulate(c, d_data_local, n, npix_local, d_t, d_G, d_E_local, acc, s);
        if (r != MDC_OK) return r;
        if (ncclAllReduce(acc, acc, 2, ncclDouble, ncclSum, comm, s) != ncclSuccess) return MDC_ERR_CUDA;
        double h[2];
        if (cudaMemcpyAsync(h, acc, sizeof h, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) return MDC_ERR_CUDA;
        out[0] = 1e5 * sqrt(h[0] / h[1]);
        out[1] = h[1];
        return MDC_OK;
    };
    // counts can be carried over from the first iteration only on the bulk-copy path (16-byte aligned slice of a multiple of 16 pixels)
    bool reusable = npix_local % 16 == 0 && (reinterpret_cast<uintptr_t>(d_data_local) & 15) == 0;
    {   // the ranks must agree on it, or they would disagree on which all-reduces happen
        unsigned long long flag = reusable ? 1ull : 0ull;
        if (cudaMemcpyAsync(gnum, &flag, sizeof flag, cudaMemcpyHostToDevice, s) != cudaSuccess ||
            ncclAllReduce(gnum, gnum, 1, ncclUint64, ncclMin, comm, s) != ncclSuccess ||
            cudaMemcpyAsync(&flag, gnum, sizeof flag, cudaMemcpyDeviceToHost, s) != cudaSuccess || cudaStreamSynchronize(s) != cudaSuccess) {
            cudaFree(scratch); cudaStreamDestroy(s);
            return MDC_ERR_CUDA;
        }
        reusable = flag != 0;
    }
    // every per-rank call accepts an empty slice (npix_local = 0, null data and E), so every rank makes the same calls and collectives
    rc = mdc_rc_einit(c, d_data_local, n, npix_local, d_E_local, s);
    if (rc == MDC_OK && cudaMemsetAsync(d_G, 0, 256 * sizeof(double), s) != cudaSuccess) rc = MDC_ERR_CUDA;
    for (int it = 0; it < nits && rc == MDC_OK; ++it) {
        double r[2], row[4] = {0, 0, 0, 0};
        const bool reuse = it > 0 && reusable;
        // G-step with sums that are exact across ranks: one scale for all (MAX), integer limbs + fp64 side sums (SUM)
        if ((rc = mdc_rc_gstep_scale(c, d_E_local, npix_local, d_t, n, scale, s)) != MDC_OK) break;
        if (ncclAllReduce(scale, scale, 4, ncclUint64, ncclMax, comm, s) != ncclSuccess) { rc = MDC_ERR_CUDA; break; }
        rc = mdc_rc_gstep_accumulate_exact(c, d_data_local, n, npix_local, d_t, d_E_local, scale, limbs, special, gnum, reuse ? 1 : 0, s);
        if (rc != MDC_OK) break;
        if (ncclAllReduce(limbs, limbs, 768, ncclInt64, ncclSum, comm, s) != ncclSuccess) { rc = MDC_ERR_CUDA; break; }
        if (ncclAllReduce(special, special, 256, ncclDouble, ncclSum, comm, s) != ncclSuccess) { rc = MDC_ERR_CUDA; break; }
        if (!reuse && ncclAllReduce(gnum, gnum, 256, ncclUint64, ncclSum, comm, s) != ncclSuccess) { rc = MDC_ERR_CUDA; break; }
        if ((rc = mdc_rc_gstep_finish_exact(c, scale, limbs, special, gnum, d_G, s)) != MDC_OK) break;
        if ((rc = rmse(r)) != MDC_OK) break;
        row[0] = r[0];
        if ((rc = mdc_estep(c, d_data_local, n, npix_local, d_t, d_G, d_E_local, s)) != MDC_OK) break;
        if ((rc = rmse(r)) != MDC_OK) break;
        row[1] = r[0];
        // rescale (:350-355): the factor comes from the replicated G, so every rank applies the same one to its slice and to its G
        if (cudaStreamSynchronize(s) != cudaSuccess) { rc = MDC_ERR_CUDA; break; }
        double factor = 0;
        if ((rc = mdc_rc_rescale(c, npix_local, d_E_local, d_G, &factor)) != MDC_OK) break;
        if ((rc = rmse(r)) != MDC_OK) break;
        row[2] = r[0]; row[3] = r[1];
        if (log_host) memcpy(log_host + 4 * it, row, sizeof row);
    }
    cudaStreamSynchronize(s);
    cudaFree(scratch);
    cudaStreamDestroy(s);
    return rc;
}
