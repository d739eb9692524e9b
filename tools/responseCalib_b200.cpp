// responseCalib on the GPU: a C++ host for the calibrator kernels behind include/mdc_b200.h.
//
// Same command line, same inputs and the same result files as the reference's responseCalib program
// (/root/reference/src/main_responseCalib.cpp:149-173 arguments, :191-237 loading + saturation leak padding,
// :249-259 starting irradiance, :281-362 optimisation loop, :359 log.txt rows, :367-375 pcalib.txt), with every pass over
// the image stack — padding, E-init, G-step, E-step, rescale, rmse — running in the sm_90a kernels of libmdc_b200.so.
// The reference's debug plots (plotE / plotG, imshow) are GUI output and are not produced.
//
//   responseCalib_b200 <dataset dir/> [leakPadding=2] [iterations=10] [skip=1] [device=0]
//
// Build (see tests/test_tools_cpp.py):  g++ -std=c++11 -O2 -Iinclude tools/responseCalib_b200.cpp -Lmono_dataset_code_b200/lib
//                                       -lmdc_b200 -L/usr/local/cuda/lib64 -lcudart -o responseCalib_b200
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <vector>

#include "mdc_b200.h"

namespace {

struct Options { int leak_padding = 2, iterations = 10, skip = 1, device = 0; };

void parse_option(const char* arg, Options* o) {
    int v;
    if (sscanf(arg, "leakPadding=%d", &v) == 1) { o->leak_padding = v; printf("leakPadding set to %d!\n", v); return; }
    if (sscanf(arg, "iterations=%d", &v) == 1) { o->iterations = v; printf("nits set to %d!\n", v); return; }
    if (sscanf(arg, "skip=%d", &v) == 1) { o->skip = v; printf("skipFrames set to %d!\n", v); return; }
    if (sscanf(arg, "device=%d", &v) == 1) { o->device = v; return; }
    printf("could not parse argument \"%s\"!!\n", arg);
}

#define CUDA_OR_DIE(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { printf("%s: %s\n", #expr, cudaGetErrorString(e__)); exit(2); } } while (0)
#define MDC_OR_DIE(expr) do { int r__ = (expr); if (r__ != MDC_OK) { printf("%s failed (%d): %s\n", #expr, r__, mdc_last_error()); exit(2); } } while (0)

}  // namespace

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: responseCalib_b200 <dataset dir/> [leakPadding=N] [iterations=N] [skip=N] [device=N]\n"); return 1; }
    Options opt;
    for (int i = 2; i < argc; ++i) parse_option(argv[i], &opt);
    if (opt.skip < 1) opt.skip = 1;

    // ---- the exposure sweep: every skip-th frame that decodes, with its exposure time.  The first one that decodes sets the size
    // (main_responseCalib.cpp:192-205); all of them are decoded in one call (JPEG frames on the GPU) into the device stack, and
    // frames that cannot be decoded are skipped.
    mdc_seq* seq = nullptr;
    if (mdc_seq_open(argv[1], &seq) != MDC_OK) { printf("cannot open dataset %s: %s\n", argv[1], mdc_last_error()); return 1; }
    std::vector<int> ids;
    for (int i = 0; i < mdc_seq_num_images(seq); i += opt.skip) ids.push_back(i);
    int w = 0, h = 0;
    for (int i : ids)
        if (mdc_seq_read_gray8(seq, i, nullptr, 0, &w, &h) == MDC_OK) break;       // leaves w, h at 0 if it fails
    std::vector<double> exposures;
    mdc_ctx* ctx = nullptr;
    unsigned char* d_data = nullptr;
    if (w > 0) {
        CUDA_OR_DIE(cudaSetDevice(opt.device));
        MDC_OR_DIE(mdc_ctx_create(opt.device, nullptr, nullptr, &ctx));
        const size_t frame_bytes = static_cast<size_t>(w) * h;
        CUDA_OR_DIE(cudaMalloc(&d_data, frame_bytes * ids.size()));
        std::vector<int> status(ids.size()), sizes(2 * ids.size());
        const int r = mdc_seq_read_gray8_device(ctx, seq, ids.data(), static_cast<int>(ids.size()), w, h, d_data, w, status.data(), sizes.data(), 0, nullptr);
        if (r != MDC_OK && r != MDC_ERR_FORMAT) { printf("mdc_seq_read_gray8_device failed (%d): %s\n", r, mdc_last_error()); exit(2); }
        for (size_t k = 0; k < ids.size(); ++k) {
            if (status[k] == MDC_ERR_FORMAT) continue;                                                    // undecodable frame: skipped
            if (sizes[2 * k] != w) { printf("width mismatch!\n"); return 1; }
            if (sizes[2 * k + 1] != h) { printf("height mismatch!\n"); return 1; }
            const size_t n = exposures.size();
            if (n != k) CUDA_OR_DIE(cudaMemcpy(d_data + n * frame_bytes, d_data + k * frame_bytes, frame_bytes, cudaMemcpyDeviceToDevice));
            exposures.push_back(static_cast<double>(mdc_seq_exposure(seq, ids[k])));
        }
    }
    const int n = static_cast<int>(exposures.size());
    const int npix = w * h;
    printf("loaded %d images\n", n);
    if (n < 1) return 1;

    // ---- device state: image stack (above), exposure times, irradiance E, inverse response G
    double *d_t = nullptr, *d_E = nullptr, *d_G = nullptr;
    CUDA_OR_DIE(cudaMalloc(&d_t, sizeof(double) * n));
    CUDA_OR_DIE(cudaMalloc(&d_E, sizeof(double) * npix));
    CUDA_OR_DIE(cudaMalloc(&d_G, sizeof(double) * 256));
    CUDA_OR_DIE(cudaMemcpy(d_t, exposures.data(), sizeof(double) * n, cudaMemcpyHostToDevice));
    MDC_OR_DIE(mdc_rc_leak_padding(ctx, d_data, n, w, h, opt.leak_padding, nullptr));

    if (system("rm -rf photoCalibResult") == -1) printf("could not delete old photoCalibResult folder!\n");
    if (system("mkdir photoCalibResult") == -1) printf("could not create photoCalibResult folder!\n");

    // rmse of the starting point (E = mean image, G = 0), as the reference prints it before its loop
    {
        double r[2] = {0, 0};
        CUDA_OR_DIE(cudaMemset(d_G, 0, sizeof(double) * 256));
        MDC_OR_DIE(mdc_rc_einit(ctx, d_data, n, npix, d_E, nullptr));
        MDC_OR_DIE(mdc_rc_rmse(ctx, d_data, n, npix, d_t, d_G, d_E, r));
        printf("init RMSE = %f! \t", r[0]);
    }

    // ---- the optimisation loop (prints the per-iteration rmse lines itself)
    std::vector<double> log(static_cast<size_t>(4) * (opt.iterations > 0 ? opt.iterations : 1), 0.0);
    MDC_OR_DIE(mdc_response_calib(ctx, d_data, n, npix, d_t, opt.iterations, d_E, d_G, log.data()));

    {
        std::ofstream lf("photoCalibResult/log.txt", std::ios::trunc | std::ios::out);
        lf.precision(15);
        for (int it = 0; it < opt.iterations; ++it) lf << it << " " << n << " " << log[4 * it + 3] << " " << log[4 * it + 2] << "\n";
    }
    double G[256];
    CUDA_OR_DIE(cudaMemcpy(G, d_G, sizeof G, cudaMemcpyDeviceToHost));
    {
        std::ofstream pc("photoCalibResult/pcalib.txt", std::ios::trunc | std::ios::out);
        pc.precision(15);
        for (int i = 0; i < 256; ++i) pc << G[i] << " ";
        pc << "\n";
    }
    cudaFree(d_data); cudaFree(d_t); cudaFree(d_E); cudaFree(d_G);
    mdc_ctx_destroy(ctx);
    mdc_seq_close(seq);
    return 0;
}
