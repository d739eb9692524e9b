// responseCalib on the GPU: a C++ host for the calibrator kernels behind include/mdc_b200.h.
//
// Same command line, inputs and result files as the reference's responseCalib program
// (main_responseCalib.cpp:149-173 arguments, :191-237 loading + saturation leak padding, :249-259 starting irradiance, :281-362
// optimisation loop, :359 log.txt rows, :367-375 pcalib.txt), with every pass over the image stack — padding, E-init, G-step,
// E-step, rescale, rmse — running in the sm_90a kernels of libmdc_b200.so.
// The result images are written as the reference writes them (:72-146, :273, :309-310, :344-345): E-0.png / E-016.png after E-init,
// G-k.png after each G-step and E-k.png / E-k16.png after each E-step, with the "Irradiance" and "Inv. Response" lines printed where
// the reference prints them.  The kernels of mdc_rc_plot_e / mdc_rc_plot_g make the pixels; each step's plots are copied to pinned
// host memory and compressed to PNG (mdc_png_write) on writer threads while the loop goes on.  plots=0 skips them; pcalib.txt and
// log.txt are the same either way.  The imshow windows are not produced.
//
//   responseCalib_b200 <dataset dir/> [leakPadding=2] [iterations=10] [skip=1] [device=0] [plots=1]
//
// Build (see tests/test_tools_cpp.py):  g++ -std=c++11 -O2 -Iinclude tools/responseCalib_b200.cpp -Lmono_dataset_code_b200/lib
//                                       -lmdc_b200 -L/usr/local/cuda/lib64 -lcudart -o responseCalib_b200
#include <cuda_runtime.h>

#include <algorithm>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <fstream>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "mdc_b200.h"

namespace {

struct Options { int leak_padding = 2, iterations = 10, skip = 1, device = 0, plots = 1; };

void parse_option(const char* arg, Options* o) {
    int v;
    if (sscanf(arg, "leakPadding=%d", &v) == 1) { o->leak_padding = v; printf("leakPadding set to %d!\n", v); return; }
    if (sscanf(arg, "iterations=%d", &v) == 1) { o->iterations = v; printf("nits set to %d!\n", v); return; }
    if (sscanf(arg, "skip=%d", &v) == 1) { o->skip = v; printf("skipFrames set to %d!\n", v); return; }
    if (sscanf(arg, "device=%d", &v) == 1) { o->device = v; return; }
    if (sscanf(arg, "plots=%d", &v) == 1) { o->plots = v; return; }
    printf("could not parse argument \"%s\"!!\n", arg);
}

#define CUDA_OR_DIE(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { printf("%s: %s\n", #expr, cudaGetErrorString(e__)); exit(2); } } while (0)
#define MDC_OR_DIE(expr) do { int r__ = (expr); if (r__ != MDC_OK) { printf("%s failed (%d): %s\n", #expr, r__, mdc_last_error()); exit(2); } } while (0)

// PNG files written by host threads from pinned slots: the loop takes a free slot (waiting while all are queued or being written),
// fills it, and hands it over with the files it holds.
class PlotWriter {
public:
    struct File { std::string path; size_t offset; int w, h, depth, channels; };

    PlotWriter(size_t slot_bytes, int threads) {
        for (int i = 0; i < 2 * threads; ++i) {
            void* p = nullptr;
            CUDA_OR_DIE(cudaHostAlloc(&p, slot_bytes, cudaHostAllocDefault));
            slots_.push_back(static_cast<uint8_t*>(p));
            free_.push_back(static_cast<uint8_t*>(p));
        }
        for (int i = 0; i < threads; ++i) threads_.emplace_back(&PlotWriter::run, this);
    }
    ~PlotWriter() {
        finish();
        for (uint8_t* p : slots_) cudaFreeHost(p);
    }
    uint8_t* acquire() {
        std::unique_lock<std::mutex> lock(m_);
        cv_.wait(lock, [this] { return !free_.empty(); });
        uint8_t* p = free_.back();
        free_.pop_back();
        return p;
    }
    void submit(uint8_t* slot, const std::vector<File>& files) {
        std::lock_guard<std::mutex> lock(m_);
        jobs_.push_back(Job{slot, files});
        cv_.notify_all();
    }
    // waits for every queued file, stops the threads; false if a file could not be written
    bool finish() {
        {
            std::lock_guard<std::mutex> lock(m_);
            stop_ = true;
            cv_.notify_all();
        }
        for (std::thread& t : threads_) t.join();
        threads_.clear();
        return ok_;
    }

private:
    struct Job { uint8_t* slot; std::vector<File> files; };
    void run() {
        for (;;) {
            Job job;
            {
                std::unique_lock<std::mutex> lock(m_);
                cv_.wait(lock, [this] { return stop_ || !jobs_.empty(); });
                if (jobs_.empty()) return;
                job = jobs_.front();
                jobs_.pop_front();
            }
            bool ok = true;
            for (const File& f : job.files) {
                const size_t row = static_cast<size_t>(f.w) * f.channels * (f.depth / 8);
                if (mdc_png_write(f.path.c_str(), job.slot + f.offset, f.w, f.h, row, f.depth, f.channels) != MDC_OK) {
                    printf("could not write %s: %s\n", f.path.c_str(), mdc_last_error());
                    ok = false;
                }
            }
            std::lock_guard<std::mutex> lock(m_);
            if (!ok) ok_ = false;
            free_.push_back(job.slot);
            cv_.notify_all();
        }
    }
    std::mutex m_;
    std::condition_variable cv_;
    std::vector<uint8_t*> slots_, free_;
    std::deque<Job> jobs_;
    std::vector<std::thread> threads_;
    bool stop_ = false, ok_ = true;
};

// plotE / plotG of one step of the loop (mdc_response_calib_ex's hook): the kernels make the images, the writer compresses them
struct Plots {
    mdc_ctx* ctx;
    int w, h;
    double* d_range;
    uint8_t *d_bgr, *d_g;
    uint16_t* d_e16;
    PlotWriter* writer;
};

void plot_step(int iteration, int which, const double* d_E, const double* d_G, void* user) {
    Plots* p = static_cast<Plots*>(user);
    const size_t npix = static_cast<size_t>(p->w) * p->h;
    uint8_t* slot = p->writer->acquire();
    char base[64];
    if (which == MDC_RC_STEP_E) {
        double range[4];
        MDC_OR_DIE(mdc_rc_plot_e(p->ctx, d_E, static_cast<int>(npix), p->d_range, p->d_bgr, p->d_e16, nullptr));
        CUDA_OR_DIE(cudaMemcpy(slot, p->d_bgr, 3 * npix, cudaMemcpyDeviceToHost));
        CUDA_OR_DIE(cudaMemcpy(slot + 3 * npix, p->d_e16, 2 * npix, cudaMemcpyDeviceToHost));
        CUDA_OR_DIE(cudaMemcpy(range, p->d_range, sizeof range, cudaMemcpyDeviceToHost));
        printf("Irradiance %f - %f\n", range[2], range[3]);
        snprintf(base, sizeof base, "photoCalibResult/E-%d", iteration);
        p->writer->submit(slot, {{std::string(base) + ".png", 0, p->w, p->h, 8, 3}, {std::string(base) + "16.png", 3 * npix, p->w, p->h, 16, 1}});
    } else {
        double minmax[2];
        MDC_OR_DIE(mdc_rc_plot_g(p->ctx, d_G, p->d_g, minmax, nullptr));
        CUDA_OR_DIE(cudaMemcpy(slot, p->d_g, 256 * 256, cudaMemcpyDeviceToHost));
        printf("Inv. Response %f - %f\n", minmax[0], minmax[1]);
        snprintf(base, sizeof base, "photoCalibResult/G-%d.png", iteration);
        p->writer->submit(slot, {{base, 0, 256, 256, 8, 1}});
    }
}

}  // namespace

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: responseCalib_b200 <dataset dir/> [leakPadding=N] [iterations=N] [skip=N] [device=N] [plots=0|1]\n"); return 1; }
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

    // ---- the optimisation loop (prints the per-iteration rmse lines itself; the hook plots)
    std::vector<double> log(static_cast<size_t>(4) * (opt.iterations > 0 ? opt.iterations : 1), 0.0);
    Plots plots = {ctx, w, h, nullptr, nullptr, nullptr, nullptr, nullptr};
    PlotWriter* writer = nullptr;
    if (opt.plots) {
        CUDA_OR_DIE(cudaMalloc(&plots.d_range, 4 * sizeof(double)));
        CUDA_OR_DIE(cudaMalloc(&plots.d_bgr, 3 * static_cast<size_t>(npix)));
        CUDA_OR_DIE(cudaMalloc(&plots.d_e16, 2 * static_cast<size_t>(npix)));
        CUDA_OR_DIE(cudaMalloc(&plots.d_g, 256 * 256));
        const int threads = static_cast<int>(std::max(1u, std::min(4u, std::thread::hardware_concurrency())));
        writer = plots.writer = new PlotWriter(std::max<size_t>(5 * static_cast<size_t>(npix), 256 * 256), threads);
    }
    MDC_OR_DIE(mdc_response_calib_ex(ctx, d_data, n, npix, d_t, opt.iterations, d_E, d_G, log.data(), opt.plots ? plot_step : nullptr, &plots));
    const bool plots_written = writer ? writer->finish() : true;
    delete writer;

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
    cudaFree(plots.d_range); cudaFree(plots.d_bgr); cudaFree(plots.d_e16); cudaFree(plots.d_g);
    mdc_ctx_destroy(ctx);
    mdc_seq_close(seq);
    return plots_written ? 0 : 2;
}
