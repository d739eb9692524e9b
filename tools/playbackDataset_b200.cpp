// playbackDataset's save mode on the GPU: a C++ host for the sequence feed and the JPEG encoder behind include/mdc_b200.h.
//
// Same command line and the same files as the reference's playbackDataset program (main_playbackDataset.cpp:47-85): it prints the
// dataset, the rectified size and K, and the original size, omega and K; with a second argument it writes every frame, rectified and
// without photometric correction (getImage(i, true, false, false, false)), as %05d.jpg into the current directory, the bytes
// cv::imwrite writes for the float image.  The interactive viewer (:88-127) is GUI output and is not provided.
//
//   playbackDataset_b200 <dataset dir/> [anything -> save mode] [device=0] [threads=0]
//
// An argument of the form device=N or threads=N is an option; any other argument after the dataset turns save mode on.  threads is
// the number of host threads of the sequence feed (0 = its default); frames go through the GPU in chunks of min(512, max(16,
// 32 * threads)) frames: mdc_seq_prepare_device_ex (MDC_RECTIFY, MDC_OUT_U8: cv::imwrite's conversion of the float image) ->
// mdc_jpeg_encode_device (quality 95, cv::imwrite's default) -> device-to-host copies of the files into pinned buffers, while a
// writer thread writes the previous chunk's files.  A frame that cannot be read stops the program with the library's message and
// status 1 (the reference dereferences a null image there); the files of the chunks before the frame's chunk have been written.
//
// Build (see tests/test_playback_dataset_tool.py):  g++ -std=c++11 -O2 -Iinclude tools/playbackDataset_b200.cpp
//                                                   -Lmono_dataset_code_b200/lib -lmdc_b200 -L/usr/local/cuda/lib64 -lcudart -lpthread
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "mdc_b200.h"

namespace {

#define CUDA_OR_DIE(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { printf("%s: %s\n", #expr, cudaGetErrorString(e__)); exit(2); } } while (0)
#define MDC_OR_DIE(expr) do { int r__ = (expr); if (r__ != MDC_OK) { printf("%s failed (%d): %s\n", #expr, r__, mdc_last_error()); exit(2); } } while (0)

// std::cout << Eigen::Matrix3f with Eigen's default IOFormat: every coefficient printed with the stream's precision (6 significant
// digits), right-aligned to the widest one, " " between columns, rows on their own lines, no newline after the last row
void print_matrix(const float m[9]) {
    char s[9][32];
    int width = 0;
    for (int i = 0; i < 9; ++i) width = std::max(width, snprintf(s[i], sizeof s[i], "%g", m[i]));
    for (int r = 0; r < 3; ++r) {
        for (int c = 0; c < 3; ++c) printf(c ? " %*s" : "%*s", width, s[3 * r + c]);
        if (r < 2) printf("\n");
    }
}

// The files of one chunk in a pinned buffer: frame f0 + i is bytes [at[i], at[i] + size[i])
struct Chunk {
    int f0 = 0, n = 0;
    uint8_t* pinned = nullptr;
    size_t capacity = 0;
    std::vector<size_t> at, size;
};

bool write_files(const Chunk& c) {
    for (int i = 0; i < c.n; ++i) {
        char name[32];
        snprintf(name, sizeof name, "%05d.jpg", c.f0 + i);
        FILE* f = fopen(name, "wb");
        const bool ok = f && fwrite(c.pinned + c.at[static_cast<size_t>(i)], 1, c.size[static_cast<size_t>(i)], f) == c.size[static_cast<size_t>(i)];
        if (f && fclose(f) != 0) return false;
        if (!ok) { printf("cannot write %s\n", name); return false; }
    }
    return true;
}

}  // namespace

int main(int argc, char** argv) {
    if (argc < 2) { printf("usage: playbackDataset_b200 <dataset dir/> [save] [device=N] [threads=N]\n"); return 1; }
    int device = 0, threads = 0;
    bool save = false;
    for (int i = 2; i < argc; ++i) {
        if (strncmp(argv[i], "device=", 7) == 0) { device = atoi(argv[i] + 7); continue; }
        if (strncmp(argv[i], "threads=", 8) == 0) { threads = atoi(argv[i] + 8); continue; }
        save = true;
    }
    const std::string dataset = argv[1];
    printf("Playback dataset %s!\n", dataset.c_str());

    // ---- the dataset as DatasetReader opens it (BenchmarkDatasetReader.h:85-140)
    mdc_seq* seq = nullptr;
    if (mdc_seq_open(argv[1], &seq) != MDC_OK) { printf("cannot open dataset %s: %s\n", argv[1], mdc_last_error()); return 1; }
    mdc_fov* fov = nullptr;
    mdc_fov_create((dataset + "camera.txt").c_str(), &fov);
    int in_w = 0, in_h = 0, out_w = 0, out_h = 0;
    mdc_fov_dims(fov, &in_w, &in_h, &out_w, &out_h);
    mdc_photo* photo = nullptr;
    mdc_photo_create((dataset + "pcalib.txt").c_str(), (dataset + "vignette.png").c_str(), in_w, in_h, &photo);

    float k_rect[9], k_org[9];
    mdc_fov_get_K(fov, k_rect, k_org);
    printf("Rectified Images: %d x %d. K:\n", out_w, out_h);
    print_matrix(k_rect);
    printf("\n\n");
    printf("Original Images: %d x %d. omega=%f K:\n", in_w, in_h, mdc_fov_omega(fov));
    print_matrix(k_org);
    printf("\n\n");
    if (!save) return 0;

    printf("Saving undistorted Dataset to here!\n");
    fflush(stdout);
    const int n_frames = mdc_seq_num_images(seq);
    const int t = threads > 0 ? threads : static_cast<int>(std::max(1u, std::thread::hardware_concurrency()));
    const int chunk = std::min(512, std::max(16, 32 * t));
    CUDA_OR_DIE(cudaSetDevice(device));
    mdc_ctx* ctx = nullptr;
    MDC_OR_DIE(mdc_ctx_create(device, fov, photo, &ctx));
    const size_t frame_px = static_cast<size_t>(out_w) * out_h, stride = mdc_jpeg_encode_bound(out_w, out_h);
    uint8_t *d_u8 = nullptr, *d_jpeg = nullptr;
    CUDA_OR_DIE(cudaMalloc(&d_u8, frame_px * chunk));
    CUDA_OR_DIE(cudaMalloc(&d_jpeg, stride * chunk));
    Chunk bufs[2];
    std::thread writer;
    bool write_ok = true;
    auto join_writer = [&]() { if (writer.joinable()) writer.join(); };
    int status = 0;
    for (int k = 0, f0 = 0; f0 < n_frames && status == 0; ++k, f0 += chunk) {
        const int n = std::min(chunk, n_frames - f0);
        void* level0 = d_u8;
        const int rc = mdc_seq_prepare_device_ex(ctx, seq, f0, n, MDC_RECTIFY, MDC_OUT_U8, &level0, 1, threads, nullptr);
        if (rc != MDC_OK) {
            join_writer();
            printf("%s\n", mdc_last_error());
            status = 1;
            break;
        }
        Chunk& c = bufs[k & 1];                 // its previous files (chunk k - 2) were written before chunk k - 1's writer started
        c.f0 = f0;
        c.n = n;
        c.at.resize(static_cast<size_t>(n));
        c.size.resize(static_cast<size_t>(n));
        MDC_OR_DIE(mdc_jpeg_encode_device(ctx, d_u8, out_w, n, out_w, out_h, 95, d_jpeg, stride, c.size.data(), nullptr));
        size_t total = 0;
        for (int i = 0; i < n; ++i) { c.at[static_cast<size_t>(i)] = total; total += c.size[static_cast<size_t>(i)]; }
        if (c.capacity < total) {
            if (c.pinned) CUDA_OR_DIE(cudaFreeHost(c.pinned));
            c.capacity = total + total / 4;
            CUDA_OR_DIE(cudaMallocHost(&c.pinned, c.capacity));
        }
        for (int i = 0; i < n; ++i)
            CUDA_OR_DIE(cudaMemcpyAsync(c.pinned + c.at[static_cast<size_t>(i)], d_jpeg + stride * i, c.size[static_cast<size_t>(i)], cudaMemcpyDeviceToHost, 0));
        CUDA_OR_DIE(cudaStreamSynchronize(0));
        join_writer();
        if (!write_ok) { status = 1; break; }
        writer = std::thread([&c, &write_ok]() { if (!write_files(c)) write_ok = false; });
    }
    join_writer();
    if (!write_ok) status = 1;
    for (Chunk& c : bufs)
        if (c.pinned) cudaFreeHost(c.pinned);
    cudaFree(d_u8);
    cudaFree(d_jpeg);
    mdc_ctx_destroy(ctx);
    mdc_photo_destroy(photo);
    mdc_fov_destroy(fov);
    mdc_seq_close(seq);
    return status;
}
