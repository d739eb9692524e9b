// vignetteCalib on the GPU: a C++ host for the front end and the optimiser behind include/mdc_b200.h.
//
// Same command line, inputs and result files as the reference's vignetteCalib program (main_vignetteCalib.cpp:132-180 arguments,
// :222-227 mean exposure, :230-372 front end, :395-585 optimisation loop, :531 log.txt rows, :72-93 plane.png, :570-582
// vignette.png / vignetteSmoothed.png), with every pass over the images and plane grids running in the sm_90a kernels of
// libmdc_b200.so: gamma removal (mdc_unmap_u8), exposure normalisation and gradient invalidation (mdc_vc_prepare_images),
// projection + distortion + visibility mask of the plane grid (mdc_vc_plane_maps), and the loop (mdc_vignette_calib).
//
// The homographies from the unit square to the marker (:231-262) come from one of two places:
//   homographies=detect  the tool detects the marker itself: every skip-th frame decoded once into device memory
//                        (mdc_seq_read_gray8_device) -> rectification (mdc_prepare_batch_pitched, MDC_RECTIFY) -> 8-bit
//                        frame and adaptive threshold (mdc_marker_threshold) on the GPU, in chunks of frames; then aruco's
//                        detector (mdc_marker_detect) on host threads, one frame per thread, and mdc_marker_homography.  The rows
//                        it used are written to vignetteCalibResult/homographies.txt, in the format homographies=FILE reads.
//   homographies=FILE    nine whitespace-separated numbers (the row-major 3x3 homography from marker corners to rectified pixels)
//                        per considered frame i = 0, skip, 2*skip, ...
// The frames that have a homography are decoded in one mdc_seq_read_gray8_device call (JPEG frames on the GPU), or, after detection,
// gathered from the frames it decoded.
// A row containing NaN means that the frame does not show exactly one marker: the frame is left out (:240), but its exposure
// still counts in the mean exposure, as in the reference.  The debug overlays and imshow windows (:306-368) are not produced.
//
//   vignetteCalib_b200 <dataset dir/> homographies=FILE|detect [iterations=20] [skip=1] [patternX=1000] [patternY=1000] [facW=5]
//                      [facH=5] [device=0]
//
// Build (see tests/test_vignette_calib_tool.py):  g++ -std=c++11 -O2 -Iinclude tools/vignetteCalib_b200.cpp
//                                                 -Lmono_dataset_code_b200/lib -lmdc_b200 -L/usr/local/cuda/lib64 -lcudart
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <string>
#include <thread>
#include <vector>

#include "mdc_b200.h"

namespace {

struct Options {
    int iterations = 20, skip = 1, gw = 1000, gh = 1000, device = 0;
    float facw = 5, fach = 5;
    std::string homographies;
};

void parse_option(const char* arg, Options* o) {
    int v;
    float f;
    if (strncmp(arg, "homographies=", 13) == 0) { o->homographies = arg + 13; return; }
    if (sscanf(arg, "iterations=%d", &v) == 1) { o->iterations = v; printf("nits set to %d!\n", v); return; }
    if (sscanf(arg, "skip=%d", &v) == 1) { o->skip = v; printf("skipFrames set to %d!\n", v); return; }
    if (sscanf(arg, "patternX=%d", &v) == 1) { o->gw = v; printf("patternX set to %d!\n", v); return; }
    if (sscanf(arg, "patternY=%d", &v) == 1) { o->gh = v; printf("patternY set to %d!\n", v); return; }
    if (sscanf(arg, "facW=%f", &f) == 1) { o->facw = f; printf("facw set to %f!\n", f); return; }
    if (sscanf(arg, "facH=%f", &f) == 1) { o->fach = f; printf("fach set to %f!\n", f); return; }
    if (sscanf(arg, "device=%d", &v) == 1) { o->device = v; return; }
    printf("could not parse argument \"%s\"!!\n", arg);
}

#define CUDA_OR_DIE(expr) do { cudaError_t e__ = (expr); if (e__ != cudaSuccess) { printf("%s: %s\n", #expr, cudaGetErrorString(e__)); exit(2); } } while (0)
#define MDC_OR_DIE(expr) do { int r__ = (expr); if (r__ != MDC_OK) { printf("%s failed (%d): %s\n", #expr, r__, mdc_last_error()); exit(2); } } while (0)

// cv::Mat(CV_32F) * 254.9 * 254.9 -> convertTo(CV_16U) (:570-581): two float products, then round to nearest even and saturate
// (NaN -> 0)
bool write_vignette_png(const std::string& path, const std::vector<float>& v, int w, int h) {
    std::vector<uint16_t> px(v.size());
    for (size_t i = 0; i < v.size(); ++i) {
        float a = static_cast<float>(v[i] * 254.9);
        a = static_cast<float>(a * 254.9);
        const double r = nearbyint(static_cast<double>(a));
        const unsigned u = r > 65535 ? 65535u : (r > 0 ? static_cast<unsigned>(r) : 0u);
        px[i] = static_cast<uint16_t>(u);
    }
    return mdc_png_write(path.c_str(), px.data(), w, h, 2 * static_cast<size_t>(w), 16, 1) == MDC_OK;
}

// displayImage (:72-93): grey 255*(I-vmin)/(vmax-vmin) truncated to 8 bits; NaN is BGR (0,0,255), i.e. red
bool write_plane_png(const std::string& path, const std::vector<float>& I, int w, int h) {
    float vmin = 1e10, vmax = -1e10;
    for (float v : I) {
        if (vmin > v) vmin = v;
        if (vmax < v) vmax = v;
    }
    printf("plane image values %f - %f!\n", vmin, vmax);
    std::vector<uint8_t> px(I.size() * 3);
    for (size_t i = 0; i < I.size(); ++i) {
        uint8_t* p = &px[3 * i];
        if (std::isnan(I[i])) { p[0] = 0; p[1] = 0; p[2] = 255; continue; }
        const float c = 255 * (I[i] - vmin) / (vmax - vmin);
        p[0] = p[1] = p[2] = c >= 0 && c < 256 ? static_cast<uint8_t>(c) : (c >= 256 ? 255 : 0);
    }
    return mdc_png_write(path.c_str(), px.data(), w, h, 3 * static_cast<size_t>(w), 8, 3) == MDC_OK;
}

// Every skip-th frame (ids) decoded into the device stack d_stack [ids][hI][pitch] in one call; exits at the first one that cannot be
// read as a wI x hI image, with the reader's message.
void read_frames(mdc_ctx* ctx, mdc_seq* seq, const std::vector<int>& ids, int wI, int hI, uint8_t* d_stack, size_t pitch) {
    std::vector<int> status(ids.size());
    const int r = mdc_seq_read_gray8_device(ctx, seq, ids.data(), static_cast<int>(ids.size()), wI, hI, d_stack, pitch, status.data(), nullptr, 0, nullptr);
    if (r != MDC_OK && r != MDC_ERR_FORMAT) { printf("mdc_seq_read_gray8_device failed (%d): %s\n", r, mdc_last_error()); exit(2); }
    for (size_t k = 0; k < ids.size(); ++k)
        if (status[k] != MDC_OK) {
            printf("frame %d: cannot read a %dx%d image: %s\n", ids[k], wI, hI, mdc_last_error());       // the first failed frame's message
            exit(1);
        }
}

// Homographies of frames i = 0, skip, ... by marker detection; writes them (NaN rows for frames without exactly one marker) to `out`.
// The frames are decoded once into *d_stack ([ids][hI][pitch], rows padded to 16 bytes so that the rectification keeps its TMA loader),
// which the caller gathers the frames with a marker from.
void detect_homographies(mdc_ctx* ctx, mdc_seq* seq, int skip, int wI, int hI, int w_out, int h_out, const char* out, uint8_t** d_stack, size_t* pitch) {
    const int num_images = mdc_seq_num_images(seq);
    std::vector<int> ids;
    for (int i = 0; i < num_images; i += skip) ids.push_back(i);
    *pitch = (static_cast<size_t>(wI) + 15) / 16 * 16;
    const size_t frame_bytes = *pitch * hI;
    CUDA_OR_DIE(cudaMalloc(d_stack, std::max<size_t>(1, frame_bytes * ids.size())));
    read_frames(ctx, seq, ids, wI, hI, *d_stack, *pitch);
    const size_t npx_in = static_cast<size_t>(wI) * hI, npx = static_cast<size_t>(w_out) * h_out;
    const int chunk = static_cast<int>(std::max<size_t>(1, std::min<size_t>(32, (size_t(1) << 30) / (npx * 4 + npx_in))));
    std::vector<uint8_t> grey(chunk * npx), mask(chunk * npx);
    uint8_t *d_grey = nullptr, *d_mask = nullptr;
    float* d_rect = nullptr;
    CUDA_OR_DIE(cudaMalloc(&d_rect, chunk * npx * sizeof(float)));
    CUDA_OR_DIE(cudaMalloc(&d_grey, grey.size()));
    CUDA_OR_DIE(cudaMalloc(&d_mask, mask.size()));
    std::vector<double> Hs(ids.size() * 9, NAN);
    const int threads = std::max(1u, std::thread::hardware_concurrency());
    int found = 0;
    for (size_t first = 0; first < ids.size(); first += chunk) {
        const int m = static_cast<int>(std::min<size_t>(chunk, ids.size() - first));
        MDC_OR_DIE(mdc_prepare_batch_pitched(ctx, *d_stack + first * frame_bytes, *pitch, m, MDC_RECTIFY, &d_rect, 1, nullptr));   // getImage(i, true, false, false, false)
        MDC_OR_DIE(mdc_marker_threshold(ctx, d_rect, m, w_out, h_out, d_grey, d_mask, nullptr));
        CUDA_OR_DIE(cudaMemcpy(grey.data(), d_grey, m * npx, cudaMemcpyDeviceToHost));
        CUDA_OR_DIE(cudaMemcpy(mask.data(), d_mask, m * npx, cudaMemcpyDeviceToHost));
        std::vector<int> status(m, MDC_OK);
        std::vector<std::string> errors(m);
        std::vector<std::thread> pool;
        for (int t = 0; t < std::min(threads, m); ++t)
            pool.emplace_back([&, t]() {
                for (int k = t; k < m; k += threads) {
                    mdc_marker markers[2];
                    int count = 0;
                    status[k] = mdc_marker_detect(grey.data() + k * npx, mask.data() + k * npx, w_out, h_out, markers, 2, &count);
                    if (status[k] == MDC_ERR_INVALID_ARG && count > 2) status[k] = MDC_OK;    // more than one marker: skipped (:240)
                    if (status[k] != MDC_OK) { errors[k] = mdc_last_error(); continue; }
                    if (count == 1 && mdc_marker_homography(markers[0].corners, &Hs[(first + k) * 9]) != MDC_OK)
                        for (int q = 0; q < 9; ++q) Hs[(first + k) * 9 + q] = NAN;
                }
            });
        for (std::thread& t : pool) t.join();
        for (int k = 0; k < m; ++k) {
            if (status[k] != MDC_OK) { printf("frame %d: marker detection failed: %s\n", ids[first + k], errors[k].c_str()); exit(2); }
            found += !std::isnan(Hs[(first + k) * 9]);
        }
    }
    cudaFree(d_rect); cudaFree(d_grey); cudaFree(d_mask);
    printf("found exactly one marker in %d of %zu frames\n", found, ids.size());
    FILE* f = fopen(out, "w");
    if (!f) { printf("cannot write %s\n", out); exit(1); }
    for (size_t r = 0; r < ids.size(); ++r)
        for (int q = 0; q < 9; ++q) fprintf(f, "%.17g%c", Hs[r * 9 + q], q == 8 ? '\n' : ' ');
    if (fclose(f) != 0) { printf("cannot write %s\n", out); exit(1); }
}

}  // namespace

int main(int argc, char** argv) {
    if (argc < 2) {
        printf("usage: vignetteCalib_b200 <dataset dir/> homographies=FILE|detect [iterations=N] [skip=N] [patternX=N] [patternY=N] [facW=F] [facH=F] "
               "[device=N]\n");
        return 1;
    }
    Options opt;
    for (int i = 2; i < argc; ++i) parse_option(argv[i], &opt);
    if (opt.skip < 1) opt.skip = 1;
    if (opt.homographies.empty()) { printf("homographies=FILE is required (or homographies=detect)\n"); return 1; }
    if (opt.gw < 1 || opt.gh < 1) { printf("patternX / patternY must be positive\n"); return 1; }

    if (system("rm -rf vignetteCalibResult") == -1) printf("could not delete old vignetteCalibResult folder!\n");
    if (system("mkdir vignetteCalibResult") == -1) printf("could not create vignetteCalibResult folder!\n");

    // ---- the dataset as DatasetReader opens it: frames + times.txt, camera.txt, pcalib.txt + vignette.png
    const std::string path = argv[1];
    printf("SEQUENCE NAME: %s!\n", argv[1]);
    mdc_seq* seq = nullptr;
    if (mdc_seq_open(argv[1], &seq) != MDC_OK) { printf("cannot open dataset %s: %s\n", argv[1], mdc_last_error()); return 1; }
    mdc_fov* fov = nullptr;
    if (mdc_fov_create((path + "camera.txt").c_str(), &fov) != MDC_OK) { printf("invalid camera.txt: %s\n", mdc_last_error()); return 1; }
    int wI = 0, hI = 0, w_out = 0, h_out = 0;
    mdc_fov_dims(fov, &wI, &hI, &w_out, &h_out);
    mdc_photo* photo = nullptr;
    mdc_photo_create((path + "pcalib.txt").c_str(), (path + "vignette.png").c_str(), wI, hI, &photo);      // only the response is used
    const int num_images = mdc_seq_num_images(seq);

    // :222-227: the sum runs over every skip-th frame but is divided by the number of ALL frames
    float mean_exposure = 0;
    for (int i = 0; i < num_images; i += opt.skip) mean_exposure += mdc_seq_exposure(seq, i);
    mean_exposure = mean_exposure / num_images;
    if (mean_exposure == 0) mean_exposure = 1;

    CUDA_OR_DIE(cudaSetDevice(opt.device));
    mdc_ctx* ctx = nullptr;
    MDC_OR_DIE(mdc_ctx_create(opt.device, fov, photo, &ctx));
    uint8_t* d_stack = nullptr;            // homographies=detect: every skip-th frame, decoded for the detection
    size_t stack_pitch = 0;
    if (opt.homographies == "detect") {
        opt.homographies = "vignetteCalibResult/homographies.txt";
        detect_homographies(ctx, seq, opt.skip, wI, hI, w_out, h_out, opt.homographies.c_str(), &d_stack, &stack_pitch);
    }

    // ---- frames that have a homography, as [n][wI*hI] on the device: gathered from the detection's stack, or decoded in one call
    FILE* hf = fopen(opt.homographies.c_str(), "r");
    if (!hf) { printf("cannot open %s\n", opt.homographies.c_str()); return 1; }
    const size_t npx = static_cast<size_t>(wI) * hI;
    std::vector<int> ids;
    std::vector<float> exposures;
    std::vector<double> Hs;
    int missing = -1;                      // first frame without a row: reported after the frames before it have been read
    for (int i = 0; i < num_images; i += opt.skip) {
        double H[9];
        bool complete = true;
        for (int k = 0; k < 9 && complete; ++k) complete = fscanf(hf, "%lf", &H[k]) == 1;
        if (!complete) { missing = i; break; }
        bool found = true;
        for (double v : H) found = found && !std::isnan(v);
        if (!found) continue;                                   // no marker in this frame (:240)
        ids.push_back(i);
        exposures.push_back(mdc_seq_exposure(seq, i));
        Hs.insert(Hs.end(), H, H + 9);
    }
    fclose(hf);
    uint8_t* d_frames = nullptr;
    if (!ids.empty()) {
        CUDA_OR_DIE(cudaMalloc(&d_frames, npx * ids.size()));
        if (!d_stack) {
            read_frames(ctx, seq, ids, wI, hI, d_frames, wI);
        } else {
            for (size_t k = 0; k < ids.size(); ++k)
                CUDA_OR_DIE(cudaMemcpy2D(d_frames + k * npx, wI, d_stack + static_cast<size_t>(ids[k] / opt.skip) * stack_pitch * hI, stack_pitch, wI, hI,
                                         cudaMemcpyDeviceToDevice));
        }
    }
    cudaFree(d_stack);
    if (missing >= 0) { printf("%s: no homography for frame %d\n", opt.homographies.c_str(), missing); return 1; }
    const int n = static_cast<int>(exposures.size());
    printf("loaded %d images with a marker\n", n);
    const size_t gwgh = static_cast<size_t>(opt.gw) * opt.gh;

    // ---- front end on the device: gamma removal, normalisation + gradient invalidation, plane-to-image maps
    float *d_images = nullptr, *d_p2x = nullptr, *d_p2y = nullptr, *d_plane = nullptr, *d_vig = nullptr, *d_smoothed = nullptr;
    CUDA_OR_DIE(cudaMalloc(&d_images, npx * n * sizeof(float) + 4));
    CUDA_OR_DIE(cudaMalloc(&d_p2x, gwgh * n * sizeof(float) + 4));
    CUDA_OR_DIE(cudaMalloc(&d_p2y, gwgh * n * sizeof(float) + 4));
    CUDA_OR_DIE(cudaMalloc(&d_plane, gwgh * sizeof(float)));
    CUDA_OR_DIE(cudaMalloc(&d_vig, npx * sizeof(float)));
    CUDA_OR_DIE(cudaMalloc(&d_smoothed, npx * sizeof(float)));
    if (n > 0) {
        MDC_OR_DIE(mdc_unmap_u8(ctx, d_frames, d_images, static_cast<int>(npx), n, MDC_REMOVE_GAMMA, nullptr));      // getImage(i,false,true,false,false)
        CUDA_OR_DIE(cudaFree(d_frames));
        MDC_OR_DIE(mdc_vc_prepare_images(ctx, d_images, n, wI, hI, exposures.data(), mean_exposure, 255, d_images, nullptr));
        MDC_OR_DIE(mdc_vc_plane_maps(fov, Hs.data(), n, opt.gw, opt.gh, opt.facw, opt.fach, d_p2x, d_p2y, opt.device, nullptr));
    }

    // ---- the optimisation loop: plane colour starts at 0 (the reference reads it uninitialised), vignette at 1 (:391)
    CUDA_OR_DIE(cudaMemset(d_plane, 0, gwgh * sizeof(float)));
    {
        std::vector<float> ones(npx, 1.0f);
        CUDA_OR_DIE(cudaMemcpy(d_vig, ones.data(), npx * sizeof(float), cudaMemcpyHostToDevice));
    }
    std::vector<double> log(static_cast<size_t>(4) * (opt.iterations > 0 ? opt.iterations : 1), 0.0);
    MDC_OR_DIE(mdc_vignette_calib(ctx, d_images, d_p2x, d_p2y, n, opt.gw, opt.gh, wI, hI, opt.iterations, 15, 1, d_plane, d_vig, d_smoothed,
                                  log.data()));

    {
        std::ofstream lf("vignetteCalibResult/log.txt", std::ios::trunc | std::ios::out);
        lf.precision(15);
        for (int it = 0; it < opt.iterations; ++it)
            lf << it << " " << n << " " << log[4 * it + 3] << " " << sqrtf(static_cast<float>(log[4 * it + 2] / log[4 * it + 3])) << "\n";
    }
    int rc = 0;
    if (opt.iterations > 0) {
        std::vector<float> vig(npx), smoothed(npx), plane(gwgh);
        CUDA_OR_DIE(cudaMemcpy(vig.data(), d_vig, npx * sizeof(float), cudaMemcpyDeviceToHost));
        CUDA_OR_DIE(cudaMemcpy(smoothed.data(), d_smoothed, npx * sizeof(float), cudaMemcpyDeviceToHost));
        CUDA_OR_DIE(cudaMemcpy(plane.data(), d_plane, gwgh * sizeof(float), cudaMemcpyDeviceToHost));
        if (!write_plane_png("vignetteCalibResult/plane.png", plane, opt.gw, opt.gh) ||
            !write_vignette_png("vignetteCalibResult/vignetteSmoothed.png", smoothed, wI, hI) ||
            !write_vignette_png("vignetteCalibResult/vignette.png", vig, wI, hI)) {
            printf("could not write the result images\n");
            rc = 1;
        }
    }
    cudaFree(d_images); cudaFree(d_p2x); cudaFree(d_p2y); cudaFree(d_plane); cudaFree(d_vig); cudaFree(d_smoothed);
    mdc_ctx_destroy(ctx);
    mdc_photo_destroy(photo);
    mdc_fov_destroy(fov);
    mdc_seq_close(seq);
    return rc;
}
