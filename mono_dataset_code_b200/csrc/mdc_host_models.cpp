// Host-side calibration models: parsing of camera.txt / pcalib.txt / vignette image and
// construction of the four lookup tables (remapX, remapY, GInv, vignetteMapInv).
//
// This is init-time code (tens of milliseconds once per sequence), deliberately kept on the
// CPU: the tables must be BIT-IDENTICAL to the reference's, and they depend on glibc's
// atanf/tan/sqrtf and on the exact float/double promotion pattern of the reference's
// expressions (SURVEY.md §3.4, §7 "bit-exact tables are toolchain-sensitive").  CUDA's own
// atanf is not glibc's (the device-side distortCoordinates uses the restatement in mdc_atanf.h,
// which is).  Compile with -ffp-contract=off and no -ffast-math/-march.
//
// Behaviour mirrored (file:line in /root/reference/src):
//   camera.txt parsing and validity rules ......... FOVUndistorter.cpp:55-126
//   output-camera selection (omega==0/crop/full/K)  FOVUndistorter.cpp:131-218
//   distortCoordinates ............................ FOVUndistorter.cpp:280-319
//   remap table + clamping + black marking ........ FOVUndistorter.cpp:224-251
//   Krect / Korg .................................. FOVUndistorter.cpp:257-268
//   pcalib.txt parsing, GInv normalisation, G ..... PhotometricUndistorter.cpp:56-110
//   vignette normalisation and reciprocal ......... PhotometricUndistorter.cpp:119-156
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>

#include "mdc_atanf.h"
#include "mdc_internal.h"

// ------------------------------------------------------------------------- error slot
static thread_local char g_err[512] = "";
void mdc_set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof g_err, fmt, ap);
    va_end(ap);
}
extern "C" const char* mdc_last_error(void) { return g_err; }
extern "C" const char* mdc_version(void) { return "mdc_b200 0.1 (sm_90a)"; }

// ------------------------------------------------------------------ FOV model helpers
namespace {

// The reference calls unqualified tan()/sqrt() on float arguments; depending on the
// headers in scope these are the double functions (result narrowed on assignment) or the
// float overloads.  Both behaviours are kept, selected by float_math.
struct MathSel {
    int fm;
    // 2.0f * tan(dist / 2.0f)
    float d2t(float dist) const {
        if (fm) return 2.0f * tanf(dist / 2.0f);
        double t = tan(static_cast<double>(dist / 2.0f));
        return static_cast<float>(2.0 * t);
    }
    // tan(radius * dist) / d2t
    float trans(float radius, float dist, float d2t_) const {
        float arg = radius * dist;
        if (fm) return tanf(arg) / d2t_;
        return static_cast<float>(tan(static_cast<double>(arg)) / static_cast<double>(d2t_));
    }
    float root(float v) const { return fm ? sqrtf(v) : static_cast<float>(sqrt(static_cast<double>(v))); }
};

inline float pick_max(float a, float b) { return (a < b) ? b : a; }

// value - 0.5 with a DOUBLE literal, narrowed to float (FOVUndistorter.cpp:137-138 etc.)
inline float minus_half_d(float v) { return static_cast<float>(static_cast<double>(v) - 0.5); }

struct Intrinsics { float fx, fy, cx, cy; };

Intrinsics input_intrinsics(const mdc_fov* f) {
    Intrinsics k;
    k.fx = f->in_calib[0] * f->in_w;
    k.fy = f->in_calib[1] * f->in_h;
    k.cx = minus_half_d(f->in_calib[2] * f->in_w);
    k.cy = minus_half_d(f->in_calib[3] * f->in_h);
    return k;
}

}  // namespace

// the ten per-calibration constants of distortCoordinates, evaluated exactly like the reference does (FOVUndistorter.cpp:286-301)
void mdc_fov_distort_constants(const mdc_fov* f, mdc_distort_constants* k) {
    const MathSel m{f->float_math};
    k->omega = f->in_calib[4];
    k->d2t = m.d2t(k->omega);
    const Intrinsics in = input_intrinsics(f);
    k->fx = in.fx; k->fy = in.fy; k->cx = in.cx; k->cy = in.cy;
    // note: here the reference subtracts a FLOAT 0.5f (FOVUndistorter.cpp:300-301)
    k->ofx = f->out_calib[0] * f->out_w;
    k->ofy = f->out_calib[1] * f->out_h;
    k->ocx = f->out_calib[2] * f->out_w - 0.5f;
    k->ocy = f->out_calib[3] * f->out_h - 0.5f;
}

void mdc_fov_distort(const mdc_fov* f, float* xs, float* ys, int n) {
    mdc_distort_constants k;
    mdc_fov_distort_constants(f, &k);
    for (int i = 0; i < n; ++i) {
        float nx = (xs[i] - k.ocx) / k.ofx;
        float ny = (ys[i] - k.ocy) / k.ofy;
        float rad = sqrtf(nx * nx + ny * ny);
        float scale = 1;
        if (!(rad == 0 || k.omega == 0)) scale = atanf(rad * k.d2t) / (k.omega * rad);
        xs[i] = k.fx * scale * nx + k.cx;
        ys[i] = k.fy * scale * ny + k.cy;
    }
}

// HK = H * K_p2idx^-1 of main_vignetteCalib.cpp:195-200, :254-271, in float with the arithmetic of the stand-in Eigen the runnable
// reference program is built against (oracle/shim/Eigen/Core): inverse by adjugate / determinant, product summed left to right.
// Real Eigen may order the inverse differently and differ in the last bit.
void mdc_vc_plane_matrix(const double H[9], int gw, int gh, float facw, float fach, float HK[9]) {
    float K[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, Ki[9], Hf[9];
    K[0] = gw / facw; K[4] = gh / fach; K[2] = gw / 2; K[5] = gh / 2; K[8] = 1;      // gw / 2 is an int division
    const float c00 = K[4] * K[8] - K[5] * K[7], c01 = K[5] * K[6] - K[3] * K[8], c02 = K[3] * K[7] - K[4] * K[6];
    const float det = K[0] * c00 + K[1] * c01 + K[2] * c02;
    Ki[0] = c00 / det; Ki[3] = c01 / det; Ki[6] = c02 / det;
    Ki[1] = (K[2] * K[7] - K[1] * K[8]) / det;
    Ki[4] = (K[0] * K[8] - K[2] * K[6]) / det;
    Ki[7] = (K[1] * K[6] - K[0] * K[7]) / det;
    Ki[2] = (K[1] * K[5] - K[2] * K[4]) / det;
    Ki[5] = (K[2] * K[3] - K[0] * K[5]) / det;
    Ki[8] = (K[0] * K[4] - K[1] * K[3]) / det;
    for (int i = 0; i < 9; ++i) Hf[i] = static_cast<float>(H[i]);          // Eigen::Matrix3f H from the double cv::Mat, :255-263
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) HK[r * 3 + c] = Hf[r * 3] * Ki[c] + Hf[r * 3 + 1] * Ki[3 + c] + Hf[r * 3 + 2] * Ki[6 + c];
}

// the restated atanf (mdc_atanf.h) evaluated on the host, so that it can be compared with the platform's libm without a GPU
extern "C" void mdc_atanf_host(const float* in, float* out, size_t n) {
    for (size_t i = 0; i < n; ++i) out[i] = mdc_atanf(in[i]);
}

void mdc_fov_build(mdc_fov* f, int mode, const float out_calib_in[5]) {
    const MathSel m{f->float_math};
    const float omega = f->in_calib[4];
    const float d2t = m.d2t(omega);
    const Intrinsics in = input_intrinsics(f);
    const int W = f->in_w, H = f->in_h, OW = f->out_w, OH = f->out_h;
    float ofx, ofy, ocx, ocy;

    if (omega == 0) {
        // no distortion: same relative intrinsics at the output size
        ofx = f->in_calib[0] * OW;
        ofy = f->in_calib[1] * OH;
        ocx = minus_half_d(f->in_calib[2] * OW);
        ocy = minus_half_d(f->in_calib[3] * OH);
    } else if (mode == MDC_FOV_CROP || mode == MDC_FOV_FULL) {
        // normalised radii of the four image borders as seen from the principal point
        const float rl = in.cx / in.fx, rr = (W - 1 - in.cx) / in.fx;
        const float rt = in.cy / in.fy, rb = (H - 1 - in.cy) / in.fy;
        if (mode == MDC_FOV_CROP) {
            const float tl = m.trans(rl, omega, d2t), tr = m.trans(rr, omega, d2t);
            const float tt = m.trans(rt, omega, d2t), tb = m.trans(rb, omega, d2t);
            ofy = in.fy * ((rt + rb) / (tt + tb)) * ((float)OH / (float)H);
            ocy = (tt / rt) * ofy * in.cy / in.fy;
            ofx = in.fx * ((rl + rr) / (tl + tr)) * ((float)OW / (float)W);
            ocx = (tl / rl) * ofx * in.cx / in.fx;
            printf("new K: %f %f %f %f\n", ofx, ofy, ocx, ocy);
            printf("old K: %f %f %f %f\n", in.fx, in.fy, in.cx, in.cy);
        } else {
            // corner radii and their undistorted counterparts
            const float c_tl = m.root(rl * rl + rt * rt), c_tr = m.root(rr * rr + rt * rt);
            const float c_bl = m.root(rl * rl + rb * rb), c_br = m.root(rr * rr + rb * rb);
            const float u_tl = m.trans(c_tl, omega, d2t), u_tr = m.trans(c_tr, omega, d2t);
            const float u_bl = m.trans(c_bl, omega, d2t), u_br = m.trans(c_br, omega, d2t);
            const float span_h = pick_max(c_br, c_tr) + pick_max(c_bl, c_tl);
            const float span_v = pick_max(c_tr, c_tl) + pick_max(c_bl, c_br);
            const float uspan_h = pick_max(u_br, u_tr) + pick_max(u_bl, u_tl);
            const float uspan_v = pick_max(u_tr, u_tl) + pick_max(u_bl, u_br);
            ofy = in.fy * (span_v / uspan_v) * ((float)OH / (float)H);
            ocy = pick_max(u_tl / c_tl, u_tr / c_tr) * ofy * in.cy / in.fy;
            ofx = in.fx * (span_h / uspan_h) * ((float)OW / (float)W);
            ocx = pick_max(u_bl / c_bl, u_tl / c_tl) * ofx * in.cx / in.fx;
            printf("new K: %f %f %f %f\n", ofx, ofy, ocx, ocy);
            printf("old K: %f %f %f %f\n", in.fx, in.fy, in.cx, in.cy);
        }
    } else {
        ofx = out_calib_in[0] * OW;
        ofy = out_calib_in[1] * OH;
        ocx = minus_half_d(out_calib_in[2] * OW);
        ocy = minus_half_d(out_calib_in[3] * OH);
    }

    // store the output camera relative to the output size (centre shifted back by +0.5, in double)
    f->out_calib[0] = ofx / OW;
    f->out_calib[1] = ofy / OH;
    f->out_calib[2] = static_cast<float>((static_cast<double>(ocx) + 0.5) / static_cast<double>(OW));
    f->out_calib[3] = static_cast<float>((static_cast<double>(ocy) + 0.5) / static_cast<double>(OH));
    f->out_calib[4] = 0;

    // identity grid -> distorted source coordinates
    const size_t n_out = static_cast<size_t>(OW) * OH;
    f->remap_x.resize(n_out);
    f->remap_y.resize(n_out);
    for (int y = 0; y < OH; ++y) {
        float* rx = &f->remap_x[static_cast<size_t>(y) * OW];
        float* ry = &f->remap_y[static_cast<size_t>(y) * OW];
        for (int x = 0; x < OW; ++x) { rx[x] = (float)x; ry[x] = (float)y; }
    }
    mdc_fov_distort(f, f->remap_x.data(), f->remap_y.data(), static_cast<int>(n_out));

    // nudge exact-border hits inwards, then blacken everything not strictly inside, so that
    // the 4 bilinear taps of every surviving entry are in bounds
    const float x_hi = (float)(W - 1), y_hi = (float)(H - 1);
    const float x_hi_in = static_cast<float>(W - 1.01), y_hi_in = static_cast<float>(H - 1.01);
    const float lo_in = static_cast<float>(0.01);
    f->has_black = false;
    for (size_t i = 0; i < n_out; ++i) {
        float& sx = f->remap_x[i];
        float& sy = f->remap_y[i];
        if (sx == 0) sx = lo_in;
        if (sy == 0) sy = lo_in;
        if (sx == x_hi) sx = x_hi_in;
        if (sy == y_hi) sy = y_hi_in;
        const bool inside = sx > 0 && sy > 0 && sx < x_hi && sy < y_hi;
        if (!inside) { sx = -1; sy = -1; f->has_black = true; }
    }
    if (f->has_black) printf("\n\nFOV Undistorter: Warning! Image has black pixels.\n\n\n");

    // pinhole matrices of the rectified and the original camera (row-major 3x3)
    auto fill_K = [](float* k, const float c[5], int w, int h) {
        for (int i = 0; i < 9; ++i) k[i] = 0;
        k[0] = c[0] * w;
        k[4] = c[1] * h;
        k[2] = minus_half_d(c[2] * w);
        k[5] = minus_half_d(c[3] * h);
        k[8] = 1;
    };
    fill_K(f->k_rect, f->out_calib, OW, OH);
    fill_K(f->k_org, f->in_calib, W, H);
}

// Sizes come from files: everything allocated from them (remap tables, vignette maps, device buffers) stays below 2^28 pixels per image,
// the limit the image decoders use too, so that a crafted header cannot make an allocation throw across the C ABI.
static bool size_ok(int w, int h) { return static_cast<long long>(w) * h <= (1LL << 28); }

// -------------------------------------------------------------- FOV model: C entry points
static int fov_from_file(const char* path, int float_math, mdc_fov** out) {
    if (!out) { mdc_set_error("mdc_fov_create: out is NULL"); return MDC_ERR_INVALID_ARG; }
    mdc_fov* f = new mdc_fov();
    f->float_math = float_math ? 1 : 0;
    *out = f;

    std::ifstream file(path ? path : "");
    if (!file.good()) {
        printf("Failed to read camera calibration (invalid format?)\nCalibration file: %s\n", path ? path : "(null)");
        mdc_set_error("cannot open camera calibration %s", path ? path : "(null)");
        return MDC_ERR_IO;
    }
    std::string line[4];
    for (int i = 0; i < 4; ++i) std::getline(file, line[i]);

    float* c = f->in_calib;
    if (!(std::sscanf(line[0].c_str(), "%f %f %f %f %f", c, c + 1, c + 2, c + 3, c + 4) == 5 &&
          std::sscanf(line[1].c_str(), "%d %d", &f->in_w, &f->in_h) == 2)) {
        printf("Failed to read camera calibration (invalid format?)\nCalibration file: %s\n", path);
        mdc_set_error("camera calibration %s: lines 1-2 malformed", path);
        return MDC_ERR_FORMAT;
    }
    f->dims_known = true;
    printf("Input resolution: %d %d\n", f->in_w, f->in_h);
    printf("Input Calibration (fx fy cx cy): %f %f %f %f %f\n", f->in_w * c[0], f->in_h * c[1], f->in_w * c[2],
           f->in_h * c[3], c[4]);

    int mode;
    float oc[5] = {0, 0, 0, 0, 0};
    if (line[2] == "crop") { mode = MDC_FOV_CROP; printf("Out: Crop\n"); }
    else if (line[2] == "full") { mode = MDC_FOV_FULL; printf("Out: Full\n"); }
    else if (line[2] == "none") {
        printf("NO RECTIFICATION\n");
        mdc_set_error("camera calibration %s: rectification disabled ('none')", path);
        return MDC_ERR_INVALID_OBJECT;
    } else if (std::sscanf(line[2].c_str(), "%f %f %f %f %f", oc, oc + 1, oc + 2, oc + 3, oc + 4) == 5) {
        mode = MDC_FOV_EXPLICIT;
        printf("Out: %f %f %f %f %f\n", oc[0], oc[1], oc[2], oc[3], oc[4]);
    } else {
        printf("Out: Failed to Read Output pars... not rectifying.\n");
        mdc_set_error("camera calibration %s: line 3 malformed", path);
        return MDC_ERR_FORMAT;
    }
    if (std::sscanf(line[3].c_str(), "%d %d", &f->out_w, &f->out_h) != 2) {
        printf("Out: Failed to Read Output resolution... not rectifying.\n");
        mdc_set_error("camera calibration %s: line 4 malformed", path);
        return MDC_ERR_FORMAT;
    }
    printf("Output resolution: %d %d\n", f->out_w, f->out_h);
    if (f->in_w < 2 || f->in_h < 2 || f->out_w < 1 || f->out_h < 1) {
        mdc_set_error("camera calibration %s: non-positive image size", path);
        return MDC_ERR_FORMAT;
    }
    if (!size_ok(f->in_w, f->in_h) || !size_ok(f->out_w, f->out_h)) {      // the tables below are allocated from these numbers
        mdc_set_error("camera calibration %s: image larger than 2^28 pixels", path);
        return MDC_ERR_FORMAT;
    }
    f->valid = true;
    mdc_fov_build(f, mode, oc);
    return MDC_OK;
}

extern "C" int mdc_fov_create(const char* camera_txt, mdc_fov** out) { return fov_from_file(camera_txt, 0, out); }
extern "C" int mdc_fov_create_ex(const char* camera_txt, int float_math, mdc_fov** out) {
    return fov_from_file(camera_txt, float_math, out);
}

extern "C" int mdc_fov_create_from_params(const float in_calib[5], int in_w, int in_h, int mode,
                                          const float out_calib[5], int out_w, int out_h, int float_math,
                                          mdc_fov** out) {
    if (!out || !in_calib) { mdc_set_error("mdc_fov_create_from_params: NULL argument"); return MDC_ERR_INVALID_ARG; }
    if (in_w < 2 || in_h < 2 || out_w < 1 || out_h < 1 || !size_ok(in_w, in_h) || !size_ok(out_w, out_h)) { mdc_set_error("mdc_fov_create_from_params: bad size"); return MDC_ERR_INVALID_ARG; }
    if (mode == MDC_FOV_EXPLICIT && !out_calib) { mdc_set_error("mdc_fov_create_from_params: explicit mode needs out_calib"); return MDC_ERR_INVALID_ARG; }
    mdc_fov* f = new mdc_fov();
    f->float_math = float_math ? 1 : 0;
    memcpy(f->in_calib, in_calib, sizeof(float) * 5);
    f->in_w = in_w; f->in_h = in_h; f->out_w = out_w; f->out_h = out_h;
    f->dims_known = true;
    f->valid = true;
    const float zero[5] = {0, 0, 0, 0, 0};
    mdc_fov_build(f, mode, out_calib ? out_calib : zero);
    *out = f;
    return MDC_OK;
}

extern "C" void mdc_fov_destroy(mdc_fov* f) { delete f; }
extern "C" int mdc_fov_is_valid(const mdc_fov* f) { return f && f->valid ? 1 : 0; }
extern "C" int mdc_fov_dims(const mdc_fov* f, int* in_w, int* in_h, int* out_w, int* out_h) {
    if (!f) return MDC_ERR_INVALID_ARG;
    if (in_w) *in_w = f->in_w;
    if (in_h) *in_h = f->in_h;
    if (out_w) *out_w = f->out_w;
    if (out_h) *out_h = f->out_h;
    return f->dims_known ? MDC_OK : MDC_ERR_INVALID_OBJECT;
}
extern "C" int mdc_fov_get_K(const mdc_fov* f, float k_rect[9], float k_org[9]) {
    if (!f) return MDC_ERR_INVALID_ARG;
    if (k_rect) memcpy(k_rect, f->k_rect, sizeof f->k_rect);
    if (k_org) memcpy(k_org, f->k_org, sizeof f->k_org);
    return f->valid ? MDC_OK : MDC_ERR_INVALID_OBJECT;
}
extern "C" float mdc_fov_omega(const mdc_fov* f) { return f ? f->in_calib[4] : 0.0f; }
extern "C" int mdc_fov_original_calibration(const mdc_fov* f, float v[5]) {
    if (!f || !v) return MDC_ERR_INVALID_ARG;
    v[0] = f->in_calib[0] * f->in_w;
    v[1] = f->in_calib[1] * f->in_h;
    v[2] = minus_half_d(f->in_calib[2] * f->in_w);
    v[3] = minus_half_d(f->in_calib[3] * f->in_h);
    v[4] = f->in_calib[4];
    return MDC_OK;
}
extern "C" int mdc_fov_distort_coordinates(const mdc_fov* f, float* x, float* y, int n) {
    if (!f || !x || !y || n < 0) return MDC_ERR_INVALID_ARG;
    if (!f->valid) {
        printf("ERROR: invalid UndistorterFOV!\n");
        mdc_set_error("distortCoordinates on an invalid rectifier");
        return MDC_ERR_INVALID_OBJECT;
    }
    mdc_fov_distort(f, x, y, n);
    return MDC_OK;
}
extern "C" const float* mdc_fov_remap_x(const mdc_fov* f) { return f && f->valid ? f->remap_x.data() : nullptr; }
extern "C" const float* mdc_fov_remap_y(const mdc_fov* f) { return f && f->valid ? f->remap_y.data() : nullptr; }

// ------------------------------------------------------------------- photometric model
bool mdc_photo_set_gamma(mdc_photo* p, const float raw[256]) {
    for (int i = 0; i < 256; ++i) p->GInv[i] = raw[i];
    for (int i = 0; i + 1 < 256; ++i)
        if (p->GInv[i + 1] <= p->GInv[i]) {
            printf("PhotometricUndistorter: G invalid! it has to be strictly increasing, but it isnt!\n");
            return false;
        }
    // stretch to 0..255: float difference, then double multiply/divide, one narrowing
    const float lo = p->GInv[0], hi = p->GInv[255];
    const float range = hi - lo;
    for (int i = 0; i < 256; ++i) {
        const float d = p->GInv[i] - lo;
        p->GInv[i] = static_cast<float>(255.0 * static_cast<double>(d) / static_cast<double>(range));
    }
    // forward response by bracket search + linear interpolation (nobody downstream reads it)
    for (int level = 1; level < 255; ++level) {
        for (int s = 1; s < 255; ++s) {
            if (p->GInv[s] <= level && p->GInv[s + 1] >= level) {
                p->G[level] = s + (level - p->GInv[s]) / (p->GInv[s + 1] - p->GInv[s]);
                break;
            }
        }
    }
    p->G[0] = 0;
    p->G[255] = 255;
    p->valid_gamma = true;
    return true;
}

void mdc_photo_set_vignette(mdc_photo* p, const void* pixels, int depth) {
    const size_t n = static_cast<size_t>(p->w) * p->h;
    float peak = 0;
    if (depth == 8) {
        const uint8_t* px = static_cast<const uint8_t*>(pixels);
        for (size_t i = 0; i < n; ++i) if (px[i] > peak) peak = px[i];
        for (size_t i = 0; i < n; ++i) p->vmap[i] = px[i] / peak;
    } else {
        const uint16_t* px = static_cast<const uint16_t*>(pixels);
        for (size_t i = 0; i < n; ++i) if (px[i] > peak) peak = px[i];
        for (size_t i = 0; i < n; ++i) p->vmap[i] = px[i] / peak;
    }
    for (size_t i = 0; i < n; ++i) p->vinv[i] = 1.0f / p->vmap[i];
    p->valid_vignette = true;
}

static mdc_photo* new_photo(int w, int h) {
    mdc_photo* p = new mdc_photo();
    p->w = w; p->h = h;
    for (int i = 0; i < 256; ++i) { p->G[i] = 0; p->GInv[i] = 0; }
    return p;
}

extern "C" int mdc_photo_create(const char* pcalib_txt, const char* vignette_image, int w, int h, mdc_photo** out) {
    if (!out) { mdc_set_error("mdc_photo_create: out is NULL"); return MDC_ERR_INVALID_ARG; }
    mdc_photo* p = new_photo(w, h);
    *out = p;
    const std::string calib = pcalib_txt ? pcalib_txt : "", vig = vignette_image ? vignette_image : "";
    if (calib == "" || vig == "") { mdc_set_error("photometric calibration: empty file name"); return MDC_ERR_INVALID_OBJECT; }

    std::ifstream f(calib.c_str());
    printf("Reading Photometric Calibration from file %s\n", calib.c_str());
    if (!f.good()) {
        printf("PhotometricUndistorter: Could not open file!\n");
        mdc_set_error("cannot open %s", calib.c_str());
        return MDC_ERR_IO;
    }
    std::string first;
    std::getline(f, first);
    std::istringstream tokens(first);
    std::vector<float> raw;
    for (float v; tokens >> v;) raw.push_back(v);
    if (raw.size() != 256) {
        printf("PhotometricUndistorter: invalid format! got %d entries in first line, expected 256!\n", (int)raw.size());
        mdc_set_error("%s: %d entries in first line, expected 256", calib.c_str(), (int)raw.size());
        return MDC_ERR_FORMAT;
    }
    if (!mdc_photo_set_gamma(p, raw.data())) { mdc_set_error("%s: response not strictly increasing", calib.c_str()); return MDC_ERR_FORMAT; }
    if (w < 1 || h < 1 || !size_ok(w, h)) { mdc_set_error("photometric calibration: bad image size %d x %d", w, h); return MDC_ERR_INVALID_ARG; }

    printf("Reading Vignette Image from %s\n", vig.c_str());
    p->vmap.assign(static_cast<size_t>(w) * h, 0.0f);
    p->vinv.assign(static_cast<size_t>(w) * h, 0.0f);
    mdc_gray_image img;
    const bool readable = mdc_read_gray_image(vig, &img);
    if (img.rows != h || img.cols != w) {
        printf("PhotometricUndistorter: Invalid vignette image size! got %d x %d, expected %d x %d. Set vignette to 1.\n",
               img.cols, img.rows, w, h);
        if (readable) mdc_set_error("%s: vignette is %d x %d, expected %d x %d", vig.c_str(), img.cols, img.rows, w, h);
        return readable ? MDC_ERR_FORMAT : MDC_ERR_IO;
    }
    mdc_photo_set_vignette(p, img.px.data(), img.depth);
    printf("Successfully read photometric calibration!\n");
    return MDC_OK;
}

extern "C" int mdc_photo_create_from_arrays(const float* ginv_raw256, const void* vignette_pixels, int depth,
                                            int rows, int cols, int w, int h, mdc_photo** out) {
    if (!out) { mdc_set_error("mdc_photo_create_from_arrays: out is NULL"); return MDC_ERR_INVALID_ARG; }
    mdc_photo* p = new_photo(w, h);
    *out = p;
    if (!ginv_raw256 || !vignette_pixels) { mdc_set_error("photometric calibration: missing table"); return MDC_ERR_INVALID_OBJECT; }
    if (!mdc_photo_set_gamma(p, ginv_raw256)) { mdc_set_error("response not strictly increasing"); return MDC_ERR_FORMAT; }
    if (w < 1 || h < 1 || !size_ok(w, h)) { mdc_set_error("photometric calibration: bad image size"); return MDC_ERR_INVALID_ARG; }
    p->vmap.assign(static_cast<size_t>(w) * h, 0.0f);
    p->vinv.assign(static_cast<size_t>(w) * h, 0.0f);
    if (rows != h || cols != w || (depth != 8 && depth != 16)) {
        printf("PhotometricUndistorter: Invalid vignette image size! got %d x %d, expected %d x %d. Set vignette to 1.\n", cols, rows, w, h);
        mdc_set_error("vignette is %d x %d (depth %d), expected %d x %d", cols, rows, depth, w, h);
        return MDC_ERR_FORMAT;
    }
    mdc_photo_set_vignette(p, vignette_pixels, depth);
    return MDC_OK;
}

extern "C" void mdc_photo_destroy(mdc_photo* p) { delete p; }
extern "C" int mdc_photo_valid_gamma(const mdc_photo* p) { return p && p->valid_gamma ? 1 : 0; }
extern "C" int mdc_photo_valid_vignette(const mdc_photo* p) { return p && p->valid_vignette ? 1 : 0; }
extern "C" float* mdc_photo_ginv(mdc_photo* p) { return p && p->valid_gamma ? p->GInv : nullptr; }
extern "C" float* mdc_photo_g(mdc_photo* p) { return p && p->valid_gamma ? p->G : nullptr; }
extern "C" const float* mdc_photo_vignette_map(const mdc_photo* p) { return p && p->valid_vignette ? p->vmap.data() : nullptr; }
extern "C" const float* mdc_photo_vignette_map_inv(const mdc_photo* p) { return p && p->valid_vignette ? p->vinv.data() : nullptr; }
