// Host half of vignetteCalib's marker detection: aruco 1.3.0's MarkerDetector::detect with its default settings (ADPT_THRES 7/7,
// LINES corners, 56-pixel warp, FiducidalMarkers::detect as the id reader), from the grey image and the adaptive-threshold mask that
// mdc_marker_threshold computes on the GPU.  Paths are relative to aruco-1.3.0/src/ unless a file of the reference is named.
//
// The OpenCV primitives aruco calls are restated here from their documented algorithms so that the results are the same
// integers and the same float bits: findContours (Suzuki-Abe border following, CV_RETR_LIST, CV_CHAIN_APPROX_NONE), approxPolyDP
// (closed-curve Douglas-Peucker), isContourConvex, getPerspectiveTransform (8x8 LU in double), warpPerspective (INTER_NEAREST,
// inverse map, BORDER_CONSTANT 0), threshold(THRESH_OTSU).  The two fp32 least-squares solves of the LINES corner refinement
// (solve(..., DECOMP_SVD)) are computed in double and rounded to float: within 1e-3 px of OpenCV's fp32 SVD, not the same bits.
//
// Everything lives on the stack of the call or in vectors it owns: the functions are re-entrant, one frame per thread.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <utility>
#include <vector>

#include "mdc_internal.h"

namespace {

constexpr int64_t kMaxPixels = int64_t(1) << 28;   // the bound every image size of the library is held to
constexpr int kMaxContours = 1 << 22;               // a noise mask of 2^23 pixels has about 2^21 contours
constexpr int kMaxCandidates = 1 << 14;             // the too-near test is quadratic in this
constexpr int kWarp = 56;                            // _markerWarpSize, markerdetector.cpp:59

struct Pt { int x, y; };
struct Pf { float x, y; };

struct Candidate {
    Pf c[4];
    std::vector<Pt> contour;
};

struct Marker {
    int id;
    Pf c[4];
};

bool check_size(int w, int h, const char* who) {
    if (w < 1 || h < 1 || static_cast<int64_t>(w) * h > kMaxPixels) {
        mdc_set_error("%s: image size %d x %d outside 1 .. 2^28 pixels", who, w, h);
        return false;
    }
    return true;
}

// ---- findContours(CV_RETR_LIST, CV_CHAIN_APPROX_NONE) ----------------------------------------------------------------------
// The mask is copied to signed bytes (non-zero -> 1) with the outer rows and columns cleared, as cvStartFindContours does.  Traced
// pixels become 2, or kRight when the pixel to their right is background (a right edge): an outer border starts at a 1 after a 0,
// a hole border at a 0 after a positive pixel.  Contours are produced in raster order of their start; findContours lists them
// last-found first.
constexpr int8_t kRight = static_cast<int8_t>(2 | -128);
const int kCodeDx[8] = {1, 1, 0, -1, -1, -1, 0, 1};   // chain code s: (dx, dy) with y down
const int kCodeDy[8] = {0, -1, -1, -1, 0, 1, 1, 1};

class ContourScanner {
public:
    ContourScanner(const uint8_t* mask, int w, int h) : w_(w), h_(h), img_(static_cast<size_t>(w) * h) {
        for (int y = 1; y + 1 < h; ++y)
            for (int x = 1; x + 1 < w; ++x) img_[static_cast<size_t>(y) * w + x] = mask[static_cast<size_t>(y) * w + x] != 0;
        for (int s = 0; s < 16; ++s) delta_[s] = static_cast<ptrdiff_t>(kCodeDy[s & 7]) * w + kCodeDx[s & 7];
        y_ = 1; x_ = 1; prev_ = 0;
    }

    // Next contour in discovery order into *out; false when the image is exhausted.
    bool next(std::vector<Pt>* out) {
        for (; y_ + 1 < h_; ++y_, x_ = 1, prev_ = 0) {
            int8_t* row = img_.data() + static_cast<size_t>(y_) * w_;
            for (; x_ + 1 < w_; ++x_) {
                const int p = row[x_];
                if (p == prev_) continue;
                int hole = 0;
                if (!(prev_ == 0 && p == 1)) {
                    if (p != 0 || prev_ < 1) { prev_ = p; continue; }
                    hole = 1;
                }
                fetch(row + x_ - hole, Pt{x_ - hole, y_}, hole, out);
                prev_ = row[x_];
                ++x_;
                return true;
            }
        }
        return false;
    }

private:
    // icvFetchContour with CV_CHAIN_APPROX_NONE: every border pixel once per visit, starting at the start pixel
    void fetch(int8_t* i0, Pt pt, int hole, std::vector<Pt>* out) {
        out->clear();
        int s = hole ? 0 : 4, s_end = s;
        int8_t* i1;
        do {
            s = (s - 1) & 7;
            i1 = i0 + delta_[s];
        } while (*i1 == 0 && s != s_end);
        if (s == s_end) {                      // isolated pixel
            *i0 = kRight;
            out->push_back(pt);
            return;
        }
        int8_t* i3 = i0;
        int8_t* i4 = nullptr;
        for (;;) {
            s_end = s;
            while (s < 15) {
                i4 = i3 + delta_[++s];
                if (*i4 != 0) break;
            }
            s &= 7;
            if (static_cast<unsigned>(s - 1) < static_cast<unsigned>(s_end)) *i3 = kRight;
            else if (*i3 == 1) *i3 = 2;
            out->push_back(pt);
            pt.x += kCodeDx[s];
            pt.y += kCodeDy[s];
            if (i4 == i0 && i3 == i1) break;
            i3 = i4;
            s = (s + 4) & 7;
        }
    }

    int w_, h_;
    std::vector<int8_t> img_;
    ptrdiff_t delta_[16];
    int y_, x_, prev_;
};

// ---- approxPolyDP(contour, eps, closed = true) -------------------------------------------------------------------------------
// Start point: three rounds of "farthest point from the current start", the last start and its farthest point split the curve;
// then iterative Douglas-Peucker on a stack of slices (last pushed first) and a clean-up pass over nearly straight vertices.
// cv2 4.13 picks another split on about 1 in 3000 tiny (< 70 point) self-touching noise contours; marker-sized contours agree.
void approx_poly_closed(const std::vector<Pt>& src, double eps, std::vector<Pt>* dst_out) {
    const int count = static_cast<int>(src.size());
    std::vector<Pt>& dst = *dst_out;
    dst.assign(count, Pt{0, 0});
    if (count == 0) { dst.clear(); return; }
    struct Range { int start, end; };
    std::vector<Range> stack;
    Range slice{0, 0}, right{0, 0};
    Pt start_pt{-1000000, -1000000}, end_pt{0, 0}, pt{0, 0};
    int pos = 0, new_count = 0;
    bool le_eps = false;
    auto read = [&](Pt& p, int& q) { p = src[q]; if (++q >= count) q = 0; };
    eps *= eps;
    for (int it = 0; it < 3; ++it) {
        double max_dist = 0;
        pos = (pos + right.start) % count;
        read(start_pt, pos);
        for (int j = 1; j < count; ++j) {
            read(pt, pos);
            const double dx = pt.x - start_pt.x, dy = pt.y - start_pt.y;
            const double dist = dx * dx + dy * dy;
            if (dist > max_dist) { max_dist = dist; right.start = j; }
        }
        le_eps = max_dist <= eps;
    }
    if (!le_eps) {
        right.end = slice.start = pos % count;
        slice.end = right.start = (right.start + slice.start) % count;
        stack.push_back(right);
        stack.push_back(slice);
    } else {
        dst[new_count++] = start_pt;
    }
    while (!stack.empty()) {
        slice = stack.back();
        stack.pop_back();
        end_pt = src[slice.end];
        pos = slice.start;
        read(start_pt, pos);
        if (pos != slice.end) {
            double max_dist = 0;
            const double dx = end_pt.x - start_pt.x, dy = end_pt.y - start_pt.y;
            while (pos != slice.end) {
                read(pt, pos);
                const double dist = std::fabs((pt.y - start_pt.y) * dx - (pt.x - start_pt.x) * dy);
                if (dist > max_dist) { max_dist = dist; right.start = (pos + count - 1) % count; }
            }
            le_eps = max_dist * max_dist <= eps * (dx * dx + dy * dy);
        } else {
            le_eps = true;
            start_pt = src[slice.start];
        }
        if (le_eps) {
            dst[new_count++] = start_pt;
        } else {
            right.end = slice.end;
            slice.end = right.start;
            stack.push_back(right);
            stack.push_back(slice);
        }
    }
    // clean-up: drop a vertex that lies within sqrt(eps/2) of the chord of its neighbours (closed curve)
    const int n = new_count;
    auto read_dst = [&](Pt& p, int& q) { p = dst[q]; if (++q >= n) q = 0; };
    pos = n - 1;
    read_dst(start_pt, pos);
    int wpos = pos;
    read_dst(pt, pos);
    for (int i = 0; i < n && new_count > 2; ++i) {
        read_dst(end_pt, pos);
        const double dx = end_pt.x - start_pt.x, dy = end_pt.y - start_pt.y;
        const double dist = std::fabs((pt.x - start_pt.x) * dy - (pt.y - start_pt.y) * dx);
        const double inner = static_cast<double>(pt.x - start_pt.x) * (end_pt.x - pt.x) + static_cast<double>(pt.y - start_pt.y) * (end_pt.y - pt.y);
        if (dist * dist <= 0.5 * eps * (dx * dx + dy * dy) && dx != 0 && dy != 0 && inner >= 0) {
            new_count--;
            dst[wpos] = start_pt = end_pt;
            if (++wpos >= n) wpos = 0;
            read_dst(pt, pos);
            i++;
            continue;
        }
        dst[wpos] = start_pt = pt;
        if (++wpos >= n) wpos = 0;
        pt = end_pt;
    }
    dst.resize(new_count);
}

// isContourConvex on integer points: every turn strictly the same way (a straight vertex is not convex)
bool is_convex(const std::vector<Pt>& p) {
    const int n = static_cast<int>(p.size());
    if (n == 0) return false;
    Pt prev = p[(n - 2 + n) % n], cur = p[n - 1];
    int64_t dx0 = cur.x - prev.x, dy0 = cur.y - prev.y;
    int orientation = 0;
    for (int i = 0; i < n; ++i) {
        prev = cur;
        cur = p[i];
        const int64_t dx = cur.x - prev.x, dy = cur.y - prev.y;
        const int64_t dxdy0 = dx * dy0, dydx0 = dy * dx0;
        orientation |= dydx0 > dxdy0 ? 1 : (dydx0 < dxdy0 ? 2 : 3);
        if (orientation == 3) return false;
        dx0 = dx;
        dy0 = dy;
    }
    return true;
}

// MarkerDetector::perimeter, markerdetector.cpp:755: float side lengths added into an int (truncating at every step)
int perimeter(const Pf* a) {
    int sum = 0;
    for (int i = 0; i < 4; ++i) {
        const int i2 = (i + 1) % 4;
        const float dx = a[i].x - a[i2].x, dy = a[i].y - a[i2].y;
        sum = static_cast<int>(static_cast<float>(sum) + std::sqrt(dx * dx + dy * dy));
    }
    return sum;
}

// ---- detectRectangles, markerdetector.cpp:287-430 --------------------------------------------------------------------------
int find_candidates(const uint8_t* mask, int w, int h, std::vector<Candidate>* out) {
    const int m = std::max(w, h);
    const int min_size = static_cast<int>(0.04 * m * 4), max_size = static_cast<int>(0.5 * m * 4);   // _minSize, _maxSize
    ContourScanner scanner(mask, w, h);
    std::vector<Pt> contour, approx;
    std::vector<Candidate> found;        // discovery order; findContours lists the contours the other way round
    int contours = 0;
    while (scanner.next(&contour)) {
        if (++contours > kMaxContours) {
            mdc_set_error("mdc_marker_detect: more than %d contours in the mask", kMaxContours);
            return MDC_ERR_UNSUPPORTED;
        }
        const int64_t n = static_cast<int64_t>(contour.size());
        if (!(min_size < n && n < max_size)) continue;
        approx_poly_closed(contour, static_cast<double>(n) * 0.05, &approx);
        if (approx.size() != 4 || !is_convex(approx)) continue;
        float min_dist = 1e10f;
        for (int j = 0; j < 4; ++j) {
            const Pt& a = approx[j];
            const Pt& b = approx[(j + 1) % 4];
            const float d = std::sqrt(static_cast<float>(a.x - b.x) * (a.x - b.x) + static_cast<float>(static_cast<int64_t>(a.y - b.y) * (a.y - b.y)));
            if (d < min_dist) min_dist = d;
        }
        if (!(min_dist > 10)) continue;
        if (found.size() >= static_cast<size_t>(kMaxCandidates)) {
            mdc_set_error("mdc_marker_detect: more than %d marker candidates in the mask", kMaxCandidates);
            return MDC_ERR_UNSUPPORTED;
        }
        found.emplace_back();
        for (int j = 0; j < 4; ++j) found.back().c[j] = Pf{static_cast<float>(approx[j].x), static_cast<float>(approx[j].y)};
        found.back().contour = contour;
    }
    std::reverse(found.begin(), found.end());
    // corners anti-clockwise in image coordinates: swap 1 and 3 when the third corner is left of 0 -> 1 (the contour follows)
    std::vector<char> swapped(found.size(), 0);
    for (size_t i = 0; i < found.size(); ++i) {
        Pf* c = found[i].c;
        const double dx1 = c[1].x - c[0].x, dy1 = c[1].y - c[0].y, dx2 = c[2].x - c[0].x, dy2 = c[2].y - c[0].y;
        if (dx1 * dy2 - dy1 * dx2 < 0.0) { std::swap(c[1], c[3]); swapped[i] = 1; }
    }
    // of two candidates whose corners are all closer than 6 px, the one with the smaller perimeter goes (the first on a tie)
    std::vector<char> remove(found.size(), 0);
    for (size_t i = 0; i < found.size(); ++i)
        for (size_t j = i + 1; j < found.size(); ++j) {
            bool near = true;
            for (int c = 0; c < 4 && near; ++c) {
                const float dx = found[i].c[c].x - found[j].c[c].x, dy = found[i].c[c].y - found[j].c[c].y;
                near = std::sqrt(dx * dx + dy * dy) < 6;
            }
            if (near) {
                if (perimeter(found[i].c) > perimeter(found[j].c)) remove[j] = 1;
                else remove[i] = 1;
            }
        }
    out->clear();
    for (size_t i = 0; i < found.size(); ++i) {
        if (remove[i]) continue;
        out->push_back(std::move(found[i]));
        if (swapped[i]) std::reverse(out->back().contour.begin(), out->back().contour.end());
    }
    return MDC_OK;
}

// ---- warp + FiducidalMarkers::detect ---------------------------------------------------------------------------------------
// cv::solve(DECOMP_LU) of an n x n system: partial pivoting, 0 when a pivot is below 100 DBL_EPSILON
bool lu_solve(double* A, double* b, int m) {
    for (int i = 0; i < m; ++i) {
        int k = i;
        for (int j = i + 1; j < m; ++j)
            if (std::fabs(A[j * m + i]) > std::fabs(A[k * m + i])) k = j;
        if (std::fabs(A[k * m + i]) < 100 * 2.220446049250313e-16) return false;
        if (k != i) {
            for (int j = i; j < m; ++j) std::swap(A[i * m + j], A[k * m + j]);
            std::swap(b[i], b[k]);
        }
        const double d = -1 / A[i * m + i];
        for (int j = i + 1; j < m; ++j) {
            const double alpha = A[j * m + i] * d;
            for (int q = i + 1; q < m; ++q) A[j * m + q] += alpha * A[i * m + q];
            b[j] += alpha * b[i];
        }
        A[i * m + i] = -d;
    }
    for (int i = m - 1; i >= 0; --i) {
        double s = b[i];
        for (int q = i + 1; q < m; ++q) s -= A[i * m + q] * b[q];
        b[i] = s * A[i * m + i];
    }
    return true;
}

// getPerspectiveTransform(quad -> 56 x 56 square), inverted (3x3 adjugate / determinant) for warpPerspective's backward map
bool warp_matrix(const Pf* quad, double Minv[9]) {
    const float dx[4] = {0, kWarp - 1, kWarp - 1, 0}, dy[4] = {0, 0, kWarp - 1, kWarp - 1};
    double a[64] = {0}, b[8];
    for (int i = 0; i < 4; ++i) {
        a[i * 8 + 0] = a[(i + 4) * 8 + 3] = quad[i].x;
        a[i * 8 + 1] = a[(i + 4) * 8 + 4] = quad[i].y;
        a[i * 8 + 2] = a[(i + 4) * 8 + 5] = 1;
        a[i * 8 + 6] = -quad[i].x * dx[i];            // float products, as with Point2f
        a[i * 8 + 7] = -quad[i].y * dx[i];
        a[(i + 4) * 8 + 6] = -quad[i].x * dy[i];
        a[(i + 4) * 8 + 7] = -quad[i].y * dy[i];
        b[i] = dx[i];
        b[i + 4] = dy[i];
    }
    if (!lu_solve(a, b, 8)) return false;
    double M[9];
    for (int i = 0; i < 8; ++i) M[i] = b[i];
    M[8] = 1.;
    auto S = [&](int r, int c) { return M[r * 3 + c]; };
    double d = S(0, 0) * (S(1, 1) * S(2, 2) - S(1, 2) * S(2, 1)) - S(0, 1) * (S(1, 0) * S(2, 2) - S(1, 2) * S(2, 0)) +
               S(0, 2) * (S(1, 0) * S(2, 1) - S(1, 1) * S(2, 0));
    if (d == 0.) return false;
    d = 1. / d;
    Minv[0] = (S(1, 1) * S(2, 2) - S(1, 2) * S(2, 1)) * d;
    Minv[1] = (S(0, 2) * S(2, 1) - S(0, 1) * S(2, 2)) * d;
    Minv[2] = (S(0, 1) * S(1, 2) - S(0, 2) * S(1, 1)) * d;
    Minv[3] = (S(1, 2) * S(2, 0) - S(1, 0) * S(2, 2)) * d;
    Minv[4] = (S(0, 0) * S(2, 2) - S(0, 2) * S(2, 0)) * d;
    Minv[5] = (S(0, 2) * S(1, 0) - S(0, 0) * S(1, 2)) * d;
    Minv[6] = (S(1, 0) * S(2, 1) - S(1, 1) * S(2, 0)) * d;
    Minv[7] = (S(0, 1) * S(2, 0) - S(0, 0) * S(2, 1)) * d;
    Minv[8] = (S(0, 0) * S(1, 1) - S(0, 1) * S(1, 0)) * d;
    return true;
}

int sat_short(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }

// warpPerspective(INTER_NEAREST): per destination pixel W = 1/W (0 stays 0), source = round-half-even of X*W, Y*W clamped to int
// then to short; outside the image -> 0.  A 56-pixel row is one block, so each row starts from x = 0.
bool warp_patch(const uint8_t* grey, int w, int h, const Pf* quad, uint8_t* patch) {
    double M[9];
    if (!warp_matrix(quad, M)) return false;
    for (int y = 0; y < kWarp; ++y) {
        const double X0 = M[0] * 0 + M[1] * y + M[2], Y0 = M[3] * 0 + M[4] * y + M[5], W0 = M[6] * 0 + M[7] * y + M[8];
        for (int x = 0; x < kWarp; ++x) {
            double W = W0 + M[6] * x;
            W = W != 0 ? 1. / W : 0;
            const double fX = std::max(static_cast<double>(INT32_MIN), std::min(static_cast<double>(INT32_MAX), (X0 + M[0] * x) * W));
            const double fY = std::max(static_cast<double>(INT32_MIN), std::min(static_cast<double>(INT32_MAX), (Y0 + M[3] * x) * W));
            const int X = sat_short(static_cast<int>(std::nearbyint(fX))), Y = sat_short(static_cast<int>(std::nearbyint(fY)));
            patch[y * kWarp + x] = (X >= 0 && X < w && Y >= 0 && Y < h) ? grey[static_cast<size_t>(Y) * w + X] : 0;
        }
    }
    return true;
}

// threshold(THRESH_OTSU): the first bin that maximises the between-class variance (bins whose class weight is within
// FLT_EPSILON of 0 or 1 skipped)
int otsu(const uint8_t* p, int n) {
    int hist[256] = {0};
    for (int i = 0; i < n; ++i) hist[p[i]]++;
    const double scale = 1. / n;
    double mu = 0;
    for (int i = 0; i < 256; ++i) mu += i * static_cast<double>(hist[i]);
    mu *= scale;
    double mu1 = 0, q1 = 0, max_sigma = 0, max_val = 0;
    const double feps = 1.1920928955078125e-07;
    for (int i = 0; i < 256; ++i) {
        const double p_i = hist[i] * scale;
        mu1 *= q1;
        q1 += p_i;
        const double q2 = 1. - q1;
        if (std::min(q1, q2) < feps || std::max(q1, q2) > 1. - feps) continue;
        mu1 = (mu1 + i * p_i) / q1;
        const double mu2 = (mu - q1 * mu1) / q2;
        const double sigma = q1 * q2 * (mu1 - mu2) * (mu1 - mu2);
        if (sigma > max_sigma) { max_sigma = sigma; max_val = i; }
    }
    return static_cast<int>(max_val);
}

// hammDistMarker, arucofidmarkers.cpp:308: per row the distance to the nearest of the four code words
int hamming(const uint8_t bits[25]) {
    static const uint8_t words[4][5] = {{1, 0, 0, 0, 0}, {1, 0, 1, 1, 1}, {0, 1, 0, 0, 1}, {0, 1, 1, 1, 0}};
    int dist = 0;
    for (int y = 0; y < 5; ++y) {
        int best = 100000;
        for (int p = 0; p < 4; ++p) {
            int sum = 0;
            for (int x = 0; x < 5; ++x) sum += bits[y * 5 + x] != words[p][x];
            best = std::min(best, sum);
        }
        dist += best;
    }
    return dist;
}

// FiducidalMarkers::detect on a warped patch (thresholded in place): id, or -1
int read_id(uint8_t* patch, int* thresh_out, int* rotations) {
    const int t = otsu(patch, kWarp * kWarp);
    if (thresh_out) *thresh_out = t;
    for (int i = 0; i < kWarp * kWarp; ++i) patch[i] = patch[i] > t ? 255 : 0;
    const int cell = kWarp / 7;
    auto white = [&](int cx, int cy) {
        int nz = 0;
        for (int y = 0; y < cell; ++y)
            for (int x = 0; x < cell; ++x) nz += patch[(cy * cell + y) * kWarp + cx * cell + x] != 0;
        return nz > cell * cell / 2;
    };
    *rotations = 0;
    for (int y = 0; y < 7; ++y)
        for (int x = 0; x < 7; x += (y == 0 || y == 6) ? 1 : 6)
            if (white(x, y)) return -1;
    uint8_t rot[4][25];
    for (int y = 0; y < 5; ++y)
        for (int x = 0; x < 5; ++x) rot[0][y * 5 + x] = white(x + 1, y + 1);
    int best = hamming(rot[0]), best_r = 0;
    for (int r = 1; r < 4; ++r) {
        for (int i = 0; i < 5; ++i)
            for (int j = 0; j < 5; ++j) rot[r][i * 5 + j] = rot[r - 1][(5 - j - 1) * 5 + i];   // FiducidalMarkers::rotate, :290
        const int d = hamming(rot[r]);
        if (d < best) { best = d; best_r = r; }
    }
    *rotations = best_r;
    if (best != 0) return -1;
    int id = 0;
    for (int y = 0; y < 5; ++y) {
        id = (id << 1) | rot[best_r][y * 5 + 1];
        id = (id << 1) | rot[best_r][y * 5 + 3];
    }
    return id;
}

// ---- refineCandidateLines, markerdetector.cpp:779-928 ------------------------------------------------------------------------
// Least squares for [u 1] (a, c)^T = v (solve(DECOMP_SVD) of the n x 2 system), the minimum-norm solution when all u are equal
void fit_line(const std::vector<Pf>& pts, bool x_major, float* a_out, float* c_out) {
    const size_t n = pts.size();
    double su = 0, sv = 0;
    for (const Pf& p : pts) { su += x_major ? p.x : p.y; sv += x_major ? p.y : p.x; }
    const double mu = su / n, mv = sv / n;
    double suu = 0, suv = 0;
    for (const Pf& p : pts) {
        const double u = (x_major ? p.x : p.y) - mu, v = (x_major ? p.y : p.x) - mv;
        suu += u * u;
        suv += u * v;
    }
    double a, c;
    if (suu > 0) {
        a = suv / suu;
        c = mv - a * mu;
    } else {
        a = mv * mu / (mu * mu + 1);
        c = mv / (mu * mu + 1);
    }
    *a_out = static_cast<float>(a);
    *c_out = static_cast<float>(c);
}

// getCrossPoint: the 2x2 system [l1.x l1.y; l2.x l2.y] p = -[l1.z; l2.z] (pseudo-inverse when singular)
Pf cross_point(const float* l1, const float* l2) {
    const double a = l1[0], b = l1[1], c = l2[0], d = l2[1], r0 = -static_cast<double>(l1[2]), r1 = -static_cast<double>(l2[2]);
    const double det = a * d - b * c;
    if (det != 0) return Pf{static_cast<float>((d * r0 - b * r1) / det), static_cast<float>((a * r1 - c * r0) / det)};
    const double f = a * a + b * b + c * c + d * d;
    if (f == 0) return Pf{0, 0};
    return Pf{static_cast<float>((a * r0 + c * r1) / f), static_cast<float>((b * r0 + d * r1) / f)};
}

void refine_lines(Candidate& cand) {
    const std::vector<Pt>& contour = cand.contour;
    const int size = static_cast<int>(contour.size());
    unsigned idx[4] = {0, 0, 0, 0};
    for (int j = 0; j < size; ++j)
        for (int k = 0; k < 4; ++k)
            if (contour[j].x == cand.c[k].x && contour[j].y == cand.c[k].y) idx[k] = j;
    bool inverse;
    if (idx[1] > idx[0] && (idx[2] > idx[1] || idx[2] < idx[0])) inverse = false;
    else if (idx[2] > idx[1] && idx[2] < idx[0]) inverse = false;
    else inverse = true;
    const int inc = inverse ? -1 : 1;
    float lines[4][3];
    std::vector<Pf> run;
    for (int l = 0; l < 4; ++l) {
        run.clear();
        const int stop = static_cast<int>(idx[(l + 1) % 4]);
        for (int j = static_cast<int>(idx[l]); j != stop; j += inc) {
            if (j == size && !inverse) j = 0;
            else if (j == 0 && inverse) j = size - 1;
            run.push_back(Pf{static_cast<float>(contour[j].x), static_cast<float>(contour[j].y)});
            if (j == stop) break;
        }
        if (run.empty()) run.push_back(Pf{static_cast<float>(contour[stop].x), static_cast<float>(contour[stop].y)});
        float minx = run[0].x, maxx = run[0].x, miny = run[0].y, maxy = run[0].y;
        for (const Pf& p : run) {
            minx = std::min(minx, p.x); maxx = std::max(maxx, p.x);
            miny = std::min(miny, p.y); maxy = std::max(maxy, p.y);
        }
        float a, c;
        if (maxx - minx > maxy - miny) {
            fit_line(run, true, &a, &c);          // y = a x + c  ->  (a, -1, c)
            lines[l][0] = a; lines[l][1] = -1.f; lines[l][2] = c;
        } else {
            fit_line(run, false, &a, &c);         // x = a y + c  ->  (-1, a, c)
            lines[l][0] = -1.f; lines[l][1] = a; lines[l][2] = c;
        }
    }
    for (unsigned i = 0; i < 4; ++i) cand.c[i] = cross_point(lines[(i - 1) % 4], lines[i]);
}

}  // namespace

extern "C" int mdc_marker_candidates(const uint8_t* mask, int w, int h, float* quads, int capacity, int* count) {
    if (!mask || !count || capacity < 0 || (capacity > 0 && !quads)) { mdc_set_error("mdc_marker_candidates: bad argument"); return MDC_ERR_INVALID_ARG; }
    if (!check_size(w, h, "mdc_marker_candidates")) return MDC_ERR_INVALID_ARG;
    std::vector<Candidate> cands;
    const int r = find_candidates(mask, w, h, &cands);
    if (r != MDC_OK) return r;
    *count = static_cast<int>(cands.size());
    for (int i = 0; i < *count && i < capacity; ++i)
        for (int k = 0; k < 4; ++k) { quads[8 * i + 2 * k] = cands[i].c[k].x; quads[8 * i + 2 * k + 1] = cands[i].c[k].y; }
    if (*count > capacity) { mdc_set_error("mdc_marker_candidates: %d candidates, capacity %d", *count, capacity); return MDC_ERR_INVALID_ARG; }
    return MDC_OK;
}

extern "C" int mdc_marker_contours(const uint8_t* mask, int w, int h, int* xy, size_t point_capacity, int* lengths, int contour_capacity,
                                   int* n_contours, size_t* n_points) {
    if (!mask || !n_contours || !n_points || contour_capacity < 0 || (point_capacity && !xy) || (contour_capacity && !lengths)) {
        mdc_set_error("mdc_marker_contours: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    if (!check_size(w, h, "mdc_marker_contours")) return MDC_ERR_INVALID_ARG;
    ContourScanner scanner(mask, w, h);
    std::vector<std::vector<Pt>> all;
    std::vector<Pt> c;
    size_t total = 0;
    while (scanner.next(&c)) {
        if (static_cast<int64_t>(all.size()) >= kMaxContours) { mdc_set_error("mdc_marker_contours: more than %d contours", kMaxContours); return MDC_ERR_UNSUPPORTED; }
        total += c.size();
        all.push_back(c);
    }
    *n_contours = static_cast<int>(all.size());
    *n_points = total;
    if (all.size() > static_cast<size_t>(contour_capacity) || total > point_capacity) {
        mdc_set_error("mdc_marker_contours: %zu contours / %zu points, capacity %d / %zu", all.size(), total, contour_capacity, point_capacity);
        return MDC_ERR_INVALID_ARG;
    }
    size_t q = 0;
    for (size_t i = 0; i < all.size(); ++i) {
        const std::vector<Pt>& a = all[all.size() - 1 - i];
        lengths[i] = static_cast<int>(a.size());
        for (const Pt& p : a) { xy[2 * q] = p.x; xy[2 * q + 1] = p.y; ++q; }
    }
    return MDC_OK;
}

extern "C" int mdc_marker_approx_poly(const int* xy, int n, double eps, int* out_xy, int* n_out) {
    if (n < 0 || (n && (!xy || !out_xy)) || !n_out) { mdc_set_error("mdc_marker_approx_poly: bad argument"); return MDC_ERR_INVALID_ARG; }
    std::vector<Pt> src(n), dst;
    for (int i = 0; i < n; ++i) src[i] = Pt{xy[2 * i], xy[2 * i + 1]};
    approx_poly_closed(src, eps, &dst);
    *n_out = static_cast<int>(dst.size());
    for (size_t i = 0; i < dst.size(); ++i) { out_xy[2 * i] = dst[i].x; out_xy[2 * i + 1] = dst[i].y; }
    return MDC_OK;
}

extern "C" int mdc_marker_read_patch(const uint8_t* grey, int w, int h, const float quad[8], uint8_t* patch, int* otsu_threshold, int* id,
                                     int* rotations) {
    if (!grey || !quad || !patch || !otsu_threshold || !id || !rotations) { mdc_set_error("mdc_marker_read_patch: bad argument"); return MDC_ERR_INVALID_ARG; }
    if (!check_size(w, h, "mdc_marker_read_patch")) return MDC_ERR_INVALID_ARG;
    Pf q[4];
    for (int k = 0; k < 4; ++k) q[k] = Pf{quad[2 * k], quad[2 * k + 1]};
    if (!warp_patch(grey, w, h, q, patch)) { mdc_set_error("mdc_marker_read_patch: singular perspective transform"); return MDC_ERR_INVALID_ARG; }
    std::vector<uint8_t> work(patch, patch + kWarp * kWarp);
    *id = read_id(work.data(), otsu_threshold, rotations);
    return MDC_OK;
}

extern "C" int mdc_marker_detect(const uint8_t* grey, const uint8_t* mask, int w, int h, mdc_marker* out, int capacity, int* count) {
    if (!grey || !mask || !count || capacity < 0 || (capacity > 0 && !out)) { mdc_set_error("mdc_marker_detect: bad argument"); return MDC_ERR_INVALID_ARG; }
    *count = 0;
    if (!check_size(w, h, "mdc_marker_detect")) return MDC_ERR_INVALID_ARG;
    std::vector<Candidate> cands;
    const int r = find_candidates(mask, w, h, &cands);
    if (r != MDC_OK) return r;
    std::vector<Marker> markers;
    uint8_t patch[kWarp * kWarp];
    for (Candidate& cand : cands) {                                       // markerdetector.cpp:166-191
        if (!warp_patch(grey, w, h, cand.c, patch)) continue;
        int rot = 0;
        const int id = read_id(patch, nullptr, &rot);
        if (id == -1) continue;
        refine_lines(cand);
        Marker m;
        m.id = id;
        std::copy(cand.c, cand.c + 4, m.c);
        std::rotate(m.c, m.c + 4 - rot, m.c + 4);
        markers.push_back(m);
    }
    std::sort(markers.begin(), markers.end(), [](const Marker& a, const Marker& b) { return a.id < b.id; });   // :218
    std::vector<char> remove(markers.size(), 0);
    for (int i = 0; i < static_cast<int>(markers.size()) - 1; ++i)                                                   // :221-228
        if (markers[i].id == markers[i + 1].id && !remove[i + 1]) {
            if (perimeter(markers[i].c) > perimeter(markers[i + 1].c)) remove[i + 1] = 1;
            else remove[i] = 1;
        }
    const int bx = static_cast<int>(0.025 * static_cast<float>(w)), by = static_cast<int>(0.025 * static_cast<float>(h));   // :232-243
    for (size_t i = 0; i < markers.size(); ++i)
        for (const Pf& p : markers[i].c)
            if (p.x < bx || p.y < by || p.x > w - bx || p.y > h - by) remove[i] = 1;
    int n = 0;
    for (size_t i = 0; i < markers.size(); ++i) {
        if (remove[i]) continue;
        if (n < capacity) {
            out[n].id = markers[i].id;
            for (int k = 0; k < 4; ++k) { out[n].corners[2 * k] = markers[i].c[k].x; out[n].corners[2 * k + 1] = markers[i].c[k].y; }
        }
        ++n;
    }
    *count = n;
    if (n > capacity) { mdc_set_error("mdc_marker_detect: %d markers, capacity %d", n, capacity); return MDC_ERR_INVALID_ARG; }
    return MDC_OK;
}

extern "C" int mdc_marker_homography(const float corners[8], double H[9]) {
    if (!corners || !H) { mdc_set_error("mdc_marker_homography: bad argument"); return MDC_ERR_INVALID_ARG; }
    static const double P[4][2] = {{-0.5, 0.5}, {0.5, 0.5}, {0.5, -0.5}, {-0.5, -0.5}};   // main_vignetteCalib.cpp:246-249
    double q[4][2], scale = 0;
    for (int i = 0; i < 4; ++i) {
        q[i][0] = corners[2 * i];
        q[i][1] = corners[2 * i + 1];
        if (!std::isfinite(q[i][0]) || !std::isfinite(q[i][1])) { mdc_set_error("mdc_marker_homography: corner %d is not finite", i); return MDC_ERR_INVALID_ARG; }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) scale = std::max(scale, std::hypot(q[i][0] - q[j][0], q[i][1] - q[j][1]));
    // no three corners on one line (that includes two equal corners): the homography would be singular
    for (int i = 0; i < 4; ++i) {
        const double* a = q[(i + 1) % 4];
        const double* b = q[(i + 2) % 4];
        const double* c = q[(i + 3) % 4];
        const double cross = (b[0] - a[0]) * (c[1] - a[1]) - (b[1] - a[1]) * (c[0] - a[0]);
        if (!(std::fabs(cross) > 1e-9 * scale * scale)) { mdc_set_error("mdc_marker_homography: degenerate quad (three corners on a line)"); return MDC_ERR_INVALID_ARG; }
    }
    double A[8][8] = {{0}}, b[8];
    for (int i = 0; i < 4; ++i) {
        const double X = P[i][0], Y = P[i][1], x = q[i][0], y = q[i][1];
        double* r0 = A[2 * i];
        double* r1 = A[2 * i + 1];
        r0[0] = X; r0[1] = Y; r0[2] = 1; r0[6] = -x * X; r0[7] = -x * Y;
        r1[3] = X; r1[4] = Y; r1[5] = 1; r1[6] = -y * X; r1[7] = -y * Y;
        b[2 * i] = x;
        b[2 * i + 1] = y;
    }
    for (int col = 0; col < 8; ++col) {                    // Gaussian elimination with partial pivoting
        int piv = col;
        for (int r = col + 1; r < 8; ++r)
            if (std::fabs(A[r][col]) > std::fabs(A[piv][col])) piv = r;
        if (!(std::fabs(A[piv][col]) > 1e-12 * std::max(1.0, scale))) { mdc_set_error("mdc_marker_homography: singular system"); return MDC_ERR_INVALID_ARG; }
        if (piv != col) {
            std::swap(A[piv], A[col]);
            std::swap(b[piv], b[col]);
        }
        for (int r = col + 1; r < 8; ++r) {
            const double f = A[r][col] / A[col][col];
            for (int k = col; k < 8; ++k) A[r][k] -= f * A[col][k];
            b[r] -= f * b[col];
        }
    }
    for (int r = 7; r >= 0; --r) {
        double s = b[r];
        for (int k = r + 1; k < 8; ++k) s -= A[r][k] * b[k];
        b[r] = s / A[r][r];
    }
    for (int i = 0; i < 8; ++i) H[i] = b[i];
    H[8] = 1;
    for (int i = 0; i < 9; ++i)
        if (!std::isfinite(H[i])) { mdc_set_error("mdc_marker_homography: no finite solution"); return MDC_ERR_INVALID_ARG; }
    return MDC_OK;
}
