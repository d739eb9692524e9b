// CPU harness of the GPU JPEG decoder's core (csrc/mdc_jpeg_entropy.cuh, compiled here by the host compiler): parse the header and split
// the scan like mdc_jpeg_decode_device, decode every restart segment with mdcj::mdc_jpeg_decode_segment (what kernel J1 runs), then
// transform every visible block with mdcj::idct_block (what J2 computes) and crop.  Each segment's bytes are copied into a heap block of
// exactly their size and decoded into a zeroed coefficient plane of its own, so AddressSanitizer sees any read outside [begin, end) and
// the harness sees any coefficient written outside the segment's own blocks.  Built and run by tests/test_jpeg_entropy_host.py.
//
// usage: jpeg_entropy_harness <list>   (one file path per line).  Prints per file:
//   <index> host=<0|1> core=<0|1> same=<0|1> | <host message> | <core message>
// same = both accepted with identical pixels, or both rejected with the same message.  Exit status 1 if a segment wrote outside its
// blocks.
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "mdc_internal.h"
#include "mdc_jpeg.h"

static std::string g_error;
void mdc_set_error(const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g_error = buf;
}

static const uint8_t kZigZag[64] = MDC_JPEG_ZIGZAG;
static bool g_wrote_outside = false;

static bool core_decode(const std::vector<uint8_t>& file, const std::string& name, std::vector<uint8_t>* px, std::string* msg) {
    static mdc_jpeg_header h;
    if (!mdc_jpeg_parse_header(file.data(), file.size(), name, &h)) { *msg = g_error; return false; }
    std::vector<mdc_jpeg_segment> segs;
    const bool complete = mdc_jpeg_split_segments(file.data(), file.size(), h, &segs);
    const size_t bw = static_cast<size_t>(h.blocks_w()), bh = static_cast<size_t>(h.blocks_h());
    std::vector<int32_t> coef(bw * bh * 64, 0), scratch(bw * bh * 64, 0);
    mdcj::SegmentFrame f;
    f.ncomp = h.ncomp; f.mcus_x = h.mcus_x; f.blocks_w = h.blocks_w(); f.qzz = h.qzz;
    for (int c = 0; c < 3; ++c) {
        const mdc_jpeg_component& comp = h.comp[c < h.ncomp ? c : 0];
        f.h[c] = comp.h; f.v[c] = comp.v; f.dc[c] = &h.dc[comp.td]; f.ac[c] = &h.ac[comp.ta];
    }
    for (size_t k = 0; k < segs.size(); ++k) {
        const mdc_jpeg_segment& s = segs[k];
        const size_t len = s.end - s.begin;
        uint8_t* bytes = static_cast<uint8_t*>(malloc(len ? len : 1));
        if (len) memcpy(bytes, file.data() + s.begin, len);
        std::fill(scratch.begin(), scratch.end(), 0);
        const int rc = mdcj::mdc_jpeg_decode_segment(bytes, bytes + len, f, s.first_mcu, s.n_mcus, scratch.data());
        free(bytes);
        // blocks of this segment's MCUs: the only slots it may have written
        std::vector<char> mine(bw * bh, 0);
        for (int m = s.first_mcu; m < s.first_mcu + s.n_mcus; ++m) {
            const int my = m / h.mcus_x, mx = m % h.mcus_x;
            for (int by = 0; by < h.yv; ++by)
                for (int bx = 0; bx < h.yh; ++bx) mine[(static_cast<size_t>(my) * h.yv + by) * bw + static_cast<size_t>(mx) * h.yh + bx] = 1;
        }
        for (size_t b = 0; b < bw * bh; ++b)
            for (int i = 0; i < 64; ++i) {
                const int32_t v = scratch[b * 64 + i];
                if (v == 0) continue;
                if (!mine[b]) g_wrote_outside = true;
                coef[b * 64 + i] = v;
            }
        if (rc != mdcj::kSegOk) {
            *msg = name + ": " + (rc == mdcj::kBlockBadDc ? "corrupt JPEG data (DC)" : rc == mdcj::kBlockBadAc ? "corrupt JPEG data (AC)" : "corrupt JPEG data (run past the block)");
            return false;
        }
    }
    if (!complete) { *msg = name + ": missing restart marker"; return false; }
    px->assign(static_cast<size_t>(h.width) * h.height, 0);
    int32_t natural[64];
    uint8_t tile[64];
    for (int by = 0; by < (h.height + 7) / 8; ++by)
        for (int bx = 0; bx < (h.width + 7) / 8; ++bx) {
            const int32_t* zz = &coef[(static_cast<size_t>(by) * bw + bx) * 64];
            for (int k = 0; k < 64; ++k) natural[kZigZag[k]] = zz[k];
            mdcj::idct_block(natural, tile, 8);
            for (int y = 0; y < 8 && by * 8 + y < h.height; ++y)
                for (int x = 0; x < 8 && bx * 8 + x < h.width; ++x) (*px)[static_cast<size_t>(by * 8 + y) * h.width + bx * 8 + x] = tile[y * 8 + x];
        }
    return true;
}

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: jpeg_entropy_harness <list>\n"); return 2; }
    std::ifstream list(argv[1]);
    std::string path;
    int index = 0;
    while (std::getline(list, path)) {
        std::ifstream f(path, std::ios::binary);
        const std::vector<uint8_t> file((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        mdc_gray_image img;
        g_error.clear();
        const bool host_ok = mdc_decode_jpeg_gray(file, "frame", &img);
        const std::string host_msg = host_ok ? "" : g_error;
        std::vector<uint8_t> px;
        std::string core_msg;
        const bool core_ok = core_decode(file, "frame", &px, &core_msg);
        const bool same = host_ok == core_ok && (host_ok ? px == img.px : host_msg == core_msg);
        printf("%d host=%d core=%d same=%d | %s | %s\n", index++, host_ok ? 1 : 0, core_ok ? 1 : 0, same ? 1 : 0, host_msg.c_str(), core_msg.c_str());
    }
    if (g_wrote_outside) { printf("a segment wrote coefficients outside its own blocks\n"); return 1; }
    return 0;
}
