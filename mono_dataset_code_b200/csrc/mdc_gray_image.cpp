// Greyscale image decode for the vignette map (the one image the hot path's INIT reads;
// the reference uses cv::imread(..., CV_LOAD_IMAGE_UNCHANGED), PhotometricUndistorter.cpp:120).
// Supported: PNG colour type 0 (grey), bit depth 8 or 16, non-interlaced — the format of
// the TUM monoVO vignette.png files — and binary PGM (P5).  Anything else is reported as
// unreadable, which the photometric model treats like the reference treats a wrong-size
// image (vignette stays invalid).  Frame decode (JPEG/zip) is out of scope (SURVEY.md §8f N1).
#include <zlib.h>

#include <cctype>
#include <cstdio>
#include <cstring>
#include <fstream>
#include <exception>
#include <iterator>

#include "mdc_internal.h"

namespace {

constexpr uint64_t kMaxImagePixels = 1ull << 28;

uint32_t be32(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }

int paeth(int a, int b, int c) {
    int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    if (pa <= pb && pa <= pc) return a;
    return pb <= pc ? b : c;
}

bool decode_png(const std::vector<uint8_t>& file, const std::string& path, mdc_gray_image* out) {
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
    if (file.size() < 8 + 25 || memcmp(file.data(), sig, 8) != 0) return false;
    size_t pos = 8;
    uint32_t width = 0, height = 0;
    int depth = 0, color = -1, interlace = 0;
    std::vector<uint8_t> idat;
    bool seen_end = false;
    while (pos + 12 <= file.size() && !seen_end) {
        const uint32_t len = be32(&file[pos]);
        const uint8_t* tag = &file[pos + 4];
        if (pos + 12 + static_cast<size_t>(len) > file.size()) { mdc_set_error("%s: truncated PNG chunk", path.c_str()); return false; }
        const uint8_t* body = &file[pos + 8];
        if (!memcmp(tag, "IHDR", 4) && len >= 13) {
            width = be32(body); height = be32(body + 4);
            depth = body[8]; color = body[9]; interlace = body[12];
        } else if (!memcmp(tag, "IDAT", 4)) {
            idat.insert(idat.end(), body, body + len);
        } else if (!memcmp(tag, "IEND", 4)) {
            seen_end = true;
        }
        pos += 12 + static_cast<size_t>(len);
    }
    if (color != 0 || (depth != 8 && depth != 16) || interlace != 0 || width == 0 || height == 0) {
        mdc_set_error("%s: unsupported PNG (need non-interlaced 8/16-bit greyscale; got colour type %d, depth %d, interlace %d)",
                      path.c_str(), color, depth, interlace);
        return false;
    }
    // untrusted dimensions: bound them before anything is sized from them (same 2^28-pixel cap as the JPEG path)
    if (width > 0x7fffffffu || height > 0x7fffffffu || static_cast<uint64_t>(width) * height > kMaxImagePixels) {
        mdc_set_error("%s: implausible PNG dimensions %u x %u", path.c_str(), width, height);
        return false;
    }
    if (idat.empty()) { mdc_set_error("%s: PNG without image data", path.c_str()); return false; }
    const size_t bpp = depth / 8, stride = static_cast<size_t>(width) * bpp;
    std::vector<uint8_t> raw((stride + 1) * height);
    uLongf raw_len = static_cast<uLongf>(raw.size());
    if (idat.empty() || uncompress(raw.data(), &raw_len, idat.data(), static_cast<uLong>(idat.size())) != Z_OK ||
        raw_len != raw.size()) {
        mdc_set_error("%s: PNG zlib stream corrupt", path.c_str());
        return false;
    }
    // undo the per-scanline filters in place (filter byte precedes each row)
    std::vector<uint8_t> img(stride * height);
    for (uint32_t y = 0; y < height; ++y) {
        const uint8_t ft = raw[(stride + 1) * y];
        const uint8_t* src = &raw[(stride + 1) * y + 1];
        uint8_t* cur = &img[stride * y];
        const uint8_t* up = y ? &img[stride * (y - 1)] : nullptr;
        for (size_t i = 0; i < stride; ++i) {
            const int a = i >= bpp ? cur[i - bpp] : 0;
            const int b = up ? up[i] : 0;
            const int c = (up && i >= bpp) ? up[i - bpp] : 0;
            int v = src[i];
            switch (ft) {
                case 0: break;
                case 1: v += a; break;
                case 2: v += b; break;
                case 3: v += (a + b) >> 1; break;
                case 4: v += paeth(a, b, c); break;
                default: mdc_set_error("%s: bad PNG filter type %d", path.c_str(), ft); return false;
            }
            cur[i] = static_cast<uint8_t>(v);
        }
    }
    out->rows = static_cast<int>(height);
    out->cols = static_cast<int>(width);
    out->depth = depth;
    if (depth == 8) out->px.swap(img);
    else {  // big-endian samples -> host uint16
        out->px.resize(img.size());
        uint16_t* dst = reinterpret_cast<uint16_t*>(out->px.data());
        for (size_t i = 0; i < static_cast<size_t>(width) * height; ++i) dst[i] = static_cast<uint16_t>((img[2 * i] << 8) | img[2 * i + 1]);
    }
    return true;
}

bool decode_pgm(const std::vector<uint8_t>& file, const std::string& path, mdc_gray_image* out) {
    if (file.size() < 7 || file[0] != 'P' || file[1] != '5') return false;
    size_t pos = 2;
    int vals[3], got = 0;
    while (got < 3 && pos < file.size()) {
        if (file[pos] == '#') { while (pos < file.size() && file[pos] != '\n') ++pos; continue; }
        if (isspace(file[pos])) { ++pos; continue; }
        long long v = 0; bool any = false;
        while (pos < file.size() && isdigit(file[pos])) {
            v = v * 10 + (file[pos] - '0'); ++pos; any = true;
            if (v > 0x7fffffffLL) { mdc_set_error("%s: malformed PGM header (number too large)", path.c_str()); return false; }
        }
        if (!any) { mdc_set_error("%s: malformed PGM header", path.c_str()); return false; }
        vals[got++] = static_cast<int>(v);
    }
    if (got != 3) { mdc_set_error("%s: malformed PGM header", path.c_str()); return false; }
    ++pos;  // the single whitespace after maxval
    const int w = vals[0], h = vals[1], maxv = vals[2];
    const size_t n = static_cast<size_t>(w) * h, bpp = maxv < 256 ? 1 : 2;
    if (w <= 0 || h <= 0 || maxv <= 0 || maxv > 65535 || n > kMaxImagePixels || pos + n * bpp > file.size()) { mdc_set_error("%s: truncated PGM", path.c_str()); return false; }
    out->rows = h; out->cols = w; out->depth = bpp == 1 ? 8 : 16;
    out->px.resize(n * bpp);
    if (bpp == 1) memcpy(out->px.data(), &file[pos], n);
    else {
        uint16_t* dst = reinterpret_cast<uint16_t*>(out->px.data());
        for (size_t i = 0; i < n; ++i) dst[i] = static_cast<uint16_t>((file[pos + 2 * i] << 8) | file[pos + 2 * i + 1]);
    }
    return true;
}

}  // namespace

// No exception leaves the decoders: allocation failures on hostile input become an ordinary "unreadable image" (the callers sit
// behind extern "C" entry points and std::async workers).
bool mdc_decode_gray_image(const std::vector<uint8_t>& file, const std::string& name, mdc_gray_image* out) {
    mdc_set_error("%s: not a PNG, PGM or JPEG image", name.c_str());
    try {
        if (file.size() >= 2 && file[0] == 'P' && file[1] == '5') return decode_pgm(file, name, out);
        if (file.size() >= 2 && file[0] == 0xff && file[1] == 0xd8) return mdc_decode_jpeg_gray(file, name, out);
        return decode_png(file, name, out);
    } catch (const std::exception& e) {
        mdc_set_error("%s: cannot decode (%s)", name.c_str(), e.what());
        return false;
    }
}

bool mdc_read_file(const std::string& path, std::vector<uint8_t>* file) {
    std::ifstream f(path.c_str(), std::ios::binary | std::ios::ate);
    if (!f.good()) { mdc_set_error("cannot open image %s", path.c_str()); return false; }
    const std::streamoff size = f.tellg();
    if (size < 0) { mdc_set_error("cannot read image %s", path.c_str()); return false; }
    file->resize(static_cast<size_t>(size));
    f.seekg(0);
    if (size > 0 && !f.read(reinterpret_cast<char*>(file->data()), size)) { mdc_set_error("cannot read image %s", path.c_str()); return false; }
    return true;
}

bool mdc_read_gray_image(const std::string& path, mdc_gray_image* out) {
    try {
        static thread_local std::vector<uint8_t> file;      // per-thread scratch, read in one go (see mdc_jpeg.cpp on why not per frame)
        return mdc_read_file(path, &file) && mdc_decode_gray_image(file, path, out);
    } catch (const std::exception& e) {
        mdc_set_error("%s: cannot read (%s)", path.c_str(), e.what());
        return false;
    }
}
