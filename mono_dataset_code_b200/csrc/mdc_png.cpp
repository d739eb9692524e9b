// PNG files of 8-bit or 16-bit grey or colour images, from the pixels cv::imwrite takes (BGR order, host-order 16-bit samples).
// The decoded pixels are what matters, not libpng's bytes: every row is stored unfiltered (filter type 0) and the stream is deflated
// at zlib level 1 with the RLE strategy, the fastest setting that still shrinks flat and saturated regions.
#include <zlib.h>

#include <cstdio>
#include <cstring>
#include <vector>

#include "mdc_internal.h"

namespace {

void be32(uint8_t* p, uint32_t v) { p[0] = v >> 24; p[1] = v >> 16; p[2] = v >> 8; p[3] = v; }

bool chunk(FILE* f, const char* tag, const uint8_t* data, size_t len) {
    uint8_t head[8], tail[4];
    be32(head, static_cast<uint32_t>(len));
    memcpy(head + 4, tag, 4);
    uLong crc = crc32(0L, head + 4, 4);
    if (len) crc = crc32(crc, data, static_cast<uInt>(len));
    be32(tail, static_cast<uint32_t>(crc));
    return fwrite(head, 1, 8, f) == 8 && (len == 0 || fwrite(data, 1, len, f) == len) && fwrite(tail, 1, 4, f) == 4;
}

}  // namespace

extern "C" int mdc_png_write(const char* path, const void* pixels, int w, int h, size_t row_bytes, int depth, int channels) {
    const size_t bpp = static_cast<size_t>(channels) * (depth / 8);          // bytes per pixel
    if (!path || !pixels || w < 1 || h < 1 || (depth != 8 && depth != 16) || (channels != 1 && channels != 3) ||
        row_bytes < static_cast<size_t>(w) * bpp || (static_cast<size_t>(w) * bpp + 1) * h > 0xffffffffu) {   // one deflate call
        mdc_set_error("mdc_png_write: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    const size_t stride = static_cast<size_t>(w) * bpp;
    std::vector<uint8_t> raw((stride + 1) * h);
    for (int y = 0; y < h; ++y) {
        const uint8_t* src = static_cast<const uint8_t*>(pixels) + y * row_bytes;
        uint8_t* px = &raw[y * (stride + 1)];
        *px++ = 0;                                                     // filter type 0: the row as it is
        if (depth == 8 && channels == 1) {                             // PNG order: RGB, big-endian samples
            memcpy(px, src, stride);
        } else if (depth == 8) {
            for (int x = 0; x < w; ++x) { px[3 * x] = src[3 * x + 2]; px[3 * x + 1] = src[3 * x + 1]; px[3 * x + 2] = src[3 * x]; }
        } else {
            const int n = w * channels;
            for (int i = 0; i < n; ++i) {
                const int from = channels == 3 ? i - i % 3 + 2 - i % 3 : i;
                uint16_t v;
                memcpy(&v, src + 2 * from, 2);
                px[2 * i] = static_cast<uint8_t>(v >> 8);
                px[2 * i + 1] = static_cast<uint8_t>(v);
            }
        }
    }
    z_stream z;
    memset(&z, 0, sizeof z);
    if (deflateInit2(&z, 1, Z_DEFLATED, 15, 8, Z_RLE) != Z_OK) { mdc_set_error("mdc_png_write: deflateInit2 failed"); return MDC_ERR_IO; }
    std::vector<uint8_t> idat(deflateBound(&z, raw.size()));
    z.next_in = raw.data();
    z.avail_in = static_cast<uInt>(raw.size());
    z.next_out = idat.data();
    z.avail_out = static_cast<uInt>(idat.size());
    const int zr = deflate(&z, Z_FINISH);
    idat.resize(z.total_out);
    deflateEnd(&z);
    if (zr != Z_STREAM_END) { mdc_set_error("mdc_png_write: deflate failed"); return MDC_ERR_IO; }

    FILE* f = fopen(path, "wb");
    if (!f) { mdc_set_error("mdc_png_write: cannot open %s", path); return MDC_ERR_IO; }
    static const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1a, '\n'};
    uint8_t ihdr[13];
    be32(ihdr, static_cast<uint32_t>(w));
    be32(ihdr + 4, static_cast<uint32_t>(h));
    ihdr[8] = static_cast<uint8_t>(depth);
    ihdr[9] = channels == 3 ? 2 : 0;                                   // colour type: RGB or grey
    ihdr[10] = ihdr[11] = ihdr[12] = 0;
    bool ok = fwrite(sig, 1, 8, f) == 8 && chunk(f, "IHDR", ihdr, 13) && chunk(f, "IDAT", idat.data(), idat.size()) && chunk(f, "IEND", nullptr, 0);
    ok = (fclose(f) == 0) && ok;
    if (!ok) { mdc_set_error("mdc_png_write: cannot write %s", path); return MDC_ERR_IO; }
    return MDC_OK;
}
