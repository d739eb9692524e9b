// Sanitizer fuzz of the host marker detector (csrc/mdc_marker.cpp): random masks, adversarial ones (checkerboards, edges set,
// nested squares, single pixels, lines) and zero, negative or huge sizes go through mdc_marker_detect and its stages; the only thing
// checked is that the process survives under -fsanitize=address,undefined.  Built and run by tests/test_marker_detect.py.
// usage: marker_fuzz <rounds>
#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "mdc_internal.h"

void mdc_set_error(const char*, ...) {}

int main(int argc, char** argv) {
    if (argc < 2) { fprintf(stderr, "usage: marker_fuzz <rounds>\n"); return 2; }
    const int rounds = atoi(argv[1]);
    std::mt19937 rng(4321);
    mdc_marker out[8];
    int found = 0;
    for (int r = 0; r < rounds; ++r) {
        const int w = 1 + static_cast<int>(rng() % (r % 5 == 0 ? 400 : 48)), h = 1 + static_cast<int>(rng() % (r % 5 == 0 ? 300 : 48));
        std::vector<uint8_t> mask(static_cast<size_t>(w) * h), grey(mask.size());
        for (size_t i = 0; i < mask.size(); ++i) grey[i] = static_cast<uint8_t>(rng());
        const int kind = r % 6;
        for (int y = 0; y < h; ++y)
            for (int x = 0; x < w; ++x) {
                uint8_t v;
                switch (kind) {
                    case 0: v = (rng() & 1) ? 255 : 0; break;                                   // noise
                    case 1: v = ((x + y) & 1) ? 255 : 0; break;                                 // 1-pixel checkerboard
                    case 2: v = (x == 0 || y == 0 || x == w - 1 || y == h - 1) ? 255 : 0; break;   // edges only
                    case 3: v = ((std::min(std::min(x, y), std::min(w - 1 - x, h - 1 - y)) / 3) & 1) ? 255 : 0; break;   // nested squares
                    case 4: v = (x % 7 == 3 || y % 5 == 2) ? 255 : 0; break;                    // lines
                    default: v = (rng() % 97 == 0) ? 255 : 0;                                   // single pixels
                }
                mask[static_cast<size_t>(y) * w + x] = v;
                if (kind == 3) grey[static_cast<size_t>(y) * w + x] = v ? 10 : 240;
            }
        int count = 0;
        mdc_marker_detect(grey.data(), mask.data(), w, h, out, 8, &count);
        found += count;
        float quads[8 * 16];
        mdc_marker_candidates(mask.data(), w, h, quads, 16, &count);
        int nc = 0;
        size_t np_ = 0;
        mdc_marker_contours(mask.data(), w, h, nullptr, 0, nullptr, 0, &nc, &np_);
        uint8_t patch[56 * 56];
        int t, id, rot;
        const float quad[8] = {static_cast<float>(rng() % 600) - 100, static_cast<float>(rng() % 600) - 100, static_cast<float>(rng() % 600),
                               static_cast<float>(rng() % 600), static_cast<float>(rng() % 600), 1e30f, -1e30f, static_cast<float>(rng() % 9)};
        mdc_marker_read_patch(grey.data(), w, h, quad, patch, &t, &id, &rot);
        double H[9];
        mdc_marker_homography(quad, H);
    }
    const int sizes[][2] = {{0, 0}, {0, 5}, {5, 0}, {-3, 7}, {1 << 16, 1 << 13}, {1 << 30, 1 << 30}, {-2147483647 - 1, -1}};
    uint8_t one = 255;
    int count = 0;
    for (const auto& s : sizes) mdc_marker_detect(&one, &one, s[0], s[1], out, 8, &count);
    printf("%d rounds, %d markers\n", rounds, found);
    return 0;
}
