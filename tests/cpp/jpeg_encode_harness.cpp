// The JPEG encoder's per-block core (csrc/mdc_jpeg_encode.cuh) on the host, for tests/test_jpeg_encode_core.py.  Each line of the list
// file is "<raw frame> <w> <h> <row pitch> <quality> <out file>": the raw file holds h rows of `pitch` bytes.  The frame is encoded
// into a heap block of exactly mdc_jpeg_encode_bound(w, h) bytes (under AddressSanitizer a write past it stops the run) and written
// to the out file.  Prints "<out file> <size> <bound>" per frame.
#include <cstdio>
#include <fstream>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "mdc_jpeg_encode.cuh"

int main(int argc, char** argv) {
    if (argc != 2) { fprintf(stderr, "usage: jpeg_encode_harness <list>\n"); return 2; }
    std::ifstream list(argv[1]);
    std::string line;
    while (std::getline(list, line)) {
        std::istringstream in(line);
        std::string raw, out;
        int w, h, q;
        size_t pitch;
        if (!(in >> raw >> w >> h >> pitch >> q >> out)) continue;
        std::ifstream f(raw, std::ios::binary);
        std::vector<uint8_t> px((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
        if (px.size() != pitch * h) { fprintf(stderr, "%s: %zu bytes, expected %zu\n", raw.c_str(), px.size(), pitch * h); return 2; }
        const size_t bound = mdcje::encode_bound(w, h);
        uint8_t* buf = new uint8_t[bound];
        const size_t n = mdcje::encode_frame_host(px.data(), pitch, w, h, q, buf);
        std::ofstream o(out, std::ios::binary);
        o.write(reinterpret_cast<const char*>(buf), static_cast<std::streamsize>(n));
        delete[] buf;
        printf("%s %zu %zu\n", out.c_str(), n, bound);
    }
    return 0;
}
