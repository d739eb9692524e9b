// Baseline-JPEG encoding of single-channel 8-bit frames, to the bytes cv::imwrite(".jpg") writes (libjpeg's defaults for one component:
// JFIF APP0, one quantisation table scaled from T.81 Annex K, the standard luminance Huffman tables, the accurate integer forward DCT,
// no restart markers, no Huffman optimisation).  Written once for the host and the device like mdc_jpeg_entropy.cuh: MDC_HD is
// __host__ __device__ under nvcc and plain inline under a host compiler, so the kernels of mdc_jpeg_encode.cu and a CPU harness
// (tests/test_jpeg_encode_core.py) run the same per-block code.  tests/jpeg_encode_spec.py restates the rules in numpy.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

#include "mdc_jpeg_entropy.cuh"      // MDC_HD, MDC_JPEG_ZIGZAG

namespace mdcje {

constexpr int kHeaderBytes = 328;     // SOI, APP0, DQT, SOF0, DHT (DC), DHT (AC), SOS
constexpr int kMaxDcBits = 9 + 11;    // longest DC code (size 11) + 11 magnitude bits
constexpr int kMaxAcBits = 16 + 10;   // a 16-bit AC code with 10 magnitude bits

// T.81 Annex K, Table K.1 (natural order) and Tables K.3 / K.5 (code-length counts for lengths 1..16, then the symbols)
constexpr uint8_t kLumaQuant[64] = {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                                    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                                    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
constexpr uint8_t kDcBits[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
constexpr uint8_t kDcVals[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
constexpr uint8_t kAcBits[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
constexpr uint8_t kAcVals[162] = {
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32, 0x81,
    0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18,
    0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75,
    0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99,
    0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5,
    0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa};

// What the per-block code needs: the quantisation divisors (8 q[k], natural order: the transform's outputs are 8 times the DCT) and
// the Huffman codes by symbol (length 0 = no code).  Small enough to pass by value to a kernel.
struct EncTables {
    int32_t div[64];
    uint16_t dc_code[16];
    uint8_t dc_len[16];
    uint16_t ac_code[256];
    uint8_t ac_len[256];
};

// libjpeg's jpeg_quality_scaling + baseline jpeg_add_quant_table: natural order, every entry in 1..255
inline void quant_table(int quality, int32_t q[64]) {
    const int s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    for (int k = 0; k < 64; ++k) {
        const int32_t v = (kLumaQuant[k] * s + 50) / 100;
        q[k] = v < 1 ? 1 : (v > 255 ? 255 : v);
    }
}

// T.81 Annex C: canonical codes from the code-length counts
inline void canonical_codes(const uint8_t bits[16], const uint8_t* vals, uint16_t* code_of, uint8_t* len_of) {
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        for (int i = 0; i < bits[l - 1]; ++i, ++k, ++code) {
            code_of[vals[k]] = static_cast<uint16_t>(code);
            len_of[vals[k]] = static_cast<uint8_t>(l);
        }
        code <<= 1;
    }
}

inline void make_tables(int quality, EncTables* t) {
    memset(t, 0, sizeof *t);
    int32_t q[64];
    quant_table(quality, q);
    for (int k = 0; k < 64; ++k) t->div[k] = 8 * q[k];
    canonical_codes(kDcBits, kDcVals, t->dc_code, t->dc_len);
    canonical_codes(kAcBits, kAcVals, t->ac_code, t->ac_len);
}

// The 328 bytes in front of the entropy-coded data of a w x h frame (1 <= w, h <= 65535)
inline void write_header(int w, int h, int quality, uint8_t out[kHeaderBytes]) {
    static const uint8_t kZz[64] = MDC_JPEG_ZIGZAG;
    static const uint8_t kApp0[20] = {0xff, 0xd8, 0xff, 0xe0, 0x00, 0x10, 'J', 'F', 'I', 'F', 0x00, 0x01, 0x01, 0x00, 0x00, 0x01, 0x00, 0x01, 0x00, 0x00};
    int32_t q[64];
    quant_table(quality, q);
    uint8_t* p = out;
    memcpy(p, kApp0, sizeof kApp0); p += sizeof kApp0;
    const uint8_t dqt[5] = {0xff, 0xdb, 0x00, 0x43, 0x00};
    memcpy(p, dqt, 5); p += 5;
    for (int k = 0; k < 64; ++k) *p++ = static_cast<uint8_t>(q[kZz[k]]);
    const uint8_t sof[15] = {0xff, 0xc0, 0x00, 0x0b, 0x08, static_cast<uint8_t>(h >> 8), static_cast<uint8_t>(h), static_cast<uint8_t>(w >> 8),
                             static_cast<uint8_t>(w), 0x01, 0x01, 0x11, 0x00};
    memcpy(p, sof, 13); p += 13;
    const uint8_t dht_dc[5] = {0xff, 0xc4, 0x00, 2 + 1 + 16 + 12, 0x00};
    memcpy(p, dht_dc, 5); p += 5;
    memcpy(p, kDcBits, 16); p += 16;
    memcpy(p, kDcVals, 12); p += 12;
    const uint8_t dht_ac[5] = {0xff, 0xc4, 0x00, 2 + 1 + 16 + 162, 0x10};
    memcpy(p, dht_ac, 5); p += 5;
    memcpy(p, kAcBits, 16); p += 16;
    memcpy(p, kAcVals, 162); p += 162;
    const uint8_t sos[10] = {0xff, 0xda, 0x00, 0x08, 0x01, 0x01, 0x00, 0x00, 0x3f, 0x00};
    memcpy(p, sos, 10);
}

// Blocks of a w x h frame, and the most bits one block's code can take at any quality
inline size_t block_count(int w, int h) { return static_cast<size_t>((w + 7) / 8) * static_cast<size_t>((h + 7) / 8); }
constexpr int kMaxBlockBits = kMaxDcBits + 63 * kMaxAcBits;
// header, the worst-case scan twice over (every byte could be 0xFF and take a stuffed 0x00), EOI
inline size_t encode_bound(int w, int h) { return kHeaderBytes + 2 * ((block_count(w, h) * kMaxBlockBits + 7) / 8) + 2; }

// ---------------------------------------------------------------------------------------------------------- forward DCT
// The accurate integer method (13-bit constants, 2 extra bits between the passes), 32-bit arithmetic, round-half-up descaling.
// pass 1 (rows): in = samples minus 128, out scaled up by 2^2; pass 2 (columns): out = 8 x the DCT coefficient.
constexpr int kConstBits = 13, kPass1Bits = 2;
MDC_HD int32_t descale(int32_t x, int n) { return (x + (1 << (n - 1))) >> n; }
MDC_HD void fdct_1d(const int32_t d[8], int32_t o[8], bool pass1) {
    const int32_t t0 = d[0] + d[7], t7 = d[0] - d[7], t1 = d[1] + d[6], t6 = d[1] - d[6];
    const int32_t t2 = d[2] + d[5], t5 = d[2] - d[5], t3 = d[3] + d[4], t4 = d[3] - d[4];
    const int32_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    const int s = pass1 ? kConstBits - kPass1Bits : kConstBits + kPass1Bits;
    o[0] = pass1 ? (t10 + t11) * (1 << kPass1Bits) : descale(t10 + t11, kPass1Bits);
    o[4] = pass1 ? (t10 - t11) * (1 << kPass1Bits) : descale(t10 - t11, kPass1Bits);
    const int32_t z1e = (t12 + t13) * 4433;                           // FIX(0.541196100)
    o[2] = descale(z1e + t13 * 6270, s);                              // FIX(0.765366865)
    o[6] = descale(z1e - t12 * 15137, s);                             // FIX(1.847759065)
    const int32_t z5 = (t4 + t6 + t5 + t7) * 9633;                    // FIX(1.175875602)
    const int32_t z1 = (t4 + t7) * -7373, z2 = (t5 + t6) * -20995;    // FIX(0.899976223), FIX(2.562915447)
    const int32_t z3 = (t4 + t6) * -16069 + z5, z4 = (t5 + t7) * -3196 + z5;   // FIX(1.961570560), FIX(0.390180644)
    o[7] = descale(t4 * 2446 + z1 + z3, s);                           // FIX(0.298631336)
    o[5] = descale(t5 * 16819 + z2 + z4, s);                          // FIX(2.053119869)
    o[3] = descale(t6 * 25172 + z2 + z3, s);                          // FIX(3.072711026)
    o[1] = descale(t7 * 12299 + z1 + z4, s);                          // FIX(1.501321110)
}
// c: 8 x the DCT coefficient; d = 8 q[k].  Rounds half away from zero, as libjpeg's quantiser.
MDC_HD int16_t quantise(int32_t c, int32_t d) {
    const int32_t a = ((c < 0 ? -c : c) + (d >> 1)) / d;
    return static_cast<int16_t>(c < 0 ? -a : a);
}

MDC_HD int min_i(int a, int b) { return a < b ? a : b; }
// Samples of block (bx, by) of a frame with rows `pitch` bytes apart: the right edge repeats the last pixel of each row, the bottom
// edge the last row.  Row r of the block, minus 128.
MDC_HD void load_row(const uint8_t* frame, size_t pitch, int w, int h, int bx, int by, int r, int32_t d[8]) {
    const int y = min_i(by * 8 + r, h - 1);
    const uint8_t* row = frame + static_cast<size_t>(y) * pitch;
    for (int i = 0; i < 8; ++i) d[i] = static_cast<int32_t>(row[min_i(bx * 8 + i, w - 1)]) - 128;
}

// ---------------------------------------------------------------------------------------------------------- Huffman coding
// T.81 F.1.2.1: the size category of v, and the `size` low bits that follow its code (v, or v - 1 for v < 0)
MDC_HD int magnitude_size(int v) {
    const unsigned a = static_cast<unsigned>(v < 0 ? -v : v);
#if defined(__CUDA_ARCH__)
    return 32 - __clz(a);
#else
    return a ? 32 - __builtin_clz(a) : 0;
#endif
}
MDC_HD uint32_t magnitude_bits(int v, int size) { return static_cast<uint32_t>(v < 0 ? v - 1 : v) & ((1u << size) - 1u); }

// Walks a block's code in stream order: put(value, length) for every code-plus-magnitude token (length <= kMaxAcBits).  zz: the 64
// quantised coefficients in zig-zag order; pred: the previous block's quantised DC (0 for the first block of the scan).
template <class Put>
MDC_HD void code_block(const int16_t* zz, int pred, const EncTables& t, Put& put) {
    const int diff = zz[0] - pred;
    const int ds = magnitude_size(diff);
    put((static_cast<uint32_t>(t.dc_code[ds]) << ds) | magnitude_bits(diff, ds), t.dc_len[ds] + ds);
    int run = 0;
    for (int k = 1; k < 64; ++k) {
        const int v = zz[k];
        if (v == 0) { ++run; continue; }
        for (; run > 15; run -= 16) put(t.ac_code[0xf0], t.ac_len[0xf0]);       // ZRL
        const int s = magnitude_size(v), sym = (run << 4) | s;
        put((static_cast<uint32_t>(t.ac_code[sym]) << s) | magnitude_bits(v, s), t.ac_len[sym] + s);
        run = 0;
    }
    if (run > 0) put(t.ac_code[0x00], t.ac_len[0x00]);                          // EOB only when the block ends in zeros
}

struct CountBits {
    uint32_t n = 0;
    MDC_HD void operator()(uint32_t, int len) { n += static_cast<uint32_t>(len); }
};
// Bits of a block's code given its DC predictor
MDC_HD uint32_t block_bits(const int16_t* zz, int pred, const EncTables& t) {
    CountBits c;
    code_block(zz, pred, t, c);
    return c.n;
}

// Writes a run of bits starting at bit `pos` of a stream held in 32-bit words whose memory bytes are the stream's bytes (each word
// big-endian in bit order, so word i holds bytes 4i..4i+3).  The words the run touches must start out holding zero bits where the run
// goes; or_word(i, v) ORs v (bytes in memory order) into word i, so runs of neighbouring blocks may share a word.
template <class OrWord>
struct BitWriter {
    OrWord& or_word;
    uint64_t word;       // the word the pending bits go to
    uint64_t acc;        // its pending bits are the low n bits (n < 32 between calls; the first bits of a run's first word count as 0s)
    int n;
    MDC_HD BitWriter(OrWord& o, uint64_t pos) : or_word(o), word(pos >> 5), acc(0), n(static_cast<int>(pos & 31)) {}
    MDC_HD void operator()(uint32_t v, int len) {
        acc = (acc << len) | v;
        n += len;
        if (n >= 32) {
            n -= 32;
            or_word(word++, bswap(static_cast<uint32_t>(acc >> n)));
        }
    }
    MDC_HD void flush() {
        if (n > 0) or_word(word, bswap(static_cast<uint32_t>(acc << (32 - n))));
        n = 0;
    }
    MDC_HD static uint32_t bswap(uint32_t x) { return (x >> 24) | ((x >> 8) & 0xff00u) | ((x << 8) & 0xff0000u) | (x << 24); }
};

// Emits a block's code at bit `pos` (see BitWriter)
template <class OrWord>
MDC_HD void emit_block(const int16_t* zz, int pred, const EncTables& t, uint64_t pos, OrWord& or_word) {
    BitWriter<OrWord> bw(or_word, pos);
    code_block(zz, pred, t, bw);
    bw.flush();
}

// The 1-bits that pad a scan of `bits` bits to a whole byte, ORed in like a block's code
template <class OrWord>
MDC_HD void emit_padding(uint64_t bits, OrWord& or_word) {
    const int pad = static_cast<int>((8 - (bits & 7)) & 7);
    if (!pad) return;
    BitWriter<OrWord> bw(or_word, bits);
    bw((1u << pad) - 1u, pad);
    bw.flush();
}

// ---------------------------------------------------------------------------------------------------------- host encoder
// One frame, block after block on one thread: what the kernels compute in parallel, for the CPU harness.  out must hold
// encode_bound(w, h) bytes; returns the file's length.
inline size_t encode_frame_host(const uint8_t* frame, size_t pitch, int w, int h, int quality, uint8_t* out) {
    EncTables t;
    make_tables(quality, &t);
    static const uint8_t kZz[64] = MDC_JPEG_ZIGZAG;
    const int bw = (w + 7) / 8, bh = (h + 7) / 8;
    const size_t words = (block_count(w, h) * kMaxBlockBits + 31) / 32 + 1;
    uint32_t* scan = new uint32_t[words]();
    struct OrHost {
        uint32_t* w;
        void operator()(uint64_t i, uint32_t v) { w[i] |= v; }
    } sink{scan};
    uint64_t pos = 0;
    int pred = 0;
    for (int by = 0; by < bh; ++by)
        for (int bx = 0; bx < bw; ++bx) {
            int32_t ws[64], col[8], o[8];
            for (int r = 0; r < 8; ++r) {
                int32_t d[8];
                load_row(frame, pitch, w, h, bx, by, r, d);
                fdct_1d(d, ws + 8 * r, true);
            }
            int16_t nat[64], zz[64];
            for (int c = 0; c < 8; ++c) {
                for (int r = 0; r < 8; ++r) col[r] = ws[8 * r + c];
                fdct_1d(col, o, false);
                for (int r = 0; r < 8; ++r) nat[8 * r + c] = quantise(o[r], t.div[8 * r + c]);
            }
            for (int k = 0; k < 64; ++k) zz[k] = nat[kZz[k]];
            emit_block(zz, pred, t, pos, sink);
            pos += block_bits(zz, pred, t);
            pred = zz[0];
        }
    emit_padding(pos, sink);
    write_header(w, h, quality, out);
    const uint8_t* bytes = reinterpret_cast<const uint8_t*>(scan);
    size_t n = kHeaderBytes;
    for (uint64_t i = 0; i < (pos + 7) / 8; ++i) {
        out[n++] = bytes[i];
        if (bytes[i] == 0xff) out[n++] = 0x00;
    }
    out[n++] = 0xff;
    out[n++] = 0xd9;
    delete[] scan;
    return n;
}

}  // namespace mdcje
