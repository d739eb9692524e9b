// Baseline-JPEG entropy decoding of one restart segment, and the accurate-integer inverse DCT, written once for the host and the
// device: MDC_HD is __host__ __device__ (inlined) under nvcc and plain inline under a host compiler, so the same code runs in the GPU kernels of
// mdc_jpeg_gpu.cu (J1, J2), in the host decoder (mdc_jpeg.cpp, its scalar transform) and in a CPU harness that checks it under
// AddressSanitizer (tests/test_jpeg_entropy_host.py).
//
// Safety: mdc_jpeg_decode_segment reads only bytes in [begin, end) and writes only the coefficient slots of the luminance blocks of
// the MCUs it is given, whatever the bytes are.  Huffman tables come from HuffTable::build, which refuses over-subscribed code
// lengths, so every table look-up below stays inside its table.
#pragma once
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define MDC_HD __host__ __device__ __forceinline__
#else
#define MDC_HD inline
#endif

namespace mdcj {

constexpr int kLookBits = 9;      // Huffman codes up to this length are resolved by one table look-up
constexpr int kFastBits = 10;     // window of the combined code + magnitude look-up of the AC tables

// T.81 Figure A.6: natural (row-major) index of the k-th coefficient in stream order
#define MDC_JPEG_ZIGZAG {0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, \
                         35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63}

struct HuffTable {
    bool defined = false;
    uint8_t bits[17] = {0};
    uint8_t vals[256] = {0};
    // canonical decoding tables (T.81 Annex F.2.2.3) + a prefix table for the short codes
    int mincode[17], maxcode[18], valptr[17];
    uint16_t look[1 << kLookBits];      // (code length << 8) | symbol, 0 = longer than kLookBits
    // AC tables: a kFastBits-wide window resolves in one look-up every code that fits it TOGETHER with its magnitude bits, and the
    // two symbols without magnitude bits: entry = (value << 16) | (kind << 9) | (run << 5) | total bits consumed;
    // kind 0 = not covered (general path), 1 = coefficient, 2 = end of block, 3 = run of 16 zeros
    int32_t fast[1 << kFastBits];
    void build_fast() {
        memset(fast, 0, sizeof fast);
        int code = 0, k = 0;
        for (int l = 1; l <= 16; ++l) {
            for (int i = 0; i < bits[l]; ++i, ++code, ++k) {
                if (l > kFastBits) continue;
                const int run = vals[k] >> 4, mag = vals[k] & 15, spare = kFastBits - l;
                for (int suffix = 0; suffix < (1 << spare); ++suffix) {
                    int32_t e = 0;
                    if (mag == 0) {
                        e = ((run == 15 ? 3 : 2) << 9) | l;            // anything but ZRL ends the block, like the general path
                    } else if (mag <= spare) {
                        int v = suffix >> (spare - mag);                // the magnitude bits that follow the code
                        if (v < (1 << (mag - 1))) v += 1 - (1 << mag);  // T.81 F.2.2.1 EXTEND
                        e = (v * 65536) | (1 << 9) | (run << 5) | (l + mag);
                    }
                    fast[(code << spare) | suffix] = e;
                }
            }
            code <<= 1;
        }
    }
    // false = over-subscribed table (more codes of some length than the prefix code space has left; libjpeg's
    // JERR_BAD_HUFF_TABLE).  Must be checked before look[] / fast[] are filled: such a table would index past their end.
    bool build() {
        int code = 0, k = 0;
        memset(look, 0, sizeof look);
        for (int l = 1; l <= 16; ++l) {
            if (code + bits[l] > (1 << l)) return false;
            valptr[l] = k;
            mincode[l] = code;
            for (int i = 0; i < bits[l]; ++i, ++code, ++k)
                if (l <= kLookBits) {
                    const int first = code << (kLookBits - l), span = 1 << (kLookBits - l);
                    for (int j = 0; j < span; ++j) look[first + j] = static_cast<uint16_t>((l << 8) | vals[k]);
                }
            maxcode[l] = bits[l] ? code - 1 : -1;
            code <<= 1;
        }
        maxcode[17] = 0x7fffffff;
        return true;
    }
};

// ---------------------------------------------------------------------------------------------------------- entropy decoding
// Bit reader over [p, end): 0xFF 0x00 is a stuffed 0xFF; 0xFF followed by anything else, a 0xFF as the last byte, and everything
// from `end` on read as zero bits (the host decoder's rule for a marker or a truncated scan).
struct SegmentReader {
    const uint8_t* p;
    const uint8_t* end;
    uint64_t acc;          // the next bits of the stream, left-aligned
    int n;                 // how many of them are valid
    bool hit_marker;
    MDC_HD void fill() {
        // eight plain bytes ahead (no 0xFF among them): take as many whole bytes as fit at once.  The eight loads are independent,
        // so the GPU has one memory round trip per refill instead of one per byte.  Bits of a partly fitting next byte come along
        // below the counted ones; the next refill ORs the same byte over them (as the host decoder's reader does).
        if (!hit_marker && end - p >= 8) {
            uint64_t v = 0;
            bool ff = false;
            for (int i = 0; i < 8; ++i) { const uint64_t b = p[i]; ff |= b == 0xff; v = (v << 8) | b; }
            if (!ff) {
                const int bytes = (64 - n) >> 3;
                acc |= v >> n;
                p += bytes;
                n += 8 * bytes;
                return;
            }
        }
        while (n <= 56) {
            uint64_t b = 0;
            if (!hit_marker && p < end) {
                b = *p;
                if (b == 0xff) {
                    if (p + 1 < end && p[1] == 0x00) p += 2;
                    else { hit_marker = true; b = 0; }
                } else {
                    ++p;
                }
            }
            acc |= b << (56 - n);
            n += 8;
        }
    }
    MDC_HD int peek(int count) {                       // count in 1..25
        if (n < count) fill();
        return static_cast<int>(acc >> (64 - count));
    }
    MDC_HD void skip(int count) { acc <<= count; n -= count; }
    MDC_HD int bits(int count) {
        if (count == 0) return 0;
        const int v = peek(count);
        skip(count);
        return v;
    }
};

MDC_HD int decode_symbol(SegmentReader& br, const HuffTable& t) {
    const int look = t.look[br.peek(kLookBits)];
    if (look) { br.skip(look >> 8); return look & 0xff; }
    int l = kLookBits + 1;                             // longer code: canonical search from kLookBits + 1 bits on
    int code = br.peek(l);
    while (l <= 16 && code > t.maxcode[l]) { ++l; code = br.peek(l); }
    if (l > 16) return -1;
    br.skip(l);
    return t.vals[(t.valptr[l] + code - t.mincode[l]) & 255];      // < 256 for every table build() accepts
}
// T.81 F.2.2.1 EXTEND
MDC_HD int extend(int v, int t) { return (t && v < (1 << (t - 1))) ? v - (1 << t) + 1 : v; }

enum { kSegOk = 0, kBlockBadDc = 1, kBlockBadAc = 2, kBlockBadRun = 3 };

// One block: DC difference, then AC coefficients until end of block.  coef == nullptr for components that are only skipped
// (chroma): same bits consumed, nothing written.  Coefficients are stored dequantised in zig-zag (stream) order: coef[k] = v * q[k].
MDC_HD int decode_block(SegmentReader& br, const HuffTable& dct, const HuffTable& act, int& pred, int32_t* coef, const int32_t* qzz) {
    if (br.n < 32) br.fill();
    const int t = decode_symbol(br, dct);
    if (t < 0 || t > 15) return kBlockBadDc;
    // libjpeg stores coefficients as 16-bit JCOEF: the running DC value wraps there (only corrupt data gets that far)
    pred = static_cast<int16_t>(static_cast<uint32_t>(pred) + static_cast<uint32_t>(extend(br.bits(t), t)));
    if (coef) coef[0] = pred * qzz[0];             // |pred| <= 2^15, q <= 65535: fits int32
    for (int k = 1; k < 64;) {
        if (br.n < 32) br.fill();
        const int32_t fe = act.fast[br.acc >> (64 - kFastBits)];
        const int kind = (fe >> 9) & 3;
        if (kind == 1) {                       // code + magnitude in one look-up
            k += (fe >> 5) & 15;
            if (k > 63) return kBlockBadRun;
            br.skip(fe & 31);
            if (coef) coef[k] = (fe >> 16) * qzz[k];
            ++k;
            continue;
        }
        if (kind == 2) { br.skip(fe & 31); break; }
        if (kind == 3) { br.skip(fe & 31); k += 16; continue; }
        const int rs = decode_symbol(br, act);
        if (rs < 0) return kBlockBadAc;
        const int r = rs >> 4, sz = rs & 15;
        if (sz == 0) {
            if (r != 15) break;                // EOB
            k += 16;
            continue;
        }
        k += r;
        if (k > 63) return kBlockBadRun;
        const int v = extend(br.bits(sz), sz);
        if (coef) coef[k] = v * qzz[k];        // |v| < 2^15, q <= 65535: fits int32
        ++k;
    }
    return kSegOk;
}

// What a segment needs to know about its frame.  Luminance block (bx, by) of the padded plane has its 64 coefficients at
// coef + 64 * (by * blocks_w + bx).  For a single-component scan an MCU is one block (T.81 A.2.2); otherwise component c contributes
// h[c] x v[c] blocks per MCU, and only component 0 (luminance, which carries the maximum factors) is stored.
struct SegmentFrame {
    int ncomp, mcus_x, blocks_w;
    int h[3], v[3];
    const HuffTable* dc[3];
    const HuffTable* ac[3];
    const int32_t* qzz;          // luminance quantisation steps in zig-zag order
};

// Decode the MCUs [first_mcu, first_mcu + n_mcus) of one restart segment whose entropy-coded bytes are [begin, end); predictors start
// at zero.  The coefficient slots of those MCUs' luminance blocks must be zero on entry.  Returns kSegOk or the first error met.
MDC_HD int mdc_jpeg_decode_segment(const uint8_t* begin, const uint8_t* end, const SegmentFrame& f, int first_mcu, int n_mcus,
                                          int32_t* coef) {
    SegmentReader br{begin, end, 0, 0, false};
    int pred0 = 0, pred1 = 0, pred2 = 0;          // scalars, not an array: a dynamically indexed array would live in local memory on the GPU
    const bool single = f.ncomp == 1;
    const int yh = single ? 1 : f.h[0], yv = single ? 1 : f.v[0];
    for (int m = first_mcu; m < first_mcu + n_mcus; ++m) {
        const int my = m / f.mcus_x, mx = m - my * f.mcus_x;
        for (int c = 0; c < f.ncomp; ++c) {
            const int bh = single ? 1 : f.h[c], bv = single ? 1 : f.v[c];
            const HuffTable& dct = *f.dc[c];
            const HuffTable& act = *f.ac[c];
            int pred = c == 0 ? pred0 : (c == 1 ? pred1 : pred2);
            for (int by = 0; by < bv; ++by)
                for (int bx = 0; bx < bh; ++bx) {
                    int32_t* slot = nullptr;
                    if (c == 0) slot = coef + 64 * (static_cast<size_t>(my * yv + by) * f.blocks_w + static_cast<size_t>(mx) * yh + bx);
                    const int rc = decode_block(br, dct, act, pred, slot, f.qzz);
                    if (rc != kSegOk) return rc;
                }
            if (c == 0) pred0 = pred; else if (c == 1) pred1 = pred; else pred2 = pred;
        }
    }
    return kSegOk;
}

// ---------------------------------------------------------------------------------------------------------- inverse DCT
// Accurate integer method (13-bit constants, 2 guard bits between the passes).  Temporaries are 64-bit like libjpeg's (its JLONG is
// `long`), so no input — not even a corrupt one — can overflow.
typedef int64_t wide;
constexpr int kConstBits = 13, kPass1Bits = 2;
constexpr wide F_0_298631336 = 2446, F_0_390180644 = 3196, F_0_541196100 = 4433, F_0_765366865 = 6270, F_0_899976223 = 7373,
               F_1_175875602 = 9633, F_1_501321110 = 12299, F_1_847759065 = 15137, F_1_961570560 = 16069, F_2_053119869 = 16819,
               F_2_562915447 = 20995, F_3_072711026 = 25172;
MDC_HD wide descale(wide x, int n) { return (x + (wide(1) << (n - 1))) >> n; }      // arithmetic shift (floor), as in libjpeg
MDC_HD uint8_t clamp_sample(wide v) { v += 128; return static_cast<uint8_t>(v < 0 ? 0 : (v > 255 ? 255 : v)); }

struct Butterfly { wide e0, e1, e2, e3, o0, o1, o2, o3; };      // out[k] = e_k + o_(3-k), out[7-k] = e_k - o_(3-k)
MDC_HD Butterfly idct_1d(wide c0, wide c1, wide c2, wide c3, wide c4, wide c5, wide c6, wide c7) {
    Butterfly r;
    // even part
    wide z1 = (c2 + c6) * F_0_541196100;
    const wide t2 = z1 + c6 * (-F_1_847759065), t3 = z1 + c2 * F_0_765366865;
    const wide t0 = (c0 + c4) * (wide(1) << kConstBits), t1 = (c0 - c4) * (wide(1) << kConstBits);
    r.e0 = t0 + t3; r.e3 = t0 - t3; r.e1 = t1 + t2; r.e2 = t1 - t2;
    // odd part
    wide a0 = c7, a1 = c5, a2 = c3, a3 = c1;
    z1 = a0 + a3;
    wide z2 = a1 + a2, z3 = a0 + a2, z4 = a1 + a3;
    const wide z5 = (z3 + z4) * F_1_175875602;
    a0 *= F_0_298631336; a1 *= F_2_053119869; a2 *= F_3_072711026; a3 *= F_1_501321110;
    z1 *= -F_0_899976223; z2 *= -F_2_562915447; z3 *= -F_1_961570560; z4 *= -F_0_390180644;
    z3 += z5; z4 += z5;
    r.o0 = a0 + z1 + z3; r.o1 = a1 + z2 + z4; r.o2 = a2 + z2 + z3; r.o3 = a3 + z1 + z4;
    return r;
}

// Pass 1, column c: coef = dequantised coefficients in natural order -> ws[8 * r + c].  A column whose AC terms are all zero takes a
// shortcut that gives exactly what the full butterfly gives for it (dc << 2).
MDC_HD void idct_column(const int32_t* coef, int c, wide* ws) {
    if ((coef[8 + c] | coef[16 + c] | coef[24 + c] | coef[32 + c] | coef[40 + c] | coef[48 + c] | coef[56 + c]) == 0) {
        const wide v = wide(coef[c]) * (1 << kPass1Bits);
        ws[c] = ws[8 + c] = ws[16 + c] = ws[24 + c] = ws[32 + c] = ws[40 + c] = ws[48 + c] = ws[56 + c] = v;
        return;
    }
    const Butterfly b = idct_1d(coef[c], coef[8 + c], coef[16 + c], coef[24 + c], coef[32 + c], coef[40 + c], coef[48 + c], coef[56 + c]);
    const int s = kConstBits - kPass1Bits;
    ws[c] = descale(b.e0 + b.o3, s);       ws[56 + c] = descale(b.e0 - b.o3, s);
    ws[8 + c] = descale(b.e1 + b.o2, s);   ws[48 + c] = descale(b.e1 - b.o2, s);
    ws[16 + c] = descale(b.e2 + b.o1, s);  ws[40 + c] = descale(b.e2 - b.o1, s);
    ws[24 + c] = descale(b.e3 + b.o0, s);  ws[32 + c] = descale(b.e3 - b.o0, s);
}
// Pass 2, row r of ws -> o[0..7].  A row whose AC terms are all zero: every sample is (ws0 + 16) >> 5, what the butterfly gives.
MDC_HD void idct_row(const wide* ws, int r, uint8_t* o) {
    const wide* w = ws + 8 * r;
    if ((w[1] | w[2] | w[3] | w[4] | w[5] | w[6] | w[7]) == 0) {
        const uint8_t v = clamp_sample(descale(w[0], kPass1Bits + 3));
        for (int i = 0; i < 8; ++i) o[i] = v;
        return;
    }
    const Butterfly b = idct_1d(w[0], w[1], w[2], w[3], w[4], w[5], w[6], w[7]);
    const int s = kConstBits + kPass1Bits + 3;
    o[0] = clamp_sample(descale(b.e0 + b.o3, s));  o[7] = clamp_sample(descale(b.e0 - b.o3, s));
    o[1] = clamp_sample(descale(b.e1 + b.o2, s));  o[6] = clamp_sample(descale(b.e1 - b.o2, s));
    o[2] = clamp_sample(descale(b.e2 + b.o1, s));  o[5] = clamp_sample(descale(b.e2 - b.o1, s));
    o[3] = clamp_sample(descale(b.e3 + b.o0, s));  o[4] = clamp_sample(descale(b.e3 - b.o0, s));
}
// coef: dequantised coefficients in natural order; out: 8 rows of 8 samples, `stride` apart
MDC_HD void idct_block(const int32_t coef[64], uint8_t* out, size_t stride) {
    wide ws[64];
    for (int c = 0; c < 8; ++c) idct_column(coef, c, ws);
    for (int r = 0; r < 8; ++r) idct_row(ws, r, out + r * stride);
}

}  // namespace mdcj
