// Baseline JPEG -> 8-bit grey, for the frames of the published sequences (images.zip holds JPEGs; the reference reads them with
// cv::imread(..., CV_LOAD_IMAGE_GRAYSCALE), BenchmarkDatasetReader.h:252, :274).
//
// The image has no libjpeg to link, so this is a small decoder of its own, written to give the SAME BYTES as the decoder behind
// cv::imread (libjpeg / libjpeg-turbo with its default settings) for the files it accepts:
//   * baseline sequential DCT, Huffman coding, 8-bit samples (SOF0; SOF1 with 8-bit tables works the same), 1 or 3 components,
//     any sampling factors, restart intervals.  Progressive / arithmetic / 12-bit / lossless files are rejected (MDC_ERR_FORMAT).
//   * grey output = the luminance component only — what libjpeg does for out_color_space = JCS_GRAYSCALE: chroma blocks are
//     entropy-decoded (they share the bit stream) and dropped, so no upsampling or colour conversion is involved.
//   * inverse DCT = the "accurate integer" method (JDCT_ISLOW, libjpeg's default): the Loeffler-Ligtenberg-Moschytz
//     factorisation in 13-bit fixed point with 2 extra bits kept between the column and the row pass, as published in the
//     Independent JPEG Group's jidctint.c; libjpeg-turbo's SIMD versions are bit-exact with it.  Restated here from that
//     description (ITU-T T.81 for the entropy coding); tests/test_jpeg_decoder.py compares the result with cv2's decoder on
//     grey and colour files of several qualities, sampling modes and restart intervals, byte for byte.
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "mdc_internal.h"
#include "mdc_jpeg.h"
#if defined(__x86_64__) && defined(__GNUC__)
#include <immintrin.h>
#endif

namespace {

using mdcj::HuffTable;
using mdcj::kLookBits;
using mdcj::kFastBits;

struct BitReader {
    const uint8_t* p;
    const uint8_t* end;
    uint64_t acc = 0;      // the next bits of the stream, left-aligned
    int n = 0;             // how many of them are valid
    bool hit_marker = false;
    // entropy-coded bytes: 0xFF 0x00 is a stuffed 0xFF, 0xFF followed by anything else is a marker (zero bits from then on)
    void fill() {
        if (!hit_marker && end - p >= 8) {      // eight plain bytes ahead (no 0xFF among them): take as many whole bytes as fit at once
            uint64_t v;
            memcpy(&v, p, 8);
            const uint64_t x = ~v;
            if (!((x - 0x0101010101010101ull) & ~x & 0x8080808080808080ull)) {
                const int bytes = (64 - n) >> 3;
                // bits of a partly fitting next byte come along below the counted ones; the next fill ORs the same byte over them
                acc |= __builtin_bswap64(v) >> n;
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
    inline int peek(int count) {                       // count in 1..25
        if (n < count) fill();
        return static_cast<int>(acc >> (64 - count));
    }
    inline void skip(int count) { acc <<= count; n -= count; }
    inline int bits(int count) {
        if (count == 0) return 0;
        const int v = peek(count);
        skip(count);
        return v;
    }
    void reset() { acc = 0; n = 0; hit_marker = false; }
};

inline int decode_symbol(BitReader& br, const HuffTable& t) {
    const int look = t.look[br.peek(kLookBits)];
    if (look) { br.skip(look >> 8); return look & 0xff; }
    // longer code: canonical search from kLookBits + 1 bits on
    int l = kLookBits + 1;
    int code = br.peek(l);
    while (l <= 16 && code > t.maxcode[l]) { ++l; code = br.peek(l); }
    if (l > 16) return -1;
    br.skip(l);
    return t.vals[t.valptr[l] + code - t.mincode[l]];
}
// T.81 F.2.2.1 EXTEND
inline int extend(int v, int t) { return (t && v < (1 << (t - 1))) ? v - (1 << t) + 1 : v; }

const uint8_t kZigZag[64] = MDC_JPEG_ZIGZAG;

// One block: DC difference, then AC coefficients until end of block.  kStore = false for components that are only skipped (chroma of a
// colour file): same bits consumed, nothing written.  The bit reader is copied into a local so that its state lives in registers (a
// coefficient store could alias `n` otherwise); at least 32 bits are made available before every symbol — more than the longest
// code + magnitude — so nothing below checks the fill level again.  Returns < 0 on corrupt data, else 1 if an AC coefficient was stored.
enum { kBlockBadDc = -1, kBlockBadAc = -2, kBlockBadRun = -3 };
template <bool kStore>
inline int decode_block(BitReader& reader, const HuffTable& dct, const HuffTable& act, int& pred, int32_t* coef, const int32_t* qzz) {
    BitReader br = reader;
    if (br.n < 32) br.fill();
    const int t = decode_symbol(br, dct);
    if (t < 0 || t > 15) return kBlockBadDc;
    // libjpeg stores coefficients as 16-bit JCOEF: the running DC value wraps there (only corrupt data gets that far)
    pred = static_cast<int16_t>(static_cast<uint32_t>(pred) + static_cast<uint32_t>(extend(br.bits(t), t)));
    if (kStore) coef[0] = pred * qzz[0];
    int any_ac = 0;
    for (int k = 1; k < 64;) {
        if (br.n < 32) br.fill();
        const int32_t fe = act.fast[br.acc >> (64 - kFastBits)];
        const int kind = (fe >> 9) & 3;
        if (kind == 1) {                       // code + magnitude in one look-up
            k += (fe >> 5) & 15;
            if (k > 63) return kBlockBadRun;
            br.skip(fe & 31);
            if (kStore) { coef[kZigZag[k]] = (fe >> 16) * qzz[k]; any_ac = 1; }
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
        if (kStore) { coef[kZigZag[k]] = v * qzz[k]; any_ac = 1; }
        ++k;
    }
    reader = br;
    return any_ac;
}

// ---- inverse DCT, accurate integer method: the 64-bit scalar transform is mdcj::idct_block (mdc_jpeg_entropy.cuh), shared with the
// GPU decoder
using mdcj::wide; using mdcj::kConstBits; using mdcj::kPass1Bits; using mdcj::descale; using mdcj::clamp_sample; using mdcj::idct_block;
using mdcj::F_0_298631336; using mdcj::F_0_390180644; using mdcj::F_0_541196100; using mdcj::F_0_765366865; using mdcj::F_0_899976223;
using mdcj::F_1_175875602; using mdcj::F_1_501321110; using mdcj::F_1_847759065; using mdcj::F_1_961570560; using mdcj::F_2_053119869;
using mdcj::F_2_562915447; using mdcj::F_3_072711026;

// ---- the same transform with AVX2: eight columns (pass 1) resp. eight rows (pass 2) per instruction, 32-bit lanes.  Dequantised
// coefficients of a valid stream fit 16 bits, so no lane can overflow and the results equal the 64-bit scalar code bit for bit
// (and what libjpeg-turbo's SIMD returns); only corrupt streams can tell the two apart.  Chosen at run time (cpu_has_avx2).
#if defined(__x86_64__) && defined(__GNUC__)
#define MDC_JPEG_AVX2 1
#define AVX2_FN __attribute__((target("avx2"), always_inline)) inline
typedef __m256i V8;
AVX2_FN V8 vmul(V8 a, int c) { return _mm256_mullo_epi32(a, _mm256_set1_epi32(c)); }
AVX2_FN V8 vadd(V8 a, V8 b) { return _mm256_add_epi32(a, b); }
AVX2_FN V8 vsub(V8 a, V8 b) { return _mm256_sub_epi32(a, b); }
struct ButterflyV { V8 e0, e1, e2, e3, o0, o1, o2, o3; };
AVX2_FN ButterflyV idct_1d_v(V8 c0, V8 c1, V8 c2, V8 c3, V8 c4, V8 c5, V8 c6, V8 c7) {
    ButterflyV r;
    V8 z1 = vmul(vadd(c2, c6), static_cast<int>(F_0_541196100));
    const V8 t2 = vadd(z1, vmul(c6, -static_cast<int>(F_1_847759065))), t3 = vadd(z1, vmul(c2, static_cast<int>(F_0_765366865)));
    const V8 t0 = _mm256_slli_epi32(vadd(c0, c4), kConstBits), t1 = _mm256_slli_epi32(vsub(c0, c4), kConstBits);
    r.e0 = vadd(t0, t3); r.e3 = vsub(t0, t3); r.e1 = vadd(t1, t2); r.e2 = vsub(t1, t2);
    V8 a0 = c7, a1 = c5, a2 = c3, a3 = c1;
    z1 = vadd(a0, a3);
    V8 z2 = vadd(a1, a2), z3 = vadd(a0, a2), z4 = vadd(a1, a3);
    const V8 z5 = vmul(vadd(z3, z4), static_cast<int>(F_1_175875602));
    a0 = vmul(a0, static_cast<int>(F_0_298631336)); a1 = vmul(a1, static_cast<int>(F_2_053119869));
    a2 = vmul(a2, static_cast<int>(F_3_072711026)); a3 = vmul(a3, static_cast<int>(F_1_501321110));
    z1 = vmul(z1, -static_cast<int>(F_0_899976223)); z2 = vmul(z2, -static_cast<int>(F_2_562915447));
    z3 = vadd(vmul(z3, -static_cast<int>(F_1_961570560)), z5); z4 = vadd(vmul(z4, -static_cast<int>(F_0_390180644)), z5);
    r.o0 = vadd(vadd(a0, z1), z3); r.o1 = vadd(vadd(a1, z2), z4); r.o2 = vadd(vadd(a2, z2), z3); r.o3 = vadd(vadd(a3, z1), z4);
    return r;
}
template <int kShift> AVX2_FN V8 vdescale(V8 x) { return _mm256_srai_epi32(vadd(x, _mm256_set1_epi32(1 << (kShift - 1))), kShift); }
// rows r0..r7 of an 8x8 int32 matrix -> its columns
AVX2_FN void transpose8(V8& r0, V8& r1, V8& r2, V8& r3, V8& r4, V8& r5, V8& r6, V8& r7) {
    const V8 a0 = _mm256_unpacklo_epi32(r0, r1), a1 = _mm256_unpackhi_epi32(r0, r1), a2 = _mm256_unpacklo_epi32(r2, r3), a3 = _mm256_unpackhi_epi32(r2, r3);
    const V8 a4 = _mm256_unpacklo_epi32(r4, r5), a5 = _mm256_unpackhi_epi32(r4, r5), a6 = _mm256_unpacklo_epi32(r6, r7), a7 = _mm256_unpackhi_epi32(r6, r7);
    const V8 b0 = _mm256_unpacklo_epi64(a0, a2), b1 = _mm256_unpackhi_epi64(a0, a2), b2 = _mm256_unpacklo_epi64(a1, a3), b3 = _mm256_unpackhi_epi64(a1, a3);
    const V8 b4 = _mm256_unpacklo_epi64(a4, a6), b5 = _mm256_unpackhi_epi64(a4, a6), b6 = _mm256_unpacklo_epi64(a5, a7), b7 = _mm256_unpackhi_epi64(a5, a7);
    r0 = _mm256_permute2x128_si256(b0, b4, 0x20); r1 = _mm256_permute2x128_si256(b1, b5, 0x20);
    r2 = _mm256_permute2x128_si256(b2, b6, 0x20); r3 = _mm256_permute2x128_si256(b3, b7, 0x20);
    r4 = _mm256_permute2x128_si256(b0, b4, 0x31); r5 = _mm256_permute2x128_si256(b1, b5, 0x31);
    r6 = _mm256_permute2x128_si256(b2, b6, 0x31); r7 = _mm256_permute2x128_si256(b3, b7, 0x31);
}
__attribute__((target("avx2"))) void idct_block_avx2(const int32_t* coef, uint8_t* out, size_t stride) {
    const V8* c = reinterpret_cast<const V8*>(coef);      // 32-byte aligned by the caller; row r = lanes (columns) of one vector
    // pass 1: columns
    ButterflyV b = idct_1d_v(_mm256_load_si256(c), _mm256_load_si256(c + 1), _mm256_load_si256(c + 2), _mm256_load_si256(c + 3),
                             _mm256_load_si256(c + 4), _mm256_load_si256(c + 5), _mm256_load_si256(c + 6), _mm256_load_si256(c + 7));
    constexpr int s1 = kConstBits - kPass1Bits;
    V8 w0 = vdescale<s1>(vadd(b.e0, b.o3)), w7 = vdescale<s1>(vsub(b.e0, b.o3)), w1 = vdescale<s1>(vadd(b.e1, b.o2)), w6 = vdescale<s1>(vsub(b.e1, b.o2));
    V8 w2 = vdescale<s1>(vadd(b.e2, b.o1)), w5 = vdescale<s1>(vsub(b.e2, b.o1)), w3 = vdescale<s1>(vadd(b.e3, b.o0)), w4 = vdescale<s1>(vsub(b.e3, b.o0));
    // pass 2: rows — lanes become rows
    transpose8(w0, w1, w2, w3, w4, w5, w6, w7);
    b = idct_1d_v(w0, w1, w2, w3, w4, w5, w6, w7);
    constexpr int s2 = kConstBits + kPass1Bits + 3;
    const V8 bias = _mm256_set1_epi32(128);
    const V8 o0 = vadd(vdescale<s2>(vadd(b.e0, b.o3)), bias), o7 = vadd(vdescale<s2>(vsub(b.e0, b.o3)), bias);
    const V8 o1 = vadd(vdescale<s2>(vadd(b.e1, b.o2)), bias), o6 = vadd(vdescale<s2>(vsub(b.e1, b.o2)), bias);
    const V8 o2 = vadd(vdescale<s2>(vadd(b.e2, b.o1)), bias), o5 = vadd(vdescale<s2>(vsub(b.e2, b.o1)), bias);
    const V8 o3 = vadd(vdescale<s2>(vadd(b.e3, b.o0)), bias), o4 = vadd(vdescale<s2>(vsub(b.e3, b.o0)), bias);
    // o_k: lane = row, value = sample k of that row.  Saturating packs clamp to 0..255; per 128-bit half the bytes come out as
    // [k0: r0-3][k1: r0-3][k2: r0-3][k3: r0-3] and have to be regrouped by row
    const V8 p0123 = _mm256_packus_epi16(_mm256_packs_epi32(o0, o1), _mm256_packs_epi32(o2, o3));
    const V8 p4567 = _mm256_packus_epi16(_mm256_packs_epi32(o4, o5), _mm256_packs_epi32(o6, o7));
    const V8 by_row = _mm256_setr_epi8(0, 4, 8, 12, 1, 5, 9, 13, 2, 6, 10, 14, 3, 7, 11, 15, 0, 4, 8, 12, 1, 5, 9, 13, 2, 6, 10, 14, 3, 7, 11, 15);
    const V8 q0 = _mm256_shuffle_epi8(p0123, by_row), q1 = _mm256_shuffle_epi8(p4567, by_row);      // dword j of a half = samples 0-3 (q0) / 4-7 (q1) of row j
    const V8 rows01 = _mm256_unpacklo_epi32(q0, q1), rows23 = _mm256_unpackhi_epi32(q0, q1);         // low half: rows 0,1 / 2,3; high half: rows 4,5 / 6,7
    const __m128i lo01 = _mm256_castsi256_si128(rows01), lo23 = _mm256_castsi256_si128(rows23);
    const __m128i hi45 = _mm256_extracti128_si256(rows01, 1), hi67 = _mm256_extracti128_si256(rows23, 1);
    _mm_storel_epi64(reinterpret_cast<__m128i*>(out), lo01);
    _mm_storel_epi64(reinterpret_cast<__m128i*>(out + stride), _mm_unpackhi_epi64(lo01, lo01));
    _mm_storel_epi64(reinterpret_cast<__m128i*>(out + 2 * stride), lo23);
    _mm_storel_epi64(reinterpret_cast<__m128i*>(out + 3 * stride), _mm_unpackhi_epi64(lo23, lo23));
    _mm_storel_epi64(reinterpret_cast<__m128i*>(out + 4 * stride), hi45);
    _mm_storel_epi64(reinterpret_cast<__m128i*>(out + 5 * stride), _mm_unpackhi_epi64(hi45, hi45));
    _mm_storel_epi64(reinterpret_cast<__m128i*>(out + 6 * stride), hi67);
    _mm_storel_epi64(reinterpret_cast<__m128i*>(out + 7 * stride), _mm_unpackhi_epi64(hi67, hi67));
}
// MDC_JPEG_SCALAR=1 forces the scalar transform (tests compare both against OpenCV's decoder)
const bool cpu_has_avx2 = [] {
    __builtin_cpu_init();
    const char* e = getenv("MDC_JPEG_SCALAR");
    return __builtin_cpu_supports("avx2") != 0 && !(e && e[0] == '1');
}();
#endif

// a block whose AC coefficients are all zero: every sample is the rounded DC term (what both passes' shortcuts give)
inline void idct_dc_only(int32_t dc, uint8_t* out, size_t stride) {
    const uint8_t v = clamp_sample(descale(wide(dc) * (1 << kPass1Bits), kPass1Bits + 3));
    for (int r = 0; r < 8; ++r) memset(out + r * stride, v, 8);
}

inline int be16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

}  // namespace

bool mdc_jpeg_parse_header(const uint8_t* d, size_t n, const std::string& name, mdc_jpeg_header* h) {
    if (n < 4 || d[0] != 0xff || d[1] != 0xd8) { mdc_set_error("%s: not a JPEG file", name.c_str()); return false; }
    uint16_t quant[4][64];
    bool quant_defined[4] = {false, false, false, false};
    HuffTable* dc = h->dc;
    HuffTable* ac = h->ac;
    for (int t = 0; t < 4; ++t) dc[t].defined = ac[t].defined = false;
    mdc_jpeg_component* comps = h->comp;
    int ncomp = 0;
    int width = 0, height = 0, restart_interval = 0;
    bool have_frame = false;
    size_t pos = 2;
    auto fail = [&](const char* what) { mdc_set_error("%s: %s", name.c_str(), what); return false; };
    while (pos + 4 <= n) {
        if (d[pos] != 0xff) return fail("corrupt JPEG (marker expected)");
        while (pos < n && d[pos] == 0xff) ++pos;             // fill bytes
        if (pos >= n) break;
        const int marker = d[pos++];
        if (marker == 0xd8 || (marker >= 0xd0 && marker <= 0xd7) || marker == 0x01) continue;
        if (marker == 0xd9) break;
        if (pos + 2 > n) return fail("truncated JPEG");
        const int len = be16(d + pos);
        if (len < 2 || pos + len > n) return fail("truncated JPEG segment");
        const uint8_t* seg = d + pos + 2;
        const int seg_len = len - 2;
        if (marker == 0xdb) {                                  // DQT
            int i = 0;
            while (i < seg_len) {
                const int pq = seg[i] >> 4, tq = seg[i] & 15;
                ++i;
                if (tq > 3 || i + (pq ? 128 : 64) > seg_len) return fail("bad quantisation table");
                for (int k = 0; k < 64; ++k) {
                    quant[tq][kZigZag[k]] = static_cast<uint16_t>(pq ? be16(seg + i + 2 * k) : seg[i + k]);
                }
                i += pq ? 128 : 64;
                quant_defined[tq] = true;
            }
        } else if (marker == 0xc4) {                           // DHT
            int i = 0;
            while (i + 17 <= seg_len) {
                const int tc = seg[i] >> 4, th = seg[i] & 15;
                if (tc > 1 || th > 3) return fail("bad Huffman table id");
                HuffTable& t = tc ? ac[th] : dc[th];
                int total = 0;
                t.bits[0] = 0;
                for (int l = 1; l <= 16; ++l) { t.bits[l] = seg[i + l]; total += t.bits[l]; }
                i += 17;
                if (total > 256 || i + total > seg_len) return fail("bad Huffman table");
                memcpy(t.vals, seg + i, static_cast<size_t>(total));
                i += total;
                t.defined = t.build();
                if (!t.defined) return fail("bad Huffman table (over-subscribed code lengths)");
                if (tc) t.build_fast();
            }
        } else if (marker == 0xc0 || marker == 0xc1) {         // SOF0 / SOF1 (Huffman, sequential)
            if (seg_len < 6) return fail("bad frame header");
            if (seg[0] != 8) return fail("only 8-bit JPEG samples are supported");
            height = be16(seg + 1);
            width = be16(seg + 3);
            const int nc = seg[5];
            if ((nc != 1 && nc != 3) || seg_len < 6 + 3 * nc || width < 1 || height < 1) return fail("unsupported JPEG frame (components / size)");
            if (static_cast<long long>(width) * height > (1LL << 28)) return fail("JPEG frame larger than 2^28 pixels");
            ncomp = nc;
            for (int c = 0; c < nc; ++c) {
                comps[c] = mdc_jpeg_component();
                comps[c].id = seg[6 + 3 * c];
                comps[c].h = seg[7 + 3 * c] >> 4;
                comps[c].v = seg[7 + 3 * c] & 15;
                comps[c].tq = seg[8 + 3 * c];
                if (comps[c].h < 1 || comps[c].h > 4 || comps[c].v < 1 || comps[c].v > 4 || comps[c].tq > 3) return fail("bad component description");
            }
            have_frame = true;
        } else if (marker == 0xc2 || (marker >= 0xc3 && marker <= 0xcf && marker != 0xc4 && marker != 0xc8 && marker != 0xcc)) {
            return fail("progressive / lossless / arithmetic-coded JPEG is not supported (baseline only)");
        } else if (marker == 0xdd) {                           // DRI
            if (seg_len < 2) return fail("bad restart interval");
            restart_interval = be16(seg);
        } else if (marker == 0xda) {                           // SOS: the one scan of a baseline file
            if (!have_frame) return fail("scan before frame header");
            if (seg_len < 1) return fail("bad scan header");
            const int ns = seg[0];
            if (ns != ncomp || seg_len < 1 + 2 * ns + 3) return fail("non-interleaved multi-scan JPEG is not supported");
            for (int k = 0; k < ns; ++k) {
                const int cid = seg[1 + 2 * k];
                bool found = false;
                for (int c = 0; c < ncomp; ++c)
                    if (comps[c].id == cid) { comps[c].td = seg[2 + 2 * k] >> 4; comps[c].ta = seg[2 + 2 * k] & 15; found = true; }
                if (!found) return fail("scan names an unknown component");
            }
            pos += static_cast<size_t>(len);
            int hmax = 1, vmax = 1;
            for (int c = 0; c < ncomp; ++c) { hmax = std::max(hmax, comps[c].h); vmax = std::max(vmax, comps[c].v); }
            const mdc_jpeg_component& Y = comps[0];
            if (!quant_defined[Y.tq]) return fail("missing quantisation table");
            for (int c = 0; c < ncomp; ++c)
                if (comps[c].td > 3 || comps[c].ta > 3 || !dc[comps[c].td].defined || !ac[comps[c].ta].defined) return fail("missing Huffman table");
            const bool single = ncomp == 1;
            // a single-component scan is not interleaved: its MCU is one block whatever the sampling factors say (T.81 A.2.2)
            const int mcu_w = single ? 8 : 8 * hmax, mcu_h = single ? 8 : 8 * vmax;
            // luminance plane padded to whole blocks; for subsampled colour files Y has h x v blocks per MCU at full resolution
            // only if Y carries the maximum factors (always the case for files written by libjpeg/OpenCV); otherwise Y itself
            // is subsampled and a grey read would need upsampling, which is not supported
            if (!single && (Y.h != hmax || Y.v != vmax)) return fail("JPEG with a subsampled luminance component is not supported");
            h->width = width; h->height = height; h->ncomp = ncomp; h->restart_interval = restart_interval;
            h->mcus_x = (width + mcu_w - 1) / mcu_w;
            h->mcus_y = (height + mcu_h - 1) / mcu_h;
            h->yh = single ? 1 : Y.h;
            h->yv = single ? 1 : Y.v;
            for (int k = 0; k < 64; ++k) h->qzz[k] = quant[Y.tq][kZigZag[k]];
            h->scan_begin = pos;
            return true;
        }
        pos += static_cast<size_t>(len);
    }
    return fail("JPEG without image data");
}

// The host decoder's restart walk (mdc_decode_jpeg_gray): after an interval it searches for FF D0..D7 from the byte its reader
// stopped at.  That reader never passes the first marker after the interval's start, and no FF D0..D7 lies in front of that marker
// (an FF inside the interval is stuffed, FF 00), so searching from the interval's start finds the same marker.
bool mdc_jpeg_split_segments(const uint8_t* d, size_t n, const mdc_jpeg_header& h, std::vector<mdc_jpeg_segment>* segs) {
    segs->clear();
    const int total = h.mcus_x * h.mcus_y;
    const int per = h.restart_interval ? h.restart_interval : total;
    size_t begin = h.scan_begin;
    for (int first = 0; first < total; first += per) {
        if (first > 0) {
            size_t q = begin;
            while (q + 1 < n && !(d[q] == 0xff && d[q + 1] >= 0xd0 && d[q + 1] <= 0xd7)) ++q;
            if (q + 1 >= n) return false;
            begin = q + 2;
        }
        size_t end = begin;                   // the first marker: an FF not followed by 00 (an FF as the last byte counts as one)
        while (end < n && !(d[end] == 0xff && !(end + 1 < n && d[end + 1] == 0x00))) end += d[end] == 0xff ? 2 : 1;
        segs->push_back(mdc_jpeg_segment{begin, end, first, std::min(per, total - first)});
    }
    return true;
}

bool mdc_decode_jpeg_gray(const std::vector<uint8_t>& file, const std::string& name, mdc_gray_image* out) {
    const uint8_t* d = file.data();
    const size_t n = file.size();
    static thread_local mdc_jpeg_header hdr;      // 46 KB of Huffman tables: not on the decode threads' stacks
    if (!mdc_jpeg_parse_header(d, n, name, &hdr)) return false;
    const mdc_jpeg_header& h = hdr;
    auto fail = [&](const char* what) { mdc_set_error("%s: %s", name.c_str(), what); return false; };
    const int width = h.width, height = h.height, restart_interval = h.restart_interval;
    const int mcus_x = h.mcus_x, mcus_y = h.mcus_y, yh = h.yh, yv = h.yv;
    const bool single = h.ncomp == 1;
    int pred[3] = {0, 0, 0};
    const size_t pw = static_cast<size_t>(mcus_x) * yh * 8, ph = static_cast<size_t>(mcus_y) * yv * 8;
    // per-thread scratch, reused from frame to frame: a fresh 2 MB vector per frame means mmap + page faults + munmap on
    // every decode, and with dozens of decode threads those serialise on the process's address-space lock
    // When the width is a whole number of blocks the padded plane is the image plus spare rows: decode straight into the
    // result and cut the spare rows off afterwards (one 2 MB copy less per frame).
    static thread_local std::vector<uint8_t> scratch_plane;
    const bool in_place = pw == static_cast<size_t>(width);
    std::vector<uint8_t>& plane = in_place ? out->px : scratch_plane;
    plane.resize(pw * ph);      // every block of the padded plane is written by the loop below
    BitReader br{d + h.scan_begin, d + n};
    alignas(32) int32_t coef[64] = {0};      // all zero between blocks: a block clears what it wrote
    const int32_t* qzz = h.qzz;              // luminance quantisation steps in zig-zag (= stream) order
    int until_restart = restart_interval;
    for (int my = 0; my < mcus_y; ++my)
        for (int mx = 0; mx < mcus_x; ++mx) {
            if (restart_interval && until_restart == 0) {
                // byte-align, expect RSTn, reset predictors
                const uint8_t* q = br.p;
                while (q + 1 < br.end && !(q[0] == 0xff && q[1] >= 0xd0 && q[1] <= 0xd7)) ++q;
                if (q + 1 >= br.end) return fail("missing restart marker");
                br.p = q + 2;
                br.reset();
                pred[0] = pred[1] = pred[2] = 0;
                until_restart = restart_interval;
            }
            for (int c = 0; c < h.ncomp; ++c) {
                const mdc_jpeg_component& comp = h.comp[c];
                const int bh = single ? 1 : comp.h, bv = single ? 1 : comp.v;
                for (int by = 0; by < bv; ++by)
                    for (int bx = 0; bx < bh; ++bx) {
                        const int rc = c == 0 ? decode_block<true>(br, h.dc[comp.td], h.ac[comp.ta], pred[c], coef, qzz)
                                              : decode_block<false>(br, h.dc[comp.td], h.ac[comp.ta], pred[c], nullptr, qzz);
                        if (rc < 0) return fail(rc == kBlockBadDc ? "corrupt JPEG data (DC)" : rc == kBlockBadAc ? "corrupt JPEG data (AC)" : "corrupt JPEG data (run past the block)");
                        const bool any_ac = rc != 0;
                        if (c == 0) {
                            const size_t x0 = (static_cast<size_t>(mx) * yh + bx) * 8, y0 = (static_cast<size_t>(my) * yv + by) * 8;
                            uint8_t* dst = plane.data() + y0 * pw + x0;
                            if (!any_ac) {
                                idct_dc_only(coef[0], dst, pw);
                                coef[0] = 0;
                            } else {
#ifdef MDC_JPEG_AVX2
                                if (cpu_has_avx2) idct_block_avx2(coef, dst, pw);
                                else
#endif
                                    idct_block(coef, dst, pw);
                                memset(coef, 0, sizeof coef);
                            }
                        }
                    }
            }
            if (restart_interval) --until_restart;
        }
    out->rows = height; out->cols = width; out->depth = 8;
    out->px.resize(static_cast<size_t>(width) * height);
    if (!in_place)
        for (int y = 0; y < height; ++y) memcpy(out->px.data() + static_cast<size_t>(y) * width, plane.data() + static_cast<size_t>(y) * pw, static_cast<size_t>(width));
    return true;
}
