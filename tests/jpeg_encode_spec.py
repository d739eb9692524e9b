"""A numpy restatement of what cv::imwrite(".jpg") / cv2.imencode writes for a single-channel 8-bit image: libjpeg's baseline defaults
for one component (JFIF APP0, one 8-bit quantisation table scaled from the Annex K luminance table, the standard luminance Huffman
tables, the accurate integer forward DCT, no restart markers, no Huffman optimisation).  encode(img, q) must equal
cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, q]) byte for byte; csrc/mdc_jpeg_encode.cuh is checked against it.

The float path: cv2.imencode of a float32 image converts it with saturate_cast<uchar> first (conv_u8)."""
import numpy as np

# T.81 Annex K, Table K.1: luminance quantisation table, natural (row-major) order
ANNEX_K_LUMA = np.array([
    16, 11, 10, 16, 24, 40, 51, 61,
    12, 12, 14, 19, 26, 58, 60, 55,
    14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77,
    24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101,
    72, 92, 95, 98, 112, 100, 103, 99], dtype=np.int64)

# T.81 Figure A.6: natural index of the k-th coefficient in zig-zag order
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
                   35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55,
                   62, 63])

# T.81 Annex K.3, Tables K.3 and K.5: standard luminance DC and AC Huffman tables (code-length counts 1..16, symbols)
DC_BITS = [0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0]
DC_VALS = list(range(12))
AC_BITS = [0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d]
AC_VALS = [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5,
    0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
    0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa]

HEADER_BYTES = 328


def huffman_codes(bits, vals):
    """Canonical codes (T.81 Annex C): symbol -> (code, length)."""
    code_of, code, k = {}, 0, 0
    for length in range(1, 17):
        for _ in range(bits[length - 1]):
            code_of[vals[k]] = (code, length)
            code += 1
            k += 1
        code <<= 1
    return code_of


DC_CODES = huffman_codes(DC_BITS, DC_VALS)
AC_CODES = huffman_codes(AC_BITS, AC_VALS)


def quant_table(quality):
    """libjpeg's jpeg_quality_scaling + jpeg_add_quant_table (baseline): natural order, entries in 1..255."""
    q = min(max(int(quality), 1), 100)
    s = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((ANNEX_K_LUMA * s + 50) // 100, 1, 255)


def header(w, h, quality):
    """SOI, APP0 JFIF 1.01, DQT, SOF0, DHT (DC), DHT (AC), SOS: the 328 bytes in front of the entropy-coded data."""
    qt = quant_table(quality)
    out = bytearray(b"\xff\xd8")
    out += b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00"
    out += b"\xff\xdb\x00\x43\x00" + bytes(int(v) for v in qt[ZIGZAG])
    out += b"\xff\xc0\x00\x0b\x08" + bytes([h >> 8, h & 255, w >> 8, w & 255]) + b"\x01\x01\x11\x00"
    out += b"\xff\xc4" + (2 + 1 + 16 + len(DC_VALS)).to_bytes(2, "big") + b"\x00" + bytes(DC_BITS) + bytes(DC_VALS)
    out += b"\xff\xc4" + (2 + 1 + 16 + len(AC_VALS)).to_bytes(2, "big") + b"\x10" + bytes(AC_BITS) + bytes(AC_VALS)
    out += b"\xff\xda\x00\x08\x01\x01\x00\x00\x3f\x00"
    assert len(out) == HEADER_BYTES
    return bytes(out)


# jfdctint.c's accurate integer method: 13-bit constants, 2 extra bits of precision between the passes
CONST_BITS, PASS1_BITS = 13, 2
FIX = dict(F_0_298631336=2446, F_0_390180644=3196, F_0_541196100=4433, F_0_765366865=6270, F_0_899976223=7373, F_1_175875602=9633,
           F_1_501321110=12299, F_1_847759065=15137, F_1_961570560=16069, F_2_053119869=16819, F_2_562915447=20995, F_3_072711026=25172)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, pass1):
    """One 1-D pass over the last axis (8 values, int64 arrays), scaled as libjpeg's islow pass 1 (rows) or pass 2 (columns)."""
    F = FIX
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    s = CONST_BITS - PASS1_BITS if pass1 else CONST_BITS + PASS1_BITS
    o = np.empty_like(d)
    if pass1:
        o[..., 0] = (t10 + t11) << PASS1_BITS
        o[..., 4] = (t10 - t11) << PASS1_BITS
    else:
        o[..., 0] = _descale(t10 + t11, PASS1_BITS)
        o[..., 4] = _descale(t10 - t11, PASS1_BITS)
    z1 = (t12 + t13) * F["F_0_541196100"]
    o[..., 2] = _descale(z1 + t13 * F["F_0_765366865"], s)
    o[..., 6] = _descale(z1 - t12 * F["F_1_847759065"], s)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * F["F_1_175875602"]
    t4, t5, t6, t7 = t4 * F["F_0_298631336"], t5 * F["F_2_053119869"], t6 * F["F_3_072711026"], t7 * F["F_1_501321110"]
    z1, z2 = z1 * -F["F_0_899976223"], z2 * -F["F_2_562915447"]
    z3, z4 = z3 * -F["F_1_961570560"] + z5, z4 * -F["F_0_390180644"] + z5
    o[..., 7] = _descale(t4 + z1 + z3, s)
    o[..., 5] = _descale(t5 + z2 + z4, s)
    o[..., 3] = _descale(t6 + z2 + z3, s)
    o[..., 1] = _descale(t7 + z1 + z4, s)
    return o


def blocks(img):
    """Edge-padded 8x8 blocks in raster order: [n_blocks, 8, 8] int64 samples minus 128."""
    img = np.asarray(img, np.uint8)
    h, w = img.shape
    ph, pw = -(-h // 8) * 8, -(-w // 8) * 8
    p = np.pad(img, ((0, ph - h), (0, pw - w)), mode="edge").astype(np.int64) - 128
    return p.reshape(ph // 8, 8, pw // 8, 8).transpose(0, 2, 1, 3).reshape(-1, 8, 8)


def quantised_blocks(img, quality):
    """[n_blocks, 64] quantised coefficients in zig-zag order."""
    b = blocks(img)
    c = _fdct_1d(b, True)                                             # rows
    c = _fdct_1d(c.transpose(0, 2, 1), False).transpose(0, 2, 1)      # columns
    c = c.reshape(-1, 64)
    d = 8 * quant_table(quality)
    q = np.sign(c) * ((np.abs(c) + d // 2) // d)
    return q[:, ZIGZAG]


def magnitude(v):
    """(size category, the size low bits that follow the code) of T.81 F.1.2.1: v for v > 0, v - 1 (low bits) for v < 0."""
    v = np.asarray(v, np.int64)
    a = np.abs(v)
    size = np.zeros_like(a)
    nz = a > 0
    size[nz] = np.floor(np.log2(a[nz])).astype(np.int64) + 1
    bits = np.where(v < 0, v - 1, v) & ((np.int64(1) << size) - 1)
    return size, bits


def entropy_tokens(zz):
    """The scan's bits as (value, length) tokens in stream order, from [n_blocks, 64] zig-zag coefficients."""
    nb = zz.shape[0]
    dc = zz[:, 0]
    diff = dc - np.concatenate([[0], dc[:-1]])
    dsize, dbits = magnitude(diff)
    dcode = np.array([DC_CODES[s][0] for s in range(12)])[dsize]
    dlen = np.array([DC_CODES[s][1] for s in range(12)])[dsize]
    keys, vals, lens = [np.arange(nb) * 66 * 4], [(dcode << dsize) | dbits], [dlen + dsize]

    ac = zz[:, 1:]
    b, k = np.nonzero(ac)                                             # row-major: blocks in order, k increasing
    k = k + 1
    prev = np.zeros_like(k)
    same = np.zeros(b.size, bool)
    same[1:] = b[1:] == b[:-1]
    prev[same] = k[np.flatnonzero(same) - 1]
    run = k - prev - 1
    size, mbits = magnitude(ac[b, k - 1])
    sym = ((run & 15) << 4) | size
    ac_code = np.zeros(256, np.int64)
    ac_len = np.zeros(256, np.int64)
    for s, (c, l) in AC_CODES.items():
        ac_code[s], ac_len[s] = c, l
    nzrl = run >> 4
    keys.append((b * 66 + k) * 4 + nzrl)
    vals.append((ac_code[sym] << size) | mbits)
    lens.append(ac_len[sym] + size)
    for j in range(3):                                                # runs of 16 zeros in front of the coefficient
        m = nzrl > j
        keys.append((b[m] * 66 + k[m]) * 4 + j)
        vals.append(np.full(m.sum(), ac_code[0xf0]))
        lens.append(np.full(m.sum(), ac_len[0xf0]))
    last = np.zeros(nb, np.int64)
    last[b] = k                                                       # last nonzero index per block (0 if none)
    eob = last < 63
    keys.append(np.flatnonzero(eob) * 66 * 4 + 65 * 4)
    vals.append(np.full(eob.sum(), ac_code[0x00]))
    lens.append(np.full(eob.sum(), ac_len[0x00]))
    key = np.concatenate(keys)
    order = np.argsort(key, kind="stable")
    return np.concatenate(vals)[order], np.concatenate(lens)[order]


def pack(vals, lens):
    """Tokens MSB first, the last byte padded with 1-bits, then 0xFF bytes stuffed with 0x00."""
    total = int(lens.sum())
    pad = (-total) % 8
    vals = np.concatenate([vals, [(1 << pad) - 1]]) if pad else vals
    lens = np.concatenate([lens, [pad]]) if pad else lens
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    idx = np.repeat(np.arange(len(lens)), lens)
    j = np.arange(total + pad) - starts[idx]
    bitv = ((vals[idx] >> (lens[idx] - 1 - j)) & 1).astype(np.uint8)
    data = np.packbits(bitv)
    ff = np.flatnonzero(data == 0xFF)
    out = np.repeat(data, 1 + (data == 0xFF))
    out[ff + np.arange(ff.size) + 1] = 0                              # the i-th 0xFF has moved i bytes on
    return out.tobytes()


def encode(img, quality=95):
    """The file cv2.imencode('.jpg', img, [cv2.IMWRITE_JPEG_QUALITY, quality]) writes for a 2-D uint8 image."""
    img = np.asarray(img)
    assert img.ndim == 2 and img.dtype == np.uint8
    h, w = img.shape
    vals, lens = entropy_tokens(quantised_blocks(img, quality))
    return header(w, h, quality) + pack(vals, lens) + b"\xff\xd9"


def conv_u8(a):
    """cv::saturate_cast<uchar>(float) on x86-64 (what cv::imwrite applies to a CV_32F image): round half to even; NaN, +-inf and
    anything outside int32 become 0; the rest is clamped to [0, 255]."""
    a = np.asarray(a, np.float32)
    inside = (a >= -2.0 ** 31) & (a < 2.0 ** 31)
    with np.errstate(invalid="ignore"):
        r = np.where(inside, np.rint(a.astype(np.float64)), -2.0 ** 31)
    return np.clip(r, 0, 255).astype(np.uint8)


def encode_bound(w, h):
    """mdc_jpeg_encode_bound: header + twice (for stuffing) the worst-case scan + EOI.  A block's worst case is the longest DC code
    with size 11, then 63 coefficients each with the longest (AC code length + size) of the table."""
    dc = max(l for (_, l) in DC_CODES.values()) + 11
    ac = max(l + (s & 15) for s, (_, l) in AC_CODES.items())
    n_blocks = (-(-w // 8)) * (-(-h // 8))
    return HEADER_BYTES + 2 * -(-(n_blocks * (dc + 63 * ac)) // 8) + 2


# ------------------------------------------------------------------------------------------------ the test corpus
SIZES = [(1, 1), (1, 9), (9, 1), (7, 7), (8, 8), (9, 9), (17, 23), (333, 217), (640, 480), (1280, 1024)]
QUALITIES = [1, 10, 49, 50, 51, 75, 90, 95, 100]
KINDS = ["noise", "gradient", "zeros", "full", "checker", "blurred", "ffbytes"]


def frame(kind, w, h, seed=0):
    """A w x h uint8 frame of one corpus kind."""
    rng = np.random.default_rng(seed + 7919 * w + 104729 * h)
    y, x = np.mgrid[0:h, 0:w]
    if kind == "noise":
        return rng.integers(0, 256, (h, w), dtype=np.uint8)
    if kind == "gradient":
        return ((x * 3 + y * 5) & 255).astype(np.uint8)
    if kind == "zeros":
        return np.zeros((h, w), np.uint8)
    if kind == "full":
        return np.full((h, w), 255, np.uint8)
    if kind == "checker":
        return (((x + y) & 1) * 255).astype(np.uint8)
    if kind == "blurred":
        n = rng.integers(0, 256, (h + 4, w + 4)).astype(np.float64)
        k = np.array([1, 4, 6, 4, 1], np.float64) / 16
        n = sum(k[i] * n[i:i + h, :] for i in range(5))
        n = sum(k[i] * n[:, i:i + w] for i in range(5))
        return np.clip(np.rint(n), 0, 255).astype(np.uint8)
    if kind == "ffbytes":
        # flat blocks whose DC steps by +-1 between neighbours: DC codes of size 1 ("010" + one bit) and EOBs ("1010") alternate into
        # runs of 1-bits, with bright saturated rows that code as long strings of ones
        v = np.where(((x // 8) + (y // 8)) % 2 == 0, 128, 136).astype(np.uint8)
        v[(y % 16) < 3] = 255
        return v
    raise ValueError(kind)


def corpus(sizes=SIZES, qualities=QUALITIES, kinds=KINDS, big_qualities=(1, 50, 95, 100)):
    """(name, image, quality) of the corpus: every kind and quality at the small sizes; the frames of 640x480 and up at fewer qualities
    (their coding paths are the same ones, only longer)."""
    out = []
    for (w, h) in sizes:
        qs = qualities if w * h < 640 * 480 else [q for q in qualities if q in big_qualities]
        for kind in kinds:
            img = frame(kind, w, h)
            for q in qs:
                out.append((f"{kind}_{w}x{h}_q{q}", img, q))
    return out
