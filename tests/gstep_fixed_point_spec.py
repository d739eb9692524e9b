"""The G-step's fixed-point summation (DESIGN.md §4 N2) written out in numpy / Python integers — the specification the CUDA kernels are
compared with bit for bit (tests/test_gpu_parity.py, tests/test_response_calib_scale.py) and the stand-in the world-size-2 gloo test
drives through the sharded host loop (tests/test_sharding_gloo.py).  Test infrastructure.

  scale_words(E, t)                 -> [bits(max finite |E|), bits(max finite |t|), 1 if a t is not finite else 0, 0]   (ranks: elementwise MAX)
  accumulate(data, t, E, words)     -> limbs int64[768], special float64[256], counts int64[256]                         (ranks: SUM)
  finish(words, limbs, special, n)  -> G float64[256]  (sum / count, gaps extrapolated as in main_responseCalib.cpp:300-304)

Every product E[k]*t[i] is rounded to fp64 as the reference rounds it, scaled by 2^s (exactly, or below 2^-1022 where it rounds to
integer 0 anyway) and rounded to an integer; the integers are summed exactly.  Non-finite products are summed in fp64 on the side
(only ±inf and NaN reach that sum, so its value does not depend on the order).  Word 2 (a non-finite t) tells the kernels to
range-check every sample of the pass; the result does not depend on it.
"""
import math

import numpy as np

LIMIT = float(2 ** 48)          # scaled products stay below it
LIMB_BITS = 43
MIN_S = 48 - 1024               # every finite product is below 2^1024
HALF_BITS = 24                  # accumulate(): a scaled product (|v| < 2^48) as two halves whose bincount sums stay exact
CHUNK = 1 << 24                 # samples per bincount: 2^24 halves below 2^24 sum to less than 2^48 < 2^53


def _bits(x):
    return int(np.float64(x).view(np.int64))


def _from_bits(b):
    return float(np.int64(b).view(np.float64))


def scale_words(E, t):
    e = np.abs(E[np.isfinite(E)])
    tt = np.abs(t[np.isfinite(t)])
    return np.array([_bits(e.max()) if e.size else 0, _bits(tt.max()) if tt.size else 0, int(not np.all(np.isfinite(t))), 0], np.int64)


def exponent(words):
    """s with |E*t| * 2^s < 2^48 for every finite product: 47 - ilogb(max|E| * max|t|), the product's exponent taken from the
    factors' exponents and the product of their mantissas (so that it exists when the product overflows or underflows), and at
    least 48 - 1024."""
    e, t = _from_bits(words[0]), _from_bits(words[1])
    if not (e > 0.0 and t > 0.0):
        return 0
    ee, et = math.frexp(e)[1] - 1, math.frexp(t)[1] - 1          # ilogb, subnormals included
    k = math.frexp(math.ldexp(e, -ee) * math.ldexp(t, -et))[1] - 1
    return max(MIN_S, 47 - (ee + et + k))


def _scaled(data, t, E, s):
    """(products, scaled products, unsaturated mask) of a block of rows"""
    with np.errstate(invalid="ignore", over="ignore", under="ignore"):
        p = E[None, :] * t[:, None]                      # rounded like the reference's E[k] * t[i] (:295)
        x = np.ldexp(p, s)                               # exact, or below 2^-1022 (an integer 0 either way)
    return p, x, data != 255                             # :293


def limbs_of(totals):
    """exact per-bin integer sums (Python ints) -> the three 43-bit limbs a rank all-reduces"""
    limbs = np.zeros(768, np.int64)
    mask = (1 << LIMB_BITS) - 1
    for b in range(256):
        limbs[b], limbs[256 + b], limbs[512 + b] = totals[b] & mask, (totals[b] >> LIMB_BITS) & mask, totals[b] >> (2 * LIMB_BITS)
    limbs[255] = limbs[511] = limbs[767] = 0             # value 255 is never summed
    return limbs


def accumulate_loop(data, t, E, words):
    """accumulate() one sample at a time in Python integers: the plain statement of the sums, for small inputs."""
    s = exponent(words)
    p, x, keep = _scaled(data, t, E, s)
    with np.errstate(invalid="ignore"):
        ok = keep & (np.abs(x) < LIMIT)                  # False for NaN
    counts = np.bincount(data[keep].ravel(), minlength=256)[:256].astype(np.int64)
    special = np.zeros(256)
    odd = keep & ~ok
    with np.errstate(invalid="ignore"):
        np.add.at(special, data[odd], p[odd])
    totals = [0] * 256
    v = np.rint(x[ok]).astype(np.int64)                  # round to nearest even, exact below 2^48
    for b, val in zip(data[ok].tolist(), v.tolist()):
        totals[b] += val
    return limbs_of(totals), special, counts


def accumulate(data, t, E, words):
    """The same sums, vectorised: each rounded product split into two 24-bit halves, the halves summed per bin with np.bincount in
    blocks of at most 2^24 samples (exact in fp64), the block sums joined in Python integers."""
    s = exponent(words)
    n, npix = data.shape
    rows = max(1, CHUNK // max(npix, 1))
    totals = [0] * 256
    counts = np.zeros(256, np.int64)
    special = np.zeros(256)
    for r0 in range(0, n, rows):
        d = data[r0:r0 + rows]
        p, x, keep = _scaled(d, t[r0:r0 + rows], E, s)
        with np.errstate(invalid="ignore"):
            ok = keep & (np.abs(x) < LIMIT)
        counts += np.bincount(d[keep].ravel(), minlength=256)[:256]
        odd = keep & ~ok
        if odd.any():
            special += np.bincount(d[odd], weights=p[odd], minlength=256)[:256]      # ±inf / NaN only: order-free
        b = d[ok]
        v = np.rint(x[ok]).astype(np.int64)
        lo = np.bincount(b, weights=(v & ((1 << HALF_BITS) - 1)).astype(np.float64), minlength=256)
        hi = np.bincount(b, weights=(v >> HALF_BITS).astype(np.float64), minlength=256)
        for k in np.flatnonzero((lo != 0) | (hi != 0)):
            totals[k] += int(lo[k]) + (int(hi[k]) << HALF_BITS)
    return limbs_of(totals), special, counts


def sums(words, limbs, special):
    s = exponent(words)
    out = np.zeros(256)
    for b in range(256):
        v = int(limbs[b]) + (int(limbs[256 + b]) << LIMB_BITS) + (int(limbs[512 + b]) << (2 * LIMB_BITS))
        lo, hi = v & ((1 << 64) - 1), v >> 64
        with np.errstate(over="ignore", invalid="ignore"):
            out[b] = np.ldexp(np.float64(float(hi) * 18446744073709551616.0 + float(lo)), -s) + special[b]      # inf where 2^-s > 1 overflows it
    return out


def finish(words, limbs, special, counts):
    with np.errstate(divide="ignore", invalid="ignore"):
        g = sums(words, limbs, special) / counts.astype(np.float64)
    for i in range(2, 256):                             # main_responseCalib.cpp:300-304, sequential
        if not np.isfinite(g[i]):
            g[i] = g[i - 1] + (g[i - 1] - g[i - 2])
    return g


def gstep(data, t, E):
    """The whole G-step on one rank."""
    w = scale_words(E, t)
    limbs, special, counts = accumulate(data, t, E, w)
    return finish(w, limbs, special, counts)
