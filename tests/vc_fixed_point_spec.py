"""vignetteCalib's vignette step (main_vignetteCalib.cpp:458-533, DESIGN.md §4 N4) as the CUDA kernels compute it, written out in
numpy: the specification `vc_vignette_kernel` / `vc_divide_kernel` / `vc_normalise_kernel` are compared with bit for bit
(tests/test_vignette_calib_optimiser.py).  Test infrastructure.

Every term is the reference's fp32 product (:489-503).  A finite term is scaled by 2^s and rounded to the nearest integer, ties to
even; the integers of one pixel are summed exactly (int64).  A term that is not finite goes to an fp32 side sum instead, which then
only ever holds +-inf or NaN, so its value does not depend on the order.  The pixel's sum is float(double(int64) * 2^-s) + side sum.

  bounds(images, p2x, p2y, plane, wI)          -> (bits of max finite |plane|, bits of max finite |image|, max footprint count)
  scale_exponent(plane_bits, image_bits, count) -> s
  vignette_step(...)                            -> dict(vignette, tt, ct, tt_special, ct_special, s, E, R, ...)
"""
import math

import numpy as np

f32 = np.float32
NAN32 = f32(np.nan)
LO_BITS = 26                     # an int64 term is summed as (term >> 26) and (term & (2^26 - 1)), each exactly in float64


def _absmax_bits(v):
    a = np.abs(np.asarray(v, f32).ravel())
    a = a[np.isfinite(a)]
    return int(a.max().view(np.uint32)) if a.size else 0


def taps(x, y, wI):
    """The index/weight part of getInterpolatedElement (:52-62) on float32 arrays: (w00, w10, w01, w11, base)."""
    ix, iy = x.astype(np.int32), y.astype(np.int32)
    dx, dy = x - ix.astype(f32), y - iy.astype(f32)
    dxdy = dx * dy
    w00 = ((f32(1) - dx) - dy) + dxdy
    return w00, dx - dxdy, dy - dxdy, dxdy, ix.astype(np.int64) + iy.astype(np.int64) * wI


def blend(mat, w, wI):
    """... and its blend (:65-68), left to right in fp32."""
    w00, w10, w01, w11, b = w
    r = w11 * mat[b + 1 + wI]
    r = r + w01 * mat[b + wI]
    r = r + w10 * mat[b + 1]
    return r + w00 * mat[b]


def outlier(residual, oth2, integer_abs):
    """`abs(residual) > oth2` (:481): on the residual truncated to int (integer_abs; out-of-range and NaN never count), or fabs."""
    with np.errstate(invalid="ignore"):
        if not integer_abs:
            return np.abs(residual) > oth2
        return (residual < 2147483648.0) & (np.trunc(np.where(residual < 2147483648.0, residual, 0.0)) > oth2)


def bounds(images, p2x, p2y, plane, wI):
    """What fixes the scale: the largest finite |planeColor| and |image| as float bit patterns, and the largest number of map
    entries whose bilinear footprint starts at one pixel.  Every non-NaN map entry counts, whatever its plane colour.  Nothing is
    measured when there is no map entry at all."""
    if p2x.size == 0:
        return 0, 0, 0
    count = np.zeros(images.shape[1], np.int64)
    for img in range(p2x.shape[0]):
        ok = ~np.isnan(p2x[img])
        base = taps(p2x[img][ok], p2y[img][ok], wI)[4]
        count += np.bincount(base, minlength=count.size)
    return _absmax_bits(plane), _absmax_bits(images), int(count.max())


def ilogb(x):
    return math.frexp(x)[1] - 1


def scale_exponent(plane_bits, image_bits, count):
    """vc_scale_exponent: the largest s with |term| * 2^s < 2^50 and (4 * count + 4) * |term| * 2^s < 2^62 for every term the
    bounds allow (|w| <= 1; the factor 1.001 covers the fp32 roundings of the products)."""
    P = float(np.uint32(plane_bits).view(f32))
    I = float(np.uint32(image_bits).view(f32))
    term = P * (P if P > I else I) * 1.001
    if not term > 0.0:
        return 0
    total = term * (4.0 * count + 4.0)
    s = min(50 - (ilogb(term) + 1), 62 - (ilogb(total) + 1))
    return max(-1000, min(1000, s))


def sample_terms(images, p2x, p2y, plane, vignette, wI, oth2, integer_abs, img):
    """One image's samples (:467-503): (TT terms [4, k], CT terms [4, k], pixel offsets [4, k]) of the samples that are summed, and
    this image's share of (E, R)."""
    x = p2x[img]
    pi = np.flatnonzero(~np.isnan(x))                                                # :469
    cP = plane[pi]
    keep = ~np.isnan(cP)                                                             # :477
    pi, cP = pi[keep], cP[keep]
    with np.errstate(invalid="ignore", over="ignore"):
        w = taps(x[pi], p2y[img][pi], wI)
        cI = blend(images[img], w, wI)
        keep = ~np.isnan(cI)                                                         # :478
        w, cP, cI = tuple(a[keep] for a in w), cP[keep], cI[keep]
        fac = blend(vignette, w, wI)
        d = cI - cP * fac
        residual = (d * d).astype(np.float64)
        out = outlier(residual, oth2, integer_abs)                                   # :481-486
        keep = ~out
        counted = keep & ~np.isnan(fac)                                              # :504-505
        E = float(oth2) * int(out.sum()) + float(np.sum(residual[counted]))
        R = int(out.sum()) + int(counted.sum())
        w, cP, cI = tuple(a[keep] for a in w), cP[keep], cI[keep]
        tt = np.stack([(wk * cP) * cP for wk in w[:4]])                              # :489-503, w00 w10 w01 w11
        ct = np.stack([(wk * cI) * cP for wk in w[:4]])
    pix = np.stack([w[4], w[4] + 1, w[4] + wI, w[4] + 1 + wI])
    return tt, ct, pix, E, R


class _ExactSum:
    """Per-pixel exact int64 sums of quantised terms, and fp32 side sums of the terms that are not finite."""

    def __init__(self, npx, s):
        self.scale = math.ldexp(1.0, s)
        self.hi, self.lo = np.zeros(npx, np.int64), np.zeros(npx, np.int64)
        self.special = np.zeros(npx, f32)
        self.npx = npx

    def add(self, terms, pix):
        terms, pix = terms.ravel(), pix.ravel()
        fin = np.isfinite(terms)
        if not fin.all():
            np.add.at(self.special, pix[~fin], terms[~fin])
        q = np.rint(terms[fin].astype(np.float64) * self.scale).astype(np.int64)
        p = pix[fin]
        # each part's per-pixel sum stays far below 2^53, so the float64 bincounts are exact
        self.hi += np.rint(np.bincount(p, q >> LO_BITS, self.npx)).astype(np.int64)
        self.lo += np.rint(np.bincount(p, q & ((1 << LO_BITS) - 1), self.npx)).astype(np.int64)

    def total(self):
        return (self.hi << LO_BITS) + self.lo


def to_float(acc, s, special):
    """float(scalbn(double(acc), -s)) + side sum, as vc_divide_kernel converts a sum."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.ldexp(acc.astype(np.float64), -s).astype(f32) + special


def divide_normalise(t, c):
    """:507-523: CT/TT where TT >= 1 else NaN; the largest factor, starting from 0; every factor divided by it."""
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        v = np.where(t < 1, NAN32, c / t).astype(f32)
        pos = v[v > 0]
        m = pos.max() if pos.size else f32(0)
        return (v / m).astype(f32), m


def vignette_step(images, p2x, p2y, wI, hI, plane, vignette, oth2, integer_abs=True, on_terms=None):
    """The whole vignette step.  images [n, wI*hI], p2x / p2y [n, gw*gh], plane [gw*gh], vignette [wI*hI], all float32.
    on_terms(tt, ct, pix), if given, sees every image's summed terms (for measurements against exact sums)."""
    npx = wI * hI
    plane_bits, image_bits, count = bounds(images, p2x, p2y, plane, wI)
    s = scale_exponent(plane_bits, image_bits, count)
    TT, CT = _ExactSum(npx, s), _ExactSum(npx, s)
    E, R = 0.0, 0
    for img in range(p2x.shape[0]):
        tt, ct, pix, e, r = sample_terms(images, p2x, p2y, plane, vignette, wI, oth2, integer_abs, img)
        TT.add(tt, pix)
        CT.add(ct, pix)
        E += e
        R += r
        if on_terms is not None:
            on_terms(tt, ct, pix)
    tt_acc, ct_acc = TT.total(), CT.total()
    t, c = to_float(tt_acc, s, TT.special), to_float(ct_acc, s, CT.special)
    v, m = divide_normalise(t, c)
    return dict(vignette=v, t=t, c=c, tt=tt_acc, ct=ct_acc, tt_special=TT.special, ct_special=CT.special, s=s, max_factor=m,
                bounds=(plane_bits, image_bits, count), E=E, R=float(R))
