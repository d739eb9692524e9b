"""Independent statement of UndistorterFOV::undistort for arbitrary remap tables (test infrastructure).

FOVUndistorter.cpp:341-367, for every output pixel idx with (x, y) = (remapX[idx], remapY[idx]):

    if (x < 0) out = 0;                                  only x is tested: y may be anything, NaN included
    else {
        xi = (int)x; yi = (int)y;                        truncation toward zero: a y in (-1, 0) has row 0 and a NEGATIVE fraction
        fx = x - xi; fy = y - yi; fxy = fx * fy;         float32
        s = input + xi + yi * W;
        out = ((fxy * s[1+W] + (fy - fxy) * s[W]) + (fx - fxy) * s[1]) + (((1 - fx) - fy) + fxy) * s[0];
    }

every operation rounded to float32, no fused multiply-add, subnormals kept.  Written with numpy arrays, not by looking at
oracle/port/mdc_oracle_port.c or the kernels, so that those are checked against a second formulation.

The domain D: the entries for which the reference reads only pixels of the W x H frame.  x < 0 (black, any y), or
0 <= x < W-1 and -1 < y < H-1 (then 0 <= xi <= W-2 and 0 <= yi <= H-2).  NaN fails every comparison, so a NaN x and a NaN y
under a valid x are outside D; -0.0 is a valid x (it is not < 0) and truncates to column 0."""
import numpy as np

F32 = np.float32


def in_domain(rx, ry, in_w, in_h):
    """Boolean mask of the table entries inside D (compared in float64: W-1 and H-1 need not be floats)."""
    x = np.asarray(rx, F32).astype(np.float64)
    y = np.asarray(ry, F32).astype(np.float64)
    with np.errstate(invalid="ignore"):
        return (x < 0) | ((x >= 0) & (x < in_w - 1) & (y > -1) & (y < in_h - 1))


def taps(rx, ry, in_w, in_h):
    """(valid mask, flat index of s[0], w3, w2, w1, w0) for the entries with !(x < 0); all of the table must be inside D."""
    rx = np.asarray(rx, F32).reshape(-1)
    ry = np.asarray(ry, F32).reshape(-1)
    assert in_domain(rx, ry, in_w, in_h).all(), "table entries outside D"
    valid = ~(rx < 0)
    x, y = rx[valid], ry[valid]
    xi = np.trunc(x).astype(np.int64)
    yi = np.trunc(y).astype(np.int64)
    fx = np.subtract(x, xi.astype(F32), dtype=F32)
    fy = np.subtract(y, yi.astype(F32), dtype=F32)
    fxy = np.multiply(fx, fy, dtype=F32)
    w3 = fxy
    w2 = np.subtract(fy, fxy, dtype=F32)
    w1 = np.subtract(fx, fxy, dtype=F32)
    w0 = np.add(np.subtract(np.subtract(F32(1), fx, dtype=F32), fy, dtype=F32), fxy, dtype=F32)
    return valid, xi + yi * in_w, w3, w2, w1, w0


def undistort(rx, ry, in_w, in_h, img):
    """undistort<unsigned char> or <float>: img [in_h * in_w] uint8 or float32 -> float32 [len(rx)]."""
    s = np.asarray(img).reshape(-1)
    assert s.size == in_w * in_h and s.dtype in (np.uint8, np.float32)
    s = s.astype(F32)                    # exact for uint8
    valid, b, w3, w2, w1, w0 = taps(rx, ry, in_w, in_h)
    out = np.zeros(valid.size, F32)
    with np.errstate(all="ignore"):
        acc = np.multiply(w3, s[b + 1 + in_w], dtype=F32)
        acc = np.add(acc, np.multiply(w2, s[b + in_w], dtype=F32), dtype=F32)
        acc = np.add(acc, np.multiply(w1, s[b + 1], dtype=F32), dtype=F32)
        acc = np.add(acc, np.multiply(w0, s[b], dtype=F32), dtype=F32)
    out[valid] = acc
    return out


def unmap(ginv, vinv, raw, gamma, vignette, kill):
    """PhotometricUndistorter::unMapImage (PhotometricUndistorter.cpp:173-211) with both tables loaded: GInv[raw], times the
    inverse vignette when both are removed (vignette alone removes nothing), NaN where raw is 255 when killing."""
    raw = np.asarray(raw, np.uint8).reshape(-1)
    if vignette and not gamma:
        gamma = vignette = False
    out = raw.astype(F32)
    if gamma:
        out = np.asarray(ginv, F32)[raw]
    if gamma and vignette:
        with np.errstate(all="ignore"):
            out = np.multiply(out, np.asarray(vinv, F32).reshape(-1), dtype=F32)
    if kill:
        out = np.where(raw == 255, F32(np.nan), out)
    return out


def get_image(rx, ry, in_w, in_h, ginv, vinv, raw, rectify, gamma, vignette, kill):
    """DatasetReader::getImage (BenchmarkDatasetReader.h:210-241): undistort<uchar> of the raw frame when nothing photometric is
    asked for, else undistort<float> of the unmapped frame."""
    if not (gamma or vignette or kill):
        return undistort(rx, ry, in_w, in_h, raw) if rectify else np.asarray(raw, np.uint8).reshape(-1).astype(F32)
    u = unmap(ginv, vinv, raw, gamma, vignette, kill)
    return undistort(rx, ry, in_w, in_h, u) if rectify else u
