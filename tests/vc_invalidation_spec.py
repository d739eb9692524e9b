"""Independent statement of vignetteCalib's image preparation (main_vignetteCalib.cpp:286-301) — test infrastructure.

The reference normalises each image, image = (meanExposure * raw) / exposure in float32, and then walks the centres
2 <= x < w-2, 2 <= y < h-2 in raster order; for each it compares |centre - neighbour| > maxAbsGrad over the 5x5 window (deltax
outer, deltay inner) and sets BOTH pixels to NaN on a hit, in place.  The result depends on that order.

This file states the same result the way the GPU computes it, without replaying the in-place loop:

  1. candidates: a 24-bit mask per centre, bit k set if neighbour k (window order) compares above the threshold on the values as
     they are before the pass.  Values only ever become NaN and a comparison with NaN is false, so no other comparison can fire.
  2. greedy: visit the centres with a non-zero mask in raster order; a centre that is already dead is skipped (its comparisons
     are against NaN); otherwise it dies together with the FIRST neighbour of its mask, in window order, that is still alive
     (after that hit the centre is NaN and nothing more fires).

It is written with numpy slices and an explicit alive set, not by looking at oracle/port/mdc_oracle_port.c:oport_vc_prepare_image,
so that the C restatement, this statement and the CUDA kernels check one another."""
import numpy as np

# window order of the reference: deltax outer, deltay inner
OFFSETS = [(dx, dy) for dx in range(-2, 3) for dy in range(-2, 3)]


def normalise(raw: np.ndarray, mean_exposure, exposure) -> np.ndarray:
    t = np.float32(exposure)
    if t == 0:
        t = np.float32(1)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        return np.divide(np.multiply(np.float32(mean_exposure), raw, dtype=np.float32), t, dtype=np.float32)


def candidate_masks(img: np.ndarray, max_abs_grad) -> np.ndarray:
    """img float32 [h, w] -> uint32 [h-4, w-4] masks of the centres (bit k = OFFSETS[k])."""
    h, w = img.shape
    c = img[2:h - 2, 2:w - 2]
    masks = np.zeros(c.shape, np.uint32)
    g = np.float32(max_abs_grad)
    with np.errstate(invalid="ignore", over="ignore"):
        for k, (dx, dy) in enumerate(OFFSETS):
            nb = img[2 + dy:h - 2 + dy, 2 + dx:w - 2 + dx]
            masks |= (np.abs(np.subtract(c, nb, dtype=np.float32)) > g).astype(np.uint32) << np.uint32(k)
    return masks


def invalidate(img: np.ndarray, max_abs_grad) -> np.ndarray:
    """img float32 [h, w] (normalised) -> the invalidated copy."""
    h, w = img.shape
    out = img.copy()
    if h < 5 or w < 5:
        return out
    masks = candidate_masks(img, max_abs_grad)
    dead = np.zeros((h, w), bool)
    for cy, cx in zip(*np.nonzero(masks)):          # row-major = raster order
        y, x = cy + 2, cx + 2
        if dead[y, x]:
            continue
        m = int(masks[cy, cx])
        for k, (dx, dy) in enumerate(OFFSETS):
            if m >> k & 1 and not dead[y + dy, x + dx]:
                dead[y, x] = dead[y + dy, x + dx] = True
                break
    out[dead] = np.nan
    return out


def prepare_image(raw: np.ndarray, w: int, h: int, mean_exposure, exposure, max_abs_grad=255) -> np.ndarray:
    """raw float32 [w*h] -> the prepared image, float32 [w*h]."""
    img = normalise(np.ascontiguousarray(raw, np.float32).reshape(h, w), mean_exposure, exposure)
    return invalidate(img, max_abs_grad).reshape(-1)
