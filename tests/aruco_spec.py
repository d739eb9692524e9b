"""Specification of vignetteCalib's marker detection (main_vignetteCalib.cpp:231-262 with aruco 1.3.0's MarkerDetector, paths
below inside aruco-1.3.0/src/), restated in Python over OpenCV's own primitives (cv2), plus numpy restatements of the per-pixel
steps 1 and 3 that need no cv2, and a numpy renderer of marker scenes from the id rule of arucofidmarkers.cpp.

Steps (the numbering the tests use):
  1  grey = convertTo(CV_8U, 1, 0) of the rectified frame: round half to even, saturate (NaN -> 0)
  3  mask = adaptiveThreshold(grey, 255, ADAPTIVE_THRESH_MEAN_C, THRESH_BINARY_INV, 7, 7)        markerdetector.cpp:437-458
  4  candidates (detectRectangles, :287-430)
  5  id per candidate (:166-191, arucofidmarkers.cpp:290-465)
  6  LINES corner refinement (:779-928)
  7  filters (:218-253)
  8  homography from the unit square (main_vignetteCalib.cpp:242-253)

findContours: aruco's OpenCV (2.x) cleared the image's outer rows and columns before tracing; OpenCV 4 pads the image with zeros
instead, so the spec clears them itself.  std::sort of step 7 is not stable; the spec sorts stably, which is the same whenever no
two markers share an id or at most 16 markers are sorted (libstdc++ sorts that few by insertion).
"""
from __future__ import annotations

import numpy as np

WARP = 56
WORDS = np.array([[1, 0, 0, 0, 0], [1, 0, 1, 1, 1], [0, 1, 0, 0, 1], [0, 1, 1, 1, 0]], np.uint8)   # hammDistMarker, :308


# ---- steps 1 and 3 in numpy ------------------------------------------------------------------------------------------------
def grey_u8(rect: np.ndarray) -> np.ndarray:
    r = np.asarray(rect, np.float32)
    out = np.rint(np.nan_to_num(r, nan=0.0, posinf=255.0, neginf=0.0))
    return np.clip(out, 0, 255).astype(np.uint8)


def adaptive_threshold(grey: np.ndarray) -> np.ndarray:
    g = np.asarray(grey, np.int64)
    p = np.pad(g, 3, mode="edge")
    c = np.cumsum(np.cumsum(np.pad(p, ((1, 0), (1, 0))), 0), 1)
    h, w = g.shape
    s = c[7:7 + h, 7:7 + w] - c[0:h, 7:7 + w] - c[7:7 + h, 0:w] + c[0:h, 0:w]
    mean = np.clip(np.rint(s / 49.0), 0, 255).astype(np.int64)
    return np.where(g - mean <= -7, 255, 0).astype(np.uint8)


# ---- scenes from the id rule -----------------------------------------------------------------------------------------------
def marker_bits(marker_id: int) -> np.ndarray:
    """7x7 cells (1 = white) of marker `marker_id` at rotation 0: black border, row y of the 5x5 data is the code word whose
    columns 1 and 3 are bits 2(4-y)+1 and 2(4-y) of the id."""
    bits = np.zeros((7, 7), np.uint8)
    for y in range(5):
        two = (marker_id >> (2 * (4 - y))) & 3
        bits[y + 1, 1:6] = WORDS[two]
    return bits


def _homography(src, dst) -> np.ndarray:
    A, b = [], []
    for (X, Y), (x, y) in zip(src, dst):
        A.append([X, Y, 1, 0, 0, 0, -x * X, -x * Y]); b.append(x)
        A.append([0, 0, 0, X, Y, 1, -y * X, -y * Y]); b.append(y)
    h = np.linalg.solve(np.array(A, float), np.array(b, float))
    return np.append(h, 1.0).reshape(3, 3)


def shade(X, Y, markers, background: float = 200.0, black: float = 25.0, white: float = 225.0) -> np.ndarray:
    """Scene value at the points (X, Y): `markers` = [(bits 7x7, quad [4, 2] of the marker's outer corners (TL, TR, BR, BL of the
    bit grid))] over a flat background, each with a white quiet zone of one cell."""
    out = np.full(np.shape(X), background, np.float64)
    for bits, quad in markers:
        Hinv = np.linalg.inv(_homography([(0, 0), (7, 0), (7, 7), (0, 7)], np.asarray(quad, float)))
        W = Hinv[2, 0] * X + Hinv[2, 1] * Y + Hinv[2, 2]
        u = (Hinv[0, 0] * X + Hinv[0, 1] * Y + Hinv[0, 2]) / W
        v = (Hinv[1, 0] * X + Hinv[1, 1] * Y + Hinv[1, 2]) / W
        inside = (u >= -1) & (u < 8) & (v >= -1) & (v < 8) & (W > 0)
        cu = np.clip(np.floor(np.nan_to_num(u)), -1, 7).astype(int)
        cv = np.clip(np.floor(np.nan_to_num(v)), -1, 7).astype(int)
        in_grid = (cu >= 0) & (cu < 7) & (cv >= 0) & (cv < 7)
        val = np.where(in_grid & (bits[np.clip(cv, 0, 6), np.clip(cu, 0, 6)] == 0), black, white)
        out = np.where(inside, val, out)
    return out


def render(w: int, h: int, markers, ss: int = 3, **kw) -> np.ndarray:
    """float32 [h, w] image of shade(): each pixel the mean over ss x ss samples."""
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    off = (np.arange(ss) + 0.5) / ss - 0.5
    acc = np.zeros((h, w))
    for dy in off:
        for dx in off:
            acc += shade(xs + dx, ys + dy, markers, **kw)
    return (acc / (ss * ss)).astype(np.float32)


def square(cx, cy, size, angle_deg=0.0):
    a = np.deg2rad(angle_deg)
    r = size / 2 * np.sqrt(2)
    return np.array([[cx + r * np.cos(a + t), cy + r * np.sin(a + t)] for t in np.deg2rad([225, 315, 45, 135])])


# ---- steps 3-8 over cv2 ----------------------------------------------------------------------------------------------------
def threshold_cv2(grey):
    import cv2
    return cv2.adaptiveThreshold(np.ascontiguousarray(grey), 255, cv2.ADAPTIVE_THRESH_MEAN_C, cv2.THRESH_BINARY_INV, 7, 7)


def contours_cv2(mask):
    import cv2
    m = np.ascontiguousarray(mask).copy()
    m[0, :] = 0; m[-1, :] = 0; m[:, 0] = 0; m[:, -1] = 0
    cs, _ = cv2.findContours(m, cv2.RETR_LIST, cv2.CHAIN_APPROX_NONE)
    return [c.reshape(-1, 2).astype(np.int32) for c in cs]


def _perimeter(q) -> int:
    s = 0
    for i in range(4):
        d = np.float32(q[i]) - np.float32(q[(i + 1) % 4])
        s = int(np.float32(s) + np.sqrt(np.float32(d[0] * d[0] + d[1] * d[1])))
    return s


def candidates_cv2(mask, stages=None):
    """detectRectangles: [(quad float32 [4, 2], contour int32 [n, 2])]"""
    import cv2
    h, w = mask.shape
    mn, mx = int(0.04 * max(w, h) * 4), int(0.5 * max(w, h) * 4)
    cands = []
    for c in contours_cv2(mask):
        n = len(c)
        if not (mn < n < mx):
            continue
        ap = cv2.approxPolyDP(c.reshape(-1, 1, 2), float(n) * 0.05, True).reshape(-1, 2)
        if stages is not None:
            stages.setdefault("approx", []).append((c, ap))
        if len(ap) != 4 or not cv2.isContourConvex(ap.reshape(-1, 1, 2)):
            continue
        d = [np.sqrt(np.float32((ap[j] - ap[(j + 1) % 4]) @ (ap[j] - ap[(j + 1) % 4]))) for j in range(4)]
        if not min(d) > 10:
            continue
        cands.append([ap.astype(np.float32), c.copy()])
    swapped = []
    for cd in cands:
        q = cd[0].astype(np.float64)
        o = (q[1, 0] - q[0, 0]) * (q[2, 1] - q[0, 1]) - (q[1, 1] - q[0, 1]) * (q[2, 0] - q[0, 0])
        swapped.append(o < 0)
        if o < 0:
            cd[0][[1, 3]] = cd[0][[3, 1]]
    remove = [False] * len(cands)
    for i in range(len(cands)):
        for j in range(i + 1, len(cands)):
            dd = cands[i][0] - cands[j][0]
            if all(np.sqrt(np.float32(dd[k, 0] * dd[k, 0] + dd[k, 1] * dd[k, 1])) < 6 for k in range(4)):
                if _perimeter(cands[i][0]) > _perimeter(cands[j][0]):
                    remove[j] = True
                else:
                    remove[i] = True
    return [(q, c[::-1].copy() if s else c) for (q, c), s, r in zip(cands, swapped, remove) if not r]


def rotate_bits(b):
    """FiducidalMarkers::rotate, arucofidmarkers.cpp:290: out(i, j) = in(cols - j - 1, i)"""
    out = np.empty_like(b)
    for i in range(b.shape[0]):
        for j in range(b.shape[1]):
            out[i, j] = b[b.shape[1] - j - 1, i]
    return out


def read_bits(binary_patch):
    """the 7x7 cells of a thresholded 56x56 patch, 1 = more than half of the 64 pixels non-zero"""
    return (np.count_nonzero(binary_patch.reshape(7, 8, 7, 8), axis=(1, 3)) > 32).astype(np.uint8)


def id_from_bits(cells):
    """analyzeMarkerImage on 7x7 cells: (id or -1, rotations)"""
    if cells[0].any() or cells[6].any() or cells[:, 0].any() or cells[:, 6].any():
        return -1, 0
    rots = [cells[1:6, 1:6]]
    for _ in range(3):
        rots.append(rotate_bits(rots[-1]))
    dists = [sum(min(int(np.sum(r[y] != WORDS[p])) for p in range(4)) for y in range(5)) for r in rots]
    best = int(np.argmin(dists))
    if dists[best] != 0:
        return -1, best
    mid = 0
    for y in range(5):
        mid = (mid << 2) | (int(rots[best][y, 1]) << 1) | int(rots[best][y, 3])
    return mid, best


def read_patch_cv2(grey, quad):
    """(warped patch, Otsu threshold, id, rotations)"""
    import cv2
    dst = np.array([[0, 0], [WARP - 1, 0], [WARP - 1, WARP - 1], [0, WARP - 1]], np.float32)
    M = cv2.getPerspectiveTransform(np.asarray(quad, np.float32), dst)
    patch = cv2.warpPerspective(np.ascontiguousarray(grey), M, (WARP, WARP), flags=cv2.INTER_NEAREST)
    t, binary = cv2.threshold(patch, 125, 255, cv2.THRESH_BINARY | cv2.THRESH_OTSU)
    mid, rot = id_from_bits(read_bits(binary))
    return patch, int(t), mid, rot


def _fit_line(pts):
    import cv2
    pts = np.asarray(pts, np.float32)
    if pts[:, 0].max() - pts[:, 0].min() > pts[:, 1].max() - pts[:, 1].min():
        A = np.stack([pts[:, 0], np.ones(len(pts), np.float32)], 1)
        _, X = cv2.solve(A, pts[:, 1:2].copy(), flags=cv2.DECOMP_SVD)
        return np.float32([X[0, 0], -1.0, X[1, 0]])
    A = np.stack([pts[:, 1], np.ones(len(pts), np.float32)], 1)
    _, X = cv2.solve(A, pts[:, 0:1].copy(), flags=cv2.DECOMP_SVD)
    return np.float32([-1.0, X[0, 0], X[1, 0]])


def refine_lines_cv2(quad, contour):
    import cv2
    size = len(contour)
    idx = [0, 0, 0, 0]
    for j in range(size):
        for k in range(4):
            if contour[j, 0] == quad[k, 0] and contour[j, 1] == quad[k, 1]:
                idx[k] = j
    if idx[1] > idx[0] and (idx[2] > idx[1] or idx[2] < idx[0]):
        inverse = False
    elif idx[2] > idx[1] and idx[2] < idx[0]:
        inverse = False
    else:
        inverse = True
    inc = -1 if inverse else 1
    lines = []
    for l in range(4):
        run, j, stop = [], idx[l], idx[(l + 1) % 4]
        while j != stop:
            if j == size and not inverse:
                j = 0
            elif j == 0 and inverse:
                j = size - 1
            run.append(contour[j])
            if j == stop:
                break
            j += inc
        lines.append(_fit_line(run))
    out = np.empty((4, 2), np.float32)
    for i in range(4):
        l1, l2 = lines[(i - 1) % 4], lines[i]
        A = np.float32([[l1[0], l1[1]], [l2[0], l2[1]]])
        B = np.float32([[-l1[2]], [-l2[2]]])
        _, X = cv2.solve(A, B, flags=cv2.DECOMP_SVD)
        out[i] = X[:, 0]
    return out


def detect_cv2(grey, mask, stages=None):
    """steps 4-7: [(id, corners float32 [4, 2])] sorted by id.  stages (a dict) receives the intermediate results."""
    h, w = grey.shape
    cands = candidates_cv2(mask, stages)
    markers = []
    for q, c in cands:
        patch, t, mid, rot = read_patch_cv2(grey, q)
        if stages is not None:
            stages.setdefault("patches", []).append((patch, t, mid, rot))
        if mid == -1:
            continue
        corners = refine_lines_cv2(q, c)
        corners = np.roll(corners, rot, axis=0)            # std::rotate(begin, begin + 4 - rot, end)
        markers.append((mid, corners))
    if stages is not None:
        stages["candidates"] = [q for q, _ in cands]
    markers.sort(key=lambda m: m[0])
    remove = [False] * len(markers)
    for i in range(len(markers) - 1):
        if markers[i][0] == markers[i + 1][0] and not remove[i + 1]:
            if _perimeter(markers[i][1]) > _perimeter(markers[i + 1][1]):
                remove[i + 1] = True
            else:
                remove[i] = True
    bx, by = int(0.025 * float(np.float32(w))), int(0.025 * float(np.float32(h)))
    for i, (_, c) in enumerate(markers):
        if (c[:, 0] < bx).any() or (c[:, 1] < by).any() or (c[:, 0] > w - bx).any() or (c[:, 1] > h - by).any():
            remove[i] = True
    return [m for m, r in zip(markers, remove) if not r]


PLANE = np.array([[-0.5, 0.5], [0.5, 0.5], [0.5, -0.5], [-0.5, -0.5]], np.float32)


def homography_cv2(corners):
    import cv2
    H, _ = cv2.findHomography(PLANE, np.asarray(corners, np.float32))
    return H


def frame_homography(grey, mask, detect=None):
    """step 8: the frame's H, or None unless exactly one marker is found"""
    ms = (detect or detect_cv2)(grey, mask)
    if len(ms) != 1:
        return None, ms
    return homography_cv2(ms[0][1]), ms
