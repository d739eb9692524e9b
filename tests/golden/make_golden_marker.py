"""Generates tests/golden/marker/marker_sequence.npz: a short sequence seen through a distorting FOV camera, with markers, and what the
marker-detection specification (tests/aruco_spec.py) finds in it.

    python tests/golden/make_golden_marker.py          (needs cv2 for the specification)

Raw frames are rendered by looking up, for every raw pixel, the rectified position the FOV model maps it to (the inverse of the
rectifier's remap table, interpolated) and shading the marker scene there.  Rectification is the oracle port's undistort.  Per
frame the fixture holds sha256 of the specification's grey and mask images, the markers (id, corners) and the homography (NaN unless
exactly one marker).  Frames 2 and 5 show no marker, frame 4 two markers.
"""
import hashlib
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import aruco_spec as A  # noqa: E402
from mono_dataset_code_b200 import synthetic as S  # noqa: E402

W, H = 320, 240
OUT = os.path.join(ROOT, "tests", "golden", "marker", "marker_sequence.npz")
# (id, centre x, centre y, size, angle) in rectified pixels per frame
POSES = [[(613, 160, 120, 90, 10)], [(77, 150, 125, 80, -25)], [], [(1000, 170, 110, 100, 40)],
         [(5, 95, 120, 70, 5), (900, 225, 120, 70, -10)], [], [(613, 165, 125, 110, 80)], [(321, 155, 115, 75, 190)]]


def rectified_lookup(port_fov):
    """for every raw pixel, the rectified (x, y) that the remap table sends to it (NaN outside the rectified frame)"""
    from scipy.interpolate import griddata
    rx, ry = port_fov.tables()
    ys, xs = np.mgrid[0:H, 0:W]
    ok = rx >= 0
    pts = np.stack([rx[ok], ry[ok]], 1)
    X = griddata(pts, xs.ravel()[ok], (xs + 0.0, ys + 0.0), method="linear")
    Y = griddata(pts, ys.ravel()[ok], (xs + 0.0, ys + 0.0), method="linear")
    return X, Y


def spec_frame(port, port_fov, raw):
    rx, ry = port_fov.tables()
    rect = port.undistort(rx, ry, W, raw.ravel()).reshape(H, W)
    grey = A.grey_u8(rect)
    mask = A.adaptive_threshold(grey)
    ms = A.detect_cv2(grey, mask)
    Hm = A.homography_cv2(ms[0][1]) if len(ms) == 1 else np.full((3, 3), np.nan)
    return grey, mask, ms, Hm


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    from oracle.loader import PortOracle
    port = PortOracle()
    camera = S.camera_txt(W, H, W, H, "crop")
    with tempfile.TemporaryDirectory() as tmp:
        cam = os.path.join(tmp, "camera.txt")
        open(cam, "w").write(camera)
        pf = port.fov_from_file(cam)
    X, Y = rectified_lookup(pf)
    rng = np.random.default_rng(5)
    frames, greys, masks, ids, corners, Hs = [], [], [], [], [], []
    for i, pose in enumerate(POSES):
        markers = [(A.marker_bits(mid), A.square(cx, cy, s, a)) for mid, cx, cy, s, a in pose]
        val = np.where(np.isnan(X), 200.0, A.shade(np.nan_to_num(X), np.nan_to_num(Y), markers))
        raw = np.clip(np.rint(val * (0.8 + 0.05 * i) + rng.normal(0, 2.0, val.shape)), 0, 255).astype(np.uint8)
        grey, mask, ms, Hm = spec_frame(port, pf, raw)
        assert len(ms) == len(pose), (i, [m[0] for m in ms])
        frames.append(raw)
        greys.append(sha(grey))
        masks.append(sha(mask))
        ids.append([m[0] for m in ms] + [-1] * (2 - len(ms)))
        c = np.full((2, 4, 2), np.nan, np.float32)
        for k, m in enumerate(ms):
            c[k] = m[1]
        corners.append(c)
        Hs.append(Hm.ravel())
    times = "".join(f"{i} {1.0 + 0.05 * i:.6f} {1.0 + 0.1 * i:.6f}\n" for i in range(len(POSES)))
    np.savez_compressed(OUT, frames=np.stack(frames), camera_txt=camera, pcalib_txt=S.pcalib_txt(), times_txt=times,
                        grey_sha256=np.array(greys), mask_sha256=np.array(masks), ids=np.array(ids, np.int32),
                        corners=np.stack(corners), homographies=np.stack(Hs))
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
