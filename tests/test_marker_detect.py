"""vignetteCalib's marker detection (mdc_marker_detect, mdc_marker_homography and their stages, csrc/mdc_marker.cpp) against the
specification tests/aruco_spec.py, which restates aruco 1.3.0's MarkerDetector over OpenCV's own primitives; the specification
against those primitives; and the golden marker sequence (tests/golden/marker/marker_sequence.npz) re-derived from the specification."""
import hashlib
import os
import subprocess
import tempfile

import numpy as np
import pytest

import aruco_spec as A
from conftest import ROOT
from mono_dataset_code_b200 import api

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "marker", "marker_sequence.npz")
CORNER_TOL = 2e-3


def _scene(w, h, markers, noise=0.0, blur=0, seed=0, **kw):
    img = A.render(w, h, markers, **kw).astype(np.float64)
    if blur:
        k = np.ones(2 * blur + 1) / (2 * blur + 1)
        img = np.apply_along_axis(lambda r: np.convolve(np.pad(r, blur, mode="edge"), k, "valid"), 1, img)
        img = np.apply_along_axis(lambda r: np.convolve(np.pad(r, blur, mode="edge"), k, "valid"), 0, img)
    if noise:
        img = img + np.random.default_rng(seed).normal(0, noise, img.shape)
    return img.astype(np.float32)


def _m(mid, cx, cy, size, angle=0.0, rot=0, mirror=False, flip_bit=None):
    b = A.marker_bits(mid)
    b = np.rot90(b, rot).copy()
    if mirror:
        b = np.fliplr(b).copy()
    if flip_bit is not None:
        b[flip_bit] ^= 1
    return (b, A.square(cx, cy, size, angle))


def _persp(mid, quad):
    return (A.marker_bits(mid), np.asarray(quad, float))


SCENES = {
    "none": (640, 480, [], {}),
    "one": (640, 480, [_m(613, 300, 240, 150, 20)], {}),
    "two": (640, 480, [_m(10, 170, 240, 140, 5), _m(999, 470, 240, 140, -15)], {}),
    "same_id_twice": (640, 480, [_m(42, 170, 240, 140, 5), _m(42, 470, 240, 120, -15)], {}),
    "in_border": (640, 480, [_m(300, 70, 240, 140, 0)], {}),
    "rot90": (640, 480, [_m(613, 320, 240, 160, 12, rot=1)], {}),
    "rot180": (640, 480, [_m(613, 320, 240, 160, 12, rot=2)], {}),
    "rot270": (640, 480, [_m(613, 320, 240, 160, 12, rot=3)], {}),
    "mirrored": (640, 480, [_m(613, 320, 240, 160, 12, mirror=True)], {}),
    "one_bit_error": (640, 480, [_m(613, 320, 240, 160, 12, flip_bit=(3, 2))], {}),
    "below_min_size": (640, 480, [_m(1, 320, 240, 22, 0)], {}),
    "above_max_size": (640, 480, [_m(2, 320, 240, 420, 0)], {}),
    "perspective": (640, 480, [_persp(777, [[200, 120], [470, 170], [430, 330], [180, 390]])], {}),
    "blur_noise": (640, 480, [_m(123, 330, 230, 170, -30)], {"blur": 2, "noise": 4.0}),
    "occluded": (640, 480, [_m(456, 320, 240, 170, 8), (np.zeros((7, 7), np.uint8), [[380, 150], [470, 150], [470, 260], [380, 260]])], {}),
    "noise_only": (320, 240, [], {"noise": 30.0}),
    "odd_size": (331, 257, [_m(700, 160, 130, 90, 33)], {"noise": 2.0}),
}


def _grey_mask(name):
    w, h, markers, kw = SCENES[name]
    grey = A.grey_u8(_scene(w, h, markers, **kw))
    return grey, A.adaptive_threshold(grey)


def _special_masks():
    rng = np.random.default_rng(9)
    out = {}
    m = np.zeros((64, 80), np.uint8); m[:, :] = 255
    out["all_255"] = m
    m = (rng.random((70, 90)) < 0.5).astype(np.uint8) * 255; m[0], m[-1], m[:, 0], m[:, -1] = 255, 255, 255, 255
    out["edges_255"] = m
    yy, xx = np.mgrid[0:96, 0:96]
    out["checker1"] = (((xx + yy) % 2) * 255).astype(np.uint8)
    out["checker4"] = ((((xx // 4) + (yy // 4)) % 2) * 255).astype(np.uint8)
    r, t = np.hypot(xx - 48, yy - 48), np.arctan2(yy - 48, xx - 48)
    out["spiral"] = (((r - 3 * t) % 9 < 3) * 255).astype(np.uint8)
    m = np.zeros((60, 60), np.uint8); m[10, 5:55] = 255; m[5:55, 30] = 255; m[40:50, 40:50] = 255; m[44, 44] = 0; m[20, 20] = 255
    out["lines_holes"] = m
    for s in (1, 2, 3):
        out[f"tiny_{s}"] = (rng.random((s, s + 1)) < 0.5).astype(np.uint8) * 255
    return out


# ---- the specification against its own parts -------------------------------------------------------------------------------
@pytest.mark.parametrize("hw", [(1, 1), (1, 7), (7, 1), (3, 5), (8, 6), (64, 48), (1023, 1281)])
def test_numpy_threshold_equals_cv2(hw):
    pytest.importorskip("cv2")
    h, w = hw
    rng = np.random.default_rng(h * 7 + w)
    for img in (rng.integers(0, 256, (h, w)), np.full((h, w), 0), np.full((h, w), 255), np.full((h, w), 137),
                np.where(np.arange(w)[None, :] < w // 2, 10, 240) * np.ones((h, 1))):
        g = np.ascontiguousarray(img.astype(np.uint8))
        assert np.array_equal(A.adaptive_threshold(g), A.threshold_cv2(g))


def test_grey_rounding_is_round_half_even_and_saturating():
    v = np.array([[0.5, 1.5, 2.5, -0.5, 254.5, 255.5, 300.0, -7.0, 127.49, np.nan]], np.float32)
    assert list(A.grey_u8(v)[0]) == [0, 2, 2, 0, 254, 255, 255, 0, 127, 0]


def test_id_rule_matches_opencv_aruco_original():
    cv2 = pytest.importorskip("cv2")
    d = cv2.aruco.getPredefinedDictionary(cv2.aruco.DICT_ARUCO_ORIGINAL)
    for mid in range(1024):
        img = cv2.aruco.generateImageMarker(d, mid, 70)
        cells = (img.reshape(7, 10, 7, 10).mean(axis=(1, 3)) > 127).astype(np.uint8)
        assert np.array_equal(cells, A.marker_bits(mid)), mid
        assert A.id_from_bits(cells) == (mid, 0)


def test_rotation_convention():
    """A marker drawn at 0/90/180/270 degrees reads as the same id, and std::rotate puts corner 0 on the marker's own first corner:
    it visits each of the four image corners of the quad once."""
    pytest.importorskip("cv2")
    quad_corner = []
    for rot in range(4):
        g = A.grey_u8(A.render(480, 400, [_m(613, 240, 200, 160, 0, rot=rot)]))
        ms = A.detect_cv2(g, A.adaptive_threshold(g))
        assert [m[0] for m in ms] == [613]
        got = api.marker_detect(g, A.adaptive_threshold(g))
        assert np.abs(got[0][1] - ms[0][1]).max() <= CORNER_TOL
        quad = A.square(240, 200, 160, 0)
        quad_corner.append(int(np.argmin(np.abs(quad - ms[0][1][0]).sum(1))))
    assert sorted(quad_corner) == [0, 1, 2, 3]


# ---- mdc_marker_detect against the specification ---------------------------------------------------------------------------
def _compare_stages(grey, mask):
    stages = {}
    spec = A.detect_cv2(grey, mask, stages)
    contours = A.contours_cv2(mask)
    mine = api.marker_contours(mask)
    assert len(mine) == len(contours)
    for a, b in zip(contours, mine):
        assert np.array_equal(a, b)
    for c, ap in stages.get("approx", []):
        assert np.array_equal(api.marker_approx_poly(c, len(c) * 0.05), ap)
    cands = api.marker_candidates(mask)
    assert np.array_equal(cands.reshape(-1, 4, 2), np.array(stages["candidates"], np.float32).reshape(-1, 4, 2))
    for q, (patch, t, mid, rot) in zip(stages["candidates"], stages.get("patches", [])):
        p2, t2, mid2, rot2 = api.marker_read_patch(grey, q)
        assert np.array_equal(p2, patch) and t2 == t and mid2 == mid
        if mid != -1:
            assert rot2 == rot
    got = api.marker_detect(grey, mask)
    assert [m[0] for m in got] == [m[0] for m in spec]
    worst = 0.0
    for (_, a), (_, b) in zip(got, spec):
        worst = max(worst, float(np.abs(a - b).max()))
    assert worst <= CORNER_TOL, worst
    return got


EXPECTED = {"none": [], "one": [613], "two": [10, 999], "same_id_twice": [42], "in_border": [], "rot90": [613], "rot180": [613],
            "rot270": [613],
            # the mirror image of every marker of this code is another marker of it (rows read in the transposed rotation)
            "mirrored": [A.id_from_bits(np.fliplr(A.marker_bits(613)))[0]], "one_bit_error": [], "below_min_size": [], "above_max_size": [], "perspective": [777],
            "blur_noise": [123], "occluded": [], "noise_only": [], "odd_size": [700]}


@pytest.mark.parametrize("name", sorted(SCENES))
def test_detector_matches_the_specification(name):
    pytest.importorskip("cv2")
    grey, mask = _grey_mask(name)
    got = _compare_stages(grey, mask)
    assert [m[0] for m in got] == EXPECTED[name]


@pytest.mark.parametrize("name", sorted(_special_masks()))
def test_contours_and_candidates_on_special_masks(name):
    pytest.importorskip("cv2")
    mask = _special_masks()[name]
    grey = np.ascontiguousarray(255 - mask)
    _compare_stages(grey, mask)


def test_contours_on_random_masks():
    pytest.importorskip("cv2")
    rng = np.random.default_rng(4)
    for _ in range(200):
        h, w = rng.integers(1, 50, 2)
        m = (rng.random((h, w)) < rng.uniform(0.1, 0.9)).astype(np.uint8) * 255
        a, b = A.contours_cv2(m), api.marker_contours(m)
        assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))


def test_bad_sizes_are_rejected():
    g = np.zeros((4, 4), np.uint8)
    for w, h in ((0, 4), (4, 0), (-1, 4), (1 << 15, 1 << 14)):
        n = api.C.c_int()
        out = (api._Marker * 1)()
        assert api.lib.mdc_marker_detect(g.ctypes.data, g.ctypes.data, w, h, out, 1, api.C.byref(n)) == 1
    with pytest.raises(api.MdcError):
        api.marker_detect(np.zeros((1, 1), np.uint8), np.zeros((1, 1), np.uint8), capacity=-1)
    assert api.marker_detect(np.zeros((1, 1), np.uint8), np.zeros((1, 1), np.uint8)) == []


def test_capacity_too_small_is_an_error():
    grey, mask = _grey_mask("two")
    with pytest.raises(api.MdcError):
        api.marker_detect(grey, mask, capacity=1)


# ---- homography ------------------------------------------------------------------------------------------------------------
def test_homography_matches_find_homography():
    pytest.importorskip("cv2")
    rng = np.random.default_rng(2)
    worst = 0.0
    for _ in range(2000):
        c = A.square(*rng.uniform(100, 900, 2), rng.uniform(20, 300), rng.uniform(0, 360)) + rng.normal(0, 8, (4, 2))
        c = c.astype(np.float32)
        def cross(a, b):
            return a[0] * b[1] - a[1] * b[0]
        if cross(c[1] - c[0], c[2] - c[0]) * cross(c[2] - c[0], c[3] - c[0]) <= 0:
            continue
        ref = A.homography_cv2(c)
        got = api.marker_homography(c)
        worst = max(worst, float(np.abs(got - ref).max() / np.abs(ref).max()))
    assert worst <= 1e-12, worst


@pytest.mark.parametrize("quad", [[[0, 0], [0, 0], [10, 10], [0, 10]], [[0, 0], [5, 5], [10, 10], [0, 10]],
                                  [[0, 0], [1, 0], [2, 0], [3, 0]], [[0, 0], [np.nan, 0], [10, 10], [0, 10]],
                                  [[0, 0], [np.inf, 0], [10, 10], [0, 10]]])
def test_degenerate_quads_are_errors(quad):
    with pytest.raises(api.MdcError):
        api.marker_homography(np.array(quad, np.float32))


# ---- golden sequence -------------------------------------------------------------------------------------------------------
def test_golden_sequence_is_the_specifications():
    pytest.importorskip("cv2")
    pytest.importorskip("scipy")
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
    import make_golden_marker as G
    from oracle.loader import PortOracle
    g = np.load(GOLDEN)
    port = PortOracle()
    with tempfile.TemporaryDirectory() as tmp:
        cam = os.path.join(tmp, "camera.txt")
        open(cam, "w").write(str(g["camera_txt"]))
        pf = port.fov_from_file(cam)
    for i, raw in enumerate(g["frames"]):
        grey, mask, ms, Hm = G.spec_frame(port, pf, raw)
        assert hashlib.sha256(grey.tobytes()).hexdigest() == g["grey_sha256"][i]
        assert hashlib.sha256(mask.tobytes()).hexdigest() == g["mask_sha256"][i]
        assert [m[0] for m in ms] + [-1] * (2 - len(ms)) == list(g["ids"][i])
        for k, m in enumerate(ms):
            assert np.array_equal(m[1], g["corners"][i][k])
        assert np.array_equal(Hm.ravel(), g["homographies"][i], equal_nan=True)
        got = api.marker_detect(grey, mask)                              # the host detector on the same bytes
        assert [m[0] for m in got] == [m[0] for m in ms]
        for (_, a), (_, b) in zip(got, ms):
            assert np.abs(a - b).max() <= CORNER_TOL


# ---- sanitizer fuzz --------------------------------------------------------------------------------------------------------
def test_random_and_adversarial_masks_never_trip_the_sanitizers(tmp_path):
    exe = str(tmp_path / "marker_fuzz")
    csrc = os.path.join(ROOT, "mono_dataset_code_b200", "csrc")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-I" + os.path.join(ROOT, "include"),
           "-I" + csrc, os.path.join(ROOT, "tests", "cpp", "marker_fuzz.cpp"), os.path.join(csrc, "mdc_marker.cpp"), "-o", exe]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        pytest.skip("no sanitizer-enabled g++ here: " + r.stdout[-300:])
    r = subprocess.run([exe, "400"], env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:]
    assert "rounds" in r.stdout
