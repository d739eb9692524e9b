"""GPU side of vignetteCalib's marker detection: mdc_marker_threshold bit for bit against the numpy specification (tests/aruco_spec.py,
no cv2 needed), the library chain on the golden marker sequence, and vignetteCalib_b200 with homographies=detect."""
import hashlib
import os
import shutil
import subprocess

import numpy as np
import pytest

import aruco_spec as A
from mono_dataset_code_b200 import api
from mono_dataset_code_b200 import synthetic as S

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "marker", "marker_sequence.npz")
CORNER_TOL = 2e-3


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def ctx():
    return api.Context(None, None, 0)


def _check_threshold(ctx, rect):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(rect, np.float32)).cuda()
    grey, mask = ctx.marker_threshold(t)
    torch.cuda.synchronize()
    g, m = grey.cpu().numpy(), mask.cpu().numpy()
    for i in range(rect.shape[0]):
        eg = A.grey_u8(rect[i])
        assert np.array_equal(g[i], eg), i
        assert np.array_equal(m[i], A.adaptive_threshold(eg)), i


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(1, 1), (3, 5), (8, 6), (1023, 1281), (31, 33), (1, 300), (300, 1)])
def test_threshold_kernel_is_the_specification_on_odd_sizes(ctx, hw):
    h, w = hw
    rng = np.random.default_rng(h + 3 * w)
    rect = np.stack([rng.uniform(-3, 258, (h, w)), np.zeros((h, w)), np.full((h, w), 255.0),
                     np.round(rng.uniform(0, 255, (h, w))) + 0.5]).astype(np.float32)
    _check_threshold(ctx, rect)


@pytest.mark.gpu
def test_threshold_kernel_on_rectified_frames(tmp_path, ctx):
    """K1-rectified 1280x1024 crop frames (noise and a marker scene), one frame and a batch of 300."""
    import torch
    d = str(tmp_path)
    S.write_dataset_dir(d, 1280, 1024, 1280, 1024, "crop")
    fov = api.UndistorterFOV(os.path.join(d, "camera.txt"))
    c = api.Context(fov, None, 0)
    scene = A.render(1280, 1024, [(A.marker_bits(613), A.square(640, 512, 300, 20))], ss=1)
    rng = np.random.default_rng(1)
    raw = np.clip(scene[None] + rng.normal(0, 8, (300, 1024, 1280)), 0, 255).astype(np.uint8)
    for n in (1, 300):
        frames = torch.from_numpy(raw[:n].reshape(n, -1)).cuda()
        rect = torch.empty((n, 1024 * 1280), dtype=torch.float32, device="cuda")
        c.prepare_batch(frames, api.RECTIFY, [rect])
        grey, mask = c.marker_threshold(rect.view(n, 1024, 1280))
        torch.cuda.synchronize()
        r = rect.view(n, 1024, 1280).cpu().numpy()
        g, m = grey.cpu().numpy(), mask.cpu().numpy()
        for i in sorted({0, n // 2, n - 1}):
            eg = A.grey_u8(r[i])
            assert np.array_equal(g[i], eg) and np.array_equal(m[i], A.adaptive_threshold(eg))
        assert np.array_equal(g, A.grey_u8(r))
    c.close()


def _golden_fov(tmp_path, g):
    cam = tmp_path / "camera.txt"
    cam.write_text(str(g["camera_txt"]))
    return api.UndistorterFOV(str(cam))


@pytest.mark.gpu
def test_library_chain_reproduces_the_golden_sequence(tmp_path, golden):
    import torch
    fov = _golden_fov(tmp_path, golden)
    c = api.Context(fov, None, 0)
    frames = golden["frames"]
    n, h, w = frames.shape
    rect = torch.empty((n, h * w), dtype=torch.float32, device="cuda")
    c.prepare_batch(torch.from_numpy(frames.reshape(n, -1)).cuda(), api.RECTIFY, [rect])
    grey, mask = c.marker_threshold(rect.view(n, h, w))
    torch.cuda.synchronize()
    grey, mask = grey.cpu().numpy(), mask.cpu().numpy()
    worst_c, worst_h = 0.0, 0.0
    for i in range(n):
        assert hashlib.sha256(grey[i].tobytes()).hexdigest() == golden["grey_sha256"][i]
        assert hashlib.sha256(mask[i].tobytes()).hexdigest() == golden["mask_sha256"][i]
        ms = api.marker_detect(grey[i], mask[i])
        ids = [m[0] for m in ms]
        assert ids + [-1] * (2 - len(ids)) == list(golden["ids"][i])
        for k, (_, corners) in enumerate(ms):
            worst_c = max(worst_c, float(np.abs(corners - golden["corners"][i][k]).max()))
        if len(ms) == 1:
            H = api.marker_homography(ms[0][1]).ravel()
            ref = golden["homographies"][i]
            worst_h = max(worst_h, float(np.abs(H - ref).max() / np.abs(ref).max()))
        else:
            assert np.all(np.isnan(golden["homographies"][i]))
    print(f"worst corner difference {worst_c:.3g} px, worst H difference {worst_h:.3g} relative")
    assert worst_c <= CORNER_TOL
    assert worst_h <= 1e-4            # 2e-3 px on markers of ~80 px moves H by ~5e-5 of its largest entry
    c.close()


def _write_dataset(d, g):
    os.makedirs(d / "images")
    h, w = g["frames"].shape[1:]
    (d / "camera.txt").write_text(str(g["camera_txt"]))
    (d / "pcalib.txt").write_text(str(g["pcalib_txt"]))
    (d / "times.txt").write_text(str(g["times_txt"]))
    S.write_png_gray(str(d / "vignette.png"), S.vignette_image(w, h))
    for i, f in enumerate(g["frames"]):
        S.write_pgm(str(d / "images" / f"{i:05d}.pgm"), f)


def _run(exe, seq, work, hom, its=4):
    work.mkdir(exist_ok=True)
    r = subprocess.run([exe, str(seq) + "/", "homographies=" + hom, f"iterations={its}", "patternX=200", "patternY=200"], cwd=work,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    return r.stdout


@pytest.mark.gpu
def test_vignette_tool_detects_the_markers_itself(tmp_path, golden):
    import test_vignette_calib_tool as T
    exe = T.build_tool(tmp_path)
    seq = tmp_path / "seq"
    _write_dataset(seq, golden)
    out = _run(exe, seq, tmp_path / "detect", "detect")
    res = tmp_path / "detect" / "vignetteCalibResult"
    assert sorted(os.listdir(res)) == ["homographies.txt", "log.txt", "plane.png", "vignette.png", "vignetteSmoothed.png"]
    Hd = np.loadtxt(res / "homographies.txt", ndmin=2)
    ref = golden["homographies"]
    assert Hd.shape == ref.shape
    assert np.array_equal(np.isnan(Hd), np.isnan(ref))
    fin = ~np.isnan(ref[:, 0])
    assert f"loaded {int(fin.sum())} images with a marker" in out
    assert np.all(np.abs(Hd[fin] - ref[fin]).max(1) / np.abs(ref[fin]).max(1) <= 1e-4)

    def files(d):
        r = d / "vignetteCalibResult"
        return dict(log=np.loadtxt(r / "log.txt", ndmin=2), vignette=T.read_png(r / "vignette.png")[:, :, 0],
                    smoothed=T.read_png(r / "vignetteSmoothed.png")[:, :, 0], plane=T.read_png(r / "plane.png"))
    got = files(tmp_path / "detect")
    replay = tmp_path / "replay.txt"
    shutil.copy(res / "homographies.txt", replay)
    _run(exe, seq, tmp_path / "replay", str(replay))
    T.assert_same_files(files(tmp_path / "replay"), got)                 # detect == replay of the rows it wrote

    spec = tmp_path / "spec.txt"
    np.savetxt(spec, ref, fmt="%.17g")
    _run(exe, seq, tmp_path / "spec", str(spec))
    exp = files(tmp_path / "spec")
    # the residual count and rms: the plane is flat, so late iterations reach rms ~1e-7 grey levels, where only an absolute bound means anything
    assert np.allclose(got["log"][:, 2], exp["log"][:, 2], rtol=2e-3) and np.allclose(got["log"][:, 3], exp["log"][:, 3], rtol=2e-3, atol=1e-5)
    for k in ("vignette", "smoothed"):
        a, b = got[k].astype(np.int64), exp[k].astype(np.int64)
        assert np.mean((a == 0) == (b == 0)) >= 0.999, k
        both = (a != 0) & (b != 0)
        assert np.max(np.abs(a[both] - b[both]), initial=0) <= 13, k
