"""tools/vignetteCalib_b200.cpp — the C++ host of the vignetteCalib front end and optimiser: builds and links against include/ +
libmdc_b200.so (CPU), and on a GPU
  - reproduces what the REFERENCE PROGRAM wrote for the same sequence (tests/golden/programs/vignette_calib.npz, produced by
    main_vignetteCalib.cpp compiled unmodified against stand-in aruco / findHomography; generator
    tests/golden/make_golden_vignette_program.py): log.txt, vignette.png,
    vignetteSmoothed.png, plane.png, to the whole-loop tolerance of mdc_vignette_calib;
  - writes exactly the files that mdc_vignette_calib gives when its inputs come from the CPU restatement of the front end
    (oport_vc_plane_maps -> mdc_fov_distort_coordinates -> oport_vc_mask_maps, oport_vc_prepare_image), which pins the tool's
    own front end bit for bit;
  - drops a frame whose homography row is NaN (no marker), keeping its exposure in the mean."""
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from conftest import ROOT
from mono_dataset_code_b200 import synthetic as S

LIBDIR = os.path.join(ROOT, "mono_dataset_code_b200", "lib")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "programs", "vignette_calib.npz")


def build_tool(tmp_path):
    exe = str(tmp_path / "vignetteCalib_b200")
    cmd = ["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++11", "-O2", "-Wall", "-I" + os.path.join(ROOT, "include"),
           "-I/usr/local/cuda/include", os.path.join(ROOT, "tools", "vignetteCalib_b200.cpp"), "-o", exe, "-L" + LIBDIR, "-lmdc_b200",
           "-L/usr/local/cuda/lib64", "-lcudart", "-lz", "-Wl,-rpath," + LIBDIR + ":/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return exe


def test_vignette_tool_builds_and_prints_usage(tmp_path):
    exe = build_tool(tmp_path)
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 1 and "usage: vignetteCalib_b200" in r.stdout
    r = subprocess.run([exe, str(tmp_path) + "/"], cwd=tmp_path, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 1 and "homographies=FILE is required" in r.stdout


def read_png(path):
    """PNG written with filter 0 on every row -> uint8 [h, w, c] or uint16 [h, w, c]."""
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, ihdr = 8, b"", None
    while pos < len(data):
        ln, tag = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + ln]
        assert struct.unpack(">I", data[pos + 8 + ln:pos + 12 + ln])[0] == zlib.crc32(tag + body) & 0xFFFFFFFF
        if tag == b"IHDR":
            ihdr = struct.unpack(">IIBBBBB", body)
        elif tag == b"IDAT":
            idat += body
        pos += 12 + ln
    w, h, depth, colour = ihdr[:4]
    ch = 3 if colour == 2 else 1
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, 1 + w * ch * depth // 8)
    assert np.all(raw[:, 0] == 0)
    px = raw[:, 1:]
    if depth == 16:
        px = px.copy().view(">u2").astype(np.uint16)
    return px.reshape(h, w, ch)


def to_u16(v):
    a = (v.astype(np.float64) * 254.9).astype(np.float32)
    a = (a.astype(np.float64) * 254.9).astype(np.float32).astype(np.float64)
    r = np.rint(a)
    return np.where(np.isnan(r), 0, np.clip(r, 0, 65535)).astype(np.uint16)


def plane_rgb(plane):
    fin = np.isfinite(plane)
    vmin, vmax = np.float32(plane[fin].min()), np.float32(plane[fin].max())
    with np.errstate(invalid="ignore"):
        c = (np.float32(255) * (plane - vmin) / (vmax - vmin)).astype(np.float32)
    g = np.where(fin, np.clip(c, 0, 255), 0).astype(np.uint8)
    rgb = np.stack([g, g, g], axis=1)
    rgb[~fin] = [255, 0, 0]
    return rgb


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def write_sequence(d, g, homographies=None):
    os.makedirs(d / "images")
    wI, hI = int(g["wI"]), int(g["hI"])
    for name, key in (("camera.txt", "camera_txt"), ("pcalib.txt", "pcalib_txt"), ("times.txt", "times_txt")):
        (d / name).write_text(str(g[key]))
    S.write_png_gray(str(d / "vignette.png"), S.vignette_image(wI, hI))
    for i, f in enumerate(g["frames"]):
        S.write_pgm(str(d / "images" / f"{i:05d}.pgm"), f.reshape(hI, wI))
    Hs = g["homographies"] if homographies is None else homographies
    np.savetxt(d / "homographies.txt", Hs, fmt="%.17g")


def run_tool(tmp_path, g, homographies=None, its=None):
    seq, work = tmp_path / "seq", tmp_path / "work"
    write_sequence(seq, g, homographies)
    work.mkdir()
    exe = build_tool(tmp_path)
    its = int(g["iterations"]) if its is None else its
    r = subprocess.run([exe, str(seq) + "/", "homographies=" + str(seq / "homographies.txt"), f"iterations={its}", f"patternX={int(g['gw'])}",
                        f"patternY={int(g['gh'])}"], cwd=work, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    out = work / "vignetteCalibResult"
    return r.stdout, dict(log=np.loadtxt(out / "log.txt", ndmin=2), vignette=read_png(out / "vignette.png")[:, :, 0],
                          smoothed=read_png(out / "vignetteSmoothed.png")[:, :, 0], plane=read_png(out / "plane.png"))


def restated(g, drop=()):
    """The tool's pipeline with the CPU restatement as the front end and mdc_vignette_calib as the loop."""
    import torch
    from mono_dataset_code_b200 import api
    from oracle.loader import PortOracle
    port = PortOracle()
    wI, hI, gw, gh, its = (int(g[k]) for k in ("wI", "hI", "gw", "gh", "iterations"))
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        cam = os.path.join(tmp, "camera.txt")
        open(cam, "w").write(str(g["camera_txt"]))
        fov = api.UndistorterFOV(cam)
    ginv, _ = port.photo_tables(np.array(str(g["pcalib_txt"]).split(), np.float32))
    expo = g["exposures"]
    mean = np.float32(0)
    for e in expo:                                                   # every frame counts, dropped or not (:222-227)
        mean = np.float32(mean + e)
    mean = np.float32(mean / np.float32(len(expo)))
    images, p2x, p2y = [], [], []
    for i in range(len(expo)):
        if i in drop:
            continue
        X, Y = port.vc_plane_maps(g["homographies"][i], gw, gh)
        fov.distortCoordinates(X, Y)
        port.vc_mask_maps(X, Y, wI, hI)
        raw = port.unmap(ginv, None, g["frames"][i], True, False, False)
        images.append(port.vc_prepare_image(raw, wI, hI, mean, expo[i]))
        p2x.append(X)
        p2y.append(Y)
    ctx = api.Context(None, None, 0)
    d = [torch.from_numpy(np.stack(a)).cuda() for a in (images, p2x, p2y)]
    pc, v = torch.zeros(gw * gh, dtype=torch.float32, device="cuda"), torch.ones(wI * hI, dtype=torch.float32, device="cuda")
    smoothed, log = ctx.vignette_calib(d[0], d[1], d[2], gw, gh, wI, hI, its, 15, pc, v, True)
    vig, plane = v.cpu().numpy(), pc.cpu().numpy()
    n = len(images)
    sq = np.sqrt((log[:, 2] / log[:, 3]).astype(np.float32))
    return dict(log=np.stack([np.arange(its), np.full(its, n), log[:, 3], sq], axis=1), vignette=to_u16(vig).reshape(hI, wI),
                smoothed=to_u16(smoothed.cpu().numpy()).reshape(hI, wI), plane=plane_rgb(plane).reshape(gh, gw, 3))


def test_fixture_is_consistent_with_the_restatement(golden):
    """CPU: the whole program replayed with the C restatement (front end and loop) gives the fixture's files — the same check as
    tests/test_vignette_calib_reference_program.py, on the stored run."""
    from oracle.loader import PortOracle
    port = PortOracle()
    wI, hI, gw, gh, its = (int(golden[k]) for k in ("wI", "hI", "gw", "gh", "iterations"))
    import tempfile
    with tempfile.TemporaryDirectory() as tmp:
        cam = os.path.join(tmp, "camera.txt")
        open(cam, "w").write(str(golden["camera_txt"]))
        fov = port.fov_from_file(cam)
    ginv, _ = port.photo_tables(np.array(str(golden["pcalib_txt"]).split(), np.float32))
    expo = golden["exposures"]
    mean = np.float32(0)
    for e in expo:
        mean = np.float32(mean + e)
    mean = np.float32(mean / np.float32(len(expo)))
    images, p2x, p2y = [], [], []
    for i in range(len(expo)):
        X, Y = fov.distort(*port.vc_plane_maps(golden["homographies"][i], gw, gh))
        port.vc_mask_maps(X, Y, wI, hI)
        images.append(port.vc_prepare_image(port.unmap(ginv, None, golden["frames"][i], True, False, False), wI, hI, mean, expo[i]))
        p2x.append(X)
        p2y.append(Y)
    images, p2x, p2y = np.stack(images), np.stack(p2x), np.stack(p2y)
    plane, vig, log = np.zeros(gw * gh, np.float32), np.ones(wI * hI, np.float32), []
    for it in range(its):
        oth2 = 15 * 15 if it >= its // 2 else 10000 * 10000
        plane, _, _, _ = port.vc_plane_step(images, p2x, p2y, wI, hI, vig, plane, oth2)
        vig, _, _, vs = port.vc_vignette_step(images, p2x, p2y, wI, hI, plane, vig, oth2)
        log.append([vs[1], np.sqrt(np.float32(vs[0] / vs[1]))])
    log = np.array(log)
    assert np.array_equal(log[:, 0], golden["log"][:, 2])
    assert np.max(np.abs(log[:, 1] - golden["log"][:, 3]) / golden["log"][:, 3]) < 1e-6
    assert np.array_equal(to_u16(vig).reshape(hI, wI), golden["vignette_png"])
    assert np.array_equal(to_u16(port.vc_smooth(vig, wI, hI, 4)).reshape(hI, wI), golden["vignette_smoothed_png"])
    assert np.array_equal(plane_rgb(plane).reshape(gh, gw, 3), golden["plane_png_bgr"][:, :, ::-1])


def assert_same_files(got, exp):
    assert got["log"].shape == exp["log"].shape
    assert np.array_equal(got["log"][:, :3], exp["log"][:, :3])
    assert np.array_equal(got["log"][:, 3].astype(np.float32), exp["log"][:, 3].astype(np.float32))     # 15 digits round-trip a float
    for k in ("vignette", "smoothed", "plane"):
        assert np.array_equal(got[k], exp[k]), k


@pytest.mark.gpu
def test_vignette_tool_reproduces_the_reference_program(tmp_path, golden):
    out, got = run_tool(tmp_path, golden)
    n = len(golden["frames"])
    assert f"loaded {n} images with a marker" in out and "residual terms =>" in out
    ref = golden["log"]
    assert got["log"].shape == ref.shape and np.all(got["log"][:, 1] == n)
    assert np.allclose(got["log"][:, 2], ref[:, 2], rtol=2e-3) and np.allclose(got["log"][:, 3], ref[:, 3], rtol=2e-3)
    for k, rk in (("vignette", "vignette_png"), ("smoothed", "vignette_smoothed_png")):
        a, b = got[k].astype(np.int64), golden[rk].astype(np.int64)
        assert np.mean((a == 0) == (b == 0)) >= 0.999, k
        both = (a != 0) & (b != 0)
        assert both.mean() > 0.5 and np.max(np.abs(a[both] - b[both])) <= 13, k          # 2e-4 x 254.9^2
    bgr = golden["plane_png_bgr"]
    ref_rgb = bgr[:, :, ::-1]
    red = np.array([255, 0, 0], np.uint8)
    fin = ~np.all(got["plane"] == red, axis=2) & ~np.all(ref_rgb == red, axis=2)
    assert np.mean(np.all(got["plane"] == red, axis=2) == np.all(ref_rgb == red, axis=2)) >= 0.999
    assert fin.mean() > 0.3 and np.max(np.abs(got["plane"][fin].astype(int) - ref_rgb[fin].astype(int))) <= 1


@pytest.mark.gpu
def test_vignette_tool_front_end_is_exact(tmp_path, golden):
    _, got = run_tool(tmp_path, golden)
    assert_same_files(got, restated(golden))


@pytest.mark.gpu
def test_vignette_tool_drops_frames_without_marker(tmp_path, golden):
    Hs = golden["homographies"].copy()
    Hs[3] = np.nan
    out, got = run_tool(tmp_path, golden, homographies=Hs)
    assert f"loaded {len(Hs) - 1} images with a marker" in out
    assert_same_files(got, restated(golden, drop=(3,)))
