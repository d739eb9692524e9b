"""vignetteCalib's front end (main_vignetteCalib.cpp:266-301, :346-357): the plane-to-image maps and the prepared images.

CPU: the numpy statement of the order-dependent gradient invalidation (tests/vc_invalidation_spec.py) against the C restatement
(oport_vc_prepare_image).  GPU: mdc_vc_plane_maps against oport_vc_plane_maps -> mdc_fov_distort_coordinates (host) ->
oport_vc_mask_maps, and mdc_vc_prepare_images against oport_vc_prepare_image, bit for bit."""
import numpy as np
import pytest

import vc_invalidation_spec as spec
from conftest import CALIBS, assert_bits_equal
from mono_dataset_code_b200 import synthetic as S


def noise(h, w, seed, lo=0.0, hi=255.0):
    return np.random.default_rng(seed).uniform(lo, hi, (h, w)).astype(np.float32)


def adversarial_cases():
    """(name, raw [h, w] float32, max_abs_grad, mean_exposure, exposure)"""
    out = []
    for g in (10, 40, 120, 255):
        out.append((f"noise_g{g}", noise(121, 161, g), g, 1.3, 0.9))
    out.append(("noise_wide_g255", noise(121, 161, 5, 0.0, 700.0), 255, 1.0, 1.0))
    H, W = 121, 161
    v = np.full((H, W), 20.0, np.float32)
    v[:, 80:] = 400.0
    out.append(("vertical_edge", v, 255, 1.0, 1.0))
    v = np.full((H, W), 20.0, np.float32)
    v[60:, :] = 400.0
    out.append(("horizontal_edge", v, 255, 1.0, 1.0))
    yy, xx = np.mgrid[0:H, 0:W]
    out.append(("diagonal_edge", np.where(xx > yy + 10, 400.0, 20.0).astype(np.float32), 255, 1.0, 1.0))
    out.append(("anti_diagonal_edge", np.where(xx + yy > 140, 400.0, 20.0).astype(np.float32), 255, 1.0, 1.0))
    out.append(("staircase", (20.0 + 300.0 * (xx // 3 % 2) + 5.0 * yy).astype(np.float32), 255, 1.0, 1.0))
    out.append(("checkerboard", np.where((xx + yy) % 2 == 0, 400.0, 20.0).astype(np.float32), 255, 1.0, 1.0))
    out.append(("checkerboard_2px", np.where((xx // 2 + yy // 2) % 2 == 0, 300.0, 0.0).astype(np.float32), 255, 0.8, 1.1))
    v = noise(H, W, 11, 0.0, 200.0)
    rng = np.random.default_rng(12)
    for val in (np.inf, -np.inf, np.nan):
        v[rng.integers(0, H, 60), rng.integers(0, W, 60)] = val
    v[:, 40] = np.inf
    v[30, :] = np.nan
    out.append(("inf_nan", v, 120, 1.0, 1.0))
    out.append(("overflow_to_inf", noise(H, W, 13, 1e37, 3e38), 255, 1e3, 1.0))
    for h, w in ((5, 5), (6, 7), (4, 9), (9, 4), (3, 3), (1, 1)):
        out.append((f"tiny_{h}x{w}", noise(h, w, h * 10 + w), 60, 1.0, 1.0))
        out.append((f"tiny_{h}x{w}_checker", np.where(np.add.outer(np.arange(h), np.arange(w)) % 2 == 0, 300.0, 0.0).astype(np.float32), 255, 1.0, 1.0))
    return out


CASES = adversarial_cases()


@pytest.fixture(scope="module")
def port():
    from oracle.loader import PortOracle
    return PortOracle()


# ------------------------------------------------------------------------------------------------ CPU: spec vs restatement
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_invalidation_spec_matches_the_restatement(port, case):
    name, raw, g, mean, t = case
    h, w = raw.shape
    exp = port.vc_prepare_image(raw.ravel(), w, h, mean, t, g)
    got = spec.prepare_image(raw.ravel(), w, h, mean, t, g)
    assert_bits_equal(got, exp, name)


def test_the_cases_are_what_they_claim():
    """Dense cases really are dense: most centres have a candidate hit, and the edges reach over the full height."""
    by = {c[0]: c for c in CASES}
    for name, frac in (("noise_g10", 0.9), ("checkerboard", 0.9), ("vertical_edge", 0.02), ("diagonal_edge", 0.02), ("horizontal_edge", 0.02)):
        _, raw, g, mean, t = by[name]
        img = spec.normalise(raw, mean, t)
        m = spec.candidate_masks(img, g)
        assert (m != 0).mean() > frac, name
        out = spec.invalidate(img, g)
        assert np.isnan(out).any(), name


def test_zero_exposure_counts_as_one(port):
    raw = noise(20, 30, 3)
    assert_bits_equal(spec.prepare_image(raw.ravel(), 30, 20, 1.5, 0.0, 40), port.vc_prepare_image(raw.ravel(), 30, 20, 1.5, 1.0, 40))


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def gpu():
    torch = pytest.importorskip("torch")
    from mono_dataset_code_b200 import api
    return torch, api, api.Context(None, None, 0)


@pytest.mark.gpu
@pytest.mark.parametrize("inplace", [False, True], ids=["out_of_place", "in_place"])
def test_prepare_images_adversarial_cases(port, gpu, inplace):
    torch, _, ctx = gpu
    for name, raw, g, mean, t in CASES:
        h, w = raw.shape
        exp = port.vc_prepare_image(raw.ravel(), w, h, mean, t, g)
        d = torch.from_numpy(raw.reshape(1, -1).copy()).cuda()
        got = ctx.vc_prepare_images(d, w, h, [t], mean, g, out=d if inplace else None)
        assert (got.data_ptr() == d.data_ptr()) == inplace
        assert_bits_equal(got.cpu().numpy()[0], exp, name)


@pytest.mark.gpu
def test_prepare_images_batched_same_size_cases(port, gpu):
    """All 121x161 cases in one call, each with its own exposure."""
    torch, _, ctx = gpu
    sel = [c for c in CASES if c[1].shape == (121, 161)]
    mean = 1.1
    expo = np.array([0.5 + 0.1 * i for i in range(len(sel))], np.float32)
    expo[3] = 0.0                                                    # counts as 1
    raw = np.stack([c[1].ravel() for c in sel])
    got = ctx.vc_prepare_images(torch.from_numpy(raw).cuda(), 161, 121, expo, mean, 120).cpu().numpy()
    for i, c in enumerate(sel):
        exp = port.vc_prepare_image(raw[i], 161, 121, mean, expo[i] if expo[i] != 0 else 1.0, 120)
        assert_bits_equal(got[i], exp, c[0])


@pytest.mark.gpu
def test_prepare_images_realistic_frames(port, gpu):
    """Gamma-unmapped camera frames at the reference's size (getImage(i, false, true, false, false), :265)."""
    torch, _, ctx = gpu
    w, h, n = 1280, 1024, 3
    ginv, _ = port.photo_tables(S.ginv_raw().astype(np.float32))
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    raws = []
    for i in range(n):
        rng = np.random.default_rng(40 + i)
        scene = 45 + 25 * np.sin(xx * 0.013 + i) * np.cos(yy * 0.011 - i) + 180 * (((xx // 64) + (yy // 64)) % 2)    # a calibration pattern
        f = np.clip(np.rint(scene + rng.normal(0, 3, scene.shape)), 0, 255).astype(np.uint8).ravel()
        raws.append(port.unmap(ginv, None, f, True, False, False))
    raws = np.stack(raws)
    expo = np.array([0.7, 1.3, 2.9], np.float32)
    mean = np.float32(expo.sum() / np.float32(n))
    d = torch.from_numpy(raws.copy()).cuda()
    ctx.vc_prepare_images(d, w, h, expo, mean, 255, out=d)
    got = d.cpu().numpy()
    for i in range(n):
        exp = port.vc_prepare_image(raws[i], w, h, mean, expo[i], 255)
        assert np.isnan(exp).mean() < 0.2 and (i == 2 or np.isnan(exp).mean() > 0.001)      # the pattern's edges, at the shorter exposures
        assert_bits_equal(got[i], exp, f"frame {i}")


@pytest.mark.gpu
def test_prepare_images_many_chunks(port, gpu):
    """More images than one chunk of the invalidation holds (512), dense, in place."""
    torch, _, ctx = gpu
    n, w, h = 1100, 13, 9
    rng = np.random.default_rng(8)
    raw = rng.uniform(0, 255, (n, w * h)).astype(np.float32)
    expo = rng.uniform(0.2, 3.0, n).astype(np.float32)
    d = torch.from_numpy(raw.copy()).cuda()
    ctx.vc_prepare_images(d, w, h, expo, 1.25, 40, out=d)
    got = d.cpu().numpy()
    for i in range(n):
        assert_bits_equal(got[i], port.vc_prepare_image(raw[i], w, h, 1.25, expo[i], 40), f"image {i}")


# ---- plane maps
def homographies(wI, hI):
    """Realistic marker poses plus the corner cases: a projective row that is zero on part of the grid, far outside the image,
    an almost-identity matrix."""
    Hs = []
    s = 0.12 * min(wI, hI)
    for i in range(5):
        ang = 0.3 * np.sin(i)
        Hs.append([s * np.cos(ang), -s * np.sin(ang), wI / 2 + 8 * np.cos(i), s * np.sin(ang), s * np.cos(ang), hI / 2 + 6 * np.sin(i),
                   0.004 * np.cos(i), -0.003 * np.sin(i), 1.0])
    Hs.append([s, 0, wI / 2, 0, s, hI / 2, 0, 0, 0])                 # pp[2] == 0 everywhere
    Hs.append([s, 0, wI / 2, 0, s, hI / 2, 1, 0, 0])                 # pp[2] == 0 on the column x = gw/2 (for an even gw)
    Hs.append([s, 0, wI / 2, 0, s, hI / 2, 0, 1, 0])                 # ... on the row y = gh/2
    Hs.append([s, 0, 1e6, 0, s, -1e6, 0, 0, 1])                      # far outside
    Hs.append([1e30, 0, 0, 0, 1e30, 0, 0, 0, 1])                     # overflows to inf
    Hs.append([1 + 1e-7, 2e-8, 1e-6, -3e-8, 1 - 1e-7, 2e-6, 1e-9, -1e-9, 1])   # almost the identity
    Hs.append([2.0 * s, 0.3 * s, wI / 2, -0.2 * s, 1.7 * s, hI / 2, 0.0, 0.0, 1.0])   # grid larger than the image
    return np.array(Hs, np.float64)


PLANE_CAMS = {"crop": (CALIBS["c1_crop_640"], False), "omega0": (CALIBS["omega0"], False), "crop_float_math": (CALIBS["odd_sizes"], True)}


def plane_maps_cpu(port, fov, H, gw, gh, facw, fach):
    wI, hI = fov.getInputDims()
    X, Y = port.vc_plane_maps(H, gw, gh, facw, fach)
    fov.distortCoordinates(X, Y)                                     # mdc_fov_distort_coordinates (host)
    port.vc_mask_maps(X, Y, wI, hI)
    return X, Y


@pytest.mark.gpu
@pytest.mark.parametrize("cam", list(PLANE_CAMS), ids=list(PLANE_CAMS))
@pytest.mark.parametrize("gw,gh", [(97, 53), (1000, 1000)], ids=["97x53", "1000x1000"])
def test_plane_maps_are_bit_identical(port, gpu, dataset_dir, cam, gw, gh):
    torch, api, _ = gpu
    cfg, float_math = PLANE_CAMS[cam]
    fov = api.UndistorterFOV(dataset_dir(cfg)["camera"], float_math=float_math)
    assert fov.isValid()
    wI, hI = fov.getInputDims()
    facw, fach = (5.0, 5.0) if gw == 1000 else (3.5, 6.0)
    Hs = homographies(wI, hI)
    p2x = torch.empty((len(Hs), gw * gh), dtype=torch.float32, device="cuda")
    p2y = torch.empty_like(p2x)
    fov.vcPlaneMaps(Hs, gw, gh, p2x, p2y, facw, fach)
    gx, gy = p2x.cpu().numpy(), p2y.cpu().numpy()
    for i, H in enumerate(Hs):
        X, Y = plane_maps_cpu(port, fov, H, gw, gh, facw, fach)
        assert_bits_equal(gx[i], X, f"p2x of homography {i}")
        assert_bits_equal(gy[i], Y, f"p2y of homography {i}")
    visible = np.isfinite(gx).mean(axis=1)
    assert visible[:5].min() > 0.05 and visible[5] == 0 and visible[8] == 0
    if gw == 1000:                                                   # the zero denominators really occur on this grid
        X, _ = port.vc_plane_maps(Hs[6], gw, gh, facw, fach)
        assert not np.all(np.isfinite(X.reshape(gh, gw)[:, gw // 2]))
