"""GPU parity tests (run on the H100 box): the CUDA path, called through the C ABI, against the
plain-C oracle on the same seeded inputs and against the committed golden fixtures.

Bar: BIT-EXACT floats (NaN positions identical, payloads ignored) — stronger than the 1e-4
relative tolerance BASELINE.json asks for; TOL_REL documents that contract anyway."""
import glob
import os

import numpy as np
import pytest

import gstep_fixed_point_spec as fx_spec
import pyramid_spec
from conftest import CALIBS, BIG_CALIBS, ROOT, assert_bits_equal
from mono_dataset_code_b200 import synthetic as S

pytestmark = pytest.mark.gpu
TOL_REL = 1e-4   # north_star tolerance; the assertions below are exact, so it is never exceeded

torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def api():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from mono_dataset_code_b200 import api as a
    return a


def make_models(api, files, iw, ih):
    u = api.UndistorterFOV(files["camera"])
    p = api.PhotometricUndistorter(files["pcalib"], files["vignette"], iw, ih)
    assert u.isValid() and p.validGamma and p.validVignette
    return u, p


def oracle_tables(port, files):
    f = port.fov_from_file(files["camera"])
    rx, ry = f.tables()
    ginv, _ = port.photo_tables(np.loadtxt(files["pcalib"], dtype=np.float32))
    _, vinv = port.vignette_maps(files["vignette_pixels"])
    return rx, ry, ginv, vinv.reshape(-1)


def mixed_frames(n, w, h):
    kinds = ["uniform", "speckle", "gradient", "white", "black"]
    return np.stack([S.frame(i, w, h, kinds[i % len(kinds)]) for i in range(n)])


LOADER_ID = {"ldg": 0, "tma": 1, "tex": 2, "hybrid": 3}


def select_loader(prep, loader):
    """Force one of K1's input loaders (include/mdc_b200.h MDC_LOADER_*); skip where it cannot describe the geometry."""
    if not prep.ctx.loader_usable(loader):
        pytest.skip(f"the {loader} loader is not usable for this geometry on this device (the other loaders cover it)")
    prep.ctx.configure(use_tma=LOADER_ID[loader])


def usable_loaders(prep):
    return [i for n, i in LOADER_ID.items() if prep.ctx.loader_usable(n)]


@pytest.mark.parametrize("name", list(CALIBS))
@pytest.mark.parametrize("loader", ["hybrid", "tex", "tma", "ldg"])
def test_get_image_all_flag_combinations(name, loader, api, port, dataset_dir):
    iw, ih, ow, oh, mode, calib = CALIBS[name]
    files = dataset_dir(name, vignette_zeros=(name in ("odd_sizes", "c1_crop_640")))
    u, p = make_models(api, files, iw, ih)
    prep = api.FramePreparer(u, p)
    select_loader(prep, loader)
    rx, ry, ginv, vinv = oracle_tables(port, files)
    frames = mixed_frames(7, iw, ih)
    d_frames = torch.from_numpy(frames).cuda()
    for flags in range(16):
        rectify, g, v, k = flags & 1, (flags >> 1) & 1, (flags >> 2) & 1, (flags >> 3) & 1
        out = prep.prepare_device(d_frames, rectify, g, v, k)[0].cpu().numpy()
        for i in range(frames.shape[0]):
            exp = port.get_image(rx, ry, iw, ih, ginv, vinv, frames[i], rectify, g, v, k)
            assert_bits_equal(out[i], exp, f"{name}/{loader} flags={flags} frame={i}")


@pytest.mark.parametrize("name", ["c1_crop_640", "odd_sizes", "upscale", "full_blackpx"])
@pytest.mark.parametrize("loader", ["tex", "tma", "ldg"])
def test_pyramid_levels(name, loader, api, port, dataset_dir):
    iw, ih, ow, oh, mode, calib = CALIBS[name]
    files = dataset_dir(name)
    u, p = make_models(api, files, iw, ih)
    prep = api.FramePreparer(u, p)
    select_loader(prep, loader)
    rx, ry, ginv, vinv = oracle_tables(port, files)
    frames = mixed_frames(5, iw, ih)
    d_frames = torch.from_numpy(frames).cuda()
    for levels, flags in [(5, (1, 1, 1, 1)), (3, (1, 1, 1, 0)), (7, (1, 0, 0, 0)), (4, (0, 1, 1, 0))]:
        outs = [o.cpu().numpy() for o in prep.prepare_device(d_frames, *flags, levels=levels)]
        w0, h0 = (ow, oh) if flags[0] else (iw, ih)
        for i in range(frames.shape[0]):
            lvl0 = port.get_image(rx, ry, iw, ih, ginv, vinv, frames[i], *flags)
            exp = port.pyramid(lvl0, w0, h0, levels)
            spec = pyramid_spec.pyramid(lvl0, w0, h0, levels)      # second, independently written formulation (DSO makeImages)
            for l in range(levels):
                assert outs[l].shape[1] == (w0 >> l) * (h0 >> l)
                assert_bits_equal(outs[l][i], exp[l], f"{name}/{loader} levels={levels} flags={flags} frame={i} level={l}")
                assert_bits_equal(outs[l][i], spec[l], f"{name}/{loader} vs DSO spec levels={levels} flags={flags} frame={i} level={l}")


GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.npz")))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_against_reference_golden_vectors(path, api, tmp_path):
    """Outputs of the reference's own compiled code (tests/golden/make_golden.py)."""
    g = np.load(path)
    iw, ih, ow, oh = [int(v) for v in g["dims"]]
    cam, pc, vig = tmp_path / "camera.txt", tmp_path / "pcalib.txt", tmp_path / "vignette.png"
    cam.write_bytes(g["camera_txt"].tobytes())
    pc.write_bytes(g["pcalib_txt"].tobytes())
    S.write_png_gray(str(vig), g["vignette_pixels"])
    u = api.UndistorterFOV(str(cam))
    p = api.PhotometricUndistorter(str(pc), str(vig), iw, ih)
    prep = api.FramePreparer(u, p)
    d_frames = torch.from_numpy(g["frames"]).cuda()
    for use_tma in usable_loaders(prep) + [-1]:
        prep.ctx.configure(use_tma=use_tma)
        for flags in range(16):
            rectify, gm, v, k = flags & 1, (flags >> 1) & 1, (flags >> 2) & 1, (flags >> 3) & 1
            out = prep.prepare_device(d_frames, rectify, gm, v, k)[0].cpu().numpy()
            assert_bits_equal(out, g[f"out_{flags:02d}"], f"golden flags={flags} tma={use_tma}")
    # host-buffer entry point (what the C++ compat classes call): one frame at a time
    for flags in (0, 1, 7, 15):
        img = prep.getImage(g["frames"][1].reshape(ih, iw), 1, flags & 1, (flags >> 1) & 1, (flags >> 2) & 1, (flags >> 3) & 1)
        assert_bits_equal(img.image, g[f"out_{flags:02d}"][1], f"golden host getImage flags={flags}")


def test_standalone_operators_and_error_behaviour(api, port, dataset_dir, capfd):
    iw, ih, ow, oh, mode, calib = CALIBS["c1_crop_640"]
    files = dataset_dir("c1_crop_640")
    u, p = make_models(api, files, iw, ih)
    rx, ry, ginv, vinv = oracle_tables(port, files)
    img = S.frame(4, iw, ih, "speckle")
    # unMapImage on host buffers, all 8 flag combinations
    for g in (0, 1):
        for v in (0, 1):
            for k in (0, 1):
                out = np.zeros(iw * ih, np.float32)
                p.unMapImage(img, out, iw * ih, g, v, k)
                assert_bits_equal(out, port.unmap(ginv, vinv, img, g, v, k), f"unMapImage {g}{v}{k}")
    # undistort<uchar> and undistort<float> on host buffers
    out = np.zeros(ow * oh, np.float32)
    u.undistort(img, out, iw * ih, ow * oh)
    assert_bits_equal(out, port.undistort(rx, ry, iw, img), "undistort<uchar>")
    fl = port.unmap(ginv, vinv, img, 1, 1, 1)
    u.undistort(fl, out, iw * ih, ow * oh)
    assert_bits_equal(out, port.undistort(rx, ry, iw, fl), "undistort<float>")
    # device tensors
    d_img = torch.from_numpy(fl).cuda()
    d_out = torch.zeros(ow * oh, dtype=torch.float32, device="cuda")
    u.undistort(d_img, d_out)
    assert_bits_equal(d_out.cpu().numpy(), port.undistort(rx, ry, iw, fl), "undistort<float> device")
    # wrong pixel counts: message + output untouched (FOVUndistorter.cpp:327-338)
    out[:] = 7.0
    u.undistort(img, out, iw * ih - 1, ow * oh)
    u.undistort(img, out, iw * ih, ow * oh + 3)
    assert (out == 7.0).all()
    assert "wrong input image dismesions" in capfd.readouterr().out
    # photometric object with invalid vignette: undoVignette silently drops to gamma only
    p2 = api.PhotometricUndistorter(files["pcalib"], "/nonexistent.png", iw, ih)
    out2 = np.zeros(iw * ih, np.float32)
    p2.unMapImage(img, out2, iw * ih, True, True, False)
    assert_bits_equal(out2, port.unmap(ginv, None, img, 1, 1, 0), "gamma-only fallback")
    # getImage refuses wrong-size / wrong-type frames like the reference (returns 0)
    prep = api.FramePreparer(u, p)
    assert prep.getImage(np.zeros((ih, iw + 1), np.uint8), 0, True, True, True, False) is None
    assert prep.getImage(np.zeros((ih, iw), np.uint16), 0, True, True, True, False) is None


def test_stand_alone_pyr_down_matches_fused_epilogue(api, port, dataset_dir):
    iw, ih, ow, oh, mode, calib = CALIBS["odd_sizes"]
    files = dataset_dir("odd_sizes")
    u, p = make_models(api, files, iw, ih)
    prep = api.FramePreparer(u, p)
    d_frames = torch.from_numpy(mixed_frames(3, iw, ih)).cuda()
    outs = prep.prepare_device(d_frames, 1, 1, 1, 0, levels=5)
    for l in range(1, 5):
        dst = torch.empty_like(outs[l])
        prep.ctx.pyr_down(outs[l - 1], ow >> (l - 1), oh >> (l - 1), dst, n_frames=3)
        assert_bits_equal(dst.cpu().numpy(), outs[l].cpu().numpy(), f"K2 vs fused level {l}")


@pytest.mark.parametrize("name", list(BIG_CALIBS))
def test_full_size_configs(name, api, port, dataset_dir):
    """BASELINE.json configs[1]/[3] geometry: a handful of frames against the oracle, then the
    size-independent properties on a larger batch (batch position independence; pyramid closure)."""
    iw, ih, ow, oh, mode, calib = BIG_CALIBS[name]
    files = dataset_dir(name)
    u, p = make_models(api, files, iw, ih)
    prep = api.FramePreparer(u, p)
    rx, ry, ginv, vinv = oracle_tables(port, files)
    frames = mixed_frames(4, iw, ih)
    n_big = 64
    big = torch.from_numpy(np.concatenate([frames] * (n_big // 4))).cuda()
    for use_tma in usable_loaders(prep) + [-1]:
        prep.ctx.configure(use_tma=use_tma)
        outs = prep.prepare_device(big, 1, 1, 1, 1, levels=5)
        lv = [o.cpu().numpy() for o in outs]
        for i in range(4):
            exp = port.pyramid(port.get_image(rx, ry, iw, ih, ginv, vinv, frames[i], 1, 1, 1, 1), ow, oh, 5)
            for l in range(5):
                assert_bits_equal(lv[l][i], exp[l], f"{name} tma={use_tma} frame={i} level={l}")
        # every replica of a frame in the batch gives the same bits, wherever the schedule put it
        for l in range(5):
            a = lv[l].reshape(n_big // 4, 4, -1)
            assert np.array_equal(a.view(np.uint32), np.broadcast_to(a[:1], a.shape).view(np.uint32)), f"batch position dependence, level {l}"


def test_batch_beyond_4gb_and_2g_elements(api, port, dataset_dir):
    """1700 C2 frames in ONE call: 2.2 GB of input, level 0 alone is 8.9 GB = 2.2e9 floats, so every frame offset past
    ~frame 1638 needs 64-bit element arithmetic (and every one past ~819 64-bit byte arithmetic).  Frames repeat with period 4:
    the first four are checked against the oracle, all others against those, on the device."""
    name = "c2_crop_1280"
    iw, ih, ow, oh, mode, calib = BIG_CALIBS[name]
    files = dataset_dir(name)
    u, p = make_models(api, files, iw, ih)
    prep = api.FramePreparer(u, p)
    rx, ry, ginv, vinv = oracle_tables(port, files)
    frames = mixed_frames(4, iw, ih)
    n = 1700
    big = torch.from_numpy(frames).cuda().repeat(n // 4, 1)
    assert big.shape == (n, iw * ih)
    for use_tma in usable_loaders(prep) + [-1]:
        prep.ctx.configure(use_tma=use_tma)
        outs = prep.prepare_device(big, 1, 1, 1, 1, levels=3)
        for i in range(4):
            exp = port.pyramid(port.get_image(rx, ry, iw, ih, ginv, vinv, frames[i], 1, 1, 1, 1), ow, oh, 3)
            for l in range(3):
                assert_bits_equal(outs[l][i].cpu().numpy(), exp[l], f"tma={use_tma} frame={i} level={l}")
        for l in range(3):
            a = outs[l].view(torch.int32).view(n // 4, 4, -1)
            for lo in range(0, n // 4, 25):      # compare in slabs to bound the temporaries
                assert bool((a[lo:lo + 25] == a[:1]).all()), f"tma={use_tma} level {l}: frames {4 * lo}.. differ from their replicas"
        del outs
    torch.cuda.empty_cache()


@pytest.mark.parametrize("name", list(CALIBS))
def test_distort_coordinates_on_device_is_bit_identical(name, api, dataset_dir):
    """SURVEY.md §8f N3: distortCoordinates (FOVUndistorter.cpp:280-319) as a batched device op, against the host version
    (which is itself pinned against the reference build in the CPU suite)."""
    iw, ih, ow, oh, mode, calib = CALIBS[name]
    files = dataset_dir(name)
    u = api.UndistorterFOV(files["camera"])
    rng = np.random.default_rng(31)
    n = 200_003
    x = rng.uniform(-0.5 * ow, 1.5 * ow, n).astype(np.float32)
    y = rng.uniform(-0.5 * oh, 1.5 * oh, n).astype(np.float32)
    x[:4] = [0.0, ow - 1.0, u.getK_rect()[0, 2], -0.0]
    y[:4] = [0.0, oh - 1.0, u.getK_rect()[1, 2], 3.0]        # includes the principal point (radius 0 -> scale 1)
    hx, hy = x.copy(), y.copy()
    u.distortCoordinates(hx, hy)
    dx, dy = torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda()
    u.distortCoordinatesDevice(dx, dy)
    assert_bits_equal(dx.cpu().numpy(), hx, f"{name} x")
    assert_bits_equal(dy.cpu().numpy(), hy, f"{name} y")
    # the identity grid reproduces the remap tables before clamping/blackening: compare where the table keeps the value
    gx, gy = np.meshgrid(np.arange(ow, dtype=np.float32), np.arange(oh, dtype=np.float32))
    dgx, dgy = torch.from_numpy(gx.ravel().copy()).cuda(), torch.from_numpy(gy.ravel().copy()).cuda()
    u.distortCoordinatesDevice(dgx, dgy)
    rx, ry = u.remap_tables()
    keep = (rx > 0.011) & (ry > 0.011) & (rx < iw - 1.011) & (ry < ih - 1.011)
    assert keep.any() or name == "full_wrap"
    assert np.array_equal(dgx.cpu().numpy()[keep].view(np.uint32), rx[keep].view(np.uint32))
    assert np.array_equal(dgy.cpu().numpy()[keep].view(np.uint32), ry[keep].view(np.uint32))


def test_estep_bit_exact(api, port):
    rng = np.random.default_rng(11)
    # (4100, 640): more exposures than the kernel caches in shared memory -> times come through L1; (5, 130): shorter than one
    # software-pipeline group; 1001 / 130: image sizes that are not a multiple of 4 (byte-wise tail path)
    for n, npix in [(37, 4096), (20, 1001), (64, 12 * 1024), (4100, 640), (5, 130), (27, 1536 * 300 + 16)]:
        data = rng.integers(0, 256, (n, npix), dtype=np.uint8)
        data[:, 5] = 255                       # never-valid pixel -> 0/0 = NaN survives the clamp
        data[:, 7] = 0
        t = rng.uniform(0.05, 20.0, n).astype(np.float32).astype(np.float64)   # exposures come through a float (main_responseCalib.cpp:209)
        G = np.sort(rng.uniform(-5, 300, 256))
        G[3] = -2.0
        exp = port.estep(data, t, G)
        ctx = api.Context(None, None, 0)
        E = torch.zeros(npix, dtype=torch.float64, device="cuda")
        ctx.estep(torch.from_numpy(data).cuda(), torch.from_numpy(t).cuda(), torch.from_numpy(G).cuda(), E)
        assert_bits_equal(E.cpu().numpy(), exp, f"E-step n={n} npix={npix}")
        assert np.isnan(exp[5])
        # the same planes at a base address that is 4- but not 16-byte aligned: the bulk-copy loader does not apply,
        # the register-pipelined loader must give the same bits
        shifted = torch.empty(n * npix + 4, dtype=torch.uint8, device="cuda")[4:].view(n, npix)
        shifted.copy_(torch.from_numpy(data))
        E.zero_()
        ctx.estep(shifted, torch.from_numpy(t).cuda(), torch.from_numpy(G).cuda(), E)
        assert_bits_equal(E.cpu().numpy(), exp, f"E-step (unaligned base) n={n} npix={npix}")


def test_multi_gpu_style_adopted_tables(api, port, dataset_dir):
    """Context built from device tables (the path ranks > 0 take after the NCCL broadcast)."""
    iw, ih, ow, oh, mode, calib = CALIBS["c1_crop_640"]
    files = dataset_dir("c1_crop_640")
    u, p = make_models(api, files, iw, ih)
    rx, ry = u.remap_tables()
    t = [torch.from_numpy(a).cuda() for a in (rx, ry, p.getGInv(), p.vignette_maps()[1])]
    ctx = api.Context.from_device_tables(0, iw, ih, ow, oh, *t)
    frames = mixed_frames(3, iw, ih)
    d = torch.from_numpy(frames).cuda()
    out = torch.empty((3, ow * oh), dtype=torch.float32, device="cuda")
    ctx.prepare_batch(d, 1 | 2 | 4, [out])
    prx, pry, ginv, vinv = oracle_tables(port, files)
    for i in range(3):
        assert_bits_equal(out[i].cpu().numpy(), port.get_image(prx, pry, iw, ih, ginv, vinv, frames[i], 1, 1, 1, 0), f"adopted ctx frame {i}")


def test_host_pipeline_with_pyramid_and_many_chunks(api, port, dataset_dir):
    """mdc_prepare_batch_host: 3-deep chunked H2D/kernel/D2H pipeline, frame count not a multiple of the chunk,
    pyramid levels beyond the in-kernel ones (K2 chain), pageable host memory."""
    iw, ih, ow, oh, mode, calib = CALIBS["tum_explicit"]
    files = dataset_dir("tum_explicit")
    u, p = make_models(api, files, iw, ih)
    prep = api.FramePreparer(u, p)
    rx, ry, ginv, vinv = oracle_tables(port, files)
    n = 37
    frames = mixed_frames(n, iw, ih)
    levels = 6
    outs = [np.full((n, (ow >> l) * (oh >> l)), -1.0, np.float32) for l in range(levels)]
    prep.ctx.prepare_batch_host(frames, 1 | 2 | 4 | 8, outs)
    for i in (0, 1, 15, 16, 17, 35, 36):
        exp = port.pyramid(port.get_image(rx, ry, iw, ih, ginv, vinv, frames[i], 1, 1, 1, 1), ow, oh, levels)
        for l in range(levels):
            assert_bits_equal(outs[l][i], exp[l], f"host pipeline frame={i} level={l}")


def test_many_frames_cross_chunk_boundaries(api, port, dataset_dir):
    """More frames than one schedule chunk (48) on a small geometry: every frame must come out right whatever
    item/CTA processed it."""
    iw, ih, ow, oh, mode, calib = CALIBS["omega0"]
    files = dataset_dir("omega0")
    u, p = make_models(api, files, iw, ih)
    prep = api.FramePreparer(u, p)
    rx, ry, ginv, vinv = oracle_tables(port, files)
    n = 131
    frames = mixed_frames(n, iw, ih)
    d = torch.from_numpy(frames).cuda()
    for use_tma in usable_loaders(prep) + [-1]:
        prep.ctx.configure(use_tma=use_tma)
        out = prep.prepare_device(d, 1, 1, 1, 0, levels=3)
        lv = [o.cpu().numpy() for o in out]
        for i in range(n):
            exp = port.pyramid(port.get_image(rx, ry, iw, ih, ginv, vinv, frames[i], 1, 1, 1, 0), ow, oh, 3)
            for l in range(3):
                assert_bits_equal(lv[l][i], exp[l], f"tma={use_tma} frame={i} level={l}")


def test_estep_non_finite_and_negative_exposures(api, port):
    """Saturated samples are skipped, never multiplied: t[i] = inf, a negative t[i] and a NaN table entry must come out
    exactly as the reference's `continue` leaves them (main_responseCalib.cpp:329)."""
    rng = np.random.default_rng(12)
    n, npix = 9, 2048
    data = rng.integers(250, 256, (n, npix), dtype=np.uint8)       # many saturated samples
    t = rng.uniform(0.5, 2.0, n)
    t[4] = np.inf
    t[6] = -1.25
    G = np.linspace(0.0, 255.0, 256)
    G[255] = np.nan                                                # only ever met by saturated samples
    exp = port.estep(data, t, G)
    ctx = api.Context(None, None, 0)
    E = torch.zeros(npix, dtype=torch.float64, device="cuda")
    ctx.estep(torch.from_numpy(data).cuda(), torch.from_numpy(t).cuda(), torch.from_numpy(G).cuda(), E)
    assert_bits_equal(E.cpu().numpy(), exp, "E-step with t=inf")


@pytest.mark.parametrize("w,h", [(96, 64), (50, 30)], ids=["bulk_loader_16px_multiple", "generic_size"])
def test_response_calib_building_blocks(api, port, w, h):
    """SURVEY.md §8f N2: leak padding / E-init / rescale bit-exact; G-step and rmse to rounding (the reference sums
    10^5..10^9 terms sequentially, the GPU in parallel): TOL_SUM relative."""
    TOL_SUM = 1e-10
    rng = np.random.default_rng(21)
    n = 23
    npix = w * h
    data = rng.integers(0, 256, (n, npix), dtype=np.uint8)
    data[:, 100:140] = 255                          # a saturated blob
    data[3, 0] = data[5, npix - 1] = 255            # border pixels never spread
    t = rng.uniform(0.05, 20.0, n).astype(np.float32).astype(np.float64)
    ctx = api.Context(None, None, 0)
    # leak padding, 0..3 iterations
    for iters in (1, 2, 3):
        d = torch.from_numpy(data.copy()).cuda()
        ctx.rc_leak_padding(d, w, h, iters)
        exp = np.stack([port.leak_padding(data[i], w, h, iters) for i in range(n)])
        assert np.array_equal(d.cpu().numpy(), exp), f"leak padding x{iters}"
    padded = np.stack([port.leak_padding(data[i], w, h, 2) for i in range(n)])
    d = torch.from_numpy(padded).cuda()
    dt = torch.from_numpy(t).cuda()
    # E-init
    E = torch.zeros(npix, dtype=torch.float64, device="cuda")
    ctx.rc_einit(d, E)
    E_ref = port.einit(padded)
    assert_bits_equal(E.cpu().numpy(), E_ref, "E-init")
    # G-step
    G = torch.zeros(256, dtype=torch.float64, device="cuda")
    ctx.rc_gstep(d, dt, E, G)
    G_ref = port.gstep(padded, t, E_ref)
    g = G.cpu().numpy()
    assert np.array_equal(np.isnan(g), np.isnan(G_ref))
    m = ~np.isnan(G_ref)
    assert np.max(np.abs(g[m] - G_ref[m]) / np.maximum(np.abs(G_ref[m]), 1e-300)) < TOL_SUM
    # rmse
    r = ctx.rc_rmse(d, dt, G, E)
    r_ref = port.rmse(padded, t, G_ref, E_ref)
    assert r[1] == r_ref[1] and abs(r[0] - r_ref[0]) <= TOL_SUM * 10 * abs(r_ref[0])
    # rescale (bit-exact on identical inputs)
    Gc, Ec = torch.from_numpy(G_ref.copy()).cuda(), torch.from_numpy(E_ref.copy()).cuda()
    f = ctx.rc_rescale(Ec, Gc)
    E2, G2 = E_ref.copy(), G_ref.copy()
    f_ref = port.rescale(E2, G2)
    assert f == f_ref
    assert_bits_equal(Ec.cpu().numpy(), E2, "rescaled E")
    assert_bits_equal(Gc.cpu().numpy(), G2, "rescaled G")


@pytest.mark.parametrize("npix", [96 * 64, 50 * 30 + 7], ids=["bulk_loader", "generic_kernel"])
def test_gstep_sums_are_exact_and_repeatable(api, port, npix):
    """The G-step sums E[k]*t[i] in 128-bit fixed point (DESIGN.md §4 N2): the bits of G must not depend on the run, on the tile
    width of the launch or on the order of the atomics, and each bin must be the correctly rounded EXACT sum of the fp64 products
    (math.fsum) to well inside the distance between the reference's own sequential chain and that exact sum."""
    import math
    rng = np.random.default_rng(5)
    n = 37
    data = rng.integers(0, 256, (n, npix), dtype=np.uint8)
    data[:, 11:40] = 255
    data[:, 200:260] = 7                                   # one crowded bin: thousands of colliding atomics
    t = rng.uniform(0.05, 20.0, n)
    t[3] = -1.25                                           # the arithmetic has no sign assumption
    E = np.exp(rng.uniform(-12.0, 6.0, npix))              # 8 decades of irradiance
    ctx = api.Context(None, None, 0)
    d, dt, dE = torch.from_numpy(data).cuda(), torch.from_numpy(t).cuda(), torch.from_numpy(E).cuda()
    runs = []
    for warps in ("", "10", "14", "3", ""):
        if warps:
            os.environ["MDC_STREAM_WARPS"] = warps
        else:
            os.environ.pop("MDC_STREAM_WARPS", None)
        G = torch.zeros(256, dtype=torch.float64, device="cuda")
        ctx.rc_gstep(d, dt, dE, G)
        runs.append(G.cpu().numpy())
    os.environ.pop("MDC_STREAM_WARPS", None)
    for r in runs[1:]:
        assert_bits_equal(r, runs[0], "G-step, repeated / other tile widths")
    assert_bits_equal(runs[0], fx_spec.gstep(data, t, E), "G-step vs the numpy specification of the fixed-point sums")
    prod = E[None, :] * t[:, None]                         # fp64 products, rounded like the reference rounds them
    G_ref = port.gstep(data, t, E)
    pmax = np.abs(E).max() * np.abs(t).max()
    worst = 0.0
    for b in range(255):
        m = data == b
        cnt = int(m.sum())
        if cnt == 0:
            continue
        exact = math.fsum(prod[m].tolist()) / cnt
        # every sample is rounded to a multiple of 2^-s <= 2^-47 * pmax, so a bin's MEAN is off by at most 2^-48 * pmax = 3.6e-15 * pmax (+ the final roundings)
        assert abs(runs[0][b] - exact) <= 4e-15 * pmax + 1e-15 * abs(exact), b
        worst = max(worst, abs(G_ref[b] - exact) / abs(exact))
    assert worst < 1e-10                                   # the oracle's sequential chain, for scale
    # a NaN irradiance poisons exactly the bins its pixel has samples in, as in the reference
    E2 = E.copy(); E2[500] = np.nan
    G = torch.zeros(256, dtype=torch.float64, device="cuda")
    ctx.rc_gstep(d, dt, torch.from_numpy(E2).cuda(), G)
    assert np.array_equal(np.isnan(G.cpu().numpy()), np.isnan(port.gstep(data, t, E2)))
    assert_bits_equal(G.cpu().numpy(), fx_spec.gstep(data, t, E2), "G-step with a NaN irradiance vs the specification")


def test_streaming_ring_reused_many_times(api, port):
    """300 exposures = 38 plane groups through the 3-stage bulk-copy ring of the calibrator's streaming kernels: every stage is refilled a
    dozen times per tile while the consumers are still a group or two behind, and the G-step folds its limb histograms in mid-run.
    E must be the oracle's bits, G exact, rmse the oracle's count, on every one of several runs (compute-sanitizer's racecheck cannot
    follow the empty-barrier hand-over of a 1-D bulk copy and reports it as a hazard; this is the functional check of that hand-over)."""
    import math
    rng = np.random.default_rng(31)
    n, npix = 300, 1792 * 3 + 128
    data = rng.integers(0, 256, (n, npix), dtype=np.uint8)
    data[:, 5:25] = 255
    t = rng.uniform(0.05, 20.0, n)
    G = np.sort(rng.uniform(0.0, 255.0, 256))
    ctx = api.Context(None, None, 0)
    d, dt, dG = torch.from_numpy(data).cuda(), torch.from_numpy(t).cuda(), torch.from_numpy(G).cuda()
    E_ref = port.estep(data, t, G)
    r_ref = port.rmse(data, t, G, E_ref)
    first = None
    for _ in range(4):
        E = torch.zeros(npix, dtype=torch.float64, device="cuda")
        ctx.estep(d, dt, dG, E)
        assert_bits_equal(E.cpu().numpy(), E_ref, "E-step over a reused ring")
        G2 = torch.zeros(256, dtype=torch.float64, device="cuda")
        ctx.rc_gstep(d, dt, E, G2)
        r = ctx.rc_rmse(d, dt, dG, E)
        assert r[1] == r_ref[1] and abs(r[0] - r_ref[0]) <= 1e-9 * abs(r_ref[0])
        if first is None:
            first = (G2.cpu().numpy(), r)
        else:
            assert_bits_equal(G2.cpu().numpy(), first[0], "G-step over a reused ring, repeated")
            assert r == first[1]
    prod = E_ref[None, :] * t[:, None]
    pmax = np.nanmax(np.abs(E_ref)) * np.abs(t).max()
    for b in range(0, 255, 17):
        m = (data == b) & np.isfinite(prod)
        exact = math.fsum(prod[m].tolist()) / int((data == b).sum())
        assert abs(first[0][b] - exact) <= 4e-15 * pmax + 1e-15 * abs(exact), b


def test_response_calib_loop(api, port):
    """mdc_response_calib = E-init + nits x {G-step, E-step, rescale} against the same loop composed from the oracle."""
    rng = np.random.default_rng(22)
    n, npix = 40, 4096
    # a synthetic exposure sweep of a fixed scene through a gamma response, so that the loop converges sensibly
    scene = rng.uniform(5.0, 120.0, npix)
    t = np.geomspace(0.1, 8.0, n).astype(np.float32).astype(np.float64)
    irr = np.clip(scene[None, :] * t[:, None], 0, 255.0)
    data = np.clip(np.rint(255.0 * (irr / 255.0) ** (1 / 2.2) + rng.normal(0, 1.0, irr.shape)), 0, 255).astype(np.uint8)
    nits = 4
    E_ref = port.einit(data)
    G_ref = np.zeros(256)
    for _ in range(nits):
        G_ref = port.gstep(data, t, E_ref)
        E_ref = port.estep(data, t, G_ref)
        port.rescale(E_ref, G_ref)
    r_ref = port.rmse(data, t, G_ref, E_ref)
    ctx = api.Context(None, None, 0)
    d, dt = torch.from_numpy(data).cuda(), torch.from_numpy(t).cuda()
    E = torch.zeros(npix, dtype=torch.float64, device="cuda")
    G = torch.zeros(256, dtype=torch.float64, device="cuda")
    log = ctx.response_calib(d, dt, nits, E, G)
    g, e = G.cpu().numpy(), E.cpu().numpy()
    m = np.isfinite(G_ref)
    assert np.array_equal(np.isfinite(g), m)
    assert np.max(np.abs(g[m] - G_ref[m]) / np.maximum(np.abs(G_ref[m]), 1e-12)) < 1e-8
    me = np.isfinite(E_ref)
    assert np.max(np.abs(e[me] - E_ref[me]) / np.maximum(np.abs(E_ref[me]), 1e-12)) < 1e-8
    assert log.shape == (nits, 4) and abs(log[-1, 2] - r_ref[0]) <= 1e-7 * abs(r_ref[0]) and log[-1, 3] == r_ref[1]
    assert abs(g[255] - 255.0) < 1e-9


def test_response_calib_against_the_reference_programs_own_output(api):
    """tests/golden/programs/response_calib.npz holds what the reference's responseCalib PROGRAM (main_responseCalib.cpp, unmodified)
    wrote for a small sequence: the GPU calibrator is compared with it directly, not through the restatement."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "programs", "response_calib.npz"))
    w, h, nits, leak = int(g["w"]), int(g["h"]), int(g["nits"]), int(g["leak_padding"])
    ctx = api.Context(None, None, 0)
    d = torch.from_numpy(g["frames"]).cuda()
    ctx.rc_leak_padding(d, w, h, leak)
    E = torch.zeros(w * h, dtype=torch.float64, device="cuda")
    G = torch.zeros(256, dtype=torch.float64, device="cuda")
    log = ctx.response_calib(d, torch.from_numpy(g["exposures"]).cuda(), nits, E, G)
    got, ref = G.cpu().numpy(), g["G"]
    fin = np.isfinite(ref)
    assert np.array_equal(np.isfinite(got), fin)
    assert np.max(np.abs(got[fin] - ref[fin]) / np.maximum(np.abs(ref[fin]), 1e-300)) < 1e-9      # parallel fp64 sums vs sequential ones
    assert np.array_equal(log[:, 3], g["log_num"])                                                # sample counts: exact
    assert np.max(np.abs(log[:, 2] - g["log_rmse"]) / g["log_rmse"]) < 1e-9


@pytest.mark.parametrize("cfg", [
    (1280, 1024, 64, 48, "crop", S.TUM_CALIB),          # 20x minification: boxes far too large to stage -> direct global-gather tiles
    (800, 608, 96, 40, "0.9 1.2 0.5 0.5 0", S.TUM_CALIB),   # mixed: some tiles staged, some direct, some black
    (64, 48, 1, 1, "crop", S.TUM_CALIB),                # single output pixel
    (16, 2, 33, 7, "crop", (0.5, 0.5, 0.5, 0.5, 0.3)),  # degenerate input height (only row 0..1 usable)
], ids=["minify20", "mixed_modes", "one_pixel", "thin_input"])
def test_unusual_geometries(cfg, api, port, dataset_dir):
    iw, ih, ow, oh, mode, calib = cfg
    files = dataset_dir(cfg)
    u, p = make_models(api, files, iw, ih)
    prep = api.FramePreparer(u, p)
    rx, ry, ginv, vinv = oracle_tables(port, files)
    frames = mixed_frames(5, iw, ih)
    d = torch.from_numpy(frames).cuda()
    for use_tma in usable_loaders(prep) + [-1]:
        prep.ctx.configure(use_tma=use_tma)
        for flags in ((1, 1, 1, 1), (1, 0, 0, 0), (1, 1, 0, 1)):
            levels = 4
            outs = [o.cpu().numpy() for o in prep.prepare_device(d, *flags, levels=levels)]
            for i in range(frames.shape[0]):
                exp = port.pyramid(port.get_image(rx, ry, iw, ih, ginv, vinv, frames[i], *flags), ow, oh, levels)
                for l in range(levels):
                    assert_bits_equal(outs[l][i], exp[l], f"{cfg[:4]} tma={use_tma} flags={flags} frame={i} level={l}")


@pytest.mark.parametrize("npix,split", [(96 * 64, 3072), (50 * 30, 701)], ids=["bulk_loader_slices", "ragged_slices"])
def test_pixel_sharded_calibrator_partials_one_gpu(api, port, npix, split):
    """SURVEY.md §8e row 2 on one device: the image stack cut into two pixel slices, each processed as a rank would
    (mdc_rc_gstep_accumulate / mdc_rc_rmse_accumulate on its slice), the partial accumulators summed like the all-reduce does,
    then finished — against the unsharded kernels and the oracle; then the whole sharded host loop (world size 1) against
    mdc_response_calib."""
    from mono_dataset_code_b200 import sharding
    rng = np.random.default_rng(77)
    n = 19
    data = rng.integers(0, 256, (n, npix), dtype=np.uint8)
    data[:, 40:90] = 255
    t = rng.uniform(0.05, 20.0, n).astype(np.float32).astype(np.float64)
    ctx = api.Context(None, None, 0)
    dev = torch.device("cuda", 0)
    dt = torch.from_numpy(t).to(dev)
    slices = [torch.from_numpy(np.ascontiguousarray(data[:, :split])).to(dev), torch.from_numpy(np.ascontiguousarray(data[:, split:])).to(dev)]
    E_ref = port.einit(data)
    Es = []
    for s in slices:
        E = torch.zeros(s.shape[1], dtype=torch.float64, device=dev)
        ctx.rc_einit(s, E)
        Es.append(E)
    assert_bits_equal(torch.cat(Es).cpu().numpy(), E_ref, "sliced E-init")
    gsum = torch.zeros(256, dtype=torch.float64, device=dev)
    gnum = torch.zeros(256, dtype=torch.int64, device=dev)
    acc = torch.zeros(2, dtype=torch.float64, device=dev)
    tot_sum, tot_num = torch.zeros_like(gsum), torch.zeros_like(gnum)
    for s, E in zip(slices, Es):
        ctx.rc_gstep_accumulate(s, dt, E, gsum, gnum, False)
        tot_sum += gsum
        tot_num += gnum
    G = torch.zeros(256, dtype=torch.float64, device=dev)
    ctx.rc_gstep_finish(tot_sum, tot_num, G)
    # the same through the rank-count-independent protocol: one scale for both slices (MAX), integer limbs summed -> the unsharded bits
    scale4, s4 = torch.zeros(4, dtype=torch.int64, device=dev), torch.zeros(4, dtype=torch.int64, device=dev)
    for s, E in zip(slices, Es):
        ctx.rc_gstep_scale(E, dt, s4)
        scale4 = torch.maximum(scale4, s4)
    limbs, special, gn = (torch.zeros(768, dtype=torch.int64, device=dev), torch.zeros(256, dtype=torch.float64, device=dev),
                          torch.zeros(256, dtype=torch.int64, device=dev))
    tot_l, tot_s, tot_n = torch.zeros_like(limbs), torch.zeros_like(special), torch.zeros_like(gn)
    for s, E in zip(slices, Es):
        ctx.rc_gstep_accumulate_exact(s, dt, E, scale4, limbs, special, gn, False)
        tot_l += limbs; tot_s += special; tot_n += gn
    Gx = torch.zeros(256, dtype=torch.float64, device=dev)
    ctx.rc_gstep_finish_exact(scale4, tot_l, tot_s, tot_n, Gx)
    G_whole = torch.zeros(256, dtype=torch.float64, device=dev)
    ctx.rc_gstep(torch.from_numpy(data).to(dev), dt, torch.cat(Es), G_whole)
    assert_bits_equal(Gx.cpu().numpy(), G_whole.cpu().numpy(), "G from two slices (exact protocol) vs the unsharded G-step")
    G_ref = port.gstep(data, t, E_ref)
    g = G.cpu().numpy()
    assert np.array_equal(np.isnan(g), np.isnan(G_ref))
    m = ~np.isnan(G_ref)
    assert np.max(np.abs(g[m] - G_ref[m]) / np.maximum(np.abs(G_ref[m]), 1e-300)) < 1e-10
    counts = np.array([np.count_nonzero(data == b) for b in range(256)])
    counts[255] = 0
    assert np.array_equal(tot_num.cpu().numpy(), counts)
    tot = torch.zeros_like(acc)
    for s, E in zip(slices, Es):
        ctx.rc_rmse_accumulate(s, dt, G, E, acc)
        tot += acc
    r_ref = port.rmse(data, t, g, E_ref)
    a = tot.cpu().numpy()
    assert a[1] == r_ref[1] and abs(1e5 * np.sqrt(a[0] / a[1]) - r_ref[0]) <= 1e-9 * abs(r_ref[0])
    # the sharded host loop with a single rank == the C loop
    full = torch.from_numpy(data).to(dev)
    E1, G1 = torch.zeros(npix, dtype=torch.float64, device=dev), torch.zeros(256, dtype=torch.float64, device=dev)
    E2, G2 = torch.zeros_like(E1), torch.zeros_like(G1)
    log1 = ctx.response_calib(full, dt, 3, E1, G1)
    log2 = sharding.response_calib_sharded(ctx, full, dt, 3, E2, G2)
    np.testing.assert_allclose(G2.cpu().numpy(), G1.cpu().numpy(), rtol=1e-10, equal_nan=True)
    np.testing.assert_allclose(E2.cpu().numpy(), E1.cpu().numpy(), rtol=1e-10, equal_nan=True)
    np.testing.assert_allclose(log2, log1, rtol=1e-9)


def _sharded_calib_worker(rank, world, port_no, data_path, out_dir, nits):
    import sys
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    from mono_dataset_code_b200 import api as A, sharding as sh
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port_no)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    z = np.load(data_path)
    data, t = z["data"], z["t"]
    lo, hi = sh.shard_pixels(data.shape[1], rank, world)
    local = torch.from_numpy(np.ascontiguousarray(data[:, lo:hi])).to(dev)
    dt = torch.from_numpy(t).to(dev)
    ctx = A.Context(None, None, rank)
    out = {}
    # (a) host loop in Python, all-reduces through torch.distributed (NCCL)
    E, G = torch.zeros(hi - lo, dtype=torch.float64, device=dev), torch.zeros(256, dtype=torch.float64, device=dev)
    out["log_py"] = sh.response_calib_sharded(ctx, local, dt, nits, E, G)
    out["E_py"], out["G_py"] = E.cpu().numpy(), G.cpu().numpy()
    # (b) the same loop entirely in C++ on a native communicator (libmdc_b200_nccl.so)
    comm = sh.NativeComm(rank)
    E2, G2 = torch.zeros_like(E), torch.zeros_like(G)
    out["log_cc"] = comm.response_calib_sharded(ctx, local, dt, nits, E2, G2)
    out["E_cc"], out["G_cc"] = E2.cpu().numpy(), G2.cpu().numpy()
    out["nccl_version"] = comm.version
    comm.close()
    np.savez(os.path.join(out_dir, f"gpu_calib{rank}.npz"), lo=lo, hi=hi, **out)
    dist.barrier()
    dist.destroy_process_group()


def test_pixel_sharded_calibrator_two_gpus_nccl(api, port, tmp_path):
    """SURVEY.md §8e row 2 on two GPUs: both ranks end with the same G and E, bit-identical to the single-GPU loop, through the Python
    host loop (torch.distributed NCCL all-reduce) and through the native C++ loop (ncclAllReduce in libmdc_b200_nccl.so)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket
    import torch.multiprocessing as mp
    rng = np.random.default_rng(9)
    n, npix, nits = 40, 256 * 192, 3
    t = np.linspace(0.5, 12.0, n)
    scene = rng.uniform(2.0, 30.0, npix)
    data = np.clip(scene[None, :] * t[:, None] ** 0.9 + rng.normal(0, 1.5, (n, npix)), 0, 255).astype(np.uint8)
    np.savez(tmp_path / "stack.npz", data=data, t=t)
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port_no = s.getsockname()[1]
    mp.spawn(_sharded_calib_worker, args=(2, port_no, str(tmp_path / "stack.npz"), str(tmp_path), nits), nprocs=2, join=True)
    a, b = np.load(tmp_path / "gpu_calib0.npz"), np.load(tmp_path / "gpu_calib1.npz")
    ctx = api.Context(None, None, 0)
    d, dt = torch.from_numpy(data).cuda(), torch.from_numpy(t).cuda()
    E1, G1 = torch.zeros(npix, dtype=torch.float64, device="cuda"), torch.zeros(256, dtype=torch.float64, device="cuda")
    log1 = ctx.response_calib(d, dt, nits, E1, G1)
    for tag in ("py", "cc"):
        assert np.array_equal(a["G_" + tag], b["G_" + tag], equal_nan=True), tag
        # exact integer sums across ranks: not "close", identical
        assert_bits_equal(a["G_" + tag], G1.cpu().numpy(), f"G on 2 GPUs ({tag}) vs 1 GPU")
        assert_bits_equal(np.concatenate([a["E_" + tag], b["E_" + tag]]), E1.cpu().numpy(), f"E on 2 GPUs ({tag}) vs 1 GPU")
        np.testing.assert_allclose(a["log_" + tag], log1, rtol=1e-9)
        assert np.array_equal(a["log_" + tag], b["log_" + tag])


@pytest.mark.parametrize("name", ["odd_sizes", "c1_crop_640"])
def test_padded_rows_keep_odd_widths_on_the_fast_loaders(name, api, port, dataset_dir):
    """VERDICT r1 #10: a width that is not a multiple of 16 bytes cannot be described to TMA when the rows are tightly packed, but it
    can with a padded row pitch — mdc_prepare_batch_pitched on the device, and mdc_prepare_batch_host pads during its H2D copy.
    Every loader that accepts the padded layout must reproduce the oracle bit for bit, pyramid included."""
    iw, ih, ow, oh, mode, calib = CALIBS[name]
    files = dataset_dir(name)
    u, p = make_models(api, files, iw, ih)
    prep = api.FramePreparer(u, p)
    rx, ry, ginv, vinv = oracle_tables(port, files)
    frames = mixed_frames(9, iw, ih)
    exp = [port.pyramid(port.get_image(rx, ry, iw, ih, ginv, vinv, f, 1, 1, 1, 1), ow, oh, 4) for f in frames]
    pitch = (iw + 63) & ~31                       # 32-byte multiple, strictly larger than the width
    padded = torch.full((frames.shape[0], ih, pitch), 77, dtype=torch.uint8, device="cuda")
    padded[:, :, :iw] = torch.from_numpy(frames.reshape(-1, ih, iw)).cuda()
    shapes = prep.level_shapes(True, 4)
    ran = []
    for loader in (-1, 0, 1, 2, 3):
        prep.ctx.configure(use_tma=loader)
        outs = [torch.zeros((frames.shape[0], w * h), dtype=torch.float32, device="cuda") for (w, h) in shapes]
        try:
            prep.ctx.prepare_batch_pitched(padded, pitch, 1 | 2 | 4 | 8, outs)
        except api.MdcError as exc:                # a loader that cannot take this layout says so instead of computing something else
            assert exc.code == 6 and loader > 0, (loader, str(exc))
            continue
        ran.append(loader)
        for i in range(frames.shape[0]):
            for l in range(4):
                assert_bits_equal(outs[l][i].cpu().numpy(), exp[i][l], f"{name} pitched loader={loader} frame={i} level={l}")
    assert -1 in ran and 0 in ran and 1 in ran, ran       # auto, LDG and — thanks to the padding — TMA
    # host path: tightly packed odd-width frames in, padded on the way to the device
    prep.ctx.configure(use_tma=-1)
    host_out = [np.zeros((frames.shape[0], w * h), np.float32) for (w, h) in shapes]
    prep.ctx.prepare_batch_host(frames, 1 | 2 | 4 | 8, host_out)
    for i in range(frames.shape[0]):
        for l in range(4):
            assert_bits_equal(host_out[l][i], exp[i][l], f"{name} host path frame={i} level={l}")
