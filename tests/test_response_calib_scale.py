"""responseCalib's passes (main_responseCalib.cpp:206-355) pinned at the reference's problem sizes and at the edges of their
arithmetic: leak padding, E-init, E-step, G-step, rmse and rescale, one pass at a time and as the whole loop.  They are compared with
the plain-C oracle, with tests/gstep_fixed_point_spec.py (the G-step's fixed-point sums in numpy) and, where numpy would be too slow,
with the same integer sums formed in torch on the device.

- The reference's scale: 1700 frames of 1280x1024 (2.2e9 samples, more than 2^31), and 3300 frames (4.3 GB, more than 2^32 bytes).
- Exposure counts either side of every boundary of the streaming kernels (plane groups of 8, the fold interval of 160 exposures,
  constant-memory exposure times up to 1024), in the bulk-copy, register-pipelined and byte-tail layouts and at several tile widths.
- Limb slots of the G-step histogram loaded to the bound its static_assert promises.
- Exposure times, irradiances, residuals and response values at the edges of fp64."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import gstep_fixed_point_spec as fx
from conftest import assert_bits_equal
from test_gstep_fixed_point_spec import EXTREME, assert_matches_reference, extreme

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from mono_dataset_code_b200 import api
    return api.Context(None, None, 0)


def need_free_memory(gb):
    free, total = torch.cuda.mem_get_info()
    if free < gb * 1e9:
        pytest.skip(f"needs {gb:.1f} GB of free device memory, {free / 1e9:.1f} of {total / 1e9:.1f} GB are free")


# ------------------------------------------------------------------------------------------------ inputs
def exposures(n, seed):
    """n exposure times over 0.05 .. 20 in a shuffled order, rounded through a float like times.txt (:209)"""
    t = np.geomspace(0.05, 20.0, n) if n else np.zeros(0)
    return np.random.default_rng(seed).permutation(t).astype(np.float32).astype(np.float64)


def response_table():
    G = 255.0 * (np.arange(256) / 255.0) ** 2.2
    G[255] = 300.0
    return G


def sweep_host(n, npix, seed):
    """A fixed scene seen at n exposures through a gamma-like response, with noise, a blob that is saturated in every frame and a
    saturated strip in every 7th frame (numpy, for the small problems)."""
    rng = np.random.default_rng(seed)
    t = exposures(n, seed)
    scene = rng.uniform(0.5, 40.5, npix)
    v = 255.0 * np.clip(scene[None, :] * t[:, None] / 255.0, 0.0, 1.0) ** (1 / 2.2) + rng.normal(0.0, 1.5, (n, npix))
    data = np.clip(np.rint(v), 0, 255).astype(np.uint8)
    data[:, 100:140] = 255
    data[::7, :9] = 255
    return data, t


def sweep_device(n, w, h, t, seed, rows=64):
    """The same kind of stack generated on the device, frame block by frame block: uint8 [n, w*h].  The blob is saturated in every
    frame (its pixels have no usable sample), the first row and column in every 7th frame (border pixels never spread)."""
    npix = w * h
    g = torch.Generator(device="cuda").manual_seed(seed)
    scene = torch.rand(npix, generator=g, device="cuda", dtype=torch.float64) * 40.0 + 0.5
    dt = torch.from_numpy(t).cuda()
    out = torch.empty((n, npix), dtype=torch.uint8, device="cuda")
    for r0 in range(0, n, rows):
        r1 = min(n, r0 + rows)
        v = 255.0 * torch.clamp(scene[None, :] * dt[r0:r1, None] / 255.0, 0.0, 1.0) ** (1 / 2.2)
        v += torch.randn((r1 - r0, npix), generator=g, device="cuda", dtype=torch.float64) * 1.5
        out[r0:r1] = torch.clamp(torch.round(v), 0, 255).to(torch.uint8)
    img = out.view(n, h, w)
    img[:, h // 3:h // 3 + h // 10, w // 2:w // 2 + w // 10] = 255
    img[::7, 0, :] = 255
    img[::7, :, 0] = 255
    return out


def upload(data, layout):
    """uint8 [n, npix] on the device: 'bulk' (a fresh allocation: 16-byte aligned), 'aligned4' (4 bytes past such a base: the
    register-pipelined E-step and the fallback G-step and rmse kernels); odd npix gives the byte-tail paths either way.  (torch
    passes null pointers for a stack of no frames; the C ABI accepts them when n = 0.)"""
    n, npix = data.shape
    off = 4 if layout == "aligned4" else 0
    buf = torch.empty(n * npix + off + 16, dtype=torch.uint8, device="cuda")
    d = buf[off:off + n * npix].view(n, npix)
    if n:
        d.copy_(torch.from_numpy(data))
    return d


def f64(a):
    a = np.asarray(a, np.float64)
    buf = torch.empty(a.size + 1, dtype=torch.float64, device="cuda")
    d = buf[:a.size]
    if a.size:
        d.copy_(torch.from_numpy(a))
    return d


# ------------------------------------------------------------------------------------------------ references
def per_pixel(fn, data, *args, parts=None):
    """A per-pixel oracle pass (E-init, E-step) over column slices in a thread pool: ctypes releases the GIL, and a pixel's bits do
    not depend on which other pixels share its call."""
    npix = data.shape[1]
    parts = parts or max(1, min(os.cpu_count() or 1, 32))
    cuts = np.linspace(0, npix, parts + 1).astype(np.int64)
    out = np.empty(npix)

    def run(i):
        a, b = cuts[i], cuts[i + 1]
        out[a:b] = fn(np.ascontiguousarray(data[:, a:b]), *args)

    with ThreadPoolExecutor(parts) as ex:
        list(ex.map(run, range(parts)))
    return out


def leak_padding_torch(data, w, h, iters, rows=64):
    """main_responseCalib.cpp:212-236 as a torch formulation: per iteration, the 255-mask of interior pixels (x in [1, w-2],
    y in [1, h-2]), dilated by a 3x3 max-pool, sets the pixel to 255."""
    n = data.shape[0]
    out = data.clone().view(n, h, w)
    interior = torch.zeros((h, w), dtype=torch.bool, device=data.device)
    interior[1:h - 1, 1:w - 1] = True
    for r0 in range(0, n, rows):
        x = out[r0:r0 + rows]
        for _ in range(iters):
            src = ((x == 255) & interior).to(torch.float32).unsqueeze(1)
            spread = torch.nn.functional.max_pool2d(src, 3, stride=1, padding=1).squeeze(1) > 0
            x = torch.where(spread, torch.full_like(x, 255), x)
        out[r0:r0 + rows] = x
    return out.view(n, h * w)


def device_fixed_point(d, dt, dE, t, E, rows=32):
    """The G-step's sums of gstep_fixed_point_spec formed on the device: fp64 products E*t, scaled by 2^s, torch.round (half to
    even), split into two 24-bit halves that are summed per bin with scatter_add_ in int64 (exact up to 2^39 samples), joined in
    Python integers.  -> (G, GNum, the largest |sum| of a bin in units of 2^-s)"""
    words = fx.scale_words(E, t)
    s = fx.exponent(words)
    assert -1022 <= s <= 1023, s                          # 2^s is a double: p * 2^s is the spec's ldexp(p, s)
    scale = 2.0 ** s
    lo = torch.zeros(256, dtype=torch.int64, device="cuda")
    hi, cnt = torch.zeros_like(lo), torch.zeros_like(lo)
    special = torch.zeros(256, dtype=torch.float64, device="cuda")
    for r0 in range(0, d.shape[0], rows):
        b = d[r0:r0 + rows].reshape(-1).long()
        p = (dE[None, :] * dt[r0:r0 + rows, None]).reshape(-1)
        x = p * scale
        keep = b != 255
        ok = keep & (x.abs() < fx.LIMIT)
        odd = keep & ~ok
        cnt += torch.bincount(b[keep], minlength=256)
        if bool(odd.any()):
            special.index_add_(0, b[odd], p[odd])
        v, bo = torch.round(x[ok]).long(), b[ok]
        lo.scatter_add_(0, bo, v & ((1 << 24) - 1))
        hi.scatter_add_(0, bo, v >> 24)
    lo, hi = lo.cpu().tolist(), hi.cpu().tolist()
    totals = [lo[k] + (hi[k] << 24) for k in range(256)]
    counts = cnt.cpu().numpy()
    return fx.finish(words, fx.limbs_of(totals), special.cpu().numpy(), counts), counts, max(abs(v) for v in totals)


def gstep(ctx, d, dt, dE):
    G = torch.empty(256, dtype=torch.float64, device="cuda")
    ctx.rc_gstep(d, dt, dE, G)
    return G


def estep(ctx, d, dt, dG):
    E = torch.empty(d.shape[1] + 1, dtype=torch.float64, device="cuda")[:d.shape[1]]
    ctx.estep(d, dt, dG, E)
    return E


def assert_rmse(r, r_ref, what, tol=1e-10):
    assert r[1] == r_ref[1], f"{what}: rmse counts {r[1]} vs {r_ref[1]}"
    if np.isfinite(r_ref[0]):
        assert np.isfinite(r[0]) and abs(r[0] - r_ref[0]) <= tol * abs(r_ref[0]), f"{what}: rmse {r[0]!r} vs {r_ref[0]!r}"
    else:
        assert np.array_equal(np.isnan(r[0]), np.isnan(r_ref[0])) and (np.isnan(r[0]) or r[0] == r_ref[0]), f"{what}: rmse {r[0]!r} vs {r_ref[0]!r}"


# ------------------------------------------------------------------------------------------------ (a) the reference's scale
def composed_loop(ctx, d, dt, nits):
    """mdc_response_calib's loop built from the single passes (fresh G-step counts every iteration)"""
    npix = d.shape[1]
    E = torch.empty(npix, dtype=torch.float64, device="cuda")
    ctx.rc_einit(d, E)
    G = torch.zeros(256, dtype=torch.float64, device="cuda")
    log = []
    for _ in range(nits):
        ctx.rc_gstep(d, dt, E, G)
        r0 = ctx.rc_rmse(d, dt, G, E)
        ctx.estep(d, dt, G, E)
        r1 = ctx.rc_rmse(d, dt, G, E)
        ctx.rc_rescale(E, G)
        r2 = ctx.rc_rmse(d, dt, G, E)
        log.append([r0[0], r1[0], r2[0], r2[1]])
    return E, G, np.array(log)


def test_reference_scale_1700_frames_of_1280x1024(ctx, port):
    n, w, h = 1700, 1280, 1024
    npix = w * h
    need_free_memory(4 * n * npix / 1e9 + 6.0)
    t = exposures(n, 1)
    dt = torch.from_numpy(t).cuda()
    raw = sweep_device(n, w, h, t, seed=2)
    assert n * npix > 2 ** 31
    # leak padding: 2 iterations end in the caller's buffer, 3 in scratch and are copied back
    frames = (0, n // 2, n - 1)
    for iters in (3, 2):
        d = raw.clone()
        ctx.rc_leak_padding(d, w, h, iters)
        assert torch.equal(d, leak_padding_torch(raw, w, h, iters)), f"leak padding x{iters} vs the torch formulation"
        for i in frames:
            exp = port.leak_padding(raw[i].cpu().numpy(), w, h, iters)
            assert np.array_equal(d[i].cpu().numpy(), exp), f"leak padding x{iters}, frame {i}"
    del raw
    host = d.cpu().numpy()
    assert (host == 255).mean() > 0.05 and (host < 8).mean() > 0.002
    # E-init
    E0 = torch.empty(npix, dtype=torch.float64, device="cuda")
    ctx.rc_einit(d, E0)
    E0_ref = per_pixel(port.einit, host)
    assert_bits_equal(E0.cpu().numpy(), E0_ref, "E-init")
    # G-step: bit for bit against the device's integer formulation, to rounding against the reference's sequential chain
    G = gstep(ctx, d, dt, E0)
    g = G.cpu().numpy()
    G_int, counts, biggest = device_fixed_point(d, dt, E0, t, E0_ref)
    assert_bits_equal(g, G_int, "G-step vs the integer sums on the device")
    assert_bits_equal(gstep(ctx, d, dt, E0).cpu().numpy(), g, "G-step, repeated")
    G_ref = port.gstep(host, t, E0_ref)
    assert_matches_reference(g, G_ref, "G-step vs the oracle")
    gsum = torch.zeros(256, dtype=torch.float64, device="cuda")
    gnum = torch.zeros(256, dtype=torch.int64, device="cuda")
    ctx.rc_gstep_accumulate(d, dt, E0, gsum, gnum, False)
    assert np.array_equal(gnum.cpu().numpy(), counts), "GNum vs a bincount"
    assert biggest > 2 ** 64                                  # some bin's sum needs the high word of the 128-bit accumulator
    # rmse
    r = ctx.rc_rmse(d, dt, G, E0)
    assert_rmse(r, port.rmse(host, t, g, E0_ref), "rmse")
    # E-step
    E1 = estep(ctx, d, dt, G)
    E1_ref = per_pixel(port.estep, host, t, g)
    assert_bits_equal(E1.cpu().numpy(), E1_ref, "E-step")
    # rescale
    Ec, Gc = E1.clone(), G.clone()
    f = ctx.rc_rescale(Ec, Gc)
    E2, G2 = E1_ref.copy(), g.copy()
    assert f == port.rescale(E2, G2)
    assert_bits_equal(Ec.cpu().numpy(), E2, "rescaled E")
    assert_bits_equal(Gc.cpu().numpy(), G2, "rescaled G")
    del Ec, Gc, E1, host
    # the whole loop (G-step counts reused from the second iteration on) against the loop composed from the single passes
    El, Gl = torch.empty(npix, dtype=torch.float64, device="cuda"), torch.empty(256, dtype=torch.float64, device="cuda")
    log = ctx.response_calib(d, dt, 3, El, Gl)
    Ec, Gc, log_c = composed_loop(ctx, d, dt, 3)
    assert_bits_equal(Gl.cpu().numpy(), Gc.cpu().numpy(), "loop G")
    assert_bits_equal(El.cpu().numpy(), Ec.cpu().numpy(), "loop E")
    assert_bits_equal(log, log_c, "loop log")
    del El, Ec
    # pixel-sharded protocol on one device: three uneven slices (two not a multiple of 16 pixels), one scale, integer limbs summed
    cuts = [0, 524288, 524288 + 393223, npix]
    scale4, s4 = torch.zeros(4, dtype=torch.int64, device="cuda"), torch.zeros(4, dtype=torch.int64, device="cuda")
    for a, b in zip(cuts[:-1], cuts[1:]):
        ctx.rc_gstep_scale(E0[a:b], dt, s4)
        scale4 = torch.maximum(scale4, s4)
    limbs, special = torch.zeros(768, dtype=torch.int64, device="cuda"), torch.zeros(256, dtype=torch.float64, device="cuda")
    gn = torch.zeros(256, dtype=torch.int64, device="cuda")
    tot_l, tot_s, tot_n = torch.zeros_like(limbs), torch.zeros_like(special), torch.zeros_like(gn)
    for a, b in zip(cuts[:-1], cuts[1:]):
        part = d[:, a:b].contiguous()
        ctx.rc_gstep_accumulate_exact(part, dt, E0[a:b].contiguous(), scale4, limbs, special, gn, False)
        tot_l += limbs
        tot_s += special
        tot_n += gn
        del part
    Gx = torch.empty(256, dtype=torch.float64, device="cuda")
    ctx.rc_gstep_finish_exact(scale4, tot_l, tot_s, tot_n, Gx)
    assert_bits_equal(Gx.cpu().numpy(), g, "G from three slices (exact protocol) vs the unsharded G-step")


# ------------------------------------------------------------------------------------------------ (b) beyond 2^32 bytes
def test_beyond_4gb_3300_frames_of_1280x1024(ctx, port):
    n, w, h = 3300, 1280, 1024
    npix = w * h
    need_free_memory(n * npix / 1e9 + 5.0)
    t = exposures(n, 3)
    dt = torch.from_numpy(t).cuda()
    d = sweep_device(n, w, h, t, seed=4)
    assert n * npix > 2 ** 32
    E0 = torch.empty(npix, dtype=torch.float64, device="cuda")
    ctx.rc_einit(d, E0)
    G = gstep(ctx, d, dt, E0)
    g = G.cpu().numpy()
    G_int, _, _ = device_fixed_point(d, dt, E0, t, E0.cpu().numpy())
    assert_bits_equal(g, G_int, "G-step vs the integer sums on the device")
    E1 = estep(ctx, d, dt, G)
    e0, e1 = E0.cpu().numpy(), E1.cpu().numpy()
    for a in (0, 128 * 4099 + 3, npix // 2 + 64, npix - 128):
        col = np.ascontiguousarray(d[:, a:a + 128].cpu().numpy())
        assert_bits_equal(e0[a:a + 128], port.einit(col), f"E-init, pixels {a}..{a + 127}")
        assert_bits_equal(e1[a:a + 128], port.estep(col, t, g), f"E-step, pixels {a}..{a + 127}")
    r = ctx.rc_rmse(d, dt, G, E1)
    count, err = 0, torch.zeros((), dtype=torch.float64, device="cuda")
    for r0 in range(0, n, 32):
        blk = d[r0:r0 + 32]
        res = G[blk.long()] - dt[r0:r0 + 32, None] * E1[None, :]
        ok = (blk != 255) & torch.isfinite(res)
        count += int(ok.sum())
        err += torch.where(ok, res * res * 1e-10, torch.zeros_like(res)).sum()
    assert r[1] == count
    assert abs(r[0] - 1e5 * np.sqrt(float(err) / count)) <= 1e-9 * r[0]


# ------------------------------------------------------------------------------------------------ (c) boundaries
N_EDGES = [0, 1, 7, 8, 9, 159, 160, 161, 1023, 1024, 1025, 4096, 4097]
LAYOUTS = {"bulk": ("bulk", 3600), "aligned4": ("aligned4", 3600), "odd_npix": ("bulk", 3601)}


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("n", N_EDGES)
def test_exposure_count_boundaries(ctx, port, monkeypatch, n, layout):
    kind, npix = LAYOUTS[layout]
    data, t = sweep_host(n, npix, seed=100 + n)
    d, dt = upload(data, kind), f64(t)
    G0 = response_table()
    E_ref = port.estep(data, t, G0)
    runs = [estep(ctx, d, dt, f64(G0)).cpu().numpy() for _ in range(2)]
    assert_bits_equal(runs[0], E_ref, f"E-step n={n} {layout}")
    assert_bits_equal(runs[1], runs[0], f"E-step n={n} {layout}, repeated")
    dE = f64(E_ref)
    G_spec = fx.gstep(data, t, E_ref)
    Gs = []
    for warps in (None, "1", "5", "14", None):
        if warps is None:
            monkeypatch.delenv("MDC_STREAM_WARPS", raising=False)
        else:
            monkeypatch.setenv("MDC_STREAM_WARPS", warps)
        Gs.append(gstep(ctx, d, dt, dE).cpu().numpy())
    monkeypatch.delenv("MDC_STREAM_WARPS", raising=False)
    assert_bits_equal(Gs[0], G_spec, f"G-step n={n} {layout} vs the specification")
    for G in Gs[1:]:
        assert_bits_equal(G, Gs[0], f"G-step n={n} {layout}, repeated / other tile widths")
    g = Gs[0]
    r_ref = port.rmse(data, t, g, E_ref)
    r1, r2 = ctx.rc_rmse(d, dt, f64(g), dE), ctx.rc_rmse(d, dt, f64(g), dE)
    assert_rmse(r1, r_ref, f"rmse n={n} {layout}")
    assert np.array_equal(np.array(r1), np.array(r2), equal_nan=True), f"rmse n={n} {layout}, repeated"


# ------------------------------------------------------------------------------------------------ (d) the limb bound
@pytest.mark.parametrize("sign", [1.0, -1.0], ids=["positive", "negative"])
def test_limb_slots_at_their_bound(ctx, sign):
    """Every sample in one bin, every scaled product 2^48 - 1 units (or its negative): each add puts the largest value the signed
    limb can take into its slot, and every CTA works through three full tiles of 2000 exposures, folding its histograms in
    between.  A fold interval longer than the static_assert allows overflows a slot and changes G."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n, npix = 2000, sms * 28 * 128 * 3
    need_free_memory(n * npix / 1e9 + 1.0)
    e = sign * (2.0 - 2.0 ** -47)                          # e * 1.0 * 2^47 = +-(2^48 - 1)
    d = torch.full((n, npix), 77, dtype=torch.uint8, device="cuda")
    t = np.ones(n)
    G = gstep(ctx, d, f64(t), torch.full((npix,), e, dtype=torch.float64, device="cuda")).cpu().numpy()
    words = fx.scale_words(np.array([e]), t)
    assert fx.exponent(words) == 47
    totals = [0] * 256
    totals[77] = n * npix * int(np.rint(np.ldexp(e, 47)))
    counts = np.zeros(256, np.int64)
    counts[77] = n * npix
    assert_bits_equal(G, fx.finish(words, fx.limbs_of(totals), np.zeros(256), counts), f"G-step, limbs at their bound ({sign:+})")
    assert abs(G[77] - e) <= 1e-15


# ------------------------------------------------------------------------------------------------ (e) extreme values
@pytest.mark.parametrize("layout", ["bulk", "fallback"])
@pytest.mark.parametrize("case", EXTREME)
def test_gstep_extreme_values(ctx, port, case, layout):
    data, t, E = extreme(case, npix=896 if layout == "bulk" else 900)
    d, dt, dE = upload(data, "bulk"), f64(t), f64(E)
    G = gstep(ctx, d, dt, dE).cpu().numpy()
    with np.errstate(invalid="ignore", over="ignore"):
        G_spec, G_ref = fx.gstep(data, t, E), port.gstep(data, t, E)
    assert_matches_reference(G, G_ref, f"G-step {case} ({layout})")
    assert_bits_equal(G, G_spec, f"G-step {case} ({layout}) vs the specification")
    assert_bits_equal(gstep(ctx, d, dt, dE).cpu().numpy(), G, f"G-step {case} ({layout}), repeated")


@pytest.mark.parametrize("layout", ["bulk", "fallback"])
@pytest.mark.parametrize("case", ["residuals_near_1e153", "residual_overflows", "nan_residuals"])
def test_rmse_extreme_residuals(ctx, port, case, layout):
    rng = np.random.default_rng(41)
    n, npix = 64, 896 if layout == "bulk" else 900
    data = rng.integers(0, 255, (n, npix), dtype=np.uint8)
    t = rng.uniform(1.0, 1.2, n)
    E = rng.uniform(1.0, 100.0, npix)
    G = np.linspace(0.0, 255.0, 256)
    if case in ("residuals_near_1e153", "residual_overflows"):
        E[:600] = rng.uniform(1.0, 1.3, 600) * 1e153      # each square finite, a thread's sum of them is not
    if case == "residual_overflows":
        E[7] = 2e154                                       # r * r = inf: so is the reference's long double sum
    if case == "nan_residuals":
        E[::9] = np.nan
        G[17] = np.inf
    r = ctx.rc_rmse(upload(data, "bulk"), f64(t), f64(G), f64(E))
    r_ref = port.rmse(data, t, G, E)
    assert_rmse(r, r_ref, f"rmse {case} ({layout})")
    if case == "residual_overflows":
        assert r[0] == np.inf
    else:
        assert np.isfinite(r[0])
    if case == "nan_residuals":
        assert r[1] < np.count_nonzero(data != 255)


@pytest.mark.parametrize("layout", ["bulk", "aligned4", "odd_npix"])
@pytest.mark.parametrize("n", [40, 1030])
@pytest.mark.parametrize("case", ["t_squared_underflows", "t_squared_overflows", "special_G"])
def test_estep_extreme_values(ctx, port, case, n, layout):
    kind, npix = LAYOUTS[layout]
    rng = np.random.default_rng(n)
    data = rng.integers(0, 256, (n, npix), dtype=np.uint8)
    t = rng.uniform(0.5, 2.0, n)
    G = np.linspace(-3.0, 255.0, 256)
    if case == "t_squared_underflows":
        t[::2] *= 1e-170                                   # t * t = 0
        data[1::2, :50] = 255                              # pixels that only see those frames: esum / 0
    elif case == "t_squared_overflows":
        t[::3] *= 1e160                                    # t * t = inf
        data[1::3, :50] = 255
        data[2::3, :50] = 255
    else:
        G[3], G[4], G[5], G[6], G[7], G[8] = np.inf, -np.inf, -0.0, 5e-324, 2.2e-310, np.nan
        data[:, :30] = rng.choice(np.array([3, 4, 5, 6, 7, 8, 255], np.uint8), (n, 30))
    E = estep(ctx, upload(data, kind), f64(t), f64(G)).cpu().numpy()
    assert_bits_equal(E, port.estep(data, t, G), f"E-step {case} n={n} {layout}")


@pytest.mark.parametrize("w,h", [(1, 1), (1, 6), (6, 1), (2, 2), (2, 7), (7, 2), (3, 3), (3, 8), (8, 3)])
def test_leak_padding_thin_images(ctx, port, w, h):
    rng = np.random.default_rng(w * 10 + h)
    n = 5
    data = np.where(rng.random((n, w * h)) < 0.3, 255, rng.integers(0, 255, (n, w * h))).astype(np.uint8)
    data[2] = 255                                          # a fully saturated frame
    for iters in range(1, 6):
        d = upload(data, "bulk")
        ctx.rc_leak_padding(d, w, h, iters)
        exp = np.stack([port.leak_padding(data[i], w, h, iters) for i in range(n)])
        got = d.cpu().numpy()
        assert np.array_equal(got, exp), f"leak padding {w}x{h} x{iters}"
        assert torch.equal(d, leak_padding_torch(upload(data, "bulk"), w, h, iters))
