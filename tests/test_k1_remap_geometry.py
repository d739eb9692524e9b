"""K1 (the fused prepare kernel) and K1b (undistort<float>) on remap tables the FOV model never produces (tests/remap_families.py),
adopted through mdc_ctx_create_from_device_tables, and the refusal of tables outside the domain D.

Each family runs with a real photometric model (a vignette with zeros, so its inverse holds inf) and with arbitrary GInv / inverse
vignette arrays holding NaN, +-inf, -0.0, subnormals and huge values, through every usable loader with packed rows and, at 333 x 217,
with pitched rows (a 16-multiple and an odd pitch).  Every output is compared bit for bit with the plain-C oracle (getImage, then the
pyramid), whose pyramid is itself checked against pyramid_spec; undistort<uchar> / <float> are compared with the oracle and with
undistort_spec.  The tile plan each family exists for is asserted from the MDC_VERBOSE plan line, not assumed."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import pyramid_spec
import remap_families as RF
import undistort_spec as spec
from conftest import assert_bits_equal

try:
    import torch
except ImportError:
    torch = None

gpu = pytest.mark.gpu
F32 = np.float32
SENTINEL = -12345.0
MAX_LEVELS = 8
PLAN_RE = re.compile(r"\[mdc\] plan: (\d+) tiles \((\d+) staged, (\d+) direct, (\d+) empty, (\d+) with black pixels\), (\d+) TMA box classes "
                     r"at row granularity (\d+)")
ALL_FLAGS = [(f & 1, (f >> 1) & 1, (f >> 2) & 1, (f >> 3) & 1) for f in range(16)]
LARGE_FLAGS = [(1, 1, 1, 1), (1, 0, 0, 0)]
# families whose boxes are too narrow for the pitch search to matter run with it off, so the class count is known exactly
NO_PITCH_SEARCH = ("many_classes_g16_1920x1080", "many_classes_g32_1920x1080")


@pytest.fixture(scope="module")
def api():
    if torch is None or not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from mono_dataset_code_b200 import api as a
    return a


def real_photometric(port, n, seed):
    """GInv of a gamma-like response, and the inverse of a vignette image with zero pixels (inf in its inverse)."""
    raw = (255.0 * (np.arange(256) / 255.0) ** 1.7 + 0.01 * np.arange(256)).astype(F32)
    ginv, _ = port.photo_tables(raw)
    r = np.random.default_rng(seed)
    px = r.integers(40, 256, n).astype(np.uint8)
    px[r.random(n) < 0.05] = 0
    px[0] = 0
    _, vinv = port.vignette_maps(px)
    assert np.isinf(vinv).any()
    return ginv, vinv


def plan_of(err):
    lines = PLAN_RE.findall(err)
    assert lines, f"no plan line in the MDC_VERBOSE output: {err[-2000:]}"
    t, staged, direct, empty, black, classes, gran = map(int, lines[-1])    # the plan of the last (kept) granularity
    return dict(tiles=t, staged=staged, direct=direct, empty=empty, black=black, classes=classes, gran=gran)


def adopt(api, f, ginv, vinv, monkeypatch, capfd, env=None):
    """Context.from_device_tables (which keeps the device tables alive) with MDC_VERBOSE set -> (ctx, plan dict)."""
    for k in [k for k in os.environ if k.startswith("MDC_")]:
        monkeypatch.delenv(k)
    monkeypatch.setenv("MDC_VERBOSE", "1")
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    tens = [torch.from_numpy(np.ascontiguousarray(a, F32)).cuda() for a in (f.rx, f.ry, ginv, vinv)]
    torch.cuda.synchronize()
    capfd.readouterr()
    ctx = api.Context.from_device_tables(0, f.in_w, f.in_h, f.out_w, f.out_h, *tens)
    return ctx, plan_of(capfd.readouterr().err)


def check_plan(name, f, ctx, plan):
    """The library's plan against the plan model, and the branch each family exists for."""
    model = RF.plan_model(f, plan["gran"])
    assert plan["tiles"] == -(-f.out_w // RF.TILE) * -(-f.out_h // RF.TILE)
    for k in ("staged", "direct", "empty", "black"):
        assert plan[k] == model[k], f"{name}: {plan[k]} {k} tiles in the plan, the model says {model[k]} (plan {plan})"
    if name in NO_PITCH_SEARCH:
        assert plan["gran"] == RF.granularity_without_pitch_search(f) and plan["classes"] == len(model["classes"]), (name, plan)
    if f.in_w % 16 == 0:       # TMA describes packed rows of this width: usable exactly when the plan has staged tiles
        assert ctx.loader_usable("tma") == (plan["staged"] > 0), (name, plan)
    if name.startswith(("scatter", "to_40x30")):
        assert plan["staged"] == 0 and not ctx.loader_usable("tma"), (name, plan)
    if name.startswith("many_classes_g16"):
        assert plan["gran"] >= 16 and ctx.loader_usable("tma"), plan
    if name.startswith("many_classes_g32"):
        assert plan["gran"] == 32 and ctx.loader_usable("tma"), plan
    if name.startswith("checkerboard"):
        assert plan["staged"] and plan["direct"] and plan["empty"] and plan["black"] > plan["empty"], plan
    if name == "minify_ramp_1920x1080":
        assert plan["staged"] and plan["direct"], plan


class Oracle:
    """getImage then the pyramid through the plain-C oracle, per (frame, flags), with the pyramid checked against pyramid_spec."""

    def __init__(self, port, f, ginv, vinv, frames):
        self.port, self.f, self.ginv, self.vinv, self.frames = port, f, ginv, vinv, frames
        self.cache = {}

    def dims(self, rectify):
        return (self.f.out_w, self.f.out_h) if rectify else (self.f.in_w, self.f.in_h)

    def levels(self, i, flags):
        key = (i, flags)
        if key not in self.cache:
            f = self.f
            l0 = self.port.get_image(f.rx, f.ry, f.in_w, f.in_h, self.ginv, self.vinv, self.frames[i], *flags)
            w, h = self.dims(flags[0])
            pyr = self.port.pyramid(l0, w, h, MAX_LEVELS)
            for a, b in zip(pyr, pyramid_spec.pyramid(l0, w, h, MAX_LEVELS)):
                assert_bits_equal(a, b, f"{f.name}: oracle pyramid vs pyramid_spec flags={flags}")
            self.cache[key] = pyr
        return self.cache[key]


def k1(api, ctx, d, n, pitch, flags, levels, w, h):
    """One synchronous mdc_prepare_batch(_pitched) call; levels without pixels get a NULL pointer.  -> (status, output tensors)."""
    from mono_dataset_code_b200._lib import lib
    outs = [torch.full((n, (w >> l) * (h >> l)), SENTINEL, dtype=torch.float32, device="cuda") if (w >> l) * (h >> l) else None
            for l in range(levels)]
    arr = (C.c_void_p * levels)(*[o.data_ptr() if o is not None else None for o in outs])
    bits = flags[0] | flags[1] << 1 | flags[2] << 2 | flags[3] << 3
    torch.cuda.synchronize()
    if pitch:
        rc = lib.mdc_prepare_batch_pitched(ctx._h, C.c_void_p(d.data_ptr()), pitch, n, bits, arr, levels, None)
    else:
        rc = lib.mdc_prepare_batch(ctx._h, C.c_void_p(d.data_ptr()), n, bits, arr, levels, None)
    return rc, outs


def check_outputs(oracle, outs, idx, flags, what):
    for l, o in enumerate(outs):
        if o is None:
            continue
        a = o.cpu().numpy()
        for i, k in enumerate(idx):
            assert_bits_equal(a[i], oracle.levels(k, flags)[l], f"{what} frame={i} level={l}")


def frames_for(f, n, seed):
    fr = np.stack([RF.frame_u8(f.in_w * f.in_h, seed + i) for i in range(n)])
    fr[0, :] = np.where(np.arange(f.in_w * f.in_h) % 7 == 0, 255, fr[0, :])     # saturated pixels for the kill flag
    return fr


def layouts(f):
    """(row pitch, loaders that must run, loaders that may refuse with MDC_ERR_UNSUPPORTED) for this family."""
    out = [(0, ["auto", "ldg"], ["tma", "tex", "hybrid"])]
    if f.in_w == 333:
        out += [(336, ["auto", "ldg"], ["tma", "tex", "hybrid"]), (335, ["auto", "ldg"], ["tma", "tex", "hybrid"])]
    return out


@gpu
@pytest.mark.parametrize("photo", ["real", "arbitrary"])
@pytest.mark.parametrize("name", sorted(RF.REGISTRY))
def test_family(name, photo, api, port, monkeypatch, capfd):
    f = RF.get(name)
    large = RF.REGISTRY[name][1]
    n_in = f.in_w * f.in_h
    seed = sum(map(ord, name))
    ginv, vinv = real_photometric(port, n_in, seed) if photo == "real" else RF.arbitrary_photometric(n_in, seed)
    env = {"MDC_PITCH_SEARCH": "0"} if name in NO_PITCH_SEARCH else {}
    ctx, plan = adopt(api, f, ginv, vinv, monkeypatch, capfd, env)
    n = 3 if large else 4
    frames = frames_for(f, n, seed)
    oracle = Oracle(port, f, ginv, vinv, frames)
    idx = list(range(n))
    d_packed = torch.from_numpy(frames).cuda()
    ran = set()
    for pitch, must, may in layouts(f):
        if pitch:
            d = torch.full((n, f.in_h, pitch), 77, dtype=torch.uint8, device="cuda")
            d[:, :, :f.in_w] = d_packed.view(n, f.in_h, f.in_w)
        else:
            d = d_packed
        # TMA must run where it can describe the rows: the plan has box classes, the pitch is a 16-multiple
        must = must + (["tma"] if plan["staged"] and (pitch or f.in_w) % 16 == 0 else [])
        loaders = must + [x for x in may if x not in must]
        for flags in (LARGE_FLAGS if large else ALL_FLAGS):
            if not flags[0] and pitch:
                continue                                  # padded rows: rectifying mode only
            for loader in (loaders if flags[0] else ["auto"]):
                ctx.configure(use_tma=loader)
                for levels in (1, MAX_LEVELS):
                    w, h = oracle.dims(flags[0])
                    rc, outs = k1(api, ctx, d, n, pitch, flags, levels, w, h)
                    what = f"{name} photo={photo} loader={loader} pitch={pitch} flags={flags} levels={levels}"
                    if rc == 6 and loader in may and loader not in must:
                        continue
                    assert rc == 0, f"{what}: status {rc}"
                    ran.add(loader)
                    check_outputs(oracle, outs, idx, flags, what)
    assert {"auto", "ldg"} <= ran
    check_plan(name, f, ctx, plan)       # after the runs, so that a kernel that goes wrong reports its wrong bits first
    ctx.configure(use_tma="auto")
    # the host-buffer pipeline once, every level
    flags = (1, 1, 1, 1)
    host = [np.full(n * (f.out_w >> l) * (f.out_h >> l), SENTINEL, F32) for l in range(MAX_LEVELS)]
    ctx.prepare_batch_host(frames, 15, host)
    for l in range(MAX_LEVELS):
        hl = host[l].reshape(n, -1)
        for i in idx:
            assert_bits_equal(hl[i], oracle.levels(i, flags)[l], f"{name} photo={photo} prepare_batch_host frame={i} level={l}")
    # undistort<uchar> and undistort<float> (K1b), batched, against the oracle and the spec
    if photo == "real":
        imgf = np.stack([RF.special_floats(n_in, seed + 100 + i) for i in range(2)])
        for src in (frames[:2], imgf):
            d_src = torch.from_numpy(np.ascontiguousarray(src)).cuda()
            out = torch.full((2, f.out_w * f.out_h), SENTINEL, dtype=torch.float32, device="cuda")
            ctx.undistort_device(d_src, out, n_in, f.out_w * f.out_h, n_frames=2)
            torch.cuda.synchronize()
            o = out.cpu().numpy()
            for i in range(2):
                exp = port.undistort(f.rx, f.ry, f.in_w, src[i])
                assert_bits_equal(exp, spec.undistort(f.rx, f.ry, f.in_w, f.in_h, src[i]), f"{name}: oracle vs spec {src.dtype}")
                assert_bits_equal(o[i], exp, f"{name}: mdc_undistort {src.dtype} frame={i}")
    ctx.close()


@gpu
def test_checkerboard_batch_spreads_every_tile_kind_over_every_cta(api, port, monkeypatch, capfd):
    """Staged, direct, empty and black tiles interleaved, 96 frames in two chunks: 2560 work items, several per CTA, with staged
    and direct items alternating in each CTA's TMA ring.  Replicas of three frames are compared on the device, a few frames with
    the oracle."""
    f = RF.get("checkerboard_1280x1024")
    n_in = f.in_w * f.in_h
    ginv, vinv = RF.arbitrary_photometric(n_in, 5)
    ctx, plan = adopt(api, f, ginv, vinv, monkeypatch, capfd)
    check_plan("checkerboard", f, ctx, plan)
    frames = frames_for(f, 3, 77)
    oracle = Oracle(port, f, ginv, vinv, frames)
    n = 96
    idx = [i % 3 for i in range(n)]
    d = torch.from_numpy(frames).cuda()[torch.tensor(idx, device="cuda")].contiguous()
    for loader in ["auto", "ldg", "tma"] + [x for x in ("tex", "hybrid") if ctx.loader_usable(x)]:
        ctx.configure(use_tma=loader)
        for flags in LARGE_FLAGS:
            rc, outs = k1(api, ctx, d, n, 0, flags, 3, f.out_w, f.out_h)
            assert rc == 0, (loader, flags, rc)
            for l, o in enumerate(outs):
                b = o.view(torch.int32).view(n // 3, 3, -1)
                assert bool((b == b[:1]).all()), f"checkerboard loader={loader} flags={flags} level={l}: replicas differ on the device"
            check_outputs(oracle, [o[:3] for o in outs], idx[:3], flags, f"checkerboard batch loader={loader} flags={flags}")
            check_outputs(oracle, [o[-3:] for o in outs], idx[-3:], flags, f"checkerboard batch tail loader={loader} flags={flags}")
    ctx.close()


# ------------------------------------------------------------------------------------------------ tables outside D are refused
W, H, OW, OH = 64, 48, 40, 30
BAD = [
    ("x_eq_w_minus_1", W - 1.0, 10.0),
    ("x_in_last_column", W - 0.5, 10.0),
    ("x_just_below_w", float(np.nextafter(F32(W), F32(0))), 10.0),
    ("y_eq_h_minus_1", 10.0, H - 1.0),
    ("y_eq_minus_1", 10.0, -1.0),
    ("nan_x", float("nan"), 10.0),
    ("nan_y_under_valid_x", 10.0, float("nan")),
    ("inf_x", float("inf"), 10.0),
    ("inf_y", 10.0, float("inf")),
]


@gpu
@pytest.mark.parametrize("case", BAD, ids=[b[0] for b in BAD])
def test_tables_outside_the_domain_are_refused(case, api, monkeypatch):
    from mono_dataset_code_b200._lib import MdcError
    for k in [k for k in os.environ if k.startswith("MDC_")]:
        monkeypatch.delenv(k)
    _, bx, by = case
    u, v = np.meshgrid(np.arange(OW), np.arange(OH))
    rx = (u + 0.5).astype(F32).reshape(-1)
    ry = (v + 0.5).astype(F32).reshape(-1)
    rx[7], ry[7] = -1, np.nan                            # black with a NaN y: inside D
    ry[8] = np.float32(-0.75)                            # y in (-1, 0): inside D
    assert spec.in_domain(rx, ry, W, H).all()
    ginv = torch.linspace(0, 255, 256, device="cuda")
    vinv = torch.ones(W * H, device="cuda")
    ok = api.Context.from_device_tables(0, W, H, OW, OH, torch.from_numpy(rx).cuda(), torch.from_numpy(ry).cuda(), ginv, vinv)
    ok.close()
    first, second = 3 * OW + 5, 20 * OW + 2              # output pixels (5, 3) and (2, 20)
    for i in (first, second):
        rx[i], ry[i] = bx, by
    assert not spec.in_domain(rx, ry, W, H)[[first, second]].any()
    with pytest.raises(MdcError) as e:
        api.Context.from_device_tables(0, W, H, OW, OH, torch.from_numpy(rx).cuda(), torch.from_numpy(ry).cuda(), ginv, vinv)
    assert e.value.code == 1, e.value
    assert "output pixel (5, 3)" in str(e.value), e.value
