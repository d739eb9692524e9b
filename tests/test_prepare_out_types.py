"""Prepared levels stored as float16 or uint8 (MDC_OUT_F16 / MDC_OUT_U8, the mdc_*_ex calls and the dtype= keyword).

The rule: level l of type T is conv_T(R_l), where R_l is what the same call with MDC_OUT_F32 returns, pixel for pixel and bit for
bit.  conv_f16 / conv_u8 below are the oracle; the CPU tests pin them to torch's and OpenCV's own conversions, the GPU tests compare
every narrow call with conv_T of the same call's fp32 result, and count launches, so that a separate conversion pass fails."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import CALIBS
from mono_dataset_code_b200 import _lib, synthetic as S

try:
    import torch
except ImportError:
    torch = None

lib = _lib.lib
OK, INVALID_ARG, FORMAT = 0, 1, 3
F32, F16, U8 = _lib.OUT_F32, _lib.OUT_F16, _lib.OUT_U8
gpu = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------ the oracle
def conv_f16(a):
    """IEEE round to nearest even into binary16 (__float2half_rn): numpy's astype(float16)."""
    with np.errstate(over="ignore", invalid="ignore"):
        return np.asarray(a, np.float32).astype(np.float16)


def conv_u8(a):
    """cv::saturate_cast<uchar>(float) as OpenCV computes it on x86-64: cvRound = cvtss2si (round half to even; NaN, +-inf and
    anything outside int32 give INT_MIN), then the clamp to [0, 255]."""
    a = np.asarray(a, np.float32)
    inside = (a >= -2.0 ** 31) & (a < 2.0 ** 31)             # False for NaN
    with np.errstate(invalid="ignore"):
        r = np.where(inside, np.rint(a.astype(np.float64)), -2.0 ** 31)
    return np.clip(r, 0, 255).astype(np.uint8)


CONV = {F16: conv_f16, U8: conv_u8}


def assert_conv_equal(got, ref32, out_type, what):
    """got (numpy, narrow type) == conv(ref32) bit for bit; NaN compared with isnan."""
    exp = CONV[out_type](ref32)
    assert got.dtype == exp.dtype and got.shape == exp.shape, (what, got.dtype, got.shape, exp.shape)
    if out_type == U8:
        bad = np.flatnonzero(got != exp)
    else:
        gn, en = np.isnan(got), np.isnan(exp)
        bad = np.flatnonzero((gn != en) | (~gn & (got.view(np.uint16) != exp.view(np.uint16))))
    assert bad.size == 0, f"{what}: {bad.size} pixels differ, first at {bad[0]}: got {got.reshape(-1)[bad[0]]}, " \
                          f"expected {exp.reshape(-1)[bad[0]]} from {np.asarray(ref32).reshape(-1)[bad[0]]}"


SPECIAL = [0.5, -0.5, 255.4, 255.5, 255.6, -0.4, -0.6, np.nan, np.inf, -np.inf, 2.0 ** 31, -2.0 ** 31 - 256, 1e10,
           0.0, -0.0, 1.0, 254.5, 65504.0, 65519.0, 65520.0, -65520.0, 1e-8, 6e-8, -3e-8, 2.0 ** -24, 3.0 * 2.0 ** -26]


# ------------------------------------------------------------------------------------------------ CPU: the oracle itself
def test_conv_u8_is_opencvs_convert_to_8u():
    """cv2.imencode('.png', float32) converts with convertTo(CV_8U) before it encodes; decode and compare."""
    cv2 = pytest.importorskip("cv2")
    v = np.array(SPECIAL + [k + 0.5 for k in range(256)] + [k + 0.25 for k in range(-3, 260)] + [k - 0.25 for k in range(-3, 260)],
                 np.float32)
    rng = np.random.default_rng(7)
    v = np.concatenate([v, rng.uniform(-300, 600, 4000).astype(np.float32), rng.normal(0, 1e6, 1000).astype(np.float32)])
    ok, enc = cv2.imencode(".png", v.reshape(1, -1))
    assert ok
    assert np.array_equal(cv2.imdecode(enc, cv2.IMREAD_UNCHANGED).reshape(-1), conv_u8(v))
    # the cases the output-type rule names
    assert list(conv_u8(np.array([0.5, 1.5, 2.5, 255.6, 127.5, 128.5], np.float32))) == [0, 2, 2, 255, 128, 128]
    assert not conv_u8(np.array([np.nan, np.inf, -np.inf, 2.0 ** 31, 1e10], np.float32)).any()


def test_conv_f16_is_torchs_conversion():
    t = pytest.importorskip("torch")
    rng = np.random.default_rng(11)
    bits = rng.integers(0, 2 ** 32, 200000, dtype=np.uint64).astype(np.uint32)
    v = np.concatenate([np.array(SPECIAL, np.float32), bits.view(np.float32), rng.uniform(-70000, 70000, 20000).astype(np.float32),
                        (np.arange(-2048, 2048, dtype=np.float32) * 2.0 ** -25)])
    a = conv_f16(v)
    b = t.from_numpy(v).to(t.float16).numpy()
    an, bn = np.isnan(a), np.isnan(b)
    assert np.array_equal(an, bn) and np.array_equal(np.isnan(v), an)
    assert np.array_equal(a[~an].view(np.uint16), b[~bn].view(np.uint16))


# ------------------------------------------------------------------------------------------------ CPU: argument checks of the _ex calls
def _err():
    return lib.mdc_last_error().decode()


def test_unknown_out_type_is_refused_before_anything_else():
    """No context, no frames, no levels: the output type is checked first, and needs no device."""
    dummy = (C.c_void_p * 1)(None)
    for t in (-1, 3, 7, 1 << 20):
        assert lib.mdc_prepare_batch_ex(None, None, 0, 1, 15, t, dummy, 1, None) == INVALID_ARG
        assert f"unknown output type {t}" in _err()
        assert lib.mdc_prepare_batch_host_ex(None, None, 1, 15, t, dummy, 1) == INVALID_ARG
        assert f"unknown output type {t}" in _err()
        assert lib.mdc_seq_prepare_ex(None, None, 0, 1, 15, t, dummy, 1, 0) == INVALID_ARG
        assert f"unknown output type {t}" in _err()
        assert lib.mdc_seq_prepare_device_ex(None, None, 0, 1, 15, t, dummy, 1, 0, None) == INVALID_ARG
        assert f"unknown output type {t}" in _err()


def test_ex_argument_checks_without_a_device(tmp_path):
    """Levels out of range, NULL level arrays and NULL contexts are refused for every output type as for the fp32 calls."""
    from mono_dataset_code_b200 import api
    folder = tmp_path / "seq"
    S.write_dataset_dir(str(folder), 32, 24, 32, 24, "crop")
    os.makedirs(folder / "images")
    cv2 = pytest.importorskip("cv2")
    for i in range(3):
        cv2.imwrite(str(folder / "images" / f"{i:05d}.png"), np.full((24, 32), 40 * i, np.uint8))
    seq = api.Sequence(str(folder) + "/")
    assert seq.getNumImages() == 3
    one = (C.c_void_p * 9)(*([None] * 9))
    frames = np.zeros(32 * 24, np.uint8)
    for t in (F32, F16, U8):
        for levels in (0, -1, 9):
            assert lib.mdc_prepare_batch_ex(None, frames.ctypes.data, 0, 1, 15, t, one, levels, None) == INVALID_ARG
            assert lib.mdc_prepare_batch_host_ex(None, frames.ctypes.data, 1, 15, t, one, levels) == INVALID_ARG
            assert lib.mdc_seq_prepare_ex(None, seq._h, 0, 1, 15, t, one, levels, 0) == INVALID_ARG
            assert "pyramid levels" in _err()
            assert lib.mdc_seq_prepare_device_ex(None, seq._h, 0, 1, 15, t, one, levels, 0, None) == INVALID_ARG
            assert "pyramid levels" in _err()
        # a NULL level array, frames outside the sequence, a NULL context
        assert lib.mdc_prepare_batch_ex(None, frames.ctypes.data, 0, 1, 15, t, None, 1, None) == INVALID_ARG
        assert lib.mdc_prepare_batch_host_ex(None, frames.ctypes.data, 1, 15, t, None, 1) == INVALID_ARG
        assert lib.mdc_seq_prepare_ex(None, seq._h, 0, 1, 15, t, None, 1, 0) == INVALID_ARG
        assert lib.mdc_seq_prepare_ex(None, seq._h, 2, 2, 15, t, one, 1, 0) == INVALID_ARG and "outside the sequence" in _err()
        assert lib.mdc_seq_prepare_device_ex(None, seq._h, 2, 2, 15, t, one, 1, 0, None) == INVALID_ARG and "outside the sequence" in _err()
        assert lib.mdc_seq_prepare_ex(None, seq._h, 0, 1, 15, t, one, 1, 0) == INVALID_ARG
        assert lib.mdc_seq_prepare_device_ex(None, seq._h, 0, 1, 15, t, one, 1, 0, None) == INVALID_ARG
    seq.close()


def test_python_dtype_keyword_without_a_device():
    from mono_dataset_code_b200 import api
    assert api._out_type(None) == F32
    assert api._out_type(np.float16) == F16 and api._out_type(np.uint8) == U8 and api._out_type("float32") == F32
    if torch is not None:
        assert api._out_type(torch.float16) == F16 and api._out_type(torch.uint8) == U8 and api._out_type(torch.float32) == F32
    for bad in (np.float64, np.int16, "bfloat16"):
        with pytest.raises((ValueError, TypeError)):
            api._out_type(bad)
    with pytest.raises(ValueError):
        api._check_out_dtype([np.zeros(4, np.float32)], np.uint8)
    api._check_out_dtype([np.zeros(4, np.uint8), 1234], np.uint8)      # raw addresses are taken as they are


def test_header_and_bindings_declare_the_ex_calls():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    header = open(os.path.join(root, "include", "mdc_b200.h")).read()
    for name in ("mdc_prepare_batch_ex", "mdc_prepare_batch_host_ex", "mdc_seq_prepare_ex", "mdc_seq_prepare_device_ex"):
        assert f"int {name}(" in header and name in _lib.SIGNATURES
    for name, v in (("MDC_OUT_F32", 0), ("MDC_OUT_F16", 1), ("MDC_OUT_U8", 2)):
        assert f"#define {name} {v}" in header


# ------------------------------------------------------------------------------------------------ GPU
GEOMS = {
    "c1_crop_640": CALIBS["c1_crop_640"],
    "mixed_modes": (800, 608, 96, 40, "0.9 1.2 0.5 0.5 0", S.TUM_CALIB),
    "odd_sizes": CALIBS["odd_sizes"],
    "full_blackpx": CALIBS["full_blackpx"],
    "omega0": CALIBS["omega0"],
}
KINDS = ["uniform", "speckle", "gradient", "white", "black", "speckle", "gradient"]
LOADERS = {"auto": -1, "ldg": 0, "tma": 1, "tex": 2, "hybrid": 3}
TORCH_DT = {}
# two sentinels per type that no pixel can equal both of: a pixel the call never writes differs from conv(R) in one of the two runs
# (binary16 bit patterns of +-1.0009766; 0 and 255)
SENTINELS = {F16: (0x3C01, 0xBC01), U8: (0x00, 0xFF)}


def i16(bits):
    """A 16-bit pattern as the int16 torch.full takes."""
    return bits - 0x10000 if bits >= 0x8000 else bits


@pytest.fixture(scope="module")
def dev():
    if torch is None or not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    TORCH_DT.update({F32: torch.float32, F16: torch.float16, U8: torch.uint8})
    from mono_dataset_code_b200 import api
    return api


class Setup:
    def __init__(self, api, root, name, tables=None):
        """tables = (ginv [256], vinv [ih*iw]): adopted as they are (mdc_ctx_create_from_device_tables), so that values the
        photometric model's own normalisation never produces — negative, huge or infinite — reach the kernels."""
        self.iw, self.ih, self.ow, self.oh, mode, calib = GEOMS[name]
        files = S.write_dataset_dir(os.path.join(root, name), self.iw, self.ih, self.ow, self.oh, mode, calib)
        u = api.UndistorterFOV(files["camera"])
        p = api.PhotometricUndistorter(files["pcalib"], files["vignette"], self.iw, self.ih)
        assert u.isValid() and p.validGamma and p.validVignette
        self.api, self.u, self.p = api, u, p
        if tables is None:
            self.ctx = api.Context(u, p, 0)
        else:
            rx, ry = u.remap_tables()
            t = [torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in (rx, ry, tables[0], tables[1])]
            self.ctx = api.Context.from_device_tables(0, self.iw, self.ih, self.ow, self.oh, *t)
        self.frames = np.stack([S.frame(i, self.iw, self.ih, k) for i, k in enumerate(KINDS)])
        self.d_frames = torch.from_numpy(self.frames).cuda()

    def shapes(self, flags, levels):
        w, h = (self.ow, self.oh) if flags & 1 else (self.iw, self.ih)
        return [(w >> l, h >> l) for l in range(levels)]

    def outs(self, n, flags, levels, out_type, fill):
        dt = TORCH_DT[out_type]
        res = []
        for (w, h) in self.shapes(flags, levels):
            if out_type == F16:
                res.append(torch.full((n, w * h), i16(fill), dtype=torch.int16, device="cuda").view(torch.float16))
            else:
                res.append(torch.full((n, w * h), fill if out_type == U8 else -12345.0, dtype=dt, device="cuda"))
        return res

    def frames_for(self, pitch):
        if not pitch:
            return self.d_frames.view(len(KINDS), -1)
        d = torch.full((len(KINDS), self.ih, pitch), 77, dtype=torch.uint8, device="cuda")
        d[:, :, :self.iw] = self.d_frames.view(len(KINDS), self.ih, self.iw)
        return d

    def call(self, d, pitch, flags, levels, out_type, fill=0):
        """One prepare_batch(_pitched) call -> (outputs as numpy, launches)."""
        outs = self.outs(d.shape[0], flags, levels, out_type, fill)
        before = self.ctx.launch_count
        if pitch:
            self.ctx.prepare_batch_pitched(d, pitch, flags, outs, dtype=TORCH_DT[out_type])
        else:
            self.ctx.prepare_batch(d, flags, outs, dtype=TORCH_DT[out_type])
        torch.cuda.synchronize()
        return [o.cpu().numpy() for o in outs], self.ctx.launch_count - before

    def check(self, flags, levels, pitch=0, what="", types=(F16, U8)):
        d = self.frames_for(pitch)
        ref, n32 = self.call(d, pitch, flags, levels, F32)
        for t in types:
            for fill in SENTINELS[t]:
                got, n = self.call(d, pitch, flags, levels, t, fill)
                assert n == n32, f"{what} flags={flags} levels={levels} type={t}: {n} launches, the fp32 call takes {n32}"
                for l in range(levels):
                    assert_conv_equal(got[l], ref[l], t, f"{what} flags={flags} levels={levels} pitch={pitch} type={t} level={l}")
        return ref


@pytest.fixture(scope="module")
def setups(dev, tmp_path_factory):
    root = str(tmp_path_factory.mktemp("outtypes"))
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = Setup(dev, root, name)
        return cache[name]
    return get


@gpu
@pytest.mark.parametrize("layout", [("c1_crop_640", 0), ("mixed_modes", 0), ("odd_sizes", 0), ("odd_sizes", 352),
                                    ("full_blackpx", 0), ("omega0", 0)])
def test_every_flag_combination_and_level_count(layout, setups):
    name, pitch = layout
    s = setups(name)
    s.ctx.configure(use_tma=-1)
    for flags in range(16):
        if pitch and not flags & 1:
            continue                         # padded rows: rectifying mode only
        s.check(flags, 5, pitch, name)
    for levels in (1, 2, 3, 4):
        s.check(15, levels, pitch, name)
        if not pitch:
            s.check(14, levels, pitch, name)


@gpu
@pytest.mark.parametrize("loader", list(LOADERS))
@pytest.mark.parametrize("layout", [("c1_crop_640", 0), ("mixed_modes", 0), ("odd_sizes", 0), ("odd_sizes", 352)])
def test_every_loader(loader, layout, setups):
    name, pitch = layout
    s = setups(name)
    s.ctx.configure(use_tma=LOADERS[loader])
    try:
        for flags, levels in ((15, 5), (7, 3), (1, 4), (13, 1)):
            try:
                s.check(flags, levels, pitch, f"{name} loader={loader}")
            except s.api.MdcError as e:
                # a forced loader that cannot describe these frames refuses the fp32 call as well (test_k1_configurations pins when)
                assert e.code == 6, e
                return
    finally:
        s.ctx.configure(use_tma=-1)


@gpu
def test_inf_nan_and_negative_values_reach_the_conversion(dev, tmp_path):
    """Zero vignette entries (vinv = 1/0 = inf; 0 * inf = NaN) and an inverse response with negative, half-way and large values,
    adopted as device tables: inf, NaN, negatives and values above 255 / 65504 reach both conversions, on every path."""
    iw, ih = GEOMS["c1_crop_640"][:2]
    vinv = np.full((ih, iw), 1.25, np.float32)
    vinv[::7, :] = np.inf
    vinv[:, ::11] = np.inf
    vinv[3::5, 2::9] = 0.5
    ginv = np.linspace(-300.0, 70000.0, 256).astype(np.float32)
    ginv[0] = 0.0
    ginv[17:21] = (-0.5, 0.5, 2.5, 127.5)
    s = Setup(dev, str(tmp_path), "c1_crop_640", tables=(ginv, vinv.reshape(-1)))
    seen = set()
    for loader in ("auto", "ldg", "tex"):
        s.ctx.configure(use_tma=LOADERS[loader])
        if loader == "tex" and not s.ctx.loader_usable("tex"):
            continue
        for flags in (15, 7, 3, 14, 6, 2, 9):
            ref = s.check(flags, 5, 0, f"extreme loader={loader}")
            r = np.concatenate([x.reshape(-1) for x in ref])
            seen |= {"nan"} if np.isnan(r).any() else set()
            seen |= {"inf"} if np.isinf(r).any() else set()
            seen |= {"neg"} if (r < 0).any() else set()
            seen |= {"big"} if (r > 65520).any() else set()
    s.ctx.configure(use_tma=-1)
    assert seen == {"nan", "inf", "neg", "big"}, seen


@gpu
@pytest.mark.parametrize("out_type", [F16, U8])
def test_caller_stream_orders_input_and_output(out_type, setups):
    """The narrow call runs on torch's current stream: it reads frames written there just before and its levels are read there
    just after, with a long kernel in front so that an unordered access would see the wrong bytes."""
    s = setups("c1_crop_640")
    ref, _ = s.call(s.frames_for(0), 0, 15, 5, F32)
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        d = torch.zeros_like(s.frames_for(0))
        torch.cuda._sleep(20_000_000)
        d.copy_(s.frames_for(0))
        outs = s.outs(d.shape[0], 15, 5, out_type, SENTINELS[out_type][0])
        s.ctx.prepare_batch(d, 15, outs, dtype=TORCH_DT[out_type])
        copies = [o.clone() for o in outs]
    st.synchronize()
    for l in range(5):
        assert_conv_equal(copies[l].cpu().numpy(), ref[l], out_type, f"stream level {l}")


@gpu
def test_python_entry_points_allocate_and_check_the_dtype(setups):
    s = setups("odd_sizes")
    prep = s.api.FramePreparer(s.u, s.p, 0)
    ref = prep.prepare_device(s.d_frames.view(len(KINDS), -1), 1, 1, 1, 1, levels=4)
    for dt, t in ((torch.float16, F16), (torch.uint8, U8)):
        got = prep.prepare_device(s.d_frames.view(len(KINDS), -1), 1, 1, 1, 1, levels=4, dtype=dt)
        assert all(g.dtype == dt for g in got)
        for l in range(4):
            assert_conv_equal(got[l].cpu().numpy(), ref[l].cpu().numpy(), t, f"FramePreparer level {l}")
    with pytest.raises(ValueError):
        prep.prepare_device(s.d_frames.view(len(KINDS), -1), 1, 1, 1, 1, levels=2, out=ref[:2], dtype=torch.uint8)
    with pytest.raises(ValueError):
        s.ctx.prepare_batch_host(s.frames.reshape(len(KINDS), -1), 15, [np.zeros((len(KINDS), s.ow * s.oh), np.float32)], dtype=np.float16)


@gpu
@pytest.mark.parametrize("flags,levels", [(15, 5), (14, 3), (1, 1), (7, 4)])
def test_host_pipeline_gives_the_device_bytes(flags, levels, setups, monkeypatch):
    """mdc_prepare_batch_host_ex (chunks of 3 frames over the three pipe streams, a short last chunk) == the device call."""
    monkeypatch.setenv("MDC_HOST_CHUNK", "3")
    s = setups("odd_sizes")
    frames = s.frames.reshape(len(KINDS), -1)
    for t, npdt in ((F32, np.float32), (F16, np.float16), (U8, np.uint8)):
        dev_out, _ = s.call(s.frames_for(0), 0, flags, levels, t, SENTINELS.get(t, (0,))[0])
        host = [np.zeros((len(KINDS), w * h), npdt) for (w, h) in s.shapes(flags, levels)]
        s.ctx.prepare_batch_host(frames, flags, host, dtype=npdt)
        for l in range(levels):
            assert np.array_equal(host[l].view(np.uint8), dev_out[l].view(np.uint8)), (t, l)


def _sequence(dev, folder, n=70, bad=None):
    """A folder sequence of grey and 4:2:0 colour JPEGs, 8-bit PNGs and PGMs (threads = 1: chunks of 32 frames on the device feed,
    16 on the host feed); `bad` = index of an undecodable frame."""
    cv2 = pytest.importorskip("cv2")
    w, h = 64, 48
    rng = np.random.default_rng(3)
    yy, xx = np.mgrid[0:h, 0:w]
    imgs = [np.clip(xx * 3.0 + yy * 1.2 + 25 * np.sin((xx + 7 * i) * 0.09) + rng.normal(0, 4, (h, w)), 0, 255).astype(np.uint8) for i in range(9)]
    S.write_dataset_dir(str(folder), w, h, w, h, "crop")
    os.makedirs(folder / "images", exist_ok=True)
    f420 = [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420] if hasattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR") else []
    for i in range(n):
        im = imgs[i % len(imgs)]
        k = i % 4
        if i == bad:
            ext, b = "jpg", cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
        elif k == 0:
            ext, b = "jpg", cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
        elif k == 1:
            ext, b = "jpg", cv2.imencode(".jpg", np.stack([im, 255 - im, im // 2], 2), [cv2.IMWRITE_JPEG_QUALITY, 85] + f420)[1].tobytes()
        elif k == 2:
            ext, b = "png", cv2.imencode(".png", im)[1].tobytes()
        else:
            ext, b = "pgm", cv2.imencode(".pgm", im)[1].tobytes()
        (folder / "images" / f"{i:05d}.{ext}").write_bytes(b)
    with open(folder / "times.txt", "w") as f:
        for i in range(n):
            f.write(f"{i} {i * 0.05:.3f} 1.0\n")
    fov = dev.UndistorterFOV(str(folder / "camera.txt"))
    photo = dev.PhotometricUndistorter(str(folder / "pcalib.txt"), str(folder / "vignette.png"), w, h)
    return dev.Context(fov, photo, 0), dev.Sequence(str(folder) + "/"), fov, photo


@gpu
def test_sequence_feeds_give_the_device_bytes(dev, tmp_path):
    ctx, seq, fov, photo = _sequence(dev, tmp_path / "ok")
    raw = np.stack([seq.getImageRaw_internal(i) for i in range(2, 67)])
    d = torch.from_numpy(raw.reshape(raw.shape[0], -1)).cuda()
    for flags, levels in ((15, 5), (6, 3), (1, 2)):
        w, h = ctx.level_dims(0) if flags & 1 else ctx.in_dims
        shapes = [(w >> l, h >> l) for l in range(levels)]
        ref32 = [torch.empty((65, a * b), dtype=torch.float32, device="cuda") for a, b in shapes]
        ctx.prepare_batch(d, flags, ref32)
        for t, tdt, npdt in ((F16, torch.float16, np.float16), (U8, torch.uint8, np.uint8)):
            host = seq.prepare(ctx, shapes, 2, 65, flags & 1, flags & 2, flags & 4, flags & 8, threads=1, dtype=npdt)
            devo = seq.prepare_device(ctx, 2, 65, flags & 1, flags & 2, flags & 4, flags & 8, levels=levels, threads=1, dtype=tdt)
            for l in range(levels):
                r = ref32[l].cpu().numpy()
                assert_conv_equal(host[l], r, t, f"mdc_seq_prepare_ex flags={flags} level={l}")
                assert_conv_equal(devo[l].cpu().numpy(), r, t, f"mdc_seq_prepare_device_ex flags={flags} level={l}")


@gpu
@pytest.mark.parametrize("out_type", [F16, U8])
def test_sequence_feeds_stop_at_the_bad_frames_chunk(out_type, dev, tmp_path):
    """threads = 1; frame 40 cannot be decoded.  Host feed (chunks of 16): frames 0..31 written, nothing from 32 on.  Device feed
    (chunks of 32): frames 0..31 written, nothing from 32 on.  Both return MDC_ERR_FORMAT."""
    ctx, seq, fov, photo = _sequence(dev, tmp_path / "bad", n=70, bad=40)
    _, good, _, _ = _sequence(dev, tmp_path / "good", n=70)
    npdt = {F16: np.float16, U8: np.uint8}[out_type]
    tdt = {F16: torch.float16, U8: torch.uint8}[out_type]
    fill = SENTINELS[out_type][0]
    w, h = ctx.level_dims(0)
    shapes = [(w >> l, h >> l) for l in range(2)]
    ref = good.prepare(ctx, shapes, 0, 70, 1, 1, 1, 1, threads=1, dtype=npdt)
    host = [np.full((70, a * b), fill, np.uint16 if out_type == F16 else np.uint8).view(npdt) for a, b in shapes]
    ptrs = (C.c_void_p * 2)(*[o.ctypes.data for o in host])
    assert lib.mdc_seq_prepare_ex(ctx._h, seq._h, 0, 70, 15, out_type, ptrs, 2, 1) == FORMAT
    devo = [torch.full((70, a * b), i16(fill) if out_type == F16 else fill, dtype=torch.int16 if out_type == F16 else torch.uint8,
                       device="cuda").view(tdt) for a, b in shapes]
    ptrs = (C.c_void_p * 2)(*[o.data_ptr() for o in devo])
    assert lib.mdc_seq_prepare_device_ex(ctx._h, seq._h, 0, 70, 15, out_type, ptrs, 2, 1, None) == FORMAT
    for l in range(2):
        dv = devo[l].cpu().numpy()
        for got, what in ((host[l], "host feed"), (dv, "device feed")):
            assert np.array_equal(got[:32].view(np.uint8), ref[l][:32].view(np.uint8)), (what, l)
            sent = np.full(got[32:].shape, fill, np.uint16 if out_type == F16 else np.uint8)
            assert np.array_equal(got[32:].view(sent.dtype), sent), (what, l)
