"""K1 (the fused unmap + rectify + pyramid kernel) in the configurations a caller can reach besides each loader's default: the MDC_*
knobs a context reads when it is created, mdc_ctx_configure, the alignment of the frame and output pointers, the caller's streams,
and the host-side caches of texture objects and TMA descriptors.

Every run is compared bit for bit with the plain-C oracle (get_image, then pyramid).  A forced loader may refuse a call with
MDC_ERR_UNSUPPORTED (code 6) only where `LoaderModel` (a restatement of the loader rules of csrc/mdc_capi.cu) says it cannot
describe the pointer, pitch or chunk; wrong bits, any other error and any refusal the model does not predict fail.  Every call
also checks the launch-count delta the model predicts, so that a silent fall-back to another kernel fails the test."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import CALIBS, ROOT, assert_bits_equal
from mono_dataset_code_b200 import synthetic as S

try:
    import torch
except ImportError:          # the CPU guard below does not need it
    torch = None

gpu = pytest.mark.gpu

GEOMS = {
    "c1_crop_640": CALIBS["c1_crop_640"],                                   # every loader usable
    "mixed_modes": (800, 608, 96, 40, "0.9 1.2 0.5 0.5 0", S.TUM_CALIB),   # staged, direct and black tiles
    "odd_sizes": CALIBS["odd_sizes"],                                       # packed: LDG only; pitched: TMA and texture too
    "full_blackpx": CALIBS["full_blackpx"],
    "omega0": CALIBS["omega0"],
}
KINDS = ["uniform", "speckle", "gradient", "white", "black"] + ["uniform", "speckle", "gradient"] * 2
N_DISTINCT = len(KINDS)          # 11 distinct frames; batch position i holds frame (7 i + 3) % 11, so any 11 neighbours differ
MAX_LEVELS = 5                   # levels 0..2 come from the kernel's epilogue, 3..4 from the K2 chain
IN_KERNEL_LEVELS = 3
SENTINEL = -12345.0              # outputs start as this, so a pixel the kernel never writes fails the comparison
SLEEP_CYCLES = 20_000_000        # ~10 ms of spinning on a stream: long enough for an unordered reader to see the wrong bytes

# Device constants of the texture path (cudaDeviceProp on sm_90): texturePitchAlignment, textureAlignment, and the height limit of
# 2-D texture gather (maxTexture2DGather[1]).  The gather limit only matters here through MDC_TEX_MAX_ROWS, which lowers it.
TEX_PITCH_ALIGN, TEX_BASE_ALIGN, TEX_GATHER_ROWS = 32, 512, 32768
MAX_TEX_PER_LAUNCH = 128         # texture objects (chunks) one texture-gather launch takes (kMaxTex)
LOADER_IDS = {"auto": -1, "ldg": 0, "tma": 1, "tex": 2, "hybrid": 3}

REFUSE_TMA = "TMA loader requested but unusable for this geometry/pointer"
REFUSE_TEX_CHECK = "texture-gather loader requested, but its self-check did not pass"
REFUSE_TEX_GEOM = "texture-gather loader requested but unusable for this geometry/pointer"
REFUSE_PITCHED_UNMAP = "padded rows are supported in rectifying mode only"


@pytest.fixture(scope="module")
def api():
    if torch is None or not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from mono_dataset_code_b200 import api as a
    return a


class Geom:
    """One calibration: the product's models, the oracle's tables, N_DISTINCT frames and their oracle outputs."""

    def __init__(self, name, root, api, port):
        self.name = name
        self.iw, self.ih, self.ow, self.oh, mode, calib = GEOMS[name]
        files = S.write_dataset_dir(os.path.join(root, name), self.iw, self.ih, self.ow, self.oh, mode, calib)
        self.u = api.UndistorterFOV(files["camera"])
        self.p = api.PhotometricUndistorter(files["pcalib"], files["vignette"], self.iw, self.ih)
        assert self.u.isValid() and self.p.validGamma and self.p.validVignette
        f = port.fov_from_file(files["camera"])
        self.rx, self.ry = f.tables()
        self.ginv, _ = port.photo_tables(np.loadtxt(files["pcalib"], dtype=np.float32))
        _, vinv = port.vignette_maps(files["vignette_pixels"])
        self.vinv = vinv.reshape(-1)
        self.frames = np.stack([S.frame(i, self.iw, self.ih, k) for i, k in enumerate(KINDS)])
        self.d_frames = torch.from_numpy(self.frames).cuda()
        self.port = port
        self._exp = {}

    def context(self, api):
        return api.Context(self.u, self.p, 0)

    def expected(self, flags):
        """[N_DISTINCT][MAX_LEVELS] oracle outputs for flags = (rectify, gamma, vignette, kill)."""
        if flags not in self._exp:
            w, h = (self.ow, self.oh) if flags[0] else (self.iw, self.ih)
            self._exp[flags] = [self.port.pyramid(self.port.get_image(self.rx, self.ry, self.iw, self.ih, self.ginv, self.vinv, f, *flags),
                                                  w, h, MAX_LEVELS) for f in self.frames]
        return self._exp[flags]

    def level_shapes(self, rectify, levels):
        w, h = (self.ow, self.oh) if rectify else (self.iw, self.ih)
        return [(w >> l, h >> l) for l in range(levels)]

    @staticmethod
    def batch_index(n, first=0):
        return [(7 * (first + i) + 3) % N_DISTINCT for i in range(n)]

    def write_batch(self, dst, idx, pitch):
        """Copy frames `idx` into the uint8 tensor dst ([n, ih * (pitch or iw)]) on the current stream; padding bytes get 77."""
        src = self.d_frames[torch.tensor(idx, device="cuda")]
        if pitch:
            dst.fill_(77)
            dst.view(len(idx), self.ih, pitch)[:, :, :self.iw].copy_(src.view(len(idx), self.ih, self.iw))
        else:
            dst.copy_(src)

    def batch(self, idx, pitch=0):
        d = torch.empty((len(idx), self.ih * (pitch or self.iw)), dtype=torch.uint8, device="cuda")
        self.write_batch(d, idx, pitch)
        return d

    def outputs(self, n, rectify, levels, misaligned=False):
        """Output levels; misaligned puts every level at an address that is 4 but not 16 bytes past a 16-byte boundary."""
        outs = []
        for (w, h) in self.level_shapes(rectify, levels):
            if not misaligned:
                outs.append(torch.full((n, w * h), SENTINEL, dtype=torch.float32, device="cuda"))
                continue
            raw = torch.full((n * w * h + 4,), SENTINEL, dtype=torch.float32, device="cuda")
            k = ((4 - raw.data_ptr() % 16) % 16) // 4
            o = raw[k:k + n * w * h].view(n, w * h)
            assert o.data_ptr() % 16 == 4
            outs.append(o)
        return outs

    def check(self, outs, idx, flags, what):
        exp = self.expected(flags)
        for l, o in enumerate(outs):
            a = o.cpu().numpy()
            for i, k in enumerate(idx):
                assert_bits_equal(a[i], exp[k][l], f"{self.name} {what} flags={flags} frame={i} level={l}")


@pytest.fixture(scope="module")
def geoms(api, port, tmp_path_factory):
    root = str(tmp_path_factory.mktemp("k1cfg"))
    cache = {}

    def get(name):
        if name not in cache:
            cache[name] = Geom(name, root, api, port)
        return cache[name]
    return get


@pytest.fixture(scope="module")
def device_tex_ok(api, geoms):
    """Whether the texture-gather self-check passes on this device, from a context created with no MDC_* variable set."""
    saved = {k: os.environ.pop(k) for k in list(os.environ) if k.startswith("MDC_")}
    try:
        ctx = geoms("c1_crop_640").context(api)
        ok = ctx.loader_usable("tex")
        ctx.close()
    finally:
        os.environ.update(saved)
    return ok


def _env_int(env, key, default):
    return int(env[key]) if key in env else default


def tex_chunk(g, ptr, pitch, want, max_rows):
    """Frames per texture object for frames at `ptr` with row pitch `pitch` (tex_chunk_frames); 0 = not describable."""
    if pitch % TEX_PITCH_ALIGN or g.ih < 2 or ptr % TEX_BASE_ALIGN:
        return 0
    for n in range(min(want, max_rows // g.ih), 0, -1):
        if (pitch * g.ih * n) % TEX_BASE_ALIGN == 0:
            return n
    return 0


def deep_launches(levels):
    """K2 launches after the fused kernel: levels past the epilogue, two per launch."""
    return (max(levels - IN_KERNEL_LEVELS, 0) + 1) // 2


class LoaderModel:
    """What a context created under `env` does with a rectifying call: the number of fused-kernel launches, or the refusal.  A
    restatement of run_fused / run_fused_hybrid / auto_loader / tex_selfcheck in csrc/mdc_capi.cu."""

    def __init__(self, g, env, device_tex_ok):
        self.g = g
        chunk = _env_int(env, "MDC_CHUNK_FRAMES", 0)
        self.want = chunk if chunk > 0 else 48
        self.max_rows = _env_int(env, "MDC_TEX_MAX_ROWS", TEX_GATHER_ROWS)
        self.pct = max(0, min(100, _env_int(env, "MDC_HYB_TEX_PCT", 40)))
        self.auto_hybrid = _env_int(env, "MDC_AUTO_HYBRID", 0) != 0
        self.env_loader = _env_int(env, "MDC_USE_TMA", -1)
        # the self-check runs three frames whose rows are padded to the texture pitch alignment, at a 512-byte aligned address
        padded = -(-g.iw // TEX_PITCH_ALIGN) * TEX_PITCH_ALIGN
        self.tex_ok = bool(device_tex_ok and _env_int(env, "MDC_USE_TEX", 1) != 0 and tex_chunk(g, 0, padded, self.want, self.max_rows) > 0)

    def tma_ok(self, ptr, pitch):
        # every geometry here has staged tiles, so the tile plan has TMA box classes (checked through loader_usable where it can be)
        return pitch % 16 == 0 and (pitch * self.g.ih) % 16 == 0 and ptr % 16 == 0

    def _tex_launches(self, n, chunk):
        return -(-(-(-n // chunk)) // MAX_TEX_PER_LAUNCH)

    def outcome(self, loader, ptr, pitch, n):
        """-> (fused-kernel launches, None) or (None, refusal message).  loader None = the context's own setting."""
        lid = self.env_loader if loader is None else LOADER_IDS[loader]
        forced_tex = lid >= 2            # only a texture / hybrid loader the caller chose refuses; "auto" falls back instead
        tma = self.tma_ok(ptr, pitch)
        if lid < 0:
            lid = 3 if (self.tex_ok and tma and self.auto_hybrid) else 1 if tma else 2 if self.tex_ok else 0
        if lid == 0:
            return 1, None
        if lid == 1:
            return (1, None) if tma else (None, REFUSE_TMA)
        if forced_tex and not self.tex_ok:
            return None, REFUSE_TEX_CHECK
        chunk = tex_chunk(self.g, ptr, pitch, self.want, self.max_rows)
        if chunk == 0:
            return (None, REFUSE_TEX_GEOM) if forced_tex else (1, None)
        if lid == 2:
            return self._tex_launches(n, chunk), None
        n_chunks = -(-n // chunk)
        tex_chunks = max(0, min(n_chunks, (n_chunks * self.pct + 50) // 100))
        n_tex = min(n, tex_chunks * chunk)
        if n_tex == n:
            return self._tex_launches(n, chunk), None
        if n_tex == 0 or not tma:
            return 1, None
        return 1 + self._tex_launches(n_tex, chunk), None


def k1_call(api, ctx, g, model, loader, d, idx, pitch, flags, levels, what, misaligned_out=False, outs=None):
    """One prepare_batch(_pitched) call on torch's current stream, checked against the model and the oracle.  Returns whether it ran.
    outs: output levels from g.outputs, or None to allocate them here."""
    n = len(idx)
    outs = g.outputs(n, flags[0], levels, misaligned_out) if outs is None else outs
    if flags[0]:
        launches, refusal = model.outcome(loader, d.data_ptr(), pitch or g.iw, n)
        launches = None if launches is None else launches + deep_launches(levels)
    else:
        launches, refusal = (None, REFUSE_PITCHED_UNMAP) if pitch and pitch != g.iw else (levels, None)
    bits = flags[0] | flags[1] << 1 | flags[2] << 2 | flags[3] << 3
    what = f"{what} loader={loader} pitch={pitch} levels={levels}"
    before = ctx.launch_count
    try:
        if pitch:
            ctx.prepare_batch_pitched(d, pitch, bits, outs)
        else:
            ctx.prepare_batch(d, bits, outs)
    except api.MdcError as e:
        assert refusal is not None, f"{what}: refused, but this loader can describe the call: {e}"
        assert e.code == 6 and refusal in str(e), f"{what}: expected code 6 '{refusal}', got {e}"
        return False
    assert refusal is None, f"{what}: ran, but the loader should have refused ({refusal})"
    assert ctx.launch_count - before == launches, f"{what}: {ctx.launch_count - before} launches, expected {launches}"
    g.check(outs, idx, flags, what)
    return True


def make_context(api, g, monkeypatch, env, device_tex_ok):
    for k in [k for k in os.environ if k.startswith("MDC_")]:
        monkeypatch.delenv(k)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    ctx = g.context(api)
    model = LoaderModel(g, env, device_tex_ok)
    # the model's view of the context agrees with the library's own, wherever loader_usable (packed rows) can tell
    if g.iw % 16 == 0 and (g.iw * g.ih) % 16 == 0:
        assert ctx.loader_usable("tma")
    if g.iw % TEX_PITCH_ALIGN == 0:
        assert ctx.loader_usable("tex") == model.tex_ok, (env, model.tex_ok)
    return ctx, model


# ---------------------------------------------------------------------------------------------------------------- 1. knob matrix
ALL = ["auto", "ldg", "tma", "tex", "hybrid"]
CF2 = {"MDC_CHUNK_FRAMES": "2"}        # chunks of two frames, so that nine frames give the hybrid loader five chunks to split
# (id, environment at context creation, ctas_per_sm passed to configure, loaders to force (None = leave the context as created), batch)
KNOBS = [
    ("chunk1", {"MDC_CHUNK_FRAMES": "1"}, 0, ALL, 5),
    ("chunk2", {"MDC_CHUNK_FRAMES": "2"}, 0, ALL, 9),
    ("chunk7", {"MDC_CHUNK_FRAMES": "7"}, 0, ALL, 9),
    ("chunk48", {"MDC_CHUNK_FRAMES": "48"}, 0, ALL, 50),
    ("chunk64_beyond_batch", {"MDC_CHUNK_FRAMES": "64"}, 0, ALL, 9),
    ("tma_stages2", {"MDC_TMA_STAGES": "2"}, 0, ["tma"], 9),
    ("tma_stages3", {"MDC_TMA_STAGES": "3"}, 0, ["tma"], 9),
    ("tma_stages8", {"MDC_TMA_STAGES": "8"}, 0, ["tma"], 9),
    ("ctas1", {}, 1, ["ldg", "tma", "tex"], 9),
    ("ctas2", {}, 2, ["ldg", "tma", "tex"], 9),
    ("ctas3", {}, 3, ["ldg", "tma", "tex"], 9),      # with levels > 1: the staged pyramid variant compiled for 3 CTAs/SM
    ("ctas4", {}, 4, ["ldg", "tma", "tex"], 9),      # texture kernel compiled for 4 CTAs/SM
    ("ctas2_from_env", {"MDC_CTAS_PER_SM": "2"}, 0, [None], 9),
    ("tex_tiles1", {"MDC_TEX_TILES": "1"}, 0, ["tex"], 9),
    ("tex_tiles4", {"MDC_TEX_TILES": "4"}, 0, ["tex"], 9),
    ("tex_prefetch", {"MDC_TEX_PREFETCH": "1"}, 0, ["tex"], 9),
    ("tex_prefetch_ctas2", {"MDC_TEX_PREFETCH": "1"}, 2, ["tex"], 9),
    ("hybrid_tex_pct0", {**CF2, "MDC_HYB_TEX_PCT": "0"}, 0, ["hybrid"], 9),
    ("hybrid_tex_pct40", {**CF2, "MDC_HYB_TEX_PCT": "40"}, 0, ["hybrid"], 9),
    ("hybrid_tex_pct100", {**CF2, "MDC_HYB_TEX_PCT": "100"}, 0, ["hybrid"], 9),
    ("hybrid_staged_ctas1", {**CF2, "MDC_HYB_STG_CTAS": "1"}, 0, ["hybrid"], 9),
    ("hybrid_staged_ctas3", {**CF2, "MDC_HYB_STG_CTAS": "3"}, 0, ["hybrid"], 9),
    ("carveout50", {"MDC_K1_CARVEOUT": "50"}, 0, ["ldg", "tma", "tex", "hybrid"], 9),
    ("pitch_search_off", {"MDC_PITCH_SEARCH": "0"}, 0, ["ldg", "tma", "tex"], 9),
    ("auto_hybrid", {**CF2, "MDC_AUTO_HYBRID": "1"}, 0, ["auto"], 9),
    ("no_texture", {"MDC_USE_TEX": "0"}, 0, ["auto", "tex", "hybrid"], 9),
    ("chunk7_stages2_ctas3", {"MDC_CHUNK_FRAMES": "7", "MDC_TMA_STAGES": "2"}, 3, ["ldg", "tma"], 16),
    ("tex_chunk1_tiles4_prefetch_ctas4", {"MDC_CHUNK_FRAMES": "1", "MDC_TEX_TILES": "4", "MDC_TEX_PREFETCH": "1"}, 4, ["tex"], 5),
    ("hybrid_pct60_stg3_tiles1_prefetch", {**CF2, "MDC_HYB_TEX_PCT": "60", "MDC_HYB_STG_CTAS": "3", "MDC_TEX_TILES": "1",
                                           "MDC_TEX_PREFETCH": "1"}, 0, ["hybrid"], 9),
    ("no_pitch_search_stages8_carveout100", {"MDC_PITCH_SEARCH": "0", "MDC_TMA_STAGES": "8", "MDC_K1_CARVEOUT": "100"}, 2,
     ["ldg", "tma", "tex"], 9),
]
LAYOUTS = [("c1_crop_640", 0), ("mixed_modes", 0), ("odd_sizes", 0), ("odd_sizes", 352), ("full_blackpx", 0)]


@gpu
@pytest.mark.parametrize("layout", LAYOUTS, ids=[f"{n}_{'pitch%d' % p if p else 'packed'}" for n, p in LAYOUTS])
@pytest.mark.parametrize("knob", KNOBS, ids=[k[0] for k in KNOBS])
def test_knob_matrix(knob, layout, api, geoms, device_tex_ok, monkeypatch):
    name, env, ctas, loaders, n = knob
    g = geoms(layout[0])
    pitch = layout[1]
    ctx, model = make_context(api, g, monkeypatch, env, device_tex_ok)
    if env.get("MDC_AUTO_HYBRID") == "1" and ctx.loader_usable("hybrid"):
        assert ctx.auto_loader() == "hybrid"
    if env.get("MDC_USE_TEX") == "0":
        assert not ctx.loader_usable("tex") and not ctx.loader_usable("hybrid") and ctx.auto_loader() != "tex"
    idx = g.batch_index(n)
    d = g.batch(idx, pitch)
    for loader in loaders:
        if loader is not None:
            ctx.configure(use_tma=loader, ctas_per_sm=ctas)
        for flags in ((1, 1, 1, 1), (1, 0, 0, 0)):
            for levels in (1, 3, 5):
                k1_call(api, ctx, g, model, loader, d, idx, pitch, flags, levels, name)
    ctx.close()


# ------------------------------------------------------------------------------------------------ 2. the intended path really ran
@gpu
def test_hybrid_splits_the_batch_for_every_flag_combination(api, geoms, device_tex_ok, monkeypatch):
    """Seven frames in chunks of two: four go to the texture kernel and three to the staged kernel, on two streams."""
    g = geoms("c1_crop_640")
    ctx, model = make_context(api, g, monkeypatch, CF2, device_tex_ok)
    if not ctx.loader_usable("hybrid"):
        pytest.skip("the texture self-check does not pass on this device, so the hybrid loader cannot run")
    ctx.configure(use_tma="hybrid")
    idx = g.batch_index(7)
    d = g.batch(idx)
    assert model.outcome("hybrid", d.data_ptr(), g.iw, 7) == (2, None)
    for f in range(16):
        flags = (f & 1, (f >> 1) & 1, (f >> 2) & 1, (f >> 3) & 1)
        # k1_call asserts two fused launches (staged + texture) for every rectifying call
        assert k1_call(api, ctx, g, model, "hybrid", d, idx, 0, flags, 1, "hybrid split")
    ctx.close()


@gpu
def test_texture_loader_takes_two_launches_beyond_128_chunks(api, geoms, device_tex_ok, monkeypatch):
    """MDC_TEX_MAX_ROWS = one frame's height: 131 frames are 131 texture objects, more than one launch can take."""
    g = geoms("omega0")
    ctx, model = make_context(api, g, monkeypatch, {"MDC_TEX_MAX_ROWS": str(g.ih)}, device_tex_ok)
    if not ctx.loader_usable("tex"):
        pytest.skip("the texture self-check does not pass on this device")
    ctx.configure(use_tma="tex")
    idx = g.batch_index(131)
    d = g.batch(idx)
    assert tex_chunk(g, d.data_ptr(), g.iw, model.want, model.max_rows) == 1
    for levels in (1, 3, 5):
        for flags in ((1, 1, 1, 1), (1, 0, 0, 0)):
            before = ctx.launch_count
            assert k1_call(api, ctx, g, model, "tex", d, idx, 0, flags, levels, "131 one-frame chunks")
            assert ctx.launch_count - before == 2 + deep_launches(levels)
    ctx.close()


# ----------------------------------------------------------------------------------------------------------- 3. alignment classes
OFFSETS = {"tex_describable": 0, "tma_only": 16, "ldg_words": 4, "ldg_bytes": 1}


@gpu
@pytest.mark.parametrize("layout", [("c1_crop_640", 0), ("c1_crop_640", 704), ("odd_sizes", 0), ("odd_sizes", 352)],
                         ids=["c1_packed", "c1_pitch704", "odd_packed", "odd_pitch352"])
@pytest.mark.parametrize("offset", list(OFFSETS), ids=list(OFFSETS))
def test_pointer_alignment_classes(offset, layout, api, geoms, device_tex_ok, monkeypatch):
    """Frames at byte offsets 0 / 16 / 4 / 1 from a 512-byte boundary: texture-describable, TMA-only, LDG word loads, LDG byte loads.
    Output levels at 16-byte aligned addresses and at addresses 4 bytes past one.  Non-rectifying calls run unmap_kernel, whose
    vector path needs a 4-byte aligned input and 16-byte aligned output."""
    g = geoms(layout[0])
    pitch = layout[1]
    ctx, model = make_context(api, g, monkeypatch, {}, device_tex_ok)
    n = 6
    idx = g.batch_index(n, first=2)
    nbytes = n * g.ih * (pitch or g.iw)
    raw = torch.empty(nbytes + 2 * TEX_BASE_ALIGN, dtype=torch.uint8, device="cuda")
    start = (-raw.data_ptr()) % TEX_BASE_ALIGN + OFFSETS[offset]
    d = raw[start:start + nbytes].view(n, -1)
    assert d.data_ptr() % TEX_BASE_ALIGN == OFFSETS[offset]
    g.write_batch(d, idx, pitch)
    ran = []
    for loader in ALL:
        ctx.configure(use_tma=loader)
        for misaligned in (False, True):
            if k1_call(api, ctx, g, model, loader, d, idx, pitch, (1, 1, 1, 1), 4, f"offset={offset} misaligned_out={misaligned}", misaligned):
                ran.append(loader)
    assert "auto" in ran and "ldg" in ran
    # not rectifying: no loader involved; padded rows are refused (rectifying mode only)
    ctx.configure(use_tma="auto")
    for misaligned in (False, True):
        for flags in ((0, 1, 1, 1), (0, 1, 0, 0)):
            k1_call(api, ctx, g, model, "auto", d, idx, pitch, flags, 2, f"unmap offset={offset} misaligned_out={misaligned}", misaligned)
    ctx.close()


# -------------------------------------------------------------------------------------------------------------------- 4. streams
@gpu
@pytest.mark.parametrize("loader", ALL)
def test_caller_stream_orders_input_and_output(loader, api, geoms, device_tex_ok, monkeypatch):
    """K1 on a non-default torch stream whose frames are written behind a sleep on that stream: the kernels (for the hybrid both of
    them, forked onto the context's auxiliary stream) must wait for the write, and the K2 chain after them for both halves.
    Streams share a few hardware queues, so a caller stream can be serialised with the auxiliary stream by accident, which would
    hide a missing fork; three caller streams created one after the other do not all share its queue."""
    g = geoms("c1_crop_640")
    ctx, model = make_context(api, g, monkeypatch, CF2, device_tex_ok)
    if loader in ("tex", "hybrid") and not ctx.loader_usable(loader):
        pytest.skip(f"the {loader} loader is not usable on this device")
    ctx.configure(use_tma=loader)
    idx = g.batch_index(7)
    src = g.batch(idx)
    torch.cuda.synchronize()
    for rep in range(3):
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            # allocate before the sleep: a cudaMalloc behind it could make the host wait for the sleep and hide a missing dependency
            d = torch.full_like(src, 200)
            outs = g.outputs(7, 1, 5)
            torch.cuda._sleep(SLEEP_CYCLES)
            d.copy_(src)         # device to device: nothing from here to the K1 call waits on the host, so the sleep is still running
            assert k1_call(api, ctx, g, model, loader, d, idx, 0, (1, 1, 1, 1), 5, f"caller stream {rep}", outs=outs)
        s.synchronize()
    ctx.close()


@gpu
@pytest.mark.parametrize("loader", ALL)
def test_two_streams_share_one_context(loader, api, geoms, device_tex_ok, monkeypatch):
    g = geoms("c1_crop_640")
    ctx, model = make_context(api, g, monkeypatch, CF2, device_tex_ok)
    if loader in ("tex", "hybrid") and not ctx.loader_usable(loader):
        pytest.skip(f"the {loader} loader is not usable on this device")
    ctx.configure(use_tma=loader)
    batches = [(g.batch_index(n, first), torch.cuda.Stream()) for first, n in ((0, 7), (5, 9))]
    srcs = [g.batch(idx) for idx, _ in batches]
    torch.cuda.synchronize()
    jobs = []
    expected_launches = 0
    before = ctx.launch_count
    for (idx, s), src in zip(batches, srcs):
        with torch.cuda.stream(s):       # as in the test above, nothing after the sleep waits on the host
            d = torch.full_like(src, 200)
            outs = g.outputs(len(idx), 1, 4)
            torch.cuda._sleep(SLEEP_CYCLES)
            d.copy_(src)
            ctx.prepare_batch(d, 15, outs)
        jobs.append((s, idx, d, outs))
        expected_launches += model.outcome(loader, d.data_ptr(), g.iw, len(idx))[0] + deep_launches(4)
    assert ctx.launch_count - before == expected_launches
    for s, idx, d, outs in jobs:
        s.synchronize()
        g.check(outs, idx, (1, 1, 1, 1), f"two streams loader={loader}")
    ctx.close()


@gpu
@pytest.mark.parametrize("loader", ALL)
def test_context_stream_entry_points_are_synchronous(loader, api, geoms, device_tex_ok, monkeypatch):
    """stream = NULL: the call runs on the context's own stream and returns when it is done (mdc_prepare_batch, mdc_unmap_u8 and the
    batched mdc_undistort_u8 / _f32), read back without any further synchronisation."""
    from mono_dataset_code_b200._lib import lib
    g = geoms("c1_crop_640")
    ctx, model = make_context(api, g, monkeypatch, CF2, device_tex_ok)
    if loader in ("tex", "hybrid") and not ctx.loader_usable(loader):
        pytest.skip(f"the {loader} loader is not usable on this device")
    ctx.configure(use_tma=loader)
    n = 7
    idx = g.batch_index(n)
    d = g.batch(idx)
    torch.cuda.synchronize()            # the inputs come from torch's stream, which the context's stream does not wait for
    outs = g.outputs(n, 1, 5)
    torch.cuda.synchronize()
    arr = (C.c_void_p * 5)(*[o.data_ptr() for o in outs])
    assert lib.mdc_prepare_batch(ctx._h, C.c_void_p(d.data_ptr()), n, 15, arr, 5, None) == 0
    g.check(outs, idx, (1, 1, 1, 1), f"context stream loader={loader}")
    # unmapImage, batched
    un = torch.full((n, g.iw * g.ih), SENTINEL, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    assert lib.mdc_unmap_u8(ctx._h, C.c_void_p(d.data_ptr()), C.c_void_p(un.data_ptr()), g.iw * g.ih, n, 2 | 4 | 8, None) == 0
    un_h = un.cpu().numpy()
    for i, k in enumerate(idx):
        assert_bits_equal(un_h[i], g.port.unmap(g.ginv, g.vinv, g.frames[k], 1, 1, 1), f"mdc_unmap_u8 frame={i}")
    # undistort<uchar> and undistort<float>, batched
    for src, fn, host_in in ((d, lib.mdc_undistort_u8, g.frames[idx]), (un, lib.mdc_undistort_f32, un_h)):
        out = torch.full((n, g.ow * g.oh), SENTINEL, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        assert fn(ctx._h, C.c_void_p(src.data_ptr()), C.c_void_p(out.data_ptr()), g.iw * g.ih, g.ow * g.oh, n, None) == 0
        o = out.cpu().numpy()
        for i in range(n):
            assert_bits_equal(o[i], g.port.undistort(g.rx, g.ry, g.iw, host_in[i]), f"{fn.__name__} frame={i}")
        # the same through torch's stream
        out2 = torch.full_like(out, SENTINEL)
        ctx.undistort_device(src, out2, g.iw * g.ih, g.ow * g.oh, n_frames=n)
        assert_bits_equal(out2.cpu().numpy(), o, f"{fn.__name__} on torch's stream")
    ctx.close()


# ----------------------------------------------------------------------------------------------------------- 5. cache eviction
@gpu
@pytest.mark.parametrize("loader,keys", [("tex", 34), ("tma", 10)])
def test_host_caches_evict_and_rebuild(loader, keys, api, geoms, device_tex_ok, monkeypatch):
    """More (frames pointer, batch size) keys than the host caches hold (32 texture-object sets, 8 TMA descriptor sets); then the
    first keys again, after they have been evicted."""
    g = geoms("c1_crop_640")
    ctx, model = make_context(api, g, monkeypatch, {}, device_tex_ok)
    if not ctx.loader_usable(loader):
        pytest.skip(f"the {loader} loader is not usable on this device")
    ctx.configure(use_tma=loader)
    idx_all = g.batch_index(keys // 2 + 2)
    d_all = g.batch(idx_all)
    assert (g.iw * g.ih) % TEX_BASE_ALIGN == 0 and d_all.data_ptr() % TEX_BASE_ALIGN == 0      # every frame is a describable start
    key_list = [(s, n) for s in range(keys // 2) for n in (1, 2)][:keys]
    assert len({(d_all[s:s + n].data_ptr(), n) for s, n in key_list}) == keys
    for s, n in key_list + key_list[:4]:
        assert k1_call(api, ctx, g, model, loader, d_all[s:s + n], idx_all[s:s + n], 0, (1, 1, 1, 1), 1, f"cache key ({s}, {n})")
    ctx.close()


# ------------------------------------------------------------------------------- 6. MDC_USE_TMA=2/3 and the texture self-check
@gpu
@pytest.mark.parametrize("use_tma", ["2", "3"], ids=["tex", "hybrid"])
def test_texture_self_check_ignores_the_loader_setting(use_tma, api, geoms, device_tex_ok, monkeypatch):
    """Choosing the texture or hybrid loader through MDC_USE_TMA (the only way the C++ compat headers have) must not disable it."""
    if not device_tex_ok:
        pytest.skip("the texture self-check does not pass on this device even with no MDC_USE_TMA")
    g = geoms("c1_crop_640")
    ctx0, _ = make_context(api, g, monkeypatch, CF2, device_tex_ok)
    usable = ctx0.loader_usable("tex")
    ctx0.close()
    env = {**CF2, "MDC_USE_TMA": use_tma}
    ctx, model = make_context(api, g, monkeypatch, env, device_tex_ok)
    assert ctx.loader_usable("tex") == usable
    idx = g.batch_index(7)
    d = g.batch(idx)
    for levels in (1, 3):
        # loader None: the context as created; the model expects one texture launch, or the hybrid's two
        assert k1_call(api, ctx, g, model, None, d, idx, 0, (1, 1, 1, 1), levels, f"MDC_USE_TMA={use_tma}")
    ctx.close()


# ---------------------------------------------------------------------------------------------------------------- 7. CPU guard
NOT_K1_KNOBS = {
    "MDC_K1_STUDY": "floor-study variants that compute garbage by design",
    "MDC_VERBOSE": "diagnostic output only",
    "MDC_NUMA_BIND": "host-buffer pipeline, not K1",
    "MDC_HOST_CHUNK": "host-buffer pipeline, not K1",
}


def test_every_k1_knob_is_exercised_here():
    """A K1 knob read in mdc_capi.cu must be set somewhere in this module, so that a new knob cannot land untested."""
    with open(os.path.join(ROOT, "mono_dataset_code_b200", "csrc", "mdc_capi.cu")) as f:
        read = set(re.findall(r'getenv\("(MDC_\w+)"\)', f.read()))
    assert {"MDC_USE_TMA", "MDC_CHUNK_FRAMES", "MDC_TEX_MAX_ROWS"} <= read, read      # the parse finds the knobs
    assert set(NOT_K1_KNOBS) <= read, set(NOT_K1_KNOBS) - read                        # no stale exemption
    with open(os.path.abspath(__file__)) as f:
        src = f.read()
    set_here = {k for _, env, _, _, _ in KNOBS for k in env}
    set_here |= set(re.findall(r'"(MDC_\w+)": ', src.split("NOT_K1_KNOBS = {")[0]))
    set_here |= set(re.findall(r'setenv\("(MDC_\w+)"', src))
    missing = read - set(NOT_K1_KNOBS) - set_here
    assert not missing, f"K1 knobs no test in this module sets: {sorted(missing)}"
