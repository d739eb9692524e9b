"""The pixel-sharded responseCalib pinned on one GPU, with the real kernels, for any number of ranks and any slice layout.

G and E are bit-identical for any number of ranks because the G-step's per-rank sums cross the ranks as integers: the ranks agree
on one fixed-point scale (mdc_rc_gstep_scale, all-reduce MAX), each slice's sums leave as 43-bit limbs (mdc_rc_gstep_accumulate_exact,
all-reduce SUM) and the summed limbs are joined (mdc_rc_gstep_finish_exact).  Here that is checked

(A) with simulated ranks in one process: the stack cut into pixel slices (bulk, ragged, 4-byte based, one-pixel and empty), the scale
    words combined with torch.maximum, the limbs summed with torch — each slice's limbs against tests/gstep_fixed_point_spec.py, G
    against the unsharded G-step and the specification, on extreme values and at the reference's 1700 x 1 MP scale;
(B) through sharding.response_calib_sharded at world sizes 2-4 on one device (gloo, one process and one context per rank), against
    mdc_response_calib on the whole stack, and the table broadcast at world size 3;
(C) through the native loop and broadcast of libmdc_b200_nccl.so at world size 1.

Ranks run in child processes that are joined against a deadline: a rank that fails fails the test, and none outlives it."""
import ctypes as C
import datetime
import os
import socket
import sys
import time

import numpy as np
import pytest

import gstep_fixed_point_spec as fx
from conftest import ROOT, assert_bits_equal
from test_gstep_fixed_point_spec import EXTREME, extreme
from test_response_calib_scale import exposures, need_free_memory, sweep_device, sweep_host
from mono_dataset_code_b200 import sharding

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

NCCL_LIB = os.path.join(ROOT, "mono_dataset_code_b200", "lib", "libmdc_b200_nccl.so")
MDC_ERR_UNSUPPORTED = 6


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from mono_dataset_code_b200 import api
    return api.Context(None, None, 0)


def f64(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float64)).cuda()


# ------------------------------------------------------------------------------------------------ (A) simulated ranks in one process
def layouts(npix):
    """name -> (cuts, base offsets in bytes or None) for npix >= 700"""
    out = {}
    for world in (1, 2, 3, 5, 8):
        for align in (128, 16):
            cuts = [sharding.shard_pixels(npix, r, world, align)[0] for r in range(world)] + [npix]
            out[f"shard_pixels(world={world}, align={align})"] = (cuts, None)
    out["bulk and ragged"] = ([0, 256, 263, 512, 611, npix], None)               # 256 | 7 | 249 | 99 | the rest
    out["4-byte base"] = ([0, 256, 512, npix], [0, 4, 0])                        # a multiple of 16 pixels that cannot take the bulk copy
    out["one-pixel slices"] = ([0, 1, 2, 130, 131, npix], None)
    out["empty slices"] = ([0, 0, 384, 384, npix, npix], None)                  # first, middle and last
    return out


def slice_copy(d, a, b, offset=0):
    """pixels [a, b) of every frame as a contiguous copy `offset` bytes past a fresh allocation; an empty slice is an empty tensor
    (torch gives it a null data pointer, as a rank without pixels has)"""
    n = d.shape[0]
    if a == b:
        return torch.empty((n, 0), dtype=torch.uint8, device="cuda")
    buf = torch.empty(n * (b - a) + offset + 16, dtype=torch.uint8, device="cuda")
    out = buf[offset:offset + n * (b - a)].view(n, b - a)
    out.copy_(d[:, a:b])
    return out


def reusable(ds):
    return ds.shape[1] % 16 == 0 and ds.data_ptr() % 16 == 0


def sharded_gstep(ctx, d, dt, dE, cuts, offsets=None):
    """The exact protocol over the slices [cuts[i], cuts[i+1]) -> (G, scale4, [(slice data, limbs, special, counts)])"""
    slices = []
    for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
        slices.append((slice_copy(d, a, b, offsets[i] if offsets else 0), dE[a:b].clone()))
    scale4, s4 = torch.zeros(4, dtype=torch.int64, device="cuda"), torch.empty(4, dtype=torch.int64, device="cuda")
    for ds, Es in slices:
        ctx.rc_gstep_scale(Es, dt, s4)
        scale4 = torch.maximum(scale4, s4)                                     # the all-reduce MAX
    parts = []
    for ds, Es in slices:
        limbs, special = torch.empty(768, dtype=torch.int64, device="cuda"), torch.empty(256, dtype=torch.float64, device="cuda")
        gnum = torch.empty(256, dtype=torch.int64, device="cuda")
        ctx.rc_gstep_accumulate_exact(ds, dt, Es, scale4, limbs, special, gnum, False)
        parts.append((ds, Es, limbs, special, gnum))
    G = finish(ctx, scale4, parts)
    return G, scale4, parts


def finish(ctx, scale4, parts):
    """the all-reduce SUM of limbs, side sums and counts, then the join"""
    tot_l = torch.stack([p[2] for p in parts]).sum(0)
    tot_s = torch.stack([p[3] for p in parts]).sum(0)
    tot_n = torch.stack([p[4] for p in parts]).sum(0)
    G = torch.empty(256, dtype=torch.float64, device="cuda")
    ctx.rc_gstep_finish_exact(scale4, tot_l, tot_s, tot_n, G)
    return G


def unsharded_gstep(ctx, d, dt, dE):
    G = torch.empty(256, dtype=torch.float64, device="cuda")
    ctx.rc_gstep(d, dt, dE, G)
    return G.cpu().numpy()


def max_E_in_one_slice(npix):
    """the largest |E| at one pixel, every other E 2^-60 of it: a slice's own scale would lie 60 binades from the agreed one"""
    data, t = sweep_host(40, npix, seed=21)
    E = np.random.default_rng(21).uniform(1.0, 2.0, npix) * 2.0 ** -60
    E[npix // 2 + 5] = 1.75
    return data, t, E


def saturated_slice(npix):
    """pixels [384, npix) saturated in every frame: E-init gives NaN there, so a slice inside that range has a zero E scale word"""
    data, t = sweep_host(40, npix, seed=22)
    data[:, 384:] = 255
    E = np.full(npix, np.nan)
    E[:384] = np.random.default_rng(22).uniform(0.5, 40.0, 384)
    return data, t, E


def negative_exposures(npix):
    """exposure times of alternating sign and two busy bins: a bin's sum is positive over the first tenth of the pixels and
    negative over the rest, slices' sums exceed 2^64 units and have opposite signs, and the total is negative"""
    n = 512
    rng = np.random.default_rng(23)
    t = rng.uniform(0.5, 1.0, n) * np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
    even = (np.arange(n) % 2 == 0)[:, None]
    first = (np.arange(npix) < npix // 10)[None, :]
    data = np.where(even == first, 10, 11).astype(np.uint8)                  # bin 10: +t in the first tenth, -t elsewhere
    data[rng.random((n, npix)) < 0.01] = 255
    E = rng.uniform(1.5, 2.0, npix)
    return data, t, E


def with_einit_E(n):
    def make(npix):
        data, t = sweep_host(n, npix, seed=n)
        return data, t, data.astype(np.float64).mean(0) + np.random.default_rng(n).uniform(-0.25, 0.25, npix)
    return make


DATA = {**{c: (lambda npix, c=c: extreme(c, npix=npix)) for c in EXTREME},
        "max_E_in_one_slice": max_E_in_one_slice, "saturated_slice": saturated_slice, "negative_exposures": negative_exposures,
        "n1024": with_einit_E(1024), "n1025": with_einit_E(1025)}


@pytest.mark.parametrize("npix", [900, 3000])
@pytest.mark.parametrize("case", list(DATA))
def test_slices_of_any_layout_give_the_unsharded_G(ctx, case, npix):
    data, t, E = DATA[case](npix)
    d, dt, dE = torch.from_numpy(data).cuda(), f64(t), f64(E)
    with np.errstate(invalid="ignore", over="ignore"):
        words = fx.scale_words(E, t)
        G_spec = fx.gstep(data, t, E)
    G_whole = unsharded_gstep(ctx, d, dt, dE)
    assert_bits_equal(G_whole, G_spec, f"{case}: unsharded G-step vs the specification")
    if case == "negative_exposures":
        limbs, _, _ = fx.accumulate(data, t, E, words)
        total = int(limbs[10]) + (int(limbs[266]) << 43) + (int(limbs[522]) << 86)
        assert total < -2 ** 64 and G_spec[10] < 0
    for name, (cuts, offsets) in layouts(npix).items():
        what = f"{case}, {name}"
        G, scale4, parts = sharded_gstep(ctx, d, dt, dE, cuts, offsets)
        assert np.array_equal(scale4.cpu().numpy(), words), f"{what}: agreed scale words"
        for (a, b), (ds, Es, limbs, special, gnum) in zip(zip(cuts[:-1], cuts[1:]), parts):
            if offsets:
                assert (ds.data_ptr() % 16 == 0) == (offsets[cuts.index(a)] % 16 == 0)
            with np.errstate(invalid="ignore", over="ignore"):
                l_ref, s_ref, n_ref = fx.accumulate(data[:, a:b], t, E[a:b], words)
            assert np.array_equal(limbs.cpu().numpy(), l_ref), f"{what}: limbs of pixels {a}..{b}"
            assert_bits_equal(special.cpu().numpy(), s_ref, f"{what}: side sums of pixels {a}..{b}")
            assert np.array_equal(gnum.cpu().numpy(), n_ref), f"{what}: counts of pixels {a}..{b}"
        g = G.cpu().numpy()
        assert_bits_equal(g, G_whole, f"{what}: sharded G vs the unsharded G-step")
        assert_bits_equal(g, G_spec, f"{what}: sharded G vs the specification")
        # kept counts: a second pass over the bulk slices with reuse_counts=1 must leave their counts alone and give the same G
        kept = [p[4].clone() for p in parts]
        for ds, Es, limbs, special, gnum in parts:
            if reusable(ds):
                ctx.rc_gstep_accumulate_exact(ds, dt, Es, scale4, limbs, special, gnum, True)
        assert all(torch.equal(k, p[4]) for k, p in zip(kept, parts)), f"{what}: reuse_counts changed counts"
        assert_bits_equal(finish(ctx, scale4, parts).cpu().numpy(), g, f"{what}: G with kept counts")


def test_reuse_counts_is_refused_on_a_ragged_or_misaligned_slice(ctx):
    from mono_dataset_code_b200 import api
    data, t = sweep_host(24, 1000, seed=5)
    d, dt = torch.from_numpy(data).cuda(), f64(t)
    E = f64(data.astype(np.float64).mean(0))
    scale4 = torch.empty(4, dtype=torch.int64, device="cuda")
    ctx.rc_gstep_scale(E, dt, scale4)
    bufs = [torch.empty(768, dtype=torch.int64, device="cuda"), torch.empty(256, dtype=torch.float64, device="cuda"),
            torch.empty(256, dtype=torch.int64, device="cuda")]
    for ds, Es in ((slice_copy(d, 0, 1000), E), (slice_copy(d, 0, 999), E[:999].clone()), (slice_copy(d, 0, 512, 4), E[:512].clone())):
        with pytest.raises(api.MdcError) as err:
            ctx.rc_gstep_accumulate_exact(ds, dt, Es, scale4, *bufs, True)
        assert err.value.code == MDC_ERR_UNSUPPORTED, str(err.value)


def test_reference_scale_over_8_slices(ctx):
    """1700 frames of 1280x1024 over eight slices, two of them ragged: the unsharded G, with fresh and with kept counts"""
    n, w, h = 1700, 1280, 1024
    npix = w * h
    need_free_memory(2.5 * n * npix / 1e9 + 4.0)
    t = exposures(n, 31)
    dt = f64(t)
    d = sweep_device(n, w, h, t, seed=32)
    E = torch.empty(npix, dtype=torch.float64, device="cuda")
    ctx.rc_einit(d, E)
    G_whole = unsharded_gstep(ctx, d, dt, E)
    cuts = [sharding.shard_pixels(npix, r, 8)[0] for r in range(8)] + [npix]
    cuts[3] += 7
    cuts[6] += 3
    G, scale4, parts = sharded_gstep(ctx, d, dt, E, cuts)
    del d
    assert [reusable(p[0]) for p in parts] == [True, True, False, False, True, False, False, True]
    assert_bits_equal(G.cpu().numpy(), G_whole, "1700 x 1 MP over 8 slices vs the unsharded G-step")
    for ds, Es, limbs, special, gnum in parts:
        if reusable(ds):
            ctx.rc_gstep_accumulate_exact(ds, dt, Es, scale4, limbs, special, gnum, True)
    assert_bits_equal(finish(ctx, scale4, parts).cpu().numpy(), G_whole, "1700 x 1 MP over 8 slices, kept counts")


def test_empty_slice_is_accepted_by_every_per_rank_call(ctx):
    """a rank without pixels: null data and E pointers, and the whole loop on one rank returns"""
    n = 12
    d = torch.empty((n, 0), dtype=torch.uint8, device="cuda")
    E = torch.empty(0, dtype=torch.float64, device="cuda")
    assert d.data_ptr() == 0 and E.data_ptr() == 0
    dt = f64(exposures(n, 3))
    G = f64(np.linspace(1.0, 300.0, 256))
    ctx.rc_einit(d, E)
    ctx.estep(d, dt, G, E)
    f = 255.0 / 300.0
    assert ctx.rc_rescale(E, G) == f
    assert G[255].item() == 300.0 * f
    acc = torch.full((2,), 7.0, dtype=torch.float64, device="cuda")
    ctx.rc_rmse_accumulate(d, dt, G, E, acc)
    assert acc.tolist() == [0.0, 0.0]
    log = sharding.response_calib_sharded(ctx, d, dt, 2, E, G)
    assert log.shape == (2, 4) and np.all(log[:, 3] == 0)


# ------------------------------------------------------------------------------------------------ ranks in child processes
def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run_ranks(world, job, *args, timeout=240.0):
    """job(rank, world, *args) on `world` processes joined in a gloo group (every rank on device 0).  A rank that raises fails the
    test at once (the others are terminated); ranks still running at the deadline are terminated and the test fails."""
    import torch.multiprocessing as mp
    pc = mp.spawn(_rank_main, args=(world, free_port(), job, args), nprocs=world, join=False)
    deadline = time.monotonic() + timeout
    try:
        while not pc.join(timeout=5.0):
            if time.monotonic() > deadline:
                pytest.fail(f"{job.__name__}: ranks still running after {timeout:.0f} s")
    finally:
        for p in pc.processes:
            if p.is_alive():
                p.terminate()
        for p in pc.processes:
            p.join(10)
            if p.is_alive():
                p.kill()
                p.join()


def _rank_main(rank, world, port_no, job, args):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port_no)
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=120))
    try:
        job(rank, world, *args)
    finally:
        dist.destroy_process_group()


def _gloo_int64_job(rank, world, out_dir):
    import torch.distributed as dist
    big = 2 ** 62 + 12345
    x = torch.tensor([big + rank, -big - rank, 1 << 52 | rank, rank], dtype=torch.int64, device="cuda")
    res = {}
    for name, op in (("max", dist.ReduceOp.MAX), ("min", dist.ReduceOp.MIN), ("sum", dist.ReduceOp.SUM)):
        y = x.clone()
        dist.all_reduce(y, op=op)
        res[name] = y.cpu().numpy()
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), **res)


def test_gloo_all_reduces_cuda_int64_exactly(tmp_path):
    """the Python loop's collectives on CUDA int64 tensors (the scale words, the count vote, limbs) through gloo: exact, MAX and MIN"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    run_ranks(2, _gloo_int64_job, str(tmp_path))
    big = 2 ** 62 + 12345
    for r in range(2):
        z = np.load(tmp_path / f"rank{r}.npz")
        assert z["max"].tolist() == [big + 1, -big, 1 << 52 | 1, 1]
        assert z["min"].tolist() == [big, -big - 1, 1 << 52, 0]
        assert z["sum"].tolist()[2:] == [(1 << 53) + 1, 1]


class RecordingOps:
    """api.Context with a record of the reuse_counts argument of every G-step pass"""

    def __init__(self, ctx):
        self.ctx, self.reuse = ctx, []

    def __getattr__(self, name):
        return getattr(self.ctx, name)

    def rc_gstep_accumulate_exact(self, *args):
        self.reuse.append(bool(args[-1]))
        return self.ctx.rc_gstep_accumulate_exact(*args)


def _python_loop_job(rank, world, stack, align, nits, out_dir):
    from mono_dataset_code_b200 import api
    z = np.load(stack)
    data, t = z["data"], z["t"]
    lo, hi = sharding.shard_pixels(data.shape[1], rank, world, align)
    local = torch.from_numpy(np.ascontiguousarray(data[:, lo:hi])).cuda()
    E = torch.zeros(hi - lo, dtype=torch.float64, device="cuda")
    G = torch.zeros(256, dtype=torch.float64, device="cuda")
    ops = RecordingOps(api.Context(None, None, 0))
    log = sharding.response_calib_sharded(ops, local, torch.from_numpy(t).cuda(), nits, E, G)
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), lo=lo, hi=hi, E=E.cpu().numpy(), G=G.cpu().numpy(), log=log,
             reuse=np.array(ops.reuse))


PY_CASES = {                    # name -> (world, n, npix, align, slices that take the bulk copy)
    "bulk_slices": (3, 40, 3840, 128, [True, True, True]),
    "one_ragged_slice": (2, 40, 1000, 128, [True, False]),
    "n1030": (3, 1030, 2000, 16, [True, True, True]),
    "empty_slice": (4, 30, 300, 128, [True, True, False, True]),
    "nan_t_in_one_slice": (2, 40, 2048, 128, [True, True]),
}


def unsharded_loop(ctx, data, t, nits):
    E = torch.zeros(data.shape[1], dtype=torch.float64, device="cuda")
    G = torch.zeros(256, dtype=torch.float64, device="cuda")
    log = ctx.response_calib(torch.from_numpy(data).cuda(), f64(t), nits, E, G)
    return E.cpu().numpy(), G.cpu().numpy(), log


def assert_logs_agree(log, ref, what):
    assert log.shape == ref.shape, what
    np.testing.assert_allclose(log[:, :3], ref[:, :3], rtol=1e-9, err_msg=what)
    assert np.array_equal(log[:, 3], ref[:, 3]), f"{what}: sample counts"


@pytest.mark.parametrize("case", list(PY_CASES))
def test_python_loop_on_ranks_of_one_gpu(ctx, case, tmp_path):
    world, n, npix, align, bulk = PY_CASES[case]
    nits = 3
    data, t = sweep_host(n, npix, seed=n + npix)
    if case == "nan_t_in_one_slice":           # non-finite products (the side sums) in rank 0's pixels only
        t[3] = np.nan
        data[3] = 255
        data[3, :64] = np.arange(64) % 21
    np.savez(tmp_path / "stack.npz", data=data, t=t)
    run_ranks(world, _python_loop_job, str(tmp_path / "stack.npz"), align, nits, str(tmp_path))
    E1, G1, log1 = unsharded_loop(ctx, data, t, nits)
    ranks = [np.load(tmp_path / f"rank{r}.npz") for r in range(world)]
    spans = [(int(z["lo"]), int(z["hi"])) for z in ranks]
    assert [(b - a) % 16 == 0 for a, b in spans] == bulk, spans
    if case == "empty_slice":
        assert spans[-1] == (300, 300)
    reuse = all(bulk)                                      # the MIN vote: counts are kept only if every slice can keep them
    for r, z in enumerate(ranks):
        assert z["reuse"].tolist() == [False] + [reuse] * (nits - 1), f"rank {r}: reuse_counts per iteration"
        assert_bits_equal(z["G"], G1, f"{case}: G on rank {r} vs the unsharded loop")
        assert_logs_agree(z["log"], log1, f"{case}: log of rank {r}")
        assert np.array_equal(z["log"], ranks[0]["log"], equal_nan=True), f"{case}: log of rank {r} vs rank 0"
    assert_bits_equal(np.concatenate([z["E"] for z in ranks]), E1, f"{case}: E of the {world} slices vs the unsharded loop")


def _broadcast_job(rank, world, files, frames_path, out_dir):
    from mono_dataset_code_b200 import api
    fov = photo = None
    iw = ih = 0
    if rank == 0:
        fov = api.UndistorterFOV(files["camera"])
        iw, ih = fov.getInputDims()
        photo = api.PhotometricUndistorter(files["pcalib"], files["vignette"], iw, ih)
    dims, tabs = sharding.broadcast_calibration(fov, photo, torch.device("cuda", 0))
    if rank == 0:
        return
    c = api.Context.from_device_tables(0, *dims, *tabs)
    np.savez(os.path.join(out_dir, f"rank{rank}.npz"), dims=np.array(dims), **k1_all_flags(c, dims, np.load(frames_path)))


def k1_all_flags(c, dims, frames):
    from mono_dataset_code_b200 import api
    iw, ih, ow, oh = dims
    d = torch.from_numpy(frames).cuda()
    out = {}
    for flags in range(16):
        r, g, v, k = flags & 1, (flags >> 1) & 1, (flags >> 2) & 1, (flags >> 3) & 1
        o = torch.empty((frames.shape[0], ow * oh if r else iw * ih), dtype=torch.float32, device="cuda")
        c.prepare_batch(d, api._flags(r, g, v, k), [o])
        out[f"k1_{flags}"] = o.cpu().numpy()
    return out


def oracle_tables(port, files, vignette=True):
    rx, ry = port.fov_from_file(files["camera"]).tables()
    ginv, _ = port.photo_tables(np.loadtxt(files["pcalib"], dtype=np.float32))
    vinv = port.vignette_maps(files["vignette_pixels"])[1].reshape(-1) if vignette else None
    return rx, ry, ginv, vinv


def assert_k1_matches_oracle(port, z, tables, dims, frames, what):
    iw, ih = dims[:2]
    for flags in range(16):
        r, g, v, k = flags & 1, (flags >> 1) & 1, (flags >> 2) & 1, (flags >> 3) & 1
        for i in range(frames.shape[0]):
            exp = port.get_image(*tables[:2], iw, ih, *tables[2:], frames[i], r, g, v, k)
            assert_bits_equal(z[f"k1_{flags}"][i], exp, f"{what}: flags {flags}, frame {i}")


FRAME_KINDS = ["uniform", "speckle", "gradient", "white", "black"]


def test_table_broadcast_on_ranks_of_one_gpu(ctx, port, dataset_dir, tmp_path):
    from mono_dataset_code_b200 import synthetic as S
    iw, ih, ow, oh = 320, 240, 288, 200
    files = dataset_dir((iw, ih, ow, oh, "crop", (0.35, 0.44, 0.49, 0.5, 0.93)))
    frames = np.stack([S.frame(i, iw, ih, FRAME_KINDS[i % 5]) for i in range(5)])
    np.save(tmp_path / "frames.npy", frames)
    run_ranks(3, _broadcast_job, files, str(tmp_path / "frames.npy"), str(tmp_path))
    tables = oracle_tables(port, files)
    for r in (1, 2):
        z = np.load(tmp_path / f"rank{r}.npz")
        assert z["dims"].tolist() == [iw, ih, ow, oh]
        assert_k1_matches_oracle(port, z, tables, (iw, ih), frames, f"rank {r}, adopted tables")


# ------------------------------------------------------------------------------------------------ (C) the native loop at world size 1
NATIVE_CASES = {"bulk": (40, 3840), "ragged": (40, 1001), "n1030": (1030, 2000)}


class _DeviceArray:
    """a raw device pointer as a torch-importable array (__cuda_array_interface__)"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f4", "data": (ptr, False), "version": 2, "strides": None}


def device_tables(c, sizes):
    from mono_dataset_code_b200._lib import lib, check
    ptrs = [C.c_void_p() for _ in range(4)]
    check(lib.mdc_ctx_device_tables(c._h, *[C.byref(p) for p in ptrs]), "mdc_ctx_device_tables")
    return [torch.as_tensor(_DeviceArray(p.value, n), device="cuda").cpu().numpy() if p.value else None for p, n in zip(ptrs, sizes)]


def _native_job(rank, world, stacks, files, frames_path, out_dir):
    from mono_dataset_code_b200 import api
    comm = sharding.NativeComm(0)
    try:
        c = api.Context(None, None, 0)
        nits = 3
        for name, path in stacks.items():
            z = np.load(path)
            d, dt = torch.from_numpy(z["data"]).cuda(), torch.from_numpy(z["t"]).cuda()
            E, G = torch.zeros(d.shape[1], dtype=torch.float64, device="cuda"), torch.zeros(256, dtype=torch.float64, device="cuda")
            log = comm.response_calib_sharded(c, d, dt, nits, E, G)
            np.savez(os.path.join(out_dir, f"native_{name}.npz"), E=E.cpu().numpy(), G=G.cpu().numpy(), log=log)
        # a rank without pixels: null data and E, every call of the loop accepts them
        d = torch.empty((12, 0), dtype=torch.uint8, device="cuda")
        E = torch.empty(0, dtype=torch.float64, device="cuda")
        G = torch.zeros(256, dtype=torch.float64, device="cuda")
        log = comm.response_calib_sharded(c, d, torch.from_numpy(exposures(12, 1)).cuda(), 2, E, G)
        np.save(os.path.join(out_dir, "native_empty_log.npy"), log)
        # the table broadcast, with and without a vignette
        fov = api.UndistorterFOV(files["camera"])
        iw, ih = fov.getInputDims()
        ow, oh = fov.getOutputDims()
        frames = np.load(frames_path)
        for tag, vig in (("vignette", files["vignette"]), ("no_vignette", "/nonexistent/vignette.png")):
            photo = api.PhotometricUndistorter(files["pcalib"], vig, iw, ih)
            assert photo.validGamma and photo.validVignette == (tag == "vignette")
            cb = comm.create_context(fov, photo)
            got = device_tables(cb, (ow * oh, ow * oh, 256, iw * ih))
            exp = list(fov.remap_tables()) + [photo.getGInv(), photo.vignette_maps()[1]]
            for k, (g_, e_) in enumerate(zip(got, exp)):
                assert (g_ is None) == (e_ is None), (tag, k)
                if e_ is not None:
                    assert np.array_equal(g_.view(np.uint32), e_.view(np.uint32)), (tag, "table", k)
            np.savez(os.path.join(out_dir, f"native_k1_{tag}.npz"), **k1_all_flags(cb, (iw, ih, ow, oh), frames))
            cb.close()
    finally:
        comm.close()


@pytest.mark.skipif(not os.path.exists(NCCL_LIB), reason="libmdc_b200_nccl.so was not built (no NCCL headers)")
def test_native_loop_and_broadcast_at_world_1(ctx, port, dataset_dir, tmp_path):
    from mono_dataset_code_b200 import synthetic as S
    stacks, ref = {}, {}
    for name, (n, npix) in NATIVE_CASES.items():
        data, t = sweep_host(n, npix, seed=n + npix + 1)
        stacks[name] = str(tmp_path / f"{name}.npz")
        np.savez(stacks[name], data=data, t=t)
        ref[name] = unsharded_loop(ctx, data, t, 3)
    iw, ih, ow, oh = 333, 217, 301, 199
    files = dataset_dir((iw, ih, ow, oh, "crop", (0.41, 0.52, 0.47, 0.52, 0.8)))
    frames = np.stack([S.frame(i, iw, ih, FRAME_KINDS[i % 5]) for i in range(5)])
    np.save(tmp_path / "frames.npy", frames)
    run_ranks(1, _native_job, stacks, files, str(tmp_path / "frames.npy"), str(tmp_path))
    for name, (E1, G1, log1) in ref.items():
        z = np.load(tmp_path / f"native_{name}.npz")
        assert_bits_equal(z["G"], G1, f"native loop {name}: G vs mdc_response_calib")
        assert_bits_equal(z["E"], E1, f"native loop {name}: E vs mdc_response_calib")
        assert_logs_agree(z["log"], log1, f"native loop {name}")
    assert np.all(np.load(tmp_path / "native_empty_log.npy")[:, 3] == 0)
    for tag in ("vignette", "no_vignette"):
        z = np.load(tmp_path / f"native_k1_{tag}.npz")
        assert_k1_matches_oracle(port, z, oracle_tables(port, files, tag == "vignette"), (iw, ih), frames, f"native broadcast, {tag}")
