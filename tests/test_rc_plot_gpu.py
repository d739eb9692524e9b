"""responseCalib's result images on the GPU (csrc/mdc_rc_plot.cu) against the plain-C restatement of plotE / plotG
(tests/rc_plot_oracle.py, itself pinned to the reference program's images by tests/test_rc_plot_reference_program.py):
  - mdc_rc_plot_e bit for bit on E from real loop iterations, log-uniform E over 1e-300..1e300, E placed on the truncation
    boundaries of the colour index and channel and of the 16-bit value, the special cases (max = min, +inf, near DBL_MAX, all NaN,
    negative, one pixel), 1 x 1 to 1920 x 1080, and on repeated runs;
  - the ranges of 1-8 slices (ragged and empty ones included) join into the whole image's range, and the slices' maps concatenate
    into the whole image's map;
  - mdc_rc_plot_g bit for bit; mdc_response_calib_ex returns what mdc_response_calib returns and calls back 1 + 2 nits times in the
    reference's order;
  - responseCalib_b200 on tests/golden/programs/response_calib_plots.npz: every PNG decodes to the library's plot of the E / G the loop
    had at that step, and is within one step of the reference program's image (see test_tool_writes_the_reference_programs_images);
    pcalib.txt and log.txt are the same with plots=0."""
import os
import re
import subprocess

import numpy as np
import pytest

import rc_plot_oracle as O
from mono_dataset_code_b200 import api
from mono_dataset_code_b200 import synthetic as S

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "programs", "response_calib_plots.npz")


@pytest.fixture(scope="module")
def ctx():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return api.Context(None, None, 0)


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def u16(t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def assert_plot_e(ctx, E, what, w=None, h=None):
    E = np.ascontiguousarray(E, np.float64).reshape(-1)
    w, h = (E.size, 1) if w is None else (w, h)
    bgr, e16, rng = ctx.rc_plot_e(cuda(E), w, h)
    obgr, oe16, orng = O.plot_e(E)
    assert tuple(bgr.shape) == (h, w, 3) and tuple(e16.shape) == (h, w)
    assert np.array_equal(np.array(rng).view(np.uint64), orng.view(np.uint64)), (what, rng, orng)      # the sign of a zero too
    bad = np.flatnonzero(np.any(bgr.cpu().numpy().reshape(-1, 3) != obgr, axis=1))
    assert bad.size == 0, f"{what}: {bad.size} BGR pixels differ, first E {E[bad[:4]]}"
    bad = np.flatnonzero(u16(e16).reshape(-1) != oe16)
    assert bad.size == 0, f"{what}: {bad.size} 16-bit pixels differ, first E {E[bad[:4]]}"
    return obgr, oe16


def golden_loop(ctx, on_step=None):
    g = np.load(GOLDEN)
    w, h, nits, leak = int(g["w"]), int(g["h"]), int(g["nits"]), int(g["leak_padding"])
    d = cuda(g["frames"])
    ctx.rc_leak_padding(d, w, h, leak)
    t = cuda(g["exposures"])
    E = torch.empty(w * h, dtype=torch.float64, device="cuda")
    G = torch.empty(256, dtype=torch.float64, device="cuda")
    log = ctx.response_calib(d, t, nits, E, G, on_step=on_step)
    return g, E, G, log


def loop_steps(ctx):
    """[(iteration, which, E or G as numpy, the library's plot of it)] for the golden sequence's loop"""
    steps = []

    def on_step(it, which, E, G):
        if which == "E":
            bgr, e16, rng = ctx.rc_plot_e(E, E.numel(), 1)
            steps.append((it, which, E.cpu().numpy(), (bgr.cpu().numpy().reshape(-1, 3), u16(e16).reshape(-1), rng)))
        else:
            img, mm = ctx.rc_plot_g(G)
            steps.append((it, which, G.cpu().numpy(), (img.cpu().numpy(), mm)))

    golden_loop(ctx, on_step)
    return steps


def test_plot_e_on_the_loops_irradiance(ctx):
    steps = loop_steps(ctx)
    for it, which, v, plot in steps:
        if which == "E":
            obgr, oe16, orng = O.plot_e(v)
            assert np.array_equal(plot[0], obgr) and np.array_equal(plot[1], oe16) and np.array_equal(np.array(plot[2]), orng), it


def test_plot_e_log_uniform_and_sizes(ctx):
    rng = np.random.default_rng(11)
    for w, h in [(1, 1), (3, 5), (17, 9), (1280, 1024), (1920, 1080)]:
        assert_plot_e(ctx, 10.0 ** rng.uniform(-300, 300, w * h), f"log-uniform {w}x{h}", w, h)
        E = rng.uniform(0, 600, w * h)
        E[rng.random(w * h) < 0.01] = np.nan
        assert_plot_e(ctx, E, f"uniform with NaN {w}x{h}", w, h)


def test_plot_e_on_truncation_boundaries(ctx):
    lo, hi = 0.0, 4000.0
    lmin, lmax = np.log(lo + 20), np.log(hi + 20)
    # val = 3 (exp(t) - 1) / 1.7183 at j + c / 255: the colour index and each channel's truncation
    val = (np.arange(3)[:, None] + np.arange(256)[None, :] / 255.0).reshape(-1)
    val = val[val <= 3 * (np.e - 1) / 1.7183]
    E = np.exp(lmin + np.log1p(val * 1.7183 / 3) * (lmax - lmin)) - 20
    # 16-bit value q: E = Emin + q (Emax - Emin) / 65025
    E = np.concatenate([E, lo + np.arange(0, 65026, 7) * (hi - lo) / 65025])
    ulps = np.arange(-3, 4)
    E = (E[:, None].view(np.int64) + ulps[None, :]).view(np.float64).reshape(-1)
    E = np.concatenate([[lo, hi], E[(E > lo) & (E < hi)]])
    obgr, oe16 = assert_plot_e(ctx, E, "boundaries")
    assert len(np.unique(obgr, axis=0)) > 700 and len(np.unique(oe16)) > 9000      # every segment and channel value is reached


def test_plot_e_special_cases(ctx):
    big = np.finfo(np.float64).max
    cases = {
        "constant": np.full(100, 37.5),                        # max = min: 0 / 0
        "with +inf": np.array([1.0, 5.0, np.inf, 300.0]),
        "near DBL_MAX": np.array([0.0, 1.0, big / 2, big, 1e308]),     # 65025 (E - Emin) overflows
        "all NaN": np.full(33, np.nan),
        "NaN and one value": np.array([np.nan, 4.0, np.nan]),
        "one pixel": np.array([12.0]),
        "negative": np.array([-25.0, -20.0, -19.5, -0.0, 0.0, 10.0, 1e3]),
        "zeros of both signs": np.array([0.0, -0.0, 3.0, -0.0]),
        "-0 first": np.array([-0.0, 0.0, 3.0, 0.0]),
        "-0 first, max 0": np.array([-0.0, -5.0, 0.0, -1.0]),
        "huge range": np.array([1e-300, 1e300, 1.0, 1e10]),
    }
    for name, E in cases.items():
        assert_plot_e(ctx, E, name)


def test_plot_e_range_keeps_the_first_of_equal_zeros(ctx):
    """+0 and -0 compare equal; the reference's scan keeps the one it meets first, whichever CTA or lane sees it"""
    rng = np.random.default_rng(31)
    for n in (300, 70_000, 1280 * 1024):
        for first in (0.0, -0.0):
            E = rng.uniform(1.0, 50.0, n)
            zeros = rng.choice(n, 400 if n > 400 else 50, replace=False)
            E[zeros] = np.where(rng.random(zeros.size) < 0.5, 0.0, -0.0)
            E[zeros.min()] = first
            assert_plot_e(ctx, E, f"signed zeros n={n} first={first}")
            assert_plot_e(ctx, -E, f"signed zeros, max, n={n} first={first}")


def test_plot_e_repeated_runs_agree(ctx):
    E = cuda(10.0 ** np.random.default_rng(3).uniform(-5, 5, 1280 * 1024))
    first = [x.cpu().numpy() if hasattr(x, "cpu") else x for x in ctx.rc_plot_e(E, 1280, 1024)]
    for _ in range(3):
        again = [x.cpu().numpy() if hasattr(x, "cpu") else x for x in ctx.rc_plot_e(E, 1280, 1024)]
        assert all(np.array_equal(np.asarray(a), np.asarray(b)) for a, b in zip(first, again))


def test_slices_join_into_the_whole_image(ctx):
    rng = np.random.default_rng(21)
    E = 10.0 ** rng.uniform(-3, 4, 640 * 480)
    E[rng.random(E.size) < 0.02] = np.nan
    E[rng.random(E.size) < 0.001] = 0.0
    E[rng.random(E.size) < 0.001] = -0.0                        # the first zero's sign must survive the join
    dE = cuda(E)
    whole = ctx.rc_plot_e_range(dE)
    wbgr, we16 = ctx.rc_plot_e_map(dE, whole)
    for k in range(1, 9):
        cuts = np.sort(np.concatenate([[0, E.size], rng.integers(0, E.size + 1, k - 1)]))
        if k >= 3:
            cuts[1] = cuts[2]                                     # an empty slice
        parts = [(a, b) for a, b in zip(cuts[:-1], cuts[1:])]
        joined = np.array(api.rc_plot_join_ranges([ctx.rc_plot_e_range(dE[a:b]) for a, b in parts]))
        assert np.array_equal(joined.view(np.uint64), whole.cpu().numpy().view(np.uint64)), k
        assert np.array_equal(joined.view(np.uint64), O.plot_e_range(E).view(np.uint64)), k
        maps = [ctx.rc_plot_e_map(dE[a:b], whole) for a, b in parts]
        assert np.array_equal(torch.cat([m[0] for m in maps]).cpu().numpy(), wbgr.cpu().numpy()), k
        assert np.array_equal(np.concatenate([u16(m[1]) for m in maps]), u16(we16)), k
    empty = ctx.rc_plot_e_range(dE[:0]).cpu().numpy()
    assert np.array_equal(empty, [1e10, -1e10, 1e10, -1e10])


def test_plot_g(ctx):
    rng = np.random.default_rng(8)
    steps = [v for _, which, v, _ in loop_steps(ctx) if which == "G"]
    nan_g = np.linspace(0, 300, 256)
    nan_g[:2] = np.nan
    cases = steps + [np.linspace(0, 255, 256), np.sort(rng.uniform(0, 1000, 256)), rng.normal(0, 1, 256), nan_g, np.full(256, 3.0),
                     np.r_[np.linspace(0, 1, 255), np.inf], np.r_[-np.inf, np.linspace(0, 1, 255)], 10.0 ** rng.uniform(-300, 300, 256),
                     np.full(256, np.nan)]
    for i, G in enumerate(cases):
        img, mm = ctx.rc_plot_g(cuda(G))
        oimg, omm = O.plot_g(G)
        assert np.array_equal(img.cpu().numpy(), oimg), i
        assert np.array_equal(np.array(mm), np.array(omm)), i


def test_response_calib_ex_hook_changes_nothing(ctx):
    g, E0, G0, log0 = golden_loop(ctx)
    calls = []
    _, E1, G1, log1 = golden_loop(ctx, lambda it, which, E, G: calls.append((it, which)))
    nits = int(g["nits"])
    assert calls == [(0, "E")] + [(k, w) for k in range(1, nits + 1) for w in ("G", "E")]
    for a, b in ((E0, E1), (G0, G1)):
        assert np.array_equal(a.cpu().numpy().view(np.uint64), b.cpu().numpy().view(np.uint64))
    assert np.array_equal(log0.view(np.uint64), log1.view(np.uint64))

    # work the hook leaves queued on torch's stream is finished before the loop writes E and G again: asynchronous clones, queued
    # behind a ~1 ms spin on torch's stream, equal the values a second run's hook copies to the host
    clones, copies = [], []

    def snapshot(it, which, E, G):
        torch.cuda._sleep(2_000_000)
        clones.append(E.clone() if which == "E" else G.clone())
    golden_loop(ctx, snapshot)
    golden_loop(ctx, lambda it, which, E, G: copies.append((E if which == "E" else G).cpu().numpy().copy()))
    assert len(clones) == len(copies) == 1 + 2 * nits
    for k, (c, host) in enumerate(zip(clones, copies)):
        assert np.array_equal(c.cpu().numpy().view(np.uint64), host.view(np.uint64)), k

    def boom(it, which, E, G):
        raise ValueError("from the hook")
    with pytest.raises(ValueError, match="from the hook"):
        golden_loop(ctx, boom)


def colour_position(bgr):
    """position along plotE's colour map, 0..764: (0, 0, c) -> c, (0, c, 255) -> 255 + c, (c, 255, 255) -> 510 + c"""
    b, g, r = (bgr[..., i].astype(np.int64) for i in range(3))
    return np.where(r < 255, r, np.where(g < 255, 255 + g, 510 + b))


def run_tool(tmp_path, g, tag, plots):
    from test_tools_cpp import build_tool
    w, h = int(g["w"]), int(g["h"])
    seq = tmp_path / "seq"
    if not seq.exists():
        os.makedirs(seq / "images")
        with open(seq / "times.txt", "w") as t:
            for i, (f, e) in enumerate(zip(g["frames"], g["exposures"])):
                S.write_pgm(str(seq / "images" / f"{i:05d}.pgm"), f.reshape(h, w))
                t.write(f"{i} {100.0 + 0.05 * i:.6f} {float(e):.9g}\n")
    exe = tmp_path / "responseCalib_b200"
    if not exe.exists():
        build_tool(tmp_path)
    work = tmp_path / tag
    work.mkdir()
    r = subprocess.run([str(exe), str(seq) + "/", f"iterations={int(g['nits'])}", f"leakPadding={int(g['leak_padding'])}", f"plots={plots}"],
                       cwd=work, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    return work / "photoCalibResult", r.stdout


def test_tool_writes_the_reference_programs_images(ctx, tmp_path):
    """Bound against the reference program: the GPU's G-step and rmse are within 1e-9 (relative) of the reference's, so E and G at
    every step are too, which moves plotE's colour-map position val * 255 and the 16-bit value by far less than one step; a pixel
    can only change where the reference's value lies within that distance of a truncation boundary, and then by one step.  So
    every pixel of E-k.png is within one step of the reference's along the colour map, every E-k16.png pixel within 1, and every
    G-k.png pixel within 1."""
    cv2 = pytest.importorskip("cv2")
    g = np.load(GOLDEN)
    nits, w, h = int(g["nits"]), int(g["w"]), int(g["h"])
    out1, stdout = run_tool(tmp_path, g, "plots1", 1)
    out0, stdout0 = run_tool(tmp_path, g, "plots0", 0)
    for name in ("pcalib.txt", "log.txt"):
        assert (out1 / name).read_bytes() == (out0 / name).read_bytes(), name
    assert sorted(os.listdir(out0)) == ["log.txt", "pcalib.txt"] and "Irradiance" not in stdout0
    expect = {f"E-{k}.png" for k in range(nits + 1)} | {f"E-{k}16.png" for k in range(nits + 1)} | {f"G-{k}.png" for k in range(1, nits + 1)}
    assert set(os.listdir(out1)) == expect | {"log.txt", "pcalib.txt"}

    steps = loop_steps(ctx)
    printed = re.findall(r"(Irradiance|Inv\. Response) (\S+) - (\S+)\n", stdout)
    assert len(printed) == len(steps) == 1 + 2 * nits
    assert [p[0] for p in printed] == [("Irradiance" if s[1] == "E" else "Inv. Response") for s in steps]
    assert re.search(r"init RMSE = \S+! \tIrradiance", stdout) and re.search(r"optG RMSE = \S+! \tInv\. Response", stdout)
    for (it, which, _, plot), (_, lo, hi), ref_lohi in zip(steps, printed, g["printed_ranges"]):
        read = lambda n: cv2.imread(str(out1 / n), cv2.IMREAD_UNCHANGED)      # noqa: E731
        if which == "E":
            bgr, e16 = read(f"E-{it}.png"), read(f"E-{it}16.png")
            assert bgr.shape == (h, w, 3) and e16.shape == (h, w) and e16.dtype == np.uint16
            assert np.array_equal(bgr.reshape(-1, 3), plot[0]) and np.array_equal(e16.reshape(-1), plot[1]), it
            assert (lo, hi) == (f"{plot[2][2]:f}", f"{plot[2][3]:f}"), it
            dpos = np.abs(colour_position(bgr) - colour_position(g["E_bgr"][it]))
            assert dpos.max() <= 1, (it, int((dpos > 1).sum()))
            assert np.abs(e16.astype(np.int64) - g["E16"][it]).max() <= 1, it
        else:
            img = read(f"G-{it}.png")
            assert img.shape == (256, 256) and np.array_equal(img, plot[0]), it
            assert (lo, hi) == (f"{plot[1][0]:f}", f"{plot[1][1]:f}"), it
            assert np.abs(img.astype(np.int64) - g["G8"][it - 1]).max() <= 1, it
        assert np.allclose([float(lo), float(hi)], ref_lohi, rtol=1e-8, atol=2e-6), (it, which)
