"""vignetteCalib's optimiser (main_vignetteCalib.cpp:395-585) pinned bit for bit at the shapes, densities and values where it can go
wrong: the plane step against the oracle's restatement, the vignette step against tests/vc_fixed_point_spec.py (its fixed-point
arithmetic in numpy), the whole loop against the loop composed of the two, and the smoothing against the oracle.  On the CPU the
specification itself is checked against the oracle's fp32 chain and against exact sums of the same terms."""
import math

import numpy as np
import pytest

import vc_fixed_point_spec as fx
from conftest import assert_bits_equal
from mono_dataset_code_b200 import synthetic as S
from oracle.loader import PortOracle

f32 = np.float32
NO_OUTLIERS = 10000 * 10000


@pytest.fixture(scope="module")
def port():
    return PortOracle()


# ------------------------------------------------------------------------------------------------ problems
def random_maps(rng, n, gwgh, wI, hI, nan_frac=0.2):
    """Uniform positions over every valid footprint: taps reach the last row and column (x < wI - 1, y < hI - 1)."""
    xmax, ymax = np.nextafter(f32(wI - 1), f32(0)), np.nextafter(f32(hI - 1), f32(0))
    x = np.minimum(rng.uniform(0, wI - 1, (n, gwgh)).astype(f32), xmax)
    y = np.minimum(rng.uniform(0, hI - 1, (n, gwgh)).astype(f32), ymax)
    off = rng.random((n, gwgh)) < nan_frac
    x[off] = y[off] = np.nan
    return x, y


def values(rng, kind, size, lo=20.0, hi=220.0):
    if kind == "normal":
        return rng.uniform(lo, hi, size).astype(f32)
    # extreme: log-uniform magnitudes over 1e-20 .. 1e19, both signs, and zeros
    v = (np.exp(rng.uniform(math.log(1e-20), math.log(1e19), size)) * rng.choice([-1.0, 1.0], size)).astype(f32)
    v[rng.random(size) < 0.05] = 0.0
    return v


def make_problem(n, gw, gh, wI, hI, seed=0, maps="random", vals="normal"):
    """A problem of the given shape.  maps: random | integer (points at integer coordinates, incl. the last valid ones) | dense
    (hundreds of plane points start a footprint at a few pixels) | synthetic (synthetic.vignette_calib_problem)."""
    rng = np.random.default_rng(seed)
    gwgh, npx = gw * gh, wI * hI
    if maps == "synthetic":
        pr = S.vignette_calib_problem(n, gw, gh, wI, hI, seed=seed)
        images, p2x, p2y = pr["images"], pr["p2x"], pr["p2y"]
    else:
        p2x, p2y = random_maps(rng, n, gwgh, wI, hI)
        if maps == "integer":
            p2x, p2y = np.floor(p2x), np.floor(p2y)
            p2x[:, :4], p2y[:, :4] = [0, wI - 2, 0, wI - 2], [0, 0, hI - 2, hI - 2]
        elif maps == "dense":
            hot = min(3, wI - 2)
            k = rng.random((n, gwgh)) < 0.6             # most points start their footprint in a 3x2 corner of pixels
            p2x[k] = rng.integers(0, hot, k.sum()) + rng.uniform(0, 1, k.sum()).astype(f32) * f32(0.999)
            p2y[k] = rng.integers(0, 2, k.sum()) + rng.uniform(0, 1, k.sum()).astype(f32) * f32(0.999)
        if n > 1:
            p2x[1] = p2y[1] = np.nan                    # one image sees nothing
        images = values(rng, vals, (n, npx))
        images[rng.random((n, npx)) < 0.01] = np.nan
    plane = values(rng, vals, gwgh, 60.0, 180.0)
    plane[rng.random(gwgh) < 0.02] = np.nan
    vig = rng.uniform(0.5, 1.0, npx).astype(f32)
    vig[rng.random(npx) < 0.01] = np.nan
    return dict(images=np.ascontiguousarray(images), p2x=np.ascontiguousarray(p2x), p2y=np.ascontiguousarray(p2y), plane=plane, vig=vig,
                shape=(n, gw, gh, wI, hI))


def coarse_quantum(seed=0):
    """Where 2^-s is about one fp32 ulp of the sums: tens of thousands of footprints start at a few pixels and one plane colour
    of 1e4 sets the term bound, while the other colours and the images are 1 .. 3.  Rounding the terms any other way, or another
    s, shows in the result."""
    pr = make_problem(17, 150, 100, 31, 29, seed=seed, maps="dense")
    rng = np.random.default_rng(seed)
    pr["images"] = rng.uniform(1, 3, pr["images"].shape).astype(f32)
    pr["plane"] = rng.uniform(1, 3, pr["plane"].shape).astype(f32)
    pr["plane"][0] = 1e4
    return pr


def overflow_problem(seed=0):
    """Finite colours whose products w*cP*cP overflow fp32 (|w*cP*cP| > FLT_MAX at cP = 3e19, w > 0.38): plane colours of
    0.5e19 .. 1.5e19, images of 0.5e15 .. 1.5e15, and 3e19 at the 10% of the points that all start their footprint at pixel (2, 2)
    with w00 > 0.49.  That pixel's TT gets many +inf terms, its CT stays finite; the other sums stay well above 2^-s."""
    pr = make_problem(6, 40, 30, 17, 13, seed=seed)
    rng = np.random.default_rng(seed)
    hot = rng.random(40 * 30) < 0.1
    pr["p2x"][:, hot] = f32(2) + rng.uniform(0.05, 0.3, (6, hot.sum())).astype(f32)
    pr["p2y"][:, hot] = f32(2) + rng.uniform(0.05, 0.3, (6, hot.sum())).astype(f32)
    pr["plane"] = rng.uniform(0.5e19, 1.5e19, 40 * 30).astype(f32)
    pr["plane"][hot] = f32(3e19)
    pr["images"] = rng.uniform(0.5e15, 1.5e15, pr["images"].shape).astype(f32)
    return pr


def overflow_three(seed=0):
    """Exactly three overflowing terms at pixel (2, 2), from one image; without them the problem is overflow_problem's.  Three is
    the smallest number of +inf terms whose integer stand-ins (bits(inf) - bits(1.5 * 2^52) each) would wrap an int64 sum."""
    pr = overflow_problem(seed)
    pr["plane"] = np.minimum(pr["plane"], f32(1.5e19))
    pr["plane"][:3] = f32(3e19)
    pr["p2x"][:, :3] = pr["p2y"][:, :3] = np.nan
    pr["p2x"][0, :3] = pr["p2y"][0, :3] = f32(2.1)
    return pr


def special_problem(seed=0, single=False):
    """+-inf in the images and the plane colours (the side sums).  single: few enough that no pixel gets two infinite terms."""
    pr = make_problem(5, 30, 20, 23, 19, seed=seed)
    rng = np.random.default_rng(seed + 1)
    k_img, k_pl = (3, 2) if single else (40, 25)
    for i in range(pr["images"].shape[0]):
        pr["images"][i, rng.integers(0, pr["images"].shape[1], k_img)] = rng.choice([np.inf, -np.inf], k_img)
    pr["plane"][rng.integers(0, pr["plane"].size, k_pl)] = rng.choice([np.inf, -np.inf], k_pl)
    return pr


def oracle_vignette(port, pr, oth2, ia, plane=None):
    n, gw, gh, wI, hI = pr["shape"]
    return port.vc_vignette_step(pr["images"], pr["p2x"], pr["p2y"], wI, hI, pr["plane"] if plane is None else plane, pr["vig"], oth2, ia)


def spec_vignette(pr, oth2, ia, plane=None, vig=None, on_terms=None):
    n, gw, gh, wI, hI = pr["shape"]
    return fx.vignette_step(pr["images"], pr["p2x"], pr["p2y"], wI, hI, pr["plane"] if plane is None else plane,
                            pr["vig"] if vig is None else vig, oth2, ia, on_terms)


class Terms:
    """Collects the summed fp32 terms of every pixel (for exact sums and error bounds)."""

    def __init__(self):
        self.tt, self.ct, self.pix = [], [], []

    def __call__(self, tt, ct, pix):
        self.tt.append(tt.ravel()), self.ct.append(ct.ravel()), self.pix.append(pix.ravel())

    def arrays(self):
        cat = lambda a, dt: np.concatenate(a) if a else np.zeros(0, dt)
        return cat(self.tt, f32), cat(self.ct, f32), cat(self.pix, np.int64)


# ------------------------------------------------------------------------------------------------ CPU: the specification
CPU_PROBLEMS = {
    "synthetic": lambda: make_problem(14, 96, 80, 120, 90, seed=3, maps="synthetic"),
    "random_odd": lambda: make_problem(5, 101, 79, 131, 67, seed=4),
    "integer": lambda: make_problem(3, 50, 40, 23, 17, seed=5, maps="integer"),
    "dense": lambda: make_problem(17, 150, 100, 31, 29, seed=6, maps="dense"),
    "tiny": lambda: make_problem(4, 30, 30, 5, 5, seed=7),
    "extreme": lambda: make_problem(4, 60, 50, 41, 37, seed=8, vals="extreme"),
    "coarse_quantum": lambda: coarse_quantum(10),
    "overflow": lambda: overflow_problem(9),
    "overflow_three": lambda: overflow_three(9),
}
CPU_MODES = [(NO_OUTLIERS, True), (400, True), (400, False)]


def exact_sums(terms, pix, npx):
    """math.fsum of every pixel's finite terms (correctly rounded exact sums), and each pixel's number of finite terms."""
    fin = np.isfinite(terms)
    t, p = terms[fin].astype(np.float64), pix[fin]
    order = np.argsort(p, kind="stable")
    t, p = t[order], p[order]
    cuts = np.flatnonzero(np.diff(p)) + 1
    out = np.zeros(npx)
    for grp, px in zip(np.split(t, cuts), p[np.r_[0, cuts]] if p.size else []):
        out[px] = math.fsum(grp)
    return out, np.bincount(p, minlength=npx)


@pytest.mark.parametrize("oth2,ia", CPU_MODES, ids=["no_outliers", "th20_int_abs", "th20_fabs"])
@pytest.mark.parametrize("name", list(CPU_PROBLEMS))
def test_spec_matches_the_oracle_chain_and_the_exact_sums(port, name, oth2, ia):
    pr = CPU_PROBLEMS[name]()
    n, gw, gh, wI, hI = pr["shape"]
    terms = Terms()
    got = spec_vignette(pr, oth2, ia, on_terms=terms)
    exp, tt_o, ct_o, st = oracle_vignette(port, pr, oth2, ia)
    tt, ct, pix = terms.arrays()
    s = got["s"]
    kk = np.bincount(pix, minlength=wI * hI)
    slack = {}
    for which, acc, t32, oracle_sum, tr in (("TT", got["tt"], got["t"], tt_o, tt), ("CT", got["ct"], got["c"], ct_o, ct)):
        # against the exact sums: every term is rounded to a multiple of 2^-s, so a pixel's K terms are off by at most K * 2^-(s+1)
        ex, k = exact_sums(tr, pix, wI * hI)
        fixed = np.ldexp(acc.astype(np.float64), -s)
        assert np.all(np.abs(fixed - ex) <= k * math.ldexp(0.5, -s) + np.abs(ex) * 2.0 ** -52), which
        # against the oracle's sequential fp32 chain: it is off by at most (K-1) * 2^-24 * sum|term|, the spec by the final rounding
        # and the fixed-point bound above
        with np.errstate(over="ignore", invalid="ignore"):
            mag = np.bincount(pix, np.abs(tr.astype(np.float64)), wI * hI) if pix.size else np.zeros(wI * hI)
            slack[which] = (kk + 1) * 2.0 ** -24 * mag + k * math.ldexp(0.5, -s)
            fin = np.isfinite(oracle_sum) & np.isfinite(t32)
            assert np.array_equal(np.isnan(oracle_sum), np.isnan(t32)), which
            assert np.array_equal(np.isposinf(oracle_sum), np.isposinf(t32)) and np.array_equal(np.isneginf(oracle_sum), np.isneginf(t32)), which
            err = np.abs(oracle_sum[fin].astype(np.float64) - t32[fin].astype(np.float64))
            assert np.all(err <= slack[which][fin]), which
    # TT >= 1 decides NaN: where the oracle's TT is farther from 1 than that bound, the masks must agree
    with np.errstate(invalid="ignore"):
        firm = ~(np.abs(tt_o.astype(np.float64) - 1.0) <= slack["TT"])
    assert np.array_equal(np.isnan(got["vignette"])[firm], np.isnan(exp)[firm])
    # (not where CT cancels and 2^-s is coarse next to most sums, nor where the oracle's chain of ~10^4 terms is itself off by more)
    if name not in ("extreme", "coarse_quantum"):
        m = np.isfinite(exp) & np.isfinite(got["vignette"]) & (np.abs(exp) > 1e-3)
        assert np.all(np.abs(got["vignette"][m] - exp[m]) <= 2e-5 * np.abs(exp[m]))
        assert m.sum() > 20 or name.startswith("overflow")
    assert got["R"] == st[1]
    assert got["E"] == st[0] or abs(got["E"] - st[0]) <= 1e-9 * abs(st[0]) or (math.isnan(got["E"]) and math.isnan(st[0]))


@pytest.mark.parametrize("make", [overflow_problem, overflow_three], ids=["many", "three"])
def test_overflowing_products_make_tt_infinite_as_in_the_reference(port, make):
    """w*cP*cP of finite colours can overflow fp32.  The reference's TT becomes +inf and the factor CT/inf = 0; so must the spec's."""
    pr = make(9)
    n, gw, gh, wI, hI = pr["shape"]
    got = spec_vignette(pr, NO_OUTLIERS, True)
    exp, tt_o, _, _ = oracle_vignette(port, pr, NO_OUTLIERS, True)
    hot = 2 + 2 * wI
    assert np.isposinf(tt_o[hot]) and np.isposinf(got["t"][hot]) and got["tt_special"][hot] == np.inf
    assert exp[hot] == 0 and got["vignette"][hot] == 0
    assert np.array_equal(np.isposinf(tt_o), np.isposinf(got["t"]))


def test_scale_exponent_edges():
    bits = lambda v: int(f32(v).view(np.uint32))
    assert fx.scale_exponent(0, 0, 0) == 0 and fx.scale_exponent(0, bits(5.0), 10) == 0
    # one colour of 1, no footprint: term bound 1.001 -> s = 50 - 1; 1000 footprints: total 4004 * 1.001 < 2^12 -> s = 62 - 12
    assert fx.scale_exponent(bits(1.0), bits(1.0), 0) == 49
    # the total bound 1.001 * (4c + 4) reaches 2^13 between c = 2044 and 2045: s_total = 62 - 14 takes over from s_term = 49
    assert fx.scale_exponent(bits(1.0), bits(1.0), 2044) == 49 and fx.scale_exponent(bits(1.0), bits(1.0), 2045) == 48
    # the larger of the two colour bounds; tiny colours give a large s
    assert fx.scale_exponent(bits(2.0), bits(8.0), 0) == 50 - 5 and fx.scale_exponent(bits(8.0), bits(2.0), 0) == 50 - 7
    assert fx.scale_exponent(bits(1e-20), 0, 5) == 50 - (fx.ilogb(float(f32(1e-20)) ** 2 * 1.001) + 1) == 182
    assert fx.scale_exponent(bits(3e38), bits(3e38), 2 ** 31) == 62 - (fx.ilogb(float(f32(3e38)) ** 2 * 1.001 * (4.0 * 2 ** 31 + 4)) + 1)


def dense_real_shape(n, seed=11):
    """1000x1000 plane points seen from n poses in 1280x1024 images, each pose squeezing the grid into about 200x200 pixels around
    the image centre (about 25 footprints per pixel and pose), and exposure-normalised values from 1 to 1e4."""
    rng = np.random.default_rng(seed)
    gw = gh = 1000
    wI, hI = 1280, 1024
    gy, gx = np.mgrid[0:gh, 0:gw].astype(np.float64)
    u, v = (gx / gw - 0.5).ravel(), (gy / gh - 0.5).ravel()
    p2x, p2y = np.empty((n, gw * gh), f32), np.empty((n, gw * gh), f32)
    for i in range(n):
        ang, sc = rng.uniform(-0.5, 0.5), rng.uniform(170, 230)
        tx, ty = 640 + rng.uniform(-20, 20), 512 + rng.uniform(-20, 20)
        p2x[i] = tx + sc * (np.cos(ang) * u - np.sin(ang) * v)
        p2y[i] = ty + sc * (np.sin(ang) * u + np.cos(ang) * v)
    images = np.exp(rng.uniform(0.0, math.log(1e4), (n, wI * hI))).astype(f32)
    plane = np.exp(rng.uniform(0.0, math.log(1e4), gw * gh)).astype(f32)
    vig = np.ones(wI * hI, f32)
    return dict(images=images, p2x=p2x, p2y=p2y, plane=plane, vig=vig, shape=(n, gw, gh, wI, hI))


def test_fixed_point_error_at_the_real_shape_and_density():
    """The fixed-point sums against the exact sums of the same fp32 terms at the reference's shape, with thousands of footprints per
    pixel and values up to 1e4.  A term is rounded to a multiple of 2^-s; the exact sum is sum(q) - sum(q - term * 2^s) scaled by
    2^-s, where each rounding error q - term * 2^s is exact in float64 and their sum (<= K/2 in magnitude) is accurate to ~1e-12."""
    pr = dense_real_shape(64)
    n, gw, gh, wI, hI = pr["shape"]
    npx = wI * hI
    err, cnt = np.zeros(npx), np.zeros(npx)
    sc = math.ldexp(1.0, fx.scale_exponent(*fx.bounds(pr["images"], pr["p2x"], pr["p2y"], pr["plane"], wI)))

    def on_terms(tt, ct, pix):
        x = tt.ravel().astype(np.float64) * sc
        err[:] += np.bincount(pix.ravel(), np.rint(x) - x, npx)
        cnt[:] += np.bincount(pix.ravel(), minlength=npx)

    got = spec_vignette(pr, NO_OUTLIERS, True, on_terms=on_terms)
    s, (_, _, max_count) = got["s"], got["bounds"]
    assert max_count >= 1000
    fixed = np.ldexp(got["tt"].astype(np.float64), -s)
    exact = fixed - np.ldexp(err, -s)
    abs_err = np.abs(fixed - exact)
    # what the code guarantees: K terms are off by at most K * 2^-(s+1); 2^-s <= max(2^-49, (4c+4) * 2^-61) * 1.001 * P * max(P, I)
    assert np.all(abs_err <= cnt * math.ldexp(0.5, -s) * (1 + 1e-9))
    P, I = float(f32(pr["plane"].max())), float(f32(pr["images"].max()))
    assert math.ldexp(1.0, -s) <= max(2.0 ** -49, (4 * max_count + 4) * 2.0 ** -61) * 1.001 * P * max(P, I)
    # what that means where the reference divides (TT >= 1): the error relative to the sum, and in fp32 ulps of the sum
    live = exact >= 1.0
    rel = abs_err[live] / exact[live]
    ulp = np.spacing(exact[live].astype(f32)).astype(np.float64)
    worst_rel, worst_ulp = float(rel.max()), float((abs_err[live] / ulp).max())
    print(f"\nfixed point at n={n}, {gw}x{gh} points, {wI}x{hI} px: max_count={max_count}, s={s}, "
          f"max error at TT >= 1: {worst_rel:.3g} relative, {worst_ulp:.3g} fp32 ulps; at TT >= 1e6: "
          f"{float((abs_err / np.maximum(exact, 1))[exact >= 1e6].max()):.3g} relative")
    assert worst_rel < 2e-5                           # the tolerance the suite allows the vignette against the reference


# ------------------------------------------------------------------------------------------------ GPU: bit for bit
@pytest.fixture(scope="module")
def gpu():
    torch = pytest.importorskip("torch")
    from mono_dataset_code_b200 import api
    return torch, api.Context(None, None, 0)


def to_dev(torch, a):
    """A CUDA copy; an empty array becomes an empty view of a one-row buffer, so that its pointer is not null."""
    if a.size == 0:
        return torch.zeros((1,) + a.shape[1:], dtype=torch.float32, device="cuda")[:0]
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gpu_steps(gpu, pr, oth2, ia, plane, vig, repeats=2):
    """The plane step (from `plane`, with `vig`) and the vignette step (from `plane`, `vig`) on the device, each run `repeats` times;
    the repeats must give the same bits.  Returns ((plane, E, R), (vignette, E, R))."""
    torch, ctx = gpu
    n, gw, gh, wI, hI = pr["shape"]
    d = [to_dev(torch, pr[k]) for k in ("images", "p2x", "p2y")]
    res = []
    for step in ("plane", "vignette"):
        outs = []
        for _ in range(repeats):
            if step == "plane":
                pc = torch.from_numpy(plane.copy()).cuda()
                E, R = ctx.vc_plane_step(*d, gw, gh, wI, hI, torch.from_numpy(vig).cuda(), pc, oth2, ia)
                outs.append((pc.cpu().numpy(), E, R))
            else:
                v = torch.from_numpy(vig.copy()).cuda()
                E, R = ctx.vc_vignette_step(*d, gw, gh, wI, hI, torch.from_numpy(plane).cuda(), v, oth2, ia)
                outs.append((v.cpu().numpy(), E, R))
        for o in outs[1:]:
            assert np.array_equal(o[0].view(np.uint32), outs[0][0].view(np.uint32)), f"{step} step: a repeat gave other bits"
            assert (o[1], o[2]) == (outs[0][1], outs[0][2]) or (math.isnan(o[1]) and math.isnan(outs[0][1])), f"{step} step: a repeat gave other stats"
        res.append(outs[0])
    return res


def assert_stats(E, R, E_exp, R_exp, what):
    assert R == R_exp, (what, R, R_exp)
    assert E == E_exp or abs(E - E_exp) <= 1e-9 * abs(E_exp) or (math.isnan(E) and math.isnan(E_exp)), (what, E, E_exp)


def check_steps(port, gpu, pr, oth2, ia, plane=None, vig=None):
    n, gw, gh, wI, hI = pr["shape"]
    plane = pr["plane"] if plane is None else plane
    vig = pr["vig"] if vig is None else vig
    (p_got, pE, pR), (v_got, vE, vR) = gpu_steps(gpu, pr, oth2, ia, plane, vig)
    p_exp, _, _, pst = port.vc_plane_step(pr["images"], pr["p2x"], pr["p2y"], wI, hI, vig, plane, oth2, ia)
    assert_bits_equal(p_got, p_exp, "plane step")
    assert_stats(pE, pR, pst[0], pst[1], "plane step")
    spec = fx.vignette_step(pr["images"], pr["p2x"], pr["p2y"], wI, hI, plane, vig, oth2, ia)
    assert_bits_equal(v_got, spec["vignette"], "vignette step")
    assert_stats(vE, vR, spec["E"], spec["R"], "vignette step")
    return p_got, v_got, spec


def resid_problem(seed=0):
    """Points at integer coordinates (cI is one image pixel), plane 1, vignette 1: residuals (image - 1)^2 of exactly 400, just
    either side of it, and at or above 2^31 (46341^2), where the truncating outlier test never fires and fabs does."""
    pr = make_problem(3, 40, 30, 29, 21, seed=seed, maps="integer")
    rng = np.random.default_rng(seed)
    d = rng.choice(np.array([0.5, 19.99, 20.0, 20.01, 46340.0, 46341.0, 1e5, 1e6], f32), pr["images"].shape)
    pr["images"] = (f32(1) + d * rng.choice(np.array([1, -1], f32), d.shape)).astype(f32)
    pr["plane"] = np.ones_like(pr["plane"])
    pr["vig"] = np.ones_like(pr["vig"])
    return pr


def all_nan_vignette(seed=0):
    pr = make_problem(4, 33, 21, 19, 15, seed=seed)
    pr["vig"][:] = np.nan
    return pr


def no_positive_factor(seed=0):
    """Negative images and positive plane colours: every CT/TT < 0, so the maximum stays 0 and the normalisation divides by 0."""
    pr = make_problem(4, 33, 21, 19, 15, seed=seed)
    pr["images"] = -np.abs(pr["images"])
    return pr


def tiny_colours(seed=0):
    """Plane colours of 1e-20: every TT < 1, the vignette is NaN everywhere."""
    pr = make_problem(4, 33, 21, 19, 15, seed=seed)
    pr["plane"] = np.full_like(pr["plane"], 1e-20)
    return pr


GPU_PROBLEMS = {
    **{f"n{n}": (lambda n=n: make_problem(n, 37, 29, 41, 23, seed=20 + n)) for n in (0, 1, 2, 3, 4, 5, 17)},
    "points_1": lambda: make_problem(6, 1, 1, 11, 9, seed=30),
    "points_7919": lambda: make_problem(4, 7919, 1, 53, 41, seed=31),
    "points_70001": lambda: make_problem(3, 70001, 1, 97, 61, seed=32),
    "points_1100x1000": lambda: make_problem(3, 1100, 1000, 64, 48, seed=33),
    "image_5x5": lambda: make_problem(5, 23, 19, 5, 5, seed=34),
    "image_131x67": lambda: make_problem(5, 101, 79, 131, 67, seed=35),
    "image_1280x1024": lambda: make_problem(2, 300, 200, 1280, 1024, seed=36),
    "integer_points": lambda: make_problem(4, 50, 40, 23, 17, seed=37, maps="integer"),
    "dense": lambda: make_problem(17, 150, 100, 31, 29, seed=38, maps="dense"),
    "extreme": lambda: make_problem(4, 60, 50, 41, 37, seed=39, vals="extreme"),
    "coarse_quantum": lambda: coarse_quantum(47),
    "overflow": lambda: overflow_problem(40),
    "overflow_three": lambda: overflow_three(48),
    "residuals": lambda: resid_problem(41),
    "vignette_all_nan": lambda: all_nan_vignette(42),
    "no_positive_factor": lambda: no_positive_factor(43),
    "tiny_colours": lambda: tiny_colours(44),
    "infinite_single": lambda: special_problem(45, single=True),
    "infinite_many": lambda: special_problem(46),
}
GPU_MODES = [(NO_OUTLIERS, True), (400, True), (400, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("oth2,ia", GPU_MODES, ids=["no_outliers", "th20_int_abs", "th20_fabs"])
@pytest.mark.parametrize("name", list(GPU_PROBLEMS))
def test_steps_are_bit_identical(port, gpu, name, oth2, ia):
    """Plane step = the oracle, vignette step = the spec, bit for bit (NaN positions included), on every shape and value regime."""
    pr = GPU_PROBLEMS[name]()
    _, v_got, spec = check_steps(port, gpu, pr, oth2, ia)
    if name.startswith("infinite") or name.startswith("overflow"):
        # the side sums: where the oracle's fp32 chain is NaN / +-inf / 0, so is the device's
        exp, tt_o, ct_o, _ = oracle_vignette(port, pr, oth2, ia)
        for what, a in (("nan", np.isnan), ("+inf", np.isposinf), ("-inf", np.isneginf)):
            assert np.array_equal(a(spec["t"]), a(tt_o)) and np.array_equal(a(spec["c"]), a(ct_o)), what
        assert np.array_equal(np.isnan(v_got), np.isnan(exp)) and np.array_equal(v_got == 0, exp == 0)
    if name.startswith("overflow") and ia:           # (with fabs, residuals of ~1e38 are all outliers)
        wI = pr["shape"][3]
        assert np.isposinf(spec["t"][2 + 2 * wI]) and v_got[2 + 2 * wI] == 0


@pytest.mark.gpu
def test_real_shape_once(port, gpu):
    """The reference's scale: 1000x1000 plane points, 1280x1024 images, 256 poses."""
    n, gw, gh, wI, hI = 256, 1000, 1000, 1280, 1024
    pr = S.vignette_calib_problem(n, gw, gh, wI, hI, seed=2)
    rng = np.random.default_rng(2)
    plane = rng.uniform(60, 180, gw * gh).astype(f32)
    plane[rng.integers(0, gw * gh, 5000)] = np.nan
    vig = (pr["true_vignette"] * rng.uniform(0.95, 1.05, wI * hI)).astype(f32)
    pr = dict(images=pr["images"], p2x=pr["p2x"], p2y=pr["p2y"], plane=plane, vig=vig, shape=(n, gw, gh, wI, hI))
    _, v_got, spec = check_steps(port, gpu, pr, 400, True)
    assert spec["bounds"][2] > 100 and np.isfinite(v_got).mean() > 0.5


def composed_loop(port, pr, iters, th, ia):
    """mdc_vignette_calib's loop from the oracle's plane step and the spec's vignette step."""
    n, gw, gh, wI, hI = pr["shape"]
    plane, vig, log = pr["plane"].copy(), pr["vig"].copy(), []
    for it in range(iters):
        oth2 = th * th if it >= iters // 2 else NO_OUTLIERS
        plane, _, _, ps = port.vc_plane_step(pr["images"], pr["p2x"], pr["p2y"], wI, hI, vig, plane, oth2, ia)
        r = fx.vignette_step(pr["images"], pr["p2x"], pr["p2y"], wI, hI, plane, vig, oth2, ia)
        vig = r["vignette"]
        log.append([ps[0], ps[1], r["E"], r["R"]])
    return plane, vig, np.array(log)


@pytest.mark.gpu
@pytest.mark.parametrize("int_abs", [True, False], ids=["int_abs", "fabs"])
@pytest.mark.parametrize("name", ["synthetic", "random_odd"])
def test_whole_loop_is_bit_identical_to_the_composed_steps(port, gpu, name, int_abs):
    torch, ctx = gpu
    pr = CPU_PROBLEMS[name]()
    n, gw, gh, wI, hI = pr["shape"]
    iters, th = 6, 15
    plane_e, vig_e, log_e = composed_loop(port, pr, iters, th, int_abs)
    d = [to_dev(torch, pr[k]) for k in ("images", "p2x", "p2y")]
    pc, v = torch.from_numpy(pr["plane"].copy()).cuda(), torch.from_numpy(pr["vig"].copy()).cuda()
    smoothed, log = ctx.vignette_calib(*d, gw, gh, wI, hI, iters, th, pc, v, int_abs)
    got_v = v.cpu().numpy()
    assert_bits_equal(pc.cpu().numpy(), plane_e, "plane colour")
    assert_bits_equal(got_v, vig_e, "vignette")
    assert np.array_equal(log[:, 1], log_e[:, 1]) and np.array_equal(log[:, 3], log_e[:, 3])
    assert np.all(np.abs(log[:, [0, 2]] - log_e[:, [0, 2]]) <= 1e-9 * np.abs(log_e[:, [0, 2]]))
    assert_bits_equal(smoothed.cpu().numpy(), port.vc_smooth(got_v, wI, hI, 4), "smoothed output")


def smooth_inputs():
    rng = np.random.default_rng(50)
    out = {}
    for wI, hI in ((1, 1), (1, 37), (37, 1), (5, 5), (1280, 1024)):
        v = rng.uniform(0.2, 1.0, wI * hI).astype(f32)
        v[rng.random(wI * hI) < 0.2] = np.nan
        if wI * hI > 100:
            v.reshape(hI, wI)[100:140, 200:300] = np.nan          # wider than 6 rounds can close
        out[f"{wI}x{hI}"] = (wI, hI, v)
        out[f"{wI}x{hI}_all_nan"] = (wI, hI, np.full(wI * hI, np.nan, f32))
    return out


@pytest.mark.gpu
def test_smoothing_is_bit_identical(port, gpu):
    torch, ctx = gpu
    for name, (wI, hI, v) in smooth_inputs().items():
        for iters in range(7):
            exp = port.vc_smooth(v, wI, hI, iters)
            got = ctx.vc_smooth(torch.from_numpy(v).cuda(), wI, hI, iters).cpu().numpy()
            assert_bits_equal(got, exp, f"smoothing {name} x{iters}")
