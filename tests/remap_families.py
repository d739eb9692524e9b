"""Remap tables the FOV model never produces, all inside the domain D of undistort_spec (test infrastructure).

Every K1 test before these fed the kernel tables from UndistorterFOV's constructor: smooth radial maps strictly inside
(0, W-1) x (0, H-1), or exactly -1.  The families here reach the parts of the tile plan (csrc/mdc_capi.cu, build_plan) and of the
arithmetic those tables never reach: integer and negative-fraction coordinates, -0.0, subnormal fractions, all-direct plans, boxes
at the staged-size and LDG-word limits, more than 64 TMA box classes at row granularity 8, and tile kinds interleaved in one CTA's
work.  Each family is seeded, so a run is reproducible.

`plan_model` restates the part of build_plan that does not depend on the shared-memory pitch search: per tile the input box, whether
it is staged, direct or empty, whether it has black pixels, and (with the pitch search off, i.e. box width = smallest width) the TMA
box classes at each row granularity."""
import numpy as np

F32 = np.float32
TILE = 32
MAX_STAGED_PX = 8192
MAX_BOX_WORDS = 8
THREADS = 256
MAX_CLASSES = 64


class Family:
    def __init__(self, name, in_w, in_h, out_w, out_h, rx, ry):
        self.name, self.in_w, self.in_h, self.out_w, self.out_h = name, in_w, in_h, out_w, out_h
        self.rx = np.ascontiguousarray(rx, F32).reshape(-1)
        self.ry = np.ascontiguousarray(ry, F32).reshape(-1)
        assert self.rx.size == out_w * out_h and self.ry.size == out_w * out_h


def _grid(out_w, out_h):
    v, u = np.mgrid[0:out_h, 0:out_w]
    return u.astype(np.float64), v.astype(np.float64)


def _black_outside(fam_name, W, H, OW, OH, x, y):
    """Entries outside D become the reference's (-1, -1)."""
    x = np.asarray(x, np.float64).astype(F32)
    y = np.asarray(y, np.float64).astype(F32)
    xd, yd = x.astype(np.float64), y.astype(np.float64)
    ok = (xd >= 0) & (xd < W - 1) & (yd > -1) & (yd < H - 1)
    return Family(fam_name, W, H, OW, OH, np.where(ok, x, F32(-1)), np.where(ok, y, F32(-1)))


def identity(W, H, offset):
    """out = in; the last column and row have no right / lower neighbour, so they are black."""
    u, v = _grid(W, H)
    return _black_outside(f"identity_{'int' if offset == 0 else 'half'}", W, H, W, H, u + offset, v + offset)


def flip(W, H):
    """Both axes mirrored, with a 0.25 / 0.75 fraction."""
    u, v = _grid(W, H)
    return _black_outside("flip_xy", W, H, W, H, (W - 2) - u + 0.25, (H - 2) - v + 0.75)


def transpose(W, H):
    """out = H x W: out (u, v) reads in (v + 0.5, u + 0.5)."""
    u, v = _grid(H, W)
    return _black_outside("transpose", W, H, H, W, v + 0.5, u + 0.5)


def rot90(W, H):
    """out = H x W, a quarter turn: the last output column reads y = -0.5, inside (-1, 0)."""
    u, v = _grid(H, W)
    return _black_outside("rot90", W, H, H, W, v + 0.125, (H - 1.5) - u)


def minify(W, H, k):
    """Minification by k: boxes of 32k input pixels a side."""
    OW, OH = int((W - 2) / k), int((H - 2) / k)
    u, v = _grid(OW, OH)
    return _black_outside(f"minify{k:g}", W, H, OW, OH, u * k + 0.3, v * k + 0.6)


def minify_ramp(W, H, OW, OH):
    """x = (W-1.01) t^1.6, t = u / OW: the zoom runs from strong magnification at the left/top edge to ~4.8x minification at the
    right/bottom edge, so the boxes straddle the 8192-pixel staged limit and the LDG word bound (bw 80-128 needs bh <= 64)."""
    u, v = _grid(OW, OH)
    return _black_outside(f"minify_ramp_{OW}x{OH}", W, H, OW, OH, (W - 1.01) * (u / OW) ** 1.6, (H - 1.01) * (v / OH) ** 1.6)


def to_size(W, H, OW, OH):
    """Whole frame into OW x OH (40 x 30 from 1280 x 1024: every tile direct)."""
    u, v = _grid(OW, OH)
    return _black_outside(f"to_{OW}x{OH}", W, H, OW, OH, u * ((W - 1.5) / OW) + 0.25, v * ((H - 1.5) / OH) + 0.25)


def magnify16(W, H):
    """16x magnification of a region whose right part runs past the frame: 2-pixel boxes, whose 16-aligned origin plus pitch runs
    past the right edge near it."""
    u, v = _grid(W, H)
    return _black_outside("magnify16", W, H, W, H, (W - 70.0) + u / 16.0 + 0.03, 3.0 + v / 16.0 + 0.01)


def scatter(W, H, OW, OH, seed, black_frac=0.0):
    """Uniformly random coordinates over D: every tile's box is about the whole frame, so every tile is direct.  With black_frac,
    that share of the entries is black with a mix of negative x (-1, -1e-45, -inf, -1e30) and y (-1, NaN, +-inf, anything)."""
    r = np.random.default_rng(seed)
    n = OW * OH
    x = r.uniform(0, W - 1, n).astype(F32)
    y = r.uniform(-1, H - 1, n).astype(F32)
    x = np.where(x.astype(np.float64) >= W - 1, F32(0), x)
    y = np.where(y.astype(np.float64) <= -1, F32(0), y)
    y = np.where(y.astype(np.float64) >= H - 1, F32(0), y)
    name = f"scatter_{OW}x{OH}"
    if black_frac:
        b = r.random(n) < black_frac
        bx = r.choice(np.array([-1.0, -1e-45, -np.inf, -1e30], F32), n)
        by = r.choice(np.array([-1.0, np.nan, np.inf, -np.inf, 5.0, -0.0], F32), n)
        x, y = np.where(b, bx, x), np.where(b, by, y)
        name = f"scatter_black_{OW}x{OH}"
    return Family(name, W, H, OW, OH, x, y)


def edges(W, H, seed):
    """out = in with every edge value at its natural place: column 0 maps to x = +0.0 / -0.0, the last column to
    x = nextafter(W-1, 0), row 0 to y in (-1, 0) or +-0.0, the last row to y = nextafter(H-1, 0); the interior has random fractions
    and some integer coordinates."""
    r = np.random.default_rng(seed)
    u, v = _grid(W, H)
    x = (u + r.random((H, W)) * 0.999).astype(F32)
    y = (v + r.random((H, W)) * 0.999).astype(F32)
    ints = r.random((H, W)) < 0.2
    x = np.where(ints, u.astype(F32), x)
    y = np.where(ints, v.astype(F32), y)
    x[:, 0] = np.where(r.random(H) < 0.5, F32(0.0), F32(-0.0))
    x[:, W - 1] = np.nextafter(F32(W - 1), F32(0))
    x[:, W - 2] = np.minimum(x[:, W - 2], np.nextafter(F32(W - 1), F32(0)))
    y[0, :] = np.where(r.random(W) < 0.3, np.where(r.random(W) < 0.5, F32(0.0), F32(-0.0)), -r.uniform(0, 1, W).astype(F32))
    y[0, :] = np.where(y[0, :] <= -1, F32(-0.5), y[0, :])
    y[H - 1, :] = np.nextafter(F32(H - 1), F32(0))
    y[H - 2, :] = np.minimum(y[H - 2, :], np.nextafter(F32(H - 1), F32(0)))
    return Family("edges", W, H, W, H, x, y)


def subnormal(W, H, seed):
    """Subnormal fractions: column 0 reads x in (0, 2^-126) or -0.0, row 0 reads y = +-subnormal, so fx / fy (and their products)
    are subnormal; the rest is the identity with a quarter-pixel offset."""
    r = np.random.default_rng(seed)
    u, v = _grid(W - 1, H - 1)
    x = (u + 0.25).astype(F32)
    y = (v + 0.25).astype(F32)
    tiny = lambda n: (r.integers(1, 1 << 23, n).astype(np.uint32)).view(F32)       # every positive subnormal
    x[:, 0] = np.where(r.random(H - 1) < 0.8, tiny(H - 1), F32(-0.0))
    y[0, :] = tiny(W - 1) * np.where(r.random(W - 1) < 0.5, F32(1), F32(-1))
    return Family("subnormal", W, H, W - 1, H - 1, x, y)


def many_classes(W, H, OW, OH, heights, widths, name):
    """Per tile a box of a chosen smallest width bw (a multiple of 16, 16-aligned origin) and height bh, cycling through all
    (bw, bh) pairs: with the pitch search off, the (bw, ceil(bh / g) g) classes decide the row granularity g."""
    tx, ty = -(-OW // TILE), -(-OH // TILE)
    pairs = [(bw, bh) for bw in widths for bh in heights]
    x = np.zeros((OH, OW), np.float64)
    y = np.zeros((OH, OW), np.float64)
    ox, oy = 0, 0
    for t in range(tx * ty):
        bw, bh = pairs[t % len(pairs)]
        wspan, hspan = bw - 2, bh - 2           # xi spans x0 .. x0 + bw - 2, so xhi - x0 + 1 = bw; yi spans bh - 1 rows
        if ox + bw + 16 > W:
            ox = 0
            oy += 37
        if oy + bh + 2 > H:
            oy = 0
        c0, r0 = (t % tx) * TILE, (t // tx) * TILE
        cu = np.arange(min(TILE, OW - c0))
        rv = np.arange(min(TILE, OH - r0))
        xs = ox + np.floor(cu * wspan / max(len(cu) - 1, 1)) + 0.25
        ys = oy + np.floor(rv * hspan / max(len(rv) - 1, 1)) + 0.5
        x[r0:r0 + len(rv), c0:c0 + len(cu)] = xs[None, :]
        y[r0:r0 + len(rv), c0:c0 + len(cu)] = ys[:, None]
        ox += 16 * (1 + (bw // 16) % 3)
    return _black_outside(name, W, H, OW, OH, x, y)


def checkerboard(W, H, seed):
    """out = in = W x H; tile (i, j) is, by (i + 2 j) % 4: staged (identity + fraction), direct (random coordinates from the whole
    frame), empty (all black) or staged with a black diagonal."""
    r = np.random.default_rng(seed)
    u, v = _grid(W, H)
    x = (u + 0.375).astype(F32)
    y = (v + 0.625).astype(F32)
    kind = ((u // TILE).astype(int) + 2 * (v // TILE).astype(int)) % 4
    rx_rand = r.uniform(0, W - 1.01, (H, W)).astype(F32)
    ry_rand = r.uniform(-0.99, H - 1.01, (H, W)).astype(F32)
    x = np.where(kind == 1, rx_rand, x)
    y = np.where(kind == 1, ry_rand, y)
    black = (kind == 2) | ((kind == 3) & ((u % TILE) == (v % TILE)))
    x = np.where(black, F32(-1), x)
    y = np.where(black, F32(-1), y)
    fam = _black_outside("checkerboard", W, H, W, H, x, y)
    return fam


def pinhole_radtan(W, H, OW, OH):
    """A non-FOV camera an adopter could upload: pinhole output, strong radial-tangential input distortion, computed in float64,
    rounded to float32 and sanitised by the reference's rule (FOVUndistorter.cpp:237-247)."""
    u, v = _grid(OW, OH)
    fx, fy, cx, cy = 0.45 * OW, 0.6 * OH, 0.5 * OW - 0.5, 0.5 * OH - 0.5
    k1, k2, p1, p2 = -0.42, 0.19, 0.012, -0.008
    xn, yn = (u - cx) / fx, (v - cy) / fy
    r2 = xn * xn + yn * yn
    rad = 1 + k1 * r2 + k2 * r2 * r2
    xd = xn * rad + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn)
    yd = yn * rad + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn
    x = (xd * 0.5 * W + (0.5 * W - 0.5)).astype(F32)
    y = (yd * 0.6 * H + (0.5 * H - 0.5)).astype(F32)
    x = np.where(x == 0, F32(0.01), x)
    y = np.where(y == 0, F32(0.01), y)
    x = np.where(x == W - 1, F32(W - 1.01), x)
    y = np.where(y == H - 1, F32(H - 1.01), y)
    ok = (x > 0) & (y > 0) & (x < W - 1) & (y < H - 1)
    return Family("pinhole_radtan", W, H, OW, OH, np.where(ok, x, F32(-1)), np.where(ok, y, F32(-1)))


def tiny(W, H, OW, OH, seed):
    """Random entries of D (black ones included) for the smallest geometries: 2x2 -> 1x1, 3x2 -> 33x1 and 1x33."""
    r = np.random.default_rng(seed)
    n = OW * OH
    x = r.choice(np.array([0.0, -0.0, 0.5, np.nextafter(F32(W - 1), F32(0)), -1.0, 1e-40], F32), n)
    x = np.where(x.astype(np.float64) >= W - 1, np.nextafter(F32(W - 1), F32(0)), x)
    y = r.choice(np.array([0.0, -0.0, -0.5, np.nextafter(F32(H - 1), F32(0)), 0.25, -1e-45], F32), n)
    return Family(f"tiny_{W}x{H}_to_{OW}x{OH}", W, H, OW, OH, x, y)


MANY_CLASSES_G16 = dict(widths=(16, 32, 48), heights=tuple(8 * k - 3 for k in range(1, 33)))     # 80 classes at g = 8, 40 at 16
MANY_CLASSES_G32 = dict(widths=tuple(range(16, 257, 16)), heights=tuple(8 * k - 3 for k in range(1, 33)))   # 160 at 8, 80 at 16


def registry():
    """name -> (factory, large).  `large`: 1280 x 1024 or more, run with fewer flag combinations on the GPU."""
    R = {}

    def add(name, large, fn):
        R[name] = (fn, large)
    for W, H in ((1280, 1024), (333, 217)):
        big = W > 1000
        add(f"identity_int_{W}x{H}", big, lambda W=W, H=H: identity(W, H, 0))
        add(f"flip_xy_{W}x{H}", big, lambda W=W, H=H: flip(W, H))
        add(f"transpose_{W}x{H}", big, lambda W=W, H=H: transpose(W, H))
        add(f"magnify16_{W}x{H}", big, lambda W=W, H=H: magnify16(W, H))
        add(f"scatter_{W}x{H}", big, lambda W=W, H=H: scatter(W, H, min(W, 640), min(H, 480), 11))
        add(f"scatter_black_{W}x{H}", big, lambda W=W, H=H: scatter(W, H, min(W, 640), min(H, 480), 12, black_frac=0.3))
        add(f"edges_{W}x{H}", big, lambda W=W, H=H: edges(W, H, 13))
        add(f"subnormal_{W}x{H}", big, lambda W=W, H=H: subnormal(W, H, 14))
    for W, H in ((1920, 1080), (333, 217)):
        big = W > 1000
        add(f"identity_half_{W}x{H}", big, lambda W=W, H=H: identity(W, H, 0.5))
        add(f"rot90_{W}x{H}", big, lambda W=W, H=H: rot90(W, H))
    add("minify3_1280x1024", True, lambda: minify(1280, 1024, 3))
    add("minify4_1920x1080", True, lambda: minify(1920, 1080, 4))
    add("minify3.5_333x217", False, lambda: minify(333, 217, 3.5))
    add("minify8_1280x1024", True, lambda: minify(1280, 1024, 8))
    add("minify_ramp_1920x1080", True, lambda: minify_ramp(1920, 1080, 640, 360))
    add("minify_ramp_333x217", False, lambda: minify_ramp(333, 217, 200, 150))
    add("to_40x30_1280x1024", False, lambda: to_size(1280, 1024, 40, 30))
    add("many_classes_g16_1920x1080", True, lambda: many_classes(1920, 1080, 640, 480, name="many_classes_g16", **MANY_CLASSES_G16))
    add("many_classes_g32_1920x1080", True, lambda: many_classes(1920, 1080, 1280, 1024, name="many_classes_g32", **MANY_CLASSES_G32))
    add("checkerboard_1280x1024", True, lambda: checkerboard(1280, 1024, 15))
    add("pinhole_radtan_1280x1024", True, lambda: pinhole_radtan(1280, 1024, 1280, 1024))
    add("pinhole_radtan_333x217", False, lambda: pinhole_radtan(333, 217, 301, 199))
    add("tiny_2x2_to_1x1", False, lambda: tiny(2, 2, 1, 1, 16))
    add("tiny_3x2_to_33x1", False, lambda: tiny(3, 2, 33, 1, 17))
    add("tiny_3x2_to_1x33", False, lambda: tiny(3, 2, 1, 33, 18))
    return R


REGISTRY = registry()
_cache = {}


def get(name):
    if name not in _cache:
        _cache[name] = REGISTRY[name][0]()
    return _cache[name]


# ------------------------------------------------------------------------------------------------------------------ inputs
def special_floats(n, seed):
    """float32 image with NaN, +-inf, -0.0, subnormals and values near FLT_MAX among ordinary ones."""
    r = np.random.default_rng(seed)
    img = r.uniform(-300, 300, n).astype(F32)
    pool = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1e-45, -1e-45, 1e-40, 1.1754942e-38, 3.4028235e38, -3.4028235e38,
                     3.0e38, 1.7e38], F32)
    pick = r.random(n) < 0.3
    return np.where(pick, r.choice(pool, n), img)


def frame_u8(n, seed):
    r = np.random.default_rng(seed)
    img = r.integers(0, 256, n).astype(np.uint8)
    img[r.random(n) < 0.1] = 255
    img[r.random(n) < 0.1] = 0
    return img


def arbitrary_photometric(n, seed):
    """GInv with NaN, +-inf, -0.0, subnormals and huge values; an inverse vignette with the same kinds of entries."""
    r = np.random.default_rng(seed)
    ginv = np.linspace(0, 255, 256).astype(F32)
    ginv[r.integers(0, 256, 40)] = r.choice(np.array([np.nan, np.inf, -np.inf, -0.0, 1e-20, 1e-44, 3e38], F32), 40)
    vinv = r.uniform(0.5, 3, n).astype(F32)
    m = r.random(n) < 0.2
    vinv[m] = r.choice(np.array([np.nan, np.inf, -np.inf, -0.0, 1e-20, 1e-30, 2e38], F32), int(m.sum()))
    return ginv, vinv


# ------------------------------------------------------------------------------------------------------------------ plan model
def plan_model(fam, gran):
    """build_plan's per-tile decisions at row granularity `gran`: dict with counts of staged / direct / empty tiles, tiles with black
    pixels, and the set of (smallest box width, box height rounded to gran) of the staged tiles."""
    OW, OH = fam.out_w, fam.out_h
    rx = fam.rx.reshape(OH, OW)
    ry = fam.ry.reshape(OH, OW)
    out = {"staged": 0, "direct": 0, "empty": 0, "black": 0, "classes": set()}
    for ty0 in range(0, OH, TILE):
        for tx0 in range(0, OW, TILE):
            x = rx[ty0:ty0 + TILE, tx0:tx0 + TILE].reshape(-1)
            y = ry[ty0:ty0 + TILE, tx0:tx0 + TILE].reshape(-1)
            black = x < 0
            out["black"] += bool(black.any())
            if black.all():
                out["empty"] += 1
                continue
            xi = np.trunc(x[~black]).astype(np.int64)
            yi = np.trunc(y[~black]).astype(np.int64)
            xlo, xhi, ylo, yhi = xi.min(), xi.max() + 1, yi.min(), yi.max() + 1
            x0 = xlo & ~15
            bh = yhi - ylo + 1
            bh8 = -(-bh // gran) * gran
            bw = ((xhi - x0 + 1) + 15) & ~15
            lg = 2
            while (4 << lg) < bw:
                lg += 1
            rstep = max(1, THREADS >> lg)
            if bw <= 256 and bh8 <= 256 and bw * bh8 <= MAX_STAGED_PX and -(-bh // rstep) <= MAX_BOX_WORDS:
                out["staged"] += 1
                out["classes"].add((int(bw), int(bh8)))
            else:
                out["direct"] += 1
    return out


def granularity_without_pitch_search(fam):
    """The row granularity build_plan settles on when every box is as narrow as it can be (MDC_PITCH_SEARCH=0)."""
    g = 8
    while g < 256 and len(plan_model(fam, g)["classes"]) > MAX_CLASSES:
        g *= 2
    return g
