"""The decode-ahead sequence feed (mdc_seq_prepare, csrc/mdc_sequence.cpp) frame for frame on JPEG sequences.

A feed like this one goes wrong as the right arithmetic on the wrong frame: a staging buffer refilled before it is consumed, a
pipe buffer reused before its device-to-host copy has finished, an offset wrong by one chunk, a call that returns before pinned
output has landed.  So every sequence here cycles P distinct payloads over its entries, P prime and dividing neither any chunk
size the module uses nor twice one: a frame taken from the wrong slot, the wrong chunk or a stale buffer never equals the
expectation of its own index.  Every output frame of every call is compared bit for bit, at every level, with the plain-C oracle
(oracle/port, pinned to the reference by the CPU suite) applied to payload (first + k) mod P, decoded by cv2.imdecode.  Every
level buffer has a guard row before and after the frames a call may write; all rows start as a sentinel bit pattern.

CPU part: the library's decoder against cv2.imdecode at full size, the expectation helper, and the argument checks that can run
without a context (the range and level-count checks; the NULL-level check needs the context's geometry).
GPU part: chunk boundaries, flags and levels, loaders, host-pipeline chunking, state kept across calls, the benchmark's call
pattern, errors in the middle of a call, arguments.
"""
import ctypes as C
import os
import threading
import zipfile

import numpy as np
import pytest

from mono_dataset_code_b200 import _lib, api, synthetic as S

cv2 = pytest.importorskip("cv2")
lib = _lib.lib

RECT, GAMMA, VIG, NAN = 1, 2, 4, 8
ALL = RECT | GAMMA | VIG | NAN
BENCH_FLAGS = RECT | GAMMA | VIG           # bench.py's FLAGS_ALL
MAX_LEVELS = 8                             # MDC_MAX_PYR_LEVELS
INT_MAX = 2 ** 31 - 1
OK, INVALID_ARG, FORMAT, UNSUPPORTED = 0, 1, 3, 6
SENTINEL = np.uint32(0xDEADBEEF)           # -6.3e18 as a float: no getImage output

# name -> in_w, in_h, out_w, out_h (camera.txt "crop"), entries of the main sequences, P.
# A chunk is even, so an odd prime P divides a chunk C (or 2C) only if C is a multiple of 2P (of P): P = 131 > 128 divides no
# chunk 16..256 and no twice one, whatever the default thread count of the host.  At 1920x1080 the payloads cost 8 MB each, so
# P = 37 there, which divides none of the chunks the c4 tests use (16, 34 and those of at most 24 threads: up to 48).
C4_MAX_SWEEP_THREADS = 24                       # keeps the c4 calls' pinned output under 1.3 GB on hosts with more CPUs
C4_ENTRIES = 3 * min(256, 2 * C4_MAX_SWEEP_THREADS) + 1 + 15      # the longest benchmark-pattern call, and room to wrap
GEOMS = {
    "c4": (1920, 1080, 1920, 1080, C4_ENTRIES, 37),      # the benchmark's sequence geometry
    "odd": (1241, 376, 621, 189, 800, 131),     # width not a multiple of 16: the feed pads rows to 1248 in its H2D copy
    "tiny": (33, 17, 33, 17, 800, 131),         # partial JPEG MCUs; levels 5 and up have no pixels
}
SMALL_N = 60                                    # entries of the colour and mixed sequences (fewer than P)
KINDS = ("grey", "colour", "mixed")             # baseline grey JPEG / colour 4:2:0 JPEG read as grey / JPEG + 16-bit PNG + PGM


# ------------------------------------------------------------------ the feed's documented chunk rule
def default_decode_threads():
    """mdc_seq_prepare's threads = 0: the CPUs the process may run on, capped by the cgroup v2 CPU quota."""
    n = max(1, min(os.cpu_count() or 1, len(os.sched_getaffinity(0))))
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:
            q, per = f.read().split()[:2]
        if q != "max" and int(q) > 0 and int(per) > 0:
            n = max(1, min(n, int(q) // int(per)))
    except (OSError, ValueError):
        pass
    return n


def chunk_of(threads):
    """Frames per chunk: two per decode thread, 16..256 (include/mdc_b200.h)."""
    t = threads if threads >= 1 else default_decode_threads()
    return min(256, max(16, 2 * t))


def bench_threads():
    """bench.py's decode thread count on one GPU: the CPUs of the affinity mask, capped by the CPU quota."""
    n = len(os.sched_getaffinity(0))
    try:
        with open("/sys/fs/cgroup/cpu.max") as f:
            q, per = f.read().split()[:2]
        if q != "max":
            n = max(1, min(n, int(float(q) / float(per))))
    except (OSError, ValueError):
        pass
    return n


# ------------------------------------------------------------------ payloads and sequences
def scene(p, w, h):
    """bench.py's textured scene for payload p, plus a fully saturated block (MCU-aligned, so it stays 255 through JPEG) that
    moves with p and a black block in the bottom-right corner."""
    rng = np.random.default_rng(7919 * p + w)
    yy, xx = np.mgrid[0:h, 0:w]
    img = (xx * (150.0 / w) + yy * (60.0 / h) + 40 * np.sin((xx + 13 * p) * 0.05) * np.cos((yy - 7 * p) * 0.04)
           + ((xx // 64 + yy // 64 + p) % 2) * 30 + rng.normal(0, 1.5, (h, w)))
    img = np.clip(np.rint(img), 0, 255).astype(np.uint8)
    b = 32 if w >= 128 else 16
    nx, ny = max(1, (w // 2 - b) // 16 + 1), max(1, (h - b) // 16 + 1)
    x0, y0 = 16 * ((5 * p) % nx), 16 * ((3 * p) % ny)
    img[y0:y0 + b, x0:x0 + b] = 255
    img[h - min(h, b):, w - min(w, b) // 2 - 1:] = 0
    return img


def payload(kind, p, w, h, scratch):
    """(file extension, bytes) of payload p."""
    img = scene(p, w, h)
    if kind == "grey" or (kind == "mixed" and p % 3 == 0):
        ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])
        assert ok
        return ".jpg", enc.tobytes()
    if kind == "colour":
        bgr = np.stack([img, np.roll(img, 5, axis=1), 255 - img], axis=-1)
        bgr[img == 255] = 255
        bgr[img == 0] = 0
        ok, enc = cv2.imencode(".jpg", bgr, [cv2.IMWRITE_JPEG_QUALITY, 90,
                                             cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
        assert ok
        return ".jpg", enc.tobytes()
    if p % 3 == 1:                         # 16-bit PNG: the frame is the high byte
        low = np.random.default_rng(p).integers(0, 256, img.shape, dtype=np.uint16)
        path = os.path.join(scratch, "p.png")
        S.write_png_gray(path, (img.astype(np.uint16) << 8) | low)
        with open(path, "rb") as f:
            return ".png", f.read()
    return ".pgm", b"P5\n%d %d\n255\n" % (w, h) + img.tobytes()


def decode_like_opencv(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_GRAYSCALE)


def write_times(folder, n):
    with open(os.path.join(folder, "times.txt"), "w") as t:
        for i in range(n):
            t.write(f"{i} {i * 0.05:.3f} 1.0\n")


def write_sequence(folder, entries, fmt):
    """entries: [(name, bytes)] in name order.  fmt: 'stored' / 'deflated' zip (written out of name order) or 'folder'."""
    os.makedirs(folder, exist_ok=True)
    if fmt == "folder":
        os.makedirs(os.path.join(folder, "images"))
        for name, blob in entries:
            with open(os.path.join(folder, "images", name), "wb") as f:
                f.write(blob)
    else:
        order = list(reversed(range(len(entries)))) if fmt == "stored" else list(np.random.default_rng(5).permutation(len(entries)))
        method = zipfile.ZIP_STORED if fmt == "stored" else zipfile.ZIP_DEFLATED
        with zipfile.ZipFile(os.path.join(folder, "images.zip"), "w", method, compresslevel=None if fmt == "stored" else 1) as z:
            for i in order:
                z.writestr(entries[i][0], entries[i][1])
    write_times(folder, len(entries))


class World:
    """One geometry: calibration files, payloads, sequences, contexts and the oracle's tables."""

    def __init__(self, root, geom):
        self.root, self.geom = str(root), geom
        self.iw, self.ih, self.ow, self.oh, self.n, self.P = GEOMS[geom]
        self.files = S.write_dataset_dir(os.path.join(self.root, "calib"), self.iw, self.ih, self.ow, self.oh, "crop")
        self._payloads, self._raws, self._seqs, self._ctx, self._tables = {}, {}, {}, None, None

    def payload(self, kind, p):
        """(extension, bytes) of payload p, made on first use."""
        key = (kind, p)
        if key not in self._payloads:
            self._payloads[key] = payload(kind, p, self.iw, self.ih, self.root)
        return self._payloads[key]

    def raw(self, kind, p):
        """What cv::imread(..., IMREAD_GRAYSCALE) makes of payload p."""
        key = (kind, p)
        if key not in self._raws:
            self._raws[key] = decode_like_opencv(self.payload(kind, p)[1])
        return self._raws[key]

    def variant(self, kind, base, replaced):
        """A payload kind that is `base` except for the raw frames in replaced {p: raw} (expectations follow the kind)."""
        for p in range(self.P):
            self._raws[(kind, p)] = replaced[p] if p in replaced else self.raw(base, p)
        for key in [k for k in _EXPECT if k[0] == self.geom and k[1] == kind]:
            del _EXPECT[key]

    def entries(self, kind, n):
        return [(f"{i:05d}{self.payload(kind, i % self.P)[0]}", self.payload(kind, i % self.P)[1]) for i in range(n)]

    def seq_dir(self, kind, fmt):
        key = (kind, fmt)
        if key not in self._seqs:
            folder = os.path.join(self.root, f"{kind}_{fmt}")
            write_sequence(folder, self.entries(kind, self.n if kind == "grey" else SMALL_N), fmt)
            self._seqs[key] = folder
        return self._seqs[key]

    def seq(self, kind="grey", fmt="stored"):
        s = api.Sequence(self.seq_dir(kind, fmt))
        assert s.status == 0 and s.getNumImages() == (self.n if kind == "grey" else SMALL_N)
        return s

    def new_ctx(self):
        fov = api.UndistorterFOV(self.files["camera"])
        photo = api.PhotometricUndistorter(self.files["pcalib"], self.files["vignette"], self.iw, self.ih)
        ctx = api.Context(fov, photo)
        ctx._models = (fov, photo)
        return ctx

    @property
    def ctx(self):
        if self._ctx is None:
            self._ctx = self.new_ctx()
        return self._ctx

    def shapes(self, flags, levels):
        w, h = (self.ow, self.oh) if flags & RECT else (self.iw, self.ih)
        return [(w >> l, h >> l) for l in range(levels)]

    def tables(self):
        if self._tables is None:
            from oracle.loader import PortOracle
            port = PortOracle()
            rx, ry = port.fov_from_file(self.files["camera"]).tables()
            ginv, _ = port.photo_tables(np.loadtxt(self.files["pcalib"], dtype=np.float32))
            _, vinv = port.vignette_maps(self.files["vignette_pixels"])
            self._tables = (port, rx, ry, ginv, vinv.reshape(-1))
        return self._tables


_EXPECT = {}


def expected(world, kind, flags, p, levels):
    """[(bits with NaN made canonical, has NaN)] per level: getImage + pyramid of payload p from the plain-C oracle."""
    key = (world.geom, kind, flags, p)
    have = _EXPECT.get(key)
    if have is None or len(have) < levels:
        port, rx, ry, ginv, vinv = world.tables()
        lvl0 = port.get_image(rx, ry, world.iw, world.ih, ginv, vinv, world.raw(kind, p),
                              int(bool(flags & RECT)), int(bool(flags & GAMMA)), int(bool(flags & VIG)), int(bool(flags & NAN)))
        (w, h), = world.shapes(flags, 1)
        have = []
        for a in port.pyramid(lvl0, w, h, max(levels, 1)):
            have.append((a.view(np.uint32), bool(np.isnan(a).any())))
        _EXPECT[key] = have
    return have[:levels]


def same_bits(row, exp):
    """Equal bits, except that a NaN may carry another payload than the oracle's NaN (in the same place)."""
    bits, has_nan = exp
    differ = row != bits
    if not differ.any():
        return True
    if not has_nan:
        return False
    at = np.flatnonzero(differ)
    return bool(np.isnan(row[at].view(np.float32)).all() and np.isnan(bits[at].view(np.float32)).all())


@pytest.fixture(autouse=True)
def _bounded_expectations():
    """Expectations are kept for the next tests (most use the same flags) while they hold less than 250 MB."""
    yield
    if sum(bits.nbytes for levels in _EXPECT.values() for bits, _ in levels) > 250 << 20:
        _EXPECT.clear()


@pytest.fixture(scope="module")
def world(tmp_path_factory):
    made = {}

    def get(geom):
        if geom not in made:
            made[geom] = World(tmp_path_factory.mktemp(geom), geom)
        return made[geom]
    yield get
    for w in made.values():
        if w._ctx is not None:
            w._ctx.close()


# ------------------------------------------------------------------ output buffers with guard rows
class Out:
    """Host level buffers for `count` frames, each with one guard row before and after, every row set to SENTINEL.  pool: a
    uint32 view of pinned memory to carve the levels from (None: pageable numpy arrays).  Levels without pixels get NULL."""

    def __init__(self, shapes, count, pool=None):
        self.count, self.rows, off = count, [], 0
        for (w, h) in shapes:
            n = w * h
            if n == 0:
                self.rows.append(None)
                continue
            m = (count + 2) * n
            if pool is None:
                a = np.empty(m, np.uint32)
            else:
                assert off + m <= pool.size, "pinned pool too small"
                a, off = pool[off:off + m], off + m
            a[:] = SENTINEL
            self.rows.append(a.reshape(count + 2, n))

    def ptrs(self, null_level=None, extra=0):
        p = [None if (a is None or l == null_level) else a[1:].ctypes.data for l, a in enumerate(self.rows)]
        return (C.c_void_p * (len(p) + extra))(*p)

    def untouched(self):
        return all(a is None or (a == SENTINEL).all() for a in self.rows)


@pytest.fixture()
def pinned():
    """pinned(nbytes) -> uint32 view of mdc_host_alloc memory, freed after the test."""
    blocks = []

    def alloc(nbytes):
        h = C.c_void_p()
        _lib.check(lib.mdc_host_alloc(C.byref(h), nbytes), "mdc_host_alloc")
        blocks.append(h.value)
        return np.ctypeslib.as_array((C.c_uint32 * (nbytes // 4)).from_address(h.value))
    yield alloc
    if blocks:
        import torch
        torch.cuda.synchronize()            # no copy of a call that returned too early may land in freed memory
    for b in blocks:
        lib.mdc_host_free(b)


def pool_bytes(world, flags, levels, count):
    return sum(w * h for w, h in world.shapes(flags, levels)) * (count + 2) * 4


def check_out(world, out, kind, flags, first, written, what):
    """Rows 1..written hold frames first .. first+written-1 bit for bit; the guard rows and the rows after `written` are untouched."""
    # the rows that land last are read first: a call that returned before its copies finished shows here
    tail = [a[written].copy() if (a is not None and written) else None for a in out.rows]
    levels = len(out.rows)
    for l, a in enumerate(out.rows):
        if a is None:
            continue
        assert (a[0] == SENTINEL).all(), f"{what}: level {l}: the guard row before the frames was written"
        assert (a[out.count + 1] == SENTINEL).all(), f"{what}: level {l}: the guard row after the frames was written"
        if written < out.count:
            assert (a[written + 1:out.count + 1] == SENTINEL).all(), f"{what}: level {l}: rows after frame {written - 1} were written"
    for k in range(written):
        exp = expected(world, kind, flags, (first + k) % world.P, levels)
        for l, a in enumerate(out.rows):
            if a is None:
                continue
            row = tail[l] if k == written - 1 else a[1 + k]
            if same_bits(row, exp[l]):
                continue
            if (row == SENTINEL).all():
                raise AssertionError(f"{what}: frame {k} (entry {first + k}) level {l} was not written")
            match = [q for q in range(world.P) if same_bits(row, expected(world, kind, flags, q, levels)[l])]
            raise AssertionError(f"{what}: frame {k} (entry {first + k}, payload {(first + k) % world.P}) level {l} differs from the "
                                 f"oracle; it holds payload {match if match else 'none'}: "
                                 f"{np.count_nonzero(row != exp[l][0])} of {row.size} words differ")


def seq_call(world, ctx, seq, first, count, flags, levels, threads, pool=None, kind="grey", what=""):
    out = Out(world.shapes(flags, levels), count, pool)
    rc = lib.mdc_seq_prepare(ctx._h, seq._h, first, count, flags, out.ptrs(), levels, threads)
    assert rc == OK, f"{what}: mdc_seq_prepare -> {rc}: {lib.mdc_last_error().decode()}"
    check_out(world, out, kind, flags, first, count, what or f"first {first} count {count} flags {flags} levels {levels} threads {threads}")


def capped_bench_sweep():
    cap = min(bench_threads(), C4_MAX_SWEEP_THREADS)
    return sorted({max(1, cap // 4), max(1, cap // 2), cap})


# ================================================================== CPU part
@pytest.mark.parametrize("geom,kind", [("c4", "grey"), ("c4", "colour"), ("odd", "grey"), ("odd", "colour"), ("odd", "mixed"),
                                       ("tiny", "grey"), ("tiny", "colour"), ("tiny", "mixed")])
def test_payloads_decode_like_opencv(world, geom, kind, tmp_path):
    """Every payload, from a zip and from a folder, decodes to cv2.imdecode(..., IMREAD_GRAYSCALE) at full size."""
    w = world(geom)
    entries = w.entries(kind, w.P)
    for fmt in ("stored", "folder"):
        folder = str(tmp_path / fmt)
        write_sequence(folder, entries, fmt)
        seq = api.Sequence(folder)
        assert seq.getNumImages() == w.P
        for p in range(w.P):
            got, exp = seq.getImageRaw_internal(p), w.raw(kind, p)
            assert exp.shape == (w.ih, w.iw)
            assert got is not None, f"{fmt} payload {p} ({entries[p][0]}): {lib.mdc_last_error().decode()}"
            assert np.array_equal(got, exp), f"{fmt} payload {p} ({entries[p][0]}): {np.count_nonzero(got != exp)} pixels differ"
        seq.close()


def test_payload_count_divides_no_chunk():
    """A frame one or two chunks off holds another payload, on any host: odd and tiny for every chunk the feed can choose, c4 for
    the chunks of the c4 tests (3 and 17 threads, and the benchmark's sweep up to C4_MAX_SWEEP_THREADS)."""
    for geom in ("odd", "tiny"):
        P = GEOMS[geom][5]
        assert all(c % P and (2 * c) % P for c in range(16, 257, 2)), geom
    P = GEOMS["c4"][5]
    c4_chunks = {chunk_of(3), chunk_of(17)} | {chunk_of(t) for t in range(1, C4_MAX_SWEEP_THREADS + 1)}
    assert all(c % P and (2 * c) % P for c in c4_chunks)
    assert {chunk_of(t) for t in capped_bench_sweep()} <= c4_chunks
    assert 3 * max(c4_chunks) + 1 + 12 <= GEOMS["c4"][4]          # the benchmark-pattern test's longest call and its wrap


@pytest.mark.parametrize("geom", ["odd", "tiny"])
def test_expectations_tell_every_payload_apart(world, geom):
    """The helper the GPU part compares with: level shapes as the library lays them out, every payload's frame distinct from
    every other's (so a frame from a wrong slot cannot pass), saturated pixels NaN under nanOverexposed, black pixels present."""
    w = world(geom)
    for kind in KINDS:
        raws = [w.raw(kind, p) for p in range(w.P)]
        assert all((r == 255).any() and (r == 0).any() for r in raws), kind
        for flags in (ALL, GAMMA | VIG | NAN, GAMMA | VIG):
            exp = [expected(w, kind, flags, p, MAX_LEVELS) for p in range(w.P)]
            shapes = w.shapes(flags, MAX_LEVELS)
            for l, (lw, lh) in enumerate(shapes):
                assert all(e[l][0].shape == (lw * lh,) for e in exp), (kind, flags, l)
            assert len({e[0][0].tobytes() for e in exp}) == w.P, (kind, flags)
            nan_frames = sum(e[0][1] for e in exp)      # rectified: the crop may leave a payload's saturated block outside
            assert (nan_frames >= w.P // 2 if flags & RECT else nan_frames == w.P) if flags & NAN else nan_frames == 0, (kind, flags, nan_frames)
    if geom == "tiny":
        assert [wh for wh in w.shapes(ALL, MAX_LEVELS)][5:] == [(1, 0), (0, 0), (0, 0)]


def test_argument_checks_without_a_context(world):
    """mdc_seq_prepare checks the range and the level count before it looks at the context, so these run without a GPU; the
    NULL-level check needs the context's geometry and is in the GPU part.  Nothing is written."""
    w = world("tiny")
    seq = w.seq()
    n = seq.getNumImages()
    out = Out(w.shapes(ALL, 2), 4)
    for first, count, levels, msg in ((-1, 4, 2, b"outside"), (0, -1, 2, b"outside"), (n - 3, 4, 2, b"outside"),
                                      (1, INT_MAX, 2, b"outside"), (INT_MAX, 1, 2, b"outside"), (0, 4, 0, b"pyramid levels"),
                                      (0, 4, 9, b"pyramid levels")):
        rc = lib.mdc_seq_prepare(None, seq._h, first, count, ALL, out.ptrs(extra=8), levels, 4)
        assert rc == INVALID_ARG and msg in lib.mdc_last_error(), (first, count, levels, rc, lib.mdc_last_error())
    assert lib.mdc_seq_prepare(None, seq._h, 0, 4, ALL, out.ptrs(), 2, 4) == INVALID_ARG          # no context
    assert lib.mdc_seq_prepare(None, None, 0, 4, ALL, out.ptrs(), 2, 4) == INVALID_ARG            # no sequence
    assert lib.mdc_seq_prepare(None, seq._h, 0, 4, ALL, None, 2, 4) == INVALID_ARG                # no level array
    assert out.untouched()
    seq.close()


def test_broken_entries_on_the_host(world, tmp_path):
    """The bad frames of the GPU error cases fail on the host already: a file cut inside its table segments, a progressive file,
    a file of the wrong size.  A file cut inside its entropy-coded scan is not an error: like libjpeg, the decoder reads the
    missing scan data as zero bits, so it must decode to what OpenCV makes of the file with its missing bytes given as zeros."""
    w = world("odd")
    bad = bad_payloads(w)
    write_sequence(str(tmp_path), [(f"{i:05d}.jpg", b) for i, b in enumerate(bad.values())], "folder")
    seq = api.Sequence(str(tmp_path))
    assert seq.getImageRaw_internal(0) is None and b"truncated" in lib.mdc_last_error()
    assert seq.getImageRaw_internal(1) is None and b"baseline only" in lib.mdc_last_error()
    assert seq.getImageRaw_internal(2).shape == (w.ih, w.iw - 1)
    seq.close()
    for geom in ("odd", "tiny"):
        g = world(geom)
        blob, raw = scan_cut(g)
        folder = str(tmp_path / geom)
        write_sequence(folder, [("00000.jpg", blob)], "folder")
        seq = api.Sequence(folder)
        got = seq.getImageRaw_internal(0)
        assert got is not None and np.array_equal(got, raw), geom
        assert not np.array_equal(raw, g.raw("grey", 3)), geom           # the cut removed real image data
        seq.close()


def bad_payloads(w):
    """Frames that stop a call: cut inside the table segments (before the scan), progressive, one column short."""
    img = scene(3, w.iw, w.ih)
    good = w.payload("grey", 3)[1]
    sos = good.find(b"\xff\xda")
    ok, prog = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_PROGRESSIVE, 1])
    ok2, small = cv2.imencode(".jpg", img[:, :-1], [cv2.IMWRITE_JPEG_QUALITY, 90])
    assert ok and ok2 and sos > 0
    return {"cut_in_headers": good[:sos - 40], "progressive": prog.tobytes(), "wrong_size": small.tobytes()}


def scan_cut(w):
    """Payload 3 cut halfway through its entropy-coded scan, and the frame libjpeg makes of it: the same bytes followed by zero
    bytes in place of the missing scan data (zero bits, as libjpeg substitutes at a premature end of data) and an EOI marker."""
    good = w.payload("grey", 3)[1]
    sos = good.find(b"\xff\xda")
    cut = good[:(sos + len(good)) // 2]
    raw = decode_like_opencv(cut + bytes(w.iw * w.ih) + b"\xff\xd9")
    assert raw is not None and raw.shape == (w.ih, w.iw)
    return cut, raw


# ================================================================== GPU part
THREADS = [1, 3, 8, 17, 64, 128, 0]
FMT_OF_THREADS = {1: "stored", 3: "deflated", 8: "folder", 17: "stored", 64: "deflated", 128: "folder", 0: "stored"}


@pytest.mark.gpu
@pytest.mark.parametrize("threads", THREADS)
@pytest.mark.parametrize("geom", ["odd", "tiny"])
def test_chunk_boundaries(world, pinned, geom, threads):
    """Counts C-1, C, C+1, 2C+1, 3C+1 and 1 at first offsets 0, 1 and ending at the last entry; levels 1 (pageable output) and 5
    (pinned output); rectify + gamma + vignette + NaN."""
    w = world(geom)
    c = chunk_of(threads)
    seq = w.seq("grey", FMT_OF_THREADS[threads])
    counts = sorted({c - 1, c, c + 1, 2 * c + 1, 3 * c + 1, 1})
    pool = pinned(pool_bytes(w, ALL, 5, max(counts)))
    for levels in (1, 5):
        for count in counts:
            for first in (0, 1, w.n - count):
                seq_call(w, w.ctx, seq, first, count, ALL, levels, threads, pool if levels == 5 else None,
                         what=f"{geom} {FMT_OF_THREADS[threads]} threads {threads} (chunk {c}) first {first} count {count} levels {levels}")
    seq.close()


@pytest.mark.gpu
def test_chunk_boundaries_c4(world, pinned):
    """The reduced set at the benchmark's size: counts C-1, C+1 and 2C+1, starting at entry 1 or ending at the last entry."""
    w = world("c4")
    seq = w.seq("grey", "stored")
    pool = pinned(pool_bytes(w, ALL, 5, 2 * 16 + 1))
    for threads, levels in ((3, 5), (17, 1)):
        c = chunk_of(threads)
        for i, count in enumerate((c - 1, c + 1, 2 * c + 1)):
            for first in ((1, w.n - count) if i == 2 else (1,) if i == 0 else (w.n - count,)):
                seq_call(w, w.ctx, seq, first, count, ALL, levels, threads, pool if levels == 5 else None,
                         what=f"c4 threads {threads} first {first} count {count} levels {levels}")
    seq.close()


SOURCES = [("grey", "stored"), ("grey", "deflated"), ("grey", "folder"), ("colour", "folder"), ("mixed", "folder")]


@pytest.mark.gpu
@pytest.mark.parametrize("flags", range(16))
@pytest.mark.parametrize("geom", ["odd", "tiny"])
def test_flags_and_levels(world, pinned, geom, flags):
    """Every flag combination at 1 and MDC_MAX_PYR_LEVELS levels; non-rectifying calls go through unmap + K2 at the input size
    with unpadded rows.  On tiny, the levels without pixels are passed as NULL."""
    w = world(geom)
    kind, fmt = SOURCES[flags % len(SOURCES)]
    seq = w.seq(kind, fmt)
    c = chunk_of(8)
    pool = pinned(pool_bytes(w, flags, MAX_LEVELS, 2 * c + 1))
    for levels in (1, MAX_LEVELS):
        seq_call(w, w.ctx, seq, flags + 1, 2 * c + 1, flags, levels, 8, pool if levels > 1 else None, kind=kind,
                 what=f"{geom} {kind} {fmt} flags {flags} levels {levels}")
    seq.close()


@pytest.mark.gpu
@pytest.mark.parametrize("geom", ["odd", "tiny"])
def test_loaders(world, pinned, geom):
    """The feed under each input loader of the fused kernel.  These widths are not a multiple of 16, so TMA cannot read tightly
    packed frames; the host pipeline pads the rows to a multiple of 32 bytes during its copy, and the loaders see those padded
    pipe buffers.  Every loader that loader_usable admits for the padded pitch must run bit-exact (TMA among them: it is what the
    padding is for, and what auto resolves to); any other loader either runs bit-exact or is refused with nothing written."""
    w = world(geom)
    seq = w.seq("grey", "stored")
    ctx = w.new_ctx()
    pitch = (w.iw + 31) // 32 * 32
    assert not ctx.loader_usable("tma") and ctx.loader_usable("tma", pitch)
    assert ctx.auto_loader(pitch) != "ldg"
    c = chunk_of(8)
    pool = pinned(pool_bytes(w, ALL, 5, 2 * c + 1))
    ran = []
    for loader in ("auto", "ldg", "tma", "tex", "hybrid"):
        must = loader == "auto" or ctx.loader_usable(loader, pitch)
        ctx.configure(use_tma=loader)
        out = Out(w.shapes(ALL, 5), 2 * c + 1, pool)
        rc = lib.mdc_seq_prepare(ctx._h, seq._h, 5, 2 * c + 1, ALL, out.ptrs(), 5, 8)
        if rc == UNSUPPORTED and not must:
            assert out.untouched()
            continue
        assert rc == OK, (loader, must, rc, lib.mdc_last_error())
        check_out(w, out, "grey", ALL, 5, 2 * c + 1, f"{geom} loader {loader}")
        ran.append(loader)
    print(f"{geom}: pitch {pitch}, auto = {ctx.auto_loader(pitch)}, loaders run bit-exact: {ran}")
    ctx.close()
    seq.close()


@pytest.mark.gpu
@pytest.mark.parametrize("host_chunk", ["1", "7", None, "1000"])
def test_host_pipeline_chunking(world, pinned, monkeypatch, host_chunk):
    """MDC_HOST_CHUNK (read on every call) through the feed, and mdc_prepare_batch_host called directly with pageable and pinned
    input and output, rectifying (padded rows) and not.  The long calls on tiny frames cross up to 40 chunk boundaries: their
    frames decode in microseconds while small host chunks keep each staged chunk in use for longer, so a staging buffer refilled
    before its chunk has been copied to the device shows there."""
    if host_chunk is None:
        monkeypatch.delenv("MDC_HOST_CHUNK", raising=False)
    else:
        monkeypatch.setenv("MDC_HOST_CHUNK", host_chunk)
    t = world("tiny")
    tseq = t.seq("grey", "stored")
    for threads in (8, 128):
        c = chunk_of(threads)
        count = min(40 * c + 1, t.n - 2) if c < 100 else 3 * c + 1
        seq_call(t, t.ctx, tseq, 1, count, ALL, 3, threads, what=f"tiny feed MDC_HOST_CHUNK={host_chunk} threads {threads} count {count}")
    tseq.close()
    w = world("odd")
    seq = w.seq("grey", "deflated")
    c = chunk_of(8)
    count = 2 * c + 1
    pool = pinned(pool_bytes(w, GAMMA | VIG | NAN, 5, count))
    for flags in (ALL, GAMMA | VIG | NAN):
        seq_call(w, w.ctx, seq, 3, count, flags, 5, 8, pool, what=f"feed MDC_HOST_CHUNK={host_chunk} flags {flags}")
    first = 11
    frames = np.stack([w.raw("grey", (first + k) % w.P).reshape(-1) for k in range(count)])
    pinned_in = pinned(frames.nbytes + 4).view(np.uint8)[:frames.nbytes].reshape(frames.shape)
    pinned_in[:] = frames
    for flags in (ALL, GAMMA | VIG | NAN):
        for src, in_name in ((frames, "pageable"), (pinned_in, "pinned")):
            for out_pool, out_name in ((None, "pageable"), (pool, "pinned")):
                out = Out(w.shapes(flags, 5), count, out_pool)
                rc = lib.mdc_prepare_batch_host(w.ctx._h, src.ctypes.data, count, flags, out.ptrs(), 5)
                assert rc == OK, lib.mdc_last_error()
                check_out(w, out, "grey", flags, first, count,
                          f"mdc_prepare_batch_host MDC_HOST_CHUNK={host_chunk} flags {flags} {in_name} in, {out_name} out")
    seq.close()


@pytest.mark.gpu
def test_state_across_calls(world, pinned):
    """One context and one sequence object through calls that grow and reuse the staging and pipe buffers and switch between
    padded and unpadded rows; then two sequences on one context, and one sequence on two contexts."""
    w = world("odd")
    ctx = w.new_ctx()
    seq = w.seq("grey", "stored")
    steps = []
    for threads in (1, 128, 8, 128):                       # staging grows and is reused
        steps.append((threads, 1, ALL))
    for levels in (1, MAX_LEVELS, 1):                      # pipe buffers grow
        steps.append((8, levels, ALL))
    for flags in (ALL, GAMMA | VIG | NAN, RECT | GAMMA, GAMMA, ALL):       # padded <-> unpadded pitch
        steps.append((3, 3, flags))

    def count_of(threads):
        c = chunk_of(threads)
        return c + 1 if c > 100 else 2 * c + 1
    pool = pinned(max(pool_bytes(w, f, lv, count_of(t)) for t, lv, f in steps))
    for i, (threads, levels, flags) in enumerate(steps):
        count = count_of(threads)
        seq_call(w, ctx, seq, 7 * i, count, flags, levels, threads, pool, what=f"step {i}: threads {threads} levels {levels} flags {flags}")
    other = w.seq("mixed", "folder")
    for i in range(4):                                     # two sequences alternating on one context
        s, kind = (seq, "grey") if i % 2 == 0 else (other, "mixed")
        seq_call(w, ctx, s, 2 + i, 2 * chunk_of(4) + 1, ALL, 2, 4, pool, kind=kind, what=f"two sequences, call {i} ({kind})")
    ctx2 = w.new_ctx()
    for i in range(4):                                     # one sequence on two contexts in turn
        seq_call(w, (ctx, ctx2)[i % 2], seq, 30 + i, 2 * chunk_of(4) + 1, ALL, 2, 4, pool, what=f"two contexts, call {i}")
    ctx2.close()
    ctx.close()
    other.close()
    seq.close()


@pytest.mark.gpu
def test_benchmark_call_pattern_c4(world, pinned):
    """bench.py's c4_sequence leg: 1 level, rectify + gamma + vignette, into one mdc_host_alloc buffer, over the thread sweep
    cap/4, cap/2, cap; every call crosses at least three chunk boundaries and one call per sweep step ends at the last entry and
    the next starts again at the first, as run_decode does."""
    w = world("c4")
    seq = w.seq("grey", "stored")
    sweep = capped_bench_sweep()
    call = 3 * chunk_of(max(sweep)) + 1
    assert call + 12 <= w.n
    pool = pinned(pool_bytes(w, BENCH_FLAGS, 1, call))
    for threads in sweep:
        v, done, n_frames = w.n - call - 10, 0, 2 * call
        wrapped = False
        while done < n_frames:
            first = v % w.n
            cnt = min(w.n - first, n_frames - done, call)
            wrapped |= first == 0 and done > 0
            seq_call(w, w.ctx, seq, first, cnt, BENCH_FLAGS, 1, threads, pool, what=f"c4 bench pattern threads {threads} first {first} count {cnt}")
            v += cnt
            done += cnt
        assert wrapped
    seq.close()


def call_with_deadline(fn, seconds=120):
    """(rc, mdc_last_error of the calling thread); fails if the call does not return."""
    box = {}

    def run():
        box["rc"] = fn()
        box["err"] = lib.mdc_last_error()
    t = threading.Thread(target=run, daemon=True)
    t.start()
    t.join(seconds)
    assert not t.is_alive(), "the call did not return"
    return box["rc"], box["err"]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["stored", "folder"])
@pytest.mark.parametrize("case", ["cut_in_headers", "progressive", "wrong_size"])
def test_error_in_the_third_chunk(world, pinned, tmp_path, fmt, case):
    """A bad frame at the start of the third chunk: MDC_ERR_FORMAT naming the entry, the two chunks before it complete and
    bit-exact, nothing written from its chunk on; the same objects then prepare good ranges bit for bit.  (A file cut inside
    its scan is no error: test_scan_cut_in_the_third_chunk.)"""
    w = world("odd")
    threads, c = 4, chunk_of(4)
    first, count = 1, 4 * c
    bad_at = first + 2 * c
    entries = w.entries("grey", 6 * c)
    name = f"{bad_at:05d}.jpg"
    entries[bad_at] = (name, bad_payloads(w)[case])
    write_sequence(str(tmp_path / "seq"), entries, fmt)
    seq = api.Sequence(str(tmp_path / "seq"))
    ctx = w.ctx
    pool = pinned(pool_bytes(w, ALL, 2, count))
    out = Out(w.shapes(ALL, 2), count, pool)
    rc, err = call_with_deadline(lambda: lib.mdc_seq_prepare(ctx._h, seq._h, first, count, ALL, out.ptrs(), 2, threads))
    assert rc == FORMAT and name.encode() in err, (rc, err)
    check_out(w, out, "grey", ALL, first, 2 * c, f"{case} {fmt}: frames before the bad chunk")
    seq_call(w, ctx, seq, first, 2 * c, ALL, 2, threads, pool, what=f"{case} {fmt}: good range before")
    seq_call(w, ctx, seq, bad_at + 1, 2 * c + 1, ALL, 2, threads, pool, what=f"{case} {fmt}: good range after")
    seq.close()


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["stored", "folder"])
def test_scan_cut_in_the_third_chunk(world, pinned, tmp_path, fmt):
    """A frame cut halfway through its entropy-coded scan, at the start of the third chunk, stops nothing: it decodes as libjpeg
    decodes it (missing scan data read as zero bits) and is prepared like every other frame of the call."""
    w = world("odd")
    threads, c = 4, chunk_of(4)
    first, count = 1, 4 * c
    bad_at = first + 2 * c
    blob, raw = scan_cut(w)
    entries = w.entries("grey", 6 * c)                     # fewer than P entries: no other entry shares the cut one's payload index
    entries[bad_at] = (entries[bad_at][0], blob)
    write_sequence(str(tmp_path / "seq"), entries, fmt)
    w.variant("grey_scan_cut", "grey", {bad_at % w.P: raw})
    seq = api.Sequence(str(tmp_path / "seq"))
    pool = pinned(pool_bytes(w, ALL, 2, count))
    seq_call(w, w.ctx, seq, first, count, ALL, 2, threads, pool, kind="grey_scan_cut", what=f"scan cut {fmt}")
    seq.close()


@pytest.mark.gpu
def test_arguments(world, monkeypatch):
    """Bad ranges, level counts and NULL levels are refused with the outputs untouched; count = 0 writes nothing."""
    w = world("tiny")
    seq = w.seq()
    n = seq.getNumImages()
    ctx = w.ctx
    out = Out(w.shapes(ALL, 2), 4)
    for first, count, levels in ((-1, 4, 2), (0, -1, 2), (n - 3, 4, 2), (1, INT_MAX, 2), (0, 4, 0), (0, 4, 9)):
        rc = lib.mdc_seq_prepare(ctx._h, seq._h, first, count, ALL, out.ptrs(extra=8), levels, 4)
        assert rc == INVALID_ARG, (first, count, levels, rc)
    assert out.untouched()
    rc = lib.mdc_seq_prepare(ctx._h, seq._h, 0, 4, ALL, out.ptrs(null_level=1), 2, 4)
    assert rc == INVALID_ARG and b"level 1 is NULL" in lib.mdc_last_error() and out.untouched()
    frames = np.stack([w.raw("grey", p).reshape(-1) for p in range(4)])
    for chunk in ("1", "16"):               # with one-frame chunks, level 0 of the first frames would be copied before level 1 fails
        monkeypatch.setenv("MDC_HOST_CHUNK", chunk)
        rc = lib.mdc_prepare_batch_host(ctx._h, frames.ctypes.data, 4, ALL, out.ptrs(null_level=1), 2)
        assert rc == INVALID_ARG and b"level 1 is NULL" in lib.mdc_last_error() and out.untouched(), chunk
    monkeypatch.delenv("MDC_HOST_CHUNK")
    assert lib.mdc_seq_prepare(ctx._h, seq._h, 5, 0, ALL, out.ptrs(), 2, 4) == OK and out.untouched()
    assert lib.mdc_prepare_batch_host(ctx._h, frames.ctypes.data, 0, ALL, out.ptrs(), 2) == OK and out.untouched()
    # levels without pixels may be NULL (tiny: level 5 is 1 x 0)
    seq_call(w, ctx, seq, 0, 3, ALL, MAX_LEVELS, 4)
    seq.close()
