"""mdc_seq_read_gray8_device (csrc/mdc_jpeg_gpu.cu): a sequence's raw 8-bit frames decoded into device memory, frame for frame what
mdc_seq_read_gray8 returns, and the two calibration programs that load their frames through it."""
import ctypes as C
import os
import subprocess
import zipfile

import numpy as np
import pytest

from conftest import ROOT
from mono_dataset_code_b200 import _lib, api, synthetic as S

lib = _lib.lib
OK, INVALID_ARG, FORMAT = 0, 1, 3
SENT = 0xA5


def write_seq(folder, entries, fmt, names=None):
    """entries: list of (ext, bytes).  fmt: folder / stored / deflated; names: entry names (default: sorted like the entries).  In a zip
    the entries are written in reverse name order, so that archive order and sequence order differ."""
    os.makedirs(folder, exist_ok=True)
    names = names or [f"{i:05d}.{ext}" for i, (ext, _) in enumerate(entries)]
    if fmt == "folder":
        os.makedirs(folder / "images", exist_ok=True)
        for name, (_, b) in zip(names, entries):
            (folder / "images" / name).write_bytes(b)
    else:
        with zipfile.ZipFile(folder / "images.zip", "w", zipfile.ZIP_STORED if fmt == "stored" else zipfile.ZIP_DEFLATED) as z:
            for name, (_, b) in sorted(zip(names, entries), reverse=True):
                z.writestr(name, b)
    return folder


# ------------------------------------------------------------------ argument checks (no device)
def test_argument_errors_need_no_device(tmp_path):
    seq = api.Sequence(str(write_seq(tmp_path / "s", [("pgm", b"P5\n4 3\n255\n" + bytes(12))] * 5, "folder")) + "/")
    assert seq.getNumImages() == 5
    fake_ctx = C.c_void_p(1)          # never dereferenced: every check below fails before the context is used
    buf = (C.c_uint8 * 64)()
    d = C.cast(buf, C.c_void_p)

    def rc(ctx, s, ids, w=4, h=3, pitch=4, out=d, n=None):
        a = np.ascontiguousarray(ids, dtype=np.int32)
        return lib.mdc_seq_read_gray8_device(ctx, s, a.ctypes.data if len(a) else None, len(a) if n is None else n, w, h, out, pitch,
                                             None, None, 0, None)
    for bad in ([5], [-1], [0, 1, 99], [4, 2, -3]):
        assert rc(fake_ctx, seq._h, bad) == INVALID_ARG
        assert "outside the sequence" in lib.mdc_last_error().decode()
    assert rc(fake_ctx, seq._h, [0], pitch=3) == INVALID_ARG                      # row_pitch < w
    assert rc(fake_ctx, seq._h, [0], w=0) == INVALID_ARG
    assert rc(fake_ctx, seq._h, [0], h=0) == INVALID_ARG
    assert rc(fake_ctx, seq._h, [0], w=-4, pitch=4) == INVALID_ARG
    assert rc(None, seq._h, [0]) == INVALID_ARG                                  # null context
    assert rc(fake_ctx, None, [0]) == INVALID_ARG                                # null sequence
    assert rc(fake_ctx, seq._h, [0], out=None) == INVALID_ARG                    # null output
    assert rc(fake_ctx, seq._h, [], n=2) == INVALID_ARG                          # null ids with n > 0
    assert rc(fake_ctx, seq._h, [0], n=-1) == INVALID_ARG
    # n = 0 is a no-op: nothing is read, nothing needs a context or a device
    status = np.full(1, -7, np.int32)
    assert lib.mdc_seq_read_gray8_device(None, None, None, 0, 4, 3, None, 4, status.ctypes.data, None, 0, None) == OK
    assert lib.mdc_seq_read_gray8_device(fake_ctx, seq._h, None, 0, 4, 3, d, 4, status.ctypes.data, None, 0, None) == OK
    assert status[0] == -7 and bytes(buf) == bytes(64)


def build_tool(tmp_path, name):
    exe = str(tmp_path / name)
    libdir = os.path.join(ROOT, "mono_dataset_code_b200", "lib")
    cmd = ["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++11", "-O2", "-Wall", "-I" + os.path.join(ROOT, "include"),
           "-I/usr/local/cuda/include", os.path.join(ROOT, "tools", name + ".cpp"), "-o", exe, "-L" + libdir, "-lmdc_b200",
           "-L/usr/local/cuda/lib64", "-lcudart", "-lz", "-Wl,-rpath," + libdir + ":/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return exe


def test_both_tools_build_and_print_usage(tmp_path):
    for name in ("responseCalib_b200", "vignetteCalib_b200"):
        r = subprocess.run([build_tool(tmp_path, name)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert r.returncode == 1 and f"usage: {name}" in r.stdout


# ------------------------------------------------------------------ GPU: equal to the host reader, frame for frame
def host_read(seq, i):
    """mdc_seq_read_gray8: (rc, w, h, pixels or None, message)."""
    w, h = C.c_int(0), C.c_int(0)
    rc = lib.mdc_seq_read_gray8(seq._h, i, None, 0, C.byref(w), C.byref(h))
    if rc != OK:
        return rc, 0, 0, None, lib.mdc_last_error().decode()
    px = np.empty((h.value, w.value), np.uint8)
    assert lib.mdc_seq_read_gray8(seq._h, i, px.ctypes.data, px.size, C.byref(w), C.byref(h)) == OK
    return OK, w.value, h.value, px, None


def check_against_host(seq, ctx, ids, W, H, pitch, threads):
    """One device call over `ids`; every status, size and row against mdc_seq_read_gray8.  Returns the first failed frame (its position
    in ids, and the host reader's message, None if the host reads it at another size) or None, and the call's message."""
    import torch
    out = torch.full((len(ids), H, pitch), SENT, dtype=torch.uint8, device="cuda:0")
    out, status, sizes = seq.read_gray8_device(ctx, ids, W, H, row_pitch=pitch, threads=threads, out=out)
    msg = lib.mdc_last_error().decode()
    got = out.cpu().numpy()
    first_bad = None
    for k, i in enumerate(ids):
        rc, w, h, px, hmsg = host_read(seq, int(i))
        if rc != OK:
            exp_status, exp_size = FORMAT, (0, 0)
        elif (w, h) != (W, H):
            exp_status, exp_size = INVALID_ARG, (w, h)
        else:
            exp_status, exp_size = OK, (W, H)
        assert status[k] == exp_status and tuple(sizes[k]) == exp_size, (k, i, status[k], sizes[k], exp_status, exp_size, hmsg)
        if exp_status == OK:
            assert np.array_equal(got[k, :, :W], px), (k, i, np.count_nonzero(got[k, :, :W] != px))
            assert (got[k, :, W:] == SENT).all(), (k, i, "padding written")
        else:
            assert (got[k] == SENT).all(), (k, i, "rows of a failed frame written")
            if first_bad is None:
                first_bad = (k, hmsg)
    return first_bad, msg


def gradient(w, h, i, rng):
    yy, xx = np.mgrid[0:h, 0:w]
    return np.clip(xx * (150.0 / w) + yy * (60.0 / h) + 30 * np.sin((xx + 13 * i) * 0.05) + rng.normal(0, 3, (h, w)), 0, 255).astype(np.uint8)


def mixed_entries(cv2, W, H, n, seed):
    """n frames cycling grey / 4:2:0 colour JPEGs (qualities 35..95, with and without restart intervals), 8- and 16-bit PNG and PGM.
    The cycle has 11 kinds, prime, so it divides no chunk size."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        im = gradient(W, H, i, rng)
        k = i % 11
        if k in (0, 1, 2, 3):
            params = [cv2.IMWRITE_JPEG_QUALITY, (35, 60, 90, 95)[k]] + ([cv2.IMWRITE_JPEG_RST_INTERVAL, 1 + k] if k % 2 else [])
            out.append(("jpg", cv2.imencode(".jpg", im, params)[1].tobytes()))
        elif k in (4, 5, 6):
            bgr = np.stack([im, 255 - im, np.roll(im, 5, 1)], 2)
            params = [cv2.IMWRITE_JPEG_QUALITY, (50, 80, 92)[k - 4]] + ([cv2.IMWRITE_JPEG_RST_INTERVAL, 2] if k == 5 else [])
            if hasattr(cv2, "IMWRITE_JPEG_SAMPLING_FACTOR"):
                params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420]
            out.append(("jpg", cv2.imencode(".jpg", bgr, params)[1].tobytes()))
        elif k == 7:
            out.append(("png", cv2.imencode(".png", im)[1].tobytes()))
        elif k == 8:
            out.append(("png", cv2.imencode(".png", im.astype(np.uint16) * 257 + (i % 200))[1].tobytes()))
        elif k == 9:
            out.append(("pgm", cv2.imencode(".pgm", im)[1].tobytes()))
        else:
            out.append(("jpg", cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, 75, cv2.IMWRITE_JPEG_OPTIMIZE, 1])[1].tobytes()))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["folder", "stored", "deflated"])
def test_equals_the_host_reader_per_id(tmp_path, fmt):
    """103 frames of 83 x 61 (neither a multiple of 8 nor of 16), every format mixed, plus a frame of another size and a file that is
    not an image; ids sorted, reversed, repeated and strided; three row pitches; threads = 1 (chunks of 32) and the default."""
    cv2 = pytest.importorskip("cv2")
    W, H = 83, 61
    entries = mixed_entries(cv2, W, H, 103, seed=1)
    entries[40] = ("jpg", cv2.imencode(".jpg", np.zeros((61, 82), np.uint8))[1].tobytes())
    entries[77] = ("png", b"not an image at all")
    seq = api.Sequence(str(write_seq(tmp_path / fmt, entries, fmt)) + "/")
    ctx = api.Context(None, None, 0)
    n = seq.getNumImages()
    rng = np.random.default_rng(3)
    id_sets = {"sorted": np.arange(n), "reversed": np.arange(n)[::-1], "strided": np.arange(1, n, 3),
               "repeated": rng.integers(0, n, 150), "one": np.array([40])}
    for name, ids in id_sets.items():
        for pitch in (W, 96, 131):
            for threads in (1, 0):
                if name != "sorted" and threads == 0 and pitch != 96:
                    continue
                first_bad, msg = check_against_host(seq, ctx, ids, W, H, pitch, threads)
                assert (first_bad is not None) == bool(np.isin(ids, [40, 77]).any()), name
                if first_bad is not None and first_bad[1] is None:      # another size: the host reads it, the call explains
                    assert msg.startswith("expected image dimensions 83 x 61; found 82 x 61"), (name, msg)
                elif first_bad is not None:
                    assert msg == first_bad[1], (name, msg, first_bad)
    # a call without failing frames returns MDC_OK
    ids = np.array([i for i in range(n) if i not in (40, 77)][:70])
    out, status, sizes = seq.read_gray8_device(ctx, ids, W, H)
    assert (status == OK).all() and (sizes == [W, H]).all()
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("damage", ["entropy", "truncated", "crc", "not_an_image", "other_size"])
def test_a_failed_frame_in_the_middle_chunk(tmp_path, damage):
    """threads = 1, 96 frames: chunks of 32.  Frame 45 of the middle chunk fails as the host reader fails on it (FORMAT) or reads at
    another size (INVALID_ARG with that size); every other frame is still decoded; the call returns MDC_ERR_FORMAT with frame 45's
    message."""
    cv2 = pytest.importorskip("cv2")
    import torch
    W, H = 64, 48
    rng = np.random.default_rng(8)
    imgs = [gradient(W, H, i, rng) for i in range(96)]
    entries = [("jpg", cv2.imencode(".jpg", imgs[i], [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_RST_INTERVAL, 4])[1].tobytes())
               for i in range(96)]
    blob = bytearray(entries[45][1])
    if damage == "entropy":
        at = blob.find(b"\xff\xda")
        s = at + 2 + ((blob[at + 2] << 8) | blob[at + 3])
        blob[s:s + 12] = b"\xff\x00" * 6            # stuffed 0xFF bytes: a run of 1 bits no DC code of the standard tables matches
    elif damage == "truncated":
        blob = blob[:150]
    elif damage == "not_an_image":
        blob = bytearray(b"%PDF-1.4 this is no frame")
    elif damage == "other_size":
        blob = bytearray(cv2.imencode(".jpg", cv2.resize(imgs[0], (40, 30)))[1].tobytes())
    entries[45] = ("jpg", bytes(blob))
    fmt = "stored"
    folder = write_seq(tmp_path / damage, entries, fmt)
    if damage == "crc":                              # flip one byte of entry 45's data in the archive: the reader's CRC check fails
        data = bytearray((folder / "images.zip").read_bytes())
        at = data.find(entries[45][1][-40:-8])       # entropy-coded bytes: unique to the frame (the headers are not)
        assert at > 0 and data.find(entries[45][1][-40:-8], at + 1) < 0
        data[at] ^= 0x55
        (folder / "images.zip").write_bytes(bytes(data))
    seq = api.Sequence(str(folder) + "/")
    ctx = api.Context(None, None, 0)
    ids = np.arange(96)
    out = torch.full((96, H, W), SENT, dtype=torch.uint8, device="cuda:0")
    rc = lib.mdc_seq_read_gray8_device(ctx._h, seq._h, ids.astype(np.int32).ctypes.data, 96, W, H, C.c_void_p(out.data_ptr()), W, None,
                                       None, 1, None)
    msg = lib.mdc_last_error().decode()
    assert rc == FORMAT
    hrc, w, h, px, hmsg = host_read(seq, 45)
    if damage == "other_size":
        assert hrc == OK and (w, h) == (40, 30)
        assert msg.startswith("expected image dimensions 64 x 48; found 40 x 30"), msg
    else:
        assert hrc == FORMAT and msg == hmsg, (msg, hmsg)
    first_bad, _ = check_against_host(seq, ctx, ids, W, H, W, 1)
    assert first_bad[0] == 45
    ctx.close()


# ------------------------------------------------------------------ GPU: the tools read JPEG zips to the same files as before
def encode_zip(cv2, folder, frames, times_txt, extra_files=None, replace=None):
    """frames as baseline JPEGs (quality 95) in images.zip, and the host decoder's bytes of the same JPEGs as PGM files in a folder
    dataset next to it.  -> (zip dataset, PGM dataset)."""
    blobs = [cv2.imencode(".jpg", f, [cv2.IMWRITE_JPEG_QUALITY, 95])[1].tobytes() for f in frames]
    for k, b in (replace or {}).items():
        blobs[k] = b
    zd, pd = folder / "zip", folder / "pgm"
    write_seq(zd, [("jpg", b) for b in blobs], "deflated")
    seq = api.Sequence(str(zd) + "/")
    os.makedirs(pd / "images")
    for i in range(len(blobs)):
        g = seq.getImageRaw_internal(i)
        if g is not None:
            S.write_pgm(str(pd / "images" / f"{i:05d}.pgm"), g)
        else:
            (pd / "images" / f"{i:05d}.pgm").write_bytes(b"P5 broken")
    seq.close()
    for d in (zd, pd):
        (d / "times.txt").write_text(times_txt)
        for name, data in (extra_files or {}).items():
            (d / name).write_bytes(data)
    return zd, pd


def run(exe, seq, work, *args):
    work.mkdir(parents=True, exist_ok=True)
    return subprocess.run([exe, str(seq) + "/", *args], cwd=work, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)


def lines_with(out, word):
    return [l for l in out.splitlines() if word in l]


def same_files(a, b, names):
    for n in names:
        assert (a / n).read_bytes() == (b / n).read_bytes(), n


@pytest.mark.gpu
def test_response_calib_reads_a_jpeg_zip_like_its_pgm_frames(tmp_path):
    cv2 = pytest.importorskip("cv2")
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "programs", "response_calib.npz"))
    w, h = int(g["w"]), int(g["h"])
    frames = [f.reshape(h, w) for f in g["frames"]]
    times = "".join(f"{i} {100.0 + 0.05 * i:.6f} {float(e):.9g}\n" for i, e in enumerate(g["exposures"]))
    exe = build_tool(tmp_path, "responseCalib_b200")
    zd, pd = encode_zip(cv2, tmp_path / "a", frames, times)
    outs = {}
    for name, d in (("zip", zd), ("pgm", pd)):
        r = run(exe, d, tmp_path / ("w" + name), "iterations=5")
        assert r.returncode == 0, r.stdout[-3000:]
        outs[name] = r.stdout
    assert lines_with(outs["zip"], "loaded") == lines_with(outs["pgm"], "loaded") == [f"loaded {len(frames)} images"]
    same_files(tmp_path / "wzip" / "photoCalibResult", tmp_path / "wpgm" / "photoCalibResult", ("pcalib.txt", "log.txt"))

    # an undecodable frame at a skip-aligned position is skipped
    zd, pd = encode_zip(cv2, tmp_path / "b", frames, times, replace={4: b"\xff\xd8\xff\xdb\x00"})
    n_skip = (len(frames) + 1) // 2
    for d in (zd, pd):
        r = run(exe, d, tmp_path / "wb", "iterations=2", "skip=2")
        assert r.returncode == 0 and lines_with(r.stdout, "loaded") == [f"loaded {n_skip - 1} images"], r.stdout[-2000:]
    # a frame of another size stops the tool, in id order
    for k, shape, word in ((6, (h, w + 8), "width"), (3, (h + 8, w), "height")):
        other = cv2.imencode(".jpg", np.full(shape, 90, np.uint8))[1].tobytes()
        zd, pd = encode_zip(cv2, tmp_path / f"c{k}", frames, times, replace={k: other})
        r = run(exe, zd, tmp_path / f"wc{k}", "iterations=2")
        assert r.returncode == 1 and f"{word} mismatch!" in r.stdout and "loaded" not in r.stdout, r.stdout[-2000:]


@pytest.mark.gpu
def test_vignette_calib_reads_a_jpeg_zip_like_its_pgm_frames(tmp_path):
    cv2 = pytest.importorskip("cv2")
    exe = build_tool(tmp_path, "vignetteCalib_b200")
    files = ("log.txt", "homographies.txt", "vignette.png", "vignetteSmoothed.png", "plane.png")
    # homographies=detect on the marker sequence
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "marker", "marker_sequence.npz"))
    hI, wI = g["frames"].shape[1:]
    extra = {"camera.txt": str(g["camera_txt"]).encode(), "pcalib.txt": str(g["pcalib_txt"]).encode()}
    zd, pd = encode_zip(cv2, tmp_path / "m", list(g["frames"]), str(g["times_txt"]), extra)
    for d in (zd, pd):
        S.write_png_gray(str(d / "vignette.png"), S.vignette_image(wI, hI))
    outs = {}
    for name, d in (("zip", zd), ("pgm", pd)):
        r = run(exe, d, tmp_path / ("m" + name), "homographies=detect", "iterations=4", "patternX=200", "patternY=200")
        assert r.returncode == 0, r.stdout[-3000:]
        outs[name] = r.stdout
    assert lines_with(outs["zip"], "loaded") == lines_with(outs["pgm"], "loaded")
    assert lines_with(outs["zip"], "found exactly one marker") == lines_with(outs["pgm"], "found exactly one marker")
    same_files(tmp_path / "mzip" / "vignetteCalibResult", tmp_path / "mpgm" / "vignetteCalibResult", files)

    # homographies=FILE on the reference program's fixture, with skip = 2
    v = np.load(os.path.join(os.path.dirname(__file__), "golden", "programs", "vignette_calib.npz"))
    wI, hI = int(v["wI"]), int(v["hI"])
    extra = {"camera.txt": str(v["camera_txt"]).encode(), "pcalib.txt": str(v["pcalib_txt"]).encode()}
    frames = [f.reshape(hI, wI) for f in v["frames"]]
    zd, pd = encode_zip(cv2, tmp_path / "v", frames, str(v["times_txt"]), extra)
    hom = tmp_path / "hom.txt"
    np.savetxt(hom, v["homographies"][::2], fmt="%.17g")
    outs = {}
    for name, d in (("zip", zd), ("pgm", pd)):
        S.write_png_gray(str(d / "vignette.png"), S.vignette_image(wI, hI))
        r = run(exe, d, tmp_path / ("v" + name), "homographies=" + str(hom), "iterations=3", "skip=2", "patternX=200", "patternY=200")
        assert r.returncode == 0, r.stdout[-3000:]
        outs[name] = r.stdout
    assert lines_with(outs["zip"], "loaded") == lines_with(outs["pgm"], "loaded")
    assert lines_with(outs["zip"], "loaded") == [f"loaded {int(np.isfinite(v['homographies'][::2, 0]).sum())} images with a marker"]
    same_files(tmp_path / "vzip" / "vignetteCalibResult", tmp_path / "vpgm" / "vignetteCalibResult", files[:1] + files[2:])

    # a frame that cannot be read stops the tool with the reader's message, in both modes
    zd, _ = encode_zip(cv2, tmp_path / "x", frames, str(v["times_txt"]), extra, replace={4: b"\xff\xd8\xff\xdb\x00"})
    S.write_png_gray(str(zd / "vignette.png"), S.vignette_image(wI, hI))
    seq = api.Sequence(str(zd) + "/")
    host_msg = host_read(seq, 4)[4]
    seq.close()
    for mode in ("homographies=" + str(hom), "homographies=detect"):
        r = run(exe, zd, tmp_path / "wx", mode, "iterations=1", "skip=2", "patternX=200", "patternY=200")
        assert r.returncode == 1, r.stdout[-2000:]
        assert f"frame 4: cannot read a {wI}x{hI} image: {host_msg}" in r.stdout, (r.stdout[-2000:], host_msg)
