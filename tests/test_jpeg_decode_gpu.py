"""JPEG decoding on the GPU (csrc/mdc_jpeg_gpu.cu): mdc_jpeg_decode_device against the host decoder, and the device feed
mdc_seq_prepare_device against mdc_seq_prepare, bit for bit."""
import ctypes as C
import os
import subprocess
import sys
import zipfile

import numpy as np
import pytest

from mono_dataset_code_b200 import _lib, api, synthetic as S

cv2 = pytest.importorskip("cv2")
torch = pytest.importorskip("torch")
import jpeg_cases as J  # noqa: E402

pytestmark = pytest.mark.gpu
lib = _lib.lib
OK, FORMAT = 0, 3
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def host_decode(tmp_path, blobs, scalar=False):
    """The host decoder's result per blob (None = rejected) and its message, in a child process when the scalar transform is wanted."""
    folder = tmp_path / ("hs" if scalar else "h")
    os.makedirs(folder / "images", exist_ok=True)
    for i, b in enumerate(blobs):
        (folder / "images" / f"{i:06d}.jpg").write_bytes(b)
    child = ("import sys, pickle, numpy as np; sys.path.insert(0, %r); from mono_dataset_code_b200 import api, _lib; s = api.Sequence(%r); "
             "r = []\nfor i in range(s.getNumImages()):\n    g = s.getImageRaw_internal(i); r.append((g, None if g is not None else _lib.lib.mdc_last_error().decode()))\n"
             "pickle.dump(r, open(%r, 'wb'))" % (ROOT, str(folder), str(folder / "out.pkl")))
    env = dict(os.environ, MDC_JPEG_SCALAR="1" if scalar else "0")
    r = subprocess.run([sys.executable, "-c", child], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    import pickle
    return pickle.load(open(folder / "out.pkl", "rb"))


def check_same(blobs, w, h, expect, what):
    pitch = (w + 15) // 16 * 16
    out = torch.full((len(blobs), h, pitch), 0xA5, dtype=torch.uint8, device="cuda:0")
    out, status = api.jpeg_decode_device(blobs, w, h, row_pitch=pitch, out=out)
    got = out.cpu().numpy()
    for i, (exp, _) in enumerate(expect):
        if exp is None:
            assert status[i] == FORMAT, (what, i)
            assert (got[i] == 0xA5).all(), (what, i, "rows of a failed frame were written")
        else:
            assert status[i] == OK, (what, i)
            assert np.array_equal(got[i, :, :w], exp), (what, i, np.count_nonzero(got[i, :, :w] != exp))
            assert (got[i, :, w:] == 0xA5).all(), (what, i, "padding written")


def test_decode_device_equals_host_on_the_corpus(tmp_path):
    files = J.corpus()
    W, H = 1920, 1080
    rng = np.random.default_rng(7)
    yy, xx = np.mgrid[0:H, 0:W]
    for i, extra in enumerate(([], [cv2.IMWRITE_JPEG_RST_INTERVAL, 5], [cv2.IMWRITE_JPEG_OPTIMIZE, 1])):
        img = np.clip(xx * 0.07 + yy * 0.05 + 40 * np.sin((xx + 13 * i) * 0.05) + rng.normal(0, 1.5, (H, W)), 0, 255).astype(np.uint8)
        files.append((W, H, cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90] + extra)[1].tobytes()))
    files += J.scan_cuts(files[:40])
    expect = host_decode(tmp_path, [b for (_, _, b) in files], scalar=True)
    by_size = {}
    for (w, h, b), e in zip(files, expect):
        by_size.setdefault((w, h), []).append((b, e))
    for (w, h), items in by_size.items():
        check_same([b for b, _ in items], w, h, [e for _, e in items], f"{w}x{h}")


def test_mixed_batches(tmp_path):
    """Restart and no-restart frames, standard and optimised Huffman tables, grey and colour, with frames the header parser rejects
    (progressive, not a JPEG, truncated header, another size) between good ones."""
    w, h = 96, 64
    rng = np.random.default_rng(9)
    good = []
    for k in range(12):
        img = J.scene(rng, h, w, ("smooth", "noise", "edges", "ramp")[k % 4])
        params = [cv2.IMWRITE_JPEG_QUALITY, 40 + 5 * k]
        if k % 3 == 1:
            params += [cv2.IMWRITE_JPEG_RST_INTERVAL, 1 + k % 4]
        if k % 3 == 2:
            params += [cv2.IMWRITE_JPEG_OPTIMIZE, 1]
        if k % 4 == 3:
            img = np.stack([img, 255 - img, np.roll(img, 5, 0)], 2)
        good.append(cv2.imencode(".jpg", img, params)[1].tobytes())
    prog = cv2.imencode(".jpg", J.scene(rng, h, w, "smooth"), [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes()
    other = cv2.imencode(".jpg", J.scene(rng, 48, 80, "smooth"))[1].tobytes()
    bad = [prog, b"not a jpeg at all", good[0][:40], other]
    blobs = []
    for k, g in enumerate(good):
        blobs.append(g)
        if k % 3 == 0:
            blobs.append(bad[(k // 3) % len(bad)])
    expect = host_decode(tmp_path, blobs)
    expect = [(e, m) if (e is not None and e.shape == (h, w)) else (None, m) for (e, m) in expect]
    check_same(blobs, w, h, expect, "mixed")
    _, status = api.jpeg_decode_device(blobs, w, h)
    first = int(np.flatnonzero(status != OK)[0])
    assert lib.mdc_last_error().decode().startswith(f"frame {first}: "), lib.mdc_last_error()


def test_damaged_streams_match_the_host(tmp_path):
    """The damaged set the CPU sanitizer test has passed (test_jpeg_entropy_host.py): the host's accept / reject decision (its
    64-bit scalar transform, which J2 restates) and its bytes where accepted; the message of the first bad frame is the host's."""
    dmg = [b for (_, b) in J.damaged_set()]
    expect = host_decode(tmp_path, dmg, scalar=True)
    w, h = 200, 120
    # a damaged header can still parse as another size: such frames are rejected by mdc_jpeg_decode_device's size rule
    exp = [(e, m) if (e is not None and e.shape == (h, w)) else (None, m) for (e, m) in expect]
    check_same(dmg, w, h, exp, "damaged")
    # (the sequence reader hands a file without the JPEG signature to its PNG decoder: the JPEG decoder's message is another one there)
    rejected = [i for i, (e, _) in enumerate(expect) if e is None and dmg[i][:2] == b"\xff\xd8"]
    assert len(rejected) > 50
    for i in rejected[:60]:
        _, status = api.jpeg_decode_device([dmg[i]], w, h)
        assert status[0] == FORMAT
        assert lib.mdc_last_error().decode() == "frame 0: " + expect[i][1].split(": ", 1)[1], (i, expect[i][1], lib.mdc_last_error())


# ------------------------------------------------------------------ the device feed
def payloads(w, h, n_distinct, seed=1):
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    return [np.clip(xx * (150.0 / w) + yy * (60.0 / h) + 30 * np.sin((xx + 13 * i) * 0.05) + rng.normal(0, 3, (h, w)), 0, 255).astype(np.uint8)
            for i in range(n_distinct)]


def write_seq(folder, w, h, entries, fmt):
    """entries: list of (ext, bytes).  fmt: folder / stored / deflated."""
    S.write_dataset_dir(str(folder), w, h, w // 2 * 2, h // 2 * 2, "crop")
    if fmt == "folder":
        os.makedirs(folder / "images", exist_ok=True)
        for i, (ext, b) in enumerate(entries):
            (folder / "images" / f"{i:05d}.{ext}").write_bytes(b)
    else:
        with zipfile.ZipFile(folder / "images.zip", "w", zipfile.ZIP_STORED if fmt == "stored" else zipfile.ZIP_DEFLATED) as z:
            for i, (ext, b) in enumerate(entries):
                z.writestr(f"{i:05d}.{ext}", b)
    with open(folder / "times.txt", "w") as f:
        for i in range(len(entries)):
            f.write(f"{i} {i * 0.05:.3f} 1.0\n")
    return folder


def make(folder, w, h, entries, fmt):
    write_seq(folder, w, h, entries, fmt)
    fov = api.UndistorterFOV(str(folder / "camera.txt"))
    photo = api.PhotometricUndistorter(str(folder / "pcalib.txt"), str(folder / "vignette.png"), w, h)
    return api.Context(fov, photo, 0), api.Sequence(str(folder) + "/")


def shapes(ctx, flags, levels):
    w, h = ctx.level_dims(0) if flags & 1 else ctx.in_dims
    return [(w >> l, h >> l) for l in range(levels)]


def host_prepare(ctx, seq, first, count, flags, levels, threads):
    outs = [np.full((count, w * h), np.nan, np.float32) for (w, h) in shapes(ctx, flags, levels)]
    ptrs = (C.c_void_p * levels)(*[o.ctypes.data for o in outs])
    rc = lib.mdc_seq_prepare(ctx._h, seq._h, first, count, flags, ptrs, levels, threads)
    return rc, outs


SENT = 0x7FBADBAD


def device_prepare(ctx, seq, first, count, flags, levels, threads):
    outs = [torch.full((count, w * h), SENT, dtype=torch.int32, device="cuda:0").view(torch.float32) for (w, h) in shapes(ctx, flags, levels)]
    ptrs = (C.c_void_p * levels)(*[o.data_ptr() for o in outs])
    rc = lib.mdc_seq_prepare_device(ctx._h, seq._h, first, count, flags, ptrs, levels, threads, None)
    return rc, [o.cpu().numpy() for o in outs]


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def compare(ctx, seq, first, count, flags, levels, threads, what):
    rc_h, host = host_prepare(ctx, seq, first, count, flags, levels, threads)
    rc_d, dev = device_prepare(ctx, seq, first, count, flags, levels, threads)
    assert rc_h == OK and rc_d == OK, (what, rc_h, rc_d, lib.mdc_last_error())
    for l in range(levels):
        assert same_bits(host[l], dev[l]), (what, l, np.count_nonzero(host[l].view(np.uint32) != dev[l].view(np.uint32)))


def jpeg_entries(imgs, n, **kw):
    params = [cv2.IMWRITE_JPEG_QUALITY, kw.get("quality", 90)] + kw.get("extra", [])
    blobs = [cv2.imencode(".jpg", im, params)[1].tobytes() for im in imgs]
    return [("jpg", blobs[i % len(blobs)]) for i in range(n)]


def test_feed_flags_levels_and_containers(tmp_path):
    w, h = 90, 70
    imgs = payloads(w, h, 7)
    entries = jpeg_entries(imgs, 40, extra=[cv2.IMWRITE_JPEG_RST_INTERVAL, 2])
    for fmt in ("folder", "stored", "deflated"):
        ctx, seq = make(tmp_path / fmt, w, h, entries, fmt)
        for flags in range(16):
            for levels in (1, 4):
                compare(ctx, seq, 3, 30, flags, levels, 1, f"{fmt} flags {flags} levels {levels}")


def test_feed_png_pgm_jpeg_mix_across_chunk_boundaries(tmp_path):
    """65 frames with threads = 1 (chunks of 32): two chunk boundaries; 8-bit PNG, 16-bit PNG, PGM and grey / colour JPEG entries."""
    w, h = 64, 48
    imgs = payloads(w, h, 11, seed=4)
    entries = []
    for i in range(70):
        im = imgs[i % len(imgs)]
        k = i % 5
        if k == 0:
            entries.append(("png", cv2.imencode(".png", im)[1].tobytes()))
        elif k == 1:
            entries.append(("png", cv2.imencode(".png", im.astype(np.uint16) * 257 + 3)[1].tobytes()))
        elif k == 2:
            entries.append(("pgm", cv2.imencode(".pgm", im)[1].tobytes()))
        elif k == 3:
            entries.append(("jpg", cv2.imencode(".jpg", np.stack([im, 255 - im, im], 2), [cv2.IMWRITE_JPEG_QUALITY, 80])[1].tobytes()))
        else:
            entries.append(("jpg", cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, 95, cv2.IMWRITE_JPEG_RST_INTERVAL, 3])[1].tobytes()))
    for fmt in ("folder", "deflated"):
        ctx, seq = make(tmp_path / fmt, w, h, entries, fmt)
        for threads in (1, 2):
            compare(ctx, seq, 2, 65, 15, 3, threads, f"{fmt} threads {threads}")
            compare(ctx, seq, 0, 65, 0, 1, threads, f"{fmt} threads {threads} raw")


@pytest.mark.parametrize("damage", ["entropy", "header", "size"])
def test_feed_error_in_the_third_chunk(tmp_path, damage):
    """threads = 1: chunks of 32 frames.  Frame 70 cannot be used — its scan is corrupt (found by J1 on the GPU), its header is
    (found on the host), or it has another size.  Both feeds return MDC_ERR_FORMAT with chunks 0 and 1 complete and nothing after."""
    w, h = 64, 48
    imgs = payloads(w, h, 5, seed=8)
    entries = jpeg_entries(imgs, 100, extra=[cv2.IMWRITE_JPEG_RST_INTERVAL, 4])
    blob = bytearray(entries[70][1])
    if damage == "entropy":
        s = J.scan_start(bytes(blob))
        blob[s:s + 12] = b"\xff\x00" * 6            # stuffed 0xFF bytes: a run of 1 bits no DC code of the standard tables matches
    elif damage == "header":
        blob = bytearray(cv2.imencode(".jpg", imgs[0], [cv2.IMWRITE_JPEG_PROGRESSIVE, 1])[1].tobytes())
    else:
        blob = bytearray(cv2.imencode(".jpg", cv2.resize(imgs[0], (32, 48)))[1].tobytes())
    entries[70] = ("jpg", bytes(blob))
    ctx, seq = make(tmp_path / damage, w, h, entries, "stored")
    rc_h, host = host_prepare(ctx, seq, 0, 100, 15, 2, 1)
    msg_h = lib.mdc_last_error().decode()
    rc_d, dev = device_prepare(ctx, seq, 0, 100, 15, 2, 1)
    msg_d = lib.mdc_last_error().decode()
    assert rc_h == FORMAT and rc_d == FORMAT, (rc_h, rc_d, msg_h, msg_d)
    assert msg_d.split(": ", 1)[1] == msg_h.split(": ", 1)[1], (msg_h, msg_d)
    for l in range(2):
        assert same_bits(host[l][:64], dev[l][:64]), l
        assert (dev[l][64:].view(np.uint32) == SENT).all(), l


def test_feed_512_frames_at_1080p(tmp_path):
    """One 512-frame call at the benchmark's geometry (1920 x 1080, quality 90, stored zip), compared frame by frame with the host feed
    on the 7 distinct payloads it cycles (7 divides no chunk)."""
    w, h, P = 1920, 1080, 7
    imgs = payloads(w, h, P, seed=11)
    entries = jpeg_entries(imgs, 512)
    ctx, seq = make(tmp_path / "c4", w, h, entries, "stored")
    rc_h, host = host_prepare(ctx, seq, 0, P, 7, 1, 0)
    assert rc_h == OK
    outs = [torch.full((512, w * h), SENT, dtype=torch.int32, device="cuda:0").view(torch.float32)]
    ptrs = (C.c_void_p * 1)(outs[0].data_ptr())
    assert lib.mdc_seq_prepare_device(ctx._h, seq._h, 0, 512, 7, ptrs, 1, 0, None) == OK, lib.mdc_last_error()
    exp = torch.from_numpy(host[0]).to("cuda:0").view(torch.int32)
    got = outs[0].view(torch.int32)
    for i in range(512):
        assert torch.equal(got[i], exp[i % P]), i
    # the Python wrapper: torch tensors on the context's device
    t = seq.prepare_device(ctx, 0, P, True, True, True, False, levels=2)
    assert torch.equal(t[0].view(torch.int32), exp)
