"""Sequence reader (csrc/mdc_sequence.cpp): the file side of DatasetReader without OpenCV / libzip, SURVEY.md §8f N1.
CPU: zip directory / inflate / CRC, folder listing, times.txt semantics, PNG / PGM frames against cv2 and the originals.
GPU: the decode-ahead feed against the oracle."""
import os
import zipfile

import numpy as np
import pytest

from mono_dataset_code_b200 import api, synthetic as S

W, H, N = 72, 40, 11


def make_frames(rng):
    fr = [rng.integers(0, 256, (H, W), dtype=np.uint8) for _ in range(N)]
    fr[3][:] = 255
    fr[4][:] = 0
    return fr


def write_frame_files(folder, frames, rng):
    """Mixed lossless formats: 8-bit PNG, 16-bit PNG (high byte = the frame), binary PGM.  Returns the file names."""
    names = []
    for i, f in enumerate(frames):
        if i % 3 == 0:
            name = f"{i:05d}.png"
            S.write_png_gray(os.path.join(folder, name), f)
        elif i % 3 == 1:
            name = f"{i:05d}.png"
            S.write_png_gray(os.path.join(folder, name), (f.astype(np.uint16) << 8) | rng.integers(0, 256, f.shape, dtype=np.uint16))
        else:
            name = f"{i:05d}.pgm"
            S.write_pgm(os.path.join(folder, name), f)
        names.append(name)
    return names


def write_times(path, n, with_exposure=True):
    with open(path, "w") as t:
        for i in range(n):
            t.write(f"{i} {1234.5 + 0.05 * i:.6f} {0.5 + 0.25 * i:.4f}\n" if with_exposure else f"{i} {1234.5 + 0.05 * i:.6f}\n")


@pytest.fixture()
def folder_seq(tmp_path):
    rng = np.random.default_rng(1)
    frames = make_frames(rng)
    os.makedirs(tmp_path / "images")
    names = write_frame_files(str(tmp_path / "images"), frames, rng)
    write_times(tmp_path / "times.txt", N)
    return str(tmp_path), frames, names


@pytest.fixture(params=[zipfile.ZIP_STORED, zipfile.ZIP_DEFLATED], ids=["stored", "deflated"])
def zip_seq(tmp_path, request):
    rng = np.random.default_rng(2)
    frames = make_frames(rng)
    stage = tmp_path / "stage"
    os.makedirs(stage)
    names = write_frame_files(str(stage), frames, rng)
    with zipfile.ZipFile(tmp_path / "images.zip", "w", request.param) as z:
        for nm in reversed(names):                      # archive order is not name order: the reader sorts (:131)
            z.write(stage / nm, nm)
    write_times(tmp_path / "times.txt", N)
    return str(tmp_path), frames, names


def check_frames(seq, frames, names):
    assert seq.status == 0 and seq.getNumImages() == N
    for i in range(N):
        assert seq.name(i).endswith(names[i])
        raw = seq.getImageRaw_internal(i)
        assert raw.dtype == np.uint8 and np.array_equal(raw, frames[i]), f"frame {i} ({names[i]})"
        assert seq.getTimestamp(i) == float(f"{1234.5 + 0.05 * i:.6f}")
        assert seq.getExposure(i) == np.float32(f"{0.5 + 0.25 * i:.4f}")
    assert seq.getTimestamp(N) == 0 and seq.getExposure(-1) == 0 and seq.name(N) is None          # :171-186


def test_folder_sequence(folder_seq, capfd):
    folder, frames, names = folder_seq
    seq = api.Sequence(folder)
    out = capfd.readouterr().out
    assert f"found {N} files in folder /images" in out and f"Got {N} files!" in out
    assert not seq.isZipped()
    check_frames(seq, frames, names)


def test_zip_sequence(zip_seq, capfd):
    folder, frames, names = zip_seq
    seq = api.Sequence(folder + "/")
    out = capfd.readouterr().out
    assert "assuming that images are zipped" in out and f"got {N} entries and {N} files from zipfile!" in out
    assert seq.isZipped()
    check_frames(seq, frames, names)


def test_sixteen_bit_png_matches_opencv_grayscale_load(tmp_path):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(3)
    os.makedirs(tmp_path / "images")
    img16 = rng.integers(0, 65536, (H, W), dtype=np.uint16)
    S.write_png_gray(str(tmp_path / "images" / "00000.png"), img16)
    write_times(tmp_path / "times.txt", 1)
    seq = api.Sequence(str(tmp_path))
    exp = cv2.imread(str(tmp_path / "images" / "00000.png"), cv2.IMREAD_GRAYSCALE)
    assert np.array_equal(seq.getImageRaw_internal(0), exp)


def test_times_txt_semantics(tmp_path, capfd):
    rng = np.random.default_rng(4)
    os.makedirs(tmp_path / "images")
    write_frame_files(str(tmp_path / "images"), make_frames(rng), rng)
    write_times(tmp_path / "times.txt", N, with_exposure=False)               # two columns: exposure 0 (:303-307)
    seq = api.Sequence(str(tmp_path))
    assert seq.getTimestamp(2) == float(f"{1234.5 + 0.1:.6f}") and seq.getExposure(2) == 0
    write_times(tmp_path / "times.txt", N - 2)                                # count mismatch: everything zero (:322-329)
    capfd.readouterr()
    seq = api.Sequence(str(tmp_path))
    assert "Mismatch between number of images and number of timestamps" in capfd.readouterr().out
    assert seq.getNumImages() == N and all(seq.getTimestamp(i) == 0 and seq.getExposure(i) == 0 for i in range(N))


def test_error_paths(tmp_path, capfd):
    empty = api.Sequence(str(tmp_path))                                       # no images/, no images.zip: the reference exits (:117-121)
    assert empty.status == 2 and empty.getNumImages() == 0                    # MDC_ERR_IO
    assert "ERROR reading archive" in capfd.readouterr().out
    os.makedirs(tmp_path / "images")
    (tmp_path / "images" / "00000.png").write_bytes(b"\x89PNG\r\n\x1a\nthis is not a png")
    (tmp_path / "images" / "00001.jpg").write_bytes(b"\xff\xd8\xff\xe0 jpeg frames are the caller's business")
    write_times(tmp_path / "times.txt", 2)
    seq = api.Sequence(str(tmp_path))
    assert seq.getNumImages() == 2 and seq.getImageRaw_internal(0) is None and seq.getImageRaw_internal(1) is None
    # corrupt payload in a zip: CRC mismatch
    z = tmp_path / "z"
    os.makedirs(z)
    with zipfile.ZipFile(z / "images.zip", "w", zipfile.ZIP_STORED) as f:
        f.writestr("00000.pgm", b"P5\n4 2\n255\n" + bytes(range(8)))
    blob = bytearray((z / "images.zip").read_bytes())
    at = blob.find(bytes(range(8)))
    blob[at + 3] ^= 0x40
    (z / "images.zip").write_bytes(bytes(blob))
    write_times(z / "times.txt", 1)
    seq = api.Sequence(str(z))
    assert seq.getNumImages() == 1 and seq.getImageRaw_internal(0) is None
    from mono_dataset_code_b200 import _lib
    assert b"CRC mismatch" in _lib.lib.mdc_last_error()


@pytest.mark.gpu
@pytest.mark.parametrize("zipped", [False, True], ids=["folder", "zip"])
def test_decode_ahead_feed_matches_the_oracle(tmp_path, zipped):
    """mdc_seq_prepare = decode (host threads) -> pinned staging -> H2D -> fused kernel -> D2H, 65 frames in chunks of 16 (two per
    decode thread, at least 16).  tests/test_sequence_feed.py pins the feed frame for frame on JPEG sequences."""
    from conftest import assert_bits_equal
    from oracle.loader import PortOracle
    port = PortOracle()
    iw, ih, ow, oh, n = 96, 80, 88, 72, 70
    files = S.write_dataset_dir(str(tmp_path), iw, ih, ow, oh, "crop")
    frames = S.frames(n, iw, ih)
    stage = tmp_path / ("stage" if zipped else "images")
    os.makedirs(stage)
    for i in range(n):
        if i % 2:
            S.write_png_gray(str(stage / f"{i:05d}.png"), frames[i].reshape(ih, iw))
        else:
            S.write_pgm(str(stage / f"{i:05d}.pgm"), frames[i].reshape(ih, iw))
    if zipped:
        with zipfile.ZipFile(tmp_path / "images.zip", "w", zipfile.ZIP_DEFLATED) as z:
            for nm in sorted(os.listdir(stage)):
                z.write(stage / nm, nm)
    write_times(tmp_path / "times.txt", n)
    u = api.UndistorterFOV(files["camera"])
    p = api.PhotometricUndistorter(files["pcalib"], files["vignette"], iw, ih)
    prep = api.FramePreparer(u, p)
    seq = api.Sequence(str(tmp_path))
    assert seq.getNumImages() == n and seq.isZipped() == zipped
    outs = seq.prepare(prep.ctx, prep.level_shapes(True, 3), 3, n - 5, True, True, True, False, threads=4)
    rx, ry = u.remap_tables()
    ginv, vinv = p.getGInv(), p.vignette_maps()[1]
    for k in (0, 1, 31, 32, 33, n - 6):
        exp = port.pyramid(port.get_image(rx, ry, iw, ih, ginv, vinv, frames[3 + k], 1, 1, 1, 0), ow, oh, 3)
        for l in range(3):
            assert_bits_equal(outs[l][k], exp[l], f"frame {3 + k} level {l}")
    # a frame of the wrong size stops the call like the reference refuses it (:194-199)
    S.write_pgm(str(tmp_path / "images" / "00010.pgm") if not zipped else str(stage / "00010.pgm"), np.zeros((ih, iw + 2), np.uint8))
    if not zipped:
        with pytest.raises(api.MdcError):
            api.Sequence(str(tmp_path)).prepare(prep.ctx, prep.level_shapes(True, 1), 0, 20, True, True, True, False, threads=2)


def test_hostile_headers_are_errors_not_crashes(tmp_path):
    """Untrusted dimensions and directory records are bounded before anything is sized from them; nothing throws across the C ABI."""
    import struct
    import zlib
    from mono_dataset_code_b200 import _lib
    os.makedirs(tmp_path / "images")

    def chunk(tag, body):
        return struct.pack(">I", len(body)) + tag + body + struct.pack(">I", zlib.crc32(tag + body))
    sig = b"\x89PNG\r\n\x1a\n"
    huge = sig + chunk(b"IHDR", struct.pack(">IIBBBBB", 0xFFFFFFFF, 0xFFFFFFFF, 8, 0, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(b"\0")) + chunk(b"IEND", b"")
    big = sig + chunk(b"IHDR", struct.pack(">IIBBBBB", 70000, 70000, 16, 0, 0, 0, 0)) + chunk(b"IDAT", zlib.compress(b"\0")) + chunk(b"IEND", b"")
    noidat = sig + chunk(b"IHDR", struct.pack(">IIBBBBB", 4, 4, 8, 0, 0, 0, 0)) + chunk(b"IEND", b"")
    (tmp_path / "images" / "00000.png").write_bytes(huge)
    (tmp_path / "images" / "00001.png").write_bytes(big)
    (tmp_path / "images" / "00002.png").write_bytes(noidat)
    (tmp_path / "images" / "00003.pgm").write_bytes(b"P5\n99999999999999999999 2\n255\n" + bytes(8))
    (tmp_path / "images" / "00004.pgm").write_bytes(b"P5\n2000000000 2000000000\n255\n" + bytes(8))
    write_times(tmp_path / "times.txt", 5)
    seq = api.Sequence(str(tmp_path))
    assert seq.getNumImages() == 5
    for i in range(5):
        assert seq.getImageRaw_internal(i) is None, i
    assert seq.getImageRaw_internal(0) is None and b"implausible PNG dimensions" in _lib.lib.mdc_last_error()
    # zip: central directory pointing outside the archive / claiming more entries than it can hold
    z = tmp_path / "z"
    os.makedirs(z)
    with zipfile.ZipFile(z / "images.zip", "w", zipfile.ZIP_STORED) as f:
        f.writestr("00000.pgm", b"P5\n4 2\n255\n" + bytes(range(8)))
    good = bytearray((z / "images.zip").read_bytes())
    eocd = good.rfind(b"PK\x05\x06")
    for field, value in ((12, 0xFFFFFFF0), (16, 0x7FFFFFFF), (10, 5000)):      # cd_size, cd_off, n_entries
        bad = bytearray(good)
        if field == 10:
            bad[eocd + field:eocd + field + 2] = struct.pack("<H", value)
        else:
            bad[eocd + field:eocd + field + 4] = struct.pack("<I", value)
        (z / "images.zip").write_bytes(bytes(bad))
        s2 = api.Sequence(str(z))
        assert s2.status == 2 and s2.getNumImages() == 0, (field, value)
        assert b"central directory" in _lib.lib.mdc_last_error()
