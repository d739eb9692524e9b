"""The decode-ahead host feed of mdc_seq_prepare (csrc/mdc_sequence.cpp) without a GPU: tests/cpp/seq_feed_harness.cpp links the
sequence reader with a stub context and a fake prepare call that copies the staged frames into level 0, and runs it under
AddressSanitizer + UndefinedBehaviorSanitizer and under ThreadSanitizer.

Folder, stored-zip and deflated-zip sequences mix grey JPEG, colour JPEG, 8- and 16-bit PNG and PGM frames, every frame different.
For chunks of 16, 34 and 256 frames, ranges at offsets 0 and 1 with counts C-1, C, C+1 and 3C+1 must give mdc_seq_read_gray8 frame
for frame.  A bad frame at the start of the third chunk must stop the call with MDC_ERR_FORMAT naming its entry, after the first two
chunks and before anything of its own chunk is written.  The argument checks give their codes and messages before any decoding."""
import os
import subprocess
import zipfile

import numpy as np
import pytest

from conftest import ROOT

cv2 = pytest.importorskip("cv2")
CSRC = os.path.join(ROOT, "mono_dataset_code_b200", "csrc")
W, H = 44, 26                                  # not a whole number of JPEG blocks
THREADS = {1: 16, 17: 34, 128: 256}            # thread count -> chunk: min(256, max(16, 2 * threads))
N = 3 * 256 + 1 + 1                            # the longest range call at offset 1
SANITIZERS = {"asan": ["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined"], "tsan": ["-fsanitize=thread"]}
ENV = {"asan": {"ASAN_OPTIONS": "detect_leaks=0"}, "tsan": {"TSAN_OPTIONS": "halt_on_error=1"}}


@pytest.fixture(scope="module", params=sorted(SANITIZERS))
def harness(request, tmp_path_factory):
    san = request.param
    exe = str(tmp_path_factory.mktemp("seq_feed_" + san) / "seq_feed_harness")
    cmd = ["g++", "-O1", "-g", "-std=c++17", *SANITIZERS[san], "-I" + os.path.join(ROOT, "include"), "-I" + CSRC,
           os.path.join(ROOT, "tests", "cpp", "seq_feed_harness.cpp"), os.path.join(CSRC, "mdc_sequence.cpp"),
           os.path.join(CSRC, "mdc_gray_image.cpp"), os.path.join(CSRC, "mdc_jpeg.cpp"), "-lz", "-lpthread", "-o", exe]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        pytest.skip(f"no {san}-enabled g++ here: " + r.stdout[-300:])

    def run(*args):
        r = subprocess.run([exe, *map(str, args)], env=dict(os.environ, **ENV[san]), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                           text=True, timeout=900)
        if "ThreadSanitizer: unexpected memory mapping" in r.stdout:
            pytest.skip("ThreadSanitizer cannot run under this kernel's address-space layout")
        assert r.returncode == 0 and "Sanitizer" not in r.stdout, f"{san}: {r.stdout[-4000:]}"
        return r.stdout
    return run


def frame(i):
    """(extension, bytes) of frame i: every frame different, five kinds in turn."""
    rng = np.random.default_rng(1000 + i)
    img = rng.integers(0, 256, (H, W), dtype=np.uint8)
    kind = i % 5
    if kind == 0:
        ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])
    elif kind == 1:
        bgr = np.stack([img, np.roll(img, 3, axis=1), 255 - img], axis=-1)
        ok, enc = cv2.imencode(".jpg", bgr, [cv2.IMWRITE_JPEG_QUALITY, 85, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                             cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
    elif kind == 2:
        ok, enc = cv2.imencode(".png", img)
    elif kind == 3:
        ok, enc = cv2.imencode(".png", (img.astype(np.uint16) << 8) | rng.integers(0, 256, (H, W), dtype=np.uint16))
    else:
        ok, enc = cv2.imencode(".pgm", img)
    assert ok
    return (".jpg", ".jpg", ".png", ".png", ".pgm")[kind], enc.tobytes()


def write_sequence(folder, entries, fmt):
    """entries: [(name, bytes)] in name order; fmt: 'folder', or a 'stored' / 'deflated' zip written out of name order."""
    os.makedirs(folder)
    if fmt == "folder":
        os.makedirs(os.path.join(folder, "images"))
        for name, blob in entries:
            with open(os.path.join(folder, "images", name), "wb") as f:
                f.write(blob)
    else:
        method = zipfile.ZIP_STORED if fmt == "stored" else zipfile.ZIP_DEFLATED
        with zipfile.ZipFile(os.path.join(folder, "images.zip"), "w", method) as z:
            for i in np.random.default_rng(5).permutation(len(entries)):
                z.writestr(*entries[i])
    with open(os.path.join(folder, "times.txt"), "w") as t:
        for i in range(len(entries)):
            t.write(f"{i} {i * 0.05:.3f} 1.0\n")
    return folder


def entries(n):
    return [(f"{i:05d}{ext}", blob) for i, (ext, blob) in ((i, frame(i)) for i in range(n))]


@pytest.fixture(scope="module")
def sequences(tmp_path_factory):
    root = tmp_path_factory.mktemp("seqs")
    good = entries(N)
    return {fmt: write_sequence(str(root / fmt), good, fmt) for fmt in ("folder", "stored", "deflated")}


def bad_entry(case):
    good = frame(0)[1]
    if case == "cut_in_headers":
        return ".jpg", good[:good.find(b"\xff\xda") - 20]
    ok, enc = cv2.imencode(".png", np.zeros((H, W - 1), np.uint8))           # wrong_size
    assert ok
    return ".png", enc.tobytes()


@pytest.mark.parametrize("fmt", ["folder", "stored", "deflated"])
def test_ranges_equal_the_frame_reader(harness, sequences, fmt):
    out = harness("range", sequences[fmt], *THREADS)
    assert "range: 24 calls passed" in out


@pytest.mark.parametrize("case", ["cut_in_headers", "wrong_size"])
@pytest.mark.parametrize("fmt", ["folder", "stored", "deflated"])
def test_bad_frame_at_the_start_of_the_third_chunk(harness, tmp_path, fmt, case):
    for threads in (1, 17):
        c = THREADS[threads]
        bad = 2 * c + 1
        seq = entries(4 * c + 2)
        ext, blob = bad_entry(case)
        seq[bad] = (f"{bad:05d}{ext}", blob)
        out = harness("bad", write_sequence(str(tmp_path / f"{threads}"), seq, fmt), bad, threads)
        name = seq[bad][0]
        assert "ERROR: " in out and name in out.split("ERROR: ", 1)[1].splitlines()[0], out[-2000:]
        if case == "wrong_size":
            assert f"expected image dimensions {W} x {H}; found {W - 1} x {H} (image " in out, out[-2000:]


def test_argument_checks(harness, sequences):
    assert "args: 21 cases passed" in harness("args", sequences["stored"])
