"""The GPU JPEG encoder's shared core (csrc/mdc_jpeg_encode.cuh) on the host, without a GPU:
  - built with g++ under AddressSanitizer + UndefinedBehaviorSanitizer into tests/cpp/jpeg_encode_harness.cpp, it must write the bytes
    of the numpy restatement (tests/jpeg_encode_spec.py, itself pinned to cv2) on the whole corpus, from padded rows, and stay inside
    mdc_jpeg_encode_bound on the worst cases;
  - the repository's own host decoder reads the restatement's files to the pixels cv2.imdecode gives;
  - the encoder kernels keep their state in registers; playbackDataset_b200 builds and prints the dataset's header."""
import os
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

import jpeg_encode_spec as E
from conftest import ROOT

CSRC = os.path.join(ROOT, "mono_dataset_code_b200", "csrc")
LIBDIR = os.path.join(ROOT, "mono_dataset_code_b200", "lib")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("jpeg_encode_core")
    exe = str(d / "jpeg_encode_harness")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-I" + os.path.join(ROOT, "include"),
           "-I" + CSRC, os.path.join(ROOT, "tests", "cpp", "jpeg_encode_harness.cpp"), "-o", exe]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        pytest.skip("no sanitizer-enabled g++ here: " + r.stdout[-300:])
    return exe, d


def run(harness, cases, tag, pad=0, fill=0xA5):
    """cases: (name, image, quality) -> {name: (file bytes, bound)}; rows are stored `pad` bytes wider than the image, filled with `fill`."""
    exe, d = harness
    folder = d / tag
    os.makedirs(folder, exist_ok=True)
    lines = []
    for i, (name, img, q) in enumerate(cases):
        h, w = img.shape
        buf = np.full((h, w + pad), fill, np.uint8)
        buf[:, :w] = img
        raw = folder / f"{i}.raw"
        buf.tofile(raw)
        lines.append(f"{raw} {w} {h} {w + pad} {q} {folder / f'{i}.jpg'}")
    (folder / "list").write_text("\n".join(lines) + "\n")
    r = subprocess.run([exe, str(folder / "list")], env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0"), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:]
    rows = r.stdout.splitlines()
    assert len(rows) == len(cases), r.stdout[-3000:]
    out = {}
    for (name, _, _), row in zip(cases, rows):
        path, size, bound = row.split()
        data = open(path, "rb").read()
        assert len(data) == int(size)
        out[name] = (data, int(bound))
    return out


def test_core_equals_spec_on_the_corpus(harness):
    cases = E.corpus()
    got = run(harness, cases, "corpus", pad=0)
    bad = [name for (name, img, q) in cases if got[name][0] != E.encode(img, q)]
    assert not bad, bad[:5]


def test_core_never_reads_row_padding(harness):
    cases = E.corpus(sizes=[(1, 9), (9, 1), (17, 23), (333, 217)], qualities=[50, 95])
    for fill in (0x00, 0xA5):
        got = run(harness, cases, f"pad{fill}", pad=13, fill=fill)
        bad = [name for (name, img, q) in cases if got[name][0] != E.encode(img, q)]
        assert not bad, (fill, bad[:5])


def worst_cases():
    out = []
    for (w, h) in [(8, 8), (9, 9), (64, 48), (333, 217)]:
        y, x = np.mgrid[0:h, 0:w]
        rng = np.random.default_rng(w * h)
        out.append((f"noise_{w}x{h}", rng.integers(0, 256, (h, w), dtype=np.uint8), 100))
        out.append((f"checker_{w}x{h}", (((x + y) & 1) * 255).astype(np.uint8), 100))
        out.append((f"checker2_{w}x{h}", ((((x // 2) + (y // 2)) & 1) * 255).astype(np.uint8), 100))
        # blocks alternating between all 0 and all 255: the largest DC differences, every one coded with size 11
        out.append((f"dcswing_{w}x{h}", ((((x // 8) + (y // 8)) & 1) * 255).astype(np.uint8), 100))
        out.append((f"ffbytes_{w}x{h}", E.frame("ffbytes", w, h), 100))
    return out


def test_worst_cases_stay_within_the_bound(harness):
    cases = worst_cases()
    got = run(harness, cases, "worst")
    for (name, img, q) in cases:
        data, bound = got[name]
        h, w = img.shape
        assert bound == E.encode_bound(w, h), name
        assert data == E.encode(img, q), name
        assert len(data) <= bound, (name, len(data), bound)
    # the bound follows from the tables: 20 bits of DC code + 63 AC codes of at most 26 bits per block, doubled for stuffing
    assert E.encode_bound(8, 8) == 328 + 2 * -(-(20 + 63 * 26) // 8) + 2


def test_host_decoder_reads_the_spec_files_like_opencv(tmp_path):
    cv2 = pytest.importorskip("cv2")
    from mono_dataset_code_b200 import api
    cases = E.corpus(sizes=[(1, 1), (9, 9), (17, 23), (333, 217), (640, 480)], qualities=[1, 50, 95, 100])
    os.makedirs(tmp_path / "images")
    for i, (name, img, q) in enumerate(cases):
        (tmp_path / "images" / f"{i:05d}.jpg").write_bytes(E.encode(img, q))
    seq = api.Sequence(str(tmp_path) + "/")
    assert seq.getNumImages() == len(cases)
    for i, (name, img, q) in enumerate(cases):
        mine = seq.getImageRaw_internal(i)
        ref = cv2.imdecode(np.frombuffer(E.encode(img, q), np.uint8), cv2.IMREAD_GRAYSCALE)
        assert mine is not None and np.array_equal(mine, ref), name


def test_encoder_kernels_do_not_spill():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-I" + os.path.join(ROOT, "include"),
                            "-I" + CSRC, "-c", os.path.join(CSRC, "mdc_jpeg_encode.cu"), "-o", os.path.join(d, "e.o")],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    lines = r.stdout.splitlines()
    for k in ("e1_fdct_quant", "e2_block_bits", "e3_scan_bits", "e4_emit", "e5_stuff"):
        at = [i for i, l in enumerate(lines) if "Function properties" in l and k in l]
        assert at, (k, r.stdout[-2000:])
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in lines[at[0] + 1], (k, lines[at[0] + 1])


def build_tool(tmp_path):
    exe = str(tmp_path / "playbackDataset_b200")
    cmd = ["/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++", "-std=c++11", "-O2", "-Wall", "-I" + os.path.join(ROOT, "include"),
           "-I/usr/local/cuda/include", os.path.join(ROOT, "tools", "playbackDataset_b200.cpp"), "-o", exe, "-L" + LIBDIR, "-lmdc_b200",
           "-L/usr/local/cuda/lib64", "-lcudart", "-lpthread", "-Wl,-rpath," + LIBDIR + ":/usr/local/cuda/lib64"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return exe


def test_playback_tool_builds_and_prints_the_header(tmp_path):
    from mono_dataset_code_b200 import api, synthetic as S
    exe = build_tool(tmp_path)
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 1 and "usage: playbackDataset_b200" in r.stdout
    ds = tmp_path / "ds"
    S.write_dataset_dir(str(ds), 640, 480, 320, 240, "0.4 0.53 0.5 0.5 0")
    os.makedirs(ds / "images")
    S.write_pgm(str(ds / "images" / "00000.pgm"), np.zeros((480, 640), np.uint8))
    r = subprocess.run([exe, str(ds) + "/", "device=0", "threads=3"], cwd=tmp_path, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=60)
    assert r.returncode == 0, r.stdout
    assert f"Playback dataset {ds}/!" in r.stdout
    assert "Rectified Images: 320 x 240. K:" in r.stdout and "Original Images: 640 x 480. omega=" in r.stdout
    assert "Saving" not in r.stdout and not list(tmp_path.glob("*.jpg"))
    fov = api.UndistorterFOV(str(ds / "camera.txt"))
    k_rect = np.array([[float(v) for v in l.split()] for l in r.stdout.split("K:\n")[1].split("\n\n")[0].splitlines()])
    assert np.allclose(k_rect, np.asarray(fov.getK_rect()).reshape(3, 3), rtol=1e-5)
