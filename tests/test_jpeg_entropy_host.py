"""The GPU JPEG decoder's core (csrc/mdc_jpeg_entropy.cuh: segment entropy decoding and the inverse DCT) built with the host compiler into
tests/cpp/jpeg_entropy_harness.cpp, under AddressSanitizer + UndefinedBehaviorSanitizer: header parse and restart split as
mdc_jpeg_decode_device does them, each segment decoded from a heap block of exactly its bytes into a coefficient plane of its own, then
mdcj::idct_block.  It must give the host decoder's bytes on every file the host decodes, and the host decoder's rejection and message
on every file it rejects, and never read outside a segment or write outside the segment's blocks.  No GPU needed."""
import os
import subprocess

import pytest

from conftest import ROOT

cv2 = pytest.importorskip("cv2")
import jpeg_cases as J  # noqa: E402

CSRC = os.path.join(ROOT, "mono_dataset_code_b200", "csrc")


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    d = tmp_path_factory.mktemp("jpeg_core")
    exe = str(d / "jpeg_entropy_harness")
    cmd = ["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-I" + os.path.join(ROOT, "include"),
           "-I" + CSRC, os.path.join(ROOT, "tests", "cpp", "jpeg_entropy_harness.cpp"), os.path.join(CSRC, "mdc_jpeg.cpp"), "-lz", "-o", exe]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        pytest.skip("no sanitizer-enabled g++ here: " + r.stdout[-300:])
    return exe, d


def run(harness, blobs, tag):
    """-> list of (host_ok, core_ok, same, line).  The host decoder uses its 64-bit scalar transform (MDC_JPEG_SCALAR=1): it is what
    the core's transform restates, and the AVX2 one may differ from it on corrupt streams only."""
    exe, d = harness
    folder = d / tag
    os.makedirs(folder, exist_ok=True)
    paths = []
    for i, b in enumerate(blobs):
        p = folder / f"{i:05d}.jpg"
        p.write_bytes(b)
        paths.append(str(p))
    (folder / "list").write_text("\n".join(paths) + "\n")
    env = dict(os.environ, MDC_JPEG_SCALAR="1", ASAN_OPTIONS="detect_leaks=0")
    r = subprocess.run([exe, str(folder / "list")], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:]
    rows = []
    for line in r.stdout.splitlines():
        f = line.split(" | ")[0].split()
        rows.append((f[1] == "host=1", f[2] == "core=1", f[3] == "same=1", line))
    assert len(rows) == len(blobs), r.stdout[-3000:]
    return rows


def test_core_equals_host_decoder_on_the_corpus(harness):
    files = J.corpus()
    rows = run(harness, [b for (_, _, b) in files], "corpus")
    assert all(h for (h, _, _, _) in rows), [l for (h, _, _, l) in rows if not h][:5]
    bad = [l for (_, _, same, l) in rows if not same]
    assert not bad, bad[:5]


def test_core_equals_host_decoder_on_cut_scans(harness):
    """A scan cut anywhere: both read zero bits from the cut on, or both miss a restart marker."""
    cuts = J.scan_cuts(J.corpus())
    rows = run(harness, [b for (_, _, b) in cuts], "cuts")
    bad = [l for (_, _, same, l) in rows if not same]
    assert not bad, bad[:5]
    assert sum(1 for (h, _, _, _) in rows if h) > len(rows) // 3          # most cuts still decode


def test_damaged_streams_never_trip_the_sanitizers_and_match_the_host(harness):
    """decoder_fuzz.cpp's damage modes, seeded: the same accept / reject decision and message as the host, the same bytes where
    accepted, no read outside a segment, no write outside its blocks."""
    dmg = J.damaged_set()
    rows = run(harness, [b for (_, b) in dmg], "damaged")
    bad = [l for (_, _, same, l) in rows if not same]
    assert not bad, bad[:5]
    assert sum(1 for (h, _, _, _) in rows if h) > 100


def test_j1_keeps_its_state_in_registers():
    """The entropy-decode kernel has no local-memory spills (nvcc -Xptxas -v, sm_90a)."""
    import shutil
    import tempfile
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("no nvcc")
    with tempfile.TemporaryDirectory() as d:
        r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-I" + os.path.join(ROOT, "include"),
                            "-I" + CSRC, "-c", os.path.join(CSRC, "mdc_jpeg_gpu.cu"), "-o", os.path.join(d, "j.o")],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-2000:]
    lines = r.stdout.splitlines()
    at = [i for i, l in enumerate(lines) if "Function properties" in l and "j1_entropy_decode" in l]
    assert at, r.stdout[-2000:]
    assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in lines[at[0] + 1], lines[at[0] + 1]
