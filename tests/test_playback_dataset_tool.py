"""tools/playbackDataset_b200.cpp in save mode on the GPU: every frame of a JPEG zip sequence written as %05d.jpg, each file the bytes
cv2.imencode('.jpg') writes for the rectified float image (mdc_seq_prepare's getImage(i, true, false, false, false)); with an
unreadable frame, status 1 after the files of the chunks before it."""
import os
import subprocess
import zipfile

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")
cv2 = pytest.importorskip("cv2")
if not torch.cuda.is_available():
    pytest.skip("no CUDA device", allow_module_level=True)

from mono_dataset_code_b200 import api, synthetic as S  # noqa: E402
from test_jpeg_encode_core import build_tool  # noqa: E402

IW, IH = 640, 480
N = 40


def make_sequence(folder, replace=None):
    S.write_dataset_dir(str(folder), IW, IH, IW, IH, "crop")
    kinds = ["uniform", "speckle", "gradient"]
    with zipfile.ZipFile(folder / "images.zip", "w", zipfile.ZIP_DEFLATED) as z:
        for i in range(N):
            blob = cv2.imencode(".jpg", S.frame(i, IW, IH, kinds[i % 3]).reshape(IH, IW), [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes()
            if replace and i in replace:
                blob = replace[i]
            z.writestr(f"{i:05d}.jpg", blob)
    with open(folder / "times.txt", "w") as t:
        for i in range(N):
            t.write(f"{i} {100.0 + 0.05 * i:.6f} {10.0 + i:.6f}\n")
    return str(folder) + "/"


def level0_f32(ds):
    fov = api.UndistorterFOV(ds + "camera.txt")
    ctx = api.Context(fov, api.PhotometricUndistorter(ds + "pcalib.txt", ds + "vignette.png", IW, IH), 0)
    seq = api.Sequence(ds)
    ow, oh = fov.getOutputDims()
    return seq.prepare(ctx, [(ow, oh)], 0, N, True, False, False, False)[0].reshape(N, oh, ow)


def test_save_mode_writes_opencv_files(tmp_path):
    ds = make_sequence(tmp_path / "seq")
    exe = build_tool(tmp_path)
    work = tmp_path / "work"
    work.mkdir()
    r = subprocess.run([exe, ds, "save", "threads=1"], cwd=work, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "Saving undistorted Dataset to here!" in r.stdout
    assert sorted(os.listdir(work)) == [f"{i:05d}.jpg" for i in range(N)]
    ref = level0_f32(ds)
    for i in range(N):
        exp = cv2.imencode(".jpg", ref[i])[1].tobytes()
        assert (work / f"{i:05d}.jpg").read_bytes() == exp, i


def test_unreadable_frame_stops_after_the_chunks_before_it(tmp_path):
    ds = make_sequence(tmp_path / "seq", replace={35: b"\xff\xd8\xff\xdb\x00"})
    exe = build_tool(tmp_path)
    work = tmp_path / "work"
    work.mkdir()
    r = subprocess.run([exe, ds, "save", "threads=1"], cwd=work, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 1, r.stdout[-3000:]
    assert "00035.jpg" in r.stdout
    # threads=1: chunks of 32 frames; the frame sits in the second chunk, so exactly the first chunk's files exist
    assert sorted(os.listdir(work)) == [f"{i:05d}.jpg" for i in range(32)]
