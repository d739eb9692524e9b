"""Generates tests/golden/programs/vignette_calib.npz from a RUN OF THE REFERENCE PROGRAM (oracle/_ref/vignetteCalib_ref =
/root/reference/src/main_vignetteCalib.cpp compiled unmodified against the stand-in aruco / cv::findHomography, which reads the
homographies from a file; `make -C oracle ref`).

Run in the authoring container (needs /root/reference):   python tests/golden/make_golden_vignette_program.py
Contents: the frames, times.txt, camera.txt, pcalib.txt and homographies of the sequence of
tests/test_vignette_calib_reference_program.py, the program's arguments, vignetteCalibResult/log.txt, and the three images it
hands to cv::imwrite (vignette.png, vignetteSmoothed.png, plane.png as the BGR Mat).  The GPU test runs tools/vignetteCalib_b200
on the same sequence and compares (tests/test_vignette_calib_tool.py).
"""
import os
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import loader  # noqa: E402
import test_vignette_calib_reference_program as V  # noqa: E402


def main():
    loader.build("ref")
    out_dir = os.path.join(ROOT, "tests", "golden", "programs")
    os.makedirs(out_dir, exist_ok=True)
    its = 8
    with tempfile.TemporaryDirectory() as tmp:
        seq, work = Path(tmp) / "seq", Path(tmp) / "work"
        seq.mkdir()
        (work / "dump").mkdir(parents=True)
        files, frames, expo, Hs = V.make_sequence(seq, np.random.default_rng(77))
        env = dict(os.environ, MDC_SHIM_DUMP_DIR=str(work / "dump"), MDC_SHIM_HOMOGRAPHIES=str(seq / "homographies.txt"))
        r = subprocess.run([V.EXE, str(seq) + "/", f"iterations={its}", f"patternX={V.GW}", f"patternY={V.GH}"], cwd=work, env=env,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-3000:]
        log = np.loadtxt(work / "vignetteCalibResult" / "log.txt", ndmin=2)
        dumps = {}
        for name, shape, typ, dt in (("vignette", (V.HI, V.WI), 2, np.uint16), ("vignetteSmoothed", (V.HI, V.WI), 2, np.uint16),
                                     ("plane", (V.GH, V.GW, 3), 16, np.uint8)):
            rows, cols, t, px = V.read_dump(work / "dump" / f"{name}.png.raw")
            assert (rows, cols, t) == (shape[0], shape[1], typ)
            dumps[name] = px.view(dt).reshape(shape)
        text = {k: open(seq / f).read() for k, f in (("camera_txt", "camera.txt"), ("pcalib_txt", "pcalib.txt"), ("times_txt", "times.txt"),
                                                      ("homographies_txt", "homographies.txt"))}
    np.savez_compressed(os.path.join(out_dir, "vignette_calib.npz"), frames=frames, exposures=expo, homographies=Hs, wI=V.WI, hI=V.HI,
                        gw=V.GW, gh=V.GH, iterations=its, log=log, vignette_png=dumps["vignette"],
                        vignette_smoothed_png=dumps["vignetteSmoothed"], plane_png_bgr=dumps["plane"],
                        **{k: np.array(v) for k, v in text.items()})
    print("wrote vignette_calib.npz:", frames.shape, "log", log[:, 2:])


if __name__ == "__main__":
    main()
