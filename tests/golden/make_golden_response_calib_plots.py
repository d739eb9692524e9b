"""Generates tests/golden/programs/response_calib_plots.npz from a RUN OF THE REFERENCE PROGRAM (oracle/_ref/responseCalib_ref =
main_responseCalib.cpp compiled unmodified, `make -C oracle ref`), with every Mat it hands to cv::imwrite dumped (MDC_SHIM_DUMP_DIR).

Run where the reference sources are available:   python tests/golden/make_golden_response_calib_plots.py
Contents: the raw frames and exposure times of a small sequence, the program's arguments, and its images: E_bgr [1 + nits, h, w, 3]
(E-0 .. E-nits, BGR), E16 [1 + nits, h, w] and G8 [nits, 256, 256] (G-1 .. G-nits after cv::imwrite's float -> 8-bit conversion),
and the printed ranges.  tests/test_rc_plot_gpu.py runs responseCalib_b200 on the same frames and compares its PNG files."""
import os
import re
import subprocess
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import loader  # noqa: E402
import rc_plot_oracle as O  # noqa: E402
import test_response_calib_reference_program as T  # noqa: E402


def main():
    loader.build("ref")
    nits, leak = 4, 2
    with tempfile.TemporaryDirectory() as tmp:
        seq, work = Path(tmp) / "seq", Path(tmp) / "work"
        seq.mkdir()
        (work / "dump").mkdir(parents=True)
        frames, t = T.write_sequence(seq, np.random.default_rng(4242))
        r = subprocess.run([T.EXE, str(seq) + "/", f"iterations={nits}", f"leakPadding={leak}"], cwd=work,
                           env=dict(os.environ, MDC_SHIM_DUMP_DIR=str(work / "dump")), stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                           text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:]
        dump = lambda name: O.read_dump(work / "dump" / f"{name}.png.raw")[3]      # noqa: E731
        E_bgr = np.stack([dump(f"E-{k}").reshape(T.H, T.W, 3) for k in range(nits + 1)])
        E16 = np.stack([dump(f"E-{k}16").reshape(T.H, T.W) for k in range(nits + 1)])
        G8 = np.stack([O.JS.conv_u8(dump(f"G-{k}")).reshape(256, 256) for k in range(1, nits + 1)])
        ranges = np.array([[float(a), float(b)] for _, a, b in re.findall(r"(Irradiance|Inv\. Response) (\S+) - (\S+)\n", r.stdout)])
    out = os.path.join(ROOT, "tests", "golden", "programs", "response_calib_plots.npz")
    np.savez_compressed(out, frames=frames, exposures=t, w=T.W, h=T.H, nits=nits, leak_padding=leak, E_bgr=E_bgr, E16=E16, G8=G8,
                        printed_ranges=ranges)
    print("wrote", out, frames.shape, E_bgr.shape, G8.shape)


if __name__ == "__main__":
    main()
