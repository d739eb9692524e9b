"""The plain-C restatement of plotE / plotG (tests/cpp/rc_plot_oracle.c, the oracle of the GPU plots) against the REFERENCE PROGRAM:
main_responseCalib.cpp compiled unmodified (oracle/_ref/responseCalib_ref) runs on two sequences and dumps every Mat it hands to
cv::imwrite.  The restatement, applied to the E and G of the restated loop (oracle/port) at each step, must give every E-k.png,
E-k16.png and G-k.png pixel for pixel (G-k after cv::imwrite's float -> 8-bit conversion of the dumped float image, and the float
image itself bit for bit), and the "Irradiance" / "Inv. Response" lines the program printed."""
import os
import re
import subprocess

import numpy as np
import pytest

import rc_plot_oracle as O
import test_response_calib_reference_program as T
from oracle.loader import PortOracle

pytestmark = pytest.mark.skipif(not os.path.exists(T.EXE), reason="oracle/_ref/responseCalib_ref not built (needs /root/reference)")


def run_reference(tmp_path, seed, nits, leak):
    seq, work = tmp_path / "seq", tmp_path / "work"
    seq.mkdir()
    (work / "dump").mkdir(parents=True)
    frames, t = T.write_sequence(seq, np.random.default_rng(seed))
    env = dict(os.environ, MDC_SHIM_DUMP_DIR=str(work / "dump"))
    r = subprocess.run([T.EXE, str(seq) + "/", f"iterations={nits}", f"leakPadding={leak}"], cwd=work, env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:]
    return frames, t, work / "dump", r.stdout


def restated_steps(frames, t, nits, leak):
    """[(name, kind, E or G)] in the order the reference plots: E-0, then G-k and E-k for k = 1..nits"""
    port = PortOracle()
    data = np.stack([port.leak_padding(f, T.W, T.H, leak) for f in frames])
    E = port.einit(data)
    steps = [("E-0", "E", E.copy())]
    for it in range(nits):
        G = port.gstep(data, t, E)
        steps.append((f"G-{it + 1}", "G", G.copy()))
        E = port.estep(data, t, G)
        steps.append((f"E-{it + 1}", "E", E.copy()))
        port.rescale(E, G)
    return steps


@pytest.mark.parametrize("seed,nits,leak", [(104, 4, 2), (203, 3, 0)])
def test_restated_plots_reproduce_the_reference_programs_images(tmp_path, seed, nits, leak):
    frames, t, dump, stdout = run_reference(tmp_path, seed, nits, leak)
    printed = re.findall(r"(Irradiance|Inv\. Response) (\S+) - (\S+)\n", stdout)
    steps = restated_steps(frames, t, nits, leak)
    assert len(printed) == len(steps) == 1 + 2 * nits
    for (name, kind, v), (label, lo, hi) in zip(steps, printed):
        if kind == "E":
            bgr, e16, rng = O.plot_e(v)
            rows, cols, typ, px = O.read_dump(dump / f"{name}.png.raw")
            assert (rows, cols, typ) == (T.H, T.W, 16) and np.array_equal(px.reshape(-1, 3), bgr), name
            rows, cols, typ, px = O.read_dump(dump / f"{name}16.png.raw")
            assert (rows, cols, typ) == (T.H, T.W, 2) and np.array_equal(px, e16), name
            assert (label, lo, hi) == ("Irradiance", f"{rng[2]:f}", f"{rng[3]:f}"), name
            assert len(np.unique(bgr, axis=0)) > 20 and len(np.unique(e16)) > 100, name          # the maps are not degenerate
        else:
            f, mm = O.plot_g_float(v)
            rows, cols, typ, px = O.read_dump(dump / f"{name}.png.raw")
            assert (rows, cols, typ) == (256, 256, 5), name
            assert np.array_equal(px.view(np.uint32), f.reshape(-1).view(np.uint32)), name
            assert np.array_equal(O.JS.conv_u8(px), O.plot_g(v)[0].reshape(-1)), name
            assert (label, lo, hi) == ("Inv. Response", f"{mm[0]:f}", f"{mm[1]:f}"), name
    assert sorted(os.listdir(dump)) == sorted([f"{n}.png.raw" for n, _, _ in steps] + [f"{n}16.png.raw" for n, k, _ in steps if k == "E"])
