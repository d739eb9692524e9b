"""Time responseCalib's result images: the plot kernels, the host PNG writer, and responseCalib_b200 with and without plots.

  python scripts/rc_plot_time.py [--reps 15] [--launches 50] [--frames 1000] [--its 10] [--runs 2] [--out FILE.json]

  kernels  per size (1280x1024, 1920x1080) on an irradiance from a calibration-like range with a few NaN: CUDA events around
           `launches` back-to-back launches of mdc_rc_plot_e_range (both of its kernels), of mdc_rc_plot_e_map and of mdc_rc_plot_g,
           the three interleaved, `reps` times; the median per call.
  png      mdc_png_write of the E-k.png (BGR), E-k16.png and G-k.png images of one step, one host thread, median over `reps`.
  tool     wall time of responseCalib_b200 on `frames` PGM frames of 1024 x 1024 (an exposure sweep of a fixed scene through a
           gamma response), `its` iterations, plots=0 and plots=1 alternated `runs` times each; checks that pcalib.txt and log.txt
           are the same.
Records the card's name and power limit and the host's CPU count.  Needs a GPU; prints one JSON document."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def time_kernels(ctx, torch, reps, launches):
    rng = np.random.default_rng(1)
    out = {}
    for w, h in [(1280, 1024), (1920, 1080)]:
        E = rng.uniform(4.0, 900.0, w * h)
        E[rng.random(w * h) < 0.001] = np.nan
        dE = torch.from_numpy(E).cuda()
        rng4 = ctx.rc_plot_e_range(dE)
        bgr, e16 = ctx.rc_plot_e_map(dE, rng4)
        G = torch.from_numpy(np.linspace(0, 255, 256) ** 1.1).cuda()
        calls = {"range": lambda: ctx.rc_plot_e_range(dE, rng4), "map": lambda: ctx.rc_plot_e_map(dE, rng4, bgr, e16),
                 "plot_g": lambda: ctx.rc_plot_g(G)}
        for f in calls.values():                      # warm-up
            f()
        times = {k: [] for k in calls}
        for _ in range(reps):
            for k, f in calls.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                a.record()
                for _ in range(launches):
                    f()
                b.record()
                b.synchronize()
                times[k].append(a.elapsed_time(b) * 1e3 / launches)
        out[f"{w}x{h}"] = {k: {"median_us": statistics.median(v), "min_us": min(v), "max_us": max(v)} for k, v in times.items()}
        out[f"{w}x{h}"]["map_bytes"] = w * h * (8 + 3 + 2)
    return out


def time_png(api, reps):
    import rc_plot_oracle as O
    rng = np.random.default_rng(2)
    out = {}
    for w, h in [(1280, 1024), (1920, 1080)]:
        E = np.exp(rng.normal(4, 1, (h, w))) + np.linspace(0, 50, w)[None, :]
        bgr, e16, _ = O.plot_e(E)
        g8, _ = O.plot_g(np.linspace(0, 255, 256) ** 1.1)
        imgs = {"E-k.png": bgr.reshape(h, w, 3), "E-k16.png": e16.reshape(h, w), "G-k.png": g8}
        res = {}
        with tempfile.TemporaryDirectory() as d:
            for name, img in imgs.items():
                ts = []
                for _ in range(reps):
                    t0 = time.perf_counter()
                    api.png_write(os.path.join(d, name), img)
                    ts.append((time.perf_counter() - t0) * 1e3)
                res[name] = {"median_ms": statistics.median(ts), "bytes": os.path.getsize(os.path.join(d, name))}
        out[f"{w}x{h}"] = res
    return out


def time_tool(frames, its, runs):
    from mono_dataset_code_b200 import synthetic as S
    from test_tools_cpp import build_tool
    from pathlib import Path
    w = h = 1024
    res = {"frames": frames, "size": f"{w}x{h}", "iterations": its, "plots0_s": [], "plots1_s": []}
    with tempfile.TemporaryDirectory() as d:
        d = Path(d)
        exe = build_tool(d)
        seq = d / "seq"
        os.makedirs(seq / "images")
        rng = np.random.default_rng(3)
        scene = rng.uniform(4.0, 90.0, w * h)
        times = np.geomspace(0.2, 6.0, frames)
        noise = rng.normal(0, 1.0, w * h)
        with open(seq / "times.txt", "w") as t:
            for i, ti in enumerate(times):
                img = np.clip(np.rint(255.0 * (np.clip(scene * ti, 0, 255.0) / 255.0) ** (1 / 2.2) + np.roll(noise, 7919 * i)), 0, 255)
                S.write_pgm(str(seq / "images" / f"{i:05d}.pgm"), img.astype(np.uint8).reshape(h, w))
                t.write(f"{i} {100.0 + 0.05 * i:.6f} {ti:.7f}\n")
        outputs = {}
        for r in range(runs):
            for plots in (0, 1):
                work = d / f"work{plots}_{r}"
                work.mkdir()
                t0 = time.perf_counter()
                p = subprocess.run([exe, str(seq) + "/", f"iterations={its}", f"plots={plots}"], cwd=work, stdout=subprocess.PIPE,
                                   stderr=subprocess.STDOUT, text=True)
                res[f"plots{plots}_s"].append(time.perf_counter() - t0)
                assert p.returncode == 0, p.stdout[-2000:]
                outputs.setdefault(plots, [(work / "photoCalibResult" / n).read_bytes() for n in ("pcalib.txt", "log.txt")])
                res["png_files"] = len([n for n in os.listdir(work / "photoCalibResult") if n.endswith(".png")]) if plots else res.get("png_files")
        res["pcalib_and_log_identical"] = outputs[0] == outputs[1]
    for k in ("plots0_s", "plots1_s"):
        res[k.replace("_s", "_median_s")] = statistics.median(res[k])
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=15)
    ap.add_argument("--launches", type=int, default=50)
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--its", type=int, default=10)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    from mono_dataset_code_b200 import api
    ctx = api.Context(None, None, 0)
    doc = {"card": card(), "host_cpus": os.cpu_count(), "kernels": time_kernels(ctx, torch, a.reps, a.launches), "png": time_png(api, a.reps)}
    if a.frames > 0:
        doc["tool"] = time_tool(a.frames, a.its, a.runs)
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        open(a.out, "w").write(s)


if __name__ == "__main__":
    main()
