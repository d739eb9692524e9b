"""How long the calibration programs take to load their frames, on a synthetic calibration sequence: 1000 frames of 1280x1024, baseline
JPEG at quality 90 in a stored images.zip, with exposure times in times.txt.  Over the same ids (every frame), alternated and repeated
`--reps` times in one process, medians reported:
  host_loop        the load the programs used to do: mdc_seq_read_gray8 on one thread (a size query, then the read, per frame) into a
                   host stack, then one H2D copy of the stack
  device_call      mdc_seq_read_gray8_device into device memory (threads = 0: the default count)
The two stacks are compared byte for byte first.  Then the wall time, from start to exit, of responseCalib_b200 (default arguments)
and vignetteCalib_b200 (homographies=detect; the synthetic frames show no marker, so this times the load, rectification, threshold
and detection over every frame, and the loop runs on no frame), built from tools/ and, with --compare-tools DIR, from the sources in
DIR as well, alternated.  Prints one JSON line with the card's name, power limit and the host's CPUs; --out FILE also writes it there.
usage: python scripts/seq_read_device_time.py [--frames N] [--reps R] [--compare-tools DIR] [--out FILE]"""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def build_tool(src, exe):
    libdir = os.path.join(ROOT, "mono_dataset_code_b200", "lib")
    subprocess.run(["g++", "-std=c++11", "-O2", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include", src, "-o", exe,
                    "-L" + libdir, "-lmdc_b200", "-L/usr/local/cuda/lib64", "-lcudart", "-lz", "-Wl,-rpath," + libdir + ":/usr/local/cuda/lib64"],
                   check=True)


def wall(cmd, cwd):
    t0 = time.perf_counter()
    r = subprocess.run(cmd, cwd=cwd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    dt = time.perf_counter() - t0
    if r.returncode != 0:
        raise RuntimeError(f"{cmd[0]} exited with {r.returncode}: {r.stdout[-2000:]}")
    return dt, [l for l in r.stdout.splitlines() if "loaded" in l or "found exactly" in l]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--compare-tools", default=None, help="a directory holding other responseCalib_b200.cpp / vignetteCalib_b200.cpp")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import cv2
    import torch
    from mono_dataset_code_b200 import _lib, api, synthetic as S
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    lib = _lib.lib
    W, H, N = 1280, 1024, args.frames
    root = tempfile.mkdtemp(prefix="mdc_seq_read_time_")
    try:
        seq_dir = os.path.join(root, "seq")
        S.write_dataset_dir(seq_dir, W, H, 640, 480, "0.4 0.53 0.5 0.5 0")
        yy, xx = np.mgrid[0:H, 0:W]
        rng = np.random.default_rng(5)
        base = xx * (120.0 / W) + yy * (60.0 / H) + 25 * np.sin(xx * 0.03) * np.cos(yy * 0.02)
        t_enc = time.perf_counter()
        with zipfile.ZipFile(os.path.join(seq_dir, "images.zip"), "w", zipfile.ZIP_STORED) as z, open(os.path.join(seq_dir, "times.txt"), "w") as t:
            for i in range(N):
                e = 0.2 + 4.8 * ((i * 37) % N) / N                       # exposures over a 24x range, shuffled
                img = np.clip((base + 40) * e * 0.5 + rng.normal(0, 2, (H, W)), 0, 255).astype(np.uint8)
                z.writestr(f"{i:05d}.jpg", cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes())
                t.write(f"{i} {i * 0.05:.6f} {e:.6f}\n")
        t_enc = time.perf_counter() - t_enc
        seq = api.Sequence(seq_dir + "/")
        ctx = api.Context(None, None, 0)
        ids = np.arange(N, dtype=np.int32)
        host = np.empty((N, H, W), np.uint8)
        d_host = torch.empty((N, H, W), dtype=torch.uint8, device="cuda:0")
        d_dev = torch.empty((N, H, W), dtype=torch.uint8, device="cuda:0")

        def host_loop():
            w, h = C.c_int(), C.c_int()
            t0 = time.perf_counter()
            for k in range(N):
                assert lib.mdc_seq_read_gray8(seq._h, int(ids[k]), None, 0, C.byref(w), C.byref(h)) == 0
                assert lib.mdc_seq_read_gray8(seq._h, int(ids[k]), host[k].ctypes.data, W * H, C.byref(w), C.byref(h)) == 0
            d_host.copy_(torch.from_numpy(host))
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        def device_call():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            _, status, _ = seq.read_gray8_device(ctx, ids, W, H, row_pitch=W, out=d_dev)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            assert (status == 0).all()
            return dt

        warm = [device_call(), host_loop()]
        assert torch.equal(d_host, d_dev), "the two loads differ"
        times = {"host_loop": [], "device_call": []}
        for _ in range(args.reps):
            times["device_call"].append(device_call())
            times["host_loop"].append(host_loop())
        del d_host, d_dev
        seq.close()
        ctx.close()
        torch.cuda.empty_cache()

        builds = {"tools": os.path.join(ROOT, "tools")}
        if args.compare_tools:
            builds["compare"] = os.path.abspath(args.compare_tools)
        exes = {}
        for tag, d in builds.items():
            for name in ("responseCalib_b200", "vignetteCalib_b200"):
                exes[(tag, name)] = os.path.join(root, f"{tag}_{name}")
                build_tool(os.path.join(d, name + ".cpp"), exes[(tag, name)])
        tool_args = {"responseCalib_b200": [], "vignetteCalib_b200": ["homographies=detect"]}
        tool_times, tool_lines = {}, {}
        for _ in range(args.reps):
            for name in tool_args:
                for tag in builds:
                    work = os.path.join(root, f"work_{tag}_{name}")
                    os.makedirs(work, exist_ok=True)
                    dt, lines = wall([exes[(tag, name)], seq_dir + "/"] + tool_args[name], work)
                    tool_times.setdefault(f"{name}[{tag}]", []).append(dt)
                    tool_lines[f"{name}[{tag}]"] = lines

        smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                             text=True).stdout.strip().splitlines()
        res = {
            "gpu": smi[0] if smi else torch.cuda.get_device_name(0),
            "host_cpus": os.cpu_count(), "cpus_allowed": len(os.sched_getaffinity(0)),
            "frames": N, "size": [W, H], "quality": 90, "zip_mb": round(os.path.getsize(os.path.join(seq_dir, "images.zip")) / 2**20, 1),
            "encode_s": round(t_enc, 1), "first_calls_s": [round(x, 3) for x in warm],
            "load_s": {k: [round(x, 3) for x in v] for k, v in times.items()},
            "load_median_s": {k: round(float(np.median(v)), 3) for k, v in times.items()},
            "tool_wall_s": {k: [round(x, 3) for x in v] for k, v in tool_times.items()},
            "tool_wall_median_s": {k: round(float(np.median(v)), 3) for k, v in tool_times.items()},
            "tool_lines": tool_lines,
        }
        res["load_speedup"] = round(res["load_median_s"]["host_loop"] / res["load_median_s"]["device_call"], 2)
        line = json.dumps(res)
        print(line)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "w") as f:
                f.write(line + "\n")
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
