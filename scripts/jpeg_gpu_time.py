"""Decode-inclusive rates of the sequence feeds on the zip bench.py's c4 leg builds (1920x1080, quality 90, 128 distinct payloads cycled
over 1024 stored entries), getImage with rectify + gamma + vignette, 512 frames per call:
  decode_only           the host decoder alone: mdc_seq_read_gray8 over the call's frames on `threads` threads
  host_feed             mdc_seq_prepare: host decode -> H2D -> K1 -> D2H into pinned host floats
  device_feed           mdc_seq_prepare_device: host parse -> H2D -> J1 -> J2 -> K1 into device floats
The three are alternated and repeated in one process, after a first call of each feed whose outputs are compared bit for bit.  J1, J2
and K1 times per call come from a torch.profiler run of its own.  Prints one JSON line with the card's name, power limit and max SM
clock.  usage: python scripts/jpeg_gpu_time.py [--threads N] [--reps R]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time
import zipfile
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import cv2
    import torch
    from mono_dataset_code_b200 import _lib, api, synthetic as S
    lib = _lib.lib
    W, H, K, UNIQUE, CALL, FLAGS = 1920, 1080, 1024, 128, 512, 7
    root = tempfile.mkdtemp(prefix="mdc_jpeg_gpu_time_")
    S.write_dataset_dir(root, W, H, W, H, "crop")
    yy, xx = np.mgrid[0:H, 0:W]
    rng = np.random.default_rng(11)
    blobs = []
    for i in range(UNIQUE):        # the scene of bench.py's c4 leg
        img = (xx * (150.0 / W) + yy * (60.0 / H) + 40 * np.sin((xx + 13 * i) * 0.05) * np.cos((yy - 7 * i) * 0.04)
               + ((xx // 64 + yy // 64 + i) % 2) * 30 + rng.normal(0, 1.5, (H, W)))
        blobs.append(cv2.imencode(".jpg", np.clip(np.rint(img), 0, 255).astype(np.uint8), [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes())
    with zipfile.ZipFile(os.path.join(root, "images.zip"), "w", zipfile.ZIP_STORED) as z:
        for i in range(K):
            z.writestr(f"{i:05d}.jpg", blobs[i % UNIQUE])
    with open(os.path.join(root, "times.txt"), "w") as f:
        for i in range(K):
            f.write(f"{i} {i * 0.05:.3f} 1.0\n")
    fov = api.UndistorterFOV(os.path.join(root, "camera.txt"))
    photo = api.PhotometricUndistorter(os.path.join(root, "pcalib.txt"), os.path.join(root, "vignette.png"), W, H)
    ctx = api.Context(fov, photo, 0)
    seq = api.Sequence(root + "/")
    n_px = W * H
    h_out = C.c_void_p()
    _lib.check(lib.mdc_host_alloc(C.byref(h_out), CALL * n_px * 4), "mdc_host_alloc")
    h_ptrs = (C.c_void_p * 1)(h_out.value)
    d_out = torch.empty((CALL, n_px), dtype=torch.float32, device="cuda:0")
    d_ptrs = (C.c_void_p * 1)(d_out.data_ptr())

    def host_feed(first):
        _lib.check(lib.mdc_seq_prepare(ctx._h, seq._h, first, CALL, FLAGS, h_ptrs, 1, args.threads), "mdc_seq_prepare")

    def device_feed(first):
        _lib.check(lib.mdc_seq_prepare_device(ctx._h, seq._h, first, CALL, FLAGS, d_ptrs, 1, args.threads, None), "mdc_seq_prepare_device")

    def decode_only(first):
        def one(i):
            buf = np.empty(n_px, np.uint8)
            w, h = C.c_int(), C.c_int()
            for k in range(i, CALL, args.threads):
                lib.mdc_seq_read_gray8(seq._h, first + k, buf.ctypes.data_as(C.c_void_p), buf.size, C.byref(w), C.byref(h))
        with ThreadPoolExecutor(args.threads) as ex:
            list(ex.map(one, range(args.threads)))

    def rate(fn, first):
        t0 = time.perf_counter()
        fn(first)
        torch.cuda.synchronize()
        return CALL / (time.perf_counter() - t0)

    # same output: device feed vs host feed on the first call
    host_feed(0)
    device_feed(0)
    host = np.ctypeslib.as_array(C.cast(h_out, C.POINTER(C.c_uint32)), (CALL * n_px,))
    identical = bool(np.array_equal(host, d_out.view(torch.int32).cpu().numpy().reshape(-1).view(np.uint32)))
    runs = {"decode_only": [], "host_feed": [], "device_feed": []}
    for r in range(args.reps):              # alternated, warm
        first = (r * CALL) % K
        runs["decode_only"].append(rate(decode_only, first))
        runs["host_feed"].append(rate(host_feed, first))
        runs["device_feed"].append(rate(device_feed, first))
    # J1 / J2 kernel times: a profiled call of its own
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        device_feed(0)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        for tag in ("j1_entropy_decode", "j2_idct", "fused"):
            if tag in e.key:
                kern.setdefault(tag, [0.0, 0])
                kern[tag][0] += e.device_time_total / 1e3 if hasattr(e, "device_time_total") else e.cuda_time_total / 1e3
                kern[tag][1] += e.count
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({
        "card": smi, "frames_per_call": CALL, "threads": args.threads, "jpeg_mean_bytes": float(np.mean([len(b) for b in blobs])),
        "identical_output": identical,
        "fps": {k: [round(v, 1) for v in vs] for k, vs in runs.items()},
        "fps_median": {k: round(float(np.median(vs)), 1) for k, vs in runs.items()},
        "device_over_host_feed": round(float(np.median(runs["device_feed"]) / np.median(runs["host_feed"])), 2),
        "kernel_ms_per_call": {k: round(v[0], 2) for k, v in kern.items()}, "kernel_launches": {k: v[1] for k, v in kern.items()},
    }))
    lib.mdc_host_free(h_out)


if __name__ == "__main__":
    main()
