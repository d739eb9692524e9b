"""Timing of vignetteCalib's marker detection on a synthetic 1280x1024 sequence (one marker per frame, noise), on the GPU:

  threshold   mdc_marker_threshold: ms per frame (CUDA events around batches of 256 rectified frames)
  detect      mdc_marker_detect on the host: ms per frame on one thread
  end-to-end  raw frames -> mdc_prepare_batch (MDC_RECTIFY) -> mdc_marker_threshold -> D2H -> mdc_marker_detect on N threads ->
              mdc_marker_homography: frames/s, for each N
  cv2 spec    tests/aruco_spec.py (adaptiveThreshold + steps 4-7 over cv2), ms per frame, if cv2 is installed

    python scripts/marker_time.py [--frames 256] [--threads 1,8,32] [--out DIR]

Prints one JSON line with the GPU's name and power limit next to the numbers."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import aruco_spec as A  # noqa: E402
from mono_dataset_code_b200 import api, synthetic as S  # noqa: E402

W, H = 1280, 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--threads", default="1,8,32")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    n = a.frames
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as d:
        S.write_dataset_dir(d, W, H, W, H, "crop")
        fov = api.UndistorterFOV(os.path.join(d, "camera.txt"))
    ctx = api.Context(fov, None, 0)
    raw = np.empty((n, H, W), np.uint8)
    for i in range(n):
        scene = A.render(W, H, [(A.marker_bits(i % 1024), A.square(640 + 40 * np.cos(i), 512 + 30 * np.sin(i), 260, 7 * i))], ss=1)
        raw[i] = np.clip(scene + rng.normal(0, 6, scene.shape), 0, 255)
    d_raw = torch.from_numpy(raw.reshape(n, -1)).cuda()
    rect = torch.empty((n, H * W), dtype=torch.float32, device="cuda")
    ctx.prepare_batch(d_raw, api.RECTIFY, [rect])
    rect3 = rect.view(n, H, W)
    grey, mask = ctx.marker_threshold(rect3)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 20
    e0.record()
    for _ in range(reps):
        ctx.marker_threshold(rect3, grey, mask)
    e1.record()
    torch.cuda.synchronize()
    thr_ms = e0.elapsed_time(e1) / (reps * n)
    g, m = grey.cpu().numpy(), mask.cpu().numpy()

    t = time.perf_counter()
    found = sum(len(api.marker_detect(g[i], m[i])) == 1 for i in range(n))
    det_ms = (time.perf_counter() - t) * 1e3 / n

    def host(i, gg, mm):
        ms = api.marker_detect(gg[i], mm[i])
        return api.marker_homography(ms[0][1]) if len(ms) == 1 else None

    e2e = {}
    chunk = 64
    for nt in [int(x) for x in a.threads.split(",")]:
        with ThreadPoolExecutor(nt) as pool:
            torch.cuda.synchronize()
            t = time.perf_counter()
            for f0 in range(0, n, chunk):
                fr = torch.from_numpy(raw[f0:f0 + chunk].reshape(-1, H * W)).cuda()
                k = fr.shape[0]
                r = torch.empty((k, H * W), dtype=torch.float32, device="cuda")
                ctx.prepare_batch(fr, api.RECTIFY, [r])
                gg, mm = ctx.marker_threshold(r.view(k, H, W))
                gg, mm = gg.cpu().numpy(), mm.cpu().numpy()
                list(pool.map(lambda i: host(i, gg, mm), range(k)))
            e2e[nt] = n / (time.perf_counter() - t)

    cv2_ms = None
    try:
        import cv2  # noqa: F401
        k = min(n, 16)
        t = time.perf_counter()
        for i in range(k):
            gi = A.grey_u8(rect3[i].cpu().numpy())
            A.detect_cv2(gi, A.threshold_cv2(gi))
        cv2_ms = (time.perf_counter() - t) * 1e3 / k
    except ImportError:
        pass
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    res = dict(gpu=smi, frames=n, size=f"{W}x{H}", frames_with_one_marker=int(found), threshold_ms_per_frame=round(thr_ms, 5),
               detect_ms_per_frame_one_thread=round(det_ms, 3), end_to_end_frames_per_s={str(k): round(v, 1) for k, v in e2e.items()},
               host_threads_available=os.cpu_count(), cv2_spec_ms_per_frame=None if cv2_ms is None else round(cv2_ms, 2))
    print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "marker_time.json"), "w") as f:
            json.dump(res, f)


if __name__ == "__main__":
    main()
