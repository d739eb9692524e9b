"""Time the GPU JPEG encoder (mdc_jpeg_encode_device) against cv2.imencode on the same frames, and playbackDataset_b200's save mode
against a host loop doing the same work.

  python scripts/jpeg_encode_time.py [--frames 256] [--reps 10] [--e2e-frames 1000] [--out FILE.json]

  encode     per size (640x480, 1280x1024, 1920x1080): `frames` realistic rectified frames (the u8 output of the fused prepare kernel on
             the synthetic sequence: rectify + gamma + vignette).  GPU: CUDA events around `reps` calls of all frames each (a call
             returns with the sizes on the host), median.  Per stage: kernel times of one call from torch.profiler.  cv2.imencode
             (quality 95) on one thread, and on all host threads (a thread pool; imencode releases the GIL).  Checks that the GPU
             files equal cv2's.
  e2e        a zip of `e2e-frames` 1280x1024 JPEG frames (quality 90): wall time of `playbackDataset_b200 <seq> save` against a host
             loop over chunks of 256 frames: mdc_seq_prepare (rectify, MDC_OUT_U8) -> cv2.imencode -> write, the encodes and writes
             on all host threads.  Checks that both wrote the same files.
Records the card's name and power limit and the host's CPU count.  Needs a GPU; prints one JSON document."""
import argparse
import concurrent.futures as cf
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import zipfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(640, 480), (1280, 1024), (1920, 1080)]
KINDS = ["uniform", "speckle", "gradient"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def rectified_u8(d, w, h, n):
    """n frames of the synthetic sequence through the fused kernel (rectify + gamma + vignette) into u8: a CUDA tensor [n, h, w]."""
    import torch
    from mono_dataset_code_b200 import api, synthetic as S
    files = S.write_dataset_dir(d, w, h, w, h, "crop")
    prep = api.FramePreparer(api.UndistorterFOV(files["camera"]), api.PhotometricUndistorter(files["pcalib"], files["vignette"], w, h), device=0)
    raw = np.stack([S.frame(i, w, h, KINDS[i % 3]) for i in range(n)])
    out = prep.prepare_device(torch.from_numpy(raw).cuda(), True, True, True, False, dtype=torch.uint8)[0]
    torch.cuda.synchronize()
    return out.reshape(n, h, w)


def time_encode(w, h, n, reps, tmp):
    import cv2
    import torch
    from mono_dataset_code_b200 import api
    from mono_dataset_code_b200._lib import lib
    frames = rectified_u8(os.path.join(tmp, f"ds_{w}"), w, h, n)
    ctx = api.Context(None, None, 0)
    stride = api.jpeg_encode_bound(w, h)
    out = torch.empty((n, stride), dtype=torch.uint8, device="cuda")
    sizes = (C.c_size_t * n)()
    s = torch.cuda.current_stream()

    def call():
        rc = lib.mdc_jpeg_encode_device(ctx._h, C.c_void_p(frames.data_ptr()), w, n, w, h, 95, C.c_void_p(out.data_ptr()), stride, sizes,
                                        C.c_void_p(s.cuda_stream or 1))
        assert rc == 0, rc
    for _ in range(3):
        call()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        call()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    gpu_ms = statistics.median(ms)
    # per stage, one call under the profiler (a separate run: tracing slows the host)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    stages = {}
    for ev in prof.key_averages():
        for k in ("e1_fdct_quant", "e2_block_bits", "e3_scan_bits", "e4_emit", "e5_stuff"):
            if k in ev.key:
                stages[k] = round(ev.device_time_total / 1000.0, 4) if hasattr(ev, "device_time_total") else round(ev.cuda_time_total / 1000.0, 4)
    host = frames.cpu().numpy()
    gpu_files = [out[k, :sizes[k]].cpu().numpy().tobytes() for k in range(n)]
    params = [cv2.IMWRITE_JPEG_QUALITY, 95]
    t0 = time.perf_counter()
    ref = [cv2.imencode(".jpg", host[k], params)[1].tobytes() for k in range(n)]
    one = time.perf_counter() - t0
    threads = os.cpu_count()
    with cf.ThreadPoolExecutor(threads) as ex:
        list(ex.map(lambda k: cv2.imencode(".jpg", host[k], params)[1], range(min(n, threads))))
        t0 = time.perf_counter()
        list(ex.map(lambda k: cv2.imencode(".jpg", host[k], params)[1], range(n)))
        allc = time.perf_counter() - t0
    same = all(g == r for g, r in zip(gpu_files, ref))
    mean_bytes = sum(len(g) for g in gpu_files) / n
    return {"size": f"{w}x{h}", "frames": n, "gpu_ms_per_call": round(gpu_ms, 3), "gpu_min_max_ms": [round(min(ms), 3), round(max(ms), 3)],
            "gpu_frames_per_s": round(n / gpu_ms * 1e3), "stage_ms": stages, "cv2_1thread_frames_per_s": round(n / one),
            "cv2_allthreads_frames_per_s": round(n / allc), "speedup_vs_allthreads": round((n / gpu_ms * 1e3) / (n / allc), 2),
            "mean_file_bytes": round(mean_bytes), "bytes_equal_cv2": same}


def e2e(n, tmp):
    import cv2
    from mono_dataset_code_b200 import api, synthetic as S
    w, h = 1280, 1024
    seq = os.path.join(tmp, "e2e")
    files = S.write_dataset_dir(seq, w, h, w, h, "crop")
    with zipfile.ZipFile(os.path.join(seq, "images.zip"), "w", zipfile.ZIP_STORED) as z:
        for i in range(n):
            z.writestr(f"{i:05d}.jpg", cv2.imencode(".jpg", S.frame(i, w, h, KINDS[i % 3]).reshape(h, w), [cv2.IMWRITE_JPEG_QUALITY, 90])[1].tobytes())
    with open(os.path.join(seq, "times.txt"), "w") as t:
        for i in range(n):
            t.write(f"{i} {i * 0.05:.6f} 10.0\n")
    exe = os.path.join(tmp, "playbackDataset_b200")
    lib = os.path.join(ROOT, "mono_dataset_code_b200", "lib")
    subprocess.run(["g++", "-std=c++11", "-O2", "-I" + os.path.join(ROOT, "include"), "-I/usr/local/cuda/include",
                    os.path.join(ROOT, "tools", "playbackDataset_b200.cpp"), "-o", exe, "-L" + lib, "-lmdc_b200", "-L/usr/local/cuda/lib64",
                    "-lcudart", "-lpthread", "-Wl,-rpath," + lib + ":/usr/local/cuda/lib64"], check=True)
    res = {"frames": n, "size": f"{w}x{h}"}
    tool_dir, host_dir = os.path.join(tmp, "out_tool"), os.path.join(tmp, "out_host")
    for k in range(2):                                      # alternated, the second round reported
        for d in (tool_dir, host_dir):
            subprocess.run(["rm", "-rf", d])
            os.makedirs(d)
        t0 = time.perf_counter()
        r = subprocess.run([exe, seq + "/", "save"], cwd=tool_dir, capture_output=True, text=True)
        res["tool_s"] = round(time.perf_counter() - t0, 3)
        assert r.returncode == 0, r.stdout[-2000:]
        t0 = time.perf_counter()
        fov = api.UndistorterFOV(files["camera"])
        ctx = api.Context(fov, api.PhotometricUndistorter(files["pcalib"], files["vignette"], w, h), 0)
        sq = api.Sequence(seq + "/")

        def write(i, img):
            with open(os.path.join(host_dir, f"{i:05d}.jpg"), "wb") as f:
                f.write(cv2.imencode(".jpg", img)[1].tobytes())
        with cf.ThreadPoolExecutor(os.cpu_count()) as ex:
            for f0 in range(0, n, 256):
                c = min(256, n - f0)
                u8 = sq.prepare(ctx, [(w, h)], f0, c, True, False, False, False, dtype=np.uint8)[0].reshape(c, h, w)
                list(ex.map(write, range(f0, f0 + c), u8))
        res["host_loop_s"] = round(time.perf_counter() - t0, 3)
    # the tool's GPU decode feed alone (mdc_seq_prepare_device into u8, the tool's chunks of 256 frames at 8 host threads), no encode
    import torch
    d = torch.empty((256, h * w), dtype=torch.uint8, device="cuda")
    t0 = time.perf_counter()
    for f0 in range(0, n, 256):
        sq.prepare_device(ctx, f0, min(256, n - f0), True, False, False, False, out=[d[:min(256, n - f0)]], dtype=torch.uint8)
    torch.cuda.synchronize()
    res["decode_feed_only_s"] = round(time.perf_counter() - t0, 3)
    res["tool_frames_per_s"] = round(n / res["tool_s"])
    res["host_loop_frames_per_s"] = round(n / res["host_loop_s"])
    res["same_files"] = all(open(os.path.join(tool_dir, f), "rb").read() == open(os.path.join(host_dir, f), "rb").read()
                            for f in sorted(os.listdir(host_dir))) and sorted(os.listdir(tool_dir)) == sorted(os.listdir(host_dir))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--e2e-frames", type=int, default=1000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    doc = {"card": card(), "host_cpus": os.cpu_count(), "quality": 95, "encode": []}
    with tempfile.TemporaryDirectory(prefix="mdc_jpeg_enc_") as tmp:
        for (w, h) in SIZES:
            doc["encode"].append(time_encode(w, h, a.frames, a.reps, tmp))
            print(json.dumps(doc["encode"][-1]), flush=True)
        if a.e2e_frames:
            doc["e2e"] = e2e(a.e2e_frames, tmp)
    text = json.dumps(doc, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
