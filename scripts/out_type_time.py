"""Time prepared levels in each output type (MDC_OUT_F32 / F16 / U8) on the benchmark's setup: 256 synthetic 1280x1024 frames,
rectify + remove gamma + remove vignette, levels 1 and 5.

  python scripts/out_type_time.py [--frames 256] [--launches 100] [--reps 5] [--out FILE.json]

  call time   CUDA events around `launches` back-to-back mdc_prepare_batch_ex calls on resident frames, `reps` repetitions with
              the output types in rotating order; per-call median and min-max over the repetitions.  With levels = 1 a call is one
              K1 launch; with levels = 5 it is K1 (levels 0-2) and one K2 launch (levels 3-4).
  e2e         frames/s through mdc_prepare_batch_host_ex (pinned frames in, pinned levels out; H2D + kernels + D2H), median of
              `reps` calls of all frames each.
  bytes       algorithmic bytes per frame of the K1 launch: 1 byte in per pixel, the levels K1 writes in the output type, and for a
              narrow type with levels > 3 the fp32 copy of level 2 that K2 reads.
Also checks, on the timed data, that each narrow result is the conversion of the fp32 one.  Needs a GPU; prints one JSON document."""
import argparse
import ctypes as C
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

W = H = None
TYPES = {"f32": 0, "f16": 1, "u8": 2}
ESIZE = {"f32": 4, "f16": 2, "u8": 1}
FLAGS = 1 | 2 | 4


def k1_bytes(name, levels, w, h):
    px = [(w >> l) * (h >> l) for l in range(min(levels, 3))]
    b = w * h + sum(px) * ESIZE[name]
    if name != "f32" and levels > 3:
        b += px[2] * 4
    return b


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:          # the numbers still stand; the card is then named by torch only
        return f"nvidia-smi unavailable ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--size", default="1280x1024")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    w, h = map(int, a.size.split("x"))

    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    from mono_dataset_code_b200 import _lib, api, synthetic as S
    lib = _lib.lib
    files = S.write_dataset_dir(tempfile.mkdtemp(prefix="mdc_outtype_"), w, h, w, h, "crop")
    fov = api.UndistorterFOV(files["camera"])
    photo = api.PhotometricUndistorter(files["pcalib"], files["vignette"], w, h)
    ctx = api.Context(fov, photo, 0)
    n = a.frames
    rng = np.random.default_rng(0)
    h_frames = rng.integers(0, 256, (n, w * h), dtype=np.uint8)
    frames = torch.from_numpy(h_frames).cuda()
    dt = {"f32": torch.float32, "f16": torch.float16, "u8": torch.uint8}
    result = {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": gpu_info(), "host_cpus": os.cpu_count(), "frames": n,
              "size": f"{w}x{h}", "flags": "rectify+gamma+vignette", "launches_per_rep": a.launches, "reps": a.reps, "levels": {}}
    for levels in (1, 5):
        outs = {k: [torch.empty((n, (w >> l) * (h >> l)), dtype=dt[k], device="cuda") for l in range(levels)] for k in TYPES}
        ptrs = {k: (C.c_void_p * levels)(*[t.data_ptr() for t in outs[k]]) for k in TYPES}
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream or 1)

        def call(k):
            _lib.check(lib.mdc_prepare_batch_ex(ctx._h, C.c_void_p(frames.data_ptr()), 0, n, FLAGS, TYPES[k], ptrs[k], levels, stream),
                       "mdc_prepare_batch_ex")
        for k in TYPES:                     # warm-up: module load, pools, descriptors
            for _ in range(3):
                call(k)
        torch.cuda.synchronize()
        # correctness on the timed data
        ref = [o.cpu().numpy() for o in outs["f32"]]
        for l in range(levels):
            with np.errstate(over="ignore", invalid="ignore"):
                e16 = ref[l].astype(np.float16)
            g16 = outs["f16"][l].cpu().numpy()
            assert np.array_equal(np.isnan(e16), np.isnan(g16)) and np.array_equal(e16[~np.isnan(e16)].view(np.uint16),
                                                                                   g16[~np.isnan(g16)].view(np.uint16)), ("f16", l)
            inside = (ref[l] >= -2.0 ** 31) & (ref[l] < 2.0 ** 31)
            with np.errstate(invalid="ignore"):
                e8 = np.clip(np.where(inside, np.rint(ref[l].astype(np.float64)), -2.0 ** 31), 0, 255).astype(np.uint8)
            assert np.array_equal(e8, outs["u8"][l].cpu().numpy()), ("u8", l)
        per_call = {k: [] for k in TYPES}
        names = list(TYPES)
        for r in range(a.reps):
            order = names[r % 3:] + names[:r % 3]
            for k in order:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.launches):
                    call(k)
                e1.record()
                e1.synchronize()
                per_call[k].append(e0.elapsed_time(e1) / a.launches)
        # end to end through the host pipeline
        e2e = {}
        for k in TYPES:
            esz = ESIZE[k]
            px = [(w >> l) * (h >> l) for l in range(levels)]
            hin, hout = C.c_void_p(), C.c_void_p()
            _lib.check(lib.mdc_host_alloc(C.byref(hin), n * w * h), "mdc_host_alloc")
            _lib.check(lib.mdc_host_alloc(C.byref(hout), n * sum(px) * esz), "mdc_host_alloc")
            C.memmove(hin.value, h_frames.ctypes.data, n * w * h)
            offs, o = [], 0
            for p in px:
                offs.append(hout.value + o)
                o += n * p * esz
            hp = (C.c_void_p * levels)(*offs)
            times = []
            for r in range(a.reps + 1):
                t0 = time.perf_counter()
                _lib.check(lib.mdc_prepare_batch_host_ex(ctx._h, hin, n, FLAGS, TYPES[k], hp, levels), "mdc_prepare_batch_host_ex")
                times.append(time.perf_counter() - t0)
            lib.mdc_host_free(hin)
            lib.mdc_host_free(hout)
            e2e[k] = n / statistics.median(times[1:])
        result["levels"][str(levels)] = {
            k: {"call_ms_median": round(statistics.median(per_call[k]), 4), "call_ms_min": round(min(per_call[k]), 4),
                "call_ms_max": round(max(per_call[k]), 4),
                "k1_bytes_per_frame": k1_bytes(k, levels, w, h),
                "k1_gbs_at_median": round(k1_bytes(k, levels, w, h) * n / (statistics.median(per_call[k]) * 1e-3) / 1e9, 1) if levels == 1 else None,
                "e2e_frames_per_s": round(e2e[k], 1), "d2h_bytes_per_frame": sum((w >> l) * (h >> l) for l in range(levels)) * ESIZE[k]}
            for k in TYPES}
    ctx.close()
    text = json.dumps(result, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
