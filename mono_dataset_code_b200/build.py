"""Builds libmdc_b200.so (CUDA kernels + C ABI + host calibration models) in-tree for sm_90a.

nvcc cross-compiles without a GPU.  The host translation units that construct the lookup
tables are compiled by g++ directly with -ffp-contract=off (bit-exact tables, see
csrc/mdc_host_models.cpp); the .cu files go through nvcc with -lineinfo for ncu source pages.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB_DIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIB_DIR, "libmdc_b200.so")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _newer(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd, log=None):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if log is not None:
        log.append(r.stdout)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout)
        raise RuntimeError("build step failed: " + cmd[0])
    return r.stdout


def build(force: bool = False, verbose: bool = False) -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    gxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"   # not $CXX: see oracle/Makefile
    inc = ["-I" + os.path.join(ROOT, "include"), "-I" + CSRC]
    headers = [os.path.join(ROOT, "include", "mdc_b200.h"), os.path.join(CSRC, "mdc_internal.h"),
               os.path.join(CSRC, "mdc_kernels.cuh"), os.path.join(CSRC, "mdc_atanf.h"), os.path.join(CSRC, "mdc_libm.h"), os.path.join(CSRC, "mdc_jpeg.h"),
               os.path.join(CSRC, "mdc_jpeg_entropy.cuh"), os.path.join(CSRC, "mdc_jpeg_encode.cuh"), os.path.join(CSRC, "mdc_feed.h"),
               os.path.abspath(__file__)]
    obj_dir = os.path.join(PKG, "build")
    os.makedirs(obj_dir, exist_ok=True)
    os.makedirs(LIB_DIR, exist_ok=True)
    objs, log, rebuilt = [], [], False
    for src in ("mdc_host_models.cpp", "mdc_gray_image.cpp", "mdc_jpeg.cpp", "mdc_sequence.cpp", "mdc_marker.cpp", "mdc_png.cpp"):
        o = os.path.join(obj_dir, src + ".o")
        s = os.path.join(CSRC, src)
        if force or _newer(o, [s] + headers):
            _run([gxx, "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-Wall", *inc, "-c", s, "-o", o], log)
            rebuilt = True
        objs.append(o)
    for src in ("mdc_kernels.cu", "mdc_capi.cu", "mdc_vignette_calib.cu", "mdc_marker.cu", "mdc_jpeg_gpu.cu", "mdc_jpeg_encode.cu",
                "mdc_rc_plot.cu"):
        o = os.path.join(obj_dir, src + ".o")
        s = os.path.join(CSRC, src)
        if force or _newer(o, [s] + headers):
            _run([nvcc, "-ccbin", gxx, *GENCODE, "-O3", "-std=c++17", "-lineinfo", "-Xptxas", "-v", "-Xcompiler", "-fPIC",
                  *inc, "-c", s, "-o", o], log)
            rebuilt = True
        objs.append(o)
    if force or rebuilt or _newer(LIB, objs):
        _run([nvcc, "-ccbin", gxx, *GENCODE, "-shared", "-o", LIB, *objs, "-lz", "-cudart", "static"], log)
    # optional native-NCCL init helper for C++ hosts (needs the system libnccl + nccl.h; skipped silently otherwise)
    nccl_src = os.path.join(CSRC, "mdc_nccl.cu")
    nccl_lib = os.path.join(LIB_DIR, "libmdc_b200_nccl.so")
    if os.path.exists("/usr/include/nccl.h") and (force or _newer(nccl_lib, [nccl_src, LIB] + headers)):
        _run([nvcc, "-ccbin", gxx, *GENCODE, "-O2", "-std=c++17", "-Xcompiler", "-fPIC", *inc, "-shared", "-o", nccl_lib, nccl_src,
              "-L" + LIB_DIR, "-lmdc_b200", "-lnccl", "-Xlinker", "-rpath=$ORIGIN", "-cudart", "static"], log)
    if verbose:
        sys.stderr.write("".join(log))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
