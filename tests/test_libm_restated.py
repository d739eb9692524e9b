"""glibc's double exp and log restated for host and device (csrc/mdc_libm.h), which plotE's colour map depends on bit for bit.
  - CPU: the host build against this process's libm (tests/cpp/libm_sweep.cpp): exp over [0, 1] at 2^30 + 1 points with random low
    mantissa bits, around every point where the table index changes, over its whole range; log over [20, DBL_MAX] binade by binade
    with random mantissas and around every table subinterval's edge, near 1, in every binade and on subnormals; +-0, +-inf, NaN.
    The sweep prints, and this test reports, the glibc version and whether the CPU has FMA and AVX2, which select glibc's FMA build.
  - GPU: the device build equals the host build and the host's libm on the same sweeps, at the same sizes."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "mono_dataset_code_b200", "csrc")


@pytest.fixture(scope="module")
def sweep_exe(tmp_path_factory):
    exe = str(tmp_path_factory.mktemp("libm_sweep") / "libm_sweep")
    cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-pthread", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC,
           os.path.join(ROOT, "tests", "cpp", "libm_sweep.cpp"), "-o", exe]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return exe


def test_restated_exp_and_log_equal_this_libm(sweep_exe):
    r = subprocess.run([sweep_exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout
    head, *rows = r.stdout.split("\n")
    print("libm variant:", head)          # e.g. "glibc 2.39 fma 1 avx2 1": glibc's FMA build of exp and log
    fields = head.split()
    if fields[3] != "1" or fields[5] != "1":
        pytest.skip(f"{head}: glibc runs its non-FMA exp and log on this CPU; csrc/mdc_libm.h restates the FMA build")
    counts = {}
    for row in filter(None, rows):
        name, n, bad, *first = row.split()
        counts[name] = int(n)
        assert int(bad) == 0, f"{name}: {bad} of {n} points differ from libm, first input bits {first}"
    assert counts["exp_dense_0_1"] >= 10 ** 9 and counts["log_20_max"] >= 1020 << 18
    assert {"exp_special", "log_special", "log_subnormal", "log_near_1", "exp_table_boundaries", "log_table_edges"} <= set(counts)


def mix(z):
    """tests/cpp/libm_sweep.cpp's hash (splitmix64), on uint64 arrays"""
    z = z + np.uint64(0x9e3779b97f4a7c15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xbf58476d1ce4e5b9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94d049bb133111eb)
    return z ^ (z >> np.uint64(31))


def bits(u):
    return np.asarray(u, np.uint64).view(np.float64)


def sweeps(chunk=1 << 25, dense=1 << 30):
    """The sweeps of tests/cpp/libm_sweep.cpp, at the same sizes, as (name, op, x) chunks"""
    def ranged(name, op, n, point):
        for a in range(0, n, chunk):
            yield name, op, point(np.arange(a, min(n, a + chunk), dtype=np.uint64))

    step = 1.0 / dense

    def exp_dense(i):
        x = np.nextafter(i.astype(np.float64) * step, 0.0) + step * (mix(i) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
        return np.where(i == dense, 1.0, x)

    def exp_edges(i):
        c = ((i // 8193).astype(np.float64) + 0.5) * 0.0054152123481245725
        return bits(c.view(np.uint64) + i % np.uint64(8193) - np.uint64(4096))

    def log_20_max(i):      # the last binade is +inf / NaN, as in the C sweep
        x = bits(((np.uint64(0x403) + (i >> np.uint64(18))) << np.uint64(52)) | (mix(i) & np.uint64(0xfffffffffffff)))
        with np.errstate(invalid="ignore"):
            return np.where(x < 20.0, x + 4.0, x)

    def log_edges(i):
        e, j = np.uint64(0x403) + i // np.uint64(128 * 129), (i // np.uint64(129)) % np.uint64(128)
        x = bits(((e << np.uint64(52)) | np.uint64(0x6000000000000)) + (j << np.uint64(45)) + i % np.uint64(129) - np.uint64(64))
        return np.maximum(x, 20.0)

    special = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, -np.nan, 1.0, -1.0, 20.0, 5e-324, 2.2250738585072014e-308,
                        1.7976931348623157e308, -1e-300, 0.9375, 1.0 + float.fromhex("0x1.09p-4"), 709.782712893384, -745.1332191019412, 1e-300])
    yield from ranged("exp_dense_0_1", "exp", dense + 1, exp_dense)
    yield from ranged("exp_table_boundaries", "exp", 200 * 8193, exp_edges)
    yield from ranged("exp_wide", "exp", 1 << 26, lambda i: -760.0 + 1480.0 * (mix(i) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53)
    yield from ranged("exp_tiny", "exp", 1 << 22, lambda i: bits((mix(i) & np.uint64(0x800fffffffffffff)) |
                                                                  ((np.uint64(0x380) + i % np.uint64(0x80)) << np.uint64(52))))
    yield from ranged("log_20_max", "log", 1021 << 18, log_20_max)
    yield from ranged("log_table_edges", "log", 1021 * 128 * 129, log_edges)
    yield from ranged("log_near_1", "log", 1 << 24, lambda i: 0.9375 + 0.1272 * (mix(i) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53)
    yield from ranged("log_all_binades", "log", 1 << 24, lambda i: bits(mix(i) & np.uint64(0x7fffffffffffffff)))
    yield from ranged("log_subnormal", "log", 1 << 20, lambda i: bits(mix(i) & np.uint64(0x000fffffffffffff)))
    yield "exp_special", "exp", special
    yield "log_special", "log", special


def same(a, b):
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint64), b[~nan].view(np.uint64))


@pytest.mark.gpu
def test_device_exp_and_log_equal_the_host_restatement_and_libm():
    """The CPU sweeps, on the device: every point equals the host restatement and the host's libm."""
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import rc_plot_oracle as O
    from mono_dataset_code_b200 import api
    points = {}
    for name, op, x in sweeps():
        dev = api.libm_device(torch.from_numpy(x).cuda(), op).cpu().numpy()
        assert same(dev, api.libm_host(x, op)), f"{name}: device differs from the host restatement"
        assert same(dev, O.libm(x, op)), f"{name}: device differs from libm"
        points[name] = points.get(name, 0) + x.size
    assert points["exp_dense_0_1"] == (1 << 30) + 1 and points["log_20_max"] == 1021 << 18, points
