"""The decode-ahead pool both sequence feeds share (csrc/mdc_feed.h), under ThreadSanitizer: tests/cpp/feed_pool_harness.cpp sweeps
thread counts 1, 2, 3, 8, 64, chunks 1, 2, 16, 256 and counts 0, 1, C-1, C, C+1, 3C+1, with a consumer that takes every chunk, one
whose read fails on a frame, and one that stops with a slot unreleased."""
import os
import subprocess

import pytest

from conftest import ROOT

CSRC = os.path.join(ROOT, "mono_dataset_code_b200", "csrc")


def test_feed_pool_under_thread_sanitizer(tmp_path):
    exe = str(tmp_path / "feed_pool_harness")
    cmd = ["g++", "-std=c++17", "-O1", "-g", "-fsanitize=thread", "-I" + os.path.join(ROOT, "include"), "-I" + CSRC,
           os.path.join(ROOT, "tests", "cpp", "feed_pool_harness.cpp"), "-lpthread", "-o", exe]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        pytest.skip("no ThreadSanitizer-enabled g++ here: " + r.stdout[-300:])
    env = dict(os.environ, TSAN_OPTIONS="halt_on_error=1")
    r = subprocess.run([exe], env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    if "ThreadSanitizer: unexpected memory mapping" in r.stdout:
        pytest.skip("ThreadSanitizer cannot run under this kernel's address-space layout")
    assert r.returncode == 0, r.stdout[-4000:]
    assert "runs passed" in r.stdout and "ThreadSanitizer" not in r.stdout, r.stdout[-4000:]
