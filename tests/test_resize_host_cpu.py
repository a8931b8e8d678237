"""The fresh groups of mrq_resize_groups, compiled for the host from the device source (tests/cpp/resize_host_test.cpp).

init_state_kernel is the one definition of a fresh group for mrq_create and for a grow.  For R = 1..8, the rotate rule
and a fixed self id, group_base 0 and a large one, with tick mode 4's compact state live or not: created rows equal a
fresh oracle's; rows a grow initialises over another run's bytes equal create's in every column (and create's compact
form where the compact state is live), and nothing outside them changes."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cuda_headers():
    inc = os.environ.get("CUDA_INC", "/usr/local/cuda/include")
    return inc if os.path.exists(os.path.join(inc, "cuda_runtime.h")) else None


def _run(target):
    inc = _cuda_headers()
    if inc is None:
        pytest.skip("CUDA headers not found (set CUDA_INC)")
    subprocess.check_call(["make", "-C", ROOT, f"CUDA_INC={inc}", target], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, target)], capture_output=True, text=True, timeout=600)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "resize_host_test: ok" in out, out[-3000:]
    assert "runtime error" not in out and "AddressSanitizer" not in out, out[-3000:]
    return out


def _rows(out):
    return int(next(ln for ln in out.splitlines() if "fresh rows checked" in ln).split()[-1])


def test_fresh_rows_equal_create_and_the_oracle():
    assert _rows(_run("tests/cpp/resize_host_test")) > 50_000


def test_fresh_rows_under_asan_and_ubsan():
    cxx = subprocess.run(["make", "-s", "--no-print-directory", "-C", ROOT, "san_cxx"], capture_output=True, text=True).stdout.strip()
    if not cxx:
        pytest.skip("no C++ compiler with the sanitizer runtimes on this machine")
    assert _rows(_run("tests/cpp/resize_host_test_san")) > 50_000
