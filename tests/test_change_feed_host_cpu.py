"""The change feed of the tick, compiled for the host from the device source (tests/cpp/change_feed_host_test.cpp).

For R = 1..8, on elections from a cold start, lag + churn and message soups, through the wide inbox (fast + general and
general only), the byte form and the compact path of tick mode 4 in 1..8-tick batches, the records the general tick
appends must equal the diff of consecutive oracle exports field for field, and every group a fast function accepts must
keep its term, vote, role and lead.  A capacity below the change count keeps the first records and counts the rest."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cuda_headers():
    inc = os.environ.get("CUDA_INC", "/usr/local/cuda/include")
    return inc if os.path.exists(os.path.join(inc, "cuda_runtime.h")) else None


def _run(target, *argv):
    inc = _cuda_headers()
    if inc is None:
        pytest.skip("CUDA headers not found (set CUDA_INC)")
    subprocess.check_call(["make", "-C", ROOT, f"CUDA_INC={inc}", target], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, target), *argv], capture_output=True, text=True, timeout=1200)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and "change_feed_host_test: ok" in out, out[-3000:]
    assert "runtime error" not in out and "AddressSanitizer" not in out, out[-3000:]
    return out


def _counts(out):
    line = next(ln for ln in out.splitlines() if "fast-path accepts checked" in ln).split()
    return int(line[3]), int(line[6])


def test_change_feed_equals_the_oracle_diff():
    out = _run("tests/cpp/change_feed_host_test")
    cases = [ln for ln in out.splitlines() if ln.strip().startswith("feed ")]
    assert len(cases) >= 40
    for R in range(1, 9):
        assert any(f" R={R} " in ln and "compact" in ln for ln in cases), R
    accepts, records = _counts(out)
    assert accepts > 500_000 and records > 100_000


def _need_sanitizers():
    cxx = subprocess.run(["make", "-s", "--no-print-directory", "-C", ROOT, "san_cxx"], capture_output=True, text=True).stdout.strip()
    if not cxx:
        pytest.skip("no C++ compiler with the sanitizer runtimes on this machine")


def test_change_feed_under_asan_and_ubsan():
    _need_sanitizers()
    out = _run("tests/cpp/change_feed_host_test_san", "quick")
    accepts, records = _counts(out)
    assert accepts > 0 and records > 0
