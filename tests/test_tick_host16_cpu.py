"""Tick mode 4's per-group functions at the library's offset width, compiled for the host and run against the oracle
(tests/cpp/tick_host16_test.cpp).

The library stores the compact offset columns as uint16_t; tests/cpp/tick_host_test.cpp checks the same functions at
the header's default 32-bit width.  Here the 16-bit instantiation runs the traces, the message soups, the window-edge
soup, a tiny span that forces a re-base every few dozen ticks, and steady leaders whose logs run past the end of the
16-bit span, every tick's out word, commit advance and the state compared with the oracle."""
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
    assert r.returncode == 0 and "tick_host16_test: ok" in out, out[-3000:]
    assert "runtime error" not in out and "AddressSanitizer" not in out, out[-3000:]
    return out


def test_16_bit_compact_columns_on_the_host_equal_the_oracle():
    out = _run("tests/cpp/tick_host16_test")
    lines = [ln for ln in out.splitlines() if ln.strip().startswith("compact u16")]
    assert len(lines) >= 25
    long_logs = [ln.split() for ln in lines if "long logs" in ln]
    assert len(long_logs) == 1
    ln = long_logs[0]
    assert int(ln[ln.index("exits") + 1]) > 0  # leaders really ran into the end of the 16-bit span


def test_16_bit_compact_columns_under_asan_and_ubsan():
    cxx = subprocess.run(["make", "-s", "--no-print-directory", "-C", ROOT, "san_cxx"], capture_output=True, text=True).stdout.strip()
    if not cxx:
        pytest.skip("no C++ compiler with the sanitizer runtimes on this machine")
    _run("tests/cpp/tick_host16_test_san", "quick")
