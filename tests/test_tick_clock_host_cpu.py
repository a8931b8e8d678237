"""Tick mode 4's per-group functions in the library's form — 16-bit offset columns and clock-relative leader timers —
compiled for the host and run against the oracle (tests/cpp/tick_clock_host_test.cpp).

tests/cpp/tick_host_test.cpp and tick_host16_test.cpp check the same functions with the timers in the meta word.  Here a
compact leader's timers are phases against the tick number: traces, message soups, the window-edge soup, ElectionTick
1 / 2 / 2047 and HeartbeatTick 1 / 2 / 255, leaders imported with timers out of range, tick numbers near 2^32 and up
to 2^64 - 1, a tick-count reset with compact state live, and the hot step switched off.  Every tick's out word and
commit advance, and after every batch the state with the timers materialise_group writes, must equal the oracle's."""
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
    assert r.returncode == 0 and "tick_clock_host_test: ok" in out, out[-3000:]
    assert "runtime error" not in out and "AddressSanitizer" not in out, out[-3000:]
    return out


def test_clock_relative_timers_on_the_host_equal_the_oracle():
    out = _run("tests/cpp/tick_clock_host_test")
    lines = [ln for ln in out.splitlines() if ln.strip().startswith("clock")]
    assert len(lines) >= 40
    for what in ("ET=1 HT=255", "ET=2047 HT=2", "imported timers out of range", "ticks up to 2^64 - 1", "ticks across 2^32",
                 "tick count reset"):
        assert any(what in ln for ln in lines), what
    # compact leaders really ran on the fast path in the leader cases
    leaders = [ln.split() for ln in lines if "imported timers" in ln]
    assert all(int(ln[ln.index("leader") + 1].rstrip(")")) > 0 for ln in leaders)


def test_clock_relative_timers_under_asan_and_ubsan():
    cxx = subprocess.run(["make", "-s", "--no-print-directory", "-C", ROOT, "san_cxx"], capture_output=True, text=True).stdout.strip()
    if not cxx:
        pytest.skip("no C++ compiler with the sanitizer runtimes on this machine")
    _run("tests/cpp/tick_clock_host_test_san", "quick")
