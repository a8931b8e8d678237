"""The state of a list of groups, compiled for the host from the device source (tests/cpp/group_state_host_test.cpp).

For R = 1..8, after lag + churn, elections from a cold start and message soups have driven the groups through the mode-4
per-group functions (16-bit offsets, leader timers on the clock) into mixed states, export_group_row must return the rows
of the materialised groups and change no byte of state, and import_group_row must leave every other group's bytes alone
and lead to the same later ticks as the oracle given the same rows."""
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
    assert r.returncode == 0 and "group_state_host_test: ok" in out, out[-3000:]
    assert "runtime error" not in out and "AddressSanitizer" not in out, out[-3000:]
    return out


def _counts(out):
    line = next(ln for ln in out.splitlines() if "export rows checked" in ln).split()
    return int(line[3]), int(line[6])


def test_group_rows_equal_the_materialised_groups_and_the_oracle():
    out = _run("tests/cpp/group_state_host_test")
    cases = [ln for ln in out.splitlines() if ln.strip().startswith("groups ")]
    for R in range(1, 9):
        assert any(f" R={R} " in ln for ln in cases), R
    rows, imported = _counts(out)
    assert rows > 20_000 and imported > 5_000


def _need_sanitizers():
    cxx = subprocess.run(["make", "-s", "--no-print-directory", "-C", ROOT, "san_cxx"], capture_output=True, text=True).stdout.strip()
    if not cxx:
        pytest.skip("no C++ compiler with the sanitizer runtimes on this machine")


def test_group_rows_under_asan_and_ubsan():
    _need_sanitizers()
    out = _run("tests/cpp/group_state_host_test_san", "quick")
    rows, imported = _counts(out)
    assert rows > 0 and imported > 0
