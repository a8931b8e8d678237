"""The quad kernel's lane-pair hot step, compact_hot_pair, compiled for the host: against two scalar hot steps
(tests/cpp/tick_pair_host_test.cpp), and inside the kernel's pair structure against the oracle
(tests/cpp/tick_pair_clock_host_test.cpp).

compact_hot_pair steps two settled leaders at once in the 16-bit lanes of the pair words.  For R = 1..8, on random
steady-state pairs and on sweeps over the lane guards, the edges of the 16-bit span, every frame byte in every row,
proposal bytes 0 / 1 / 3 / 255, pairs with one lane ineligible, and lanes where nothing moved with the commit index
below the quorum, it must accept exactly when both scalar steps accept inside its guards, then agree with them bit for
bit (state, out words, commit advances, dirty bits), and leave both groups untouched when it declines.  Run the way
tick_fast4_kernel runs a launch — groups in pairs, the pair step first, declined pairs unpacked into the scalar steps —
every case of tests/cpp/tick_clock_host_test.cpp must still equal the oracle."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cuda_headers():
    inc = os.environ.get("CUDA_INC", "/usr/local/cuda/include")
    return inc if os.path.exists(os.path.join(inc, "cuda_runtime.h")) else None


def _run(target, ok, *argv):
    inc = _cuda_headers()
    if inc is None:
        pytest.skip("CUDA headers not found (set CUDA_INC)")
    subprocess.check_call(["make", "-C", ROOT, f"CUDA_INC={inc}", target], stdout=subprocess.DEVNULL)
    r = subprocess.run([os.path.join(ROOT, target), *argv], capture_output=True, text=True, timeout=1200)
    out = r.stdout + r.stderr
    assert r.returncode == 0 and ok in out, out[-3000:]
    assert "runtime error" not in out and "AddressSanitizer" not in out, out[-3000:]
    return out


def test_pair_step_equals_two_scalar_steps():
    out = _run("tests/cpp/tick_pair_host_test", "tick_pair_host_test: ok")
    line = next(ln for ln in out.splitlines() if "pairs checked" in ln).split()
    checked, accepted = int(line[0]), int(line[3])
    assert checked > 300_000 and accepted > checked // 5


def _need_sanitizers():
    cxx = subprocess.run(["make", "-s", "--no-print-directory", "-C", ROOT, "san_cxx"], capture_output=True, text=True).stdout.strip()
    if not cxx:
        pytest.skip("no C++ compiler with the sanitizer runtimes on this machine")


def test_pair_step_under_asan_and_ubsan():
    _need_sanitizers()
    _run("tests/cpp/tick_pair_host_test_san", "tick_pair_host_test: ok")


def _pair_ticks(out):
    line = next(ln for ln in out.splitlines() if "the pair step ran" in ln)
    return int(line.split()[4])


def test_pair_structured_launch_equals_the_oracle():
    out = _run("tests/cpp/tick_pair_clock_host_test", "tick_clock_host_test: ok")
    assert len([ln for ln in out.splitlines() if ln.strip().startswith("clock")]) >= 40
    assert _pair_ticks(out) > 100_000


def test_pair_structured_launch_under_asan_and_ubsan():
    _need_sanitizers()
    out = _run("tests/cpp/tick_pair_clock_host_test_san", "tick_clock_host_test: ok", "quick")
    assert _pair_ticks(out) > 0
