"""sb::Resources (salmon_b200/csrc/resources.h), the owner of every library object's CUDA buffers, streams and events,
compiled for the host over a stub runtime (tests/host_resources.cpp): the reuse and growth rules, grow_keep's copy, and
that a failure at any step of a create-like sequence leaves no dangling pointer and nothing live after destruction --
also under AddressSanitizer, UndefinedBehaviorSanitizer and LeakSanitizer."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host_resources.cpp")
CUDA_INC = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
CHECKS = ["grow", "alloc_release", "grow_keep", "fail_kth"]
SANITIZE = ["-fsanitize=address,undefined", "-fno-sanitize-recover=undefined", "-fno-omit-frame-pointer"]


@pytest.fixture(scope="module")
def binaries(tmp_path_factory):
    if not os.path.exists(os.path.join(CUDA_INC, "cuda_runtime.h")):
        pytest.skip("CUDA headers not found (set CUDA_HOME)")
    d = tmp_path_factory.mktemp("host_resources")
    out = {}
    for mode, extra in (("plain", []), ("sanitized", SANITIZE)):
        exe = str(d / mode)
        subprocess.check_call(["/usr/bin/g++", "-O1", "-g", "-std=c++17", "-Wall", "-Werror", *extra,
                               "-I" + CUDA_INC, "-o", exe, SRC])
        out[mode] = exe
    return out


@pytest.mark.parametrize("mode", ["plain", "sanitized"])
@pytest.mark.parametrize("check", CHECKS)
def test_resources(binaries, mode, check):
    env = dict(os.environ, ASAN_OPTIONS="detect_leaks=1:abort_on_error=0", UBSAN_OPTIONS="print_stacktrace=1")
    r = subprocess.run([binaries[mode], check], capture_output=True, text=True, env=env, timeout=120)
    assert r.returncode == 0, r.stderr
