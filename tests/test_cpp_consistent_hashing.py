"""The C++ mirror of consistent_hashing (smgx::ConsistentHashingPolicy in include/smgx.hpp): tests/cpp/test_consistent_hashing.cpp ports
the reference's unit tests onto it; this module builds the program on CPU and runs it on an H100."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CPP = os.path.join(ROOT, "tests", "cpp")


def _binary():
    subprocess.check_call(["make", "-s", "-C", CPP, "-f", "consistent_hashing.mk", "test_consistent_hashing"])
    return os.path.join(CPP, "test_consistent_hashing")


def test_cpp_consistent_hashing_builds():
    assert os.path.exists(_binary())


@pytest.mark.gpu
def test_cpp_consistent_hashing():
    r = subprocess.run([_binary()], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "10 tests, 0 failures" in r.stdout, r.stdout
