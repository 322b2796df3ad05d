"""Runs the C++ host-layer keyfob test program (tests/cpp/test_keyfob_host.cpp over include/b200sdr.hpp) through the
C ABI."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIN = os.path.join(ROOT, "tests", "cpp", "test_keyfob_host")


@pytest.mark.gpu
def test_cpp_keyfob_host_layer():
    assert os.path.exists(BIN), "tests/cpp/test_keyfob_host missing: run __graft_entry__.build()"
    r = subprocess.run([BIN], capture_output=True, text=True, timeout=300)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "all checks passed" in r.stdout


def test_cpp_keyfob_host_layer_builds():
    assert os.path.exists(BIN), "tests/cpp/test_keyfob_host missing: run __graft_entry__.build()"
