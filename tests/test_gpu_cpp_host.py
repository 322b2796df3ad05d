"""Runs each C++ host-layer test program (tests/cpp/test_*.cpp over include/b200sdr.hpp, built by
__graft_entry__.build()): the reference's known-answer tests and each block's own cases replayed from compiled host code
through the C ABI."""
import glob
import os
import subprocess

import pytest

CPP = os.path.join(os.path.dirname(os.path.abspath(__file__)), "cpp")
PROGRAMS = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(CPP, "test_*.cpp")))


def _binary(prog):
    path = os.path.join(CPP, prog)
    assert os.path.exists(path), f"tests/cpp/{prog} missing: run __graft_entry__.build()"
    return path


@pytest.mark.gpu
@pytest.mark.parametrize("prog", PROGRAMS)
def test_cpp_host_layer(prog):
    r = subprocess.run([_binary(prog)], capture_output=True, text=True, timeout=300)
    print(r.stdout[-2000:], r.stderr[-2000:])
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "all checks passed" in r.stdout


@pytest.mark.parametrize("prog", PROGRAMS)
def test_cpp_host_layer_builds(prog):
    # CPU-side: the headers compile and the binary links against libb200sdr.so
    _binary(prog)
