"""The C++ host layer's owning classes are move-only (tests/cpp/handles.cpp holds the static_asserts).  A syntax-only
compile needs the headers and a C++17 compiler, no GPU and no library."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_cpp_owning_classes_are_move_only():
    r = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"),
                        os.path.join(ROOT, "tests", "cpp", "handles.cpp")], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-4000:]
