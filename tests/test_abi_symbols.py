"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol
include/b200sdr.h declares, the ctypes table matches the header, and the product's own
host-side tap design agrees with the oracle (no GPU compute calls here)."""
import ctypes as C
import os
import re
import subprocess

import numpy as np

import oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "b200sdr.h")


def _declared():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(b2s_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported_and_bound():
    from futuresdr_b200 import _lib
    names = _declared()
    assert len(names) > 40
    nm = subprocess.run(["nm", "-D", "--defined-only", _lib.SO_PATH], capture_output=True, text=True,
                        check=True).stdout
    exported = set(re.findall(r"\sT\s+(b2s_[a-z0-9_]+)", nm))
    missing = [n for n in names if n not in exported]
    assert not missing, f"declared in b200sdr.h but not exported: {missing}"
    unbound = [n for n in names if n not in _lib.SIGNATURES]
    assert not unbound, f"declared in b200sdr.h but not in the ctypes table: {unbound}"
    extra = [n for n in _lib.SIGNATURES if n not in names]
    assert not extra, f"bound in ctypes but not declared in the header: {extra}"


def test_header_compiles_as_c():
    # the boundary must be plain C (cgo / Rust bindgen consume it)
    r = subprocess.run(["/usr/bin/gcc", "-std=c99", "-fsyntax-only", "-x", "c", HEADER],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def test_version_and_errors_without_gpu():
    from futuresdr_b200 import _lib
    assert _lib.lib.b2s_version() == 100
    h = C.c_void_p()
    rc = _lib.lib.b2s_ctx_create(0, C.byref(h))
    import torch
    if not torch.cuda.is_available():
        assert rc == _lib.ECUDA and h.value is None
        assert b"CUDA" in _lib.lib.b2s_last_error(None)
    else:
        assert rc == 0
        _lib.lib.b2s_ctx_destroy(h)


def test_product_firdes_matches_oracle():
    from futuresdr_b200 import firdes
    for args in [(0.25, 0.1, 1e-4), (0.2, 0.05, 0.01), (1 / 8, 0.05, 1e-3), (0.02, 0.1, 0.1)]:
        a, b = firdes.kaiser.lowpass(*args), orc.kaiser_lowpass(*args)
        assert a.size == b.size and np.array_equal(a, b)
    for args in [(3, 2, 12, 1e-4), (1, 4, 12, 1e-4), (5, 1, 6, 1e-3), (1, 1, 12, 1e-4), (48, 125, 12, 1e-4)]:
        a, b = firdes.kaiser.multirate(*args), orc.kaiser_multirate(*args)
        assert a.size == b.size and np.array_equal(a, b)


def test_numa_helpers_without_a_gpu():
    """futuresdr_b200.numa: cpulist parsing, and binding degrades gracefully (no NVML here) and restores the CPU set."""
    from futuresdr_b200 import numa
    assert numa._cpulist("0-3,8,10-11\n") == {0, 1, 2, 3, 8, 10, 11}
    assert numa._cpulist("") == set()
    before = os.sched_getaffinity(0)
    with numa.local_to_gpu(0) as info:
        assert "bound" in info
    assert os.sched_getaffinity(0) == before
