"""Compiles and binds the block oracles' C files under tests/ (TEST INFRASTRUCTURE ONLY).

Every oracle is built with the one command below: its flags decide what a bit-exact oracle computes (no fused
multiply-add contraction, no fast-math).  The library goes to a temporary directory that is removed at exit, so the
repository tree may be read-only.
"""
from __future__ import annotations

import atexit
import ctypes as C
import os
import shutil
import subprocess
import tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
_loaded: dict[str, C.CDLL] = {}


def load_oracle(stem: str, signatures: dict) -> C.CDLL:
    """``tests/<stem>.c`` as a ctypes library, compiled at most once per process, with every
    ``{name: (restype, argtypes)}`` of ``signatures`` bound.  A missing symbol raises AttributeError."""
    if stem not in _loaded:
        tmp = tempfile.mkdtemp(prefix=stem + "_")
        atexit.register(shutil.rmtree, tmp, True)
        so = os.path.join(tmp, f"lib{stem}.so")
        subprocess.run(["/usr/bin/gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC",
                        os.path.join(_HERE, stem + ".c"), "-o", so, "-lm"], check=True)
        lib = C.CDLL(so)
        for name, (res, args) in signatures.items():
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = res, args
        _loaded[stem] = lib
    return _loaded[stem]
