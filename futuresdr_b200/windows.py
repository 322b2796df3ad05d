"""Windows (host, f64): futuredsp::windows (crates/futuredsp/src/windows.rs)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import lib


def hamming(len: int, periodic: bool = False) -> np.ndarray:
    """windows::hamming (windows.rs:109-120, gen_cos :68-94): ``len`` f64 points, symmetric or periodic."""
    w = np.zeros(int(len), np.float64)
    lib.b2s_window_hamming(int(len), int(bool(periodic)), w.ctypes.data_as(C.POINTER(C.c_double)), w.size)
    return w
