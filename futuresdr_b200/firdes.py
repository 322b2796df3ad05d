"""Tap design (host, f64): futuredsp::firdes::kaiser, firdes::lowpass and firdes::hilbert
(crates/futuredsp/src/firdes/basic.rs)."""
from __future__ import annotations

import ctypes as C

import numpy as np

from ._lib import lib


class kaiser:
    @staticmethod
    def lowpass(cutoff: float, transition_bw: float, max_ripple: float) -> np.ndarray:
        """firdes::kaiser::lowpass::<f32> (basic.rs:310-321)."""
        assert cutoff > 0.0, "cutoff must be greater than 0"
        assert transition_bw > 0.0, "transition_bw must be greater than 0"
        assert cutoff + transition_bw < 0.5, "cutoff+transition_bw must be less than 1/2"
        n = lib.b2s_firdes_kaiser_lowpass(cutoff, transition_bw, max_ripple, None, 0)
        t = np.zeros(n, np.float32)
        lib.b2s_firdes_kaiser_lowpass(cutoff, transition_bw, max_ripple,
                                      t.ctypes.data_as(C.POINTER(C.c_float)), n)
        return t

    @staticmethod
    def multirate(interp: int, decim: int, half_polyphase_len: int, max_ripple: float) -> np.ndarray:
        """firdes::kaiser::multirate::<f32> (basic.rs:412-442)."""
        assert interp > 0 and decim > 0 and half_polyphase_len > 0
        n = lib.b2s_firdes_kaiser_multirate(interp, decim, half_polyphase_len, max_ripple, None, 0)
        t = np.zeros(n, np.float32)
        lib.b2s_firdes_kaiser_multirate(interp, decim, half_polyphase_len, max_ripple,
                                        t.ctypes.data_as(C.POINTER(C.c_float)), n)
        return t


def hilbert(window) -> np.ndarray:
    """firdes::hilbert::<f32> (basic.rs:202-222): a 90-degree phase shifter with the window's (odd) length."""
    w = np.ascontiguousarray(window, dtype=np.float64)
    assert w.size % 2 == 1, "Must be an odd number"                          # basic.rs:204
    t = np.zeros(w.size, np.float32)
    lib.b2s_firdes_hilbert(w.ctypes.data_as(C.POINTER(C.c_double)), w.size, t.ctypes.data_as(C.POINTER(C.c_float)),
                           w.size)
    return t


def lowpass(cutoff: float, window) -> np.ndarray:
    """firdes::lowpass::<f32> (basic.rs:25-42): the windowed sinc with cutoff in cycles per sample, one tap per window
    entry."""
    w = np.ascontiguousarray(window, dtype=np.float64)
    assert abs(cutoff) < 0.5, "cutoff must be in ]-1/2, 1/2["                 # basic.rs:26
    t = np.zeros(w.size, np.float32)
    if w.size:
        lib.b2s_firdes_lowpass(float(cutoff), w.ctypes.data_as(C.POINTER(C.c_double)), w.size,
                               t.ctypes.data_as(C.POINTER(C.c_float)), w.size)
    return t
