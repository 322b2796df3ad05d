"""CPU oracle of futuredsp::IirFilter (TEST INFRASTRUCTURE ONLY).

ctypes front-end to ``tests/iir_oracle.c``, the C restatement of crates/futuredsp/src/iir.rs:78-178, compiled by
``native.load_oracle`` on first use.
Status codes follow ``futuredsp::ComputationStatus``: 0 InsufficientInput, 1 InsufficientOutput, 2 BothSufficient.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from native import load_oracle

_f32p = C.POINTER(C.c_float)
_f64p = C.POINTER(C.c_double)
_szp = C.POINTER(C.c_size_t)


def _work(p):
    return C.c_int, [p, C.c_size_t, p, C.c_size_t, p, _szp, p, C.c_size_t, p, C.c_size_t, _szp, _szp]


SIGNATURES = {
    "orc_iir_work_f32": _work(_f32p),
    "orc_iir_work_f64": _work(_f64p),
    "orc_iir_exact_f32": (None, [_f32p, C.c_size_t, _f32p, C.c_size_t, _f32p, C.c_size_t, _f64p]),
}


def lib() -> C.CDLL:
    return load_oracle("iir_oracle", SIGNATURES)


def _as(a, dt):
    return np.ascontiguousarray(np.asarray(a).reshape(-1), dtype=dt)


class Iir:
    """IirFilter state machine (crates/futuredsp/src/iir.rs:78-178): memory and its fill count persist across
    ``filter`` calls like the reference's ``StatefulFilter``.  dtype float32 or float64."""

    def __init__(self, a_taps, b_taps, dtype=np.float32):
        self.dtype = np.dtype(dtype)
        self.a, self.b = _as(a_taps, self.dtype), _as(b_taps, self.dtype)
        self.memory = np.zeros(max(self.a.size, 1), self.dtype)
        self.mem_len = C.c_size_t(0)
        f64 = self.dtype == np.float64
        self._fn = lib().orc_iir_work_f64 if f64 else lib().orc_iir_work_f32
        self._ptr = _f64p if f64 else _f32p

    def filter(self, x, out_cap):
        """One filter() call -> (consumed, produced, status, out[:produced])."""
        xi = _as(x, self.dtype)
        out = np.zeros(max(out_cap, 1), self.dtype)
        c, p = C.c_size_t(0), C.c_size_t(0)
        P = lambda a: a.ctypes.data_as(self._ptr)  # noqa: E731
        st = self._fn(P(self.a), self.a.size, P(self.b), self.b.size, P(self.memory), C.byref(self.mem_len), P(xi),
                      xi.size, P(out), out_cap, C.byref(c), C.byref(p))
        assert st >= 0, "n_b == 0 (iir.rs:132 asserts)"
        return c.value, p.value, st, out[: p.value].copy()


def iir(a_taps, b_taps, x, dtype=np.float32):
    """The whole stream x through one IirFilter: outputs 0 .. len(x) - n_b."""
    x = np.asarray(x)
    f = Iir(a_taps, b_taps, dtype)
    c, p, st, y = f.filter(x, x.size)
    if p == 0:                          # the call only filled memory (num_filled == len, :119-129): call again
        c, p, st, y = f.filter(x, x.size)
    return y


def iir_exact(a_taps, b_taps, x):
    """f64 evaluation of the f32 filter (taps and samples widened exactly): the arbiter of the scan tests."""
    a, b, xi = _as(a_taps, np.float32), _as(b_taps, np.float32), _as(x, np.float32)
    n = max(xi.size + 1 - b.size, 0)
    out = np.zeros(max(n, 1), np.float64)
    lib().orc_iir_exact_f32(a.ctypes.data_as(_f32p), a.size, b.ctypes.data_as(_f32p), b.size,
                            xi.ctypes.data_as(_f32p), xi.size, out.ctypes.data_as(_f64p))
    return out[:n]
