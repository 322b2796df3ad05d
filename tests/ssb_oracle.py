"""CPU oracle of the SSB transceiver's closures (TEST INFRASTRUCTURE ONLY).

ctypes front-end to ``tests/ssb_oracle.c`` (one reference call at a time, compiled by ``native.load_oracle`` on first
use).  ``Mixer`` carries a closure's oscillator across calls; ``file_level`` and ``to_i16_iq`` are stateless.  The
``py_*`` functions are an independent transcription in numpy f32 scalars, for cross-checking the C file.
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np

from native import load_oracle

_f32p = C.POINTER(C.c_float)
_i16p = C.POINTER(C.c_int16)

ROTATE, ROTATE_SCALE, WEAVER = 0, 1, 2

SIGNATURES = {
    "orc_ssb_from_polar": (None, [C.c_float, _f32p]),
    "orc_ssb_mix": (None, [C.c_int, _f32p, C.c_float, _f32p, _f32p, C.c_size_t, _f32p]),
    "orc_ssb_file_level": (None, [C.c_float, C.c_float, _f32p, C.c_size_t, _f32p]),
    "orc_ssb_to_i16_iq": (None, [C.c_float, _f32p, C.c_size_t, _i16p]),
}


def lib() -> C.CDLL:
    return load_oracle("ssb_oracle", SIGNATURES)


def _c32(x) -> np.ndarray:
    return np.ascontiguousarray(x, np.complex64)


def shift(theta) -> np.ndarray:
    """Complex32::from_polar(1.0, theta) as two f32 (libm cosf / sinf, like Rust's f32::cos / f32::sin)."""
    s = np.zeros(2, np.float32)
    lib().orc_ssb_from_polar(float(np.float32(theta)), s.ctypes.data_as(_f32p))
    return s


class Mixer:
    """One oscillator closure (op ROTATE, ROTATE_SCALE or WEAVER), called once per ``work``."""

    def __init__(self, op: int, theta, param=1.0):
        self.op, self.param = int(op), float(np.float32(param))
        self.shift = shift(theta)
        self.osc = np.array([1.0, 0.0], np.float32)

    def work(self, x) -> np.ndarray:
        x = _c32(x)
        out = np.empty(x.size, np.float32 if self.op == WEAVER else np.complex64)
        lib().orc_ssb_mix(self.op, self.shift.ctypes.data_as(_f32p), self.param, self.osc.ctypes.data_as(_f32p),
                          x.view(np.float32).ctypes.data_as(_f32p), x.size, out.view(np.float32).ctypes.data_as(_f32p))
        return out

    def run(self, x, cuts=()) -> np.ndarray:
        """work() on the slices of ``x`` between ``cuts``, concatenated."""
        edges = [0] + [c for c in cuts if 0 < c < len(x)] + [len(x)]
        parts = [self.work(x[a:b]) for a, b in zip(edges[:-1], edges[1:])]
        return np.concatenate(parts) if parts else self.work(x[:0])


def file_level(x, gain=2.0, div=0.0001) -> np.ndarray:
    x = _c32(x)
    out = np.empty_like(x)
    lib().orc_ssb_file_level(float(np.float32(gain)), float(np.float32(div)), x.view(np.float32).ctypes.data_as(_f32p),
                             x.size, out.view(np.float32).ctypes.data_as(_f32p))
    return out


def to_i16_iq(x, level=0.9) -> np.ndarray:
    x = _c32(x)
    out = np.empty(2 * x.size, np.int16)
    lib().orc_ssb_to_i16_iq(float(np.float32(level)), x.view(np.float32).ctypes.data_as(_f32p), x.size,
                            out.ctypes.data_as(_i16p))
    return out


# ---- independent numpy-f32 transcription ------------------------------------------------------------------------
F = np.float32


def py_shift(theta) -> tuple:
    """from_polar through float64 cos / sin rounded to f32 (equal to libm's cosf / sinf where the test uses it)."""
    t = float(np.float32(theta))
    return F(F(1.0) * F(math.cos(t))), F(F(1.0) * F(math.sin(t)))


def py_mix(op: int, theta, param, x, osc=(1.0, 0.0)) -> tuple:
    """The closure over ``x`` from oscillator ``osc`` -> (output, final osc), every operation on numpy f32 scalars."""
    sr, si = py_shift(theta)
    p = F(param)
    pr, pi = F(osc[0]), F(osc[1])
    x = _c32(x)
    out = np.empty(x.size, np.float32 if op == WEAVER else np.complex64)
    with np.errstate(all="ignore"):
        for k in range(x.size):
            pr, pi = F(F(pr * sr) - F(pi * si)), F(F(pi * sr) + F(pr * si))
            vr, vi = F(x[k].real), F(x[k].imag)
            if op == WEAVER:
                out[k] = F(p * F(F(vr * pr) + F(vi * pi)))
            else:
                yr, yi = F(F(vr * pr) - F(vi * pi)), F(F(vr * pi) + F(vi * pr))
                if op == ROTATE_SCALE:
                    yr, yi = F(yr * p), F(yi * p)
                out[k] = complex(yr, yi)
    return out, (pr, pi)


def py_file_level(x, gain=2.0, div=0.0001) -> np.ndarray:
    f = _c32(x).view(np.float32)
    with np.errstate(all="ignore"):
        return ((f * F(gain)) / F(div)).astype(np.float32).view(np.complex64)


def py_to_i16_iq(x, level=0.9) -> np.ndarray:
    f = _c32(x).view(np.float32)
    with np.errstate(all="ignore"):
        y = ((f * F(level)) * F(32767.0)).astype(np.float32).astype(np.float64)
    y = np.where(np.isnan(y), 0.0, np.trunc(np.clip(y, -32768.0, 32767.0)))
    return y.astype(np.int16)
