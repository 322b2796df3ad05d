"""CPU oracle of blocks::SignalSource and FixedPointPhase (TEST INFRASTRUCTURE ONLY).

ctypes front-end to ``tests/sigsrc_oracle.c``, the C restatement of src/blocks/signal_source/{mod,fxpt_nco,
fxpt_phase}.rs, fed with the reference's sine table from ``tests/golden/reference_fxpt_sine_table.json`` and compiled
by ``native.load_oracle`` on first use.
``np_*`` is a second, independent transcription in numpy float32 that the CPU tests hold the C oracle to.
"""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np

from native import load_oracle

FIXTURE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_fxpt_sine_table.json")
COS, SIN, SQUARE = 0, 1, 2
_f32p = C.POINTER(C.c_float)


def table() -> np.ndarray:
    """The reference's sine table as float32 [1024, 2] = (slope, offset)."""
    bits = np.array(json.load(open(FIXTURE))["table_bits"], dtype=np.uint32)
    return bits.view(np.float32).reshape(1024, 2)


TABLE = table()


SIGNATURES = {
    "orc_fxpt_phase_new": (C.c_int32, [C.c_float]),
    "orc_sigsrc_inc": (C.c_int32, [C.c_float, C.c_float]),
    "orc_fxpt_sin": (C.c_float, [_f32p, C.c_int32]),
    "orc_fxpt_cos": (C.c_float, [_f32p, C.c_int32]),
    "orc_sigsrc_work": (None, [_f32p, C.c_int, C.c_int, C.POINTER(C.c_int32), C.c_int32, C.c_float, _f32p,
                               C.c_size_t]),
}


def lib() -> C.CDLL:
    return load_oracle("sigsrc_oracle", SIGNATURES)


def _tp():
    return TABLE.ctypes.data_as(_f32p)


def phase_new(x) -> int:
    return int(lib().orc_fxpt_phase_new(float(np.float32(x))))


def builder_inc(frequency, sample_rate) -> int:
    return int(lib().orc_sigsrc_inc(float(np.float32(frequency)), float(np.float32(sample_rate))))


def fxpt_sin(value: int) -> np.float32:
    return np.float32(lib().orc_fxpt_sin(_tp(), int(value)))


def fxpt_cos(value: int) -> np.float32:
    return np.float32(lib().orc_fxpt_cos(_tp(), int(value)))


class Source:
    """SignalSourceBuilder::<f32 | Complex32>::{cos, sin, square}(frequency, sample_rate, amplitude, initial_phase):
    the NCO state persists across ``work`` calls like the block's."""

    def __init__(self, wave, frequency, sample_rate, amplitude, initial_phase, dtype=np.float32):
        self.wave, self.cplx = int(wave), np.dtype(dtype) == np.complex64
        self.phase = C.c_int32(phase_new(initial_phase))
        self.inc = builder_inc(frequency, sample_rate)
        self.amplitude = np.float32(amplitude)

    def work(self, n: int) -> np.ndarray:
        """One work() call on an output slice of n items."""
        out = np.empty(max(n, 1) * (2 if self.cplx else 1), np.float32)
        lib().orc_sigsrc_work(_tp(), self.wave, int(self.cplx), C.byref(self.phase), self.inc,
                              float(self.amplitude), out.ctypes.data_as(_f32p), n)
        out = out[: n * (2 if self.cplx else 1)]
        return out.view(np.complex64) if self.cplx else out


# ---- independent numpy float32 transcription ----------------------------------------------------------------------
_PI, _TAU = np.float32(np.pi), np.float32(2 * np.pi)


def _as_i32(f):
    """Rust `as i32` on float32 arrays: truncate, saturate, NaN -> 0."""
    f = np.asarray(f, np.float32)
    with np.errstate(invalid="ignore"):
        t = np.trunc(np.nan_to_num(f, nan=0.0, posinf=3e9, neginf=-3e9).astype(np.float64))
    return np.clip(t, -2.0 ** 31, 2.0 ** 31 - 1).astype(np.int64).astype(np.int32)


def np_phase_new(x):
    x = np.asarray(x, np.float32)
    with np.errstate(all="ignore"):
        d = _as_i32(np.floor(x / _TAU + np.float32(0.5)))
        xr = x - d.astype(np.float32) * _TAU
        return _as_i32(xr * np.float32(2.0 ** 31) / _PI)


def np_builder_inc(frequency, sample_rate):
    with np.errstate(all="ignore"):
        return np_phase_new(np.float32(2.0) * _PI * np.float32(frequency) / np.float32(sample_rate))


def np_lookup(ux):
    ux = np.asarray(ux, np.uint32)
    i = ux >> np.uint32(22)
    with np.errstate(all="ignore"):
        return TABLE[i, 0] * (ux & np.uint32(0x3FFFFF)).astype(np.float32) + TABLE[i, 1]


def np_work(wave, cplx, phase0: int, inc: int, amplitude, n: int):
    """(items of one work() call of n items, the phase after it)."""
    k = np.arange(n, dtype=np.uint64)
    ph = ((np.uint64(phase0 & 0xFFFFFFFF) + k * np.uint64(inc & 0xFFFFFFFF)) & np.uint64(0xFFFFFFFF)).astype(np.uint32)
    amp = np.float32(amplitude)
    cos = lambda: np_lookup(ph + np.uint32(0x40000000))  # noqa: E731  (wrapping u32 add)
    sin = lambda: np_lookup(ph)  # noqa: E731
    v = ph.view(np.int32)
    with np.errstate(all="ignore"):
        if not cplx:
            a = cos() if wave == COS else sin() if wave == SIN else np.where(v < 0, np.float32(1), np.float32(0))
            out = a.astype(np.float32) * amp
        else:
            if wave == SQUARE:
                t = v >> 30
                re = np.where(t < 0, np.float32(1), np.float32(0))
                im = np.where((t == -1) | (t == 0), np.float32(1), np.float32(0))
            else:
                re, im = cos(), sin()
            out = np.empty(2 * n, np.float32)
            out[0::2] = re.astype(np.float32) * amp
            out[1::2] = im.astype(np.float32) * amp
            out = out.view(np.complex64)
    nxt = (phase0 + n * inc) & 0xFFFFFFFF
    return out, nxt - (1 << 32) if nxt >= 1 << 31 else nxt
