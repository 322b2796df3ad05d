"""Exact references for the FIR, the decimating FIR and the rational resampler on integer data (test infrastructure).

With samples and taps that are small integers (|v| <= 8 here), every product and every partial sum of these filters is
an integer below 2^24, so every correct f32 kernel returns the exact sum whatever its summation order or FMA use, and
the split-bf16 tensor kernel does too (integers up to 256 are exact in bf16: the lo parts are zero).  Any wrong tap,
sample, phase, tile seam or slot then moves an output by at least one unit.

The references below are exact: float64 arithmetic on integer values below 2^53 (np.convolve, a gather), or a float64
FFT convolution rounded with rint for long inputs, which asserts that it was within 1e-3 of an integer before rounding.
The (consumed, produced, status) counts come from the CPU oracle (oracle.fir / decim_fir / resamp_fir).
"""
from __future__ import annotations

import numpy as np

import oracle as orc

LIM = 8                       # samples and taps in [-LIM, LIM]
_DIRECT_MACS = 1 << 26        # np.convolve up to this many multiply-adds, FFT convolution above


def int_samples(rng, n, cplx, lim=LIM):
    """n seeded integer samples in [-lim, lim] (re and im drawn independently): float32 or complex64."""
    re = rng.integers(-lim, lim + 1, n)
    if not cplx:
        return re.astype(np.float32)
    return (re + 1j * rng.integers(-lim, lim + 1, n)).astype(np.complex64)


def int_taps(rng, n, cplx=False, lim=LIM):
    """n seeded integer taps in [-lim, lim], never a constant vector for n >= 2 (AUTO keeps constant taps off the
    tensor kernel)."""
    while True:
        t = int_samples(rng, n, cplx, lim)
        if n < 2 or np.any(t != t[0]):
            return t


def conv_valid(x, taps):
    """np.convolve(x, taps, "valid") exactly, for integer-valued x and taps (real or complex)."""
    x = np.asarray(x, np.complex128 if np.iscomplexobj(x) else np.float64)
    h = np.asarray(taps, np.complex128 if np.iscomplexobj(taps) else np.float64)
    if x.size < h.size:
        return np.zeros(0, np.result_type(x, h))
    if x.size * h.size <= _DIRECT_MACS:
        return np.convolve(x, h, "valid")
    from scipy.signal import oaconvolve
    y = oaconvolve(x, h, "valid")
    r = np.rint(y.real) + 1j * np.rint(y.imag) if np.iscomplexobj(y) else np.rint(y)
    err = float(np.max(np.abs(y - r))) if y.size else 0.0
    assert err < 1e-3, f"FFT reference is not provably exact: {err} from an integer"
    return r


def fir(taps, x, decim=1, n_out=None):
    """o[k] = sum_t x[D-1 + k*D + t] * taps[N-1-t] for every k the input allows (first n_out of them)."""
    y = conv_valid(x, taps)[decim - 1::decim]
    return y if n_out is None else y[:n_out]


def resamp(taps, interp, decim, x, n_out):
    """o[k] = sum_t x[floor(k*M/L) + t] * taps[L*(T-1-t) + (k*M mod L)] for k < n_out (all must be computable)."""
    L, M = int(interp), int(decim)
    T = len(taps) // L
    xx = np.asarray(x, np.complex128 if np.iscomplexobj(x) else np.float64)
    banks = np.asarray(taps, np.float64).reshape(T, L)[::-1, :]          # banks[t, b] = taps[L*(T-1-t) + b]
    out = np.zeros(n_out, xx.dtype)
    step = max(1, (1 << 22) // max(T, 1))
    for k0 in range(0, n_out, step):
        k = np.arange(k0, min(k0 + step, n_out), dtype=np.int64)
        s, b = (k * M) // L, (k * M) % L
        assert s[-1] + T <= xx.size, "resamp: n_out needs more input"
        out[k0:k0 + k.size] = np.einsum("kt,tk->k", xx[s[:, None] + np.arange(T)], banks[:, b])
    return out


def fir_counts(n_in, ntaps, decim, out_cap):
    """(consumed, produced, status) of DecimatingFirFilter::filter, from the oracle.  They depend on n_in and ntaps
    only through n_in + 1 - ntaps, so the oracle runs a one-tap filter on n_in + 1 - ntaps zeros (cheap for any n)."""
    c, p, st, _ = orc.decim_fir(np.ones(1, np.float32), decim, np.zeros(max(n_in + 1 - ntaps, 0), np.float32), out_cap)
    return c, p, st


def resamp_counts(n_in, interp, decim, T, out_cap):
    """(consumed, produced, status) of PolyphaseResamplingFir::filter, from the oracle (T = ntaps / interp); like
    fir_counts, through a one-tap-per-bank design on n_in + 1 - T zeros."""
    c, p, st, _ = orc.resamp_fir(np.ones(interp, np.float32), interp, decim,
                                 np.zeros(max(n_in + 1 - T, 0), np.float32), out_cap)
    return c, p, st
