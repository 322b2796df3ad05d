"""futuredsp filter cores on the GPU.

Mirrors ``futuredsp::Filter`` (crates/futuredsp/src/lib.rs:48-68): ``filter(input, output) ->
(consumed, produced, ComputationStatus)`` and ``length()``; stateless and re-entrant; the
caller owns both slices and ``output[produced:]`` is left unspecified.

``input``/``output`` are either torch CUDA tensors (device slices: asynchronous, ordered on
the context stream -- the in-flowgraph case, samples stay in HBM) or numpy arrays / CPU
tensors (host slices: the literal drop-in for the Rust call; the chunked H2D -> kernel -> D2H
pipeline runs inside the library and the call returns when ``output`` is filled).
"""
from __future__ import annotations

import ctypes as C
import enum

import numpy as np

from . import _lib
from ._lib import Handle, lib, check
from .context import Context, default_context


class ComputationStatus(enum.IntEnum):
    """futuredsp::ComputationStatus (lib.rs:33-45)."""
    InsufficientInput = 0
    InsufficientOutput = 1
    BothSufficient = 2


def _kind(sample_dtype, taps: np.ndarray) -> int:
    if np.dtype(sample_dtype) == np.float64:
        if np.iscomplexobj(taps):
            raise TypeError("no futuredsp impl for f64 samples with complex taps")
        return _lib.F64_F64                                  # fir.rs:217-226
    cin = np.dtype(sample_dtype) == np.complex64
    ctap = np.iscomplexobj(taps)
    if not cin and np.dtype(sample_dtype) != np.float32:
        raise TypeError("sample type must be float32 or complex64 (f32 / Complex<f32>)")
    if not cin and ctap:
        raise TypeError("no futuredsp impl for f32 samples with complex taps")
    return _lib.C32_C32 if ctap else (_lib.C32_F32 if cin else _lib.F32_F32)


def _taps_ptr(taps, kind):
    t = np.ascontiguousarray(taps, dtype=np.complex64 if kind == _lib.C32_C32 else np.float32)
    return t, t.view(np.float32).ctypes.data_as(C.POINTER(C.c_float))


def _is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


def _buf(x, want_dtype, writable=False):
    """-> (ptr, n_items, is_device, keepalive)"""
    if _is_torch(x):
        import torch
        td = {np.dtype(np.complex64): torch.complex64, np.dtype(np.float64): torch.float64}.get(np.dtype(want_dtype), torch.float32)
        if x.dtype != td:
            raise TypeError(f"expected {td}, got {x.dtype}")
        if not x.is_contiguous():
            raise ValueError("slices must be contiguous")
        return x.data_ptr(), x.numel(), x.is_cuda, x
    a = x if isinstance(x, np.ndarray) else np.asarray(x)
    if a.dtype != np.dtype(want_dtype):
        if writable:
            raise TypeError(f"output must be {np.dtype(want_dtype)}, got {a.dtype}")
        a = a.astype(want_dtype)
    if not a.flags.c_contiguous:
        if writable:
            raise ValueError("output must be contiguous")
        a = np.ascontiguousarray(a)
    return a.ctypes.data, a.size, False, a


class _FilterBase(Handle):
    _exec = None
    _host = None
    _length = None

    def __init__(self, ctx: Context | None):
        self.ctx = ctx or default_context()
        self._h = C.c_void_p()

    def length(self) -> int:
        """Filter::length (lib.rs:65-67)."""
        return int(type(self)._length(self._h))

    def filter(self, input, output):
        """Filter::filter (lib.rs:58-64). Returns (consumed, produced, ComputationStatus)."""
        ip, n_in, idev, _k1 = _buf(input, self.sample_dtype)
        op, n_out, odev, _k2 = _buf(output, self.sample_dtype, writable=True)
        if idev != odev:
            raise ValueError("input and output must both be device slices or both host slices")
        if idev and (input.device.index != self.ctx.device or output.device.index != self.ctx.device):
            raise ValueError(f"device slices must live on the filter's context device cuda:{self.ctx.device}")
        c, p, st = C.c_size_t(0), C.c_size_t(0), C.c_int32(0)
        fn = type(self)._exec if idev else type(self)._host
        if fn is None:
            raise NotImplementedError("host slices are not supported by this filter; pass CUDA tensors")
        check(fn(self._h, C.c_void_p(ip), n_in, C.c_void_p(op), n_out, C.byref(c), C.byref(p),
                 C.byref(st)), self.ctx.handle)
        return c.value, p.value, ComputationStatus(st.value)


class DecimatingFirFilter(_FilterBase):
    """futuredsp::DecimatingFirFilter (crates/futuredsp/src/decimating_fir.rs:31-95)."""
    _exec = lib.b2s_fir_exec
    _host = lib.b2s_fir_filter_host
    _destroy = lib.b2s_fir_destroy
    _length = lib.b2s_fir_length

    def __init__(self, decimation: int, taps, sample_dtype=np.complex64, ctx: Context | None = None,
                 algo: int = _lib.ALGO_AUTO):
        super().__init__(ctx)
        self.sample_dtype = np.dtype(sample_dtype)
        self.decimation = int(decimation)
        kind = _kind(sample_dtype, np.asarray(taps))
        if kind == _lib.F64_F64:
            t = np.ascontiguousarray(taps, dtype=np.float64)
            check(lib.b2s_fir_plan_f64_f64(self.ctx.handle, t.ctypes.data_as(C.POINTER(C.c_double)), t.size,
                                           self.decimation, C.byref(self._h)), self.ctx.handle)
        else:
            t, tp = _taps_ptr(taps, kind)
            check(lib.b2s_fir_plan(self.ctx.handle, kind, tp, t.size, self.decimation, C.byref(self._h)),
                  self.ctx.handle)
        if algo != _lib.ALGO_AUTO:
            self.set_algo(algo)

    def set_algo(self, algo: int):
        check(lib.b2s_fir_set_algo(self._h, algo), self.ctx.handle)

    @property
    def algo(self) -> int:
        return lib.b2s_fir_get_algo(self._h)


class FirFilter(DecimatingFirFilter):
    """futuredsp::FirFilter (crates/futuredsp/src/fir.rs:31-91)."""

    def __init__(self, taps, sample_dtype=np.complex64, ctx: Context | None = None,
                 algo: int = _lib.ALGO_AUTO):
        super().__init__(1, taps, sample_dtype, ctx, algo)


class IirFilter(_FilterBase):
    """futuredsp::IirFilter (crates/futuredsp/src/iir.rs:33-178), a ``StatefulFilter``: ``memory`` (the last n_a
    outputs, first filled with the stream's first n_a input samples) and the fill count live in the plan, so
    consecutive ``filter`` calls continue one stream.  f32 and f64 samples (the only impls, :56-76); device slices
    only.  ``algo``: ALGO_AUTO, ALGO_DIRECT (bit-exact sequential kernel) or ALGO_SCAN (chained scan, f32 stable
    filters; numerics in include/b200sdr.h)."""
    _exec = lib.b2s_iir_exec
    _host = None
    _destroy = lib.b2s_iir_destroy
    _length = lib.b2s_iir_length

    def __init__(self, a_taps, b_taps, sample_dtype=np.float32, ctx: Context | None = None,
                 algo: int = _lib.ALGO_AUTO):
        super().__init__(ctx)
        self.sample_dtype = np.dtype(sample_dtype)
        if self.sample_dtype == np.float64:
            ct, plan = C.c_double, lib.b2s_iir_plan_f64
        elif self.sample_dtype == np.float32:
            ct, plan = C.c_float, lib.b2s_iir_plan_f32
        else:
            raise TypeError("IirFilter has f32 x f32 and f64 x f64 impls only (iir.rs:56-76)")
        a = np.ascontiguousarray(np.asarray(a_taps, dtype=self.sample_dtype).reshape(-1))
        b = np.ascontiguousarray(np.asarray(b_taps, dtype=self.sample_dtype).reshape(-1))
        self.a_taps, self.b_taps = a, b
        check(plan(self.ctx.handle, a.ctypes.data_as(C.POINTER(ct)), a.size, b.ctypes.data_as(C.POINTER(ct)), b.size,
                   C.byref(self._h)), self.ctx.handle)
        if algo != _lib.ALGO_AUTO:
            self.set_algo(algo)

    def set_algo(self, algo: int):
        check(lib.b2s_iir_set_algo(self._h, algo), self.ctx.handle)

    @property
    def algo(self) -> int:
        return lib.b2s_iir_get_algo(self._h)


class PolyphaseResamplingFir(_FilterBase):
    """futuredsp::PolyphaseResamplingFir (crates/futuredsp/src/polyphase_resampling_fir.rs:42-124)."""
    _exec = lib.b2s_resamp_exec
    _host = None
    _destroy = lib.b2s_resamp_destroy
    _length = lib.b2s_resamp_length

    def __init__(self, interp: int, decim: int, taps, sample_dtype=np.complex64,
                 ctx: Context | None = None):
        super().__init__(ctx)
        self.sample_dtype = np.dtype(sample_dtype)
        self.interp, self.decim = int(interp), int(decim)
        t = np.asarray(taps)
        if np.iscomplexobj(t):
            raise TypeError("PolyphaseResamplingFir has f32 taps only (polyphase_resampling_fir.rs:126-167)")
        # Ensure number of taps is divisible by interp (polyphase_resampling_fir.rs:56)
        assert t.size % self.interp == 0, "taps.num_taps().is_multiple_of(interp)"
        kind = _kind(sample_dtype, t)
        t, tp = _taps_ptr(t, kind)
        check(lib.b2s_resamp_plan(self.ctx.handle, kind, tp, t.size, self.interp, self.decim,
                                  C.byref(self._h)), self.ctx.handle)
