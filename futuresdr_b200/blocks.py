"""Block-level mirror of the reference's hot-path blocks, over device-resident buffers.

Reference interfaces mirrored (names, argument meaning and finish rules):
  * ``Fir`` / ``FirBuilder``      src/blocks/fir.rs:13-95, :126-233
  * ``Iir`` / ``IirBuilder``      src/blocks/iir.rs:8-176
  * ``SignalSource`` / ``SignalSourceBuilder`` / ``FixedPointPhase``   src/blocks/signal_source/{mod,fxpt_phase}.rs
  * ``Head``                      src/blocks/head.rs:22-84
  * ``Fft`` / ``FftDirection``    src/blocks/fft.rs:30-221
  * ``Apply``                     src/blocks/apply.rs:100-131 (closed catalogue of closures)
  * ``PfbArbResampler``           src/blocks/pfb/arb_resampler.rs:72-231
  * ``WorkIo``                    src/runtime/work_io.rs:11-34
  * ``Mocker``                    src/runtime/mocker.rs:33-190 (single-block harness)

A block's ``work(io)`` does what ``Kernel::work`` does: take the input/output slices of its
ports, call the core, ``consume``/``produce``, set ``io.finished`` by the reference's rule.
Ports here are device slices (torch CUDA tensors): samples stay in HBM between blocks.
"""
from __future__ import annotations

import ctypes as C
import enum
from dataclasses import dataclass
from typing import Optional

import numpy as np
import torch

from . import _lib, firdes
from ._lib import Handle, lib, check
from .context import Context, default_context
from .filters import (ComputationStatus, DecimatingFirFilter, FirFilter, IirFilter, PolyphaseResamplingFir,
                      _FilterBase)


@dataclass
class WorkIo:
    """runtime::WorkIo (work_io.rs:11-34)."""
    call_again: bool = False
    finished: bool = False


def _tdtype(np_dtype):
    return {np.dtype(np.complex64): torch.complex64, np.dtype(np.float64): torch.float64}.get(np.dtype(np_dtype),
                                                                                             torch.float32)


def _ctx_device(ctx) -> torch.device:
    """The device a block's context lives on: every port buffer of the block is allocated THERE (not on whatever
    device happens to be current), so the pointers handed to the C ABI belong to the context's GPU."""
    return torch.device("cuda", ctx.device) if ctx is not None else torch.device("cuda", torch.cuda.current_device())


class Reader:
    """mocker::Reader<T> (mocker.rs:213-290): a vector that reports finished() == true."""

    def __init__(self, dtype, device=None):
        self.dtype = np.dtype(dtype)
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.data = torch.zeros(0, dtype=_tdtype(dtype), device=self.device)
        self.pos = 0
        self._finished = True
        self.min_items = 1

    def set(self, data):
        if isinstance(data, torch.Tensor):
            if data.is_cuda and data.device != self.device:
                raise ValueError(f"input slice lives on {data.device}, the block's context on {self.device}")
            t = data.to(device=self.device, dtype=_tdtype(self.dtype))
        else:
            t = torch.from_numpy(np.ascontiguousarray(np.asarray(data), dtype=self.dtype)).to(self.device)
        self.data, self.pos = t.contiguous(), 0

    def slice(self) -> torch.Tensor:
        return self.data[self.pos:]

    def consume(self, n: int):
        assert self.pos + n <= self.data.numel()
        self.pos += n

    def finished(self) -> bool:
        return self._finished

    def set_min_items(self, n: int):
        self.min_items = max(self.min_items, n)


class Writer:
    """mocker::Writer<T> (mocker.rs:326-400): a vector with reserved capacity."""

    def __init__(self, dtype, device=None):
        self.dtype = np.dtype(dtype)
        self.device = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.data = torch.zeros(0, dtype=_tdtype(dtype), device=self.device)
        self.len = 0
        self.min_items = 1

    def reserve(self, n: int):
        self.data = torch.zeros(n, dtype=_tdtype(self.dtype), device=self.device)
        self.len = 0

    def slice(self) -> torch.Tensor:
        return self.data[self.len:]

    def produce(self, n: int):
        assert self.len + n <= self.data.numel()
        self.len += n

    def get(self) -> torch.Tensor:
        return self.data[: self.len]

    def set_min_items(self, n: int):
        self.min_items = max(self.min_items, n)


class Block:
    in_dtype = np.complex64
    out_dtype = np.complex64

    def _ports(self):
        ctx = getattr(self, "ctx", None) or getattr(getattr(self, "filter", None), "ctx", None)
        dev = _ctx_device(ctx)
        self.input = Reader(self.in_dtype, dev)
        self.output = Writer(self.out_dtype, dev)

    def work(self, io: WorkIo):          # pragma: no cover
        raise NotImplementedError


class Fir(Block):
    """blocks::Fir (src/blocks/fir.rs:13-95): generic over a ``Filter`` core."""

    def __init__(self, filter: _FilterBase):
        self.filter = filter
        self.in_dtype = self.out_dtype = filter.sample_dtype
        self._ports()
        self.input.set_min_items(filter.length())            # fir.rs:49

    def n_taps(self) -> int:
        return self.filter.length()

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()        # fir.rs:81-82
        consumed, produced, status = self.filter.filter(i, o)
        self.input.consume(consumed)
        self.output.produce(produced)
        if self.input.finished() and status != ComputationStatus.InsufficientOutput:   # fir.rs:89-91
            io.finished = True


class FirBuilder:
    """blocks::FirBuilder (src/blocks/fir.rs:126-233)."""

    @staticmethod
    def fir(taps, sample_dtype=np.complex64, ctx: Optional[Context] = None) -> Fir:
        return Fir(FirFilter(taps, sample_dtype, ctx))

    @staticmethod
    def decimating(decim: int, sample_dtype=np.complex64, ctx: Optional[Context] = None) -> Fir:
        taps = firdes.kaiser.lowpass(1.0 / decim, 0.1, 0.0001)                  # fir.rs:154
        return FirBuilder.decimating_with_taps(decim, taps, sample_dtype, ctx)

    @staticmethod
    def decimating_with_taps(decim: int, taps, sample_dtype=np.complex64, ctx=None) -> Fir:
        return Fir(DecimatingFirFilter(decim, taps, sample_dtype, ctx))

    @staticmethod
    def resampling(interp: int, decim: int, sample_dtype=np.complex64, ctx=None) -> Fir:
        g = int(np.gcd(interp, decim))                                          # fir.rs:197-199
        interp, decim = interp // g, decim // g
        taps = firdes.kaiser.multirate(interp, decim, 12, 0.0001)               # fir.rs:201
        return FirBuilder.resampling_with_taps(interp, decim, taps, sample_dtype, ctx)

    @staticmethod
    def resampling_with_taps(interp: int, decim: int, taps, sample_dtype=np.complex64, ctx=None) -> Fir:
        return Fir(PolyphaseResamplingFir(interp, decim, taps, sample_dtype, ctx))


class Iir(Block):
    """blocks::Iir (src/blocks/iir.rs:8-176): generic over a ``StatefulFilter`` core (an ``IirFilter``)."""

    def __init__(self, core: IirFilter):
        self.filter = core
        self.in_dtype = self.out_dtype = core.sample_dtype
        self._ports()
        self.input.set_min_items(core.length())              # iir.rs:133

    @classmethod
    def new(cls, a_taps, b_taps, sample_dtype=np.float32, ctx: Optional[Context] = None) -> "Iir":
        return cls(IirFilter(a_taps, b_taps, sample_dtype, ctx))

    @classmethod
    def with_core(cls, core: IirFilter) -> "Iir":
        return cls(core)

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()        # iir.rs:162-163
        consumed, produced, status = self.filter.filter(i, o)
        self.input.consume(consumed)
        self.output.produce(produced)
        if self.input.finished() and status != ComputationStatus.InsufficientOutput:   # iir.rs:170-172
            io.finished = True


class IirBuilder:
    """blocks::IirBuilder (src/blocks/iir.rs:32-64)."""

    @staticmethod
    def iir(a_taps, b_taps, sample_dtype=np.float32, ctx: Optional[Context] = None) -> Iir:
        return Iir(IirFilter(a_taps, b_taps, sample_dtype, ctx))

    @staticmethod
    def same_type(a_taps, b_taps, sample_dtype=np.float32, ctx: Optional[Context] = None) -> Iir:
        return IirBuilder.iir(a_taps, b_taps, sample_dtype, ctx)


class FixedPointPhase:
    """blocks::FixedPointPhase (src/blocks/signal_source/fxpt_phase.rs:8-99): a phase as a wrapping i32, -2^31 = -pi.
    ``new``, ``sin`` and ``cos`` run on the host through the library (b2s_fxpt_phase_new / b2s_fxpt_sin_cos)."""

    def __init__(self, value: int):
        v = int(value) & 0xFFFFFFFF
        self.value = v - (1 << 32) if v >= 1 << 31 else v

    @classmethod
    def new(cls, x: float) -> "FixedPointPhase":
        v = C.c_int32(0)
        check(lib.b2s_fxpt_phase_new(float(np.float32(x)), C.byref(v)))
        return cls(v.value)

    def _sin_cos(self):
        s, c = C.c_float(0.0), C.c_float(0.0)
        check(lib.b2s_fxpt_sin_cos(self.value, C.byref(s), C.byref(c)))
        return np.float32(s.value), np.float32(c.value)

    def sin(self) -> np.float32:
        return self._sin_cos()[0]

    def cos(self) -> np.float32:
        return self._sin_cos()[1]


class SignalWave(enum.IntEnum):
    """The phase-to-amplitude closures of SignalSourceBuilder (b2s_wave)."""
    Cos = _lib.WAVE_COS
    Sin = _lib.WAVE_SIN
    Square = _lib.WAVE_SQUARE


class SignalSource(Block, Handle):
    """blocks::SignalSource (src/blocks/signal_source/mod.rs:29-108): a source without an input port.  Each ``work``
    fills the whole output slice and the block never finishes; the samples are bit-identical to the reference's."""
    _destroy = lib.b2s_sigsrc_destroy
    in_dtype = None

    def __init__(self, wave: SignalWave, frequency: float, sample_rate: float, amplitude: float,
                 initial_phase: float, dtype=np.float32, ctx: Optional[Context] = None):
        self.out_dtype = np.dtype(dtype)
        if self.out_dtype not in (np.dtype(np.float32), np.dtype(np.complex64)):
            raise ValueError(f"SignalSource: f32 or Complex32 items, not {self.out_dtype}")
        self.ctx = ctx or default_context()
        self.wave = SignalWave(wave)
        self._h = C.c_void_p()
        check(lib.b2s_sigsrc_create(self.ctx.handle, int(self.wave), int(self.out_dtype == np.complex64),
                                    float(np.float32(frequency)), float(np.float32(sample_rate)),
                                    float(np.float32(amplitude)), float(np.float32(initial_phase)), C.byref(self._h)),
              self.ctx.handle)
        self.input = None
        self.output = Writer(self.out_dtype, _ctx_device(self.ctx))

    def set_amplitude(self, amplitude: float):
        """SignalSource::set_amplitude (mod.rs:71-73): applies from the next call."""
        check(lib.b2s_sigsrc_set_amplitude(self._h, float(np.float32(amplitude))), self.ctx.handle)

    def phase(self) -> tuple[FixedPointPhase, FixedPointPhase]:
        """(the next sample's phase, the per-sample increment) of the NCO."""
        v, inc = C.c_int32(0), C.c_int32(0)
        check(lib.b2s_sigsrc_phase(self._h, C.byref(v), C.byref(inc)), self.ctx.handle)
        return FixedPointPhase(v.value), FixedPointPhase(inc.value)

    def generate(self, o: torch.Tensor) -> int:
        """Fill the device slice ``o`` (asynchronous on the context's stream); returns the items written."""
        p = C.c_size_t(0)
        check(lib.b2s_sigsrc_exec(self._h, C.c_void_p(o.data_ptr()), o.numel(), C.byref(p)), self.ctx.handle)
        return p.value

    def work(self, io: WorkIo):
        o = self.output.slice()                                                 # mod.rs:94-104
        self.output.produce(self.generate(o))


class SignalSourceBuilder:
    """blocks::SignalSourceBuilder (src/blocks/signal_source/mod.rs:110-227); ``dtype`` picks the item type (the
    reference's type parameter): np.float32 or np.complex64."""

    @staticmethod
    def cos(frequency, sample_rate, amplitude, initial_phase, dtype=np.float32, ctx=None) -> SignalSource:
        return SignalSource(SignalWave.Cos, frequency, sample_rate, amplitude, initial_phase, dtype, ctx)

    @staticmethod
    def sin(frequency, sample_rate, amplitude, initial_phase, dtype=np.float32, ctx=None) -> SignalSource:
        return SignalSource(SignalWave.Sin, frequency, sample_rate, amplitude, initial_phase, dtype, ctx)

    @staticmethod
    def square(frequency, sample_rate, amplitude, initial_phase, dtype=np.float32, ctx=None) -> SignalSource:
        return SignalSource(SignalWave.Square, frequency, sample_rate, amplitude, initial_phase, dtype, ctx)


class Head(Block):
    """blocks::Head (src/blocks/head.rs:22-84): copies the first ``n_items`` input items and finishes once it has
    copied them all -- not when its input finishes."""

    def __init__(self, dtype, n_items: int, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.in_dtype = self.out_dtype = np.dtype(dtype)
        self.n_items = int(n_items)
        self._ports()

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()                          # head.rs:63-83
        m = min(self.n_items, i.numel(), o.numel())
        if m > 0:
            check(lib.b2s_memcpy_d2d(self.ctx.handle, C.c_void_p(o.data_ptr()), C.c_void_p(i.data_ptr()),
                                     m * self.in_dtype.itemsize), self.ctx.handle)
            self.n_items -= m
            if self.n_items == 0:
                io.finished = True
            self.input.consume(m)
            self.output.produce(m)


class FftDirection(enum.Enum):
    """blocks::FftDirection (fft.rs:48-54)."""
    Forward = 0
    Inverse = 1


class Fft(Block, Handle):
    """blocks::Fft (src/blocks/fft.rs:30-221)."""
    _destroy = lib.b2s_fft_destroy

    def __init__(self, len: int, direction: FftDirection = FftDirection.Forward, fft_shift: bool = False,
                 normalize: Optional[float] = None, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.len, self.direction, self.fft_shift, self.normalize = int(len), direction, fft_shift, normalize
        self._h = C.c_void_p()
        check(lib.b2s_fft_plan_c32(self.ctx.handle, self.len, int(direction == FftDirection.Inverse),
                                   int(fft_shift), int(normalize is not None), float(normalize or 0.0),
                                   C.byref(self._h)), self.ctx.handle)
        self._ports()
        self.input.set_min_items(self.len)
        self.output.set_min_items(self.len)

    @classmethod
    def with_direction(cls, len, direction):
        return cls(len, direction)

    @classmethod
    def with_options(cls, len, direction, fft_shift, normalize):
        return cls(len, direction, fft_shift, normalize)

    def fft_size(self, p=None):
        """The `fft_size` message handler (fft.rs:124-136): an integer re-plans (`set_fft_size`, :139-151) and answers
        "Ok"; ``None`` (Pmt::Null) answers the current length; anything else "InvalidValue"."""
        if p is None:
            return self.len
        if isinstance(p, (int, np.integer)) and not isinstance(p, bool):
            self.set_fft_size(int(p))
            return "Ok"
        return "InvalidValue"

    def set_fft_size(self, new_len: int):
        """Fft::set_fft_size (fft.rs:139-151): a new plan of the same direction / shift / normalisation.  The new plan is
        built first, so a length this build cannot plan leaves the block as it was."""
        h = C.c_void_p()
        check(lib.b2s_fft_plan_c32(self.ctx.handle, int(new_len), int(self.direction == FftDirection.Inverse),
                                   int(self.fft_shift), int(self.normalize is not None), float(self.normalize or 0.0),
                                   C.byref(h)), self.ctx.handle)
        lib.b2s_fft_destroy(self._h)
        self._h, self.len = h, int(new_len)

    def transform(self, i: torch.Tensor, o: torch.Tensor):
        """The body of Fft::work on explicit slices. Returns m (= consumed = produced)."""
        c, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_fft_exec(self._h, C.c_void_p(i.data_ptr()), i.numel(), C.c_void_p(o.data_ptr()),
                               o.numel(), C.byref(c), C.byref(p)), self.ctx.handle)
        return c.value

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()
        m = self.transform(i, o) if min(i.numel(), o.numel()) >= self.len else 0
        if m > 0:
            self.input.consume(m)
            self.output.produce(m)
        if self.input.finished() and m == (m // self.len) * self.len:           # fft.rs:216-218
            io.finished = True


class ApplyOp(enum.IntEnum):
    """The closures of the reference graphs that exist as device ops (b2s_op)."""
    ScaleF32 = _lib.OP_SCALE_F32
    ScaleC32 = _lib.OP_SCALE_C32
    QuadDemod = _lib.OP_QUAD_DEMOD
    NormSqr = _lib.OP_NORM_SQR
    QuadDemodC32 = _lib.OP_QUAD_DEMOD_C32
    ExpF32 = _lib.OP_EXP_F32
    MagC32 = _lib.OP_MAG_C32
    Log10F32 = _lib.OP_LOG10_F32


_APPLY_TYPES = {
    ApplyOp.ScaleF32: (np.float32, np.float32), ApplyOp.ScaleC32: (np.complex64, np.complex64),
    ApplyOp.QuadDemod: (np.complex64, np.float32), ApplyOp.NormSqr: (np.complex64, np.float32),
    ApplyOp.QuadDemodC32: (np.complex64, np.complex64), ApplyOp.ExpF32: (np.float32, np.float32),
    ApplyOp.MagC32: (np.complex64, np.float32), ApplyOp.Log10F32: (np.float32, np.float32),
}


class Apply(Block, Handle):
    """blocks::Apply (src/blocks/apply.rs:42-131) for the catalogue of closures in ApplyOp.
    Stateful closures (the FM demodulator's ``last`` sample) keep their state on the device."""
    _destroy = lib.b2s_apply_destroy

    def __init__(self, op: ApplyOp, param: float = 1.0, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.op = ApplyOp(op)
        self.in_dtype, self.out_dtype = _APPLY_TYPES[self.op]
        self._h = C.c_void_p()
        check(lib.b2s_apply_create(self.ctx.handle, int(self.op), float(param), C.byref(self._h)), self.ctx.handle)
        self._ports()

    def apply(self, i: torch.Tensor, o: torch.Tensor) -> int:
        c, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_apply_exec(self._h, C.c_void_p(i.data_ptr()), i.numel(), C.c_void_p(o.data_ptr()),
                                 o.numel(), C.byref(c), C.byref(p)), self.ctx.handle)
        return c.value

    def reset(self):
        check(lib.b2s_apply_reset(self._h), self.ctx.handle)

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()
        i_len = i.numel()
        m = min(i_len, o.numel())                                               # apply.rs:109
        if m > 0:
            self.apply(i, o)
            self.input.consume(m)
            self.output.produce(m)
        if self.input.finished() and m == i_len:                                 # apply.rs:126-128
            io.finished = True


class PfbArbResampler(Block, Handle):
    """blocks::PfbArbResampler (src/blocks/pfb/arb_resampler.rs:72-231)."""
    _destroy = lib.b2s_pfbarb_destroy

    def __init__(self, rate: float, taps, num_filters: int, ctx: Optional[Context] = None):
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        # validate input (arb_resampler.rs:92-104: the reference asserts)
        assert rate > 0.0, "PfbArbResampler: resampling rate must be greater than zero"
        assert taps.size >= num_filters, "PfbArbResampler: prototype filter length must be at least num_filters"
        assert num_filters != 0, "PfbArbResampler: number of filter banks must be greater than zero"
        self.ctx = ctx or default_context()
        self.rate = np.float32(rate)
        self._h = C.c_void_p()
        check(lib.b2s_pfbarb_plan_c32(self.ctx.handle, taps.ctypes.data_as(C.POINTER(C.c_float)), taps.size,
                                      int(num_filters), float(rate), C.byref(self._h)), self.ctx.handle)
        self._ports()
        self.output.set_min_items(int(np.ceil(rate)))                           # arb_resampler.rs:109

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()
        c, p, ca = C.c_size_t(0), C.c_size_t(0), C.c_int32(0)
        check(lib.b2s_pfbarb_exec(self._h, C.c_void_p(i.data_ptr()), i.numel(), C.c_void_p(o.data_ptr()),
                                  o.numel(), C.byref(c), C.byref(p), C.byref(ca)), self.ctx.handle)
        ninput = i.numel()
        self.input.consume(c.value)
        self.output.produce(p.value)
        if ca.value:
            io.call_again = True
        elif ninput - c.value == 0 and self.input.finished():                    # :208-211, :227-229
            io.finished = True

    def reset(self):
        check(lib.b2s_pfbarb_reset(self._h), self.ctx.handle)


class Rotator(Handle):
    """futuredsp::Rotator (crates/futuredsp/src/rotator.rs:13-48): mixer / frequency shifter whose
    phase recurrence is replayed bit-for-bit (see csrc/rotator.cu)."""
    _destroy = lib.b2s_rotator_destroy

    def __init__(self, phase_incr: float, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self._h = C.c_void_p()
        check(lib.b2s_rotator_create(self.ctx.handle, float(np.float32(phase_incr)), C.byref(self._h)), self.ctx.handle)

    def rotate(self, input: torch.Tensor, output: torch.Tensor):
        """Rotator::rotate -> (n, ComputationStatus)."""
        n, st = C.c_size_t(0), C.c_int32(0)
        check(lib.b2s_rotator_exec(self._h, C.c_void_p(input.data_ptr()), input.numel(),
                                   C.c_void_p(output.data_ptr()), output.numel(), C.byref(n), C.byref(st)),
              self.ctx.handle)
        return n.value, ComputationStatus(st.value)

    def rotate_inplace(self, buffer: torch.Tensor):
        self.rotate(buffer, buffer)

    def reset(self):
        check(lib.b2s_rotator_reset(self._h), self.ctx.handle)


class XlatingFir(Block):
    """blocks::XlatingFir (src/blocks/xlating_fir.rs:22-126): decimating FIR with band-pass complex
    taps followed by a Rotator at the output rate."""

    def __init__(self, decimation: int, offset: float, sample_rate: float, taps=None,
                 ctx: Optional[Context] = None):
        if taps is None:                                                        # XlatingFir::new (:42-48)
            assert decimation >= 2, "Xlating FIR: Decimation has to be >= 2"
            transition_bw = 0.1
            cutoff = min(0.5 - transition_bw - np.finfo(np.float64).eps, 1.0 / decimation)
            taps = firdes.kaiser.lowpass(cutoff, transition_bw, 0.0001)
        assert decimation != 0
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        bpf = np.zeros(taps.size, np.complex64)
        incr = C.c_float(0.0)
        check(lib.b2s_xlating_taps(taps.ctypes.data_as(C.POINTER(C.c_float)), taps.size, float(np.float32(offset)),
                                   float(np.float32(sample_rate)), int(decimation),
                                   bpf.view(np.float32).ctypes.data_as(C.POINTER(C.c_float)), C.byref(incr)))
        self.filter = DecimatingFirFilter(decimation, bpf, np.complex64, ctx)
        self.rotator = Rotator(incr.value, ctx)
        self._ports()

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()
        consumed, produced, status = self.filter.filter(i, o)
        if produced:
            self.rotator.rotate_inplace(o[:produced])                           # xlating_fir.rs:118
        self.input.consume(consumed)
        self.output.produce(produced)
        if self.input.finished() and status != ComputationStatus.InsufficientOutput:
            io.finished = True


class PfbSynthesizer(Block, Handle):
    """blocks::PfbSynthesizer (src/blocks/pfb/synthesizer.rs:32-144): N input streams (one channel-major
    device buffer ``inputs`` [N, n] with per-call read position), one output stream."""
    _destroy = lib.b2s_synth_destroy

    def __init__(self, num_channels: int, taps, ctx: Optional[Context] = None):
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        self.ctx = ctx or default_context()
        self.num_channels = int(num_channels)
        self._h = C.c_void_p()
        check(lib.b2s_synth_plan_c32(self.ctx.handle, self.num_channels, taps.ctypes.data_as(C.POINTER(C.c_float)),
                                     taps.size, C.byref(self._h)), self.ctx.handle)
        self.inputs = torch.zeros(self.num_channels, 0, dtype=torch.complex64, device=_ctx_device(self.ctx))
        self.in_pos = 0
        self.inputs_finished = True
        self.output = Writer(np.complex64, _ctx_device(self.ctx))

    def set_inputs(self, x):
        t = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x, dtype=np.complex64))
        self.inputs = t.to(device=_ctx_device(self.ctx), dtype=torch.complex64).contiguous()
        assert self.inputs.shape[0] == self.num_channels
        self.in_pos = 0

    def work(self, io: WorkIo):
        n_in = self.inputs.shape[1] - self.in_pos
        o = self.output.slice()
        c, p = C.c_size_t(0), C.c_size_t(0)
        in_ptr = self.inputs.data_ptr() + 8 * self.in_pos
        check(lib.b2s_synth_exec(self._h, C.c_void_p(in_ptr), self.inputs.shape[1], n_in, C.c_void_p(o.data_ptr()),
                                 o.numel(), C.byref(c), C.byref(p)), self.ctx.handle)
        self.in_pos += c.value
        self.output.produce(p.value)
        if n_in - c.value == 0 and self.inputs_finished:                          # :131-141
            io.finished = True


class MovingAvg(Block, Handle):
    """blocks::MovingAvg<WIDTH> (src/blocks/moving_avg.rs:24-116): exponential average per bin over
    consecutive WIDTH-item chunks, one output chunk every ``history_size`` input chunks."""
    _destroy = lib.b2s_mavg_destroy
    in_dtype = np.float32
    out_dtype = np.float32

    def __init__(self, width: int, decay_factor: float, history_size: int, ctx: Optional[Context] = None):
        assert 0.0 <= decay_factor <= 1.0, "decay_factor must be in [0, 1]"       # moving_avg.rs:58-61
        self.ctx = ctx or default_context()
        self.width = int(width)
        self._h = C.c_void_p()
        check(lib.b2s_mavg_create(self.ctx.handle, self.width, float(decay_factor), int(history_size),
                                  C.byref(self._h)), self.ctx.handle)
        self._ports()

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()
        input_len = i.numel()
        c, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_mavg_exec(self._h, C.c_void_p(i.data_ptr()), input_len, C.c_void_p(o.data_ptr()), o.numel(),
                                C.byref(c), C.byref(p)), self.ctx.handle)
        if self.input.finished() and c.value // self.width == input_len // self.width:     # :106-108
            io.finished = True
        self.input.consume(c.value)
        self.output.produce(p.value)


class SpectrumPipe(Block, Handle):
    """The spectrum flowgraph's compute chain as ONE block (SURVEY 8f-3): ``Fft::with_options(n, Forward,
    fft_shift, None)`` -> ``Apply(|x|^2)`` -> ``MovingAvg<n>::new(decay_factor, history_size)`` of
    examples/spectrum/src/bin/cpu.rs:21-28, optionally followed by ``log10_scale * log10(.)`` (what the
    reference's CubeCL kernel fuses, perf/burn/src/bin/fft-cubecl-kernel.rs:115-146).  Complex<f32> in, f32 out;
    only 8 B/sample in and ``n`` floats per ``history_size`` frames out touch HBM.  Values agree with the three
    separate blocks to rounding (blocked-scan evaluation of the average), counts are MovingAvg's."""
    _destroy = lib.b2s_spectrum_destroy
    in_dtype = np.complex64
    out_dtype = np.float32

    def __init__(self, n: int, decay_factor: float, history_size: int, fft_shift: bool = True,
                 log10_scale: float = 0.0, ctx: Optional[Context] = None):
        assert 0.0 <= decay_factor <= 1.0, "decay_factor must be in [0, 1]"       # moving_avg.rs:58-61
        self.ctx = ctx or default_context()
        self.n = int(n)
        self._h = C.c_void_p()
        check(lib.b2s_spectrum_plan(self.ctx.handle, self.n, int(bool(fft_shift)), float(decay_factor), int(history_size),
                                    float(log10_scale), C.byref(self._h)), self.ctx.handle)
        self._ports()

    def process(self, x: torch.Tensor, out: torch.Tensor):
        """(consumed items, produced floats) for device slices -- the call ``work`` makes."""
        c, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_spectrum_exec(self._h, C.c_void_p(x.data_ptr()), x.numel(), C.c_void_p(out.data_ptr()), out.numel(),
                                    C.byref(c), C.byref(p)), self.ctx.handle)
        return c.value, p.value

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()
        input_len = i.numel()
        c, p = self.process(i, o)
        if self.input.finished() and c // self.n == input_len // self.n:          # moving_avg.rs:106-108
            io.finished = True
        self.input.consume(c)
        self.output.produce(p)

    def reset(self):
        check(lib.b2s_spectrum_reset(self._h), self.ctx.handle)


class PfbChannelizer(Block, Handle):
    """blocks::PfbChannelizer (src/blocks/pfb/channelizer.rs:72-223): one input, N output streams.
    The N output ports share one channel-major device buffer ``outputs`` of shape [N, capacity];
    ``produced`` items have been written to every row."""
    _destroy = lib.b2s_chan_destroy

    def __init__(self, num_channels: int, taps, oversample_rate: float = 1.0, ctx: Optional[Context] = None):
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        # validate input (channelizer.rs:92-104: the reference asserts)
        assert num_channels > 2, "PfbChannelizer: number of channels must be at least 2"
        assert taps.size >= num_channels, "PfbChannelizer: prototype filter length must be at least num_channels"
        assert oversample_rate != 0.0 and (num_channels % oversample_rate) == 0.0, \
            "pfb_channelizer: oversample rate must be N/i for i in [1, N]"
        self.ctx = ctx or default_context()
        self.num_channels = int(num_channels)
        self._h = C.c_void_p()
        check(lib.b2s_chan_plan_c32(self.ctx.handle, self.num_channels, taps.ctypes.data_as(C.POINTER(C.c_float)),
                                    taps.size, float(oversample_rate), C.byref(self._h)), self.ctx.handle)
        self.decimation_factor = int(lib.b2s_chan_decimation(self._h))
        self.input = Reader(np.complex64, _ctx_device(self.ctx))
        self.outputs = torch.zeros(self.num_channels, 0, dtype=torch.complex64, device=_ctx_device(self.ctx))
        self.produced = 0

    def reserve_outputs(self, n: int):
        self.outputs = torch.zeros(self.num_channels, n, dtype=torch.complex64, device=_ctx_device(self.ctx))
        self.produced = 0

    def work(self, io: WorkIo):
        i = self.input.slice()
        cap = self.outputs.shape[1] - self.produced
        c, p, ca = C.c_size_t(0), C.c_size_t(0), C.c_int32(0)
        out_ptr = self.outputs.data_ptr() + 8 * self.produced
        check(lib.b2s_chan_exec(self._h, C.c_void_p(i.data_ptr()), i.numel(), C.c_void_p(out_ptr),
                                self.outputs.shape[1], cap, C.byref(c), C.byref(p), C.byref(ca)), self.ctx.handle)
        n_in = i.numel()
        self.input.consume(c.value)
        self.produced += p.value
        if ca.value:
            io.call_again = True
        elif n_in - c.value < self.decimation_factor and self.input.finished():      # :214-218
            io.finished = True


class Mocker:
    """runtime::mocker::Mocker (src/runtime/mocker.rs:33-190): run ONE block without a scheduler."""

    def __init__(self, block: Block):
        self.block = block

    def input(self, data):
        self.block.input.set(data)

    def init_output(self, n: int):
        self.block.output.reserve(n)

    def run(self, max_calls: int = 1 << 20):
        """Loop work() while call_again is set (mocker.rs:159-190)."""
        calls = 0
        while True:
            io = WorkIo()
            self.block.work(io)
            calls += 1
            if not io.call_again or calls >= max_calls:
                break
        self.block.filter.ctx.sync() if hasattr(self.block, "filter") else torch.cuda.synchronize()
        return io

    def run_until_finished(self, max_calls: int = 1 << 20):
        """Keep calling work() until the block reports finished or makes no progress."""
        for _ in range(max_calls):
            before = (self.block.input.pos, self.block.output.len)
            io = WorkIo()
            self.block.work(io)
            if io.finished:
                break
            if not io.call_again and (self.block.input.pos, self.block.output.len) == before:
                break
        torch.cuda.synchronize()
        return io

    def output(self) -> torch.Tensor:
        return self.block.output.get()
