"""Block-level mirror of the reference's hot-path blocks, over device-resident buffers.

Reference interfaces mirrored (names, argument meaning and finish rules):
  * ``Fir`` / ``FirBuilder``      src/blocks/fir.rs:13-95, :126-233
  * ``Iir`` / ``IirBuilder``      src/blocks/iir.rs:8-176
  * ``SignalSource`` / ``SignalSourceBuilder`` / ``FixedPointPhase``   src/blocks/signal_source/{mod,fxpt_phase}.rs
  * ``Head``                      src/blocks/head.rs:22-84
  * ``Fft`` / ``FftDirection``    src/blocks/fft.rs:30-221
  * ``Apply``                     src/blocks/apply.rs:100-131 (closed catalogue of closures)
  * ``ApplyNM``                   src/blocks/applynm.rs:92-121 (closed catalogue of closures)
  * ``Mixer``                     Apply over the SSB example's oscillator closures (examples/ssb); helpers in
                                  futuresdr_b200.ssb
  * ``PfbArbResampler``           src/blocks/pfb/arb_resampler.rs:72-231
  * ``Combine`` / ``Split``       src/blocks/combine.rs:31-137, split.rs:31-127 (closed catalogues of closures)
  * ``Delay``                     src/blocks/delay.rs:31-169
  * ``MovingAverage``             examples/wlan/src/moving_average.rs:27-107, examples/m17/src/moving_average.rs:5-81
  * ``StreamDuplicator`` / ``StreamDeinterleaver``   src/blocks/stream_duplicator.rs, stream_deinterleaver.rs
  * ``AdsbDemod``                 examples/adsb/src/{preamble_detector,demodulator,decoder}.rs (PreambleDetector,
                                  Demodulator and Decoder::check_crc fused; helpers in futuresdr_b200.adsb)
  * ``ClockRecoveryMm``           examples/zigbee/src/clock_recovery_mm.rs:28-97
  * ``ZigbeeDecoder``             examples/zigbee/src/decoder.rs:78-183 with Mac::check_crc (mac.rs:62-85); helpers in
                                  futuresdr_b200.zigbee
  * ``KeyfobDecoder``             examples/keyfob/src/decoder.rs:64-127 with print (:36-52); helpers in
                                  futuresdr_b200.keyfob
  * ``LoraTransmitter``           examples/lora/src/transmitter.rs:12-168 (Encoder + Modulator); helpers in
                                  futuresdr_b200.lora
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
    return {np.dtype(np.complex64): torch.complex64, np.dtype(np.float64): torch.float64,
            np.dtype(np.uint8): torch.uint8, np.dtype(np.int16): torch.int16}.get(np.dtype(np_dtype), torch.float32)


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

    # Stream ports, as the graph driver (edges.Flowgraph) addresses them: a port is an attribute name, or
    # (attribute name, index) for one port of a list of ports.  Single-input / single-output blocks keep the defaults.
    def stream_inputs(self) -> list:
        return ["input"] if self.in_dtype is not None else []

    def stream_outputs(self) -> list:
        return ["output"] if self.out_dtype is not None else []

    def port_dtype(self, port) -> np.dtype:
        name = port[0] if isinstance(port, tuple) else port
        return np.dtype(self.in_dtype if name == "input" else self.out_dtype)

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


class Iir(Fir):
    """blocks::Iir (src/blocks/iir.rs:8-176): generic over a ``StatefulFilter`` core (an ``IirFilter``).  Its input
    minimum (iir.rs:133) and its work and finish rule (iir.rs:156-175) are Fir's."""

    @classmethod
    def new(cls, a_taps, b_taps, sample_dtype=np.float32, ctx: Optional[Context] = None) -> "Iir":
        return cls(IirFilter(a_taps, b_taps, sample_dtype, ctx))

    @classmethod
    def with_core(cls, core: IirFilter) -> "Iir":
        return cls(core)


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
    DcBlockF32 = _lib.OP_DC_BLOCK_F32      # param = alpha: s = (1 - alpha) * s + alpha * x; y = x - s
    SliceF32U8 = _lib.OP_SLICE_F32_U8      # f32 -> u8: x > 0 ? 1 : 0 (the keyfob receiver's slicer)
    DivC32 = _lib.OP_DIV_C32               # c32 -> c32: x / param per part (the SSB transmitter's file level)


_APPLY_TYPES = {
    ApplyOp.ScaleF32: (np.float32, np.float32), ApplyOp.ScaleC32: (np.complex64, np.complex64),
    ApplyOp.QuadDemod: (np.complex64, np.float32), ApplyOp.NormSqr: (np.complex64, np.float32),
    ApplyOp.QuadDemodC32: (np.complex64, np.complex64), ApplyOp.ExpF32: (np.float32, np.float32),
    ApplyOp.MagC32: (np.complex64, np.float32), ApplyOp.Log10F32: (np.float32, np.float32),
    ApplyOp.DcBlockF32: (np.float32, np.float32), ApplyOp.SliceF32U8: (np.float32, np.uint8),
    ApplyOp.DivC32: (np.complex64, np.complex64),
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
        _apply_work(self, self.apply, io)


def _apply_work(block: Block, closure, io: WorkIo):
    """Apply::work (apply.rs:109-128): ``closure(i, o)`` over min(len) items of the block's slices; the block finishes
    once its input is finished and every item on it was processed."""
    i, o = block.input.slice(), block.output.slice()
    i_len = i.numel()
    m = min(i_len, o.numel())                                                   # apply.rs:109
    if m > 0:
        closure(i, o)
        block.input.consume(m)
        block.output.produce(m)
    if block.input.finished() and m == i_len:                                   # apply.rs:126-128
        io.finished = True


class ApplyNMOp(enum.IntEnum):
    """The ApplyNM closures that exist as device ops (b2s_op)."""
    C32ToI16Iq = _lib.OP_C32_TO_I16_IQ     # c32 -> 2 x i16: (re * param * 32767.0) as i16, then im (ssb transmit)


_APPLYNM_TYPES = {ApplyNMOp.C32ToI16Iq: (np.complex64, np.int16, 1, 2)}     # (in, out, N, M)


class ApplyNM(Block, Handle):
    """blocks::ApplyNM<_, A, B, N, M> (src/blocks/applynm.rs:92-121) for the closures of ApplyNMOp: N input items become
    M output items.  Rust's ``as i16`` truncates toward zero, saturates and maps NaN to 0, and so does the device."""
    _destroy = lib.b2s_apply_destroy

    def __init__(self, op: ApplyNMOp, param: float = 1.0, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.op = ApplyNMOp(op)
        self.in_dtype, self.out_dtype, self.n, self.m = _APPLYNM_TYPES[self.op]
        self._h = C.c_void_p()
        check(lib.b2s_apply_create(self.ctx.handle, int(self.op), float(param), C.byref(self._h)), self.ctx.handle)
        self._ports()

    def apply(self, i: torch.Tensor, o: torch.Tensor) -> tuple[int, int]:
        """The closure over device slices (asynchronous) -> (consumed, produced)."""
        c, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_apply_exec(self._h, _ptr(i), i.numel(), _ptr(o), o.numel(), C.byref(c), C.byref(p)),
              self.ctx.handle)
        return c.value, p.value

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()
        i_len = i.numel()
        m = min(i_len // self.n, o.numel() // self.m)                           # applynm.rs:109
        if m > 0:
            self.apply(i[:self.n * m], o[:self.m * m])
            self.input.consume(self.n * m)
            self.output.produce(self.m * m)
        if self.input.finished() and i_len - self.n * m < self.n:               # applynm.rs:118-120
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


class MixOp(enum.IntEnum):
    """The SSB example's oscillator closures, ``osc *= shift; f(v, osc)`` (b2s_mix_op)."""
    RotateC32 = _lib.MIX_ROTATE_C32             # v * osc                                  (transmit.rs:102-107)
    RotateScaleC32 = _lib.MIX_ROTATE_SCALE_C32  # v * osc * param                          (receive.rs:58-66)
    WeaverF32 = _lib.MIX_WEAVER_F32             # param * (v.re*osc.re + v.im*osc.im), f32 (receive.rs:73-83)


class Mixer(Block, Handle):
    """blocks::Apply over one oscillator closure of MixOp, with shift = Complex32::from_polar(1.0, phase_incr): the
    Rotator's recurrence replayed bit for bit (csrc/rotator.cu), so the output is the reference closure's under any
    slicing.  Work and finish rules are Apply's (apply.rs:100-131)."""
    _destroy = lib.b2s_mixer_destroy
    in_dtype = np.complex64

    def __init__(self, op: MixOp, phase_incr: float, param: float = 1.0, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.op = MixOp(op)
        self.out_dtype = np.float32 if self.op == MixOp.WeaverF32 else np.complex64
        self._h = C.c_void_p()
        check(lib.b2s_mixer_create(self.ctx.handle, int(self.op), float(np.float32(phase_incr)), float(np.float32(param)),
                                   C.byref(self._h)), self.ctx.handle)
        self._ports()

    def mix(self, i: torch.Tensor, o: torch.Tensor) -> int:
        """The closure over min(len) items of device slices (asynchronous); returns that count."""
        c, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_mixer_exec(self._h, _ptr(i), i.numel(), _ptr(o), o.numel(), C.byref(c), C.byref(p)),
              self.ctx.handle)
        return c.value

    def reset(self):
        """osc back to 1 + 0i."""
        check(lib.b2s_mixer_reset(self._h), self.ctx.handle)

    def work(self, io: WorkIo):
        _apply_work(self, self.mix, io)


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
    only 8 B/sample in and ``n`` floats per ``history_size`` frames out touch HBM.  Counts are MovingAvg's.  Values
    are the three separate blocks' to rounding: the average is a blocked scan, so every emitted value of every bin is
    within 2*B + 4*u*V of the float64 recurrence V on the same |X|^2, B being the rounding-error bound of the
    sequential f32 recurrence (tests/test_gpu_spectrum_bins.py)."""
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


def _ptr(t: torch.Tensor) -> C.c_void_p:
    return C.c_void_p(t.data_ptr())


class CombineOp(enum.IntEnum):
    """The Combine closures of the reference graphs that exist as device ops (b2s_combine_op)."""
    AddF32 = _lib.COMBINE_ADD_F32                # a + b                 (tests/combine.rs)
    SubF32 = _lib.COMBINE_SUB_F32                # i1 - i2               (m17 rx)
    MulF32 = _lib.COMBINE_MUL_F32                # a * b                 (cw)
    ConjMulC32 = _lib.COMBINE_CONJ_MUL_C32       # a * b.conj()          (wlan rx)
    MagDivC32F32 = _lib.COMBINE_MAG_DIV_C32_F32  # a.norm() / b          (wlan rx)
    ToC32 = _lib.COMBINE_TO_C32                  # Complex32::new(i, q)  (ssb USB)
    ToC32NegQ = _lib.COMBINE_TO_C32_NEG_Q        # Complex32::new(i, q * -1.0) (ssb LSB)


_F32, _C32 = np.dtype(np.float32), np.dtype(np.complex64)
_COMBINE_TYPES = {                               # (in0, in1, output)
    CombineOp.AddF32: (_F32, _F32, _F32), CombineOp.SubF32: (_F32, _F32, _F32), CombineOp.MulF32: (_F32, _F32, _F32),
    CombineOp.ConjMulC32: (_C32, _C32, _C32), CombineOp.MagDivC32F32: (_C32, _F32, _F32),
    CombineOp.ToC32: (_F32, _F32, _C32), CombineOp.ToC32NegQ: (_F32, _F32, _C32),
}


class Combine(Block):
    """blocks::Combine (src/blocks/combine.rs:31-137): two input streams ``in0``, ``in1`` -> ``output`` through one
    closure of CombineOp.  Finishes when an input has finished and everything on it was processed (:127-133)."""
    in_dtype = None

    def __init__(self, op: CombineOp, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.op = CombineOp(op)
        a, b, self.out_dtype = _COMBINE_TYPES[self.op]
        dev = _ctx_device(self.ctx)
        self.in0, self.in1, self.output = Reader(a, dev), Reader(b, dev), Writer(self.out_dtype, dev)

    def stream_inputs(self):
        return ["in0", "in1"]

    def port_dtype(self, port):
        return {"in0": self.in0.dtype, "in1": self.in1.dtype, "output": np.dtype(self.out_dtype)}[port]

    def combine(self, i0: torch.Tensor, i1: torch.Tensor, o: torch.Tensor) -> int:
        """The closure over min(len) items of device slices (asynchronous); returns that count."""
        c, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_combine_exec(self.ctx.handle, int(self.op), _ptr(i0), i0.numel(), _ptr(i1), i1.numel(), _ptr(o),
                                   o.numel(), C.byref(c), C.byref(p)), self.ctx.handle)
        return p.value

    def work(self, io: WorkIo):
        i0, i1, o = self.in0.slice(), self.in1.slice(), self.output.slice()       # combine.rs:108-115
        i0_len, i1_len = i0.numel(), i1.numel()
        m = min(i0_len, i1_len, o.numel())
        if m > 0:
            self.combine(i0, i1, o)
            self.in0.consume(m)
            self.in1.consume(m)
            self.output.produce(m)
        if self.in0.finished() and m == i0_len:                                 # :127-133
            io.finished = True
        if self.in1.finished() and m == i1_len:
            io.finished = True


class SplitOp(enum.IntEnum):
    """The Split closures that exist as device ops (b2s_split_op)."""
    ReIm = _lib.SPLIT_RE_IM                      # |a: &Complex32| (a.re, a.im)   (tests/split.rs)
    DupF32 = _lib.SPLIT_DUP_F32                  # |v: &f32| (*v, *v)             (ssb)


class Split(Block):
    """blocks::Split (src/blocks/split.rs:31-127): ``input`` -> ``output0``, ``output1`` through one closure."""

    def __init__(self, op: SplitOp, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.op = SplitOp(op)
        self.in_dtype = _C32 if self.op == SplitOp.ReIm else _F32
        self.out_dtype = None
        dev = _ctx_device(self.ctx)
        self.input = Reader(self.in_dtype, dev)
        self.output0, self.output1 = Writer(_F32, dev), Writer(_F32, dev)

    def stream_outputs(self):
        return ["output0", "output1"]

    def port_dtype(self, port):
        return np.dtype(self.in_dtype) if port == "input" else _F32

    def split(self, i: torch.Tensor, o0: torch.Tensor, o1: torch.Tensor) -> int:
        c, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_split_exec(self.ctx.handle, int(self.op), _ptr(i), i.numel(), _ptr(o0), _ptr(o1),
                                 min(o0.numel(), o1.numel()), C.byref(c), C.byref(p)), self.ctx.handle)
        return p.value

    def work(self, io: WorkIo):
        i0, o0, o1 = self.input.slice(), self.output0.slice(), self.output1.slice()   # split.rs:101-107
        i0_len = i0.numel()
        m = min(i0_len, o0.numel(), o1.numel())
        if m > 0:
            self.split(i0, o0, o1)
            self.input.consume(m)
            self.output0.produce(m)
            self.output1.produce(m)
        if self.input.finished() and m == i0_len:                               # :121-123
            io.finished = True


class Delay(Block):
    """blocks::Delay (src/blocks/delay.rs:31-169): ``n > 0`` pads n zero items in front of the stream, ``n <= 0`` skips
    -n items.  The pad is a device memset and the copy a device-to-device copy; a skip only moves the read cursor.
    ``state`` is ("pad", n), ("skip", n) or ("copy", 0)."""

    def __init__(self, dtype, n: int, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.in_dtype = self.out_dtype = np.dtype(dtype)
        n = int(n)
        self.state = ("pad", n) if n > 0 else ("skip", -n)                      # delay.rs:55-60
        self._ports()

    def new_value(self, pad: bool, value: int):
        """The ``new_value`` message handler (delay.rs:68-105): shifts the delay by +value (pad) or -value (skip)."""
        val = int(value) if pad else -int(value)
        kind, n = self.state
        new_val = (n if kind == "pad" else -n if kind == "skip" else 0) + val
        self.state = ("pad", new_val) if new_val > 0 else ("copy", 0) if new_val == 0 else ("skip", -new_val)

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()                          # delay.rs:120-123
        i_len, o_len = i.numel(), o.numel()
        isz = self.in_dtype.itemsize
        kind, n = self.state
        if kind == "pad":
            m = min(o_len, n)
            if m:
                check(lib.b2s_memset(self.ctx.handle, _ptr(o), 0, m * isz), self.ctx.handle)
            self.output.produce(m)
            if m == n:
                self.state = ("copy", 0)
                io.call_again = True
                if self.input.finished():
                    io.finished = True
            else:
                self.state = ("pad", n - m)
        elif kind == "skip":
            m = min(i_len, n)
            self.input.consume(m)
            if n == m:
                self.state = ("copy", 0)
                io.call_again = True
            else:
                self.state = ("skip", n - m)
            if self.input.finished() and m == i_len:
                io.finished = True
        else:
            m = min(i_len, o_len)
            if m > 0:
                check(lib.b2s_memcpy_d2d(self.ctx.handle, _ptr(o), _ptr(i), m * isz), self.ctx.handle)
            self.input.consume(m)
            self.output.produce(m)
            if self.input.finished() and m == i_len:
                io.finished = True


class MovingAverage(Block, Handle):
    """The WLAN and M17 receivers' MovingAverage (examples/wlan/src/moving_average.rs:27-107, f32 and Complex32;
    examples/m17/src/moving_average.rs:5-81, f32 with ``divisor=4800.0``): a box-car sum over ``len`` items, emitted
    after ``len - 1`` leading zeros, so output k is the window that ENDS at input k.  Not ``MovingAvg`` (an
    exponential average per bin over fixed-width chunks).

    Each reference work() call restarts a strict-order f32 running sum and produces at most 4000 outputs, so the
    rounding depends on where the calls fall; the device reproduces it bit for bit given the same calls.  One
    ``work()`` runs the calls the reference would make back to back on the current slices until one makes no progress
    (``max_calls=0``), or at most ``max_calls`` of them (``max_calls=1`` is exactly one reference work() call).
    ``io.call_again`` and the finish rule (:103-105) are those of the last of these calls."""
    _destroy = lib.b2s_boxavg_destroy

    def __init__(self, dtype, len: int, divisor: Optional[float] = None, max_calls: int = 0,
                 ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.in_dtype = self.out_dtype = np.dtype(dtype)
        if self.in_dtype not in (_F32, _C32):
            raise TypeError(f"MovingAverage: f32 or Complex32 items, not {self.in_dtype}")
        self.len = int(len)
        self.divisor = None if divisor is None else float(np.float32(divisor))
        self.max_calls = int(max_calls)
        self._h = C.c_void_p()
        check(lib.b2s_boxavg_create(self.ctx.handle, int(self.in_dtype == _C32), self.len, int(divisor is not None),
                                    float(self.divisor or 0.0), C.byref(self._h)), self.ctx.handle)
        self._ports()

    def average(self, i: torch.Tensor, o: torch.Tensor, max_calls: Optional[int] = None):
        """One exec over device slices (asynchronous) -> (consumed, produced, calls, call_again, done)."""
        c, p, n = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        ca, dn = C.c_int32(0), C.c_int32(0)
        check(lib.b2s_boxavg_exec(self._h, _ptr(i), i.numel(), _ptr(o), o.numel(),
                                  self.max_calls if max_calls is None else int(max_calls), C.byref(c), C.byref(p),
                                  C.byref(n), C.byref(ca), C.byref(dn)), self.ctx.handle)
        return c.value, p.value, n.value, bool(ca.value), bool(dn.value)

    def reset(self):
        check(lib.b2s_boxavg_reset(self._h), self.ctx.handle)

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()
        c, p, _, call_again, done = self.average(i, o)
        self.input.consume(c)
        self.output.produce(p)
        if call_again:                                                          # :82-84
            io.call_again = True
        if self.input.finished() and done:                                      # :103-105
            io.finished = True


class _Records:
    """One record list of a block, handed out by ``drain(handle, host, cap, &n)`` (a b2s_*_drain_* function).  ``read``
    drains it until a short read and returns every record so far, a cumulative numpy structured array of ``dtype`` in
    stream order; draining synchronises.  ``clear`` forgets the records, as the block's reset does."""
    chunk = 1 << 16        # records per drain call; the loop ends on a short read, so the result does not depend on it

    def __init__(self, drain, dtype):
        self.drain, self.dtype = drain, np.dtype(dtype)
        self.clear()

    def clear(self):
        self._parts = []

    def read(self, h, ctx_handle) -> np.ndarray:
        while True:
            buf = np.zeros(self.chunk, self.dtype)
            n = C.c_size_t(0)
            check(self.drain(h, buf.ctypes.data_as(C.c_void_p), buf.size, C.byref(n)), ctx_handle)
            self._parts.append(buf[:n.value])
            if n.value < buf.size:
                out = np.concatenate(self._parts)
                self._parts = [out]
                return out


def _payload_batch(payloads):
    """Payloads (a str as UTF-8, or bytes-like) as the push and encode calls take them: (their bytes, those joined,
    their lengths as a c_size_t array).  The array has at least one element, so an empty batch passes a valid
    pointer."""
    data = [p.encode() if isinstance(p, str) else bytes(p) for p in payloads]
    return data, b"".join(data), (C.c_size_t * max(len(data), 1))(*[len(d) for d in data])


ADSB_PACKET = np.dtype([("preamble_index", np.uint64), ("preamble_correlation", np.float32),
                        ("crc_passed", np.int32), ("bytes", np.uint8, 14)], align=True)   # b2s_adsb_packet
ADSB_DETECTION = np.dtype([("index", np.uint64), ("value", np.float32)], align=True)      # b2s_adsb_detection


class AdsbDemod(Block, Handle):
    """The ADS-B receiver's PreambleDetector -> Demodulator -> Decoder::check_crc (examples/adsb/src/
    preamble_detector.rs:65-146, demodulator.rs:49-113, decoder.rs:57-73) as one device block.  Stream inputs
    ``in_samples`` (|x|^2), ``in_nf`` (noise floor) and ``in_preamble_cor`` (preamble correlation), all f32; no stream
    output.  The detector's tags stay inside the block: ``detections()`` returns them (index, correlation ratio) and
    ``packets()`` the demodulated 112-bit frames -- only those that pass the CRC unless ``forward_failed_crc``.  Both
    are cumulative numpy structured arrays, and reading them synchronises.

    Finish rule: the reference finishes as soon as any input is finished, which depends on its scheduler.  Here the
    block finishes once some input is finished and the scan has reached the limit computed from that input's final
    length (the smallest final length, if several are finished); that is the reference's result whenever the other
    inputs hold at least as much data, as they do in the receiver's graph."""
    _destroy = lib.b2s_adsb_destroy
    in_dtype = None
    out_dtype = None

    def __init__(self, threshold: float = 10.0, forward_failed_crc: bool = False, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.threshold = float(np.float32(threshold))
        self.forward_failed_crc = bool(forward_failed_crc)
        self._h = C.c_void_p()
        check(lib.b2s_adsb_create(self.ctx.handle, self.threshold, int(self.forward_failed_crc), C.byref(self._h)),
              self.ctx.handle)
        dev = _ctx_device(self.ctx)
        self.in_samples, self.in_nf, self.in_preamble_cor = (Reader(_F32, dev) for _ in range(3))
        self._packets = _Records(lib.b2s_adsb_drain_packets, ADSB_PACKET)
        self._detections = _Records(lib.b2s_adsb_drain_detections, ADSB_DETECTION)

    def stream_inputs(self):
        return ["in_samples", "in_nf", "in_preamble_cor"]

    def port_dtype(self, port):
        return _F32

    def exec(self, s: torch.Tensor, nf: torch.Tensor, corr: torch.Tensor, finished: bool = False) -> tuple[int, bool]:
        """One exec over device slices (asynchronous) -> (consumed from each input, done)."""
        c, dn = C.c_size_t(0), C.c_int32(0)
        check(lib.b2s_adsb_exec(self._h, _ptr(s), s.numel(), _ptr(nf), nf.numel(), _ptr(corr), corr.numel(),
                                int(finished), C.byref(c), C.byref(dn)), self.ctx.handle)
        return c.value, bool(dn.value)

    def reset(self):
        check(lib.b2s_adsb_reset(self._h), self.ctx.handle)
        self._packets.clear()
        self._detections.clear()

    def packets(self) -> np.ndarray:
        """Every packet so far (ADSB_PACKET records, in index order)."""
        return self._packets.read(self._h, self.ctx.handle)

    def detections(self) -> np.ndarray:
        """Every detector tag so far (ADSB_DETECTION records, in index order; equal indices can repeat)."""
        return self._detections.read(self._h, self.ctx.handle)

    def work(self, io: WorkIo):
        ports = (self.in_samples, self.in_nf, self.in_preamble_cor)
        sl = [p.slice() for p in ports]
        L = min(t.numel() for t in sl)
        fin = [t.numel() for p, t in zip(ports, sl) if p.finished()]
        final = bool(fin) and L == min(fin)
        c, done = self.exec(*(t[:L] for t in sl), finished=final)
        for p in ports:
            p.consume(c)
        if done:
            io.finished = True


class ClockRecoveryMm(Block, Handle):
    """examples/zigbee/src/clock_recovery_mm.rs:28-97 (Mueller & Muller), f32 -> f32, bit for bit.  Consumption depends
    on the data, so every exec synchronises once to learn its counts.  A NaN latches mu (nothing is consumed from then
    on); a step that would move past the slice raises B200SdrError (ESTATE) with the block left before that step.
    Finish rule: the input is finished and what is left of it is within the look-ahead, or the call consumed nothing
    while it produced (a latched mu).  This departs from clock_recovery_mm.rs:92-94, which finishes as soon as the
    input is finished: here an input is reported finished as soon as its writer is, while it can still hold items, and
    finishing then would drop them (and the outputs they give) whenever the output buffer had cut the call short."""
    _destroy = lib.b2s_mmclock_destroy
    in_dtype = out_dtype = np.float32

    def __init__(self, omega: float, gain_omega: float, mu: float, gain_mu: float, omega_relative_limit: float,
                 ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self._h = C.c_void_p()
        check(lib.b2s_mmclock_create(self.ctx.handle, float(omega), float(gain_omega), float(mu), float(gain_mu),
                                     float(omega_relative_limit), C.byref(self._h)), self.ctx.handle)
        self.look_ahead = int(lib.b2s_mmclock_look_ahead(self._h))
        self._ports()
        self.input.set_min_items(self.look_ahead + 1)                           # :37

    def exec(self, i: torch.Tensor, o: torch.Tensor) -> tuple[int, int]:
        """One call of the reference's work loop over device slices -> (consumed, produced); synchronises."""
        c, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_mmclock_exec(self._h, _ptr(i), i.numel(), _ptr(o), o.numel(), C.byref(c), C.byref(p)),
              self.ctx.handle)
        return c.value, p.value

    def reset(self):
        check(lib.b2s_mmclock_reset(self._h), self.ctx.handle)

    def work(self, io: WorkIo):
        i, o = self.input.slice(), self.output.slice()
        c, p = self.exec(i, o)
        self.input.consume(c)
        self.output.produce(p)
        if self.input.finished() and (i.numel() - c <= self.look_ahead or (c == 0 and p > 0)):
            io.finished = True


class _Decoder(Block, Handle):
    """The body of the decoders that turn one stream input into records, with no stream output: ``exec``, ``reset``, the
    record reader and ``work``.  A subclass names its ABI functions and record type, calls ``__init__`` and then
    creates ``self._h``."""
    out_dtype = None
    _exec = _reset = _drain = _record = None

    def __init__(self, ctx: Optional[Context]):
        self.ctx = ctx or default_context()
        self.input = Reader(self.in_dtype, _ctx_device(self.ctx))
        self._records = _Records(self._drain, self._record)

    def exec(self, i: torch.Tensor) -> int:
        c = C.c_size_t(0)
        check(self._exec(self._h, _ptr(i), i.numel(), C.byref(c)), self.ctx.handle)
        return c.value

    def reset(self):
        check(self._reset(self._h), self.ctx.handle)
        self._records.clear()

    def work(self, io: WorkIo):
        i = self.input.slice()
        self.input.consume(self.exec(i))
        if self.input.finished():                       # zigbee decoder.rs:174-176, keyfob decoder.rs:120-122
            io.finished = True


ZIGBEE_FRAME = np.dtype([("index", np.uint64), ("len", np.uint32), ("crc_ok", np.int32), ("bytes", np.uint8, 128)],
                        align=True)                                                          # b2s_zigbee_frame


class ZigbeeDecoder(_Decoder):
    """examples/zigbee/src/decoder.rs:78-183 with Mac::check_crc (mac.rs:62-85) as a device block: one f32 stream
    input, no stream output.  The frames the reference posts come out of ``frames()``, a cumulative numpy structured
    array (ZIGBEE_FRAME: the stream index of the chip that completed the frame, its length, whether its FCS checks,
    its bytes); reading it synchronises.  Every exec consumes its whole slice and never synchronises."""
    _destroy = lib.b2s_zigbee_destroy
    _exec, _reset = lib.b2s_zigbee_exec, lib.b2s_zigbee_reset
    _drain, _record = lib.b2s_zigbee_drain_frames, ZIGBEE_FRAME
    in_dtype = np.float32

    def __init__(self, threshold: int = 6, ctx: Optional[Context] = None):
        super().__init__(ctx)
        self.threshold = int(threshold)
        self._h = C.c_void_p()
        check(lib.b2s_zigbee_create(self.ctx.handle, C.c_uint32(self.threshold), C.byref(self._h)), self.ctx.handle)

    def frames(self) -> np.ndarray:
        """Every frame so far (ZIGBEE_FRAME records, in stream order)."""
        return self._records.read(self._h, self.ctx.handle)


KEYFOB_CODE = np.dtype([("index", np.uint64), ("n_bits", np.uint32), ("label", np.int32), ("bits", np.uint8, 32)],
                       align=True)                                                           # b2s_keyfob_code


class KeyfobDecoder(_Decoder):
    """examples/keyfob/src/decoder.rs:64-127 with print (:36-52) as a device block: one u8 stream input, no stream
    output.  The strings the reference logs come out of ``codes()``, a cumulative numpy structured array (KEYFOB_CODE:
    the stream position of the flushing edge, the length after the prefix strip, the label of the last 8 bits, the
    first 256 bits MSB first); reading it synchronises.  Every exec consumes its whole slice and never synchronises."""
    _destroy = lib.b2s_keyfob_destroy
    _exec, _reset = lib.b2s_keyfob_exec, lib.b2s_keyfob_reset
    _drain, _record = lib.b2s_keyfob_drain_codes, KEYFOB_CODE
    in_dtype = np.uint8

    def __init__(self, ctx: Optional[Context] = None):
        super().__init__(ctx)
        self._h = C.c_void_p()
        check(lib.b2s_keyfob_create(self.ctx.handle, C.byref(self._h)), self.ctx.handle)

    def codes(self) -> np.ndarray:
        """Every code so far (KEYFOB_CODE records, in stream order)."""
        return self._records.read(self._h, self.ctx.handle)


class _Transmitter(Block, Handle):
    """The body of the device transmitters, sources with one Complex32 output: ``finish``, ``pending``, ``exec``,
    ``reset``, ``bursts`` and ``work``.  A subclass names its ABI functions and burst record type, calls ``__init__``
    and then creates ``self._h``."""
    in_dtype = None
    out_dtype = np.complex64
    _finish = _pending = _exec = _reset = _drain = _record = None

    def __init__(self, ctx: Optional[Context]):
        self.ctx = ctx or default_context()
        self.input = None
        self.output = Writer(self.out_dtype, _ctx_device(self.ctx))
        self._records = _Records(self._drain, self._record)

    def finish(self):
        check(self._finish(self._h), self.ctx.handle)

    def pending(self) -> int:
        """Queued samples not yet produced."""
        v = C.c_uint64(0)
        check(self._pending(self._h, C.byref(v)), self.ctx.handle)
        return v.value

    def exec(self, o: torch.Tensor) -> tuple[int, bool]:
        """Write the next samples into the device slice ``o`` (asynchronous) -> (produced, finished)."""
        p, f = C.c_size_t(0), C.c_int32(0)
        check(self._exec(self._h, _ptr(o), o.numel(), C.byref(p), C.byref(f)), self.ctx.handle)
        return p.value, bool(f.value)

    def reset(self):
        check(self._reset(self._h), self.ctx.handle)
        self._records.clear()

    def bursts(self) -> np.ndarray:
        """Every burst_start tag so far (the class's burst records, in stream order)."""
        return self._records.read(self._h, self.ctx.handle)

    def work(self, io: WorkIo):
        o = self.output.slice()
        p, finished = self.exec(o)
        self.output.produce(p)
        if finished:
            io.finished = True


LORA_BURST = np.dtype([("index", np.uint64), ("len", np.uint64)], align=True)                   # b2s_lora_burst


class LoraTransmitter(_Transmitter):
    """examples/lora/src/transmitter.rs:12-168 (Encoder + Modulator) as a device source: no input port, one Complex32
    output.  ``push`` is the ``msg`` handler (bytes or str payloads, encoded on the device at once), ``set_sync_word``
    the ``synch_word`` handler and ``finish`` its Pmt::Finished.  ``work`` fills the output slice with the next samples
    of the concatenated frames, across frame boundaries; the stream is bit-identical for every slicing.  ``bursts()``
    returns the burst_start tags (stream index, length) of the frames started so far, a cumulative LORA_BURST array.
    Finish rule: finished once ``finish`` has been called and every queued sample has been produced."""
    _destroy = lib.b2s_lora_tx_destroy
    _finish, _pending, _exec = lib.b2s_lora_tx_finish, lib.b2s_lora_tx_pending, lib.b2s_lora_tx_exec
    _reset, _drain, _record = lib.b2s_lora_tx_reset, lib.b2s_lora_tx_drain_bursts, LORA_BURST

    def __init__(self, sf: int, code_rate: int, has_crc: bool, ldro_enabled: bool, implicit_header: bool,
                 oversampling: int, sync_symbols, preamble_len: int, pad: int, ctx: Optional[Context] = None):
        super().__init__(ctx)
        self.sf, self.code_rate, self.has_crc = int(sf), int(code_rate), bool(has_crc)
        self.ldro_enabled, self.implicit_header = bool(ldro_enabled), bool(implicit_header)
        self.oversampling, self.preamble_len, self.pad = int(oversampling), int(preamble_len), int(pad)
        sw = (C.c_uint32 * 2)(*[int(v) for v in sync_symbols])
        self._h = C.c_void_p()
        check(lib.b2s_lora_tx_create(self.ctx.handle, self.sf, self.code_rate, int(self.has_crc),
                                     int(self.ldro_enabled), int(self.implicit_header), self.oversampling, sw,
                                     self.preamble_len, self.pad, C.byref(self._h)), self.ctx.handle)

    def push(self, *payloads):
        """Queue frames (transmitter.rs:77-78: Pmt::Blob or Pmt::String); all or nothing."""
        data, buf, lens = _payload_batch(payloads)
        check(lib.b2s_lora_tx_push(self._h, C.c_char_p(buf) if buf else None, lens, len(data)), self.ctx.handle)

    def set_sync_word(self, word):
        """transmitter.rs:88-110: a compact u8 (int, or one byte) expands as SynchWord::from(u8); two bytes are the
        expanded symbols.  A word that does not fit the spreading factor raises and leaves the old one."""
        from .lora import SynchWord
        s0, s1 = SynchWord.from_pmt(word).expand()
        check(lib.b2s_lora_tx_set_sync_word(self._h, s0, s1), self.ctx.handle)


WLAN_BURST = np.dtype([("index", np.uint64), ("len", np.uint64)], align=True)                   # b2s_wlan_burst


class WlanTransmitter(_Transmitter):
    """The WLAN transmit chain of examples/wlan/src/bin/tx.rs:44-66 (Mac -> Encoder -> Mapper -> Fft(64, Inverse,
    shift, sqrt(1/52)) -> Prefix) as a device source: no input port, one Complex32 output.  ``push`` is the Mac's
    ``tx`` handler: payloads (bytes or str) at the default MCS, or per-frame MCS numbers (-1: the default), framed and
    encoded on the device at once.  ``work`` fills the output slice with the next samples of the concatenated bursts;
    the stream is the same for every slicing.  ``bursts()`` returns the burst_start tags (stream index, length) of the
    frames started so far, a cumulative WLAN_BURST array.  Finished once ``finish`` has been called and every queued
    sample has been produced."""
    _destroy = lib.b2s_wlan_tx_destroy
    _finish, _pending, _exec = lib.b2s_wlan_tx_finish, lib.b2s_wlan_tx_pending, lib.b2s_wlan_tx_exec
    _reset, _drain, _record = lib.b2s_wlan_tx_reset, lib.b2s_wlan_tx_drain_bursts, WLAN_BURST

    def __init__(self, src_mac, dst_mac, bss_mac, default_mcs: int, pad_front: int, pad_tail: int,
                 ctx: Optional[Context] = None):
        super().__init__(ctx)
        self.addrs = tuple(bytes(a) for a in (src_mac, dst_mac, bss_mac))
        if any(len(a) != 6 for a in self.addrs):
            raise ValueError("WlanTransmitter: MAC addresses are 6 bytes")
        self.default_mcs, self.pad_front, self.pad_tail = int(default_mcs), int(pad_front), int(pad_tail)
        self._h = C.c_void_p()
        check(lib.b2s_wlan_tx_create(self.ctx.handle, *[C.c_char_p(a) for a in self.addrs], self.default_mcs,
                                     self.pad_front, self.pad_tail, C.byref(self._h)), self.ctx.handle)

    def push(self, *payloads, mcs=None):
        """Queue frames, all or nothing.  ``mcs``: None (every frame at the default MCS, Pmt::Blob) or one MCS
        number per payload, -1 meaning the default (the (data, mcs) pair)."""
        data, buf, lens = _payload_batch(payloads)
        n = len(data)
        m = None
        if mcs is not None:
            if len(mcs) != n:
                raise ValueError(f"WlanTransmitter.push: {len(mcs)} MCS for {n} payloads")
            m = (C.c_int32 * max(n, 1))(*[int(v) for v in mcs])
        check(lib.b2s_wlan_tx_push(self._h, C.c_char_p(buf) if buf else None, lens, m, n), self.ctx.handle)

    def reset(self):
        """Back to the created state: scrambler seed 1, sequence number 0, a zero bit buffer, nothing queued."""
        super().reset()


ZIGBEE_BURST = np.dtype([("index", np.uint64), ("len", np.uint64)], align=True)               # b2s_zigbee_burst


class ZigbeeTransmitter(_Transmitter):
    """The ZigBee transmit chain of examples/zigbee/src/bin/tx.rs:37-56 (Mac -> modulator -> IqDelay) as a device
    source: no input port, one Complex32 output.  ``push`` is the Mac's ``tx`` handler: each bytes-like payload is
    framed on the host and queued; one over 116 bytes is dropped on its own, as the Mac drops it, and ``push`` returns
    how many were dropped.  ``work`` fills the output slice with the next samples of the concatenated frames, each
    with ``pad`` zeros before and after it; the stream is bit-identical to the reference's for every slicing.
    ``bursts()`` returns the burst_start tags (stream index, length) of the frames started so far, a cumulative
    ZIGBEE_BURST array.  Finished once ``finish`` has been called and every queued sample has been produced."""
    _destroy = lib.b2s_zigbee_tx_destroy
    _finish, _pending, _exec = lib.b2s_zigbee_tx_finish, lib.b2s_zigbee_tx_pending, lib.b2s_zigbee_tx_exec
    _reset, _drain, _record = lib.b2s_zigbee_tx_reset, lib.b2s_zigbee_tx_drain_bursts, ZIGBEE_BURST

    def __init__(self, pad: int = _lib.ZIGBEE_PADDING, ctx: Optional[Context] = None):
        super().__init__(ctx)
        self.pad = int(pad)
        if self.pad < 0:
            raise ValueError("ZigbeeTransmitter: pad must not be negative")
        self._h = C.c_void_p()
        check(lib.b2s_zigbee_tx_create(self.ctx.handle, self.pad, C.byref(self._h)), self.ctx.handle)

    def push(self, *payloads) -> int:
        """Queue frames (Pmt::Blob payloads: bytes-like objects; a str raises TypeError) -> the number dropped for
        being over 116 bytes."""
        if any(isinstance(p, str) for p in payloads):
            raise TypeError("ZigbeeTransmitter.push: payloads are bytes-like, not str")
        data, buf, lens = _payload_batch([bytes(memoryview(p)) for p in payloads])
        dropped = C.c_size_t(0)
        check(lib.b2s_zigbee_tx_push(self._h, C.c_char_p(buf) if buf else None, lens, len(data), C.byref(dropped)),
              self.ctx.handle)
        return dropped.value

    def reset(self):
        """Back to the created state: sequence number 0, nothing queued."""
        super().reset()


class _FanOut(Block):
    """One input, ``n`` outputs in the list attribute ``self._list``, moved by one b2s_fanout_exec launch."""
    _list = ""
    _deinterleave = 0

    def __init__(self, dtype, n: int, ctx: Optional[Context] = None):
        self.ctx = ctx or default_context()
        self.in_dtype = self.out_dtype = np.dtype(dtype)
        if self.in_dtype.itemsize not in (4, 8):
            raise ValueError(f"{type(self).__name__}: items of 4 or 8 bytes, not {self.in_dtype}")
        self.n = int(n)
        if self.n < 1:
            raise ValueError(f"{type(self).__name__}: at least one output")
        if self.n > _lib.FANOUT_MAX_OUTPUTS:
            raise _lib.B200SdrError(_lib.EUNSUPPORTED, f"{type(self).__name__}: {self.n} outputs "
                                    f"(at most {_lib.FANOUT_MAX_OUTPUTS} in one launch)")
        dev = _ctx_device(self.ctx)
        self.input = Reader(self.in_dtype, dev)
        setattr(self, self._list, [Writer(self.in_dtype, dev) for _ in range(self.n)])

    def stream_outputs(self):
        return [(self._list, k) for k in range(self.n)]

    def port_dtype(self, port):
        return self.in_dtype

    def fanout(self, i: torch.Tensor, outs) -> tuple[int, int]:
        """(consumed, produced per output) of one launch over device slices."""
        ptrs = (C.c_void_p * len(outs))(*[o.data_ptr() for o in outs])
        c, p = C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_fanout_exec(self.ctx.handle, self._deinterleave, self.in_dtype.itemsize, _ptr(i), i.numel(), ptrs,
                                  len(outs), min(o.numel() for o in outs), C.byref(c), C.byref(p)), self.ctx.handle)
        return c.value, p.value


class StreamDuplicator(_FanOut):
    """blocks::StreamDuplicator<T, N> (src/blocks/stream_duplicator.rs:20-94): ``input`` copied to ``outputs[k]``."""
    _list = "outputs"

    def work(self, io: WorkIo):
        outs = [w.slice() for w in self.outputs]                                # stream_duplicator.rs:72-80
        i = self.input.slice()
        nitem_to_consume = i.numel()
        m = min(min(o.numel() for o in outs), nitem_to_consume)
        if m > 0:
            self.fanout(i, outs)
            for w in self.outputs:
                w.produce(m)
            self.input.consume(m)
        if nitem_to_consume - m == 0 and self.input.finished():                 # :89-91
            io.finished = True


class StreamDeinterleaver(_FanOut):
    """blocks::StreamDeinterleaver<T> (src/blocks/stream_deinterleaver.rs:25-98): item j N + k of ``input`` goes to
    ``output[k]``; only whole groups of N are moved, and the block finishes once fewer than N items are left."""
    _list = "output"
    _deinterleave = 1

    def work(self, io: WorkIo):
        outs = [w.slice() for w in self.output]                                 # stream_deinterleaver.rs:67-75
        i = self.input.slice()
        n_items_to_consume = i.numel()
        m = min(min(o.numel() for o in outs), n_items_to_consume // self.n)
        if m > 0:
            self.fanout(i, outs)
            for w in self.output:
                w.produce(m)
            self.input.consume(m * self.n)
        if n_items_to_consume - m * self.n < self.n and self.input.finished():   # :91-95
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
