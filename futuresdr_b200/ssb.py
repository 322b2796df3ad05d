"""The SSB transceiver (examples/ssb/{transmit,receive}.rs): its constants, the three oscillator phase increments, the
transmitter's filters, and both graphs from the block after the audio source to the block before the audio sink.

The audio devices and file formats around the graphs (AudioSink, the audio FileSource decoder, WavSink, and the
receiver's repeating FileSource) are not part of this module: the graphs start at any f32 (transmitter) or Complex32
(receiver) block, and end at blocks a VectorSink or FileSink can read."""
from __future__ import annotations

import numpy as np

from . import firdes, windows
from .blocks import (Apply, ApplyNM, ApplyNMOp, ApplyOp, Combine, CombineOp, Delay, FirBuilder, Mixer, MixOp, Split,
                     SplitOp)

FILE_RATE = 256_000                      # transmit.rs:59 (--sample-rate), receive.rs:15 (--file-rate)
# transmitter
TX_FREQUENCY = 53e3                      # transmit.rs:56 (--frequency)
AUDIO_BANDWIDTH = 3000.0                 # transmit.rs:62 (--audio-bandwidth)
LOWPASS_TRANSITION_HZ = 350.0            # transmit.rs:82
LOWPASS_RIPPLE = 0.05                    # transmit.rs:82
HILBERT_LEN = 167                        # transmit.rs:87, windows::hamming(167, false)
I16_LEVEL = 0.9                          # transmit.rs:110-111, `* 0.9 * i16::MAX as f32`
FILE_LEVEL_GAIN = 2.0                    # transmit.rs:125, `v * 2.0 / 0.0001`
# receiver
CENTER_FREQ = 51_500                     # receive.rs:28 (--center-freq)
FILE_LEVEL_ADJUSTMENT = 0.0001           # receive.rs:57, and the divisor of transmit.rs:125
VOLUME_ADJUSTMENT = 0.5                  # receive.rs:71
MID_AUDIO_SPECTRUM_FREQ = 1500           # receive.rs:72

_F32 = np.float32
_PI, _TAU = np.float32(np.pi), np.float32(2 * np.pi)        # std::f32::consts::{PI, TAU}


def xlating_phase(center_freq: int = CENTER_FREQ, file_rate: int = FILE_RATE) -> np.float32:
    """receive.rs:59-62: -2.0 * PI * (center_freq as f32) / (file_rate as f32), in f32 left to right."""
    return _F32(_F32(_F32(_F32(-2.0) * _PI) * _F32(center_freq)) / _F32(file_rate))


def weaver_phase(audio_rate: int) -> np.float32:
    """receive.rs:74-77: 2.0 * PI * (1500 as f32) / (audio_rate as f32), in f32 left to right."""
    return _F32(_F32(_F32(_F32(2.0) * _PI) * _F32(MID_AUDIO_SPECTRUM_FREQ)) / _F32(audio_rate))


def mixer_phase(frequency: float = TX_FREQUENCY, file_rate: int = FILE_RATE) -> np.float32:
    """transmit.rs:101: TAU * frequency / (file_rate as f32), in f32 left to right."""
    return _F32(_F32(_TAU * _F32(frequency)) / _F32(file_rate))


def lowpass_taps(audio_rate: float, audio_bandwidth: float = AUDIO_BANDWIDTH) -> np.ndarray:
    """transmit.rs:82: firdes::kaiser::lowpass(audio_bandwidth / audio_rate, 350.0 / audio_rate, 0.05), in f64."""
    return firdes.kaiser.lowpass(audio_bandwidth / float(audio_rate), LOWPASS_TRANSITION_HZ / float(audio_rate),
                                 LOWPASS_RIPPLE)


def hilbert_taps() -> np.ndarray:
    """transmit.rs:87-88: firdes::hilbert(&windows::hamming(167, false))."""
    return firdes.hilbert(windows.hamming(HILBERT_LEN, False))


def transmitter(fg, src, mode: str = "lsb", audio_rate: int = 48_000, frequency: float = TX_FREQUENCY,
                file_rate: int = FILE_RATE, audio_bandwidth: float = AUDIO_BANDWIDTH, ctx=None) -> dict:
    """transmit.rs:79-134 from ``src`` (an f32 audio block already in ``fg``) at ``audio_rate``: the Kaiser low-pass,
    Split(DupF32), Delay(-83) and the 167-tap Hilbert FIR, Combine(ToC32NegQ) for LSB or Combine(ToC32) for USB, the
    gcd-reduced resampler to ``file_rate``, Mixer(RotateC32) to ``frequency``, and two readers of the mixer:
    ApplyNM(C32ToI16Iq, 0.9) (the WAV samples) and Apply(ScaleC32, 2.0) -> Apply(DivC32, 0.0001) (the .dat level).
    Returns a dict of the blocks ("lowpass", "split", "delay", "hilbert", "to_complex", "resampler", "mixer",
    "to_i16_iq", "scale", "file_level"); "to_i16_iq" (i16) and "file_level" (Complex32) are the outputs."""
    mode = mode.lower()
    if mode not in ("lsb", "usb"):
        raise ValueError(f"ssb.transmitter: mode {mode!r} is not 'lsb' or 'usb'")
    lowpass = FirBuilder.fir(lowpass_taps(audio_rate, audio_bandwidth), np.float32, ctx)
    split = Split(SplitOp.DupF32, ctx)
    hilbert = FirBuilder.fir(hilbert_taps(), np.float32, ctx)
    delay = Delay(np.float32, -(HILBERT_LEN // 2), ctx)                          # window.len() as isize / -2 == -83
    to_complex = Combine(CombineOp.ToC32NegQ if mode == "lsb" else CombineOp.ToC32, ctx)
    resampler = FirBuilder.resampling(int(file_rate), int(audio_rate), np.complex64, ctx)
    mixer = Mixer(MixOp.RotateC32, mixer_phase(frequency, file_rate), ctx=ctx)
    to_i16_iq = ApplyNM(ApplyNMOp.C32ToI16Iq, I16_LEVEL, ctx)
    scale = Apply(ApplyOp.ScaleC32, FILE_LEVEL_GAIN, ctx)
    file_level = Apply(ApplyOp.DivC32, FILE_LEVEL_ADJUSTMENT, ctx)
    fg.connect(src, lowpass)
    fg.connect(lowpass, split)
    fg.connect(split, "output0", delay)
    fg.connect(delay, to_complex, "in0")
    fg.connect(split, "output1", hilbert)
    fg.connect(hilbert, to_complex, "in1")
    fg.connect(to_complex, resampler)
    fg.connect(resampler, mixer)
    fg.connect(mixer, to_i16_iq)
    fg.connect(mixer, scale)
    fg.connect(scale, file_level)
    return {"lowpass": lowpass, "split": split, "delay": delay, "hilbert": hilbert, "to_complex": to_complex,
            "resampler": resampler, "mixer": mixer, "to_i16_iq": to_i16_iq, "scale": scale, "file_level": file_level}


def receiver(fg, src, audio_rate: int = 48_000, center_freq: int = CENTER_FREQ, file_rate: int = FILE_RATE,
             ctx=None) -> dict:
    """receive.rs:54-87 from ``src`` (a Complex32 block already in ``fg``) at ``file_rate``: Mixer(RotateScaleC32,
    0.0001) to ``center_freq`` (the frequency-xlating closure), FirBuilder.resampling(audio_rate, file_rate) and
    Mixer(WeaverF32, 0.5) at 1500 Hz.  Returns a dict of the blocks ("xlating", "resampler", "weaver"); "weaver" is the
    f32 audio output.  The reference picks the audio rate with the largest gcd with the file rate among the sound
    card's rates; here it is an argument."""
    xlating = Mixer(MixOp.RotateScaleC32, xlating_phase(center_freq, file_rate), FILE_LEVEL_ADJUSTMENT, ctx)
    resampler = FirBuilder.resampling(int(audio_rate), int(file_rate), np.complex64, ctx)
    weaver = Mixer(MixOp.WeaverF32, weaver_phase(audio_rate), VOLUME_ADJUSTMENT, ctx)
    fg.connect(src, xlating)
    fg.connect(xlating, resampler)
    fg.connect(resampler, weaver)
    return {"xlating": xlating, "resampler": resampler, "weaver": weaver}

