"""A CPU model of the SSB transmit and receive graphs (TEST INFRASTRUCTURE ONLY): float64 filters, and the oracle's f32
oscillators (tests/ssb_oracle.c).  The reference's oscillator is an un-normalised f32 product recurrence whose magnitude
drifts, so an ideal complex exponential is not the model; the filters are exact convolutions, so the model is the
graph without the filters' f32 rounding.

``error_bound`` walks the same chain and bounds |device - model| from the filters' documented bounds: a FIR stage adds
``fir_rel * ||taps||_1 * max|input|`` and multiplies the error it receives by ``||taps||_1`` (a resampler: by the
largest L1 norm of one polyphase arm, since each output uses one arm); an oscillator stage multiplies the error by
the oscillator's largest magnitude times its gain and adds 8 f32 roundings of its largest output."""
from __future__ import annotations

from math import gcd

import numpy as np

import ssb_oracle as so
from fir_exact import resamp
from futuresdr_b200 import firdes, ssb

FIR_REL = 3e-5          # b200sdr.h: worst case of the split-bf16 tensor FIR (the direct kernel is within 1e-5)
U = 2.0 ** -24


def _conv(x, h):
    from scipy.signal import oaconvolve
    x = np.asarray(x, np.complex128 if np.iscomplexobj(x) else np.float64)
    return oaconvolve(x, np.asarray(h, np.float64), "valid")


def resampler_taps(interp, decim):
    g = gcd(int(interp), int(decim))
    L, M = int(interp) // g, int(decim) // g
    return L, M, firdes.kaiser.multirate(L, M, 12, 0.0001)


def resample(x, interp, decim, n_out=None):
    """FirBuilder::resampling(interp, decim) in float64: every output the input allows (the first n_out of them)."""
    L, M, taps = resampler_taps(interp, decim)
    T = taps.size // L
    n_max = max(0, ((len(x) - T) * L) // M + 1) if len(x) >= T else 0
    while n_max > 0 and ((n_max - 1) * M) // L + T > len(x):
        n_max -= 1
    return resamp(taps, L, M, x, n_max if n_out is None else min(n_out, n_max))


def arm_l1(interp, decim):
    L, _, taps = resampler_taps(interp, decim)
    return max(float(np.sum(np.abs(taps[b::L]))) for b in range(L))


def transmit(audio, mode="lsb", audio_rate=48_000) -> dict:
    """Every stream of the transmit graph: "lowpass", "to_complex", "resampler", "mixer", "file_level"."""
    lp = _conv(audio, ssb.lowpass_taps(audio_rate))
    i = lp[ssb.HILBERT_LEN // 2:]
    q = _conv(lp, ssb.hilbert_taps())
    m = min(i.size, q.size)
    c = i[:m] + (-1j if mode == "lsb" else 1j) * q[:m]
    r = resample(c, ssb.FILE_RATE, audio_rate)
    mix = so.Mixer(so.ROTATE, ssb.mixer_phase()).work(r.astype(np.complex64))
    return {"lowpass": lp, "to_complex": c, "resampler": r, "mixer": mix,
            "file_level": mix.astype(np.complex128) * (ssb.FILE_LEVEL_GAIN / ssb.FILE_LEVEL_ADJUSTMENT)}


def receive(x, audio_rate=48_000) -> dict:
    """Every stream of the receive graph: "xlating", "resampler", "weaver" (the audio)."""
    xl = so.Mixer(so.ROTATE_SCALE, ssb.xlating_phase(), ssb.FILE_LEVEL_ADJUSTMENT).work(np.asarray(x, np.complex64))
    r = resample(xl, audio_rate, ssb.FILE_RATE)
    w = so.Mixer(so.WEAVER, ssb.weaver_phase(audio_rate), ssb.VOLUME_ADJUSTMENT).work(r.astype(np.complex64))
    return {"xlating": xl, "resampler": r, "weaver": w}


def error_bound(audio, audio_rate=48_000, rx_rate=48_000, osc_max=1.0 + 1e-3) -> float:
    """A bound on |device audio - model audio| for `audio` through transmit (at audio_rate) -> file -> receive (at
    rx_rate); see the module doc.
    osc_max bounds |osc| over the streams (it drifts from 1 by far less than 1e-3 over 10^7 steps)."""
    lp_t, h_t = ssb.lowpass_taps(audio_rate), ssb.hilbert_taps()
    l1_lp, l1_h = float(np.sum(np.abs(lp_t))), float(np.sum(np.abs(h_t)))
    a = float(np.max(np.abs(audio)))
    e, mx = FIR_REL * l1_lp * a, l1_lp * a                                   # low-pass
    e = np.hypot(e, FIR_REL * l1_h * mx + l1_h * e)                           # delay (exact) and Hilbert parts
    mx = mx * np.hypot(1.0, l1_h)
    ar = arm_l1(ssb.FILE_RATE, audio_rate)                                    # resampler to the file rate
    e, mx = FIR_REL * ar * mx + ar * e, ar * mx
    e, mx = osc_max * e + 8 * U * osc_max * mx, osc_max * mx                  # mixer
    g = ssb.FILE_LEVEL_GAIN / ssb.FILE_LEVEL_ADJUSTMENT                       # file level: two roundings
    e, mx = g * e + 4 * U * g * mx, g * mx
    g = ssb.FILE_LEVEL_ADJUSTMENT                                             # xlating
    e, mx = osc_max * g * e + 8 * U * osc_max * g * mx, osc_max * g * mx
    ar = arm_l1(rx_rate, ssb.FILE_RATE)                                       # resampler to the audio rate
    e, mx = FIR_REL * ar * mx + ar * e, ar * mx
    g = ssb.VOLUME_ADJUSTMENT                                                 # Weaver: |re*c + im*s| <= |v| |osc|
    return osc_max * g * e + 8 * U * osc_max * g * mx


def spectrum_db(x, fs):
    """(frequencies, power in dB) of a Hann-windowed FFT of x, two-sided for complex x."""
    x = np.asarray(x)
    w = np.hanning(x.size)
    X = np.fft.fft(x * w) if np.iscomplexobj(x) else np.fft.rfft(x * w)
    f = np.fft.fftfreq(x.size, 1.0 / fs) if np.iscomplexobj(x) else np.fft.rfftfreq(x.size, 1.0 / fs)
    return f, 20 * np.log10(np.abs(X) + 1e-300)


def tones(freqs, audio_rate, n, amp=0.4):
    t = np.arange(n) / audio_rate
    return sum(amp * np.cos(2 * np.pi * f * t + 0.3 * k) for k, f in enumerate(freqs)).astype(np.float32)


def level_at(f, p, freq, half_width):
    sel = np.abs(f - freq) <= half_width
    return float(np.max(p[sel]))
