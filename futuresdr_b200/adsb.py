"""The ADS-B receiver (examples/adsb): its constants, the preamble correlator taps and its receive front end
(listen_adsb.rs:85-120) down to CRC-checked 112-bit frames.  ``adsb_deku`` parsing and the ``Tracker`` are host-side
message handling and not part of this package."""
from __future__ import annotations

from math import gcd

import numpy as np

from .blocks import AdsbDemod, Apply, ApplyOp, FirBuilder

DEMOD_SAMPLE_RATE = 4_000_000                                   # lib.rs
N_SAMPLES_PER_HALF_SYM = DEMOD_SAMPLE_RATE // 2_000_000
SYMBOL_ONE_TAPS = np.array([1.0, 1.0, -1.0, -1.0], np.float32)
SYMBOL_ZERO_TAPS = np.array([-1.0, -1.0, 1.0, 1.0], np.float32)
PREAMBLE = np.array([1, -1, 1, -1, -1, -1, -1, 1, -1, 1, -1, -1, -1, -1, -1, -1], np.float32)   # preamble_detector.rs
CRC_GENERATOR = 0x1FFF409                                       # decoder.rs GENERATOR_POLY, 25 bits


def preamble_correlator_taps() -> np.ndarray:
    """PREAMBLE reversed, each half-symbol repeated N_SAMPLES_PER_HALF_SYM times: 32 taps."""
    return np.repeat(PREAMBLE[::-1], N_SAMPLES_PER_HALF_SYM).astype(np.float32)


def front_end(fg, src, sample_rate: int, threshold: float = 10.0, forward_failed_crc: bool = False, ctx=None):
    """listen_adsb.rs:85-120 from ``src`` (a Complex32 block already in ``fg``): the gcd-reduced resampler to
    DEMOD_SAMPLE_RATE, Apply(NormSqr), the 32-tap noise-floor FIR of 1/32, the preamble FIR and AdsbDemod.
    Returns a dict of the blocks ("resamp", "mag2", "nf", "corr", "demod")."""
    g = gcd(int(sample_rate), DEMOD_SAMPLE_RATE)
    interp, decim = DEMOD_SAMPLE_RATE // g, int(sample_rate) // g
    resamp = FirBuilder.resampling(interp, decim, np.complex64, ctx)
    mag2 = Apply(ApplyOp.NormSqr, ctx=ctx)
    nf = FirBuilder.fir(np.full(32, 1.0 / 32.0, np.float32), np.float32, ctx)
    corr = FirBuilder.fir(preamble_correlator_taps(), np.float32, ctx)
    demod = AdsbDemod(threshold, forward_failed_crc, ctx)
    fg.connect(src, resamp)
    fg.connect(resamp, mag2)
    fg.connect(mag2, nf)
    fg.connect(mag2, corr)
    fg.connect(mag2, demod, "in_samples")
    fg.connect(nf, demod, "in_nf")
    fg.connect(corr, demod, "in_preamble_cor")
    return {"resamp": resamp, "mag2": mag2, "nf": nf, "corr": corr, "demod": demod}
