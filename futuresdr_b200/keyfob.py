"""The keyfob receiver (examples/keyfob): its constants, the low-pass taps, the string the reference logs for a code,
and its receive front end (main.rs:39-79) down to decoded key codes."""
from __future__ import annotations

from math import gcd

import numpy as np

from . import firdes, windows
from ._lib import KEYFOB_CLOSE, KEYFOB_NONE, KEYFOB_OPEN, KEYFOB_TRUNK
from .blocks import Apply, ApplyOp, FirBuilder, KeyfobDecoder

SAMPLE_RATE = 250_000                                            # main.rs:43, :54 (resampled rate)
DC_ALPHA = 0.0001                                                # main.rs:63
LOWPASS_CUTOFF_HZ = 15e3                                         # main.rs:70
LOWPASS_TAPS = 128                                               # main.rs:70, windows::hamming(128, false)
PREAMBLE = "10101111"                                            # decoder.rs:37
LABELS = {KEYFOB_NONE: "", KEYFOB_CLOSE: " (Close)", KEYFOB_OPEN: " (Open)", KEYFOB_TRUNK: " (Trunk)"}   # :42-48


def lowpass_taps() -> np.ndarray:
    """firdes::lowpass::<f32>(15e3 / 250e3, &windows::hamming(128, false)) (main.rs:70)."""
    return firdes.lowpass(LOWPASS_CUTOFF_HZ / SAMPLE_RATE, windows.hamming(LOWPASS_TAPS, False))


def code_string(rec) -> str:
    """What the reference logs after ``RXed `` for a KEYFOB_CODE record, label suffix included.  Exact for
    n_bits <= 256; a longer string keeps only its first 256 bits and ends in ``...`` before the suffix (the label
    still comes from the true last 8 bits)."""
    n = int(rec["n_bits"])
    bits = np.unpackbits(np.asarray(rec["bits"], np.uint8))[:min(n, 256)]
    s = "".join("1" if b else "0" for b in bits)
    if n > 256:
        s += "..."
    return s + LABELS[int(rec["label"])]


def front_end(fg, src, sample_rate: int = 4_000_000, ctx=None):
    """main.rs:39-79 from ``src`` (a Complex32 block already in ``fg``): the gcd-reduced resampler to 250 kHz,
    Apply(NormSqr), Apply(DcBlockF32, 0.0001) for the running-average closure, the 128-tap Hamming low-pass FIR,
    Apply(SliceF32U8) and KeyfobDecoder.  Returns a dict of the blocks ("resamp", "mag2", "avg", "low_pass", "slice",
    "decoder")."""
    g = gcd(SAMPLE_RATE, int(sample_rate))
    resamp = FirBuilder.resampling(SAMPLE_RATE // g, int(sample_rate) // g, np.complex64, ctx)
    mag2 = Apply(ApplyOp.NormSqr, ctx=ctx)
    avg = Apply(ApplyOp.DcBlockF32, DC_ALPHA, ctx=ctx)
    low_pass = FirBuilder.fir(lowpass_taps(), np.float32, ctx)
    slicer = Apply(ApplyOp.SliceF32U8, ctx=ctx)
    decoder = KeyfobDecoder(ctx)
    fg.connect(src, resamp)
    fg.connect(resamp, mag2)
    fg.connect(mag2, avg)
    fg.connect(avg, low_pass)
    fg.connect(low_pass, slicer)
    fg.connect(slicer, decoder)
    return {"resamp": resamp, "mag2": mag2, "avg": avg, "low_pass": low_pass, "slice": slicer, "decoder": decoder}
