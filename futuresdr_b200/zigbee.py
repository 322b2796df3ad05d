"""The ZigBee (IEEE 802.15.4 O-QPSK) receiver (examples/zigbee): its chip table, the Mac's FCS and its receive front
end (rx.rs:66-92) down to decoded frames.  The Mac's rftap / UDP output is host-side message handling and not part of
this package."""
from __future__ import annotations

import numpy as np

from .blocks import Apply, ApplyOp, ClockRecoveryMm, ZigbeeDecoder

CHIP_MAPPING = np.array([1618456172, 1309113062, 1826650030, 1724778362, 778887287, 2061946375, 2007919840,
                         125494990, 529027475, 838370585, 320833617, 422705285, 1368596360, 85537272, 139563807,
                         2021988657], np.uint32)                                  # decoder.rs
CHIP_MASK = 0x7FFFFFFE
DC_ALPHA = 0.00016                                                                # rx.rs:67
MM_OMEGA, MM_GAIN_OMEGA, MM_MU, MM_GAIN_MU, MM_OMEGA_RELATIVE_LIMIT = 2.0, 0.000225, 0.5, 0.03, 0.0002   # rx.rs:78-82
DECODER_THRESHOLD = 6                                                             # rx.rs:86


def calc_crc(data) -> int:
    """Mac::calc_crc (mac.rs:62-80): CRC-16, reflected polynomial 0x1021, initial value 0.  A frame whose last two
    bytes are its FCS (little endian) gives 0."""
    crc = 0
    for b in bytes(data):
        for k in range(8):
            bit = ((b >> k) & 1) ^ (crc & 1)
            crc >>= 1
            if bit:
                crc ^= 0x8408
    return crc


def front_end(fg, src, ctx=None):
    """rx.rs:66-92 from ``src`` (a Complex32 block already in ``fg``): Apply(QuadDemod) and Apply(DcBlockF32) for the
    phase-difference-minus-DC closure, ClockRecoveryMm(2.0, 0.000225, 0.5, 0.03, 0.0002) and ZigbeeDecoder(6).
    Returns a dict of the blocks ("phase", "dc", "mm", "decoder")."""
    phase = Apply(ApplyOp.QuadDemod, ctx=ctx)
    dc = Apply(ApplyOp.DcBlockF32, DC_ALPHA, ctx=ctx)
    mm = ClockRecoveryMm(MM_OMEGA, MM_GAIN_OMEGA, MM_MU, MM_GAIN_MU, MM_OMEGA_RELATIVE_LIMIT, ctx=ctx)
    decoder = ZigbeeDecoder(DECODER_THRESHOLD, ctx=ctx)
    fg.connect(src, phase)
    fg.connect(phase, dc)
    fg.connect(dc, mm)
    fg.connect(mm, decoder)
    return {"phase": phase, "dc": dc, "mm": mm, "decoder": decoder}
