"""ZigBee (IEEE 802.15.4 O-QPSK, examples/zigbee): the receiver's chip table, the Mac's FCS and its receive front end
(rx.rs:66-92) down to decoded frames; the transmitter's frame length and ``transmitter()``, the graph of tx.rs:37-56
(Mac -> modulator -> IqDelay) without its radio sink.  Together they run the transceiver of trx.rs on the device:
``transmitter()`` into ``front_end()``.

The transmitter is a source whose Complex32 stream a VectorSink, FileSink or the front end can read, and its
burst_start tags come back as records (``ZigbeeTransmitter.bursts()``).  The Mac's rftap / UDP output and its
``stats`` handler are host-side message handling and not part of this package."""
from __future__ import annotations

import numpy as np

from ._lib import ZIGBEE_MAX_PAYLOAD, ZIGBEE_PADDING
from .blocks import Apply, ApplyOp, ClockRecoveryMm, ZigbeeDecoder, ZigbeeTransmitter

CHIP_MAPPING = np.array([1618456172, 1309113062, 1826650030, 1724778362, 778887287, 2061946375, 2007919840,
                         125494990, 529027475, 838370585, 320833617, 422705285, 1368596360, 85537272, 139563807,
                         2021988657], np.uint32)                                  # decoder.rs
CHIP_MASK = 0x7FFFFFFE
DC_ALPHA = 0.00016                                                                # rx.rs:67
MM_OMEGA, MM_GAIN_OMEGA, MM_MU, MM_GAIN_MU, MM_OMEGA_RELATIVE_LIMIT = 2.0, 0.000225, 0.5, 0.03, 0.0002   # rx.rs:78-82
DECODER_THRESHOLD = 6                                                             # rx.rs:86
PADDING = ZIGBEE_PADDING                                                          # iq_delay.rs:11
MAX_PAYLOAD = ZIGBEE_MAX_PAYLOAD                                                  # MAX_FRAME_SIZE - 11 (mac.rs:155)


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


def frame_len(n: int, pad: int = PADDING) -> int:
    """Samples IqDelay makes of the frame of an n-byte payload (iq_delay.rs:112-118): the frame's n + 16 bytes at 128
    samples each, the two held Q samples, and ``pad`` zeros before and after."""
    return 2 * int(pad) + 128 * (int(n) + 16) + 2


def transmitter(fg, pad: int = PADDING, ctx=None) -> ZigbeeTransmitter:
    """tx.rs:37-56 without the radio sink: adds a ZigbeeTransmitter (Mac, modulator, IqDelay with ``pad``) to ``fg``;
    connect its "output" to a sink, or pass it to ``front_end`` as the source, and ``push`` payloads into it."""
    tx = ZigbeeTransmitter(pad, ctx)
    fg.add(tx)
    return tx
