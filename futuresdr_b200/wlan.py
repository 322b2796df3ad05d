"""The WLAN transmitter (examples/wlan): the MCS table and FrameParam (lib.rs:223-363), the device encoder, the
length of a burst, and ``transmitter()``, the graph of bin/tx.rs:44-66 without its radio sink.

The receive chain past the front end (SyncShort, SyncLong, FrameEqualizer, Decoder) and the radio sink are not part of
this module: the transmitter is a source whose Complex32 stream a VectorSink or FileSink can read, and its
burst_start tags come back as records (``WlanTransmitter.bursts()``)."""
from __future__ import annotations

import ctypes as C
import enum
from dataclasses import dataclass

import torch

from ._lib import WLAN_MAX_PAYLOAD, WLAN_MAX_PSDU, check, lib  # noqa: F401
from .blocks import WlanTransmitter, _payload_batch
from .context import default_context

PAD_FRONT = 5000                          # bin/tx.rs:40
PAD_TAIL = 5000                           # bin/tx.rs:41
SRC_MAC = bytes([0x42] * 6)               # bin/tx.rs:49
DST_MAC = bytes([0x23] * 6)
BSS_MAC = bytes([0xFF] * 6)


class Mcs(enum.IntEnum):
    """lib.rs:223-312, numbered as the reference's enum (and B2S_WLAN_*)."""
    BPSK_1_2 = 0
    BPSK_3_4 = 1
    QPSK_1_2 = 2
    QPSK_3_4 = 3
    QAM16_1_2 = 4
    QAM16_3_4 = 5
    QAM64_2_3 = 6
    QAM64_3_4 = 7

    @property
    def n_bpsc(self) -> int:
        """Coded bits per subcarrier."""
        return (1, 1, 2, 2, 4, 4, 6, 6)[self]

    @property
    def n_cbps(self) -> int:
        """Coded bits per OFDM symbol."""
        return 48 * self.n_bpsc

    @property
    def n_dbps(self) -> int:
        """Data bits per OFDM symbol."""
        return (24, 36, 48, 72, 96, 144, 192, 216)[self]

    @property
    def rate_field(self) -> int:
        """The SIGNAL field's 4 rate bits."""
        return (0x0D, 0x0F, 0x05, 0x07, 0x09, 0x0B, 0x01, 0x03)[self]

    @classmethod
    def parse(cls, s: str) -> "Mcs":
        """Mcs::parse: case-insensitive, '-' and '_' ignored ("qpsk-1-2", "QAM64_3_4")."""
        m = s.replace("-", "").replace("_", "").lower()
        names = {"bpsk12": cls.BPSK_1_2, "bpsk34": cls.BPSK_3_4, "qpsk12": cls.QPSK_1_2, "qpsk34": cls.QPSK_3_4,
                 "qam1612": cls.QAM16_1_2, "qam1634": cls.QAM16_3_4, "qam6423": cls.QAM64_2_3,
                 "qam6434": cls.QAM64_3_4}
        if m not in names:
            raise ValueError(f"Invalid MCS {s}")
        return names[m]


@dataclass(frozen=True)
class FrameParam:
    """FrameParam::new (lib.rs:323-363), computed by the library."""
    mcs: Mcs
    psdu_size: int
    n_symbols: int
    n_data_bits: int
    n_pad: int

    @classmethod
    def new(cls, mcs, psdu_size: int) -> "FrameParam":
        ns, nb, npad = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
        check(lib.b2s_wlan_frame_param(int(mcs), int(psdu_size), C.byref(ns), C.byref(nb), C.byref(npad)))
        return cls(Mcs(mcs), int(psdu_size), ns.value, nb.value, npad.value)


def frame_len(mcs, payload_len: int, pad_front: int = PAD_FRONT, pad_tail: int = PAD_TAIL) -> int:
    """Samples of the burst Prefix makes of one payload (prefix.rs:126): the PSDU adds 28 bytes, and the burst holds
    the SIGNAL symbol and the data symbols at 80 samples each."""
    n = FrameParam.new(mcs, int(payload_len) + 28).n_symbols + 1
    return int(pad_front) + 320 + 80 * n + max(int(pad_tail), 1)


def encode(payloads, mcs, src_mac=SRC_MAC, dst_mac=DST_MAC, bss_mac=BSS_MAC, sequence_number: int = 0,
           scrambler_seed: int = 1, ctx=None) -> list[torch.Tensor]:
    """Mac + Encoder + SIGNAL field of each payload as one batch on the device, from a fresh encoder: a list of device
    uint8 tensors of shape (1 + n_symbols, 48), one per payload, row 0 the SIGNAL symbol.  ``mcs`` is one MCS or one
    per payload; frame i has sequence number ``sequence_number + i`` and scrambler seed ``scrambler_seed + i``, both
    wrapping as the reference's do."""
    ctx = ctx or default_context()
    data, buf, lens = _payload_batch(payloads)
    n = len(data)
    ms = [int(mcs)] * n if isinstance(mcs, (int, enum.IntEnum)) else [int(m) for m in mcs]
    if len(ms) != n:
        raise ValueError(f"encode: {len(ms)} MCS for {n} payloads")
    rows = [1 + FrameParam.new(m, len(d) + 28).n_symbols if len(d) <= WLAN_MAX_PAYLOAD else 0
            for m, d in zip(ms, data)]
    dev = torch.device("cuda", ctx.device)
    d_pay = torch.frombuffer(bytearray(buf or b"\0"), dtype=torch.uint8).to(dev)     # a valid pointer when empty
    d_sym = torch.zeros(max(sum(rows), 1), 48, dtype=torch.uint8, device=dev)
    mc = (C.c_int32 * max(n, 1))(*ms)
    got = C.c_size_t(0)
    addrs = [C.c_char_p(bytes(a)) for a in (src_mac, dst_mac, bss_mac)]
    check(lib.b2s_wlan_encode(ctx.handle, *addrs, int(sequence_number), int(scrambler_seed),
                              C.c_void_p(d_pay.data_ptr()), lens, mc, n, C.c_void_p(d_sym.data_ptr()),
                              d_sym.shape[0], C.byref(got)), ctx.handle)
    return list(d_sym[:sum(rows)].split(rows))


def transmitter(fg, default_mcs=Mcs.QPSK_1_2, src_mac=SRC_MAC, dst_mac=DST_MAC, bss_mac=BSS_MAC,
                pad_front: int = PAD_FRONT, pad_tail: int = PAD_TAIL, ctx=None) -> WlanTransmitter:
    """bin/tx.rs:44-66 without the radio sink: adds a WlanTransmitter (Mac, Encoder at ``default_mcs``, Mapper, the
    64-point inverse Fft and Prefix) to ``fg``; connect its "output" to a sink and ``push`` payloads into it."""
    tx = WlanTransmitter(src_mac, dst_mac, bss_mac, int(default_mcs), pad_front, pad_tail, ctx)
    fg.add(tx)
    return tx
