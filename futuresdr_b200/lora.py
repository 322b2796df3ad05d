"""The LoRa transmitter (examples/lora): its enums and defaults (utils.rs, default_values.rs), the sync word's
expansion, ``sample_count``, the device encoder, and ``transmitter()``, the graph builder of lib.rs:47-74.

The receive chain (FrameSync and the blocks after it), Meshtastic encryption and the radio sinks are not part of this
module: the transmitter is a source whose Complex32 stream a VectorSink or FileSink can read."""
from __future__ import annotations

import ctypes as C
import enum
import math

import numpy as np
import torch

from ._lib import check, lib
from .blocks import LoraTransmitter, _payload_batch
from .context import default_context

PREAMBLE_LEN = 8                         # default_values.rs:7
HAS_CRC = True                           # default_values.rs:6
OVERSAMPLING_TX = 8                      # default_values.rs:10
LDRO_MAX_DURATION_MS = np.float32(16.0)  # default_values.rs:15


class SpreadingFactor(enum.IntEnum):
    SF5 = 5
    SF6 = 6
    SF7 = 7
    SF8 = 8
    SF9 = 9
    SF10 = 10
    SF11 = 11
    SF12 = 12

    def samples_per_symbol(self) -> int:
        return 1 << int(self)


class CodeRate(enum.IntEnum):
    """utils.rs:631-661: the number the header carries."""
    CR_4_5 = 1
    CR_4_6 = 2
    CR_4_7 = 3
    CR_4_8 = 4


class Bandwidth(enum.IntEnum):
    """utils.rs:278-309, in Hz."""
    BW62 = 62_500
    BW125 = 125_000
    BW250 = 250_000
    BW500 = 500_000


class LdroMode(enum.IntEnum):
    DISABLE = 0
    ENABLE = 1
    AUTO = 2

    def resolve_if_auto(self, sf, bw) -> "LdroMode":
        """utils.rs:693-705: AUTO enables LDRO when a symbol lasts longer than 16 ms, computed in f32."""
        if self != LdroMode.AUTO:
            return self
        dur = np.float32(np.float32(np.float32(1 << int(sf)) * np.float32(1e3)) / np.float32(int(bw)))
        return LdroMode.ENABLE if dur > LDRO_MAX_DURATION_MS else LdroMode.DISABLE

    def enabled(self) -> bool:
        assert self != LdroMode.AUTO
        return self == LdroMode.ENABLE


def preamble_len(sf) -> int:
    """default_values.rs:17-23."""
    return 12 if int(sf) == 5 else PREAMBLE_LEN


class SynchWord:
    """utils.rs:336-496: a compact u8 (0x12 private, 0x34 public, 0x2B Meshtastic) or two expanded symbols."""
    PRIVATE, PUBLIC, MESHTASTIC = 0x12, 0x34, 0x2B

    def __init__(self, value: int | None = None, expanded: tuple[int, int] | None = None):
        if (value is None) == (expanded is None):
            raise ValueError("SynchWord: a compact value or expanded symbols")
        self.value, self.expanded = value, expanded

    @classmethod
    def from_pmt(cls, word) -> "SynchWord":
        """transmitter.rs:95-107: an int is a u8 (TryInto::<u8> fails above 255); bytes of length 1 or 2 are
        SynchWord::try_from(&[u8])."""
        if isinstance(word, SynchWord):
            return word
        if isinstance(word, int):
            if not 0 <= word <= 0xFF:
                raise ValueError(f"SynchWord: {word} is not a u8")
            return cls(value=word)
        b = bytes(word)
        if len(b) == 1:
            return cls(value=b[0])
        if len(b) == 2:
            return cls(expanded=(b[0], b[1]))
        raise ValueError(f"invalid value for synch word: {list(b)}")

    def expand(self) -> tuple[int, int]:
        if self.expanded is not None:
            return self.expanded
        v = self.value
        return ((v & 0xF0) >> 4) << 3, (v & 0x0F) << 3

    def verify_and_expand(self, sf) -> tuple[int, int]:
        s = self.expand()
        if any(x >= (1 << int(sf)) for x in s):
            raise ValueError(f"LoRa Modulator: can not encode sync word symbols {list(s)} with SF{int(sf)}")
        return s


def sample_count(sf, preamble_len, explicit_header: bool, payload_len, has_crc, code_rate, os_factor, pad,
                 ldro_enabled) -> int:
    """utils.rs:988-1020 in its f32 arithmetic.  Its usize subtractions underflow for payloads that fit the first
    interleaver block (a panic in a debug build): that raises ValueError here."""
    sf, cr = int(sf), int(code_rate)
    f = np.float32
    pre = f(f(preamble_len) + f(4.25) + (f(2.0) if sf < 7 else f(0.0)))
    hdr = 5 if explicit_header else 0
    pay = 2 * int(payload_len) + (4 if has_crc else 0)
    sub = sf - (2 if sf >= 7 else 0)
    if pay + hdr < sub:
        raise ValueError("sample_count: the payload fits the first block (usize underflow in the reference)")
    blocks = f(math.ceil(f(f(pay + hdr - sub) / f(sf - (2 if ldro_enabled else 0)))))
    total = f(f(f(pre + f(8.0)) + f(blocks * f(4 + cr))) * f((1 << sf) * int(os_factor)))
    v = int(total) + 2 * int(pad)
    if v < int(os_factor):
        raise ValueError("sample_count: usize underflow in the reference")
    return v - int(os_factor)


def symbol_count(sf, code_rate, has_crc, ldro_enabled, implicit_header, payload_len) -> int:
    """The symbols Encoder::encode makes of a payload of ``payload_len`` bytes."""
    n = C.c_size_t(0)
    check(lib.b2s_lora_symbol_count(int(sf), int(code_rate), int(has_crc), int(ldro_enabled), int(implicit_header),
                                    int(payload_len), C.byref(n)))
    return n.value


def frame_len(sf, oversampling, preamble_len, pad, n_symbols) -> int:
    """Samples of one modulated frame (modulator.rs:46-152)."""
    N = (1 << int(sf)) * int(oversampling)
    return 2 * pad + (preamble_len + 4 + (2 if int(sf) < 7 else 0)) * N + N // 4 - oversampling + n_symbols * N


def encode(payloads, sf, code_rate, has_crc, ldro_enabled, implicit_header, ctx=None) -> list[torch.Tensor]:
    """Encoder::encode of each payload, as one batch on the device: a list of device tensors, one per payload, of its
    u16 symbols held in torch.int16 (``.cpu().numpy().view(np.uint16)`` reads them back)."""
    ctx = ctx or default_context()
    data, buf, lens = _payload_batch(payloads)
    counts = [symbol_count(sf, code_rate, has_crc, ldro_enabled, implicit_header, len(d)) for d in data]
    dev = torch.device("cuda", ctx.device)
    d_pay = torch.frombuffer(bytearray(buf or b"\0"), dtype=torch.uint8).to(dev)     # a valid pointer when empty
    d_sym = torch.zeros(max(sum(counts), 1), dtype=torch.int16, device=dev)
    n = C.c_size_t(0)
    check(lib.b2s_lora_encode(ctx.handle, int(sf), int(code_rate), int(has_crc), int(ldro_enabled),
                              int(implicit_header), C.c_void_p(d_pay.data_ptr()), lens, len(data),
                              C.c_void_p(d_sym.data_ptr()), d_sym.numel(), C.byref(n)), ctx.handle)
    return list(d_sym[:sum(counts)].split(counts))


def transmitter(fg, bw=Bandwidth.BW125, sf=SpreadingFactor.SF7, code_rate=CodeRate.CR_4_5, has_crc=HAS_CRC,
                ldro=LdroMode.AUTO, implicit_header=False, os_factor=4, sync_word=SynchWord.PRIVATE,
                preamble_len_=None, pad=0, ctx=None) -> LoraTransmitter:
    """build_lora_tx (lib.rs:47-74): resolves LDRO for the bandwidth, expands and checks the sync word, and adds a
    LoraTransmitter to ``fg``; connect its "output" to a sink."""
    ldro_enabled = LdroMode(ldro).resolve_if_auto(sf, bw).enabled()
    sync = SynchWord.from_pmt(sync_word).verify_and_expand(sf)
    tx = LoraTransmitter(int(sf), int(code_rate), has_crc, ldro_enabled, implicit_header, os_factor, sync,
                         preamble_len(sf) if preamble_len_ is None else preamble_len_, pad, ctx)
    fg.add(tx)
    return tx
