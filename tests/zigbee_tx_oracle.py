"""CPU oracle of the ZigBee transmitter: Mac, modulator and IqDelay (TEST INFRASTRUCTURE ONLY).

ctypes front-end to ``tests/zigbee_tx_oracle.c`` (the blocks' work() calls one at a time, compiled by
``native.load_oracle`` on first use).  ``Tx`` carries the chain's state across calls.  ``np_stream`` is an independent
vectorised numpy transcription built on the reference's literal DSSS table and SHAPE
(``tests/golden/zigbee_tx_dsss.json``), for cross-checking the C file.
"""
from __future__ import annotations

import ctypes as C
import json
import os

import numpy as np

import zigbee_oracle as zo
from native import load_oracle

PADDING = 40000                     # iq_delay.rs:11
MAX_PAYLOAD = 116                   # MAX_FRAME_SIZE - 11 (mac.rs:155)

_f32p = C.POINTER(C.c_float)
_u64p = C.POINTER(C.c_uint64)
_szp = C.POINTER(C.c_size_t)

SIGNATURES = {
    "orc_zbtx_dsss": (None, [_f32p]),
    "orc_zbtx_shape": (None, [_f32p]),
    "orc_zbtx_new": (C.c_void_p, [C.c_size_t, C.c_size_t, C.c_size_t]),
    "orc_zbtx_free": (None, [C.c_void_p]),
    "orc_zbtx_tx": (C.c_int, [C.c_void_p, C.c_char_p, C.c_size_t]),
    "orc_zbtx_run": (C.c_long, [C.c_void_p, _f32p, C.c_size_t, C.c_uint64, _u64p, _u64p, C.c_size_t, _szp]),
}


def lib() -> C.CDLL:
    return load_oracle("zigbee_tx_oracle", SIGNATURES)


def golden() -> dict:
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "zigbee_tx_dsss.json")) as f:
        return json.load(f)


def dsss() -> np.ndarray:
    """The C oracle's generated table, (16 nibbles, 16 chips, re / im) float32."""
    t = np.zeros((16, 16, 2), np.float32)
    lib().orc_zbtx_dsss(t.ctypes.data_as(_f32p))
    return t


def shape() -> np.ndarray:
    s = np.zeros(4, np.float32)
    lib().orc_zbtx_shape(s.ctypes.data_as(_f32p))
    return s


def frame_len(n: int, pad: int = PADDING) -> int:
    return 2 * pad + 128 * (n + 16) + 2


class Tx:
    """Mac -> modulator -> IqDelay with buffers of c1 bytes and c2 samples between the blocks."""

    def __init__(self, pad: int = PADDING, c1: int = 4096, c2: int = 1 << 16):
        self.pad = int(pad)
        self.h = C.c_void_p(lib().orc_zbtx_new(self.pad, int(c1), int(c2)))
        self.pos = 0

    def __del__(self):
        if getattr(self, "h", None):
            lib().orc_zbtx_free(self.h)
            self.h = None

    def push(self, *payloads) -> int:
        """Mac::tx per payload -> the number dropped."""
        return sum(1 - lib().orc_zbtx_tx(self.h, bytes(p), len(p)) for p in payloads)

    def run(self, cap: int):
        """Work rounds until ``cap`` samples are out or nothing moves -> (complex64 samples, [(index, len)] bursts)."""
        out = np.zeros(max(cap, 1), np.complex64)
        tcap = cap // 2 + 2
        ti, tv = np.zeros(tcap, np.uint64), np.zeros(tcap, np.uint64)
        nt = C.c_size_t(0)
        p = lib().orc_zbtx_run(self.h, out.view(np.float32).ctypes.data_as(_f32p), cap, self.pos,
                               ti.ctypes.data_as(_u64p), tv.ctypes.data_as(_u64p), tcap, C.byref(nt))
        assert p >= 0, "IqDelay: no frame start tag"
        assert nt.value <= tcap
        self.pos += p
        return out[:p], [(int(ti[k]), int(tv[k])) for k in range(nt.value)]

    def stream(self, caps=(1 << 22,)):
        """run() over the given capacities (cycled) until a call produces nothing -> (samples, bursts)."""
        outs, bursts, k = [], [], 0
        while True:
            o, b = self.run(int(caps[k % len(caps)]))
            k += 1
            outs.append(o)
            bursts += b
            if o.size == 0:
                return np.concatenate(outs), bursts


# ---- independent numpy transcription -----------------------------------------------------------------------------
def np_frame(frame: bytes, pad: int, fx=None) -> np.ndarray:
    """modulator.rs then IqDelay for one Mac frame, from the reference's literals (``golden()``), as complex64."""
    fx = fx or golden()
    table = np.asarray(fx["dsss"], np.float32)                                    # (16, 16, 2)
    shp = np.asarray(fx["shape"], np.float32)
    b = np.frombuffer(bytes(frame), np.uint8)
    nib = np.stack([b & 0x0F, b >> 4], axis=1).reshape(-1)                        # low nibble first
    chips = np.repeat(table[nib], 4, axis=1)                                      # (2 nb, 64, 2): [x; 4]
    m = (chips * np.tile(shp, 16)[None, :, None]).astype(np.float32).reshape(-1, 2)
    z2 = np.zeros(2, np.float32)
    re = np.concatenate([np.zeros(pad, np.float32), m[:, 0], z2, np.zeros(pad, np.float32)])
    im = np.concatenate([np.zeros(pad, np.float32), z2, m[:, 1], np.zeros(pad, np.float32)])
    out = np.empty(re.size, np.complex64)
    out.real, out.imag = re, im
    return out


def np_stream(payloads, pad: int, seq0: int = 0):
    """The whole stream of the payloads (oversized ones dropped) -> (complex64 samples, [(index, len)] bursts)."""
    fx = golden()
    parts, bursts, pos, seq = [], [], 0, seq0
    for p in payloads:
        if len(p) > MAX_PAYLOAD:
            continue
        f = np_frame(zo.mac_frame(p, seq), pad, fx)
        seq = (seq + 1) & 0xFF
        bursts.append((pos, f.size))
        parts.append(f)
        pos += f.size
    return (np.concatenate(parts) if parts else np.zeros(0, np.complex64)), bursts


def same_bits(a: np.ndarray, b: np.ndarray) -> bool:
    """complex64 arrays equal bit for bit (so +0.0 and -0.0 differ)"""
    a, b = np.ascontiguousarray(a, np.complex64), np.ascontiguousarray(b, np.complex64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))
