"""CPU oracle of the keyfob receiver's running average, slicer and Decoder (TEST INFRASTRUCTURE ONLY).

ctypes front-end to ``tests/keyfob_oracle.c`` (one reference call at a time, compiled by ``native.load_oracle`` on
first use).  ``Avg`` and ``Decoder`` carry a block's state across calls; ``py_decode`` is an independent pure-Python
transcription of decoder.rs for cross-checking the C file; ``code_tuple`` turns a device KEYFOB_CODE record into the
oracle's tuple form.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from native import load_oracle

_f32p = C.POINTER(C.c_float)
_u8p = C.POINTER(C.c_uint8)

LABELS = {"11010101": 1, "11100011": 2, "10111001": 3}          # Close, Open, Trunk


class DecState(C.Structure):
    _fields_ = [("n_read", C.c_uint64), ("since", C.c_uint64), ("up", C.c_uint32), ("output", C.c_uint32),
                ("s", C.c_void_p), ("len", C.c_size_t), ("cap", C.c_size_t)]


class Code(C.Structure):
    _fields_ = [("index", C.c_uint64), ("n_bits", C.c_uint32), ("label", C.c_int32), ("bits", C.c_uint8 * 32)]


SIGNATURES = {
    "orc_kf_avg": (None, [C.c_float, _f32p, _f32p, C.c_size_t, _f32p]),
    "orc_kf_slice": (None, [_f32p, C.c_size_t, _u8p]),
    "orc_kf_dec_new": (None, [C.POINTER(DecState)]),
    "orc_kf_dec_free": (None, [C.POINTER(DecState)]),
    "orc_kf_dec_work": (C.c_size_t, [C.POINTER(DecState), _u8p, C.c_size_t, C.POINTER(Code), C.c_size_t]),
}


def lib() -> C.CDLL:
    return load_oracle("keyfob_oracle", SIGNATURES)


class Avg:
    """main.rs:62-68, the running-average closure (alpha 0.0001 by default)."""

    def __init__(self, alpha=0.0001):
        self.alpha = float(np.float32(alpha))
        self.cur = C.c_float(0.0)

    def work(self, x) -> np.ndarray:
        x = np.ascontiguousarray(x, np.float32)
        y = np.empty_like(x)
        lib().orc_kf_avg(self.alpha, C.byref(self.cur), x.ctypes.data_as(_f32p), x.size, y.ctypes.data_as(_f32p))
        return y


def slice_u8(x) -> np.ndarray:
    x = np.ascontiguousarray(x, np.float32)
    y = np.empty(x.size, np.uint8)
    lib().orc_kf_slice(x.ctypes.data_as(_f32p), x.size, y.ctypes.data_as(_u8p))
    return y


def _tuple(c) -> tuple:
    return (int(c.index), int(c.n_bits), int(c.label), bytes(c.bits))


def code_tuple(rec) -> tuple:
    return (int(rec["index"]), int(rec["n_bits"]), int(rec["label"]), bytes(np.asarray(rec["bits"], np.uint8)))


class Decoder:
    """decoder.rs:64-127: one work() call at a time."""

    def __init__(self):
        self.s = DecState()
        lib().orc_kf_dec_new(C.byref(self.s))

    def __del__(self):
        try:
            lib().orc_kf_dec_free(C.byref(self.s))
        except Exception:  # noqa: BLE001
            pass

    def work(self, x) -> list:
        """One call (consumes everything) -> [(index, n_bits, label, bits[32])] of the strings it logs."""
        x = np.ascontiguousarray(x, np.uint8)
        cap = x.size // 504 + 2
        out = (Code * cap)()
        n = lib().orc_kf_dec_work(C.byref(self.s), x.ctypes.data_as(_u8p), x.size, out, cap)
        assert n <= cap
        return [_tuple(out[k]) for k in range(n)]


def decode(x, cuts=()) -> list:
    """The codes of one stream, work() called on the slices between `cuts`."""
    x = np.ascontiguousarray(x, np.uint8)
    d, got = Decoder(), []
    edges = [0] + [c for c in cuts if 0 < c < x.size] + [x.size]
    for a, b in zip(edges[:-1], edges[1:]):
        got += d.work(x[a:b])
    return got


def _pack(s: str) -> bytes:
    b = bytearray(32)
    for i, ch in enumerate(s[:256]):
        if ch == "1":
            b[i // 8] |= 0x80 >> (i % 8)
    return bytes(b)


def py_decode(x) -> list:
    """decoder.rs:36-127 transcribed literally in Python (strings, State::Up / State::Down)."""
    up, since, output, s, got = False, 0, False, "", []
    for pos, v in enumerate(np.asarray(x, np.uint8).tolist()):
        if (not up and v == 1) or (up and v == 0):
            diff = pos - since
            if 63 <= diff <= 83:
                if not output:
                    output = True
                else:
                    output = False
                    s += "1" if up else "0"
            elif 131 <= diff <= 161:
                output = False
                s += "1" if up else "0"
            else:
                off = s.find("10101111")
                t = s[off:] if off >= 0 else ""
                s = ""
                if len(t) >= 8:
                    got.append((pos, len(t), LABELS.get(t[-8:], 0), _pack(t)))
            up = not up
            since = pos
    return got


def code_text(c) -> str:
    """The string the reference logs for an oracle tuple with n_bits <= 256 (label suffix included)."""
    _, n, label, bits = c
    s = "".join("1" if (bits[i // 8] >> (7 - i % 8)) & 1 else "0" for i in range(min(n, 256)))
    return s + {0: "", 1: " (Close)", 2: " (Open)", 3: " (Trunk)"}[label]


def levels_for(bits: str, rng=None, lead: int = 300, start_level: int = 0, short=(63, 83), long=(131, 161)) -> np.ndarray:
    """A slicer stream that the decoder turns into `bits` and then flushes.  A bit b is appended by the edge that ends
    a period at level b (a low period ends in a rising edge: "0").  From level b that is one long period (131..=161
    items); from the other level a short period (63..=83, it sets `output`) first, then a short or a long one.  The
    stream starts at `start_level` for `lead` items (its first edge flushes when lead is outside both ranges) and
    ends with a 20-item period, whose edge flushes the string.  Period widths are drawn from `short` and `long`."""
    rng = rng or np.random.default_rng(0)
    out, level = [np.full(lead, start_level, np.uint8)], start_level ^ 1

    def period(lo, hi):
        nonlocal level
        out.append(np.full(int(rng.integers(lo, hi + 1)), level, np.uint8))
        level ^= 1

    for ch in bits:
        b = int(ch)
        if level != b:
            period(*short)
            if rng.random() < 0.5:
                period(*short)
                continue
        period(*long)
    period(20, 20)
    out.append(np.full(5, level, np.uint8))
    return np.concatenate(out)
