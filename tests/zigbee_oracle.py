"""CPU oracle of the ZigBee receiver's DC blocker, ClockRecoveryMm, Decoder and Mac::calc_crc (TEST INFRASTRUCTURE ONLY).

ctypes front-end to ``tests/zigbee_oracle.c`` (one reference call at a time, compiled by ``native.load_oracle`` on
first use).  ``DcBlock``, ``Mm`` and ``Decoder`` carry a block's state across calls; ``np_*`` are an independent
numpy float32 transcription for cross-checking the C file, and ``crc16_table`` a table-driven CRC for cross-checking
``calc_crc``.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from native import load_oracle

_f32p = C.POINTER(C.c_float)
_u64p = C.POINTER(C.c_uint64)
_u32p = C.POINTER(C.c_uint32)
_u8p = C.POINTER(C.c_uint8)
_szp = C.POINTER(C.c_size_t)

CHIP_MAPPING = np.array([1618456172, 1309113062, 1826650030, 1724778362, 778887287, 2061946375, 2007919840,
                         125494990, 529027475, 838370585, 320833617, 422705285, 1368596360, 85537272, 139563807,
                         2021988657], np.uint32)
MASK = 0x7FFFFFFE


class MmState(C.Structure):
    _fields_ = [("omega", C.c_float), ("omega_mid", C.c_float), ("omega_limit", C.c_float),
                ("gain_omega", C.c_float), ("mu", C.c_float), ("gain_mu", C.c_float), ("last_sample", C.c_float),
                ("pad", C.c_uint32), ("look_ahead", C.c_uint64)]


class DecState(C.Structure):
    _fields_ = [("shift_reg", C.c_uint32), ("threshold", C.c_uint32), ("chip_count", C.c_uint32),
                ("state", C.c_uint32), ("byte", C.c_int32), ("len", C.c_uint32), ("dlen", C.c_uint32),
                ("data", C.c_uint8 * 128)]


SIGNATURES = {
    "orc_zb_dc_block": (None, [C.c_float, _f32p, _f32p, C.c_size_t, _f32p]),
    "orc_zb_mm_new": (None, [C.POINTER(MmState)] + [C.c_float] * 5),
    "orc_zb_mm_work": (C.c_int, [C.POINTER(MmState), _f32p, C.c_size_t, _f32p, C.c_size_t, _szp, _szp]),
    "orc_zb_decoder_new": (None, [C.POINTER(DecState), C.c_uint32]),
    "orc_zb_decoder_work": (C.c_size_t, [C.POINTER(DecState), _f32p, C.c_size_t, C.c_uint64, _u64p, _u32p, _u8p,
                                         C.c_size_t]),
    "orc_zb_calc_crc": (C.c_uint32, [_u8p, C.c_size_t]),
}


def lib() -> C.CDLL:
    return load_oracle("zigbee_oracle", SIGNATURES)


def _f(a):
    return np.ascontiguousarray(a, np.float32)


class DcBlock:
    def __init__(self, alpha):
        self.alpha = float(np.float32(alpha))
        self.iir = C.c_float(0.0)

    def work(self, x) -> np.ndarray:
        x = _f(x)
        y = np.empty_like(x)
        lib().orc_zb_dc_block(self.alpha, C.byref(self.iir), x.ctypes.data_as(_f32p), x.size, y.ctypes.data_as(_f32p))
        return y


class Mm:
    def __init__(self, omega, gain_omega, mu, gain_mu, omega_relative_limit):
        self.s = MmState()
        lib().orc_zb_mm_new(C.byref(self.s), *(float(np.float32(v)) for v in
                                               (omega, gain_omega, mu, gain_mu, omega_relative_limit)))

    @property
    def look_ahead(self) -> int:
        return int(self.s.look_ahead)

    def work(self, x, n_out):
        """One work() call -> (consumed, outputs, err); err = 1 for a step that would move past the slice."""
        x = _f(x)
        o = np.zeros(max(1, n_out), np.float32)
        c, p = C.c_size_t(0), C.c_size_t(0)
        err = lib().orc_zb_mm_work(C.byref(self.s), x.ctypes.data_as(_f32p), x.size, o.ctypes.data_as(_f32p), n_out,
                                   C.byref(c), C.byref(p))
        return c.value, o[:p.value].copy(), err


class Decoder:
    def __init__(self, threshold):
        self.s = DecState()
        lib().orc_zb_decoder_new(C.byref(self.s), int(threshold))
        self.pos = 0

    def work(self, x):
        """One work() call (consumes everything) -> [(index, bytes)] of the frames it posts."""
        x = _f(x)
        cap = x.size // 192 + 2
        idx, lens = np.zeros(cap, np.uint64), np.zeros(cap, np.uint32)
        by = np.zeros((cap, 128), np.uint8)
        nf = lib().orc_zb_decoder_work(C.byref(self.s), x.ctypes.data_as(_f32p), x.size, self.pos,
                                       idx.ctypes.data_as(_u64p), lens.ctypes.data_as(_u32p),
                                       by.ctypes.data_as(_u8p), cap)
        assert nf <= cap
        self.pos += x.size
        return [(int(idx[k]), bytes(by[k, :lens[k]].tolist())) for k in range(nf)]


def calc_crc(data) -> int:
    b = np.frombuffer(bytes(data), np.uint8).copy() if len(data) else np.zeros(1, np.uint8)
    return int(lib().orc_zb_calc_crc(b.ctypes.data_as(_u8p), len(data)))


def crc_ok(data) -> bool:
    """What the Mac accepts (mac.rs:98): calc_crc == 0 and more than two bytes."""
    return calc_crc(data) == 0 and len(data) > 2


def mm_replay(params, x, cuts=None, n_out=None):
    """ClockRecoveryMm over a whole stream, called on growing slices: before call k the input holds cuts[k] items
    (the last call sees everything); each call may write n_out outputs (unbounded if None).  Returns (outputs,
    consumed, err) with err the call index that flagged an out-of-slice step, or None."""
    x = _f(x)
    m = Mm(*params)
    cuts = [c for c in (cuts or []) if c < x.size] + [x.size]
    pos, outs = 0, []
    for k, cut in enumerate(cuts):
        cut = max(cut, pos)
        while True:
            cap = (cut - pos + 8) if n_out is None else n_out
            c, o, err = m.work(x[pos:cut], cap)
            pos += c
            outs.append(o)
            if err:
                return np.concatenate(outs), pos, k
            if n_out is None or o.size < n_out or c == 0:
                break
    return np.concatenate(outs), pos, None


def decode_replay(threshold, x, cuts=None):
    """The Decoder over a whole stream in calls ending at cuts -> [(index, bytes)]."""
    x = _f(x)
    d = Decoder(threshold)
    edges = [0] + sorted(c for c in set(cuts or []) if 0 < c < x.size) + [x.size]
    out = []
    for a, b in zip(edges[:-1], edges[1:]):
        out += d.work(x[a:b])
    return out


# ---- independent numpy float32 transcription -------------------------------------------------------------------
def np_dc_block(alpha, x, iir=0.0):
    f32 = np.float32
    a = f32(alpha)
    oma = f32(1.0) - a
    s = f32(iir)
    y = np.empty(len(x), np.float32)
    with np.errstate(all="ignore"):
        for k, v in enumerate(_f(x)):
            s = f32(f32(oma * s) + f32(a * v))
            y[k] = f32(v - s)
    return y, s


def np_mm(params, x, n_out):
    """One call from the initial state -> (consumed, outputs, err)."""
    f32 = np.float32
    omega, gain_omega, mu, gain_mu, rel = (f32(v) for v in params)
    with np.errstate(all="ignore"):
        lim = f32(omega * rel)
        laf = np.ceil(f32(f32(omega + lim) + gain_mu))
        la = 0 if not laf > 0 else int(laf)
        mid, last = omega, f32(0.0)
        x = _f(x)
        ii, out = 0, []
        while ii + la < x.size and len(out) < n_out:
            o = f32(x[ii] + f32(mu * f32(x[ii + 1] - x[ii])))
            sl = f32(1.0) if last > 0 else f32(-1.0)
            so = f32(1.0) if o > 0 else f32(-1.0)
            mm = f32(f32(sl * o) - f32(so * last))
            om = f32(omega + f32(gain_omega * mm))
            d = f32(om - mid)
            if d < -lim:
                d = -lim
            if d > lim:
                d = lim
            om = f32(mid + d)
            nmu = f32(mu + f32(om + f32(gain_mu * mm)))
            fl = np.floor(nmu)
            step = int(fl) if fl > 0 and np.isfinite(fl) else (0 if not fl > 0 else 1 << 64)
            if step > x.size - ii:
                return ii, np.array(out, np.float32), 1
            out.append(o)
            last, omega, mu = o, om, f32(nmu - fl)
            ii += step
    return ii, np.array(out, np.float32), 0


def np_decode(threshold, x):
    """The Decoder from the initial state over one slice -> [(index, bytes)]."""
    chips = (_f(x) > 0).astype(np.uint8)
    cm = [int(c) & MASK for c in CHIP_MAPPING]

    def dist(sr, i):
        return bin((sr & MASK) ^ cm[i]).count("1")

    sr, cc, state, byte, length, data, out = 0, 0, "search", None, 0, [], []
    for k, b in enumerate(chips):
        sr = ((sr << 1) | int(b)) & 0xFFFFFFFF
        cc = (cc + 1) % 32
        if state == "search":
            if dist(sr, 0) < threshold:
                state, cc = "pre", 0
            continue
        if cc != 0:
            continue
        if state == "pre":
            if dist(sr, 7) < threshold:
                state = "sfd"
            elif not dist(sr, 0) < threshold:
                state = "search"
            continue
        if state == "sfd":
            state, byte = ("hdr", None) if dist(sr, 10) < threshold else ("search", None)
            continue
        ds = [dist(sr, i) for i in range(16)]
        i = int(np.argmin(ds))
        if not ds[i] < threshold:
            state = "search"
            continue
        if byte is None:
            byte = i
            continue
        v = (i << 4) | byte
        byte = None
        if state == "hdr":
            if v < 128:
                state, length, data = "dec", v, []
            else:
                state = "search"
        else:
            data.append(v)
            if len(data) == length:
                out.append((k, bytes(data)))
                state = "search"
    return out


_TABLE = None


def crc16_table(data) -> int:
    """Table-driven reflected CRC-16 (polynomial 0x1021 reflected = 0x8408, initial value 0)."""
    global _TABLE
    if _TABLE is None:
        t = []
        for i in range(256):
            r = i
            for _ in range(8):
                r = (r >> 1) ^ 0x8408 if r & 1 else r >> 1
            t.append(r)
        _TABLE = t
    crc = 0
    for b in bytes(data):
        crc = (crc >> 8) ^ _TABLE[(crc ^ b) & 0xFF]
    return crc


# ---- the transmitter side (examples/zigbee/src/{mac,modulator,iq_delay}.rs) ---------------------------------------
def mac_frame(payload: bytes, seq: int = 0) -> bytes:
    """Mac's tx framing (mac.rs:193-220): preamble 00 00 00 a7, length, 9 header bytes, payload, FCS (little endian)
    over length-excluded header + payload.  The receiver's decoder posts frame[5:] (what follows the length byte)."""
    hdr = bytes([0x41, 0x88, seq & 0xFF, 0xAA, 0x1A, 0xFF, 0xFF, 0x44, 0x33])   # FRAME_CONTROL, seq, PAN, dst, src
    body = hdr + bytes(payload)
    crc = calc_crc(body)
    body += bytes([crc & 0xFF, crc >> 8])
    return bytes([0, 0, 0, 0xA7, len(payload) + 11]) + body


def chips_of(frame: bytes) -> np.ndarray:
    """Each byte as two symbols, low nibble first, each symbol its 32 chips MSB first (bit 31 is sent first; the
    decoder's shift register then holds the sequence as is)."""
    out = []
    for b in frame:
        for nib in (b & 0xF, b >> 4):
            c = int(CHIP_MAPPING[nib])
            out.extend((c >> (31 - j)) & 1 for j in range(32))
    return np.array(out, np.uint8)
