"""CPU oracle of the ADS-B receiver's PreambleDetector -> Demodulator -> Decoder::check_crc (TEST INFRASTRUCTURE ONLY).

ctypes front-end to ``tests/adsb_oracle.c`` (one reference call at a time, compiled by ``native.load_oracle`` on
first use).  ``replay`` drives the three blocks over any sequence of detector calls, and ``np_detect`` /
``np_demod_bits`` are an independent numpy float32 transcription for cross-checking the C file.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from native import load_oracle

_f32p = C.POINTER(C.c_float)
_u64p = C.POINTER(C.c_uint64)
_u8p = C.POINTER(C.c_uint8)
PACKET_SAMPLES = 480
PREAMBLE_SAMPLES = 32

SIGNATURES = {
    "orc_adsb_detect": (C.c_size_t, [C.c_float, _f32p, C.c_size_t, _f32p, C.c_size_t, _f32p, C.c_size_t, C.c_size_t,
                                     _u64p, _f32p, C.c_size_t, C.POINTER(C.c_size_t)]),
    "orc_adsb_demod_bits": (None, [_f32p, C.c_size_t, _u8p]),
    "orc_adsb_check_crc": (C.c_int, [_u8p, C.c_size_t]),
}


def lib() -> C.CDLL:
    return load_oracle("adsb_oracle", SIGNATURES)


def _f(a):
    return np.ascontiguousarray(a, np.float32)


def detect(threshold, samples, nf, corr, len_out=None):
    """One PreambleDetector::work call -> (num_read, [(index, max_corr), ...]) with indices relative to the slices."""
    s, n, c = _f(samples), _f(nf), _f(corr)
    lo = min(s.size, n.size, c.size) if len_out is None else int(len_out)
    cap = max(1, lo // 31 + 2)
    idx, val, nt = np.zeros(cap, np.uint64), np.zeros(cap, np.float32), C.c_size_t(0)
    nr = lib().orc_adsb_detect(float(np.float32(threshold)), s.ctypes.data_as(_f32p), s.size,
                               n.ctypes.data_as(_f32p), n.size, c.ctypes.data_as(_f32p), c.size, lo,
                               idx.ctypes.data_as(_u64p), val.ctypes.data_as(_f32p), cap, C.byref(nt))
    assert nt.value <= cap
    return nr, list(zip(idx[:nt.value].tolist(), val[:nt.value].tolist()))


def demod_bits(samples, index) -> np.ndarray:
    s = _f(samples)
    assert index + PACKET_SAMPLES < s.size
    bits = np.zeros(112, np.uint8)
    lib().orc_adsb_demod_bits(s.ctypes.data_as(_f32p), int(index), bits.ctypes.data_as(_u8p))
    return bits


def check_crc(bits) -> bool:
    b = np.ascontiguousarray(bits, np.uint8)
    r = lib().orc_adsb_check_crc(b.ctypes.data_as(_u8p), b.size)
    assert r >= 0
    return bool(r)


def bits_to_bytes(bits) -> bytes:
    return bytes(np.packbits(np.asarray(bits, np.uint8)).tolist())


def hex_to_bits(h: str) -> np.ndarray:
    return np.unpackbits(np.frombuffer(bytes.fromhex(h), np.uint8))


def replay(threshold, samples, nf, corr, cuts=None):
    """The three blocks over a whole stream, the detector called on growing slices: before call k every input holds
    ``cuts[k]`` items (increasing; the last call sees everything, and the inputs are finished then).  The demodulator
    runs after every detector call on what the detector has produced so far (demodulator.rs:57-110).
    Returns (tags [(global index, max_corr)], packets [(index, max_corr, crc_passed, bytes)], D)."""
    s, n, c = _f(samples), _f(nf), _f(corr)
    total = min(s.size, n.size, c.size)
    cuts = [x for x in (cuts or []) if x < total] + [total]
    pos, tags, packets = 0, [], []
    dstart, next_tag = 0, 0                          # demodulator: consumed items, first tag not yet handled
    for avail in cuts:
        avail = max(avail, pos)
        nr, t = detect(threshold, s[pos:avail], n[pos:avail], c[pos:avail])
        tags += [(pos + i, v) for i, v in t]
        pos += nr
        buf_len = pos - dstart                       # the demodulator's slice: produced, not consumed
        while next_tag < len(tags) and tags[next_tag][0] - dstart + PACKET_SAMPLES < buf_len:
            g, v = tags[next_tag]
            bits = demod_bits(s[:pos], g)
            packets.append((g, v, check_crc(bits), bits_to_bytes(bits)))
            next_tag += 1
        if buf_len >= PACKET_SAMPLES:
            dstart += buf_len - PACKET_SAMPLES
    return tags, packets, pos


# ---- independent numpy float32 transcription -------------------------------------------------------------------
def np_detect(threshold, samples, nf, corr):
    f32 = np.float32
    s, n, c = _f(samples), _f(nf), _f(corr)
    limit = max(0, min(s.size, n.size, c.size) - 64)
    thr = f32(threshold)
    with np.errstate(all="ignore"):
        ratio = c / n
        trig = c > thr * n
    pos, tags = 0, []
    while pos < limit:
        if not trig[pos]:
            pos += 1
            continue
        w = ratio[pos:pos + 32]
        best, idx = w[0], 0
        for k in range(1, 32):
            if w[k] > best:
                best, idx = w[k], k
        idx += pos
        with np.errstate(all="ignore"):
            p = s[idx:idx + 32].reshape(16, 2)
            pw = (f32(-0.0) + p[:, 0]) + p[:, 1]
            hi, lo = pw[[0, 2, 7, 9]], np.delete(pw, [0, 2, 7, 9])
            if not np.all(np.isnan(hi)):
                mn, mx = np.nanmin(hi), np.nanmax(hi)
            else:
                mn = mx = f32(np.nan)
            ml = np.nanmax(lo) if not np.all(np.isnan(lo)) else f32(np.nan)
            if mn > f32(0.1) * mx and ml < mx:
                tags.append((idx, float(best)))
        pos += 31
    return pos, tags


def np_demod_bits(samples, index):
    s = _f(samples)
    x = s[index + 32:index + 32 + 448].reshape(112, 4)
    f32 = np.float32
    with np.errstate(all="ignore"):
        c0 = (((f32(0) + x[:, 0] * f32(-1)) + x[:, 1] * f32(-1)) + x[:, 2]) + x[:, 3]
        c1 = (((f32(0) + x[:, 0]) + x[:, 1]) + x[:, 2] * f32(-1)) + x[:, 3] * f32(-1)
    return np.where(c0 > c1, 0, 1).astype(np.uint8)


def crc24_table(bits) -> int:
    """Table-driven CRC-24 (generator 0xFFF409) of the first 88 bits, XOR the last 24: 0 iff the frame checks."""
    table = _table()
    data = bits_to_bytes(bits)
    crc = 0
    for b in data[:11]:
        crc = ((crc << 8) & 0xFFFFFF) ^ table[((crc >> 16) ^ b) & 0xFF]
    return crc ^ int.from_bytes(data[11:14], "big")


_TABLE = None


def _table():
    global _TABLE
    if _TABLE is None:
        t = []
        for i in range(256):
            r = i << 16
            for _ in range(8):
                r = ((r << 1) ^ 0xFFF409) if r & 0x800000 else (r << 1)
            t.append(r & 0xFFFFFF)
        _TABLE = t
    return _TABLE
