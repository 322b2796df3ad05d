"""CPU oracle of the LoRa transmitter (TEST INFRASTRUCTURE ONLY).

ctypes front-end to ``tests/lora_oracle.c`` (one reference call at a time, compiled by ``native.load_oracle`` on first
use): ``encode``, ``chirp``, ``modulate`` (samples with libm cosf / sinf, and the phase sums) and ``sample_count``.
The ``py_*`` functions are an independent transcription in Python integers and numpy f32, for cross-checking the C
file.  The reference's LoRa code has no tests, so this parity is unpinned.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from native import load_oracle

_u8p, _u16p, _f32p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint16), C.POINTER(C.c_float)
_sz = C.c_size_t

SIGNATURES = {
    "orc_lora_whitening": (None, [_u8p]),
    "orc_lora_encode": (C.c_long, [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _u8p, _sz, _u16p, _sz]),
    "orc_lora_chirp": (None, [_sz, C.c_int, _sz, C.c_int, _sz, C.c_int, _f32p]),
    "orc_lora_modulate": (_sz, [C.c_int, _sz, _u16p, _sz, _sz, _u16p, _sz, _f32p, _f32p, _sz]),
    "orc_lora_sample_count": (C.c_longlong, [C.c_int, _sz, C.c_int, _sz, C.c_int, C.c_int, _sz, _sz, C.c_int]),
}


def lib() -> C.CDLL:
    return load_oracle("lora_oracle", SIGNATURES)


def whitening() -> np.ndarray:
    out = np.zeros(255, np.uint8)
    lib().orc_lora_whitening(out.ctypes.data_as(_u8p))
    return out


def encode(payload, sf, cr, has_crc, ldro, implicit):
    """Encoder::encode -> u16 symbols, or None where the reference panics."""
    p = np.ascontiguousarray(np.frombuffer(bytes(payload), np.uint8)) if len(payload) else np.zeros(1, np.uint8)
    out = np.zeros(4096, np.uint16)
    n = lib().orc_lora_encode(sf, cr, int(has_crc), int(ldro), int(implicit), p.ctypes.data_as(_u8p), len(payload),
                              out.ctypes.data_as(_u16p), out.size)
    return None if n < 0 else out[:n].copy()


def chirp(id, sf, os, upchirp=True, n_samples=None, offset_id=False) -> np.ndarray:
    n = (1 << sf) * os if n_samples is None else n_samples
    out = np.zeros(max(n, 1), np.float32)
    lib().orc_lora_chirp(id, sf, os, int(upchirp), n, int(offset_id), out.ctypes.data_as(_f32p))
    return out[:n]


def frame_len(sf, os, preamble_len, pad, n_sym) -> int:
    N = (1 << sf) * os
    return 2 * pad + (preamble_len + 4 + (2 if sf < 7 else 0)) * N + N // 4 - os + n_sym * N


def modulate(symbols, sf, os, sync, preamble_len, pad):
    """Modulator::modulate -> (Complex32 samples, f32 phase sums)."""
    sym = np.ascontiguousarray(symbols, np.uint16)
    n = frame_len(sf, os, preamble_len, pad, sym.size)
    out, ph = np.zeros(n, np.complex64), np.zeros(n, np.float32)
    sw = np.array(sync, np.uint16)
    got = lib().orc_lora_modulate(sf, os, sw.ctypes.data_as(_u16p), preamble_len, pad,
                                  (sym if sym.size else np.zeros(1, np.uint16)).ctypes.data_as(_u16p), sym.size,
                                  out.view(np.float32).ctypes.data_as(_f32p), ph.ctypes.data_as(_f32p), n)
    assert got == n
    return out, ph


def sample_count(sf, preamble_len, explicit_header, payload_len, has_crc, cr, os, pad, ldro):
    """utils::sample_count, or None where its usize arithmetic underflows."""
    v = lib().orc_lora_sample_count(sf, preamble_len, int(explicit_header), payload_len, int(has_crc), cr, os, pad,
                                    int(ldro))
    return None if v < 0 else int(v)


# ---- independent transcription -------------------------------------------------------------------------------------
def py_whitening() -> list:
    out, s = [], 0xFF
    for _ in range(255):
        out.append(s)
        s = ((s << 1) | (bin(s & 0xB8).count("1") & 1)) & 0xFF
    return out


_WH = py_whitening()


def _int2bool(v, n):
    return [bool((v >> (n - 1 - i)) & 1) for i in range(n)]


def _bool2int(b):
    return sum(int(x) << (len(b) - 1 - i) for i, x in enumerate(b))


def py_encode(payload, sf, cr, has_crc, ldro, implicit):
    payload = list(bytes(payload))
    L = len(payload)
    if L > 255 or (has_crc and L < 2):
        return None
    frame = []
    for i, b in enumerate(payload):
        frame += [(b ^ _WH[i]) & 0x0F, (b ^ _WH[i]) >> 4]
    if not implicit:
        o = [L >> 4, L & 0x0F, (cr << 1) | int(has_crc)]
        bit = lambda x, k: (x >> k) & 1  # noqa: E731
        c4 = bit(o[0], 3) ^ bit(o[0], 2) ^ bit(o[0], 1) ^ bit(o[0], 0)
        c3 = bit(o[0], 3) ^ bit(o[1], 3) ^ bit(o[1], 2) ^ bit(o[1], 1) ^ bit(o[2], 0)
        c2 = bit(o[0], 2) ^ bit(o[1], 3) ^ bit(o[1], 0) ^ bit(o[2], 3) ^ bit(o[2], 1)
        c1 = bit(o[0], 1) ^ bit(o[1], 2) ^ bit(o[1], 0) ^ bit(o[2], 2) ^ bit(o[2], 1) ^ bit(o[2], 0)
        c0 = bit(o[0], 0) ^ bit(o[1], 1) ^ bit(o[2], 3) ^ bit(o[2], 2) ^ bit(o[2], 1) ^ bit(o[2], 0)
        frame = o + [c4, c3 << 3 | c2 << 2 | c1 << 1 | c0] + frame
    if has_crc:
        crc = 0
        for b in payload[:L - 2]:
            for _ in range(8):
                crc = ((crc << 1) ^ 0x1021) if ((crc & 0x8000) >> 8) ^ (b & 0x80) else (crc << 1)
                crc &= 0xFFFF
                b = (b << 1) & 0xFFFF
        crc ^= payload[L - 1] ^ (payload[L - 2] << 8)
        frame += [crc & 0xF, (crc >> 4) & 0xF, (crc >> 8) & 0xF, crc >> 12]
    cws = []
    for i, nib in enumerate(frame):
        cr_app = 4 if i < sf - (0 if sf < 7 else 2) else cr
        d = _int2bool(nib, 4)
        if cr_app != 1:
            p0, p1, p2, p3 = d[3] ^ d[2] ^ d[1], d[2] ^ d[1] ^ d[0], d[3] ^ d[2] ^ d[0], d[3] ^ d[1] ^ d[0]
            cws.append(_bool2int([d[3], d[2], d[1], d[0], p0, p1, p2, p3]) >> (4 - cr_app))
        else:
            cws.append(_bool2int([d[3], d[2], d[1], d[0], d[0] ^ d[1] ^ d[2] ^ d[3]]))
    out, cnt = [], 0
    while True:
        if sf >= 7:
            cw_len, use_ldro = 4 + (4 if cnt < sf - 2 else cr), cnt < sf - 2 or ldro
        else:
            cw_len, use_ldro = 4 + (4 if cnt < sf else cr), cnt >= sf and ldro
        sf_app = max(sf - 2, 0) if use_ldro else sf
        curr, cws = cws[:sf_app], cws[sf_app:]
        cw_bin = [_int2bool(x, cw_len) for x in curr + [0] * (sf_app - len(curr))]
        cnt += sf_app
        for i in range(cw_len):
            row = [False] * sf
            for j in range(sf_app):
                row[j] = cw_bin[(i - j - 1) % sf_app][i]
            if use_ldro:
                row[sf_app] = sum(row) % 2 != 0
            out.append(_bool2int(row))
        if not cws:
            break
    res = []
    for v in out:
        g = v
        for j in range(1, sf):
            g ^= v >> j
        res.append((g + 1) % (1 << sf))
    return np.array(res, np.uint16)


_F32 = np.float32


def py_chirp(id, sf, os, upchirp=True, n_samples=None, offset_id=False) -> np.ndarray:
    n = 1 << sf
    ns = n * os if n_samples is None else n_samples
    t_ds = np.arange(ns, dtype=np.float64) / np.float64(n * os)
    p = (t_ds - 0.5).astype(np.float32) + _F32(_F32((id - 1) if offset_id else id) / _F32(n))
    p = np.where(p > _F32(0.5), p - _F32(1.0), np.where(p < _F32(-0.5), p + _F32(1.0), p)).astype(np.float32)
    k = _F32(_F32(_F32(1.0 if upchirp else -1.0) * _F32(_F32(1.0) / _F32(os))) * _F32(_F32(2.0) * _F32(np.pi)))
    return (p * k).astype(np.float32)


def py_increments(symbols, sf, os, sync, preamble_len, pad) -> np.ndarray:
    N = (1 << sf) * os
    parts = [np.zeros(pad, np.float32)]
    parts += [py_chirp(0, sf, os)] * preamble_len
    parts += [py_chirp(int(sync[0]), sf, os), py_chirp(int(sync[1]), sf, os)]
    parts += [py_chirp(0, sf, os, False)] * 2 + [py_chirp(0, sf, os, False, N // 4 - os)]
    parts += [py_chirp(0, sf, os)] * (2 if sf < 7 else 0)
    parts += [py_chirp(int(s), sf, os, True, None, True) for s in symbols]
    parts += [np.zeros(pad, np.float32)]
    return np.concatenate(parts).astype(np.float32)


def py_phase(symbols, sf, os, sync, preamble_len, pad) -> np.ndarray:
    """The phase sums of samples_from_phase_diff: np.add.accumulate in f32 adds in order from +0."""
    return np.add.accumulate(py_increments(symbols, sf, os, sync, preamble_len, pad), dtype=np.float32)


def f64_samples(phase) -> np.ndarray:
    """float32(cos / sin(float64(S))): the device's rule for the samples of the phases S."""
    s = np.asarray(phase, np.float64)
    out = np.empty(s.size, np.complex64)
    out.real, out.imag = np.cos(s).astype(np.float32), np.sin(s).astype(np.float32)
    return out


def ulp_diff(a, b) -> int:
    """The largest distance in f32 units in the last place over the parts of two Complex32 arrays."""
    x = np.ascontiguousarray(a, np.complex64).view(np.float32).view(np.int32).astype(np.int64)
    y = np.ascontiguousarray(b, np.complex64).view(np.float32).view(np.int32).astype(np.int64)
    x = np.where(x < 0, -(x & 0x7FFFFFFF), x)
    y = np.where(y < 0, -(y & 0x7FFFFFFF), y)
    return int(np.max(np.abs(x - y))) if x.size else 0
