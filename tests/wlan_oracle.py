"""CPU oracle of the WLAN transmitter (TEST INFRASTRUCTURE ONLY).

ctypes front-end to ``tests/wlan_oracle.c`` (compiled by ``native.load_oracle`` on first use): ``Tx`` is a Mac +
Encoder with the reference's persistent state (sequence number, scrambler seed, the never-cleared bit buffer), ``map``
is Mapper::map, ``prefix`` the Prefix block's f32 operations on caller-given inverse-FFT outputs and ``ifft_f64`` an
f64 DFT of that transform.  The ``Py*`` / ``py_*`` names are an independent transcription in Python integers and numpy
f32, for cross-checking the C file.  Apart from the tables (tests/golden/wlan_tables.json) this parity is unpinned.
"""
from __future__ import annotations

import ctypes as C
import json
import os
import zlib

import numpy as np

from native import load_oracle

_u8p, _f32p, _f64p, _i32p = (C.POINTER(C.c_uint8), C.POINTER(C.c_float), C.POINTER(C.c_double),
                             C.POINTER(C.c_int32))
_sz, _szp = C.c_size_t, C.POINTER(C.c_size_t)

SIGNATURES = {
    "orc_wlan_mseq": (None, [_u8p]),
    "orc_wlan_crc32": (C.c_uint32, [_u8p, _sz]),
    "orc_wlan_new": (C.c_void_p, [_u8p, _u8p, _u8p]),
    "orc_wlan_free": (None, [C.c_void_p]),
    "orc_wlan_set_state": (None, [C.c_void_p, C.c_uint, C.c_uint]),
    "orc_wlan_mac": (C.c_long, [C.c_void_p, _u8p, _sz, _u8p]),
    "orc_wlan_frame_param": (None, [C.c_int, _sz, _szp, _szp, _szp]),
    "orc_wlan_encode": (C.c_long, [C.c_void_p, _u8p, _sz, C.c_int, _u8p, _sz]),
    "orc_wlan_signal_pattern": (None, [_i32p]),
    "orc_wlan_signal": (None, [C.c_int, _sz, _u8p]),
    "orc_wlan_constellation": (None, [C.c_int, _f32p]),
    "orc_wlan_map": (None, [_u8p, C.c_int, _sz, _f32p]),
    "orc_wlan_sync_words": (None, [_f32p]),
    "orc_wlan_ifft_f64": (None, [_f32p, _f64p]),
    "orc_wlan_prefix": (C.c_long, [_f32p, _sz, _sz, _sz, _f32p, _sz]),
}

N_BPSC = (1, 1, 2, 2, 4, 4, 6, 6)
N_DBPS = (24, 36, 48, 72, 96, 144, 192, 216)
RATE = (0x0D, 0x0F, 0x05, 0x07, 0x09, 0x0B, 0x01, 0x03)
SRC, DST, BSS = bytes([0x42] * 6), bytes([0x23] * 6), bytes([0xFF] * 6)
_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "wlan_tables.json")


def lib() -> C.CDLL:
    return load_oracle("wlan_oracle", SIGNATURES)


def golden() -> dict:
    with open(_GOLDEN) as f:
        return json.load(f)


def _u8(b) -> np.ndarray:
    return np.ascontiguousarray(np.frombuffer(bytes(b), np.uint8)) if len(b) else np.zeros(1, np.uint8)


def mseq() -> np.ndarray:
    out = np.zeros(127, np.uint8)
    lib().orc_wlan_mseq(out.ctypes.data_as(_u8p))
    return out


def crc32(data) -> int:
    return lib().orc_wlan_crc32(_u8(data).ctypes.data_as(_u8p), len(data))


def frame_param(mcs, psdu):
    v = [C.c_size_t(0) for _ in range(3)]
    lib().orc_wlan_frame_param(int(mcs), int(psdu), *[C.byref(x) for x in v])
    return tuple(x.value for x in v)               # n_symbols, n_data_bits, n_pad


def signal_pattern() -> np.ndarray:
    out = np.zeros(48, np.int32)
    lib().orc_wlan_signal_pattern(out.ctypes.data_as(_i32p))
    return out


def signal(mcs, psdu) -> np.ndarray:
    out = np.zeros(48, np.uint8)
    lib().orc_wlan_signal(int(mcs), int(psdu), out.ctypes.data_as(_u8p))
    return out


def constellation(bpsc) -> np.ndarray:
    out = np.zeros(2 << bpsc, np.float32)
    lib().orc_wlan_constellation(int(bpsc), out.ctypes.data_as(_f32p))
    return out.view(np.complex64)


def sync_words() -> np.ndarray:
    out = np.zeros(640, np.float32)
    lib().orc_wlan_sync_words(out.ctypes.data_as(_f32p))
    return out.view(np.complex64)


def map_symbol(sc, bpsc, index) -> np.ndarray:
    """Mapper::map of 48 subcarrier bytes -> 64 complex64."""
    out = np.zeros(128, np.float32)
    lib().orc_wlan_map(_u8(np.asarray(sc, np.uint8).tobytes()).ctypes.data_as(_u8p), int(bpsc), int(index),
                       out.ctypes.data_as(_f32p))
    return out.view(np.complex64)


def ifft_f64(x) -> np.ndarray:
    """The shifted inverse transform of one mapped symbol, times sqrt(1/52), as an f64 DFT -> complex128."""
    xi = np.ascontiguousarray(np.asarray(x, np.complex64)).view(np.float32)
    out = np.zeros(128, np.float64)
    lib().orc_wlan_ifft_f64(xi.ctypes.data_as(_f32p), out.ctypes.data_as(_f64p))
    return out.view(np.complex128)


def prefix(y, pad_front, pad_tail) -> np.ndarray:
    """Prefix of one frame from its transforms y (n_ofdm x 64 complex64)."""
    y = np.ascontiguousarray(np.asarray(y, np.complex64).reshape(-1, 64))
    n = y.shape[0]
    out = np.zeros(2 * (pad_front + 320 + 80 * n + max(pad_tail, 1)), np.float32)
    r = lib().orc_wlan_prefix(y.view(np.float32).ctypes.data_as(_f32p), n, pad_front, pad_tail,
                              out.ctypes.data_as(_f32p), out.size // 2)
    assert r == out.size // 2
    return out.view(np.complex64)


class Tx:
    """Mac + Encoder with the reference's state.  ``frame`` -> (psdu bytes, symbols (1 + n_sym) x 48 uint8 with the
    SIGNAL symbol first), or None where the Mac drops the payload."""

    def __init__(self, src=SRC, dst=DST, bss=BSS, seq=0, seed=1):
        self._h = lib().orc_wlan_new(_u8(src).ctypes.data_as(_u8p), _u8(dst).ctypes.data_as(_u8p),
                                     _u8(bss).ctypes.data_as(_u8p))
        lib().orc_wlan_set_state(self._h, seq, seed)

    def __del__(self):
        if getattr(self, "_h", None):
            lib().orc_wlan_free(self._h)

    def frame(self, payload, mcs):
        psdu = np.zeros(1528, np.uint8)
        n = lib().orc_wlan_mac(self._h, _u8(payload).ctypes.data_as(_u8p), len(payload), psdu.ctypes.data_as(_u8p))
        if n < 0:
            return None
        psdu = psdu[:n].copy()
        ns = frame_param(mcs, n)[0]
        sym = np.zeros((1 + ns, 48), np.uint8)
        assert lib().orc_wlan_encode(self._h, psdu.ctypes.data_as(_u8p), n, int(mcs),
                                     sym[1:].ctypes.data_as(_u8p), 48 * ns) == ns
        sym[0] = signal(mcs, n)
        return psdu, sym


def mapped(sym, mcs) -> np.ndarray:
    """The Mapper's output for one frame's symbols: (1 + n_sym) x 64 complex64 (SIGNAL BPSK at pilot index 0)."""
    return np.stack([map_symbol(s, 1 if i == 0 else N_BPSC[mcs], i) for i, s in enumerate(sym)])


def stream(frames, ifft, pad_front, pad_tail) -> np.ndarray:
    """The transmitter's samples for frames [(symbols, mcs)], the inverse FFT given as ifft(mapped (n x 64)) -> n x 64
    complex64."""
    return np.concatenate([prefix(ifft(mapped(s, m)), pad_front, pad_tail) for s, m in frames])


def frame_len(n_ofdm, pad_front, pad_tail) -> int:
    return pad_front + 320 + 80 * n_ofdm + max(pad_tail, 1)


# ---- independent transcription ------------------------------------------------------------------------------------
def py_mseq() -> list:
    s, out = 0x7F, []
    for _ in range(127):
        fb = ((s >> 6) ^ (s >> 3)) & 1
        out.append(fb)
        s = ((s << 1) & 0x7E) | fb
    return out


class PyTx:
    """mac.rs / encoder.rs / mapper.rs in Python integers."""
    MAX_BITS = (16 + 8 * 1528 + 6) * 2 + 288

    def __init__(self, src=SRC, dst=DST, bss=BSS, seq=0, seed=1):
        self.hdr = bytes([0x08, 0x00, 0, 0]) + bytes(src) + bytes(dst) + bytes(bss)
        self.seq, self.seed = seq, seed
        self.bits = [0] * self.MAX_BITS

    def frame(self, payload, mcs):
        if len(payload) > 1500:
            return None
        sn = (self.seq << 4) & 0xFFFF
        self.seq = (self.seq + 1) % 4096
        body = self.hdr + bytes([sn & 0xFF, sn >> 8]) + bytes(payload)
        psdu = body + zlib.crc32(body).to_bytes(4, "little")
        n = len(psdu)
        dbps, bpsc = N_DBPS[mcs], N_BPSC[mcs]
        cbps = 48 * bpsc
        n_sym = -(-(16 + 8 * n + 6) // dbps)
        nd = n_sym * dbps
        npad = nd - (16 + 8 * n + 6)
        for i, byte in enumerate(psdu):
            for b in range(8):
                self.bits[16 + 8 * i + b] = (byte >> b) & 1
        st = self.seed
        self.seed = self.seed + 1 if self.seed < 127 else 1
        scr = []
        for i in range(nd):
            fb = ((st >> 6) ^ (st >> 3)) & 1
            scr.append(fb ^ self.bits[i])
            st = ((st << 1) & 0x7E) | fb
        for i in range(nd - npad - 6, nd - npad):
            scr[i] = 0
        enc = _conv(scr)
        if mcs == 6:
            pun = [e for i, e in enumerate(enc) if i % 4 != 3]
        elif mcs & 1:
            pun = [e for i, e in enumerate(enc) if i % 6 not in (3, 4)]
        else:
            pun = enc
        s = max(bpsc // 2, 1)
        first = [s * (j // s) + (j + 16 * j // cbps) % s for j in range(cbps)]
        second = [16 * i - (cbps - 1) * (16 * i // cbps) for i in range(cbps)]
        inter = [pun[i * cbps + second[first[k]]] for i in range(n_sym) for k in range(cbps)]
        data = np.array([sum(inter[i * bpsc + k] << k for k in range(bpsc)) for i in range(48 * n_sym)], np.uint8)
        return np.frombuffer(psdu, np.uint8).copy(), np.vstack([py_signal(mcs, n), data.reshape(n_sym, 48)])


def _conv(bits) -> list:
    st, out = 0, []
    for b in bits:
        st = ((st << 1) & 0x7E) | b
        out += [bin(st & 0o155).count("1") % 2, bin(st & 0o117).count("1") % 2]
    return out


def py_signal(mcs, length) -> np.ndarray:
    r = RATE[mcs]
    sig = [(r >> (3 - i)) & 1 for i in range(4)] + [0] + [(length >> i) & 1 for i in range(12)]
    sig += [sum(sig) % 2] + [0] * 6
    enc = _conv(sig)
    out = np.zeros(48, np.uint8)
    for i in range(48):
        out[3 * (i % 16) + i // 16] = enc[i]
    return out


def py_constellation(bpsc) -> np.ndarray:
    f = np.float32
    if bpsc == 1:
        return np.array([-1, 1], np.complex64)
    if bpsc == 2:
        q = f(1 / np.sqrt(2))
        lv = [-q, q]
        return np.array([complex(lv[i & 1], lv[i >> 1]) for i in range(4)], np.complex64)
    lvl, amp = (f(0.31622776601683794), [-3, 3, -1, 1]) if bpsc == 4 else (f(0.1543033499620919),
                                                                             [-7, 7, -1, 1, -5, 5, -3, 3])
    h = bpsc // 2
    return np.array([complex(f(amp[i & ((1 << h) - 1)]) * lvl, f(amp[i >> h]) * lvl) for i in range(1 << bpsc)],
                    np.complex64)


def py_map(sc, bpsc, index) -> np.ndarray:
    pol = np.float32(1 - 2 * py_mseq()[index % 127])
    re, im = np.zeros(64, np.float32), np.zeros(64, np.float32)
    tab = py_constellation(bpsc)
    data = [c for c in range(6, 59) if c not in (11, 25, 32, 39, 53)]
    for d, c in enumerate(data):
        re[c], im[c] = tab[sc[d]].real, tab[sc[d]].imag
    for c in (11, 25, 39):
        re[c] = pol
    re[53], im[53] = -pol, np.float32(-0.0)
    return _cplx(re, im)


def _cplx(re, im) -> np.ndarray:
    out = np.empty(re.size, np.complex64)
    out.real, out.imag = re, im
    return out


def py_sync_words() -> np.ndarray:
    """The generation rule of tests/golden/wlan_tables.json's sync words, through numpy's f64 FFT."""
    short = {-24: 1, -20: -1, -16: 1, -12: -1, -8: -1, -4: 1, 4: -1, 8: -1, 12: 1, 16: 1, 20: 1, 24: 1}
    long_ = [1, 1, -1, -1, 1, 1, -1, 1, -1, 1, 1, 1, 1, 1, 1, -1, -1, 1, 1, -1, 1, -1, 1, 1, 1, 1, 0,
             1, -1, -1, 1, 1, -1, 1, -1, 1, -1, -1, -1, -1, -1, 1, 1, -1, -1, 1, -1, 1, -1, 1, 1, 1, 1]
    S, L = np.zeros(64, complex), np.zeros(64, complex)
    for k, v in short.items():
        S[k % 64] = np.sqrt(13 / 6) * v * (1 + 1j)
    for i, v in enumerate(long_):
        L[(i - 26) % 64] = v
    st = np.fft.ifft(S) * 64 * np.sqrt(1 / 52)
    lt = np.fft.ifft(L) * 64 * np.sqrt(1 / 52)
    sync = np.concatenate([st, st, st[:32], lt[32:], lt, lt])
    sync[160] = 0.5 * (lt[32] + st[0])
    return sync.astype(np.complex64)


def py_prefix(y, pad_front, pad_tail) -> np.ndarray:
    y = np.asarray(y, np.complex64).reshape(-1, 64)
    n = y.shape[0]
    tail = max(pad_tail, 1)
    re, im = np.zeros(pad_front + 320 + 80 * n + tail, np.float32), np.zeros(pad_front + 320 + 80 * n + tail,
                                                                             np.float32)
    sync = py_sync_words()
    o = pad_front + 320
    re[pad_front:o], im[pad_front:o] = sync.real, sync.imag
    for k in range(n):
        body = np.concatenate([y[k, 48:], y[k]])
        re[o + 80 * k:o + 80 * k + 80], im[o + 80 * k:o + 80 * k + 80] = body.real, body.imag
    h = np.float32(0.5)
    re[o], im[o] = h * (re[o] + sync.real[256]), h * (im[o] + sync.imag[256])
    for k in range(n):
        a, b = o + (k + 1) * 80, o + k * 80 + 16
        re[a], im[a] = h * (re[a] + re[b]), h * (im[a] + im[b])
    return _cplx(re * np.float32(0.6), im * np.float32(0.6))
