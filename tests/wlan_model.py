"""A restatement of the WLAN receive direction for ideal timing (TEST INFRASTRUCTURE ONLY): what the reference's
FrameEqualizer, Decoder and ViterbiDecoder do to a burst once it is found, without synchronisation or channel
estimation.  Per burst it removes the cyclic prefixes, takes an f64 FFT of each symbol, demaps with
``Modulation::demap`` (lib.rs:177-218), deinterleaves, depunctures with ``Mcs::depuncture_pattern`` (lib.rs:223-230),
runs a hard-decision Viterbi decoder over the K = 7 code, descrambles from the 7 SERVICE bits, checks the SIGNAL
field's parity, rate and length, and checks the FCS.
"""
from __future__ import annotations

import zlib

import numpy as np

N_BPSC = (1, 1, 2, 2, 4, 4, 6, 6)
N_DBPS = (24, 36, 48, 72, 96, 144, 192, 216)
RATE = (0x0D, 0x0F, 0x05, 0x07, 0x09, 0x0B, 0x01, 0x03)
DEPUNCTURE = {0: (1, 1), 1: (1, 1, 1, 0, 0, 1), 2: (1, 1), 3: (1, 1, 1, 0, 0, 1), 4: (1, 1), 5: (1, 1, 1, 0, 0, 1),
              6: (1, 1, 1, 0), 7: (1, 1, 1, 0, 0, 1)}
DATA_SC = [c for c in range(6, 59) if c not in (11, 25, 32, 39, 53)]
SCALE = 64 * np.sqrt(1 / 52) * 0.6           # the transmitter's IFFT normalisation and Prefix's 0.6


def demap(x: np.ndarray, bpsc: int) -> np.ndarray:
    """Modulation::demap of an array of subcarriers -> bytes."""
    re, im = x.real, x.imag
    if bpsc == 1:
        return (re > 0).astype(np.uint8)
    if bpsc == 2:
        return (2 * (im > 0) + (re > 0)).astype(np.uint8)
    if bpsc == 4:
        lv = 0.6324555320336759
        return ((re > 0) | ((abs(re) < lv) << 1) | ((im > 0) << 2) | ((abs(im) < lv) << 3)).astype(np.uint8)
    lv = 0.1543033499620919
    return ((re > 0) | ((abs(re) < 4 * lv) << 1) | (((abs(re) < 6 * lv) & (abs(re) > 2 * lv)) << 2) | ((im > 0) << 3)
            | ((abs(im) < 4 * lv) << 4) | (((abs(im) < 6 * lv) & (abs(im) > 2 * lv)) << 5)).astype(np.uint8)


_NS = np.arange(64)
_OUT = np.array([[[bin((ns | (m << 6)) & mask).count("1") % 2 for mask in (0o155, 0o117)] for m in (0, 1)]
                 for ns in range(64)])                                       # [next state][msb] -> 2 coded bits


def viterbi(coded: np.ndarray) -> np.ndarray:
    """Hard-decision Viterbi of the rate-1/2 K = 7 code; coded holds 0, 1 or -1 (erased).  Ends in state 0."""
    n = coded.size // 2
    pm = np.full(64, 1 << 30)
    pm[0] = 0
    surv = np.zeros((n, 64), np.uint8)
    for t in range(n):
        c = coded[2 * t:2 * t + 2]
        bm = np.zeros((64, 2), np.int64)
        for j in range(2):
            if c[j] >= 0:
                bm += _OUT[:, :, j] != c[j]
        prev = np.stack([(_NS >> 1), (_NS >> 1) | 32], axis=1)
        cand = pm[prev] + bm
        choice = np.argmin(cand, axis=1)
        surv[t] = choice
        pm = cand[_NS, choice]
    bits = np.zeros(n, np.uint8)
    s = 0
    for t in range(n - 1, -1, -1):
        bits[t] = s & 1
        s = (s >> 1) | (int(surv[t, s]) << 5)
    return bits


def _deinterleave(bits: np.ndarray, bpsc: int) -> np.ndarray:
    cbps = 48 * bpsc
    s = max(bpsc // 2, 1)
    first = np.array([s * (j // s) + (j + 16 * j // cbps) % s for j in range(cbps)])
    second = np.array([16 * i - (cbps - 1) * (16 * i // cbps) for i in range(cbps)])
    out = np.empty_like(bits)
    for i in range(bits.size // cbps):
        out[i * cbps + second[first]] = bits[i * cbps:(i + 1) * cbps]
    return out


def _symbols(x: np.ndarray, d0: int, n: int) -> np.ndarray:
    """Subcarriers 0..63 of n symbols from sample d0, in the Mapper's order."""
    body = np.stack([x[d0 + 80 * k + 16:d0 + 80 * k + 80] for k in range(n)]).astype(np.complex128)
    return np.roll(np.fft.fft(body, axis=1) / SCALE, 32, axis=1)


def _bits(sc: np.ndarray, bpsc: int) -> np.ndarray:
    b = demap(sc[:, DATA_SC].reshape(-1), bpsc)
    return ((b[:, None] >> np.arange(bpsc)) & 1).astype(np.int8).reshape(-1)


def decode_burst(x: np.ndarray, start: int, pad_front: int):
    """The payload of the burst at sample ``start``, and its MCS -> (payload bytes, mcs), or None if the SIGNAL or
    the FCS does not check."""
    d0 = start + pad_front + 320
    sig = _deinterleave(_bits(_symbols(x, d0, 1), 1), 1)
    b = viterbi(sig.astype(np.int8))
    if b[17] != b[:17].sum() % 2 or b[4] != 0:
        return None
    rate = int(b[0]) << 3 | int(b[1]) << 2 | int(b[2]) << 1 | int(b[3])
    if rate not in RATE:
        return None
    mcs = RATE.index(rate)
    length = sum(int(b[5 + i]) << i for i in range(12))
    n_sym = -(-(16 + 8 * length + 6) // N_DBPS[mcs])
    inter = _deinterleave(_bits(_symbols(x, d0 + 80, n_sym), N_BPSC[mcs]), N_BPSC[mcs])
    pat = DEPUNCTURE[mcs]
    nd = n_sym * N_DBPS[mcs]
    coded = np.full(2 * nd, -1, np.int8)
    keep = np.array([pat[i % len(pat)] for i in range(2 * nd)], bool)
    coded[keep] = inter[:keep.sum()]
    scr = viterbi(coded)
    st = 0
    for i in range(7):                       # SERVICE bits 0..6 are zeros: the scrambled ones are the sequence
        st = (st << 1) | int(scr[i])
    data = np.zeros(nd, np.uint8)
    for i in range(7, nd):
        fb = ((st >> 6) ^ (st >> 3)) & 1
        data[i] = scr[i] ^ fb
        st = ((st << 1) & 0x7E) | fb
    psdu = np.packbits(data[16:16 + 8 * length].reshape(-1, 8)[:, ::-1], axis=1).reshape(-1).tobytes()
    if len(psdu) < 28 or zlib.crc32(psdu[:-4]) != int.from_bytes(psdu[-4:], "little"):
        return None
    return psdu[24:-4], mcs
