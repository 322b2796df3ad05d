"""The SSB transceiver's CPU side: the C oracle of its five closures (tests/ssb_oracle.c) against an independent numpy-f32
transcription, bit for bit, on random and special values under many call slicings; the phase increments and taps of
futuresdr_b200.ssb against an independent f32 / f64 evaluation; and the header constants the new blocks mirror.  The
reference has no SSB tests, so this parity is unpinned, like the Rotator's."""
import math
import os
import struct
import subprocess

import numpy as np
import pytest

import oracle as orc
import ssb_oracle as so
from futuresdr_b200 import _lib, ssb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bits(a) -> np.ndarray:
    """Raw bit patterns: equal arrays of floats compare equal here even where they hold NaN."""
    a = np.ascontiguousarray(a)
    return a.view({2: np.uint16, 4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def _nan_equal(a, b):
    """Bit for bit, except that any NaN equals any NaN (the payload of a NaN is not part of the closures' result)."""
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype.kind == "c":
        a, b = a.view(np.float32), b.view(np.float32)
    assert a.shape == b.shape
    if a.dtype.kind == "f":
        both = np.isnan(a) & np.isnan(b)
        return np.array_equal(_bits(a)[~both], _bits(b)[~both])
    return np.array_equal(a, b)


SPECIALS = np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45, 1e-40, -3e-39, np.finfo(np.float32).tiny,
                     np.finfo(np.float32).max, -np.finfo(np.float32).max, 1.0, -1.0], np.float32)


def signal(rng, n, specials=True) -> np.ndarray:
    """n complex64 samples over many magnitudes, with special values sprinkled in both parts."""
    p = (rng.standard_normal(2 * n) * 10.0 ** rng.integers(-20, 20, 2 * n)).astype(np.float32)
    if specials and n:
        k = rng.integers(0, 2 * n, min(2 * n, 64))
        p[k] = SPECIALS[rng.integers(0, SPECIALS.size, k.size)]
    return p.view(np.complex64)


def i16_edges() -> np.ndarray:
    """c32 samples whose parts, times 0.9 * 32767, land on and next to the i16 range ends and zero."""
    k = np.float32(0.9) * np.float32(32767.0)
    ends = []
    for v in (32767.0, 32768.0, -32767.0, -32768.0, -32769.0, 0.5, -0.5, 1.0, -1.0):
        x = np.float32(v) / k
        ends += [np.nextafter(np.nextafter(x, np.float32(-np.inf)), np.float32(-np.inf)),
                 np.nextafter(x, np.float32(-np.inf)), x, np.nextafter(x, np.float32(np.inf)),
                 np.nextafter(np.nextafter(x, np.float32(np.inf)), np.float32(np.inf))]
    p = np.concatenate([np.array(ends, np.float32), SPECIALS, np.float32([1e6, -1e6, 2.0, -2.0])])
    if p.size % 2:
        p = np.append(p, np.float32(0.25))
    return np.concatenate([p, p[::-1]]).view(np.complex64)


def cuts_for(n, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "whole":
        return []
    if kind == "ones":
        return list(range(1, min(n, 40)))
    if kind in ("7", "8", "9"):
        return list(range(int(kind), n, int(kind)))
    return np.cumsum(rng.integers(1, max(2, n // 5), 12)).tolist()


PHASES = [0.1, -2.5, 1e-4, 3.0, float(ssb.xlating_phase()), float(ssb.weaver_phase(48_000)),
          float(ssb.weaver_phase(8_000)), float(ssb.mixer_phase())]


@pytest.mark.parametrize("theta", PHASES)
def test_shift_is_from_polar(theta):
    assert np.array_equal(_bits(so.shift(theta)), _bits(np.array(so.py_shift(theta), np.float32)))


@pytest.mark.parametrize("op,param", [(so.ROTATE, 1.0), (so.ROTATE_SCALE, 0.0001), (so.WEAVER, 0.5)])
@pytest.mark.parametrize("kind", ["whole", "ones", "7", "8", "9", "ragged"])
def test_mixer_oracle_equals_transcription(op, param, kind):
    rng = np.random.default_rng(op * 10 + len(kind))
    n = 3000
    x = signal(rng, n)
    for theta in (PHASES[4], PHASES[5], -2.5):
        want, _ = so.py_mix(op, theta, param, x)
        got = so.Mixer(op, theta, param).run(x, cuts_for(n, kind, op))
        assert _nan_equal(got, want)


def test_mixer_oracle_carries_the_oscillator():
    """The oscillator continues across calls from where the last call left it, and is not renormalised: after 10^5
    steps |osc| has drifted from 1 as the plain f32 recurrence does."""
    x = np.ones(100_000, np.complex64)
    m = so.Mixer(so.ROTATE, 0.37)
    y = m.run(x, [1, 8, 4097, 50_000])
    want, osc = so.py_mix(so.ROTATE, 0.37, 1.0, x)
    assert _nan_equal(y, want)
    assert np.array_equal(m.osc, np.array(osc, np.float32))
    assert abs(abs(complex(*m.osc)) - 1.0) > 1e-7


def test_file_level_and_i16_oracle_equal_transcription():
    rng = np.random.default_rng(5)
    for x in (signal(rng, 5000), i16_edges(), signal(rng, 5000, specials=False) * np.float32(1e-4)):
        assert _nan_equal(so.file_level(x), so.py_file_level(x))
        assert np.array_equal(so.to_i16_iq(x), so.py_to_i16_iq(x))
    # Rust `as i16` at the edges, written out by hand: truncation toward zero, saturation, NaN -> 0
    got = so.to_i16_iq(np.array([complex(np.inf, -np.inf), complex(np.nan, -0.0)], np.complex64))
    assert got.tolist() == [32767, -32768, 0, 0]
    k = float(np.float32(np.float32(0.9) * np.float32(32767.0)))
    x = np.array([complex(-1.4 / k, 1.9 / k)], np.complex64)
    assert so.to_i16_iq(x).tolist() == [-1, 1]


def test_file_level_is_one_rounding_per_step():
    """v * 2.0 / 0.0001 rounds the product first: the division alone by 0.00005 differs on some samples."""
    x = signal(np.random.default_rng(9), 20_000, specials=False)
    f = x.view(np.float32)
    y = so.file_level(x).view(np.float32)
    assert np.array_equal(_bits(y), _bits((f * np.float32(2.0)) / np.float32(0.0001)))


# ---- ssb.py: phase increments and taps --------------------------------------------------------------------------
def _r32(v: float) -> float:
    return struct.unpack("f", struct.pack("f", v))[0]


def test_phase_increments_are_f32_left_to_right():
    """Each product and quotient of two f32 values, formed in f64 and rounded once to f32, is the f32 operation."""
    pi32, tau32 = _r32(math.pi), _r32(2 * math.pi)
    assert float(ssb.xlating_phase()) == _r32(_r32(_r32(-2.0 * pi32) * 51_500.0) / 256_000.0)
    for rate in (8_000, 16_000, 32_000, 44_100, 48_000):
        assert float(ssb.weaver_phase(rate)) == _r32(_r32(_r32(2.0 * pi32) * 1500.0) / float(rate))
    assert float(ssb.mixer_phase()) == _r32(_r32(tau32 * 53_000.0) / 256_000.0)
    # and they are the intended angles to within f32 rounding
    assert abs(float(ssb.xlating_phase()) + 2 * math.pi * 51_500 / 256_000) < 1e-6
    assert abs(float(ssb.weaver_phase(48_000)) - 2 * math.pi * 1500 / 48_000) < 1e-7
    assert abs(float(ssb.mixer_phase()) - 2 * math.pi * 53_000 / 256_000) < 1e-6


@pytest.mark.parametrize("audio_rate", [8_000, 48_000])
def test_taps_match_the_oracle_designs(audio_rate):
    lp = ssb.lowpass_taps(audio_rate)
    assert np.array_equal(lp, orc.kaiser_lowpass(3000.0 / audio_rate, 350.0 / audio_rate, 0.05))
    g = math.gcd(audio_rate, ssb.FILE_RATE)
    for L, M in ((ssb.FILE_RATE // g, audio_rate // g), (audio_rate // g, ssb.FILE_RATE // g)):
        from futuresdr_b200 import firdes
        assert np.array_equal(firdes.kaiser.multirate(L, M, 12, 0.0001), orc.kaiser_multirate(L, M, 12, 0.0001))
    h = ssb.hilbert_taps()
    assert h.size == 167 and np.all(h[1::2] == 0) and np.allclose(h, -h[::-1], rtol=1e-6, atol=0)


# ---- header mirror -----------------------------------------------------------------------------------------------
CONSTANTS = ["OP_DIV_C32", "OP_C32_TO_I16_IQ", "MIX_ROTATE_C32", "MIX_ROTATE_SCALE_C32", "MIX_WEAVER_F32"]


@pytest.fixture(scope="module")
def header(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("ssb_probe")
    src, exe = tmp / "probe.c", tmp / "probe"
    body = "\n    ".join(f'printf("{n} %lld\\n", (long long)(B2S_{n}));' for n in CONSTANTS)
    src.write_text(f'#include <stdio.h>\n#include "b200sdr.h"\nint main(void) {{\n    {body}\n    return 0;\n}}\n')
    r = subprocess.run(["/usr/bin/gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    return {k: int(v) for k, v in (line.split() for line in out.splitlines())}


@pytest.mark.parametrize("name", CONSTANTS)
def test_header_constant(header, name):
    assert header[name] == getattr(_lib, name)


def test_apply_ops_keep_their_numbers():
    # the two SSB ops were appended to b2s_op; the ten before them keep 0..9
    assert (_lib.OP_SLICE_F32_U8, _lib.OP_DIV_C32, _lib.OP_C32_TO_I16_IQ) == (9, 10, 11)
