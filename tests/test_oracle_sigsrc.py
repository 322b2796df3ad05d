"""SignalSource / FixedPointPhase without a GPU: the library's host-side FixedPointPhase (b2s_fxpt_phase_new,
b2s_fxpt_sin_cos) and sine table against the reference's table (tests/golden/reference_fxpt_sine_table.json) and
the CPU oracle (tests/sigsrc_oracle.c), and the oracle against an independent numpy float32 transcription."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sigsrc_oracle as orc  # noqa: E402  (tests/sigsrc_oracle.py)


@pytest.fixture(scope="module")
def L():
    from futuresdr_b200 import _lib
    return _lib


def lib_phase_new(L, x):
    v = C.c_int32(0)
    assert L.lib.b2s_fxpt_phase_new(float(np.float32(x)), C.byref(v)) == L.OK
    return v.value


def lib_sin_cos(L, value):
    s, c = C.c_float(0.0), C.c_float(0.0)
    assert L.lib.b2s_fxpt_sin_cos(int(value), C.byref(s), C.byref(c)) == L.OK
    return np.float32(s.value), np.float32(c.value)


def bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def test_fixture_is_the_generating_formula():
    """f(u) = sin(u pi / 2^31), incx = (2^32 - 1) / 1024, T[i] = ((f(b) - f(a)) / (b - a), f(a)), in f64 rounded to
    f32, reproduces all 2048 literals; incx = 2^32 / 1024 would not."""
    i = np.arange(1024, dtype=np.float64)

    def gen(incx):
        a, b = i * incx, (i + 1) * incx
        f = lambda u: np.sin(u * np.pi / 2.0 ** 31)  # noqa: E731
        return np.stack([((f(b) - f(a)) / (b - a)).astype(np.float32), f(a).astype(np.float32)], 1)

    assert np.array_equal(bits(gen((2.0 ** 32 - 1) / 1024)), bits(orc.TABLE))
    assert not np.array_equal(bits(gen(2.0 ** 32 / 1024)), bits(orc.TABLE))


def test_library_table_equals_fixture_at_every_index(L):
    """Every index through b2s_fxpt_sin_cos.  A fraction of 0 returns the offset exactly (all 1024 offsets, bit for
    bit); fractions 1, 2^21, 0x3FFFFF and random ones return slope * frac + offset, the outputs the slopes make."""
    rng = np.random.default_rng(11)
    for i in range(1024):
        s, c = lib_sin_cos(L, (i << 22) - (1 << 32 if i >= 512 else 0))
        assert bits(s) == bits(orc.TABLE[i, 1]), i
        fracs = [0, 1, 1 << 21, 0x3FFFFF] + [int(f) for f in rng.integers(0, 1 << 22, 4)]
        for f in fracs:
            v = np.uint32((i << 22) | f).view(np.int32)
            s, c = lib_sin_cos(L, v)
            assert bits(s) == bits(orc.fxpt_sin(v)) and bits(c) == bits(orc.fxpt_cos(v)), (i, f)
            assert bits(s) == bits(orc.np_lookup(np.uint32((i << 22) | f))), (i, f)


def _phase_inputs():
    f32 = np.float32
    pi = f32(np.pi)
    special = [0.0, -0.0, pi, -pi, np.nextafter(pi, f32(4)), np.nextafter(pi, f32(0)), f32(2 * np.pi),
               -f32(2 * np.pi), 3 * pi, -3 * pi, 1e9, -1e9, 1e30, -1e30, 3.4e38, -3.4e38, np.inf, -np.inf, np.nan,
               1e-45, -1e-45, 1.1754942e-38, -1.1754942e-38, 1e-40, 0.5, -0.5, 1.0, 2.0 ** 31 * 2 * np.pi,
               2.0 ** 33, -(2.0 ** 33), 13493037056.0, -13493037056.0, 6.7e9, -6.7e9]
    rng = np.random.default_rng(5)
    rand = np.concatenate([rng.uniform(-10, 10, 40000), rng.uniform(-1e6, 1e6, 20000),
                           rng.standard_normal(10000) * 1e12]).astype(np.float32)
    rand_bits = rng.integers(0, 1 << 32, 30000, dtype=np.uint64).astype(np.uint32).view(np.float32)
    return np.concatenate([np.array(special, np.float32), rand, rand_bits])


def test_phase_new_equals_oracle(L):
    """FixedPointPhase::new on signed zeros, +-pi and its neighbours, +-TAU, 3 pi, huge values, infinities, NaN,
    denormals and 10^5 random values (uniform, and random bit patterns that include every class)."""
    xs = _phase_inputs()
    assert xs.size >= 100000
    got = np.array([lib_phase_new(L, x) for x in xs], np.int64)
    want = np.array([orc.phase_new(x) for x in xs], np.int64)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(float(xs[k]), int(got[k]), int(want[k])) for k in bad[:10]]
    assert lib_phase_new(L, np.nan) == 0 and lib_phase_new(L, np.inf) == orc.phase_new(np.inf)


def test_oracle_phase_new_equals_numpy():
    xs = _phase_inputs()
    want = np.array([orc.phase_new(x) for x in xs], np.int64)
    assert np.array_equal(orc.np_phase_new(xs).astype(np.int64), want)


PAIRS = [(1000.0, 48000.0), (48000.0 / 4, 48000.0), (48000.0 / 64, 48000.0), (-3000.0, 48000.0),
         (30000.0, 48000.0), (47999.0, 48000.0), (100000.0, 48000.0), (-100000.0, 48000.0), (1.0, 0.0),
         (-1.0, 0.0), (0.0, 0.0), (440.0, 44100.0), (1e-3, 1e9), (np.nan, 48000.0), (1000.0, np.inf)]


@pytest.mark.parametrize("f, fs", PAIRS)
def test_builder_increment(L, f, fs):
    """inc = FixedPointPhase::new(2 PI f / fs) in f32 (mod.rs:130-133) for negative f, f > fs/2, fs = 0 and more;
    the library's FixedPointPhase::new of that f32 value, the oracle and numpy agree."""
    w = np.float32(2.0) * np.float32(np.pi) * np.float32(f)
    with np.errstate(all="ignore"):
        w = w / np.float32(fs)
    assert lib_phase_new(L, w) == orc.builder_inc(f, fs) == int(orc.np_builder_inc(f, fs))


@pytest.mark.parametrize("dtype", [np.float32, np.complex64])
@pytest.mark.parametrize("wave", [orc.COS, orc.SIN, orc.SQUARE])
def test_oracle_work_equals_numpy_on_ragged_calls(wave, dtype):
    """The C oracle's work() over a ragged call sequence equals the numpy transcription bit for bit, phase carried
    across calls, with amplitudes that make signed zeros and NaN."""
    for f, fs, amp, ph0 in [(1000.0, 48000.0, 0.5, 0.3), (-3000.0, 48000.0, -1.0, -2.0), (12000.0, 48000.0, 0.0, 1.0),
                            (750.0, 48000.0, np.nan, 0.0), (30011.0, 48000.0, 3.0, 100.0)]:
        src = orc.Source(wave, f, fs, amp, ph0, dtype)
        phase, inc = src.phase.value, src.inc
        for n in (0, 1, 3, 4095, 70001):
            got = src.work(n)
            want, phase = orc.np_work(wave, dtype == np.complex64, phase, inc, amp, n)
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (f, amp, n)
            assert src.phase.value == phase


def test_fxpt_null_arguments_refused(L):
    v, s = C.c_int32(0), C.c_float(0)
    assert L.lib.b2s_fxpt_phase_new(1.0, None) == L.EINVAL
    assert L.lib.b2s_fxpt_sin_cos(0, None, C.byref(s)) == L.EINVAL
    assert L.lib.b2s_fxpt_sin_cos(0, C.byref(s), None) == L.EINVAL
    assert L.lib.b2s_fxpt_phase_new(1.0, C.byref(v)) == L.OK


def test_python_fixed_point_phase_mirror():
    from futuresdr_b200 import FixedPointPhase
    p = FixedPointPhase.new(np.float32(np.pi) / 2)
    assert p.value == orc.phase_new(np.float32(np.pi) / 2)
    assert bits(p.sin()) == bits(orc.fxpt_sin(p.value)) and bits(p.cos()) == bits(orc.fxpt_cos(p.value))
    assert FixedPointPhase(0xFFFFFFFF).value == -1
