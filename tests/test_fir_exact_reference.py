"""The exact integer references of tests/fir_exact.py (used by tests/test_gpu_fir_exact.py) against the CPU oracle, which
is exact on integer data too, against np.convolve, and against the reference's known-answer vectors in tests/golden/."""
import json
import os
import sys

import numpy as np
import pytest

import oracle as orc

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fir_exact as fx  # noqa: E402

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_known_answers.json")


@pytest.mark.parametrize("kind", ["f32", "c32", "c32c"])
@pytest.mark.parametrize("ntaps,decim", [(1, 1), (2, 1), (7, 1), (64, 1), (257, 1), (5, 2), (9, 3), (33, 7), (64, 64),
                                         (3, 19), (100, 40)])
def test_fir_reference_equals_oracle_bit_for_bit(kind, ntaps, decim):
    rng = np.random.default_rng(1000 * ntaps + decim)
    x = fx.int_samples(rng, 3000 + ntaps, kind != "f32")
    taps = fx.int_taps(rng, ntaps, kind == "c32c")
    for cap in (0, 1, 17, 10 ** 6):
        c, p, st, ref = orc.decim_fir(taps, decim, x, cap)
        assert fx.fir_counts(x.size, ntaps, decim, cap) == (c, p, st)
        got = fx.fir(taps, x, decim, p)
        assert got.size == p and np.array_equal(got, ref.astype(got.dtype))
    if decim == 1:
        c, p, st, ref = orc.fir(taps, x, x.size)
        assert np.array_equal(fx.fir(taps, x), ref.astype(got.dtype))


@pytest.mark.parametrize("cplx", [False, True])
@pytest.mark.parametrize("L,M,T", [(1, 1, 1), (3, 2, 24), (2, 3, 1), (1, 10, 240), (5, 1, 2), (8, 3, 5), (48, 125, 24),
                                   (160, 147, 3), (1, 100, 17), (4, 125, 24)])
def test_resampler_reference_equals_oracle_bit_for_bit(cplx, L, M, T):
    rng = np.random.default_rng(7 * L + M + T)
    x = fx.int_samples(rng, 4000 + T, cplx)
    taps = fx.int_taps(rng, L * T)
    for cap in (0, 1, L + 1, 3 * L - 1, 10 ** 7):
        c, p, st, ref = orc.resamp_fir(taps, L, M, x, cap)
        assert fx.resamp_counts(x.size, L, M, T, cap) == (c, p, st)
        got = fx.resamp(taps, L, M, x, p)
        assert np.array_equal(got, ref.astype(got.dtype))


@pytest.mark.parametrize("n,ntaps", [(1, 1), (10, 10), (9, 10), (5000, 300), (1 << 18, 257), (300000, 1000)])
def test_reference_equals_np_convolve(n, ntaps):
    """Both branches (direct and rounded FFT convolution) equal np.convolve on integers."""
    rng = np.random.default_rng(n + ntaps)
    for cplx in (False, True):
        x, taps = fx.int_samples(rng, n, cplx), fx.int_taps(rng, ntaps, cplx)
        want = np.convolve(x.astype(np.complex128), taps.astype(np.complex128), "valid") if n >= ntaps else []
        got = fx.conv_valid(x, taps)
        assert np.array_equal(got, np.asarray(want).astype(got.dtype) if cplx else np.real(want))
    # the FFT branch is taken above the direct-convolution budget
    assert 300000 * 1000 > fx._DIRECT_MACS


def test_reference_reproduces_known_answers():
    cases = json.load(open(GOLDEN))["cases"]
    seen = set()
    for case in cases:
        x = np.array(case["input"], np.float32)
        taps = np.array(case["taps"], np.float32)
        cap = case["out_cap"]
        if case["filter"] == "fir":
            counts = fx.fir_counts(x.size, taps.size, 1, cap)
            got = fx.fir(taps, x, 1, counts[1])
        elif case["filter"] == "decimating_fir":
            counts = fx.fir_counts(x.size, taps.size, case["decim"], cap)
            got = fx.fir(taps, x, case["decim"], counts[1])
        elif case["filter"] == "polyphase_resampling_fir":
            T = taps.size // case["interp"]
            counts = fx.resamp_counts(x.size, case["interp"], case["decim"], T, cap)
            got = fx.resamp(taps, case["interp"], case["decim"], x, counts[1])
        else:
            continue
        seen.add(case["filter"])
        assert counts == (case["consumed"], case["produced"], case["status"]), case["cite"]
        assert list(got) == case["output"], case["cite"]
    assert seen == {"fir", "decimating_fir", "polyphase_resampling_fir"}


def test_generators():
    rng = np.random.default_rng(1)
    x = fx.int_samples(rng, 100000, True)
    assert x.dtype == np.complex64 and x.real.min() == -8 and x.real.max() == 8 and x.imag.min() == -8
    assert not np.array_equal(x.real, x.imag)
    assert np.all(x.real == np.rint(x.real))
    for n in (2, 3, 24):
        for _ in range(200):
            t = fx.int_taps(rng, n)
            assert t.dtype == np.float32 and np.any(t != t[0])
