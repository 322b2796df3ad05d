"""Tensor-core (split-bf16) FIR on STRUCTURED signals -- everything the white-noise parity tests cannot see.

The split keeps ~16-17 bits of each operand (x = bf16 hi + bf16 lo, same for the taps; three of the four partial
products are summed), so the per-product error is bounded by ~2^-16 + 2*2^-17 of |x||g| in the worst case and is
~2^-18 rms; on white noise the errors average, on DC / tones / same-sign taps the sample-residual part is COHERENT.
Every case below reports the error three ways (printed with -s, asserted where the contract says so):
    e_f32 : vs the f32 strict-order oracle (oracle.fir  == fir.rs:77-88 on stable Rust)
    e_f64 : vs the exact f64 evaluation    (oracle.fir_c32_exact)
    e_rms : max |y - y_f64| / rms(y_f64)
all normalised:  e / (||taps||_1 * max|x|)  must be <= 1e-5  (the parity bar of SURVEY.md 7 / DESIGN.md 2).
For comparison the same three numbers are computed for the reference's OWN f32 evaluation against f64.
"""
import numpy as np
import pytest

import oracle as orc

pytestmark = pytest.mark.gpu


def _run(taps, x, algo=None):
    import torch
    import futuresdr_b200 as fb
    f = fb.FirFilter(taps, sample_dtype=x.dtype, algo=fb.ALGO_TENSOR if algo is None else algo)
    n = x.size
    xd = torch.from_numpy(x).cuda()
    yd = torch.zeros(n, dtype=xd.dtype, device="cuda")
    c, p, st = f.filter(xd, yd)
    torch.cuda.synchronize()
    return yd[:p].cpu().numpy(), p


def _three_errors(name, taps, x, y):
    _, p0, _, ref32 = orc.fir(taps, x, x.size)
    assert p0 == y.size
    ref64 = orc.fir_c32_exact(taps, x, y.size)
    scale = float(np.sum(np.abs(taps))) * float(np.max(np.abs(x)))
    e_f32 = float(np.max(np.abs(y - ref32))) / scale
    e_f64 = float(np.max(np.abs(y.astype(np.complex128) - ref64))) / scale
    rms = float(np.sqrt(np.mean(np.abs(ref64) ** 2))) or 1.0
    e_rms = float(np.max(np.abs(y.astype(np.complex128) - ref64))) / rms
    r_f64 = float(np.max(np.abs(ref32.astype(np.complex128) - ref64))) / scale
    print(f"[tensor-structured] {name:28s} e_f32 {e_f32:.2e}  e_f64 {e_f64:.2e}  e_rms {e_rms:.2e}   "
          f"(reference f32 vs f64: {r_f64:.2e})")
    return e_f32, e_f64, e_rms


def _cases():
    rng = np.random.default_rng(2024)
    n = 40000
    t = np.arange(n)
    unit = rng.uniform(-1, 1, 256).astype(np.float32)
    pos = rng.uniform(0, 1, 256).astype(np.float32)
    lp = orc.kaiser_lowpass(0.1, 0.02, 1e-4)[:257].astype(np.float32)
    noise = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    yield "dc_random_taps", unit, np.full(n, 0.7391 - 0.2957j, np.complex64)
    yield "dc_positive_taps", pos, np.full(n, 0.7391 - 0.2957j, np.complex64)
    yield "dc_lowpass", lp, np.full(n, 0.3337 + 0.9113j, np.complex64)
    yield "tone_band_edge_lowpass", lp, (0.98 * np.exp(2j * np.pi * 0.1 * t)).astype(np.complex64)
    yield "tone_fullscale_positive_taps", pos, np.exp(2j * np.pi * 0.01234 * t).astype(np.complex64)
    yield "tone_nyquist_random_taps", unit, ((-1.0) ** t * (1 + 1j)).astype(np.complex64)
    yield "mix_60dB", lp, (np.exp(2j * np.pi * 0.03 * t) + 1e-3 * np.exp(2j * np.pi * 0.31 * t) + 1e-3 * noise).astype(np.complex64)
    yield "noise_positive_taps", pos, noise
    yield "square_wave_positive_taps", pos, (np.sign(np.sin(2 * np.pi * t / 97.0)) * (0.9 + 0.4j)).astype(np.complex64)
    yield "tiny_amplitude_1e-20", unit, (1e-20 * noise).astype(np.complex64)
    yield "huge_amplitude_1e20", unit, (1e15 * noise).astype(np.complex64)


@pytest.mark.parametrize("name,taps,x", list(_cases()), ids=[c[0] for c in _cases()])
def test_structured_signals_hold_the_parity_bar(name, taps, x):
    y, p = _run(taps, x)
    e_f32, e_f64, e_rms = _three_errors(name, taps, x, y)
    assert e_f32 <= 1e-5 and e_f64 <= 1e-5, (name, e_f32, e_f64)


def test_boxcar_on_dc_documented_worst_case():
    """The adversarial corner: ALL taps equal and ALL samples equal, so every partial-product error has the same sign.
    The bound is 2^-16 + 2*2^-17 ~ 3.1e-5 of ||taps||_1 max|x| (DESIGN.md 4.2); this case sits inside THAT bound and is
    the documented reason to pick B2S_ALGO_DIRECT for boxcar / CIC-like filters on DC-heavy streams (AUTO does so for
    constant tap vectors)."""
    import futuresdr_b200 as fb
    n = 20000
    worst = 0.0
    for tv, xv in ((0.1, 0.7391), (0.3333333, 0.6180339), (0.007, 1.9999)):
        taps = np.full(64, tv, np.float32)
        x = np.full(n, xv * (1 + 1j), np.complex64)
        y, p = _run(taps, x)
        e_f32, e_f64, e_rms = _three_errors(f"boxcar {tv} on dc {xv}", taps, x, y)
        worst = max(worst, e_f64)
        assert e_f64 <= 3.1e-5
        # AUTO keeps constant-tap filters on the CUDA cores: full f32 products
        y2, _ = _run(taps, x, algo=fb.ALGO_AUTO)
        e2 = _three_errors(f"  same, ALGO_AUTO", taps, x, y2)
        assert e2[1] <= 1e-6
    print(f"[tensor-structured] boxcar-on-DC worst e_f64 {worst:.2e} (bound 3.1e-5)")


def test_denormal_samples_are_flushed_to_zero():
    """Contract (include/b200sdr.h): the tensor path treats f32 DENORMAL samples as zero (the bf16 operands of
    the tensor-core MMA may be flushed to zero), where the reference's scalar loop keeps them.  The difference is bounded by
    ||taps||_1 * 1.18e-38 (the largest denormal) -- 280 dB below full scale -- and normal samples are unaffected."""
    rng = np.random.default_rng(7)
    n = 20000
    taps = rng.uniform(-1, 1, 128).astype(np.float32)
    x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) * 1e-41).astype(np.complex64)
    y, p = _run(taps, x)
    _, _, _, ref = orc.fir(taps, x, n)
    assert np.all(np.isfinite(y.view(np.float32)))
    assert float(np.max(np.abs(y - ref))) <= float(np.sum(np.abs(taps))) * 1.18e-38
    # a stream that mixes normal samples with denormal ones: the normal part is filtered as usual
    x2 = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    x2[::3] *= np.float32(1e-41)
    y2, _ = _run(taps, x2)
    _, _, _, ref2 = orc.fir(taps, x2, n)
    assert float(np.max(np.abs(y2 - ref2))) <= 1e-5 * float(np.sum(np.abs(taps))) * float(np.max(np.abs(x2)))


@pytest.mark.parametrize("bad", [np.inf, -np.inf, np.nan])
def test_non_finite_contract(bad):
    """Contract (include/b200sdr.h, B2S_ALGO_TENSOR): a non-finite sample at index i makes every output of the
    128-sample blocks whose block-Toeplitz K-range contains it NON-FINITE (0 * Inf = NaN in the zero part of the
    operand) -- a superset, inside [i-K, i+131], of the reference's window [i-(ntaps-1), i] (fir.rs:77-88),
    K = 128*ceil((ntaps+127)/128) -- and leaves every other output exactly as if the sample were finite.
    Never a wrong FINITE value."""
    rng = np.random.default_rng(11)
    n, ntaps, i = 30000, 256, 17000
    K = 384
    taps = rng.uniform(-1, 1, ntaps).astype(np.float32)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    clean, p = _run(taps, x)
    xb = x.copy()
    xb[i] = complex(bad, 1.0)
    y, p2 = _run(taps, xb)
    assert p == p2
    k = np.arange(p)
    in_ref_window = (k >= i - (ntaps - 1)) & (k <= i)
    in_k_window = (k >= i - K) & (k <= i + 131)
    finite = np.isfinite(y.real) & np.isfinite(y.imag)
    assert not np.any(finite[in_ref_window]), "outputs the reference poisons must be non-finite"
    assert np.all(finite[~in_k_window]), "outputs outside the K window must stay finite"
    assert np.array_equal(y[~in_k_window], clean[~in_k_window]), "and bit-identical to the clean run"
