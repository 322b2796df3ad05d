"""Overlap-save FFT FIR (B2S_ALGO_FFT) against float64, on structured and extreme signals: the numerics contract of
include/b200sdr.h, case by case.

Geometry.  One CTA owns one block: block b of a call reads the NF = 4096 inputs x[s : s+NF], s = b*V (zeros past the
end of the input), and writes the V = NF - (ntaps-1) outputs y[s : s+V].  y = IFFT(FFT(x_block) . H) with
H = (1/NF) FFT(reversed taps) rounded to f32, both transforms single-precision radix-16 Stockham.

The gate.  For output k in the block that starts at s, with x_b = x[s : s+NF] and c_b its circular correlation with the
taps (the block's V outputs plus the N-1 that wrap, rms(c_b) = ||X_b . NF H||_2 / NF <= max|G| rms(x_b)):

    |y_k - y64_k| <= C * u * log2(NF) * (||taps||_2 * rms(x_b) + rms(c_b)),      u = 2^-24,  C = 8 for every case

Reasoning.  A log2(NF)-pass FFT returns X + e with ||e||_2 <= c * u * log2(NF) * ||X||_2 (c a small constant per pass:
one rounding per add, a few ulp per twiddle); ||X||_2 = sqrt(NF) ||x_b||_2 = NF * rms(x_b).  The error is spread over
the bins, so the product with H carries it through ||H||_2 = ||taps||_2 / sqrt(NF) (Parseval), and the unnormalised
inverse multiplies the 2-norm by sqrt(NF) again: the forward transform's share of the rms output error is
~ c * u * log2(NF) * ||taps||_2 * rms(x_b).  The inverse transform's own rounding, the f32 rounding of H and of the
product are relative to what the inverse transforms, the block's circular output: ~ c * u * log2(NF) * rms(c_b).  For
broadband input the two terms are equal; when the block's energy sits where |G| peaks (a passband tone, DC or a step
through all-positive taps or a boxcar) the second is up to max|G| / ||taps||_2 times the first -- 15x for 300 positive
taps, 32x for the 1024-tap boxcar, where even rounding the exact result to f32 would exceed the first term alone.  Taking
the largest of ~NF Gaussian-like errors costs a factor of ~4 over the rms, while the pass-by-pass errors add in quadrature
rather than linearly (sqrt(log2 NF) in place of log2 NF), so a correct kernel with exact twiddles sits near 1 on this
scale; the core builds each butterfly's twiddle powers by a product tree (up to four multiplies deep), which roughly
triples that (the largest case here, noise through 128 complex taps, sits at ~3.3).  C = 8 covers both, and an H kept to
16 significant bits takes most cases past it.  The error is NOT relative to the output: a stopband tone has a tiny
output and the full input-sized first term.

Every case with finite outputs and no floor also keeps the bar of tests/test_gpu_fir_fft.py (1e-5 * ||taps||_1 * max|x|
against the f32 reference loop).  Every case reports, with -s, on the gate's scale (max over k of error / the gate's
right-hand side without C):
    fft-f64 : this kernel against float64 -- asserted <= C
    fft-f32 : this kernel against the reference's f32 loop (oracle.fir)
    ref-f64 : the reference's f32 loop against float64
"""
import ctypes as C_

import numpy as np
import pytest

import oracle as orc

gpu = pytest.mark.gpu

NF = 4096
LOG2NF = 12
U = 2.0 ** -24
C = 8.0
N_OUT = 20000          # outputs per case: 5 blocks at V = 4033, 10 at V = 2048


def _v(ntaps):
    return NF - (ntaps - 1)


# ---------------------------------------------------------------------------------------------------------------------
# float64 arbiter

def conv64(taps, x, n_out):
    """o[k] = sum_t x[k+t] * taps[N-1-t] in complex128, for real or complex taps."""
    taps = np.asarray(taps).astype(np.complex128)
    x = np.asarray(x).astype(np.complex128)
    return np.convolve(x[: n_out + taps.size - 1], taps, mode="valid")[:n_out]


def y64(taps, x, n_out):
    if np.iscomplexobj(taps):
        return conv64(taps, x, n_out)
    return orc.fir_c32_exact(taps, x, n_out)


def test_conv64_matches_the_oracle_arbiter_on_real_taps():
    rng = np.random.default_rng(101)
    for ntaps, n in ((1, 10), (64, 700), (1024, 3000)):
        taps = rng.uniform(-1, 1, ntaps).astype(np.float32)
        x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
        n_out = n - ntaps + 1
        a, b = conv64(taps, x, n_out), orc.fir_c32_exact(taps, x, n_out)
        assert a.shape == b.shape == (n_out,)
        assert np.max(np.abs(a - b)) <= 1e-12 * float(np.sum(np.abs(taps))) * float(np.max(np.abs(x)))
    # complex taps: the same sum with the tap's imaginary part, against the product written out
    taps = (rng.standard_normal(5) + 1j * rng.standard_normal(5)).astype(np.complex64)
    x = (rng.standard_normal(40) + 1j * rng.standard_normal(40)).astype(np.complex64)
    want = [sum(complex(x[k + t]) * complex(taps[4 - t]) for t in range(5)) for k in range(36)]
    assert np.allclose(conv64(taps, x, 36), want, rtol=0, atol=1e-12)


# ---------------------------------------------------------------------------------------------------------------------
# the gate

def unit(taps, x, n_out, start=0):
    """u * log2(NF) * (||taps||_2 * rms(x_block) + rms(circular output of the block)), per output k; the block window
    is x[s : s+NF] with zeros past the end of x, s = start + (k // V) * V."""
    taps = np.asarray(taps).astype(np.complex128)
    V = _v(taps.size)
    g2 = float(np.sqrt(np.sum(np.abs(taps) ** 2)))
    gpad = np.zeros(NF, np.complex128)
    gpad[: taps.size] = taps[::-1]
    G = np.abs(np.fft.ifft(gpad)) * NF               # |NF * H| in exact arithmetic
    x = np.asarray(x)
    nb = -(-n_out // V)
    r = np.empty(nb)
    for b in range(nb):
        w = np.zeros(NF, np.complex128)
        seg = x[start + b * V: start + b * V + NF]
        w[: seg.size] = seg
        rms_x = np.sqrt(np.sum(np.abs(w) ** 2) / NF)
        rms_y = np.sqrt(np.sum((np.abs(np.fft.fft(w)) * G) ** 2)) / NF
        r[b] = g2 * rms_x + rms_y
    return U * LOG2NF * np.repeat(r, V)[:n_out]


def ratio(err, scale):
    """max over k of err/scale; an output with scale 0 must have err 0 (reported as inf otherwise)."""
    zero = scale == 0
    if np.any(err[zero] != 0):
        return float("inf")
    return float(np.max(err[~zero] / scale[~zero])) if np.any(~zero) else 0.0


def check_gate(name, taps, x, y, start=0, floor=0.0, nonfinite_ok=False):
    """Assert the gate (plus an absolute floor) on every output; report the three errors on the gate's scale."""
    n = y.size
    ref64 = y64(taps, x[start:], n)
    sc = unit(taps, x, n, start)
    err = np.abs(y.astype(np.complex128) - ref64)
    fin = np.isfinite(y.real) & np.isfinite(y.imag)
    if nonfinite_ok:
        err = np.where(fin, err, 0.0)
    else:
        assert np.all(fin), f"{name}: non-finite output"
    bad = err > C * sc + floor
    assert not np.any(bad), (f"{name}: {int(np.sum(bad))} outputs outside the gate, first at k = {int(np.argmax(bad))}:"
                             f" err {err[bad][0]:.3e} gate {C * sc[bad][0] + floor:.3e}")
    g = ratio(err, sc + floor / C)
    _, p0, _, ref32 = orc.fir(taps, x[start:], n)
    assert p0 == n
    r32 = np.abs(ref32.astype(np.complex128) - ref64)
    e32 = np.abs(y - ref32)
    if not nonfinite_ok and floor == 0.0:
        old = 1e-5 * float(np.sum(np.abs(taps))) * float(np.max(np.abs(x[start:start + n + len(taps) - 1])))
        assert float(np.max(e32)) <= old, f"{name}: outside the old bar"
    print(f"[fft-numerics] {name:34s} fft-f64 {g:6.3f} (margin to C {C / g if g else float('inf'):6.1f}x)  "
          f"fft-f32 {ratio(np.where(fin, e32, 0.0), sc):8.3f}  ref-f64 {ratio(r32, sc):8.3f}")
    return g


# ---------------------------------------------------------------------------------------------------------------------
# running the kernel

def _run(taps, x, cap=None, in_off=0, out_off=0):
    """One FirFilter::filter call on the FFT path; x is placed `in_off` items into its allocation, the output `out_off`
    items into its own.  Returns (produced, y)."""
    import torch
    import futuresdr_b200 as fb
    f = fb.FirFilter(taps, algo=fb.ALGO_FFT)
    assert f.algo == fb.ALGO_FFT
    n = x.size
    cap = n - len(taps) + 1 if cap is None else cap
    xb = torch.zeros(in_off + n, dtype=torch.complex64, device="cuda")
    xb[in_off:] = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    yb = torch.full((out_off + cap,), 3.0, dtype=torch.complex64, device="cuda")
    c, p, st = f.filter(xb[in_off:], yb[out_off:])
    torch.cuda.synchronize()
    return p, yb[out_off:out_off + p].cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# the case matrix

def _lowpass(ntaps, cutoff):
    return orc.firdes_lowpass(cutoff, orc.window_kaiser(ntaps, 8.0)).astype(np.float32)


def _taps():
    """name -> (taps, passband frequency, stopband frequency), frequencies in cycles per sample."""
    rng = np.random.default_rng(4096)
    lp = orc.kaiser_lowpass(0.08, 0.015, 1e-5)                 # 429 taps, unit DC gain
    return {
        "kaiser_lp_429": (lp, 0.03, 0.31),
        "uniform_64": (rng.uniform(-1, 1, 64).astype(np.float32), 0.03, 0.31),
        "uniform_1024": (rng.uniform(-1, 1, 1024).astype(np.float32), 0.03, 0.31),
        "uniform_2049": (rng.uniform(-1, 1, 2049).astype(np.float32), 0.03, 0.31),
        "positive_300": (rng.uniform(0, 1, 300).astype(np.float32), 0.0007, 0.31),
        "boxcar_1024": (np.full(1024, 1.0 / 1024, np.float32), 0.0001, 0.31),
        "xlating_c128": (orc.xlating_taps(_lowpass(128, 0.1), 0.2, 1.0), 0.21, -0.3),
        "xlating_c700": (orc.xlating_taps(_lowpass(700, 0.05), -0.125, 1.0), -0.13, 0.25),
    }


TAPS = _taps()
SIGNALS = ("dc", "stopband_tone", "passband_tone_100dB", "nyquist", "square", "noise", "bursty")


def _signal(kind, n, f_pass, f_stop, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n)
    noise = rng.standard_normal(n) + 1j * rng.standard_normal(n)
    if kind == "dc":
        x = np.full(n, 0.7391 - 0.2957j)
    elif kind == "stopband_tone":
        x = np.exp(2j * np.pi * f_stop * t)
    elif kind == "passband_tone_100dB":
        x = np.exp(2j * np.pi * f_pass * t) + 1e-5 * np.exp(2j * np.pi * f_stop * t)
    elif kind == "nyquist":
        x = (-1.0) ** t * (1 + 1j)
    elif kind == "square":
        x = np.sign(np.sin(2 * np.pi * (t + 0.5) / 97.0)) * (0.9 + 0.4j)
    elif kind == "noise":
        x = noise
    else:   # bursts of 3000 noisy samples between zero runs of 12000: every run holds at least one whole block window
        x = np.where((t % 15000) < 3000, noise, 0)
    return x.astype(np.complex64)


@gpu
@pytest.mark.parametrize("signal", SIGNALS)
@pytest.mark.parametrize("tname", list(TAPS))
def test_structured_signals_hold_the_gate(tname, signal):
    taps, f_pass, f_stop = TAPS[tname]
    N = len(taps)
    x = _signal(signal, N_OUT + N - 1, f_pass, f_stop, seed=len(tname) * 31 + SIGNALS.index(signal))
    p, y = _run(taps, x)
    assert p == N_OUT
    check_gate(f"{tname}/{signal}", taps, x, y)
    if signal == "bursty":
        V = _v(N)
        b = np.arange(p) // V
        silent = np.array([not np.any(x[i * V: i * V + NF]) for i in range(b[-1] + 1)])[b]
        assert np.any(silent)
        assert np.all(y[silent] == 0), "an all-zero block window must give exact zeros"


# ---------------------------------------------------------------------------------------------------------------------
# non-finite input

def _poisoned(p, ntaps, i):
    """Outputs k < p of every block whose window [s, s+NF) contains input i."""
    V = _v(ntaps)
    k = np.arange(p)
    s = (k // V) * V
    return (s <= i) & (i < s + NF)


@gpu
@pytest.mark.parametrize("bad", [np.nan, np.inf, -np.inf])
@pytest.mark.parametrize("where", ["one_block", "overlap", "past_the_outputs"])
def test_non_finite_sample_poisons_exactly_its_blocks(bad, where):
    """A NaN/Inf input at index i makes non-finite exactly the outputs of the blocks whose NF-sample window holds i:
    a superset of the reference's [i-N+1, i], inside [i-NF+1, i+NF-N].  Every other output is bit-identical to the
    clean run.  past_the_outputs: the output capacity ends before the last block's window does, so that block reads
    (and is poisoned by) a sample no output of the reference depends on."""
    rng = np.random.default_rng(77)
    N, n = 1024, 20000
    V = _v(N)
    taps = rng.uniform(-1, 1, N).astype(np.float32)
    x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
    i, cap = {"one_block": (V + 2000, None),             # window of block 1 only
              "overlap": (2 * V + 100, None),            # windows of blocks 1 and 2
              "past_the_outputs": (3 * V + 3500, 3 * V + 10)}[where]
    p, clean = _run(taps, x, cap)
    xb = x.copy()
    xb[i] = complex(bad, 1.0)
    p2, y = _run(taps, xb, cap)
    assert p == p2
    k = np.arange(p)
    want = _poisoned(p, N, i)
    nblocks = len(set((k[want] // V).tolist()))
    assert nblocks == {"one_block": 1, "overlap": 2, "past_the_outputs": 1}[where]
    ref_window = (k >= i - N + 1) & (k <= i)
    assert not np.any(ref_window & ~want)
    assert np.all(k[want] >= i - NF + 1) and np.all(k[want] <= i + NF - N)
    fin = np.isfinite(y.real) & np.isfinite(y.imag)
    assert np.array_equal(~fin, want), f"non-finite outputs {np.flatnonzero(~fin)[[0, -1]]} expected {k[want][[0, -1]]}"
    assert np.array_equal(y[fin].view(np.uint64), clean[fin].view(np.uint64)), "other outputs bit-identical"


# ---------------------------------------------------------------------------------------------------------------------
# amplitude range and denormals

_LP = orc.kaiser_lowpass(0.08, 0.015, 1e-5)


def _scaled(kind, n, scale):
    rng = np.random.default_rng(5)
    if kind == "dc":
        x = np.full(n, (0.6 - 0.8j) * scale)
    else:
        z = rng.standard_normal(n) + 1j * rng.standard_normal(n)
        x = z / np.max(np.abs(z)) * scale
    return x.astype(np.complex64)


def _finite_limit(taps):
    """The largest max|x| the contract keeps finite: 4096 * max|x| * max(1, ||taps||_1) < 2^128."""
    return 2.0 ** 128 / (NF * max(1.0, float(np.sum(np.abs(taps)))))


@gpu
@pytest.mark.parametrize("kind", ["dc", "noise"])
def test_amplitude_range_holds_the_gate(kind):
    """max|x| from 2^-100 up to just below the finite limit: the same gate, no floor, every output finite."""
    N = len(_LP)
    lim = _finite_limit(_LP)
    for e in (-100, -64, -20, 0, 20, 64, 100, None):
        scale = 0.99 * lim if e is None else 2.0 ** e
        x = _scaled(kind, N_OUT + N - 1, scale)
        assert np.all(np.isfinite(x.view(np.float32)))
        p, y = _run(_LP, x)
        check_gate(f"lowpass/{kind} max|x| 2^{np.log2(scale):.2f}", _LP, x, y)


@gpu
@pytest.mark.parametrize("kind", ["dc", "noise"])
def test_tiny_and_denormal_input_holds_the_gate_plus_floor(kind):
    """Below 2^-100 the products X.H (H carries the 1/NF) fall into the subnormal range and lose bits: the gate plus an
    absolute floor of ||taps||_1 * 2^-126, down to input that is denormal only."""
    N = len(_LP)
    floor = float(np.sum(np.abs(_LP))) * 2.0 ** -126
    for e in (-110, -120, -126, -135, -145):
        x = _scaled(kind, N_OUT + N - 1, 2.0 ** e)
        if e < -126:
            assert np.all(np.abs(x.view(np.float32)) < np.float32(2.0 ** -126)), "denormal only"
        p, y = _run(_LP, x)
        check_gate(f"lowpass/{kind} max|x| 2^{e}", _LP, x, y, floor=floor)


@gpu
@pytest.mark.parametrize("kind", ["dc", "noise"])
def test_beyond_the_finite_range_never_gives_a_wrong_finite_value(kind):
    """Past the limit the transforms overflow: every output is within the gate or non-finite, never a wrong finite
    value."""
    N = len(_LP)
    for scale in (2.0 ** 117, 2.0 ** 126):
        x = _scaled(kind, N_OUT + N - 1, scale)
        assert NF * float(np.max(np.abs(x))) >= 2.0 ** 128
        p, y = _run(_LP, x)
        fin = np.isfinite(y.real) & np.isfinite(y.imag)
        if kind == "dc":
            assert not np.any(fin[:_v(N)]), "DC past the limit overflows the forward transform of a full block"
        check_gate(f"lowpass/{kind} max|x| 2^{np.log2(scale):.0f} (past)", _LP, x, y, nonfinite_ok=True)


# ---------------------------------------------------------------------------------------------------------------------
# slices and calls

@gpu
@pytest.mark.parametrize("in_off,out_off", [(0, 0), (1, 0), (0, 1), (1, 1)])
def test_element_offsets(in_off, out_off):
    """Slices one item past the allocation's start (8-byte aligned, still the FFT kernel) hold the same gate."""
    taps = TAPS["uniform_1024"][0]
    x = _signal("noise", N_OUT + 1023, 0, 0, seed=91)
    p, y = _run(taps, x, in_off=in_off, out_off=out_off)
    assert p == N_OUT
    check_gate(f"uniform_1024/noise offsets {in_off},{out_off}", taps, x, y)


@gpu
def test_ragged_calls_restart_the_block_geometry():
    """A stream fed in calls of uneven length: each call's blocks start at its own first input."""
    taps = TAPS["kaiser_lp_429"][0]
    N = len(taps)
    x = _signal("square", 60000, 0, 0, seed=92) + _signal("noise", 60000, 0, 0, seed=93) * np.float32(1e-3)
    pos = 0
    for n in (N, N + 1, NF, NF + 1, 2 * _v(N) + N - 1, 9999, 17_321, 4444):
        p, y = _run(taps, x[pos:pos + n])
        assert p == n - N + 1
        check_gate(f"kaiser_lp_429 call at {pos} of {n}", taps, x, y, start=pos)
        pos += p


@gpu
def test_exec_hist_sharded_path():
    """b2s_fir_exec_hist with a 1024-tap filter and the history in its own allocation (the sharded FIR's step): the
    logical slice hist ++ in is one call, whose blocks start at the history's first item."""
    import torch
    import futuresdr_b200 as fb
    from futuresdr_b200._lib import lib, check
    N = 1024
    H = N - 1
    taps = TAPS["uniform_1024"][0]
    x = _signal("noise", H + 3 * N_OUT, 0, 0, seed=94)
    fir = fb.FirFilter(taps)
    assert fir.algo == fb.ALGO_FFT
    hist = torch.from_numpy(x[:H]).cuda()
    pad = ((H + 255) // 256) * 256
    buf = torch.zeros(pad + x.size - H, dtype=torch.complex64, device="cuda")
    buf[pad:] = torch.from_numpy(x[H:]).cuda()
    out = torch.zeros(x.size - H, dtype=torch.complex64, device="cuda")
    c, p, st = C_.c_size_t(0), C_.c_size_t(0), C_.c_int32(0)
    check(lib.b2s_fir_exec_hist(fir._h, C_.c_void_p(hist.data_ptr()), H, C_.c_void_p(buf[pad:].data_ptr()),
                                x.size - H, C_.c_void_p(out.data_ptr()), out.numel(), None,
                                C_.byref(c), C_.byref(p), C_.byref(st)), fir.ctx.handle)
    torch.cuda.synchronize()
    assert p.value == x.size - H
    check_gate("uniform_1024/noise exec_hist", taps, x, out.cpu().numpy())
