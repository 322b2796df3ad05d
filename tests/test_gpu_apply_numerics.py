"""The Apply catalogue (csrc/apply.cu) against float64, op by op, at each op's written bound.

Each reference is a plain float64 computation on the exact f32 values the kernel reads.  Inputs are stratified over the
whole f32 range (a few thousand random mantissas of both signs in every binade from the smallest denormal, 2^-149, to
2^127), a table of special values, and each op's thresholds.  An ulp is the f32 spacing at the exact value: 2^(e-23)
for 2^e <= |v| < 2^(e+1), 2^-149 below 2^-126, and 2^104 from FLT_MAX on, where an f32 inf counts as 2^128 (the value
correct rounding gives inf from).

    ScaleF32, ScaleC32, NormSqr, DivC32   bit-identical to numpy float32: each is one or three correctly rounded IEEE
                                          operations, so a flushed denormal anywhere fails (NaN: positions, not payloads)
    ExpF32                                <= 2 ulp (CUDA's expf bound)
    Log10F32 (param * log10 x)            log10f is within 2 ulp(l) of l = log10(x) (CUDA's bound) and the product is
                                          rounded once: |got - p*l| <= 2 |p| ulp(l) + ulp(p*l) / 2
    MagC32                                <= 3 ulp (CUDA's hypotf bound), and no overflow while the result is finite
    QuadDemod, QuadDemodC32               |got - atan2_64(im, re)| <= DEMOD_BOUND rad, with (re, im) the f32 product
                                          num_complex forms, un-fused; libm's special values

The demodulator's bound.  atan2_poly evaluates atan(a) = a * P(a^2) in f32 Horner form (P's own error is 1.1e-7 rad),
unfolds the octant with one or two f32 subtractions from pi/2 and pi (each rounded: up to ulp(pi)/2 = 1.2e-7 rad), and
takes the quotient a = min/max from div.approx.f32, within 2 ulp of it.  A numpy emulation of the same f32 operations
over 2e7 angles reaches 2.9e-7 rad with a correctly rounded quotient and 3.75e-7 rad with the quotient moved by 2 ulp
(d atan(a)/da <= 1, 2 ulp of a < 1 is at most 2^-23).  DEMOD_BOUND = 4e-7 rad.  On an H100 the kernel's largest error
over these tests is 3.04e-7 rad (2.90e-7 on the unit circle); each test prints its own with -s.
"""
import numpy as np
import pytest

gpu = pytest.mark.gpu

F32, F64, U32 = np.float32, np.float64, np.uint32
FMAX = float(np.finfo(F32).max)
DEMOD_BOUND = 4e-7


@pytest.fixture(scope="module")
def fb():
    import futuresdr_b200 as fb
    import futuresdr_b200.blocks  # noqa: F401
    return fb


def _bits(v):
    return np.asarray(v, F32).view(U32)


def _f32(bits):
    return np.asarray(bits, np.int64).astype(U32).view(F32)


# ±0, the smallest and largest denormals, the smallest normal, ±FLT_MAX, ±inf, NaN, ±1
SPECIALS = _f32([0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00800000, 0x80800000,
                 0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000, 0x7FC00000, 0x3F800000, 0xBF800000])


def stratified(seed, per_exp=2000):
    """per_exp f32 values in every binade 2^e <= |v| < 2^(e+1), e = -149 .. 127 (below -126: the denormals whose
    leading bit is 2^e), with uniformly random mantissa bits below the leading one and random signs."""
    rng = np.random.default_rng(seed)
    parts = []
    for e in range(-149, 128):
        if e >= -126:
            bits = ((e + 127) << 23) | rng.integers(0, 1 << 23, per_exp)
        else:
            k = e + 149
            bits = (1 << k) | rng.integers(0, 1 << k, per_exp)
        parts.append(bits | rng.integers(0, 2, per_exp) << 31)
    return _f32(np.concatenate(parts))


def neighbours(v, k):
    """The 2k+1 f32 values around the f32 rounding of v (v != 0), k steps each way."""
    b = np.int64(_bits(np.abs(F32(v))))
    return np.copysign(_f32(b + np.arange(-k, k + 1)), F32(v))


def ulp32(v):
    """The f32 ulp at each exact (float64) value."""
    e = np.frexp(np.abs(v))[1].astype(np.int64) - 1
    e = np.where(v == 0, -126, e)
    return np.ldexp(1.0, np.clip(e, -126, 127) - 23)


def ulp_err(got, exact):
    """|got - exact| in f32 ulps at exact.  An infinite got counts as +-2^128 and an exact value past +-2^128 as
    +-2^128 (check_ulp separately asserts that a result more than the bound past FLT_MAX is inf)."""
    g = got.astype(F64)
    g = np.where(np.isinf(g), np.copysign(2.0 ** 128, g), g)
    x = np.clip(exact, -2.0 ** 128, 2.0 ** 128)
    with np.errstate(invalid="ignore"):
        return np.abs(g - x) / ulp32(x)


def check_ulp(name, inp, got, exact, bound):
    """NaN exactly where the reference is NaN; elsewhere within `bound` (ulps per element, or one number), and inf
    wherever the exact value is more than the bound past FLT_MAX.  Returns the largest error in ulps."""
    gn, rn = np.isnan(got), np.isnan(exact)
    bad = np.flatnonzero(gn != rn)
    assert bad.size == 0, f"{name}: NaN mismatch at {bad.size} inputs, e.g. {inp[bad[0]]!r} -> {got[bad[0]]!r}, " \
                          f"reference {exact[bad[0]]!r}"
    ok = ~rn
    err = ulp_err(got[ok], exact[ok])
    bnd = np.broadcast_to(bound, got.shape)[ok]
    worst = int(np.argmax(err - bnd))
    i = np.flatnonzero(ok)[worst]
    assert err[worst] <= bnd[worst], f"{name}: {err[worst]:.3g} ulp (bound {bnd[worst]:.3g}) at {inp[i]!r} -> " \
                                     f"{got[i]!r}, reference {exact[i]!r}; max {err.max():.3g} ulp"
    with np.errstate(invalid="ignore"):
        over = ok & (np.abs(exact) > 2.0 ** 128 + np.broadcast_to(bound, got.shape) * 2.0 ** 104)
    miss = np.flatnonzero(over & ~(np.isinf(got) & (np.sign(got) == np.sign(exact))))
    assert miss.size == 0, f"{name}: {inp[miss[0]]!r} -> {got[miss[0]]!r}, reference {exact[miss[0]]!r} overflows"
    print(f"{name}: max {err.max():.3f} ulp over {ok.sum()} values")
    return float(err.max())


def check_bits(name, inp, got, ref):
    """Bit-identical, except that NaNs only have to sit at the same positions."""
    same = (_bits(got) == _bits(ref)) | (np.isnan(got) & np.isnan(ref))
    bad = np.flatnonzero(~same)
    assert bad.size == 0, f"{name}: {bad.size} outputs differ, e.g. {inp[bad[0]]!r} -> {got[bad[0]]!r} " \
                          f"(0x{int(_bits(got[bad[0]])):08x}), numpy {ref[bad[0]]!r} (0x{int(_bits(ref[bad[0]])):08x})"


def run(op, x, param=1.0, steps=None, blk=None):
    """Apply(op, param) over x on the device, in one call or in calls of `steps` items (the last takes the rest)."""
    import torch
    from futuresdr_b200.blocks import Apply
    if blk is None:
        blk = Apply(op, param)
    xd = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    out = torch.empty(x.size, dtype=torch.float32 if blk.out_dtype == np.float32 else torch.complex64, device="cuda")
    pos = 0
    for step in list(steps or ()) + [x.size]:
        n = min(step, x.size - pos)
        assert blk.apply(xd[pos:pos + n], out[pos:pos + n]) == n
        pos += n
    torch.cuda.synchronize()
    return out.cpu().numpy()


def cplx(re, im):
    re, im = np.broadcast_arrays(np.asarray(re, F32), np.asarray(im, F32))
    return np.stack([re, im], axis=-1).reshape(-1).view(np.complex64)


def complex_inputs(seed):
    """Stratified parts paired with a shuffled copy of themselves, and every pair of special values."""
    s = stratified(seed)
    rng = np.random.default_rng(seed + 1)
    sr, si = np.meshgrid(SPECIALS, SPECIALS)
    return cplx(np.concatenate([s, sr.ravel()]), np.concatenate([rng.permutation(s), si.ravel()]))


# ---------------------------------------------------------------------------------------------------------------------
# the yardsticks themselves (no GPU)

def test_ulp32_and_ulp_err():
    assert list(ulp32(np.array([1.0, 1.5, 2.0, 0.0, 2.0 ** -149, 2.0 ** -126, FMAX, 2.0 ** 130]))) == \
        [2.0 ** -23, 2.0 ** -23, 2.0 ** -22, 2.0 ** -149, 2.0 ** -149, 2.0 ** -149, 2.0 ** 104, 2.0 ** 104]
    one = F32(1.0)
    assert ulp_err(np.array([np.nextafter(one, F32(2))]), np.array([1.0]))[0] == 1.0
    assert ulp_err(np.array([F32(np.inf)]), np.array([1e300]))[0] == 0.0
    assert ulp_err(np.array([F32(FMAX)]), np.array([2.0 ** 128]))[0] == 1.0
    assert ulp_err(np.array([F32(0.0)]), np.array([2.0 ** -150]))[0] == 0.5


def test_stratified_inputs_cover_every_binade_with_both_signs():
    s = stratified(1, per_exp=64)
    a = np.abs(s.astype(F64))
    e = np.frexp(a)[1] - 1
    assert np.array_equal(np.bincount(e + 149), np.full(277, 64))
    assert np.all(np.isfinite(s)) and a.min() == 2.0 ** -149 and a.max() < 2.0 ** 128
    assert 0.4 < np.mean(np.signbit(s)) < 0.6


# ---------------------------------------------------------------------------------------------------------------------
# bit-exact ops: one correctly rounded operation per part, denormal inputs, outputs and params included

DENORM = float(_f32(0x00300001))       # a denormal param (about 4.4e-39)


@gpu
@pytest.mark.parametrize("param", [12.0, -0.3, DENORM, 0.0, -0.0, 3.0e38, np.inf])
def test_scale_f32_bit_exact(fb, param):
    from futuresdr_b200.blocks import ApplyOp
    x = np.concatenate([stratified(11), SPECIALS])
    with np.errstate(all="ignore"):
        ref = x * F32(param)
    check_bits(f"ScaleF32({param})", x, run(ApplyOp.ScaleF32, x, param), ref)


@gpu
@pytest.mark.parametrize("param", [0.5, -3.7, DENORM, 0.0, -0.0, 3.0e38])
def test_scale_c32_bit_exact(fb, param):
    from futuresdr_b200.blocks import ApplyOp
    x = complex_inputs(12)
    xf = x.view(F32)
    with np.errstate(all="ignore"):
        ref = xf * F32(param)                    # Complex * f32 multiplies each part (no complex product with 0i)
    check_bits(f"ScaleC32({param})", np.repeat(x, 2), run(ApplyOp.ScaleC32, x, param).view(F32), ref)


@gpu
def test_norm_sqr_bit_exact(fb):
    from futuresdr_b200.blocks import ApplyOp
    x = complex_inputs(13)
    with np.errstate(all="ignore"):
        ref = x.real * x.real + x.imag * x.imag  # f32, un-fused
    assert ref.dtype == F32
    check_bits("NormSqr", x, run(ApplyOp.NormSqr, x), ref)


@gpu
@pytest.mark.parametrize("param", [1e-4, 3.0, -7.0, DENORM, 3.0e38, 0.0, -0.0, np.inf])
def test_div_c32_bit_exact(fb, param):
    from futuresdr_b200.blocks import ApplyOp
    x = complex_inputs(14)
    with np.errstate(all="ignore"):
        ref = x.view(F32) / F32(param)
    check_bits(f"DivC32({param})", np.repeat(x, 2), run(ApplyOp.DivC32, x, param).view(F32), ref)


# ---------------------------------------------------------------------------------------------------------------------
# exp, log10, hypot: CUDA's documented ulp bounds

@gpu
def test_exp_f32_within_2ulp(fb):
    from futuresdr_b200.blocks import ApplyOp
    rng = np.random.default_rng(21)
    # overflow (exp(x) > FLT_MAX), the normal/denormal boundary (2^-126), the smallest denormal (2^-149) and the
    # round-to-zero point (2^-150)
    edges = [np.log(FMAX), -126 * np.log(2), -149 * np.log(2), -150 * np.log(2)]
    x = np.concatenate([stratified(21), SPECIALS, rng.uniform(-104.5, 89.5, 2_000_000).astype(F32),
                        np.concatenate([neighbours(v, 2000) for v in edges])])
    got = run(ApplyOp.ExpF32, x)
    with np.errstate(over="ignore"):
        exact = np.exp(x.astype(F64))
    check_ulp("ExpF32", x, got, exact, 2.0)
    sp = run(ApplyOp.ExpF32, np.array([np.inf, -np.inf, np.nan], F32))
    assert sp[0] == np.inf and _bits(sp[1]) == 0 and np.isnan(sp[2])            # exp(-inf) = +0, not -0


@gpu
@pytest.mark.parametrize("param", [10.0, 20.0, -10.0, 1.0])
def test_log10_f32_within_bound(fb, param):
    from futuresdr_b200.blocks import ApplyOp
    # the magnitudes the spectrum's dB stage gets (powers over ~60 decades), every binade, x near 1 (log10 near 0)
    rng = np.random.default_rng(22)
    x = np.concatenate([stratified(22), SPECIALS, (10.0 ** rng.uniform(-30, 30, 1_000_000)).astype(F32),
                        neighbours(1.0, 3000), F32(10.0) ** np.arange(-38, 39, dtype=F32)])
    got = run(ApplyOp.Log10F32, x, param)
    with np.errstate(divide="ignore", invalid="ignore"):
        l64 = np.log10(x.astype(F64))
        exact = F64(F32(param)) * l64
    # 2 ulp of log10 scaled by |p|, then one rounding of the product, in ulps of the product
    bound = (2 * abs(float(F32(param))) * ulp32(np.nan_to_num(l64)) + 0.5 * ulp32(np.nan_to_num(exact))) / \
        ulp32(np.nan_to_num(exact))
    check_ulp(f"Log10F32({param})", x, got, exact, bound)
    # IEEE special values: log10(+-0) = -inf, log10(x < 0) = NaN, log10(+inf) = +inf, log10(1) = +0, signs through p
    sp = np.array([0.0, -0.0, -1.0, -np.inf, -2.0 ** -149, np.inf, 1.0, np.nan], F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        ref = (F64(F32(param)) * np.log10(sp.astype(F64))).astype(F32)
    check_bits(f"Log10F32({param}) specials", sp, run(ApplyOp.Log10F32, sp, param), ref)


@gpu
def test_mag_c32_within_3ulp(fb):
    from futuresdr_b200.blocks import ApplyOp
    rng = np.random.default_rng(23)
    n = 1_500_000
    # pairs whose binary exponents differ by 0 .. 60, over the whole range (below 2^-149 a part rounds to 0)
    e1 = rng.integers(-149, 128, n)
    e2 = e1 - rng.integers(0, 61, n)
    m = rng.uniform(1, 2, (2, n)) * np.where(rng.random((2, n)) < 0.5, -1, 1)
    a, b = np.ldexp(m[0], e1).astype(F32), np.ldexp(m[1], e2).astype(F32)
    swap = rng.random(n) < 0.5
    re, im = np.where(swap, b, a), np.where(swap, a, b)
    # near overflow: both parts in [2^126, 2^128), |x| from below FLT_MAX to past it
    big = np.ldexp(rng.uniform(1, 2, (2, 200_000)), rng.integers(126, 128, (2, 200_000))).astype(F32)
    x = np.concatenate([cplx(re, im), cplx(big[0], -big[1]), complex_inputs(23)])
    got = run(ApplyOp.MagC32, x)
    exact = np.hypot(x.real.astype(F64), x.imag.astype(F64))
    assert np.any(exact > FMAX) and np.any((exact < FMAX) & (exact > 2.0 ** 127.9))
    check_ulp("MagC32", x, got, exact, 3.0)
    sp = cplx([np.inf, -np.inf, np.nan, np.nan, np.inf, np.nan], [np.nan, np.nan, np.inf, -np.inf, -np.inf, 1.0])
    got = run(ApplyOp.MagC32, sp)
    assert list(got[:5]) == [np.inf] * 5 and np.isnan(got[5])                   # hypot(+-inf, NaN) = +inf


# ---------------------------------------------------------------------------------------------------------------------
# the quadrature demodulator: arg(x[j] * conj(x[j-1])), x[-1] = the carried sample ((0, 0) after reset)

def demod_ref(x, carry=0j):
    """float64 atan2 of the f32 product num_complex forms: re = a*c - b*d, im = a*d + b*c with (c, d) = conj(last),
    each operation rounded to f32 (numpy float32, un-fused).  Returns (phase64, re, im)."""
    last = np.concatenate([np.array([carry], np.complex64), x[:-1]])
    a, b = x.real, x.imag
    c, d = last.real, -last.imag
    with np.errstate(all="ignore"):
        re = a * c - b * d
        im = a * d + b * c
    assert re.dtype == F32
    return np.arctan2(im.astype(F64), re.astype(F64)), re, im


def check_demod(name, x, got, ref):
    """NaN exactly where the reference is NaN, |got - ref| <= DEMOD_BOUND elsewhere.  Returns the largest error."""
    gn, rn = np.isnan(got), np.isnan(ref)
    bad = np.flatnonzero(gn != rn)
    last = np.concatenate([[0j], x[:-1]])
    assert bad.size == 0, f"{name}: {bad.size} NaN mismatches, e.g. x[j-1], x[j] = {last[bad[0]]!r}, " \
                          f"{x[bad[0]]!r} -> {got[bad[0]]!r}, reference {ref[bad[0]]!r}"
    err = np.abs(got[~rn].astype(F64) - ref[~rn])
    i = np.flatnonzero(~rn)[int(np.argmax(err))]
    assert err.max() <= DEMOD_BOUND, f"{name}: error {err.max():.3e} rad (bound {DEMOD_BOUND:.1e}) at x[j-1], x[j] = " \
                                     f"{last[i]!r}, {x[i]!r} -> {got[i]!r}, reference {ref[i]!r}"
    print(f"{name}: max error {err.max():.3e} rad over {(~rn).sum()} outputs")
    return float(err.max())


def after_unit(v):
    """x = (1, 0), v0, (1, 0), v1, ...: every odd output is arg(v_k), every even one arg(conj(v_k))."""
    x = np.empty(2 * v.size, np.complex64)
    x[0::2], x[1::2] = 1, v
    return x


def random_polar(seed, n, lo=-80, hi=70):
    """Independent uniform angles and log2-magnitudes in [lo, hi]: products from 2^-160 to 2^140 -- zero, denormal,
    normal, in (2^126, 2^128), and overflowed."""
    rng = np.random.default_rng(seed)
    th, lm = rng.uniform(-np.pi, np.pi, n), rng.uniform(lo, hi, n)
    return cplx(np.cos(th) * 2.0 ** lm, np.sin(th) * 2.0 ** lm)


def axis_neighbours(v):
    """A part of a unit vector at a multiple of pi/4, moved by a few ulps -- into the denormals when it is 0."""
    if v == 0:
        k = np.arange(9, dtype=F64)
        return np.concatenate([k * 2.0 ** -149, -k * 2.0 ** -149, k[1:] * 2.0 ** -24, -k[1:] * 2.0 ** -24]).astype(F32)
    return neighbours(v, 8)


@gpu
@pytest.mark.parametrize("op", ["QuadDemod", "QuadDemodC32"])
def test_quad_demod_unit_circle_sweep(fb, op):
    from futuresdr_b200.blocks import ApplyOp
    rng = np.random.default_rng(31)
    th = np.concatenate([rng.uniform(-np.pi, np.pi, 2_000_000), np.linspace(-np.pi, np.pi, 1_000_001)])
    v = [cplx(np.cos(th), np.sin(th))]
    for k in range(-4, 5):                           # within a few ulps of every multiple of pi/4
        c, s = np.cos(k * np.pi / 4), np.sin(k * np.pi / 4)
        c, s = (np.round(c), np.round(s)) if k % 2 == 0 else (c, s)
        re, im = np.meshgrid(axis_neighbours(F32(c)), axis_neighbours(F32(s)))
        v.append(cplx(re.ravel(), im.ravel()))
    x = after_unit(np.concatenate(v))
    got = run(getattr(ApplyOp, op), x)
    got = got.real.copy() if op == "QuadDemodC32" else got
    check_demod(f"{op} unit circle", x, got, demod_ref(x)[0])


@gpu
def test_quad_demod_random_magnitudes(fb):
    """Products over the whole f32 range, including the (+-inf, +-inf) and NaN (inf - inf) ones finite samples make."""
    from futuresdr_b200.blocks import ApplyOp
    x = random_polar(32, 3_000_000)
    ref, re, im = demod_ref(x)
    mag = np.maximum(np.abs(re), np.abs(im)).astype(F64)
    cover = {"zero": mag == 0, "denormal": (mag > 0) & (mag < 2.0 ** -126),
             "normal": (mag >= 2.0 ** -126) & (mag <= 2.0 ** 126), "(2^126, 2^128)": (mag > 2.0 ** 126) & (mag <= FMAX),
             "one part inf": np.isinf(re) != np.isinf(im), "(+-inf, +-inf)": np.isinf(re) & np.isinf(im),
             "NaN": np.isnan(ref)}
    for what, m in cover.items():
        assert m.sum() >= 100, what
    check_demod("QuadDemod random magnitudes", x, run(ApplyOp.QuadDemod, x), ref)


@gpu
def test_quad_demod_first_output_after_reset_signed_zeros(fb):
    """The carry starts at (0, 0), so the first product has zero parts whose signs follow v: libm's atan2 of signed
    zeros (atan2(+-0, -0) = +-pi, atan2(+-0, +0) = +-0), bit for bit."""
    from futuresdr_b200.blocks import Apply, ApplyOp
    for op in (ApplyOp.QuadDemod, ApplyOp.QuadDemodC32):
        blk = Apply(op)
        for vr in (1.0, -1.0, 0.0, -0.0):
            for vi in (1.0, -1.0, 0.0, -0.0):
                run(op, random_polar(33, 5), blk=blk)                    # leave a carry behind
                blk.reset()
                x = cplx([vr], [vi])
                got = run(op, x, blk=blk)
                got = got.real.copy() if op == ApplyOp.QuadDemodC32 else got
                ref = demod_ref(x)[0].astype(F32)
                assert _bits(got)[0] == _bits(ref)[0], (op, vr, vi, got[0], ref[0])


@gpu
def test_quad_demod_products_above_2p126(fb):
    """div.approx.f32 returns 0 for divisors in (2^126, 2^128): such products still give their angle."""
    from futuresdr_b200.blocks import ApplyOp
    rng = np.random.default_rng(34)
    th = rng.uniform(-np.pi, np.pi, 500_000)
    u = rng.uniform(0.001, 1.999, th.size)                 # max(|re|, |im|) = 2^(126 + u) after * conj(2^63)
    r = 2.0 ** (63 + u) / np.maximum(np.abs(np.cos(th)), np.abs(np.sin(th)))
    v = cplx(r * np.cos(th), r * np.sin(th))
    x = np.empty(2 * v.size, np.complex64)
    x[0::2], x[1::2] = 2.0 ** 63, v
    x = np.concatenate([cplx([1e19, 1e19], [0.0, 1e19]), x])          # (1e38, 1e38): pi/4
    ref, re, im = demod_ref(x)
    mag = np.maximum(np.abs(re), np.abs(im))[1:]
    assert np.all((mag > 2.0 ** 126) & np.isfinite(mag))
    got = run(ApplyOp.QuadDemod, x)
    assert abs(got[1] - np.pi / 4) <= DEMOD_BOUND, f"(1e38, 1e38) -> {got[1]!r}, not pi/4"
    check_demod("QuadDemod products in (2^126, 2^128)", x, got, ref)


@gpu
def test_quad_demod_overflowed_products(fb):
    """Finite samples whose product overflows both parts give (+-inf, +-inf): +-pi/4 or +-3pi/4, as libm's atan2."""
    from futuresdr_b200.blocks import ApplyOp
    h = 2e19
    quad = cplx([h, h, h, -h, h, -h, h, h], [0, h, 0, h, 0, -h, 0, -h])
    x = np.concatenate([quad, random_polar(35, 400_000, 63, 66)])
    ref, re, im = demod_ref(x)
    both = np.isinf(re) & np.isinf(im)
    assert both.sum() > 10_000
    assert np.array_equal(np.abs(ref[both]), np.where(re[both] > 0, np.pi / 4, 3 * np.pi / 4))
    got = run(ApplyOp.QuadDemod, x)
    assert np.allclose(got[1:8:2], [np.pi / 4, 3 * np.pi / 4, -3 * np.pi / 4, -np.pi / 4], rtol=0, atol=DEMOD_BOUND), \
        f"(+-inf, +-inf) -> {got[1:8:2]}, not pi/4, 3pi/4, -3pi/4, -pi/4"
    check_demod("QuadDemod overflowed products", x, got, ref)


@gpu
def test_quad_demod_nan_products(fb):
    """A NaN part (a NaN or inf sample, or inf - inf from an overflowed product) gives NaN, as libm's atan2 does;
    neighbouring finite products keep their angle."""
    from futuresdr_b200.blocks import ApplyOp
    nan, inf, h = np.nan, np.inf, 1e20
    x = cplx([1, nan, 1, 1, 0.5, nan, 1, inf, 1, 1, inf, -1, h, h, 1, 0, -2, 1],
             [0, 1, 1, nan, 0.5, nan, 0, 0, 0, 0, inf, 0, -h, h, 1, inf, 0, 1])
    x = np.concatenate([x, random_polar(36, 100_000, -20, 20)])
    x.real[1000::997] = nan
    x.imag[1500::991] = nan
    ref = demod_ref(x)[0]
    assert np.isnan(ref).sum() > 100
    got = run(ApplyOp.QuadDemod, x)
    check_demod("QuadDemod NaN products", x, got, ref)


@gpu
def test_quad_demod_c32_real_part_is_the_f32_output(fb):
    from futuresdr_b200.blocks import ApplyOp
    x = random_polar(37, 1_000_000)
    x[::1001] = np.nan
    f = run(ApplyOp.QuadDemod, x)
    c = run(ApplyOp.QuadDemodC32, x)
    assert np.array_equal(_bits(c.real.copy()), _bits(f))
    assert np.all(_bits(c.imag.copy()) == 0)                                     # +0.0, not -0.0


@gpu
@pytest.mark.parametrize("op", ["QuadDemod", "QuadDemodC32"])
def test_quad_demod_ragged_calls_and_reset(fb, op):
    """The carried sample crosses call boundaries of 1, 7 and 4096 items, and reset() puts it back to (0, 0)."""
    from futuresdr_b200.blocks import Apply, ApplyOp
    x = random_polar(38, 300_000, -20, 20)
    ref = demod_ref(x)[0]
    blk = Apply(getattr(ApplyOp, op))
    got = run(None, x, steps=(1, 7, 4096), blk=blk)
    got = got.real.copy() if op == "QuadDemodC32" else got
    check_demod(f"{op} ragged calls", x, got, ref)
    blk.reset()
    y = x[123_456:]
    got = run(None, y, steps=(4096, 1, 7), blk=blk)
    got = got.real.copy() if op == "QuadDemodC32" else got
    check_demod(f"{op} after reset", y, got, demod_ref(y)[0])
