"""PfbChannelizer, PfbSynthesizer and PfbArbResampler exactly, on integer data, at every kernel path.

Samples and taps are small integers (tests/pfb_exact.py), so each block has an exact expectation: PfbArb's outputs
equal the oracle's bit for bit, the channelizer's arm outputs (recovered from each output vector by an f64 FFT) are
the oracle's integers to within 0.25, and the synthesizer's outputs are the oracle's integers to within 0.25.  A wrong
tap, sample, window slot, arm or tile seam moves one of them by a whole unit -- what the tolerance tests of
test_gpu_channelizer.py, test_gpu_synthesizer.py and test_gpu_blocks.py cannot see.

The C ABI is driven directly: every call gets a fresh input slice with NaN in front of it and behind it (every third
call 1 item past a 16-byte boundary, which takes the channelizer off its fused path), and an output buffer pre-filled
with a non-integer sentinel that must survive outside [0, produced) -- for the channelizer on every channel row, with
a row stride larger than the capacity.  Counts are compared with the oracle's call by call.

Non-finite input: +inf, -inf and NaN injected in the window fill, in the first vector after it, at a fused tile seam and
in the last vector of a call must give exactly the oracle's set of non-finite outputs; the finite ones stay exact.
test_every_path_is_reached checks with the profiler that these shapes reach every kernel of the three blocks.
"""
import ctypes as C
import os
import re
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import pfb_exact as px  # noqa: E402

pytestmark = pytest.mark.gpu

SENT = 4097.5                       # not an integer and not a dyadic blend of small integers
ESTATE, EUNSUPPORTED = -6, -5
_f32p = C.POINTER(C.c_float)
S_, I_ = C.c_size_t, C.c_int32


@pytest.fixture(scope="module")
def ctx():
    import torch
    from futuresdr_b200.context import default_context
    assert torch.cuda.is_available()
    return default_context()


def _lib():
    from futuresdr_b200._lib import lib, check
    return lib, check


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _nan_buf(shape, ioff):
    """A NaN-filled buffer and the offset of the slice in it: 2 + ioff items, so that 16 bytes of NaN precede every
    slice and the slice is ioff items past a 16-byte boundary."""
    import torch
    return torch.full(shape, complex(float("nan"), float("nan")), dtype=torch.complex64, device="cuda"), 2 + ioff


def _ptr(t, off=0):
    return C.c_void_p(t.data_ptr() + 8 * off)


def _ioff(k):
    """Call k's slice starts 1 item past a 16-byte boundary for k = 2, 5, 8, ...; aligned otherwise."""
    return 1 if k % 3 == 2 else 0


def _kernels(fn):
    """Names of the kernels fn() launches, from torch.profiler.  A few launches warm the session up first: in a process
    that has already run profiler sessions, the first kernels of a new session were seen missing from its records."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(8):
            torch.ones(1 << 20, device="cuda").sum().item()
        fn()
        torch.cuda.synchronize()
    return {e.key for e in prof.key_averages()}


def _plan(create, env, monkeypatch):
    """create(h) under the A/B switch `env` (read at plan time)."""
    if env:
        monkeypatch.setenv(env, "1")
    else:
        for v in ("B2S_CHAN_NO_FUSED", "B2S_SYNTH_NO_FUSED", "B2S_PFBARB_NO_PERIODIC"):
            monkeypatch.delenv(v, raising=False)
    h = C.c_void_p()
    create(h)
    if env:
        monkeypatch.delenv(env)
    return h


# ---- channelizer ----------------------------------------------------------------------------------------------------
class _Chan:
    def __init__(self, ctx, N, taps, osr, nofused, monkeypatch):
        lib, check = _lib()
        t = np.ascontiguousarray(taps, np.float32)
        self.lib, self.ctx, self.N = lib, ctx, N
        self.h = _plan(lambda h: check(lib.b2s_chan_plan_c32(ctx.handle, N, t.ctypes.data_as(_f32p), t.size, float(osr),
                                                             C.byref(h)), ctx.handle),
                       "B2S_CHAN_NO_FUSED" if nofused else None, monkeypatch)

    def close(self):
        self.lib.b2s_chan_destroy(self.h)

    def call(self, xd, pos, avail, cap, ioff):
        import torch
        N = self.N
        buf, f = _nan_buf((ioff + avail + 6,), ioff)
        buf[f:f + avail] = xd[pos:pos + avail]
        S = cap + 3                                              # row stride > capacity
        out = torch.full((N * S + 8,), SENT, dtype=torch.complex64, device="cuda")
        c, p, ca = S_(), S_(), I_()
        rc = self.lib.b2s_chan_exec(self.h, _ptr(buf, f), avail, _ptr(out), S, cap, C.byref(c), C.byref(p), C.byref(ca))
        self.ctx.sync()
        o = out.cpu().numpy()
        rows = o[:N * S].reshape(N, S)
        intact = bool(np.all(rows[:, p.value:] == SENT) and np.all(o[N * S:] == SENT))
        return rc, (c.value, p.value, bool(ca.value)), rows[:, :p.value], intact


def _check_chan_call(k, call, rc, counts, y, intact):
    pos, avail, cap, want, (_, fin, arms) = call
    what = dict(call=k, pos=pos, avail=avail, cap=cap)
    assert rc == 0 and counts == want, (what, rc, counts, want)
    assert intact, ("wrote outside [0, produced) of a channel row", what)
    got_fin = np.isfinite(y)
    assert np.array_equal(got_fin, fin), ("non-finite outputs differ", what, np.argwhere(got_fin != fin)[:8])
    cols = np.flatnonzero(fin.all(axis=0))
    if cols.size:
        err = np.abs(px.chan_arms(y[:, cols]) - arms[:, cols])
        assert float(err.max()) <= 0.25, ("arm outputs", what, float(err.max()), np.argwhere(err > 0.25)[:8])


def _chan_case(ctx, monkeypatch, N, T, osr, nofused, x, taps, steps):
    calls = px.chan_run(N, taps, osr, x, steps)
    ch = _Chan(ctx, N, taps, osr, nofused, monkeypatch)
    try:
        xd = _dev(x)
        for k, call in enumerate(calls):
            pos, avail, cap = call[:3]
            _check_chan_call(k, call, *ch.call(xd, pos, avail, cap, ioff=_ioff(k)))
    finally:
        ch.close()
    return calls


@pytest.mark.parametrize("N,T,osr,nofused", px.CHAN_SHAPES)
def test_channelizer_exact(ctx, monkeypatch, N, T, osr, nofused):
    rng, taps, D = px.chan_case(N, T, osr, seed=N * 100 + T)
    x = px.int_samples(rng, N * T + px.chan_vectors(N, T, D) * D + D // 2, True, lim=px.LIM)
    for name, steps in px.chan_patterns(N, T, D).items():
        _chan_case(ctx, monkeypatch, N, T, osr, nofused, x, taps, steps)


def test_channelizer_unaligned_input_leaves_the_fused_path(ctx, monkeypatch):
    """The fused kernel copies its tile with 16-byte loads: a slice 1 item past a 16-byte boundary takes the generic
    bank, an aligned one the fused kernel."""
    N, T = 64, 5
    rng, taps, D = px.chan_case(N, T, 1.0, seed=9)
    x = px.int_samples(rng, N * T + 200 * N, True, lim=px.LIM)
    calls = px.chan_run(N, taps, 1.0, x, [(N * T, 1 << 40)])
    xd = _dev(x)
    seen = {0: set(), 1: set()}
    for ioff, expect in ((0, "chan_fused_kernel"), (1, "chan_bank_kernel")):
        # A profiler session now and then lacks the records of some kernels that ran, so the call is repeated on a
        # fresh plan (up to three sessions) until the expected kernel shows; every session counts for the asserts.
        for _ in range(3):
            ch = _Chan(ctx, N, taps, 1.0, False, monkeypatch)
            try:
                _check_chan_call(0, calls[0], *ch.call(xd, *calls[0][:3], ioff=ioff))
                seen[ioff] |= _kernels(lambda: _check_chan_call(1, calls[1], *ch.call(xd, *calls[1][:3], ioff=ioff)))
            finally:
                ch.close()
            if any(expect in n for n in seen[ioff]):
                break
    assert any("chan_fused_kernel" in n for n in seen[0])
    assert not any("chan_fused_kernel" in n for n in seen[1])
    assert any("chan_bank_kernel" in n for n in seen[1])


# ---- synthesizer ----------------------------------------------------------------------------------------------------
class _Synth:
    def __init__(self, ctx, N, taps, nofused, monkeypatch):
        lib, check = _lib()
        t = np.ascontiguousarray(taps, np.float32)
        self.lib, self.ctx, self.N = lib, ctx, N
        self.h = _plan(lambda h: check(lib.b2s_synth_plan_c32(ctx.handle, N, t.ctypes.data_as(_f32p), t.size,
                                                              C.byref(h)), ctx.handle),
                       "B2S_SYNTH_NO_FUSED" if nofused else None, monkeypatch)

    def close(self):
        self.lib.b2s_synth_destroy(self.h)

    def call(self, xd, pos, avail, cap, ioff):
        import torch
        N = self.N
        S = ioff + avail + 5                                     # stream w at w * S: NaN in front of and behind each
        buf, f = _nan_buf((N, S), ioff)
        buf[:, f:f + avail] = xd[:, pos:pos + avail]
        out = torch.full((cap + 8,), SENT, dtype=torch.complex64, device="cuda")
        c, p = S_(), S_()
        rc = self.lib.b2s_synth_exec(self.h, _ptr(buf, f), S, avail, _ptr(out), cap, C.byref(c), C.byref(p))
        self.ctx.sync()
        o = out.cpu().numpy()
        return rc, (c.value, p.value, False), o[:p.value], bool(np.all(o[p.value:] == SENT))


def _check_synth_call(k, call, rc, counts, z, intact):
    pos, avail, cap, want, (_, fin, zi) = call
    what = dict(call=k, pos=pos, avail=avail, cap=cap)
    assert rc == 0 and counts == want, (what, rc, counts, want)
    assert intact, ("wrote outside [0, produced)", what)
    got_fin = np.isfinite(z)
    assert np.array_equal(got_fin, fin), ("non-finite outputs differ", what, np.flatnonzero(got_fin != fin)[:8])
    if fin.any():
        err = np.abs(z[fin].astype(np.complex128) - zi[fin])
        assert float(err.max()) <= 0.25, ("outputs", what, float(err.max()), np.flatnonzero(fin)[err > 0.25][:8])


def _synth_case(ctx, monkeypatch, N, T, nofused, x, taps, steps):
    calls = px.synth_run(N, taps, x, steps)
    sy = _Synth(ctx, N, taps, nofused, monkeypatch)
    try:
        xd = _dev(x)
        for k, call in enumerate(calls):
            pos, avail, cap = call[:3]
            _check_synth_call(k, call, *sy.call(xd, pos, avail, cap, ioff=_ioff(k)))
    finally:
        sy.close()
    return calls


@pytest.mark.parametrize("N,T,nofused", px.SYNTH_SHAPES)
def test_synthesizer_exact(ctx, monkeypatch, N, T, nofused):
    rng, taps = px.synth_case(N, T, seed=N * 100 + T)
    x, _ = px.synth_inputs(rng, N, px.synth_vectors(N, T))
    for name, steps in px.synth_patterns(N, T).items():
        _synth_case(ctx, monkeypatch, N, T, nofused, x, taps, steps)


@pytest.mark.parametrize("N,T", [(64, 5), (64, 16), (256, 32), (4, 3)])
def test_synthesizer_many_tiles_per_cta_exact(ctx, monkeypatch, N, T):
    """One call over more tiles than CTAs (each CTA carries its ring across several tiles; 256 x 32 warms up over two
    tiles because a tile is shorter than the history)."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rng, taps = px.synth_case(N, T, seed=7 * N + T)
    x, _ = px.synth_inputs(rng, N, T + px.synth_lead(N, T) + (4 * sms + 3) * px.fused_ob(N) + 5)
    _synth_case(ctx, monkeypatch, N, T, False, x, taps, [(T, 1 << 40)])


# ---- PfbArbResampler ------------------------------------------------------------------------------------------------
class _Arb:
    def __init__(self, ctx, N, taps, rate, periodic, monkeypatch):
        lib, check = _lib()
        t = np.ascontiguousarray(taps, np.float32)
        self.lib, self.ctx = lib, ctx
        self.h = _plan(lambda h: check(lib.b2s_pfbarb_plan_c32(ctx.handle, t.ctypes.data_as(_f32p), t.size, N,
                                                               float(rate), C.byref(h)), ctx.handle),
                       None if periodic else "B2S_PFBARB_NO_PERIODIC", monkeypatch)

    def close(self):
        self.lib.b2s_pfbarb_destroy(self.h)

    def call(self, xd, pos, avail, cap, ioff):
        import torch
        buf, f = _nan_buf((ioff + avail + 6,), ioff)
        buf[f:f + avail] = xd[pos:pos + avail]
        out = torch.full((cap + 8,), SENT, dtype=torch.complex64, device="cuda")
        c, p, ca = S_(), S_(), I_()
        rc = self.lib.b2s_pfbarb_exec(self.h, _ptr(buf, f), avail, _ptr(out), cap, C.byref(c), C.byref(p), C.byref(ca))
        self.ctx.sync()
        o = out.cpu().numpy()
        return rc, (c.value, p.value, bool(ca.value)), o[:p.value], bool(np.all(o[p.value:] == SENT))


def _same(got, ref):
    """Values equal (-0.0 == 0.0), the same outputs non-finite."""
    fin = np.isfinite(ref)
    return (got.size == ref.size and np.array_equal(np.isfinite(got), fin)
            and np.array_equal(got[fin], ref[fin]))


def _arb_case(ctx, monkeypatch, N, T, rate, periodic, x, taps, steps):
    calls = px.pfbarb_run(rate, N, taps, x, steps)
    arb = _Arb(ctx, N, taps, rate, periodic, monkeypatch)
    try:
        _arb_calls(arb, x, calls)
    finally:
        arb.close()
    return calls


def _arb_calls(arb, x, calls):
    xd = _dev(x)
    for k, (pos, avail, cap, want, out) in enumerate(calls):
        rc, counts, y, intact = arb.call(xd, pos, avail, cap, ioff=_ioff(k))
        what = dict(call=k, pos=pos, avail=avail, cap=cap)
        assert intact, ("wrote outside [0, produced)", what)
        if want is None:                                   # the reference would overrun its slice: refused, no commit
            assert rc == ESTATE and counts[:2] == (0, 0), (what, rc, counts)
            continue
        assert rc == 0 and counts == want, (what, rc, counts, want)
        assert _same(y, out[0]), (what, np.flatnonzero(y != out[0])[:8])


@pytest.mark.parametrize("N,T,rate,periodic", px.PFBARB_SHAPES + px.PFBARB_HIGH_SHAPES)
def test_pfbarb_exact(ctx, monkeypatch, N, T, rate, periodic):
    """Rates above the arm count are checked against px.ArbRef (pfbarb_run picks it), which saturates the arm index
    like the reference."""
    taps, x = px.pfbarb_case(N, T, rate, seed=N + T + int(rate * 1000))
    for name, steps in px.pfbarb_patterns(rate, N, T, x.size - T).items():
        _arb_case(ctx, monkeypatch, N, T, rate, periodic, x, taps, steps)


@pytest.mark.parametrize("N,rate", [(32, 126.0), (32, 122.5), (1, 64.0)])
def test_pfbarb_plan_refuses_rates_the_descriptor_tile_cannot_hold(ctx, N, rate):
    """Above the arm count one sample can produce ceil(rate * (1 + 1/N)) outputs; shapes whose 32-sample sub-block would
    overflow a CTA's descriptor tile are refused at plan time, not when a call runs."""
    from futuresdr_b200._lib import B200SdrError
    lib, check = _lib()
    t = np.ones(N * 3, np.float32)
    h = C.c_void_p()
    with pytest.raises(B200SdrError) as e:
        check(lib.b2s_pfbarb_plan_c32(ctx.handle, t.ctypes.data_as(_f32p), t.size, N, rate, C.byref(h)), ctx.handle)
    assert e.value.code == EUNSUPPORTED and not h.value


def test_plans_refuse_windows_larger_than_shared_memory(ctx):
    """The window slide stages one window in shared memory: longer windows are refused when the plan is made."""
    import torch
    from futuresdr_b200._lib import B200SdrError
    lib, check = _lib()
    T = torch.cuda.get_device_properties(0).shared_memory_per_block_optin // 8 + 1
    t = np.ones(2 * T, np.float32)
    for create in (lambda h: lib.b2s_pfbarb_plan_c32(ctx.handle, t.ctypes.data_as(_f32p), t.size, 2, 1.0, C.byref(h)),
                   lambda h: lib.b2s_synth_plan_c32(ctx.handle, 2, t.ctypes.data_as(_f32p), t.size, C.byref(h))):
        h = C.c_void_p()
        with pytest.raises(B200SdrError) as e:
            check(create(h), ctx.handle)
        assert e.value.code == EUNSUPPORTED and not h.value


# ---- non-finite input -----------------------------------------------------------------------------------------------
BAD = [float("inf"), float("-inf"), float("nan")]


@pytest.mark.parametrize("bad", BAD, ids=["inf", "-inf", "nan"])
@pytest.mark.parametrize("N,T", [(64, 5), (16, 12), (8, 20), (64, 32), (6, 3)])
def test_channelizer_non_finite(ctx, monkeypatch, N, T, bad):
    """One bad sample in the fill, in the first vector after it, at a fused tile seam and in the last vector of a call
    (it stays in the history for the next call)."""
    rng, taps, D = px.chan_case(N, T, 1.0, seed=5 * N + T)
    ob = px.fused_ob(N)
    x = px.int_samples(rng, N * T + (px.chan_vectors(N, T, D) + 2 * ob + 2 * T) * D, True, lim=px.LIM)
    steps = px.chan_patterns(N, T, D)["ragged"]
    calls = px.chan_run(N, taps, 1.0, x, steps)
    q = next(c[0] for c in calls if c[3][1])
    pos, c_all = calls[-2][0], calls[-2][3][0]             # the last call: an aligned one, fused where the shape is
    seam = min(pos + (T - 1 + ob) * D + 3, pos + c_all - 1)   # its first fused tile seam
    last = calls[3][0] + calls[3][3][0] - 2               # the last vector of the call of T-1 vectors
    x = x.copy()
    for i in (0, q + 1, seam, last):
        x[i] = complex(bad, 1.0) if i % 2 else complex(2.0, bad)
    _chan_case(ctx, monkeypatch, N, T, 1.0, False, x, taps, steps)


@pytest.mark.parametrize("bad", BAD, ids=["inf", "-inf", "nan"])
@pytest.mark.parametrize("N,T", [(64, 5), (16, 12), (8, 20), (256, 32), (5, 3)])
def test_synthesizer_non_finite(ctx, monkeypatch, N, T, bad):
    rng, taps = px.synth_case(N, T, seed=5 * N + T)
    x, _ = px.synth_inputs(rng, N, px.synth_vectors(N, T) + px.synth_lead(N, T) + 2 * px.fused_ob(N))
    steps = px.synth_patterns(N, T)["ragged"]
    calls = px.synth_run(N, taps, x, steps)
    ob, lead = px.fused_ob(N), px.synth_lead(N, T)
    fill = 0
    first = T                                              # the first vector after the fill (inside call 2)
    last = calls[3][0] + calls[3][3][0] - 1                # the last vector of the call of T-1 vectors
    seam = calls[-2][0] + lead + ob                        # a tile seam of the last steady call
    x = x.copy()
    for v, ch in ((fill, 1), (first, 0), (last, N - 1), (min(seam, x.shape[1] - 1), N // 2)):
        x[ch, v] = complex(bad, 0.5)
    _synth_case(ctx, monkeypatch, N, T, False, x, taps, steps)


@pytest.mark.parametrize("bad", BAD, ids=["inf", "-inf", "nan"])
@pytest.mark.parametrize("N,T,rate", [(32, 5, 2.37), (32, 5, 0.768), (64, 300, 1.0)])
def test_pfbarb_non_finite(ctx, monkeypatch, N, T, rate, bad):
    taps, x = px.pfbarb_case(N, T, rate, seed=11 * N + T)
    steps = px.pfbarb_patterns(rate, N, T, x.size - T)["ragged"]
    calls = px.pfbarb_run(rate, N, taps, x, steps)
    last = calls[3][0] + calls[3][3][0] - 1                # the last sample of a call that leaves Boundary pending
    x = x.copy()
    for i in (1, T, last, T + 1024, T + 2048):             # fill, first steady sample, call end, CTA seams
        x[i] = complex(bad, 1.0)
    for periodic in (True, False):
        _arb_case(ctx, monkeypatch, N, T, rate, periodic, x, taps, steps)


# ---- the sweep reaches every kernel ---------------------------------------------------------------------------------
def test_every_path_is_reached(ctx, monkeypatch):
    """A representative subset of the shapes above under the profiler: the fused channelizer and synthesizer at every
    TPAD, padded (T < TPAD) and not, the generic banks, the window kernels, the radix and Bluestein FFTs and pfb_kernel."""
    def run():
        for N, T in ((64, 5), (64, 12), (64, 16), (64, 20), (6, 3)):
            rng, taps, D = px.chan_case(N, T, 1.0, seed=N + T)
            x = px.int_samples(rng, N * T + px.chan_vectors(N, T, D) * D, True, lim=px.LIM)
            _chan_case(ctx, monkeypatch, N, T, 1.0, False, x, taps, px.chan_patterns(N, T, D)["ragged"])
        for N, T in ((64, 5), (64, 12), (64, 16), (64, 20), (5, 3)):
            rng, taps = px.synth_case(N, T, seed=N + T)
            x, _ = px.synth_inputs(rng, N, px.synth_vectors(N, T))
            _synth_case(ctx, monkeypatch, N, T, False, x, taps, px.synth_patterns(N, T)["ragged"])
        taps, x = px.pfbarb_case(32, 5, 2.37, seed=1)
        _arb_case(ctx, monkeypatch, 32, 5, 2.37, True, x, taps, [])
    names = _kernels(run)
    found = set()
    for n in names:
        m = re.search(r"(chan|synth)_fused_kernel<\d+, (\d+), (true|false)>", n)
        if m:
            found |= {(m.group(1), int(m.group(2))), (m.group(1), m.group(3))}
        for k in ("chan_bank_kernel", "synth_bank_kernel", "pfb_push_kernel", "pfb_slide_kernel", "pfb_transpose_kernel",
                  "pfb_kernel", "fft_kernel", "bluestein_kernel"):
            if re.search(r"\b" + k + r"\b", n):
                found.add((k,))
    want = {(b, t) for b in ("chan", "synth") for t in (8, 16, 32, "true", "false")}   # every TPAD, padded or not
    want |= {(k,) for k in ("chan_bank_kernel", "synth_bank_kernel", "pfb_push_kernel", "pfb_slide_kernel",
                            "pfb_transpose_kernel", "pfb_kernel", "fft_kernel", "bluestein_kernel")}
    assert want <= found, (sorted(want - found), sorted(n for n in names if "kernel" in n))
