"""Every buffer and sub-plan an object allocates is owned by it: b2s_ctx_bytes_held rises when the object is created
and when an exec grows one of its workspaces, and returns exactly to its baseline when the object is destroyed.
Creates refused for bad arguments hold nothing and leave the out-handle NULL."""
import ctypes as C

import numpy as np
import pytest
import torch

from futuresdr_b200 import _lib
from futuresdr_b200._lib import lib, check
from futuresdr_b200.context import Context

pytestmark = pytest.mark.gpu


@pytest.fixture
def ctx():
    c = Context(own_stream=True)
    yield c
    c.close()


def _f32(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a, a.ctypes.data_as(_lib._f32p)


def _dev(n, dtype=torch.complex64):
    t = torch.zeros(n, dtype=dtype, device="cuda")
    torch.cuda.synchronize()                   # the context's own stream is not ordered after torch's
    return C.c_void_p(t.data_ptr()), t


def _taps(n, seed=1):
    return np.random.default_rng(seed).standard_normal(n).astype(np.float32) / n


def _lifecycle(ctx, create, destroy, run=None, grows=False):
    """create(h) -> create the object into h; run(h) -> one exec that may grow workspaces."""
    base = ctx.bytes_held
    h = C.c_void_p()
    check(create(h), ctx.handle)
    created = ctx.bytes_held
    assert created > base
    if run is not None:
        run(h)
        ctx.sync()
        if grows:
            assert ctx.bytes_held > created
        else:
            assert ctx.bytes_held == created
    destroy(h)
    assert ctx.bytes_held == base
    return created - base


S, I = C.c_size_t, C.c_int32


def _fir_exec(n, dtype=torch.complex64):
    def run(h):
        (di, _ki), (do, _ko) = _dev(n, dtype), _dev(n, dtype)
        c, p, st = S(), S(), I()
        check(lib.b2s_fir_exec(h, di, n, do, n, C.byref(c), C.byref(p), C.byref(st)))
    return run


@pytest.mark.parametrize("algo,kind,ntaps", [(_lib.ALGO_DIRECT, _lib.C32_F32, 16), (_lib.ALGO_TENSOR, _lib.F32_F32, 64),
                                             (_lib.ALGO_FFT, _lib.C32_F32, 300)])
def test_fir(ctx, algo, kind, ntaps):
    t, tp = _f32(_taps(ntaps))

    def create(h):
        rc = lib.b2s_fir_plan(ctx.handle, kind, tp, ntaps, 1, C.byref(h))
        return rc or lib.b2s_fir_set_algo(h, algo)
    dtype = torch.float32 if kind == _lib.F32_F32 else torch.complex64
    _lifecycle(ctx, create, lib.b2s_fir_destroy, _fir_exec(1 << 20, dtype))


def test_fir_f64(ctx):
    t = np.ascontiguousarray(np.arange(1, 33, dtype=np.float64))
    held = _lifecycle(ctx, lambda h: lib.b2s_fir_plan_f64_f64(ctx.handle, t.ctypes.data_as(C.POINTER(C.c_double)), t.size,
                                                               2, C.byref(h)),
                      lib.b2s_fir_destroy, _fir_exec(1 << 16, torch.float64))
    assert held == 32 * 8                                          # the reversed f64 taps and nothing else


@pytest.mark.parametrize("interp,decim,ntaps,sliding", [(3, 2, 24, True), (200, 199, 800, False)])
def test_resampler(ctx, interp, decim, ntaps, sliding):
    t, tp = _f32(_taps(ntaps))

    def run(h):
        (di, _ki), (do, _ko) = _dev(1 << 18), _dev(1 << 18)
        c, p, st = S(), S(), I()
        check(lib.b2s_resamp_exec(h, di, 1 << 18, do, 1 << 18, C.byref(c), C.byref(p), C.byref(st)))
    held = _lifecycle(ctx, lambda h: lib.b2s_resamp_plan(ctx.handle, _lib.C32_F32, tp, ntaps, interp, decim, C.byref(h)),
                      lib.b2s_resamp_destroy, run)
    banks = interp * ((ntaps // interp) | 1) * 4
    assert (held > banks) if sliding else (held == banks)


@pytest.mark.parametrize("n", [1024, 1000, 65536, 10007])     # shared memory, Bluestein, four-step, four-step Bluestein
def test_fft(ctx, n):
    def run(h):
        (di, _ki), (do, _ko) = _dev(2 * n), _dev(2 * n)
        c, p = S(), S()
        check(lib.b2s_fft_exec(h, di, 2 * n, do, 2 * n, C.byref(c), C.byref(p)))
    _lifecycle(ctx, lambda h: lib.b2s_fft_plan_c32(ctx.handle, n, 0, 1, 0, 1.0, C.byref(h)), lib.b2s_fft_destroy, run)


def _env(monkeypatch, name, on):
    if on:
        monkeypatch.setenv(name, "1")
    else:
        monkeypatch.delenv(name, raising=False)


@pytest.mark.parametrize("fused", [True, False])
def test_channelizer(ctx, monkeypatch, fused):
    _env(monkeypatch, "B2S_CHAN_NO_FUSED", not fused)
    N, T, n = 16, 4, 1 << 16
    t, tp = _f32(_taps(N * T))
    (di, _ki), (do, _ko) = _dev(n), _dev(n)

    def create(h):
        rc = lib.b2s_chan_plan_c32(ctx.handle, N, tp, N * T, 1.0, C.byref(h))
        if rc == 0:                                               # fill the windows: no workspace yet
            c, p, again = S(), S(), I()
            check(lib.b2s_chan_exec(h, di, n, do, n // N, n // N, C.byref(c), C.byref(p), C.byref(again)))
        return rc

    def run(h):
        c, p, again = S(), S(), I()
        check(lib.b2s_chan_exec(h, di, n, do, n // N, n // N, C.byref(c), C.byref(p), C.byref(again)))
        assert p.value > 0
    _lifecycle(ctx, create, lib.b2s_chan_destroy, run, grows=True)


@pytest.mark.parametrize("fused", [True, False])
def test_synthesizer(ctx, monkeypatch, fused):
    _env(monkeypatch, "B2S_SYNTH_NO_FUSED", not fused)
    N, T, n = 16, 4, 1 << 12
    t, tp = _f32(_taps(N * T))

    def run(h):
        (di, _ki), (do, _ko) = _dev(N * n), _dev(N * n)
        c, p = S(), S()
        check(lib.b2s_synth_exec(h, di, n, n, do, N * n, C.byref(c), C.byref(p)))
    _lifecycle(ctx, lambda h: lib.b2s_synth_plan_c32(ctx.handle, N, tp, N * T, C.byref(h)), lib.b2s_synth_destroy, run,
               grows=True)


@pytest.mark.parametrize("periodic", [True, False])
def test_pfbarb(ctx, monkeypatch, periodic):
    _env(monkeypatch, "B2S_PFBARB_NO_PERIODIC", not periodic)
    t, tp = _f32(_taps(32 * 8))
    n = 1 << 16
    (di, _ki), (do, _ko) = _dev(n), _dev(2 * n)

    def call(h):
        c, p, again = S(), S(), I()
        check(lib.b2s_pfbarb_exec(h, di, n, do, 2 * n, C.byref(c), C.byref(p), C.byref(again)))
        return p.value

    def create(h):
        rc = lib.b2s_pfbarb_plan_c32(ctx.handle, tp, t.size, 32, 0.768, C.byref(h))
        if rc == 0:
            assert call(h) == 0                                   # fills the filter history
        return rc

    def run(h):
        assert call(h) > 0
    _lifecycle(ctx, create, lib.b2s_pfbarb_destroy, run, grows=not periodic)


@pytest.mark.parametrize("a,b,algo,grows", [([0.5], [0.25, 0.25], _lib.ALGO_SCAN, True),
                                            ([0.5], [0.25, 0.25], _lib.ALGO_DIRECT, False),
                                            ([], [0.25, 0.5, 0.25], _lib.ALGO_AUTO, False)])
def test_iir(ctx, a, b, algo, grows):
    a, ap = _f32(a)
    b, bp = _f32(b)

    def create(h):
        rc = lib.b2s_iir_plan_f32(ctx.handle, ap, a.size, bp, b.size, C.byref(h))
        return rc or lib.b2s_iir_set_algo(h, algo)

    def run(h):
        (di, _ki), (do, _ko) = _dev(1 << 20, torch.float32), _dev(1 << 20, torch.float32)
        c, p, st = S(), S(), I()
        check(lib.b2s_iir_exec(h, di, 1 << 20, do, 1 << 20, C.byref(c), C.byref(p), C.byref(st)))
    held = _lifecycle(ctx, create, lib.b2s_iir_destroy, run, grows=grows)
    if not a.size:
        assert held > 4 + 3 * 4 + 4                                 # a, b, memory, and the FIR sub-plan's taps


@pytest.mark.parametrize("staging", [1, 0])
def test_ring(ctx, staging):
    held = _lifecycle(ctx, lambda h: lib.b2s_ring_create(ctx.handle, 8, 4096, 256, 3, staging, C.byref(h)),
                      lib.b2s_ring_destroy)
    device = 3 * (2048 + 32768) + 256
    assert held == device + (3 * 32768 if staging else 0)


def test_rotator(ctx):
    def run(h):
        (di, _ki), (do, _ko) = _dev(1 << 20), _dev(1 << 20)
        n, st = S(), I()
        check(lib.b2s_rotator_exec(h, di, 1 << 20, do, 1 << 20, C.byref(n), C.byref(st)))
    _lifecycle(ctx, lambda h: lib.b2s_rotator_create(ctx.handle, 0.01, C.byref(h)), lib.b2s_rotator_destroy, run,
               grows=True)


def test_signal_source(ctx):
    def run(h):
        (do, _ko) = _dev(1 << 16, torch.float32)
        p = S()
        check(lib.b2s_sigsrc_exec(h, do, 1 << 16, C.byref(p)))
    _lifecycle(ctx, lambda h: lib.b2s_sigsrc_create(ctx.handle, _lib.WAVE_SIN, 0, 1000.0, 48000.0, 1.0, 0.0, C.byref(h)),
               lib.b2s_sigsrc_destroy, run)


def test_moving_avg(ctx):
    def run(h):
        (di, _ki), (do, _ko) = _dev(1 << 16, torch.float32), _dev(1 << 16, torch.float32)
        c, p = S(), S()
        check(lib.b2s_mavg_exec(h, di, 1 << 16, do, 1 << 16, C.byref(c), C.byref(p)))
    _lifecycle(ctx, lambda h: lib.b2s_mavg_create(ctx.handle, 1024, 0.1, 4, C.byref(h)), lib.b2s_mavg_destroy, run)


def test_apply(ctx):
    def run(h):
        (di, _ki), (do, _ko) = _dev(1 << 16), _dev(1 << 16, torch.float32)
        c, p = S(), S()
        check(lib.b2s_apply_exec(h, di, 1 << 16, do, 1 << 16, C.byref(c), C.byref(p)))
    _lifecycle(ctx, lambda h: lib.b2s_apply_create(ctx.handle, _lib.OP_QUAD_DEMOD, 1.0, C.byref(h)),
               lib.b2s_apply_destroy, run)


def test_spectrum(ctx):
    n = 1024

    def run(h):
        (di, _ki), (do, _ko) = _dev(256 * n), _dev(256 * n, torch.float32)
        c, p = S(), S()
        check(lib.b2s_spectrum_exec(h, di, 256 * n, do, 256 * n, C.byref(c), C.byref(p)))
    _lifecycle(ctx, lambda h: lib.b2s_spectrum_plan(ctx.handle, n, 1, 0.1, 1, 0.0, C.byref(h)),
               lib.b2s_spectrum_destroy, run, grows=True)


def test_refused_creates_hold_nothing(ctx):
    t, tp = _f32(_taps(12))
    base = ctx.bytes_held
    refused = [
        lambda h: lib.b2s_fir_plan(ctx.handle, _lib.C32_F32, tp, 0, 1, C.byref(h)),
        lambda h: lib.b2s_resamp_plan(ctx.handle, _lib.C32_F32, tp, 12, 5, 1, C.byref(h)),
        lambda h: lib.b2s_fft_plan_c32(ctx.handle, 1, 0, 0, 0, 1.0, C.byref(h)),
        lambda h: lib.b2s_pfbarb_plan_c32(ctx.handle, tp, 12, 32, 1.5, C.byref(h)),
        lambda h: lib.b2s_chan_plan_c32(ctx.handle, 2, tp, 12, 1.0, C.byref(h)),
        lambda h: lib.b2s_synth_plan_c32(ctx.handle, 1, tp, 12, C.byref(h)),
        lambda h: lib.b2s_iir_plan_f32(ctx.handle, tp, 1, tp, 0, C.byref(h)),
        lambda h: lib.b2s_mavg_create(ctx.handle, 16, 2.0, 1, C.byref(h)),
        lambda h: lib.b2s_spectrum_plan(ctx.handle, 1000, 1, 0.1, 1, 0.0, C.byref(h)),
        lambda h: lib.b2s_apply_create(ctx.handle, 99, 1.0, C.byref(h)),
        lambda h: lib.b2s_sigsrc_create(ctx.handle, 7, 0, 1.0, 1.0, 1.0, 0.0, C.byref(h)),
        lambda h: lib.b2s_ring_create(ctx.handle, 8, 1024, 0, 0, 0, C.byref(h)),
    ]
    for create in refused:
        h = C.c_void_p(1)
        assert create(h) < 0
        assert not h.value
        assert ctx.bytes_held == base
