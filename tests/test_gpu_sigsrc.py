"""SignalSource (csrc/sigsrc.cu) and Head on the GPU against the CPU oracle (tests/sigsrc_oracle.py, the restatement of
src/blocks/signal_source/*.rs).  The phase is an exact wrapping integer, so every comparison is bit for bit (as
uint32), at any stream length."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sigsrc_oracle as orc  # noqa: E402  (tests/sigsrc_oracle.py)

pytestmark = pytest.mark.gpu

N_BIG = 64 << 20
FS = 48000.0
FREQS = {"1k": 1000.0, "48k": 48000.0, "fs4": FS / 4, "fs64": FS / 64, "neg3k": -3000.0}
WAVES = {"cos": orc.COS, "sin": orc.SIN, "square": orc.SQUARE}


def fb():
    import futuresdr_b200 as m
    return m


def u32(x):
    if isinstance(x, torch.Tensor):
        x = x.cpu().numpy()
    return np.ascontiguousarray(x).view(np.uint32)


def make(wave, f, amp, ph0, dtype):
    return fb().SignalSource(wave, f, FS, amp, ph0, dtype)


@pytest.mark.parametrize("dtype", [np.float32, np.complex64], ids=["f32", "c32"])
@pytest.mark.parametrize("wave", list(WAVES))
@pytest.mark.parametrize("freq", list(FREQS))
def test_one_big_call_bit_equal(wave, freq, dtype):
    """64 Mi items in one call equal the oracle bit for bit, and the phase afterwards is the oracle's."""
    src = make(WAVES[wave], FREQS[freq], 0.7, 0.3, dtype)
    out = torch.empty(N_BIG, dtype=torch.complex64 if dtype == np.complex64 else torch.float32, device="cuda")
    assert src.generate(out) == N_BIG
    ref = orc.Source(WAVES[wave], FREQS[freq], FS, 0.7, 0.3, dtype)
    want = ref.work(N_BIG)
    got = u32(out)
    bad = np.nonzero(got != want.view(np.uint32))[0]
    assert bad.size == 0, (bad.size, bad[:8])
    ph, inc = src.phase()
    assert (ph.value, inc.value) == (ref.phase.value, ref.inc)


@pytest.mark.parametrize("dtype", [np.float32, np.complex64], ids=["f32", "c32"])
@pytest.mark.parametrize("wave", list(WAVES))
def test_ragged_calls_equal_one_call(wave, dtype):
    """Calls of 0, 1, 3, 4095 and 2^20 + 7 items into slices that start one item past an aligned address produce the
    single call's items bit for bit; the NCO phase after every call is the oracle's.  The gap items around the slices
    keep a guard pattern, so a head or tail item written one slot early or late is caught."""
    sizes = [0, 1, 3, 4095, (1 << 20) + 7, 5, 0, 2]
    total = sum(sizes)
    tdt = torch.complex64 if dtype == np.complex64 else torch.float32
    one = make(WAVES[wave], 1000.0, 0.5, -1.0, dtype)
    whole = torch.empty(total, dtype=tdt, device="cuda")
    one.generate(whole)
    src = make(WAVES[wave], 1000.0, 0.5, -1.0, dtype)
    ref = orc.Source(WAVES[wave], 1000.0, FS, 0.5, -1.0, dtype)
    guard = np.uint32(0xA5A5A5A5)
    words = (total + len(sizes) + 1) * (2 if dtype == np.complex64 else 1)
    buf = torch.from_numpy(np.full(words, guard, np.uint32).view(dtype)).cuda()
    pos, pieces, gaps = 1, [], [0]
    for n in sizes:
        assert src.generate(buf[pos:pos + n]) == n
        pieces.append(buf[pos:pos + n])
        ref.work(n)
        ph, _ = src.phase()
        assert ph.value == ref.phase.value, n
        gaps.append(pos + n)
        pos += n + 1                                      # leave a gap: the next slice starts at another alignment
    got = torch.cat(pieces)
    assert np.array_equal(u32(got), u32(whole))
    assert np.all(u32(buf[gaps]) == guard)
    want = orc.Source(WAVES[wave], 1000.0, FS, 0.5, -1.0, dtype).work(total)
    assert np.array_equal(u32(whole), want.view(np.uint32))


@pytest.mark.parametrize("dtype", [np.float32, np.complex64], ids=["f32", "c32"])
@pytest.mark.parametrize("wave", list(WAVES))
def test_set_amplitude_between_calls(wave, dtype):
    """set_amplitude applies from the next call; amplitudes 0, -1, NaN and inf give the reference's signed zeros and NaN
    bit patterns (x86-64's: a NaN amplitude comes out quieted with its sign and payload, 0 * inf is 0xFFC00000)."""
    tdt = torch.complex64 if dtype == np.complex64 else torch.float32
    src = make(WAVES[wave], 1234.5, 2.0, 0.1, dtype)
    ref = orc.Source(WAVES[wave], 1234.5, FS, 2.0, 0.1, dtype)
    for amp in (None, 0.0, -1.0, np.nan, -0.0, 1e30, np.inf, -np.nan, -np.inf):
        if amp is not None:
            src.set_amplitude(amp)
            ref.amplitude = np.float32(amp)
        o = torch.empty(10007, dtype=tdt, device="cuda")
        src.generate(o)
        assert np.array_equal(u32(o), ref.work(10007).view(np.uint32)), amp


@pytest.mark.parametrize("f, fs", [(-3000.0, 48000.0), (30000.0, 48000.0), (100000.0, 48000.0), (1.0, 0.0),
                                   (0.0, 0.0), (np.nan, 48000.0), (1000.0, -48000.0)])
def test_increment_of_unvalidated_arguments(f, fs):
    """The builders take any frequency and sample rate (no validation, like the reference): the plan's increment is
    the oracle's FixedPointPhase::new(2 PI f / fs), and the samples follow it."""
    src = fb().SignalSourceBuilder.sin(f, fs, 1.0, 0.0)
    ref = orc.Source(orc.SIN, f, fs, 1.0, 0.0)
    assert src.phase()[1].value == ref.inc
    o = torch.empty(4099, device="cuda")
    src.generate(o)
    assert np.array_equal(u32(o), ref.work(4099).view(np.uint32))


@pytest.mark.parametrize("dtype", [np.float32, np.complex64], ids=["f32", "c32"])
def test_block_under_mocker_fills_reservation_and_never_finishes(dtype):
    from futuresdr_b200.blocks import Mocker
    src = fb().SignalSourceBuilder.square(700.0, FS, 0.25, 0.0, dtype)
    ref = orc.Source(orc.SQUARE, 700.0, FS, 0.25, 0.0, dtype)
    m = Mocker(src)
    for n in (4096, 333):
        m.init_output(n)
        io = m.run()
        assert not io.finished and not io.call_again
        out = m.output()
        assert out.numel() == n
        assert np.array_equal(u32(out), ref.work(n).view(np.uint32))


def test_chain_signal_source_head_fir_sink():
    """SignalSource -> Head(n) -> Fir(64 taps) -> VectorSink finishes with n - 63 items, within the FIR parity bar
    (1e-5 ||taps||_1 max|x|) of the oracle chain."""
    import oracle as ref_fir
    from futuresdr_b200.blocks import FirBuilder, Head
    from futuresdr_b200.edges import VectorSink, run_chain
    n = 3 * (1 << 20) + 4321
    rng = np.random.default_rng(9)
    taps = rng.uniform(-1, 1, 64).astype(np.float32)
    src = fb().SignalSourceBuilder.sin(1000.0, FS, 0.8, 0.2, np.complex64)
    snk = VectorSink(np.complex64, chunk_items=1 << 19)
    run_chain([src, Head(np.complex64, n), FirBuilder.fir(taps, np.complex64), snk], buffer_items=1 << 20)
    got = snk.items()
    x = orc.Source(orc.SIN, 1000.0, FS, 0.8, 0.2, np.complex64).work(n)
    _, _, _, want = ref_fir.fir(taps, x, n)
    assert got.size == want.size == n - 63
    assert np.max(np.abs(got - want)) <= 1e-5 * float(np.sum(np.abs(taps))) * float(np.max(np.abs(x)))


def test_head_semantics():
    """head.rs:63-83: copies min(n_items, input, output), finishes exactly when n_items reaches 0 -- not when the
    input finishes -- and an empty call changes nothing."""
    from futuresdr_b200.blocks import Head, Mocker, WorkIo
    x = np.arange(100, dtype=np.float32)
    h = Head(np.float32, 30)
    m = Mocker(h)
    m.input(x)
    m.init_output(1000)
    io = m.run()
    assert io.finished and np.array_equal(m.output().cpu().numpy(), x[:30]) and h.input.pos == 30
    h = Head(np.float32, 200)                         # input finishes early: Head does not
    m = Mocker(h)
    m.input(x)
    m.init_output(1000)
    io = m.run()
    assert not io.finished and h.n_items == 100 and np.array_equal(m.output().cpu().numpy(), x)
    io = WorkIo()
    h.work(io)                                        # nothing left: no copy, still not finished
    assert not io.finished and h.n_items == 100 and h.output.len == 100
    h = Head(np.complex64, 50)                        # the output slice limits a call
    m = Mocker(h)
    xc = (np.arange(80) + 1j).astype(np.complex64)
    m.input(xc)
    m.init_output(20)
    io = m.run()
    assert not io.finished and h.n_items == 30 and np.array_equal(m.output().cpu().numpy(), xc[:20])


def test_bad_arguments_refused():
    from futuresdr_b200 import _lib
    from futuresdr_b200.context import default_context
    L, ctx = _lib.lib, default_context()
    h = C.c_void_p()
    for wave in (3, -1, 100):
        assert L.b2s_sigsrc_create(ctx.handle, wave, 0, 1.0, 48000.0, 1.0, 0.0, C.byref(h)) == _lib.EINVAL
    assert L.b2s_sigsrc_create(None, 0, 0, 1.0, 48000.0, 1.0, 0.0, C.byref(h)) == _lib.EINVAL
    assert L.b2s_sigsrc_create(ctx.handle, 0, 0, 1.0, 48000.0, 1.0, 0.0, None) == _lib.EINVAL
    assert L.b2s_sigsrc_create(ctx.handle, 1, 1, 1.0, 48000.0, 1.0, 0.0, C.byref(h)) == _lib.OK
    p, v, i = C.c_size_t(7), C.c_int32(0), C.c_int32(0)
    o = torch.empty(16, device="cuda")
    assert L.b2s_sigsrc_exec(h, None, 4, C.byref(p)) == _lib.EINVAL
    assert L.b2s_sigsrc_exec(h, C.c_void_p(o.data_ptr() + 2), 4, C.byref(p)) == _lib.EINVAL    # not float-aligned
    assert L.b2s_sigsrc_exec(h, C.c_void_p(o.data_ptr()), 4, None) == _lib.EINVAL
    assert L.b2s_sigsrc_exec(None, C.c_void_p(o.data_ptr()), 4, C.byref(p)) == _lib.EINVAL
    assert L.b2s_sigsrc_exec(h, None, 0, C.byref(p)) == _lib.OK and p.value == 0
    assert L.b2s_sigsrc_phase(h, None, C.byref(i)) == _lib.EINVAL
    assert L.b2s_sigsrc_phase(None, C.byref(v), C.byref(i)) == _lib.EINVAL
    assert L.b2s_sigsrc_set_amplitude(None, 1.0) == _lib.EINVAL
    assert L.b2s_sigsrc_phase(h, C.byref(v), C.byref(i)) == _lib.OK
    L.b2s_sigsrc_destroy(h)
    with pytest.raises(ValueError):
        fb().SignalSource(7, 1.0, 48000.0, 1.0, 0.0)
    with pytest.raises(ValueError):
        fb().SignalSource(fb().SignalWave.Sin, 1.0, 48000.0, 1.0, 0.0, np.float64)
