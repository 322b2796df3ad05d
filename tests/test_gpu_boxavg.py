"""MovingAverage (csrc/boxavg.cu) on the GPU, bit for bit against the C oracle (tests/boxavg_oracle.c) given the same
sequence of execs: window lengths on both sides of the 4000-output run, slices at every 4-byte offset with NaN guards
and sentinel-filled outputs, ragged and one-call-at-a-time exec sequences, non-finite values at segment seams, the
refusals, and the two receive front ends (WLAN rx.rs:73-93, M17 rx.rs:109-133) with the real block."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import futuresdr_b200 as fb
from futuresdr_b200 import _lib
from futuresdr_b200._lib import lib
from futuresdr_b200.blocks import Apply, ApplyOp, Fir
from futuresdr_b200.edges import FileSource, Flowgraph, VectorSink, VectorSource

from boxavg_oracle import MAX_ITER, BoxAvgRef, replay

pytestmark = pytest.mark.gpu

SENTINEL = np.float32(-7.25e-3)
GUARD = 8                                                       # NaN words on each side of every slice


def _same(got, want):
    """Bit equality, any NaN matching any NaN."""
    g = np.ascontiguousarray(got).view(np.float32)
    w = np.ascontiguousarray(want).view(np.float32)
    assert g.shape == w.shape, (g.shape, w.shape)
    gn, wn = np.isnan(g), np.isnan(w)
    bad = np.flatnonzero(gn != wn)
    assert bad.size == 0, f"NaN mismatch at words {bad[:8]}"
    diff = np.flatnonzero(g[~gn].view(np.uint32) != w[~wn].view(np.uint32))
    assert diff.size == 0, f"{diff.size} words differ, first at {np.flatnonzero(~gn)[diff[:4]]}"


def _words(x):
    return np.ascontiguousarray(x).view(np.float32)


class Guarded:
    """One device allocation: GUARD NaN words, `off` more NaN words (so the slice starts at 4 off mod 16 bytes), the
    slice, GUARD NaN words."""

    def __init__(self, words: np.ndarray, off: int, fill=None):
        n = words.size
        host = np.full(2 * GUARD + off + n, np.nan, np.float32)
        host[GUARD + off:GUARD + off + n] = words if fill is None else fill
        self.t = torch.from_numpy(host).cuda()
        self.lo, self.n = GUARD + off, n

    def ptr(self):
        return C.c_void_p(self.t.data_ptr() + 4 * self.lo)

    def check_guards(self):
        h = self.t.cpu().numpy()
        assert np.isnan(h[:self.lo]).all() and np.isnan(h[self.lo + self.n:]).all(), "a guard word was written"
        return h[self.lo:self.lo + self.n]


def _exec(blk, x, cap, max_calls, off_in, off_out):
    """One b2s_boxavg_exec over guarded slices -> ((consumed, produced, calls, call_again, done), outputs)."""
    w = 2 if blk.in_dtype == np.complex64 else 1
    xi = Guarded(_words(x), off_in)
    o = Guarded(np.zeros(cap * w, np.float32), off_out, fill=SENTINEL)
    c, p, n = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    ca, dn = C.c_int32(0), C.c_int32(0)
    _lib.check(lib.b2s_boxavg_exec(blk._h, xi.ptr(), len(x), o.ptr(), cap, max_calls, C.byref(c), C.byref(p),
                                   C.byref(n), C.byref(ca), C.byref(dn)), blk.ctx.handle)
    torch.cuda.synchronize()
    xi.check_guards()
    out = o.check_guards()
    assert (out[p.value * w:] == SENTINEL).all(), "written past the produced items"
    got = out[:p.value * w].copy().view(blk.in_dtype)
    return (c.value, p.value, n.value, bool(ca.value), bool(dn.value)), got


def _run_plan(dtype, length, divisor, x, plan, offsets=(0, 0)):
    """Execs (n_in, cap, max_calls) on the stream x, each slice starting where consumption left it."""
    blk = fb.MovingAverage(dtype, length, divisor)
    ref = BoxAvgRef(dtype, length, divisor)
    pos = 0
    for k, (n_in, cap, mc) in enumerate(plan):
        sl = x[pos:pos + n_in]
        oi, oo = (offsets[0] + k) % 4, (offsets[1] + 3 * k) % 4
        counts, got = _exec(blk, sl, cap, mc, oi, oo)
        e = ref.run(sl, cap, mc)
        assert counts == (e.consumed, e.produced, e.calls, e.call_again, e.done), (k, n_in, cap, mc)
        _same(got, e.out)
        pos += e.consumed
    return pos


def _stream(rng, n, dtype):
    x = rng.standard_normal(n).astype(np.float32)
    if np.dtype(dtype) == np.complex64:
        z = np.empty(n, np.complex64)
        z.real, z.imag = x, rng.standard_normal(n).astype(np.float32)
        return z
    return x


SHAPES = [(np.float32, 1, None), (np.float32, 2, None), (np.float32, 3, None), (np.float32, 48, None),
          (np.float32, 64, None), (np.float32, 129, None), (np.float32, 130, None), (np.float32, 3999, None),
          (np.float32, 4000, None), (np.float32, 4001, None), (np.float32, 4800, 4800.0), (np.float32, 9001, None),
          (np.complex64, 1, None), (np.complex64, 2, None), (np.complex64, 3, None), (np.complex64, 48, None),
          (np.complex64, 64, None), (np.complex64, 3999, None), (np.complex64, 4000, None),
          (np.complex64, 4001, None), (np.complex64, 4800, None), (np.complex64, 9001, None)]
SIDS = [f"{'c32' if d == np.complex64 else 'f32'}-{n}{'-div' if v else ''}" for d, n, v in SHAPES]


@pytest.mark.parametrize("dtype,length,divisor", SHAPES, ids=SIDS)
def test_whole_stream_sizes(dtype, length, divisor):
    """n_in at len - 1, len, a segment edge +-1 and many segments; each exec the whole slice (after the pad)."""
    rng = np.random.default_rng(length)
    pad = length - 1
    for n_in in (length - 1, length, length - 1 + MAX_ITER - 1, length - 1 + MAX_ITER, length - 1 + MAX_ITER + 1,
                 length - 1 + 2 * MAX_ITER + 1, length - 1 + 37 * MAX_ITER + 123):
        x = _stream(rng, n_in, dtype)
        _run_plan(dtype, length, divisor, x, [(n_in, pad + n_in + 5, 0)], offsets=(n_in % 4, (n_in // 3) % 4))


@pytest.mark.parametrize("dtype,length,divisor", [(np.float32, 3, None), (np.float32, 64, None),
                                                  (np.complex64, 48, None), (np.float32, 4800, 4800.0),
                                                  (np.complex64, 4001, None)], ids=["f32-3", "f32-64", "c32-48",
                                                                                    "f32-4800-div", "c32-4001"])
def test_ragged_and_single_call_sequences(dtype, length, divisor):
    """Capacity 0, below the pad, exactly the pad, mid-segment capacities, max_calls = 1, and finishing short."""
    rng = np.random.default_rng(length + 1)
    n = length - 1 + 5 * MAX_ITER + 77
    x = _stream(rng, n, dtype)
    pad = length - 1
    plan = [(n, 0, 0), (n, max(pad - 1, 0), 0), (n, 1, 1), (n, 2 * MAX_ITER + 17, 0), (n, 0, 1), (n, 123, 1),
            (n, 5000, 1), (n, 3 * MAX_ITER, 2), (n, 10, 0), (n, 9000, 0), (n, 50, 0)]
    _run_plan(dtype, length, divisor, x, plan)
    x2 = _stream(rng, n, dtype)                                 # exactly the pad, then one call at a time
    plan2 = [(n, pad, 0)] + [(n, MAX_ITER + 1, 1)] * 7
    _run_plan(dtype, length, divisor, x2, plan2, offsets=(1, 2))


@pytest.mark.parametrize("off_in", range(4))
@pytest.mark.parametrize("dtype,length", [(np.float32, 64), (np.complex64, 48), (np.float32, 4800)])
def test_every_word_offset(dtype, length, off_in):
    rng = np.random.default_rng(off_in)
    n = length - 1 + 3 * MAX_ITER + 11
    x = _stream(rng, n, dtype)
    div = 4800.0 if length == 4800 else None
    for off_out in range(4):
        _run_plan(dtype, length, div, x, [(n, n + length, 0)], offsets=(off_in, off_out))


SPECIAL = np.asarray([0.0, -0.0, 1e-45, -1e-45, 1.17e-38, -3e-39, np.inf, -np.inf, np.nan, 3.4e38, -3.4e38],
                     np.float32)


@pytest.mark.parametrize("dtype,length,divisor", [(np.float32, 1, None), (np.float32, 3, None),
                                                  (np.float32, 64, None), (np.float32, 4800, 4800.0),
                                                  (np.complex64, 48, None), (np.complex64, 4001, None)],
                         ids=["f32-1", "f32-3", "f32-64", "f32-4800-div", "c32-48", "c32-4001"])
def test_non_finite_and_signed_values_at_seams(dtype, length, divisor):
    """+-0, denormals, +-inf and NaN in a segment's prefix, its leading and trailing streams and on segment edges:
    the NaN of inf - inf lasts exactly to the end of the reference call that made it."""
    rng = np.random.default_rng(99 + length)
    n = length - 1 + 4 * MAX_ITER + 5
    x = _stream(rng, n, dtype)
    w = _words(x)
    W = 2 if np.dtype(dtype) == np.complex64 else 1
    c0 = length - 1
    spots = [0, 1, c0 // 2, c0, c0 + 7, MAX_ITER - 1, MAX_ITER, MAX_ITER + 1, MAX_ITER + c0 - 1, MAX_ITER + c0,
             2 * MAX_ITER + c0 // 3, 3 * MAX_ITER - 1, 3 * MAX_ITER + c0 + 100, n - 1]
    for k, s in enumerate(spots):
        if 0 <= s < n:
            w[s * W + (k % W)] = SPECIAL[k % SPECIAL.size]
    w[(2 * MAX_ITER + 200) * W:(2 * MAX_ITER + 200 + length + 5) * W] = -0.0       # a window of -0.0
    w[(3 * MAX_ITER + 50) * W:(3 * MAX_ITER + 60) * W] = 1e-44                      # denormals only
    _run_plan(dtype, length, divisor, x, [(n, n + length, 0)])
    _run_plan(dtype, length, divisor, x, [(n, 3 * MAX_ITER // 2, 1)] * 8, offsets=(3, 1))


def test_negative_zero_fold_on_device():
    """A window of -0.0 sums to -0.0 (the f32 fold starts at -0.0); Complex32 gives +0."""
    blk = fb.MovingAverage(np.float32, 3)
    counts, got = _exec(blk, np.full(10, -0.0, np.float32), 12, 0, 0, 0)
    assert counts[:2] == (8, 10)
    assert got.view(np.uint32)[2] == 0x80000000 and got.view(np.uint32)[:2].tolist() == [0, 0]
    cblk = fb.MovingAverage(np.complex64, 3)
    counts, got = _exec(cblk, np.full(10, complex(-0.0, -0.0), np.complex64), 12, 0, 1, 2)
    assert (got.view(np.uint32)[4:] == 0).all()


@pytest.mark.parametrize("dtype,length,divisor", [(np.float32, 64, None), (np.complex64, 48, None),
                                                  (np.float32, 4800, 4800.0)], ids=["f32-64", "c32-48", "m17"])
def test_64mi_items(dtype, length, divisor):
    n = 64 << 20
    rng = np.random.default_rng(5)
    x = _stream(rng, n, dtype)
    blk = fb.MovingAverage(dtype, length, divisor)
    xd = torch.from_numpy(x).cuda()
    od = torch.empty(n + length, dtype=xd.dtype, device="cuda")
    c, p, calls, ca, dn = blk.average(xd, od)
    torch.cuda.synchronize()
    e = BoxAvgRef(dtype, length, divisor).run(x, n + length)
    assert (c, p, calls, ca, dn) == (e.consumed, e.produced, e.calls, e.call_again, e.done)
    _same(od[:p].cpu().numpy(), e.out)


def test_refusals_and_cleanup():
    ctx = fb.default_context()
    base = ctx.bytes_held
    h = C.c_void_p()
    assert lib.b2s_boxavg_create(ctx.handle, 0, 0, 0, 0.0, C.byref(h)) == _lib.EINVAL      # len == 0
    assert lib.b2s_boxavg_create(ctx.handle, 1, 48, 1, 4800.0, C.byref(h)) == _lib.EINVAL  # divisor on Complex32
    with pytest.raises(_lib.B200SdrError):
        fb.MovingAverage(np.complex64, 48, 4800.0)
    blk = fb.MovingAverage(np.float32, 4)
    buf = torch.zeros(20_000, device="cuda")
    c, p, n = C.c_size_t(0), C.c_size_t(0), C.c_size_t(0)
    ca, dn = C.c_int32(0), C.c_int32(0)
    args = (C.byref(c), C.byref(p), C.byref(n), C.byref(ca), C.byref(dn))
    ptr = buf.data_ptr()
    assert lib.b2s_boxavg_exec(blk._h, C.c_void_p(ptr), 10_000, C.c_void_p(ptr + 4 * 5000), 10_000, 0, *args) \
        == _lib.EINVAL                                          # the output overlaps the input it reads
    assert lib.b2s_boxavg_exec(blk._h, C.c_void_p(ptr + 2), 100, C.c_void_p(ptr + 4 * 10_000), 100, 0, *args) \
        == _lib.EINVAL                                          # not 4-byte aligned
    assert lib.b2s_boxavg_exec(blk._h, None, 100, C.c_void_p(ptr + 4 * 10_000), 100, 0, *args) == _lib.EINVAL
    assert lib.b2s_boxavg_exec(blk._h, C.c_void_p(ptr), 100, C.c_void_p(ptr + 4 * 10_000), 100, 0, None, *args[1:]) \
        == _lib.EINVAL
    assert lib.b2s_boxavg_exec(blk._h, C.c_void_p(ptr), 10_000, C.c_void_p(ptr + 4 * 10_000), 10_000, 0, *args) \
        == _lib.OK                                              # disjoint: fine (refusals left the pad as it was)
    assert (c.value, p.value) == (9997, 10_000)
    blk.reset()
    assert lib.b2s_boxavg_exec(blk._h, C.c_void_p(ptr), 10, C.c_void_p(ptr + 4 * 10_000), 2, 1, *args) == _lib.OK
    assert (c.value, p.value, n.value, ca.value) == (0, 2, 1, 0)
    torch.cuda.synchronize()
    blk.close()
    assert ctx.bytes_held == base


def test_profiler_sees_the_kernel():
    from torch.profiler import ProfilerActivity, profile
    blks = [fb.MovingAverage(np.float32, 64), fb.MovingAverage(np.complex64, 48),
            fb.MovingAverage(np.float32, 4800, 4800.0)]
    xs = [torch.ones(100_000, device="cuda"), torch.ones(100_000, dtype=torch.complex64, device="cuda"),
          torch.ones(100_000, device="cuda")]
    outs = [torch.empty_like(x) for x in xs]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for b, x, o in zip(blks, xs, outs):
            b.average(x, o)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages() if "boxavg_kernel" in e.key]
    assert len(names) == 3, names


# ---- graphs ----------------------------------------------------------------------------------------------------------
def _record(blk):
    """Wrap blk.work to log the slices each exec saw: (n_in, n_out_cap, max_calls)."""
    log, orig = [], blk.work

    def work(io):
        log.append((blk.input.slice().numel(), blk.output.slice().numel(), blk.max_calls))
        orig(io)
    blk.work = work
    return log


@pytest.mark.parametrize("buffer_items,max_calls", [(None, 0), (50_000, 0), (20_000, 1)],
                         ids=["big-buffers", "small-buffers", "one-call-per-work"])
def test_wlan_rx_front_end_with_moving_average(buffer_items, max_calls):
    """rx.rs:73-93 with MovingAverage<f32>(64) and MovingAverage<Complex32>(48): every stream bit-exact."""
    n = (4 << 20) if buffer_items is None else 300_000
    rng = np.random.default_rng(12)
    x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) / np.sqrt(2)).astype(np.complex64)
    fg = Flowgraph()
    src = VectorSource(x)
    delay = fb.Delay(np.complex64, 16)
    complex_to_mag_2 = Apply(ApplyOp.NormSqr)
    float_avg = fb.MovingAverage(np.float32, 64, max_calls=max_calls)
    mult_conj = fb.Combine(fb.CombineOp.ConjMulC32)
    complex_avg = fb.MovingAverage(np.complex64, 48, max_calls=max_calls)
    divide_mag = fb.Combine(fb.CombineOp.MagDivC32F32)
    logs = {"float_avg": _record(float_avg), "complex_avg": _record(complex_avg)}
    snk = {k: VectorSink(dt) for k, dt in [("delay", np.complex64), ("mag2", np.float32),
                                           ("mult_conj", np.complex64), ("complex_avg", np.complex64),
                                           ("float_avg", np.float32), ("divide_mag", np.float32)]}
    fg.connect(src, delay)
    fg.connect(src, complex_to_mag_2)
    fg.connect(src, mult_conj, "in0")
    fg.connect(complex_to_mag_2, float_avg)
    fg.connect(mult_conj, complex_avg)
    fg.connect(delay, mult_conj, "in1")
    fg.connect(complex_avg, divide_mag, "in0")
    fg.connect(float_avg, divide_mag, "in1")
    fg.connect(delay, snk["delay"])
    fg.connect(complex_to_mag_2, snk["mag2"])
    fg.connect(mult_conj, snk["mult_conj"])
    fg.connect(complex_avg, snk["complex_avg"])
    fg.connect(float_avg, snk["float_avg"])
    fg.connect(divide_mag, snk["divide_mag"])
    fg.run(buffer_items=buffer_items or n + 4096)
    got = {k: s.items() for k, s in snk.items()}
    d = np.concatenate([np.zeros(16, np.complex64), x])
    _same(got["delay"], d)
    with np.errstate(all="ignore"):
        b = d[:n]
        mc = np.empty(n, np.complex64)
        mc.real = x.real * b.real - x.imag * (-b.imag)
        mc.imag = x.real * (-b.imag) + x.imag * b.real
        mag2 = x.real * x.real + x.imag * x.imag
    _same(got["mult_conj"], mc)
    _same(got["mag2"], mag2)
    fa, fa_counts = replay(np.float32, 64, None, mag2, logs["float_avg"])
    ca, ca_counts = replay(np.complex64, 48, None, mc, logs["complex_avg"])
    assert got["float_avg"].size == n and got["complex_avg"].size == n        # len - 1 zeros, then n + 1 - len sums
    _same(got["float_avg"], fa)
    _same(got["complex_avg"], ca)
    assert sum(p for _, p in fa_counts) == fa.size
    m = got["divide_mag"].size
    assert m == min(fa.size, ca.size)
    with np.errstate(all="ignore"):
        want = np.hypot(ca[:m].real, ca[:m].imag) / fa[:m]
    _same(got["divide_mag"], want)


def test_m17_rx_front_end(tmp_path):
    """rx.rs:109-133 up to the RRC: FileSource(cf32) -> quadrature demod -> * DEMOD_GAIN -> MovingAverage(4800) / 4800
    -> Combine(i1 - i2) -> 81-tap RRC FIR.  The demod stream is sunk and replayed through the oracle, so the average
    and the subtraction are checked bit for bit; the FIR at its tolerance."""
    fx = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "reference_m17_rx.json")))
    taps = np.asarray(fx["taps"], np.float32)
    f32 = np.float32
    gain = f32(48000.0) / (f32(2.0) * f32(np.pi) * f32(800.0))  # DEMOD_GAIN, f32 constant arithmetic
    n = 1_000_003
    rng = np.random.default_rng(17)
    ph = np.cumsum(rng.standard_normal(n) * 0.3)
    x = (np.exp(1j * ph) * (1 + 0.1 * rng.standard_normal(n))).astype(np.complex64)
    path = tmp_path / "input.cf32"
    x.tofile(path)
    fg = Flowgraph()
    src = FileSource(path, np.complex64, chunk_items=1 << 18)
    demod = Apply(ApplyOp.QuadDemod)
    scale = Apply(ApplyOp.ScaleF32, float(gain))
    avg = fb.MovingAverage(np.float32, 4800, 4800.0)
    log = _record(avg)
    subtract = fb.Combine(fb.CombineOp.SubF32)
    rrc = Fir(fb.FirFilter(taps, sample_dtype=np.float32))
    snk = {k: VectorSink(np.float32) for k in ("demod", "avg", "sub", "rrc")}
    fg.connect(src, demod)
    fg.connect(demod, scale)
    fg.connect(scale, subtract, "in0")
    fg.connect(scale, avg)
    fg.connect(avg, subtract, "in1")
    fg.connect(subtract, rrc)
    fg.connect(scale, snk["demod"])
    fg.connect(avg, snk["avg"])
    fg.connect(subtract, snk["sub"])
    fg.connect(rrc, snk["rrc"])
    fg.run(buffer_items=1 << 18)
    got = {k: s.items() for k, s in snk.items()}
    dm = got["demod"]
    assert dm.size == n
    want_avg, _ = replay(np.float32, 4800, 4800.0, dm, log)
    _same(got["avg"], want_avg)
    m = got["sub"].size
    assert m == min(n, want_avg.size)
    _same(got["sub"], dm[:m] - want_avg[:m])
    sub = got["sub"]
    ref = np.convolve(sub.astype(np.float64), taps.astype(np.float64), "valid")
    assert got["rrc"].size == ref.size
    tol = 3e-5 * float(np.sum(np.abs(taps))) * float(np.max(np.abs(sub)))
    assert np.max(np.abs(got["rrc"] - ref)) <= tol
