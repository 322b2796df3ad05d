"""Combine, Split, StreamDuplicator, StreamDeinterleaver and Delay on the device (csrc/stream.cu), bit for bit against
numpy float32 restatements of the reference's closures (numpy does not contract to FMA; np.hypot on float32 is glibc's
hypotf, which is what num_complex's norm() calls).  Inputs carry +-0, denormals, +-inf and NaN; outputs are compared on
their bit patterns, NaN positions without their payload.  Slices start at every 4-byte offset mod 16 bytes, so each
stream takes the scalar or the vector path independently."""
import ctypes as C

import numpy as np
import pytest
import torch

import futuresdr_b200 as fb
from futuresdr_b200 import _lib
from futuresdr_b200._lib import lib
from futuresdr_b200.blocks import WorkIo

pytestmark = pytest.mark.gpu

SPECIAL = np.array([0.0, -0.0, 1e-45, -1e-45, 1.17e-38, -3e-39, np.inf, -np.inf, np.nan, 1.0, -2.5, 3.4e38, -3.4e38,
                    1.8e19, 1e-20, 6.5e-20], np.float32)


def _f32(n, rng):
    x = rng.standard_normal(n).astype(np.float32) * np.float32(10.0) ** rng.integers(-30, 30, n).astype(np.float32)
    k = min(n, 4 * SPECIAL.size)
    x[rng.choice(n, k, replace=False) if n >= k else slice(None)] = np.resize(SPECIAL, k)[: min(n, k)]
    return x


def _c32(n, rng):
    return (_f32(n, rng) + 1j * _f32(n, rng)[rng.permutation(n)]).astype(np.complex64)


def _same(got, want):
    g = np.ascontiguousarray(got).view(np.float32 if got.dtype != np.float64 else np.float64).ravel()
    w = np.ascontiguousarray(want).view(g.dtype).ravel()
    assert g.shape == w.shape
    gn, wn = np.isnan(g), np.isnan(w)
    assert np.array_equal(gn, wn), f"NaN positions differ at {np.flatnonzero(gn != wn)[:8]}"
    ib = np.uint32 if g.dtype == np.float32 else np.uint64
    bad = np.flatnonzero((g.view(ib) != w.view(ib)) & ~gn)
    assert bad.size == 0, f"{bad.size} items differ, first at {bad[:8]}: got {g[bad[:4]]} want {w[bad[:4]]}"


# closures of b2s_combine_op, restated in numpy float32
def _restate(op, a, b):
    with np.errstate(all="ignore"):
        if op == fb.CombineOp.AddF32:
            return a + b
        if op == fb.CombineOp.SubF32:
            return a - b
        if op == fb.CombineOp.MulF32:
            return a * b
        if op == fb.CombineOp.ConjMulC32:
            r = np.empty(a.size, np.complex64)
            cr, ci = b.real, -b.imag
            r.real = a.real * cr - a.imag * ci
            r.imag = a.real * ci + a.imag * cr
            return r
        if op == fb.CombineOp.MagDivC32F32:
            return np.hypot(a.real, a.imag) / b
        r = np.empty(a.size, np.complex64)
        r.real = a
        r.imag = b if op == fb.CombineOp.ToC32 else b * np.float32(-1.0)
        return r


_TYPES = {fb.CombineOp.AddF32: ("f", "f", np.float32), fb.CombineOp.SubF32: ("f", "f", np.float32),
          fb.CombineOp.MulF32: ("f", "f", np.float32), fb.CombineOp.ConjMulC32: ("c", "c", np.complex64),
          fb.CombineOp.MagDivC32F32: ("c", "f", np.float32), fb.CombineOp.ToC32: ("f", "f", np.complex64),
          fb.CombineOp.ToC32NegQ: ("f", "f", np.complex64)}


class _Raw:
    """A device copy of ``host`` that starts ``off_bytes`` (a multiple of 4) past a 64-byte boundary, with 64 bytes of
    a guard pattern on either side."""

    GUARD = 0xA5

    def __init__(self, host: np.ndarray, off_bytes: int):
        raw = np.ascontiguousarray(host).view(np.uint8).ravel()
        self.off = 64 + off_bytes
        self.init = np.full(raw.size + 128, self.GUARD, np.uint8)
        self.init[self.off:self.off + raw.size] = raw
        self.t = torch.from_numpy(self.init).cuda()
        self.ptr = C.c_void_p(self.t.data_ptr() + self.off)

    def get(self, dtype, n):
        b = np.dtype(dtype).itemsize * n
        return self.t[self.off:self.off + b].cpu().numpy().view(dtype)

    def assert_written_only(self, dtype, n):
        """Every byte outside the first ``n`` items still holds what the constructor put there: the rest of the slice
        and the guards on both sides.  A head or tail item written one slot early or late lands on one of them."""
        b = np.dtype(dtype).itemsize * n
        outside = np.ones(self.init.size, bool)
        outside[self.off:self.off + b] = False
        bad = np.flatnonzero((self.t.cpu().numpy() != self.init) & outside) - self.off
        assert bad.size == 0, f"{bad.size} bytes outside the {n} items changed, first at slice byte offsets {bad[:8]}"


def _ctx():
    return fb.default_context().handle


@pytest.mark.parametrize("op", list(fb.CombineOp), ids=[o.name for o in fb.CombineOp])
@pytest.mark.parametrize("n", list(range(10)) + [67, 4099, (1 << 20) + 3])
def test_combine_bit_exact(op, n):
    rng = np.random.default_rng(int(op) * 1000 + n % 997)
    ta, tb, to = _TYPES[op]
    for offs in ([(0, 0, 0), (4, 8, 12), (12, 0, 4), (8, 4, 0), (4, 12, 8)] if n < 5000 else [(0, 0, 0), (4, 12, 8)]):
        a = _c32(n, rng) if ta == "c" else _f32(n, rng)
        b = _c32(n + 3, rng) if tb == "c" else _f32(n + 3, rng)
        da, db = _Raw(a, offs[0]), _Raw(b, offs[1])
        do = _Raw(np.zeros(n, to), offs[2])
        c, p = C.c_size_t(9), C.c_size_t(9)
        before = lib.b2s_ctx_bytes_held(_ctx())
        assert lib.b2s_combine_exec(_ctx(), int(op), da.ptr, n, db.ptr, n + 3, do.ptr, n + 1, C.byref(c), C.byref(p)) == 0
        torch.cuda.synchronize()
        assert (c.value, p.value) == (n, n)
        assert lib.b2s_ctx_bytes_held(_ctx()) == before
        _same(do.get(to, n), _restate(op, a, b[:n]))
        do.assert_written_only(to, n)


def test_combine_in_place_and_overlap():
    rng = np.random.default_rng(5)
    n = 1000
    a, b = _c32(n, rng), _c32(n, rng)
    da, db = _Raw(a, 8), _Raw(b, 0)
    c, p = C.c_size_t(0), C.c_size_t(0)
    op = int(fb.CombineOp.ConjMulC32)
    # exactly in place: allowed
    assert lib.b2s_combine_exec(_ctx(), op, da.ptr, n, db.ptr, n, da.ptr, n, C.byref(c), C.byref(p)) == 0
    torch.cuda.synchronize()
    _same(da.get(np.complex64, n), _restate(fb.CombineOp.ConjMulC32, a, b))
    # shifted by one item: refused
    shifted = C.c_void_p(da.ptr.value + 8)
    assert lib.b2s_combine_exec(_ctx(), op, da.ptr, n, db.ptr, n, shifted, n, C.byref(c), C.byref(p)) == _lib.EINVAL
    assert lib.b2s_combine_exec(_ctx(), 7, da.ptr, n, db.ptr, n, shifted, n, C.byref(c), C.byref(p)) == _lib.EINVAL
    assert lib.b2s_combine_exec(_ctx(), op, None, n, db.ptr, n, shifted, n, C.byref(c), C.byref(p)) == _lib.EINVAL
    assert lib.b2s_combine_exec(_ctx(), op, None, 0, None, n, None, n, C.byref(c), C.byref(p)) == 0
    assert (c.value, p.value) == (0, 0)


@pytest.mark.parametrize("op", list(fb.SplitOp), ids=[o.name for o in fb.SplitOp])
@pytest.mark.parametrize("n", list(range(10)) + [4101, (1 << 20) + 1])
def test_split_bit_exact(op, n):
    rng = np.random.default_rng(n)
    x = _c32(n, rng) if op == fb.SplitOp.ReIm else _f32(n, rng)
    for offs in [(0, 0, 0), (4, 8, 12), (8, 12, 4), (12, 4, 0)]:
        di, d0, d1 = _Raw(x, offs[0]), _Raw(np.zeros(n, np.float32), offs[1]), _Raw(np.zeros(n, np.float32), offs[2])
        c, p = C.c_size_t(0), C.c_size_t(0)
        assert lib.b2s_split_exec(_ctx(), int(op), di.ptr, n, d0.ptr, d1.ptr, n + 5, C.byref(c), C.byref(p)) == 0
        torch.cuda.synchronize()
        assert (c.value, p.value) == (n, n)
        w0, w1 = (x.real, x.imag) if op == fb.SplitOp.ReIm else (x, x)
        _same(d0.get(np.float32, n), w0)
        _same(d1.get(np.float32, n), w1)
        d0.assert_written_only(np.float32, n)
        d1.assert_written_only(np.float32, n)


_DT = {"f32": np.float32, "c32": np.complex64, "f64": np.float64}


def _items(dt, n, rng):
    if dt == np.float64:
        return np.resize(np.concatenate([_f32(n, rng).astype(np.float64), [5e-324, -0.0, np.inf, 1e300]]), n)
    return _c32(n, rng) if dt == np.complex64 else _f32(n, rng)


@pytest.mark.parametrize("deinterleave", [0, 1], ids=["duplicate", "deinterleave"])
@pytest.mark.parametrize("dtn", list(_DT))
@pytest.mark.parametrize("N", [1, 2, 3, 7, 64, 256])
def test_fanout_bit_exact(deinterleave, dtn, N):
    dt = _DT[dtn]
    isz = np.dtype(dt).itemsize
    rng = np.random.default_rng(N * 7 + deinterleave)
    short = [(g, g, off) for g in range(10) for off in (0, 4, 8, 12)]   # lengths 0..9, the input at every offset
    for groups, cap, offs in [(0, 5, 0), (1, 1, 4), (37, 40, 12), (1029, 1000, 8), ((1 << 16) + 5, 1 << 17, 4), *short]:
        if N >= 64:                                             # keep 256 separate outputs small
            groups, cap = min(groups, 4099), min(cap, 4200)
        n_in = groups * N + (N - 1 if deinterleave else 0) if deinterleave else groups
        x = _items(dt, n_in, rng)
        di = _Raw(x, offs)
        outs = [_Raw(np.zeros(cap, dt), 4 * ((k + offs // 4) % 4)) for k in range(N)]
        ptrs = (C.c_void_p * N)(*[o.ptr.value for o in outs])
        c, p = C.c_size_t(0), C.c_size_t(0)
        before = lib.b2s_ctx_bytes_held(_ctx())
        assert lib.b2s_fanout_exec(_ctx(), deinterleave, isz, di.ptr, n_in, ptrs, N, cap, C.byref(c), C.byref(p)) == 0
        torch.cuda.synchronize()
        assert lib.b2s_ctx_bytes_held(_ctx()) == before
        m = min(cap, n_in // N) if deinterleave else min(cap, n_in)
        assert (c.value, p.value) == ((m * N if deinterleave else m), m)
        for k, o in enumerate(outs):
            want = x[k:m * N:N] if deinterleave else x[:m]
            _same(o.get(dt, m), want)
            o.assert_written_only(dt, m)


def test_fanout_limits():
    x = torch.zeros(1024, device="cuda")
    outs = [torch.zeros(4, device="cuda") for _ in range(257)]
    ptrs = (C.c_void_p * 257)(*[o.data_ptr() for o in outs])
    c, p = C.c_size_t(0), C.c_size_t(0)
    for d in (0, 1):
        assert lib.b2s_fanout_exec(_ctx(), d, 4, C.c_void_p(x.data_ptr()), 1024, ptrs, 257, 4, C.byref(c),
                                   C.byref(p)) == _lib.EUNSUPPORTED
    assert lib.b2s_fanout_exec(_ctx(), 0, 2, C.c_void_p(x.data_ptr()), 1024, ptrs, 2, 4, C.byref(c), C.byref(p)) == _lib.EINVAL
    same = (C.c_void_p * 2)(outs[0].data_ptr(), outs[0].data_ptr())
    assert lib.b2s_fanout_exec(_ctx(), 0, 4, C.c_void_p(x.data_ptr()), 1024, same, 2, 4, C.byref(c), C.byref(p)) == _lib.EINVAL
    with pytest.raises(fb.B200SdrError) as e:
        fb.StreamDuplicator(np.float32, 257)
    assert e.value.code == _lib.EUNSUPPORTED


# ---- block level: ragged (n_in, out_cap) sequences through the Mocker ports, restated work() ----------------------------
def _ragged(rng, total, steps):
    cuts = np.sort(rng.integers(0, total + 1, steps - 1))
    return list(np.diff(np.concatenate([[0], cuts, [total]])))


def _feed(port, full, avail, off):
    """Reader port sees items [pos, avail) of ``full`` placed ``off`` items into its device buffer."""
    if not hasattr(port, "_full"):
        port._full = torch.zeros(full.size + off, dtype=port.data.dtype, device="cuda")
        if full.size:
            port._full[off:].copy_(torch.from_numpy(full))
        port.pos = off
    port.data = port._full[:off + avail]


def _cap(w, cap, off, dtype, total):
    if not hasattr(w, "_full"):
        w._full = torch.zeros(total + off + 8, dtype=w.data.dtype, device="cuda")
        w.len = off
        w._off = off
    w.data = w._full[:min(w.len + cap, w._full.numel())]


@pytest.mark.parametrize("off", [0, 1, 2, 3])
@pytest.mark.parametrize("op", [fb.CombineOp.ConjMulC32, fb.CombineOp.MagDivC32F32, fb.CombineOp.ToC32NegQ,
                                fb.CombineOp.SubF32], ids=lambda o: o.name)
def test_combine_block_ragged(op, off):
    rng = np.random.default_rng(off + 10 * int(op))
    ta, tb, to = _TYPES[op]
    n0, n1 = 3001, 2777
    a = _c32(n0, rng) if ta == "c" else _f32(n0, rng)
    b = _c32(n1, rng) if tb == "c" else _f32(n1, rng)
    blk = fb.Combine(op)
    av0 = av1 = 0
    p0 = p1 = produced = 0
    got = []
    steps = 40
    g0, g1 = _ragged(rng, n0, steps), _ragged(rng, n1, steps)
    caps = np.concatenate([rng.integers(0, 300, steps), np.full(steps, 1000)])
    for s in range(2 * steps):
        av0 += g0[s] if s < steps else 0
        av1 += g1[s] if s < steps else 0
        last = s >= steps - 1
        blk.in0._finished = blk.in1._finished = last
        _feed(blk.in0, a, av0, off)
        _feed(blk.in1, b, av1, (off + 1) % 4)
        _cap(blk.output, int(caps[s]), (off + 2) % 4, to, n0)
        i0_len, i1_len, o_len = av0 - p0, av1 - p1, blk.output.data.numel() - blk.output.len
        m = min(i0_len, i1_len, o_len)                          # combine.rs:114-133 restated
        fin = (last and m == i0_len) or (last and m == i1_len)
        io = WorkIo()
        blk.work(io)
        assert (blk.in0.pos - off - p0, blk.in1.pos - (off + 1) % 4 - p1, io.finished) == (m, m, fin)
        p0, p1, produced = p0 + m, p1 + m, produced + m
        if fin:
            break
    torch.cuda.synchronize()
    o = blk.output.data[(off + 2) % 4:blk.output.len].cpu().numpy()
    assert o.size == produced == min(n0, n1)
    _same(o, _restate(op, a[:produced], b[:produced]))


@pytest.mark.parametrize("off", [0, 1, 2, 3])
@pytest.mark.parametrize("kind", ["split", "dup3", "deint5"])
def test_fanout_blocks_ragged(kind, off):
    rng = np.random.default_rng(off + len(kind))
    n = 4003
    if kind == "split":
        x, blk = _c32(n, rng), fb.Split(fb.SplitOp.ReIm)
        outs, N = [blk.output0, blk.output1], 1
    elif kind == "dup3":
        x, blk = _f32(n, rng).astype(np.float64), fb.StreamDuplicator(np.float64, 3)
        outs, N = blk.outputs, 1
    else:
        x, blk = _c32(n, rng), fb.StreamDeinterleaver(np.complex64, 5)
        outs, N = blk.output, 5
    steps = 30
    gs = _ragged(rng, n, steps)
    av = pos = produced = 0
    for s in range(2 * steps):
        av += gs[s] if s < steps else 0
        last = s >= steps - 1
        blk.input._finished = last
        _feed(blk.input, x, av, off)
        for k, w in enumerate(outs):
            _cap(w, int(rng.integers(0, 200)) if s < steps else 2000, (off + k) % 4, None, n)
        i_len = av - pos
        o_min = min(w.data.numel() - w.len for w in outs)
        m = min(o_min, i_len // N)                              # split.rs:106-123, stream_*.rs restated
        fin = last and (i_len - m * N < N if kind == "deint5" else m * N == i_len)
        io = WorkIo()
        blk.work(io)
        assert (blk.input.pos - off - pos, io.finished) == (m * N, fin)
        pos, produced = pos + m * N, produced + m
        if fin:
            break
    torch.cuda.synchronize()
    got = [w.data[w._off:w.len].cpu().numpy() for w in outs]
    if kind == "split":
        want = [x.real[:produced], x.imag[:produced]]
    elif kind == "dup3":
        want = [x[:produced]] * 3
    else:
        want = [x[k:produced * 5:5] for k in range(5)]
    for g, w in zip(got, want):
        _same(g, w)


# ---- Delay (delay.rs:114-168) ---------------------------------------------------------------------------------------
def _delay_run(blk, x, caps, fin_at):
    """work() calls with the output capped per call; returns [(consumed, produced, call_again, finished)]."""
    seq = []
    for s, cap in enumerate(caps):
        blk.input._finished = s >= fin_at
        before_i, before_o = blk.input.pos, blk.output.len
        blk.output.data = blk.output._full[:blk.output.len + cap]
        io = WorkIo()
        blk.work(io)
        seq.append((blk.input.pos - before_i, blk.output.len - before_o, io.call_again, io.finished))
        if io.finished:
            break
    torch.cuda.synchronize()
    return seq


def _delay_block(dt, n, x):
    blk = fb.Delay(dt, n)
    blk.input.set(x)
    blk.output._full = torch.full((4096,), 7.0, dtype=blk.output.data.dtype, device="cuda")
    blk.output.len = 0
    return blk


@pytest.mark.parametrize("dtn", list(_DT))
def test_delay_pad_copy(dtn):
    dt = _DT[dtn]
    x = _items(dt, 100, np.random.default_rng(1))
    blk = _delay_block(dt, 16, x)
    seq = _delay_run(blk, x, [10, 10, 50, 200], fin_at=0)
    assert seq == [(0, 10, False, False), (0, 6, True, True)]   # Pad(16): the last pad call finishes on a finished input
    blk = _delay_block(dt, 16, x)
    seq = _delay_run(blk, x, [10, 10, 50, 200], fin_at=3)
    assert seq == [(0, 10, False, False), (0, 6, True, False), (50, 50, False, False), (50, 50, False, True)]
    got = blk.output._full[:blk.output.len].cpu().numpy()
    _same(got, np.concatenate([np.zeros(16, dt), x]))


def test_delay_skip_and_new_value():
    x = _f32(300, np.random.default_rng(2))
    blk = _delay_block(np.float32, -83, x)                      # Delay::new(-83): the SSB graph's skip
    assert blk.state == ("skip", 83)
    blk.input.data = blk.input.data[:50]
    seq = _delay_run(blk, x, [20], fin_at=9)
    assert seq == [(50, 0, False, False)] and blk.state == ("skip", 33)
    blk.input.data = torch.from_numpy(x).cuda()
    seq = _delay_run(blk, x, [0, 40], fin_at=9)
    assert seq == [(33, 0, True, False), (40, 40, False, False)] and blk.state == ("copy", 0)
    blk.new_value(True, 5)                                      # pad 5 in the middle of the stream
    assert blk.state == ("pad", 5)
    seq = _delay_run(blk, x, [3, 100, 500], fin_at=2)
    assert seq == [(0, 3, False, False), (0, 2, True, False), (177, 177, False, True)]
    got = blk.output._full[:blk.output.len].cpu().numpy()
    _same(got, np.concatenate([x[83:123], np.zeros(5, np.float32), x[123:]]))
    blk.new_value(False, 7)
    assert blk.state == ("skip", 7)
    blk.new_value(True, 7)
    assert blk.state == ("copy", 0)
    blk.new_value(True, 2)
    blk.new_value(False, 9)
    assert blk.state == ("skip", 7)
    z = _delay_block(np.float32, 0, x)                          # Delay::new(0) is Skip(0)
    assert z.state == ("skip", 0)
    assert _delay_run(z, x, [0], fin_at=9) == [(0, 0, True, False)] and z.state == ("copy", 0)


def test_stream_calls_allocate_nothing():
    ctx = _ctx()
    before = lib.b2s_ctx_bytes_held(ctx)
    rng = np.random.default_rng(3)
    x = _f32(1 << 16, rng)
    for blk in (fb.Combine(fb.CombineOp.MulF32), fb.Split(fb.SplitOp.DupF32), fb.StreamDuplicator(np.float32, 4),
                fb.StreamDeinterleaver(np.float32, 4), fb.Delay(np.float32, 3)):
        for port in ("in0", "in1", "input"):
            if hasattr(blk, port):
                getattr(blk, port).set(x)
        for port in ("output", "output0", "output1", "outputs"):
            w = getattr(blk, port, None)
            for ww in (w if isinstance(w, list) else [w] if w is not None else []):
                ww.reserve(1 << 16)
        for _ in range(3):
            blk.work(WorkIo())
        torch.cuda.synchronize()
        assert lib.b2s_ctx_bytes_held(ctx) == before, type(blk).__name__
