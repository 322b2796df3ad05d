"""The SSB transceiver on the GPU against the C oracle (tests/ssb_oracle.c): the three oscillator mixers bit for bit
under every slicing, in place, across the record ring, through reset and destroy; Apply(DivC32) and
ApplyNM(C32ToI16Iq) bit for bit at unaligned starts and on edge values, with ApplyNM's counts and finish rule; both
graphs stream by stream; and a transmit -> .dat file -> receive loopback against a CPU model (tests/ssb_model.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

import futuresdr_b200 as fb
from futuresdr_b200 import _lib, ssb
from futuresdr_b200._lib import B200SdrError, lib
from futuresdr_b200.blocks import Apply, ApplyNM, ApplyNMOp, ApplyOp, Mixer, MixOp, Mocker, Rotator, WorkIo, _ptr
from futuresdr_b200.edges import FileSink, FileSource, Flowgraph, VectorSink, VectorSource

import oracle as orc
import ssb_model as sm
import ssb_oracle as so
from test_ssb_reference import _nan_equal, i16_edges, signal

pytestmark = pytest.mark.gpu

OPS = [(MixOp.RotateC32, so.ROTATE, 1.0), (MixOp.RotateScaleC32, so.ROTATE_SCALE, 0.0001),
       (MixOp.WeaverF32, so.WEAVER, 0.5)]
THETA = float(ssb.xlating_phase())


def _out_like(op, n):
    return torch.full((n,), float("nan"), dtype=torch.float32 if op == MixOp.WeaverF32 else torch.complex64,
                      device="cuda")


def _mix_sliced(blk, xd, out, steps):
    pos, k = 0, 0
    n = xd.numel()
    while pos < n:
        m = min(steps[k % len(steps)], n - pos)
        assert blk.mix(xd[pos:pos + m], out[pos:pos + m]) == m
        pos, k = pos + m, k + 1


@pytest.mark.parametrize("op,oop,param", OPS, ids=[o[0].name for o in OPS])
@pytest.mark.parametrize("steps", [[1], [7], [8], [9], [4097], "random"])
def test_mixer_bit_exact_any_slicing(op, oop, param, steps):
    rng = np.random.default_rng(int(op) * 100 + (0 if steps == "random" else steps[0]))
    n = 60_001
    x = signal(rng, n)
    if steps == "random":
        steps = rng.integers(1, 5000, 50).tolist()
    want = so.Mixer(oop, THETA, param).work(x)
    blk = Mixer(op, THETA, param)
    xd = torch.from_numpy(x).cuda()
    out = _out_like(op, n)
    _mix_sliced(blk, xd, out, steps)
    torch.cuda.synchronize()
    assert _nan_equal(out.cpu().numpy(), want)


@pytest.mark.parametrize("op,oop,param", OPS[:2], ids=[o[0].name for o in OPS[:2]])
def test_rotate_ops_in_place(op, oop, param):
    x = signal(np.random.default_rng(3), 100_003)
    want = so.Mixer(oop, -2.5, param).run(x, [5, 13, 4096, 50_000])
    blk = Mixer(op, -2.5, param)
    buf = torch.from_numpy(x).cuda()
    for a, b in zip([0, 5, 13, 4096, 50_000], [5, 13, 4096, 50_000, x.size]):
        assert blk.mix(buf[a:b], buf[a:b]) == b - a
    torch.cuda.synchronize()
    assert _nan_equal(buf.cpu().numpy(), want)


def test_mixer_40mi_stream_wraps_the_record_ring():
    """40 Mi samples: more than the 32 Mi-sample run-ahead ring, in execs that start at every residue mod 8."""
    n = 40 * 1024 * 1024 + 3
    rng = np.random.default_rng(4)
    x = np.tile(signal(rng, 1 << 20, specials=False), n // (1 << 20) + 1)[:n]
    want = so.Mixer(so.WEAVER, 0.0123, 0.5).work(x)
    blk = Mixer(MixOp.WeaverF32, 0.0123, 0.5)
    xd = torch.from_numpy(x).cuda()
    out = torch.empty(n, dtype=torch.float32, device="cuda")
    _mix_sliced(blk, xd, out, [9_000_001, 3, 12_345_677, 20_000_000])
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy().view(np.uint32), want.view(np.uint32))


def test_mixer_reset_mid_stream_and_destroy_in_flight():
    x = signal(np.random.default_rng(5), 200_000, specials=False)
    blk = Mixer(MixOp.RotateScaleC32, 1.3, 0.0001)
    xd = torch.from_numpy(x).cuda()
    out = torch.empty_like(xd)
    blk.mix(xd[:77_777], out[:77_777])
    blk.reset()                                                     # osc back to 1 + 0i
    blk.mix(xd, out)
    torch.cuda.synchronize()
    assert _nan_equal(out.cpu().numpy(), so.Mixer(so.ROTATE_SCALE, 1.3, 0.0001).work(x))
    for op in MixOp:                                                # work queued, then destroyed at once
        m = Mixer(op, 0.7, 0.5)
        o = _out_like(op, x.size)
        for _ in range(4):
            m.mix(xd, o)
        m.close()
    torch.cuda.synchronize()


def test_mixer_refusals():
    x = torch.from_numpy(signal(np.random.default_rng(6), 1000, specials=False)).cuda()
    w = Mixer(MixOp.WeaverF32, 0.1, 0.5)
    raw = x.view(torch.float32)
    with pytest.raises(B200SdrError):                               # f32 output on top of its c32 input
        w.mix(x, raw[:1000])
    with pytest.raises(B200SdrError):
        w.mix(x[1:], raw[1000:])
    r = Mixer(MixOp.RotateC32, 0.1)
    with pytest.raises(B200SdrError):                               # ROTATE: in place only exactly
        r.mix(x[:500], x[1:501])
    with pytest.raises(B200SdrError):                               # an input not aligned to a c32 item
        r.mix(_Misaligned(raw), torch.empty_like(x[:499]))
    with pytest.raises(B200SdrError):
        lib_op = C.c_void_p()
        fb._lib.check(lib.b2s_mixer_create(fb.default_context().handle, 3, 0.1, 1.0, C.byref(lib_op)))
    c, p = C.c_size_t(9), C.c_size_t(9)                             # empty slices: nothing to do
    assert lib.b2s_mixer_exec(r._h, None, 0, None, 5, C.byref(c), C.byref(p)) == 0 and (c.value, p.value) == (0, 0)


class _Misaligned:
    """A 499-item c32 view that starts 4 bytes into a c32 buffer (torch refuses to make one)."""

    def __init__(self, raw):
        self.ptr, self.n = raw.data_ptr() + 4, 499

    def data_ptr(self):
        return self.ptr

    def numel(self):
        return self.n


def test_rotate_c32_is_rotator_rotate():
    x = signal(np.random.default_rng(7), 123_457, specials=False)
    xd = torch.from_numpy(x).cuda()
    a, b = torch.empty_like(xd), torch.empty_like(xd)
    m, r = Mixer(MixOp.RotateC32, ssb.mixer_phase()), Rotator(ssb.mixer_phase())
    _mix_sliced(m, xd, a, [1000, 17])
    pos = 0
    for step in (3, 100_000, 10 ** 9):
        n = min(step, x.size - pos)
        r.rotate(xd[pos:pos + n], b[pos:pos + n])
        pos += n
    torch.cuda.synchronize()
    assert np.array_equal(a.cpu().numpy().view(np.uint64), b.cpu().numpy().view(np.uint64))


# ---- DivC32, C32ToI16Iq, ApplyNM ----------------------------------------------------------------------------------
@pytest.mark.parametrize("in_off,out_off", [(0, 0), (1, 0), (0, 1), (3, 2), (2, 3), (1, 1)])
def test_div_and_i16_bit_exact_unaligned(in_off, out_off):
    rng = np.random.default_rng(in_off * 7 + out_off)
    for x in (signal(rng, 10_007), i16_edges(), signal(rng, 3, specials=False)):
        n = x.size
        xd = torch.zeros(n + 8, dtype=torch.complex64, device="cuda")
        xd[in_off:in_off + n] = torch.from_numpy(x).cuda()
        # DivC32 after ScaleC32 by 2 is the file level
        s = torch.zeros_like(xd)
        assert Apply(ApplyOp.ScaleC32, 2.0).apply(xd[in_off:in_off + n], s[out_off:out_off + n]) == n
        o = torch.full((n + 8,), 7.0, dtype=torch.complex64, device="cuda")
        assert Apply(ApplyOp.DivC32, 0.0001).apply(s[out_off:out_off + n], o[out_off:out_off + n]) == n
        got = o.cpu().numpy()
        assert _nan_equal(got[out_off:out_off + n], so.file_level(x))
        assert (got[:out_off] == 7).all() and (got[out_off + n:] == 7).all()
        # i16 pairs at every 2-byte start (odd out_off: the pair is not 4-byte aligned)
        q = torch.full((2 * n + 8,), 99, dtype=torch.int16, device="cuda")
        blk = ApplyNM(ApplyNMOp.C32ToI16Iq, 0.9)
        assert blk.apply(xd[in_off:in_off + n], q[out_off:out_off + 2 * n]) == (n, 2 * n)
        got = q.cpu().numpy()
        assert np.array_equal(got[out_off:out_off + 2 * n], so.to_i16_iq(x))
        assert (got[:out_off] == 99).all() and (got[out_off + 2 * n:] == 99).all()


def test_i16_edges_by_hand():
    x = np.array([complex(np.inf, -np.inf), complex(np.nan, -0.0), complex(1e-45, -1e-40), complex(2.0, -2.0)],
                 np.complex64)
    q = torch.zeros(8, dtype=torch.int16, device="cuda")
    ApplyNM(ApplyNMOp.C32ToI16Iq, 0.9).apply(torch.from_numpy(x).cuda(), q)
    assert q.cpu().tolist() == [32767, -32768, 0, 0, 0, 0, 32767, -32768]


@pytest.mark.parametrize("cap", [0, 1, 2, 3, 5, 17, 2001, 4000, 4001])
def test_applynm_counts_and_finish(cap):
    """m = min(in / 1, out / 2) items (applynm.rs:109); finished once the input is finished and no item is left."""
    x = signal(np.random.default_rng(8), 2000, specials=False)
    blk = ApplyNM(ApplyNMOp.C32ToI16Iq, 0.9)
    m = Mocker(blk)
    m.input(x)
    blk.output.reserve(cap)
    io = WorkIo()
    blk.work(io)
    torch.cuda.synchronize()
    k = min(x.size, cap // 2)
    assert blk.input.pos == k and blk.output.len == 2 * k
    assert io.finished == (k == x.size)
    assert np.array_equal(blk.output.get().cpu().numpy(), so.to_i16_iq(x[:k]))
    c, p = C.c_size_t(0), C.c_size_t(0)                             # the C ABI's counts for an odd capacity
    xd = torch.from_numpy(x).cuda()
    o = torch.empty(cap + 1, dtype=torch.int16, device="cuda")
    _lib.check(lib.b2s_apply_exec(blk._h, _ptr(xd), x.size, _ptr(o), cap, C.byref(c), C.byref(p)))
    assert (c.value, p.value) == (k, 2 * k)


def test_i16_refusals():
    x = torch.from_numpy(signal(np.random.default_rng(9), 100, specials=False)).cuda()
    blk = ApplyNM(ApplyNMOp.C32ToI16Iq, 0.9)
    with pytest.raises(B200SdrError):                               # in place
        blk.apply(x, x.view(torch.int16)[:200])
    o = torch.empty(400, dtype=torch.int16, device="cuda")
    c, p = C.c_size_t(0), C.c_size_t(0)
    assert lib.b2s_apply_exec(blk._h, _ptr(x), 100, C.c_void_p(o.data_ptr() + 1), 200, C.byref(c), C.byref(p)) < 0


# ---- the graphs ---------------------------------------------------------------------------------------------------
def _fir_tol(taps, x):
    return sm.FIR_REL * float(np.sum(np.abs(taps))) * float(np.max(np.abs(x)))


def _resamp_check(x, y, interp, decim):
    L, M, taps = sm.resampler_taps(interp, decim)
    _, p, _, ref = orc.resamp_fir(taps, L, M, x, y.size + 64)
    assert p >= y.size and y.size > 0
    assert np.max(np.abs(y - ref[:y.size])) <= 1e-5 * sm.arm_l1(interp, decim) * np.max(np.abs(x))


def _transmit(audio, mode="lsb", dat=None, chunk=1 << 14):
    fg = Flowgraph()
    src = VectorSource(audio, chunk_items=chunk)
    fg.add(src)
    b = ssb.transmitter(fg, src, mode, 48_000)
    sinks = {k: VectorSink(b[k].out_dtype) for k in ("lowpass", "delay", "hilbert", "to_complex", "resampler", "mixer",
                                                     "to_i16_iq", "scale", "file_level")}
    for k, s in sinks.items():
        fg.connect(b[k], s)
    if dat is not None:
        fg.connect(b["file_level"], FileSink(dat))
    fg.run(buffer_items=1 << 16)
    return {k: s.items() for k, s in sinks.items()}


@pytest.mark.parametrize("mode", ["lsb", "usb"])
def test_transmit_graph_stream_by_stream(mode):
    audio = sm.tones([1000.0], 48_000, 30_000) + np.random.default_rng(10).uniform(-0.1, 0.1, 30_000).astype(np.float32)
    s = _transmit(audio, mode)
    lp = s["lowpass"]
    lp_taps = ssb.lowpass_taps(48_000)
    assert np.max(np.abs(lp - orc.fir(lp_taps, audio)[3][:lp.size])) <= _fir_tol(lp_taps, audio)
    assert np.array_equal(s["delay"].view(np.uint32), lp[83:83 + s["delay"].size].view(np.uint32))
    h = s["hilbert"]
    assert np.max(np.abs(h - orc.fir(ssb.hilbert_taps(), lp)[3][:h.size])) <= _fir_tol(ssb.hilbert_taps(), lp)
    c = s["to_complex"]
    assert c.size == h.size
    assert np.array_equal(c.real.view(np.uint32), s["delay"][:c.size].view(np.uint32))
    assert np.array_equal(c.imag.view(np.uint32), (-h if mode == "lsb" else h).view(np.uint32))
    _resamp_check(c, s["resampler"], ssb.FILE_RATE, 48_000)
    r, mix = s["resampler"], s["mixer"]
    assert mix.size == r.size
    assert _nan_equal(mix, so.Mixer(so.ROTATE, ssb.mixer_phase()).work(r))
    assert np.array_equal(s["to_i16_iq"], so.to_i16_iq(mix, 0.9))
    assert _nan_equal(s["file_level"], so.file_level(mix))


@pytest.mark.parametrize("audio_rate", [48_000, 8_000])
def test_receive_graph_stream_by_stream(audio_rate):
    rng = np.random.default_rng(audio_rate)
    x = (rng.standard_normal(300_001) + 1j * rng.standard_normal(300_001)).astype(np.complex64) * np.float32(5000)
    fg = Flowgraph()
    src = VectorSource(x, chunk_items=1 << 15)
    fg.add(src)
    b = ssb.receiver(fg, src, audio_rate)
    sinks = {k: VectorSink(b[k].out_dtype) for k in b}
    for k, s in sinks.items():
        fg.connect(b[k], s)
    fg.run(buffer_items=1 << 16)
    xl, r, w = (sinks[k].items() for k in ("xlating", "resampler", "weaver"))
    assert _nan_equal(xl, so.Mixer(so.ROTATE_SCALE, ssb.xlating_phase(), 0.0001).work(x))
    _resamp_check(xl, r, audio_rate, ssb.FILE_RATE)
    assert w.size == r.size
    assert _nan_equal(w, so.Mixer(so.WEAVER, ssb.weaver_phase(audio_rate), 0.5).work(r))


# ---- the loopback ---------------------------------------------------------------------------------------------------
# Bounds fixed from the CPU model (ssb_model.transmit / receive, 1 s of audio at 48 kHz, 0.4 per tone): the unwanted
# sideband at 53 kHz + f sits 86 dB (one tone) and 67 dB (two tones) under the wanted one, the strongest component of
# the file outside 53 kHz -/+ 3.5 kHz (the resampler's images) 96 dB under, and the strongest component of the audio
# more than 8 bins from a tone 65 dB under it.  The device must reach the same to within a margin.
SIDEBAND_DB, IMAGE_DB, SPUR_DB = -55.0, -75.0, -50.0


@pytest.mark.parametrize("freqs", [[1000.0], [700.0, 1900.0]], ids=["tone", "two-tone"])
def test_loopback_audio_to_audio(tmp_path, freqs):
    audio = sm.tones(freqs, 48_000, 48_000)
    dat = tmp_path / "ssb_lsb_256k.dat"
    _transmit(audio, "lsb", str(dat))
    file = np.fromfile(dat, np.complex64)
    model_file = sm.transmit(audio)["file_level"]
    # the model keeps every output its input allows; the resampler's count rule can stop one output earlier
    assert 0 <= model_file.size - file.size <= 1
    model_file = model_file[:file.size].astype(np.complex64)
    f, p = sm.spectrum_db(file[:1 << 17], ssb.FILE_RATE)
    top = max(sm.level_at(f, p, 53_000 - fa, 20) for fa in freqs)
    assert max(sm.level_at(f, p, 53_000 + fa, 20) for fa in freqs) - top <= SIDEBAND_DB
    assert float(np.max(p[(f < 49_500) | (f > 56_500)])) - top <= IMAGE_DB
    for rx_rate in (48_000, 8_000):
        fg = Flowgraph()
        src = FileSource(str(dat), np.complex64, repeat=False, chunk_items=1 << 15)
        fg.add(src)
        b = ssb.receiver(fg, src, rx_rate)
        snk = VectorSink(np.float32)
        fg.connect(b["weaver"], snk)
        fg.run(buffer_items=1 << 16)
        got = snk.items()
        want = sm.receive(model_file, rx_rate)["weaver"]
        assert 0 <= want.size - got.size <= 2            # the model keeps every output; each device resampler may stop one earlier
        bound = sm.error_bound(audio, 48_000, rx_rate)
        err = float(np.max(np.abs(got - want[:got.size])))
        assert err <= bound, (err, bound)
        N = 1 << int(np.log2(got.size))
        f2, p2 = sm.spectrum_db(got[got.size - N:], rx_rate)
        binw = rx_rate / N
        for fa in freqs:
            near = np.abs(f2 - fa) < 100
            assert abs(f2[near][np.argmax(p2[near])] - fa) <= binw
        peak = max(sm.level_at(f2, p2, fa, 3 * binw) for fa in freqs)
        away = np.ones_like(f2, bool)
        for fa in freqs:
            away &= np.abs(f2 - fa) > 8 * binw
        assert float(np.max(p2[away])) - peak <= SPUR_DB
