"""The fan-out / fan-in graph driver (edges.Flowgraph) on the reference's branching graphs: examples/multi.rs, the WLAN
receiver front end (examples/wlan/src/bin/rx.rs:73-93), the SSB transmitter (examples/ssb/transmit.rs:84-97,
:129-131), SignalSource -> Head -> VectorSink, buffer compaction with three readers, and the error paths."""
import numpy as np
import pytest
import torch

import futuresdr_b200 as fb
from futuresdr_b200.blocks import Apply, ApplyOp, Fir, Head, SignalSourceBuilder
from futuresdr_b200.edges import Flowgraph, VectorSink, VectorSource

pytestmark = pytest.mark.gpu


def _bits_equal(got, want):
    g = np.ascontiguousarray(got).view(np.uint32)
    w = np.ascontiguousarray(want).view(np.uint32)
    assert g.shape == w.shape and np.array_equal(g, w)


def _fir_tol(taps, x):
    return 1e-5 * float(np.sum(np.abs(taps))) * float(np.max(np.abs(x)))


def _multi(buffer_items, chunks):
    n_items = 20_000                                            # examples/multi.rs
    orig = np.random.default_rng(0).random(n_items, dtype=np.float32)
    fg = Flowgraph()
    src = VectorSource(orig)
    dup = fb.StreamDuplicator(np.float32, 3)
    snks = [VectorSink(np.float32, n_items, chunk_items=c) for c in chunks]
    fg.connect(src, dup)
    for k, s in enumerate(snks):
        fg.connect(dup, ("outputs", k), s)
    calls = fg.run(buffer_items=buffer_items)
    for s in snks:
        v = s.items()
        assert v.size == n_items and np.array_equal(v, orig)
    return calls


def test_multi_rs():
    _multi(4 << 20, [1 << 20] * 3)


def test_compaction_with_three_readers():
    """One output port read by three sinks that drain at different rates through a 2500-item buffer: the writer is
    held back by the slowest reader and compaction moves the unread tail to the front many times."""
    n = 50_000
    x = np.random.default_rng(1).standard_normal(n).astype(np.float32)
    fg = Flowgraph()
    src = VectorSource(x)
    snks = [VectorSink(np.float32, chunk_items=c) for c in (700, 1100, 333)]
    for s in snks:
        fg.connect(src, s)
    calls = fg.run(buffer_items=2500)
    assert calls > 3 * n // 1250
    for s in snks:
        assert np.array_equal(s.items(), x)
    _multi(2500, [700, 1100, 333])                              # and behind a StreamDuplicator


def test_wlan_rx_front_end():
    """rx.rs:73-93 with Fir(ones(64)) (f32) and Fir(ones(48)) (c32) standing in for wlan's private MovingAverage<f32>(64)
    and MovingAverage<Complex32>(48) (a sum over the same window; the example's block is not part of the library)."""
    n = 4 << 20
    rng = np.random.default_rng(11)
    x = ((rng.standard_normal(n) + 1j * rng.standard_normal(n)) / np.sqrt(2)).astype(np.complex64)
    fg = Flowgraph()
    src = VectorSource(x)
    delay = fb.Delay(np.complex64, 16)
    complex_to_mag_2 = Apply(ApplyOp.NormSqr)
    float_avg = Fir(fb.FirFilter(np.ones(64, np.float32), sample_dtype=np.float32))
    mult_conj = fb.Combine(fb.CombineOp.ConjMulC32)
    complex_avg = Fir(fb.FirFilter(np.ones(48, np.float32), sample_dtype=np.complex64))
    divide_mag = fb.Combine(fb.CombineOp.MagDivC32F32)
    snk = {k: VectorSink(dt) for k, dt in [("delay", np.complex64), ("mult_conj", np.complex64),
                                           ("complex_avg", np.complex64), ("float_avg", np.float32),
                                           ("divide_mag", np.float32)]}
    fg.connect(src, delay)                                      # the source stream is read by three blocks
    fg.connect(src, complex_to_mag_2)
    fg.connect(src, mult_conj, "in0")
    fg.connect(complex_to_mag_2, float_avg)
    fg.connect(mult_conj, complex_avg)
    fg.connect(delay, mult_conj, "in1")
    fg.connect(complex_avg, divide_mag, "in0")
    fg.connect(float_avg, divide_mag, "in1")
    fg.connect(delay, snk["delay"])
    fg.connect(mult_conj, snk["mult_conj"])
    fg.connect(complex_avg, snk["complex_avg"])
    fg.connect(float_avg, snk["float_avg"])
    fg.connect(divide_mag, snk["divide_mag"])
    fg.run(buffer_items=n + 4096)
    got = {k: s.items() for k, s in snk.items()}
    # Delay(16): 16 zeros, then the stream
    d = np.concatenate([np.zeros(16, np.complex64), x])
    _bits_equal(got["delay"], d)
    # Combine(a * b.conj()): min(n, n + 16) items, bit for bit
    with np.errstate(all="ignore"):
        b = d[:n]
        mc = np.empty(n, np.complex64)
        mc.real = x.real * b.real - x.imag * (-b.imag)
        mc.imag = x.real * (-b.imag) + x.imag * b.real
    _bits_equal(got["mult_conj"], mc)
    # the two FIR stand-ins, against f64 window sums
    ca_ref = np.convolve(mc.astype(np.complex128), np.ones(48), "valid")
    assert got["complex_avg"].size == n - 47
    assert np.max(np.abs(got["complex_avg"] - ca_ref)) <= _fir_tol(np.ones(48), mc)
    p = (x.real.astype(np.float64) ** 2 + x.imag.astype(np.float64) ** 2)
    fa_ref = np.convolve(p, np.ones(64), "valid")
    assert got["float_avg"].size == n - 63
    assert np.max(np.abs(got["float_avg"] - fa_ref)) <= _fir_tol(np.ones(64), p)
    # Combine(a.norm() / b): its inputs arrive with n - 47 and n - 63 items; m = min of the two (combine.rs:114)
    assert got["divide_mag"].size == min(n - 47, n - 63)
    m = n - 63
    ca, fa = got["complex_avg"][:m], got["float_avg"][:m]
    _bits_equal(got["divide_mag"], np.hypot(ca.real, ca.imag) / fa)


@pytest.mark.parametrize("mode", ["usb", "lsb"])
def test_ssb_transmit_topology(mode):
    n = 200_000
    rng = np.random.default_rng(3)
    audio = rng.uniform(-1, 1, n).astype(np.float32)
    window = fb.windows.hamming(167, False)
    taps = fb.firdes.hilbert(window)
    fg = Flowgraph()
    src = VectorSource(audio)
    split = fb.Split(fb.SplitOp.DupF32)                         # Split::new(|v| (*v, *v))
    hilbert = Fir(fb.FirFilter(taps, sample_dtype=np.float32))
    delay = fb.Delay(np.float32, len(window) // 2 * -1)         # window.len() as isize / -2 == -83
    to_complex = fb.Combine(fb.CombineOp.ToC32 if mode == "usb" else fb.CombineOp.ToC32NegQ)
    snk = VectorSink(np.complex64)
    fg.connect(src, split)
    fg.connect(split, "output0", delay)                         # split.output0 > delay > in0.to_complex
    fg.connect(delay, to_complex, "in0")
    fg.connect(split, "output1", hilbert)                       # split.output1 > hilbert > in1.to_complex
    fg.connect(hilbert, to_complex, "in1")
    fg.connect(to_complex, snk)
    fg.run(buffer_items=1 << 16)
    y = snk.items()
    assert y.size == n - 166                                    # min(n - 83, n - 166)
    _bits_equal(y.real.copy(), audio[83:83 + y.size])
    q = np.convolve(audio.astype(np.float64), taps.astype(np.float64), "valid")
    want_q = q if mode == "usb" else -q
    # AUTO may pick the split-bf16 tensor path for 167 taps: its bound is 3e-5 of ||taps||_1 max|x| (b200sdr.h)
    assert np.max(np.abs(y.imag - want_q)) <= 3 * _fir_tol(taps, audio)


def test_never_finishing_source_is_finished_by_its_reader():
    fg = Flowgraph()
    src = SignalSourceBuilder.sin(1000.0, 48000.0, 0.5, 0.0)
    head = Head(np.float32, 10_000)
    snk = VectorSink(np.float32)
    fg.connect(src, head)
    fg.connect(head, snk)
    fg.run(buffer_items=4096)                                   # returns: Head's finish finished the source
    ref = SignalSourceBuilder.sin(1000.0, 48000.0, 0.5, 0.0)
    o = torch.empty(10_000, device="cuda")
    ref.generate(o)
    torch.cuda.synchronize()
    _bits_equal(snk.items(), o.cpu().numpy())


def test_deadlocked_graph_raises():
    fg = Flowgraph()
    fg.connect(VectorSource(np.ones(1000, np.float32)), Fir(fb.FirFilter(np.ones(64, np.float32), sample_dtype=np.float32)))
    fg.connect(fg.blocks[1], VectorSink(np.float32))
    with pytest.raises(RuntimeError, match="no block can make progress"):
        fg.run(buffer_items=32)                                 # 64 taps never fit a 32-item buffer


def test_item_types_and_ports_are_checked():
    fg = Flowgraph()
    src = VectorSource(np.ones(10, np.float32))
    with pytest.raises(TypeError, match="item types differ"):
        fg.connect(src, fb.Combine(fb.CombineOp.ConjMulC32), "in0")
    with pytest.raises(ValueError, match="no stream input"):
        fg.connect(src, fb.Combine(fb.CombineOp.AddF32), "in2")
    comb = fb.Combine(fb.CombineOp.AddF32)
    fg.connect(src, comb, "in0")
    fg.connect(comb, VectorSink(np.float32))
    with pytest.raises(ValueError, match="in1 is not connected"):
        fg.run()
