"""The WLAN transmitter on the device (csrc/wlan.cu) against the C oracle of mac.rs / encoder.rs / mapper.rs /
prefix.rs (tests/wlan_oracle.c): subcarrier bytes bit for bit; samples bit for bit against the oracle's Prefix fed by
the library's own Fft(64, Inverse, shift, sqrtf(1/52)) block (so the fused kernel equals the unfused device chain) and
within the FFT's rounding bound of an f64 DFT; the stream under every slicing, the stale pad bits across pushes, the
handlers, the transmit graph, the WLAN receive front end on its output and a receive model decoding it."""
import math

import numpy as np
import pytest
import torch

import futuresdr_b200 as fb
from futuresdr_b200 import blocks as B, wlan
from futuresdr_b200.blocks import Apply, ApplyOp
from futuresdr_b200.edges import FileSink, Flowgraph, VectorSink, VectorSource

import wlan_model as wm
import wlan_oracle as wo

pytestmark = pytest.mark.gpu

LENGTHS = [0, 1, 2, 3, 5, 17, 100, 499, 1000, 1499, 1500]
NORM = float(np.sqrt(np.float32(1.0) / np.float32(52.0)))
U = 2.0 ** -24


def _payload(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def _tx(mcs=wlan.Mcs.QPSK_1_2, pf=37, pt=11):
    return B.WlanTransmitter(wo.SRC, wo.DST, wo.BSS, int(mcs), pf, pt)


_FFT = {}


def device_ifft(mapped: np.ndarray) -> np.ndarray:
    """The library's Fft block as tx.rs configures it, over n x 64 mapped symbols."""
    if "f" not in _FFT:
        _FFT["f"] = B.Fft(64, B.FftDirection.Inverse, True, NORM)
    x = torch.from_numpy(np.ascontiguousarray(mapped.reshape(-1))).cuda()
    y = torch.empty_like(x)
    assert _FFT["f"].transform(x, y) == x.numel()
    torch.cuda.synchronize()
    return y.cpu().numpy().reshape(-1, 64)


def oracle_frames(frames, mcs, otx=None):
    otx = otx or wo.Tx()
    return [(otx.frame(p, m)[1], m) for p, m in zip(frames, mcs)]


def oracle_stream(frames, mcs, pf, pt, otx=None):
    """The oracle's samples, with every frame's symbols transformed by one device Fft call."""
    fr = oracle_frames(frames, mcs, otx)
    maps = [wo.mapped(s, m) for s, m in fr]
    y = device_ifft(np.concatenate(maps))
    out, o = [], 0
    for mp in maps:
        out.append(wo.prefix(y[o:o + len(mp)], pf, pt))
        o += len(mp)
    return np.concatenate(out), maps


def _run(tx, caps):
    """exec over the given caps (cycled) until nothing is pending; the concatenated output on the host."""
    total = tx.pending()
    out = torch.full((total + 1,), complex(7, 7), dtype=torch.complex64, device="cuda")
    pos, k = 0, 0
    while pos < total:
        c = caps[k % len(caps)]
        k += 1
        p, _ = tx.exec(out[pos:pos + c])
        assert p == min(c, total - pos)
        pos += p
    torch.cuda.synchronize()
    assert complex(out[total].item()) == complex(7, 7)
    return out[:total].cpu().numpy()


def _same(a, b):
    assert a.shape == b.shape, (a.shape, b.shape)
    bad = np.flatnonzero(a.view(np.uint64) != b.view(np.uint64))
    assert bad.size == 0, (bad.size, int(bad[0]), a[bad[0]], b[bad[0]])


def test_encoder_symbols_equal_the_oracle_for_every_mcs(rng):
    frames = [_payload(rng, n) for n in LENGTHS for _ in range(8)]
    mcs = [m for _ in LENGTHS for m in range(8)]
    rng.shuffle(frames)                               # stale pad bits from every kind of earlier frame
    for seq, seed in ((0, 1), (4090, 120)):           # and both counters across their wraps
        got = wlan.encode(frames, mcs, sequence_number=seq, scrambler_seed=seed)
        want = oracle_frames(frames, mcs, wo.Tx(seq=seq, seed=seed))
        for g, (w, _) in zip(got, want):
            assert np.array_equal(g.cpu().numpy(), w)


def test_encode_refusals():
    with pytest.raises(fb.B200SdrError):
        wlan.encode([b"x" * 1501], 0)
    with pytest.raises(fb.B200SdrError):
        wlan.encode([b"x"], 8)
    with pytest.raises(fb.B200SdrError):
        wlan.encode([b"x"], 0, scrambler_seed=0)
    with pytest.raises(fb.B200SdrError):
        wlan.encode([b"x"], 0, sequence_number=4096)


def _f64_bound_check(got, maps, pf, pt):
    """The body of every OFDM symbol (its 64 samples after the cyclic prefix) against 0.6 sqrt(1/52) IFFT in f64,
    normwise per symbol: the library's FFT bound (tests/test_gpu_spectrum_bins.py) plus the two f32 scalings."""
    g4 = 4 * U / (1 - 4 * U)
    mu = 15 * U + 4 * math.sqrt(2) * 2 * U / (1 - 2 * U)
    eta = mu + g4 * (math.sqrt(2) + mu)
    rel = 6 * eta / (1 - 6 * eta) + 5 * U
    o = 0
    for mp in maps:
        d0 = o + pf + 320
        body = np.stack([got[d0 + 80 * k + 16:d0 + 80 * k + 80] for k in range(len(mp))]).astype(np.complex128)
        ref = 0.6 * np.stack([wo.ifft_f64(v) for v in mp])
        err = np.linalg.norm(body - ref, axis=1)
        assert np.all(err <= rel * np.linalg.norm(ref, axis=1)), float(np.max(err / np.linalg.norm(ref, axis=1)))
        o += wo.frame_len(len(mp), pf, pt)


def test_samples_equal_the_unfused_device_chain(rng):
    frames = [_payload(rng, n) for n in (0, 3, 100, 1500, 57, 1499, 600, 28)]
    mcs = [int(m) for m in rng.integers(-1, 8, len(frames))]
    tx = _tx(wlan.Mcs.QAM16_3_4, 37, 11)
    tx.push(*frames, mcs=mcs)
    got = _run(tx, [1 << 24])
    eff = [5 if m == -1 else m for m in mcs]
    want, maps = oracle_stream(frames, eff, 37, 11)
    _same(got, want)
    _f64_bound_check(got, maps, 37, 11)
    sync = np.array([complex(*v) for v in wo.golden()["sync_words"]], np.complex64)
    assert np.array_equal(got[37:37 + 320], sync * np.float32(0.6))


def test_every_slicing_gives_the_same_stream(rng):
    frames = [_payload(rng, int(n)) for n in rng.integers(0, 300, 6)]
    mcs = [int(m) for m in rng.integers(0, 8, 6)]
    tx = _tx(pf=90, pt=33)
    tx.push(*frames, mcs=mcs)
    ref = _run(tx, [1 << 24])
    _same(ref, oracle_stream(frames, mcs, 90, 33)[0])
    lens = [int(b["len"]) for b in tx.bursts()]
    caps_sets = [[1], [7], [80], [lens[0], lens[1], 1, lens[2] - 1], [lens[0] - 1, 2], [4095, 4097, 8193],
                 [int(c) for c in rng.integers(0, 5000, 60)]]
    for caps in caps_sets:
        t2 = _tx(pf=90, pt=33)
        t2.push(*frames, mcs=mcs)
        if caps == [1]:
            t2.push()                                 # an empty push changes nothing
        _same(_run(t2, caps), ref)


def test_4096_frames_of_random_length_and_mcs_in_one_push(rng):
    frames = [_payload(rng, int(n)) for n in rng.integers(0, 400, 4096)]
    mcs = [int(m) for m in rng.integers(0, 8, 4096)]
    tx = _tx(pf=20, pt=5)
    tx.push(*frames, mcs=mcs)
    got = _run(tx, [3_000_017, 1 << 30])
    want, _ = oracle_stream(frames, mcs, 20, 5)
    _same(got, want)
    b = tx.bursts()
    assert b.size == 4096 and int(b["index"][0]) == 0 and int(b["len"].sum()) == got.size
    assert list(b["len"]) == [wlan.frame_len(m, len(f), 20, 5) for f, m in zip(frames, mcs)]


def test_stale_pad_bits_carry_across_pushes(rng):
    """A long frame, then short ones whose pad bits come from it, pushed one by one and in groups, with frames of
    every length in between: the device's shadow of the bit buffer must give the reference's pad bits."""
    seqs = [[_payload(rng, 1500)], [_payload(rng, 10)], [_payload(rng, 0), _payload(rng, 40)],
            [_payload(rng, int(n)) for n in rng.integers(0, 1501, 30)], [_payload(rng, 3)], [_payload(rng, 1)]]
    mcs = [[int(m) for m in rng.integers(0, 8, len(s))] for s in seqs]
    tx = _tx(pf=5, pt=5)
    for s, m in zip(seqs, mcs):
        tx.push(*s, mcs=m)
    got = _run(tx, [1 << 24])
    flat = [p for s in seqs for p in s]
    fm = [m for ms in mcs for m in ms]
    want, _ = oracle_stream(flat, fm, 5, 5)
    _same(got, want)
    # the short frame's symbols depend on the long frame before it through its pad bits alone
    other = oracle_frames([_payload(rng, 1500), flat[1]], fm[:2])[1][0]
    assert not np.array_equal(other, oracle_frames(flat[:2], fm[:2])[1][0])


def test_pads_0_0_have_the_one_sample_tail(rng):
    p = b"lol"
    tx = _tx(wlan.Mcs.QPSK_1_2, 0, 0)
    tx.push(p)
    got = _run(tx, [1 << 20])
    want, _ = oracle_stream([p], [2], 0, 0)
    _same(got, want)
    assert got.size == wlan.frame_len(2, 3, 0, 0) == 320 + 80 * (1 + 6) + 1     # 270 data bits: 6 symbols


def test_refusals_leave_the_transmitter_as_it_was(rng):
    with pytest.raises(fb.B200SdrError):
        _tx(8)
    with pytest.raises(ValueError):
        B.WlanTransmitter(b"12345", wo.DST, wo.BSS, 0, 0, 0)
    tx = _tx(pf=3, pt=3)
    a = _payload(rng, 50)
    with pytest.raises(fb.B200SdrError):
        tx.push(a, b"x" * 1501)
    with pytest.raises(fb.B200SdrError):
        tx.push(a, mcs=[9])
    with pytest.raises(ValueError):
        tx.push(a, mcs=[1, 2])
    assert tx.pending() == 0
    tx.push(a)                                        # sequence number 0 and seed 1: nothing was consumed
    out = torch.empty(tx.pending() + 1, dtype=torch.complex64, device="cuda")
    with pytest.raises(fb.B200SdrError):              # an output slice 4 bytes off the 8-byte grid
        tx.exec(_Slice(out.data_ptr() + 4, 16))
    _same(_run(tx, [1 << 20]), oracle_stream([a], [2], 3, 3)[0])


class _Slice:
    """A slice stand-in for exec: a raw device pointer and an item count."""

    def __init__(self, ptr, n):
        self.ptr, self.n = ptr, n

    def data_ptr(self):
        return self.ptr

    def numel(self):
        return self.n


def test_finish_reset_and_destroy_in_flight(rng):
    tx = _tx()
    p = _payload(rng, 30)
    tx.push(p)
    total = tx.pending()
    out = torch.empty(total, dtype=torch.complex64, device="cuda")
    assert tx.exec(out[:100]) == (100, False)
    tx.finish()
    assert tx.exec(out[100:200]) == (100, False)
    assert tx.exec(out[200:]) == (total - 200, True)
    assert tx.exec(out[:0]) == (0, True)
    tx.push(p)                                        # frames queued after finish still go out
    assert tx.pending() == total and tx.exec(out[:10]) == (10, False)
    tx.reset()
    assert tx.pending() == 0 and tx.exec(out) == (0, False) and tx.bursts().size == 0
    tx.push(p)                                        # the created state: sequence 0, seed 1, zero bit buffer
    _same(_run(tx, [1 << 20]), oracle_stream([p], [2], 37, 11)[0])
    t2 = _tx(pf=5000, pt=5000)
    t2.push(*[_payload(rng, 1500) for _ in range(64)], mcs=[0] * 64)
    big = torch.empty(t2.pending(), dtype=torch.complex64, device="cuda")
    t2.exec(big)
    t2.close()                                        # waits for the exec, then frees
    torch.cuda.synchronize()


def test_transmitter_graph_into_vector_and_file_sinks(rng, tmp_path):
    frames = [_payload(rng, int(n)) for n in (10, 200, 1500, 0)]
    fg = Flowgraph()
    tx = wlan.transmitter(fg, pad_front=500, pad_tail=300)
    vs = VectorSink(np.complex64, chunk_items=1 << 15)
    fs = FileSink(tmp_path / "wlan.cf32", np.complex64, chunk_items=1 << 15)
    fg.connect(tx, vs)
    fg.connect(tx, fs)
    tx.push(*frames[:2])
    tx.push(*frames[2:], mcs=[wlan.Mcs.QAM16_1_2, -1])
    tx.finish()
    fg.run(buffer_items=1 << 16)
    want, _ = oracle_stream(frames, [2, 2, 4, 2], 500, 300)
    got = vs.items()
    _same(got, want)
    assert np.array_equal(np.fromfile(tmp_path / "wlan.cf32", np.complex64).view(np.uint64), got.view(np.uint64))
    b = tx.bursts()
    assert list(b["len"]) == [wlan.frame_len(m, len(f), 500, 300) for f, m in zip(frames, [2, 2, 4, 2])]
    assert list(b["index"]) == list(np.concatenate([[0], np.cumsum(b["len"])[:-1]]))


def test_wlan_rx_front_end_sees_the_short_training_field(rng):
    """rx.rs:73-93's front end (Delay 16, NormSqr -> MovingAverage 64, conj-multiply -> MovingAverage 48, magnitude
    ratio) on the transmitter's bursts: divide_mag exceeds SyncShort's threshold 0.56 over each short training field
    and nowhere in the pads."""
    pf, pt = 2000, 2000
    frames = [_payload(rng, int(n)) for n in (100, 600, 1500)]
    tx = _tx(wlan.Mcs.QPSK_1_2, pf, pt)
    tx.push(*frames)
    x = _run(tx, [1 << 24])
    rng2 = np.random.default_rng(3)
    x = (x + 1e-4 * (rng2.standard_normal(x.size) + 1j * rng2.standard_normal(x.size))).astype(np.complex64)
    fg = Flowgraph()
    src = VectorSource(x)
    delay = fb.Delay(np.complex64, 16)
    mag2 = Apply(ApplyOp.NormSqr)
    float_avg = fb.MovingAverage(np.float32, 64)
    mult_conj = fb.Combine(fb.CombineOp.ConjMulC32)
    complex_avg = fb.MovingAverage(np.complex64, 48)
    divide_mag = fb.Combine(fb.CombineOp.MagDivC32F32)
    snk = VectorSink(np.float32)
    fg.connect(src, delay)
    fg.connect(src, mag2)
    fg.connect(src, mult_conj, "in0")
    fg.connect(mag2, float_avg)
    fg.connect(mult_conj, complex_avg)
    fg.connect(delay, mult_conj, "in1")
    fg.connect(complex_avg, divide_mag, "in0")
    fg.connect(float_avg, divide_mag, "in1")
    fg.connect(divide_mag, snk)
    fg.run(buffer_items=x.size + 4096)
    d = snk.items()
    for b in tx.bursts():
        s = int(b["index"])
        stf = d[s + pf + 64:s + pf + 160]               # the averages are full of short training field samples
        assert np.all(stf > 0.56), float(stf.min())
        assert np.all(d[s + 64:s + pf] < 0.56)          # pad front (noise only)
        e = s + int(b["len"])
        assert np.all(d[e - pt + 64:e] < 0.56)          # pad tail


@pytest.mark.parametrize("snr_db", [None, 30])
def test_receive_model_decodes_the_device_samples(rng, snr_db):
    frames = [_payload(rng, int(n)) for n in (0, 77, 1500)] * 3
    mcs = [m for m in range(8)] + [2]
    tx = _tx(wlan.Mcs.QPSK_1_2, 400, 400)
    tx.push(*frames, mcs=mcs)
    x = _run(tx, [1 << 24]).astype(np.complex128)
    if snr_db is not None:
        # per-sample noise power at the given SNR against the data symbols' average power (0.36 after Prefix)
        sig = 0.36
        n0 = sig / 10 ** (snr_db / 10)
        x = x + np.sqrt(n0 / 2) * (rng.standard_normal(x.size) + 1j * rng.standard_normal(x.size))
    for b, p, m in zip(tx.bursts(), frames, mcs):
        r = wm.decode_burst(x, int(b["index"]), 400)
        assert r is not None and r[0] == p and r[1] == m
