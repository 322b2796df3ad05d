"""The ZigBee transmitter on the device (csrc/zigbee_tx.cu) bit for bit against the C oracle of mac.rs / modulator.rs /
iq_delay.rs (tests/zigbee_tx_oracle.c), compared as uint32 so that the sign of every zero counts: payloads of every
length at pads 0, 1 and 40000, 300 frames (sequence wrap), every slicing, 4096 frames in one exec, pushes between
execs, the drop rule, the handlers, the refusals, the transmit graph into VectorSink and FileSink, and the transceiver
loop (trx.rs) from payloads through ``zigbee.front_end`` to decoded frames, clean and through a channel."""
import ctypes as C

import numpy as np
import pytest
import torch

import futuresdr_b200 as fb
from futuresdr_b200 import _lib, zigbee
from futuresdr_b200._lib import lib
from futuresdr_b200.blocks import ZigbeeTransmitter
from futuresdr_b200.edges import FileSink, Flowgraph, VectorSink, VectorSource

import zigbee_oracle as zo
import zigbee_tx_oracle as zt

pytestmark = pytest.mark.gpu

MM = (zigbee.MM_OMEGA, zigbee.MM_GAIN_OMEGA, zigbee.MM_MU, zigbee.MM_GAIN_MU, zigbee.MM_OMEGA_RELATIVE_LIMIT)


def _pays(rng, lengths):
    return [rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in lengths]


def _run(tx, caps):
    """exec over the given caps (cycled) until nothing is pending; the concatenated output on the host."""
    total = tx.pending()
    out = torch.full((total + 1,), complex(7, 7), dtype=torch.complex64, device="cuda")
    pos, k = 0, 0
    while pos < total:
        c = int(caps[k % len(caps)])
        k += 1
        p, _ = tx.exec(out[pos:pos + c])
        assert p == min(c, total - pos)
        pos += p
    torch.cuda.synchronize()
    assert complex(out[total].item()) == complex(7, 7)
    return out[:total].cpu().numpy()


def _same(a, b):
    assert a.shape == b.shape, (a.shape, b.shape)
    bad = np.flatnonzero(a.view(np.uint32) != np.ascontiguousarray(b, np.complex64).view(np.uint32))
    assert bad.size == 0, (bad.size, int(bad[0]) // 2, a[bad[0] // 2], b[bad[0] // 2])


def _oracle(pays, pad, caps=(1 << 22,)):
    t = zt.Tx(pad)
    dropped = t.push(*pays)
    x, b = t.stream(caps)
    return x, b, dropped


@pytest.mark.parametrize("pad", [0, 1, 40000])
def test_every_payload_length_bit_for_bit(pad):
    rng = np.random.default_rng(pad + 1)
    lengths = list(range(0, 117))
    rng.shuffle(lengths)
    pays = _pays(rng, lengths)
    tx = ZigbeeTransmitter(pad)
    assert tx.push(*pays) == 0
    assert tx.pending() == sum(zigbee.frame_len(n, pad) for n in lengths)
    got = _run(tx, [1 << 30])
    want, wb, _ = _oracle(pays, pad)
    _same(got, want)
    assert [(int(b["index"]), int(b["len"])) for b in tx.bursts()] == wb
    assert tx.pending() == 0


def test_300_frames_wrap_the_sequence_number_and_drops_match():
    rng = np.random.default_rng(2)
    lengths = [int(n) for n in rng.integers(0, 130, 300)]
    pays = _pays(rng, lengths)
    tx = ZigbeeTransmitter(1)
    n_drop = tx.push(*pays)
    want, wb, w_drop = _oracle(pays, 1)
    assert n_drop == w_drop == sum(n > 116 for n in lengths) > 0
    assert sum(n <= 116 for n in lengths) > 256
    _same(_run(tx, [1 << 30]), want)
    assert [(int(b["index"]), int(b["len"])) for b in tx.bursts()] == wb


@pytest.mark.parametrize("pad", [0, 1, 40000])
def test_every_slicing_gives_the_same_stream(pad):
    rng = np.random.default_rng(3 + pad)
    pays = _pays(rng, [0, 116, 5, 77, 1])
    want, wb, _ = _oracle(pays, pad)
    lens = [n for _, n in wb]
    edges = [[1], [7], [4096], [lens[0] - 1, 2, lens[1] - 3, 1], [pad, 1, 1, 128, 2, 1],
             [int(c) for c in rng.integers(1, 70000, 50)]]
    for caps in edges:
        caps = [c for c in caps if c > 0] or [1]
        if caps == [1] and want.size > 400_000:
            caps = [1] * 500 + [33_333]                  # single-sample execs across the first frame's edges
        tx = ZigbeeTransmitter(pad)
        tx.push(*pays)
        _same(_run(tx, caps), want)
    # single-sample execs at every frame edge of the stream, the rest in large pieces
    tx = ZigbeeTransmitter(pad)
    tx.push(*pays)
    cuts = sorted({c for s, n in wb for e in (s, s + pad, s + n - pad - 2, s + n) for c in (e - 2, e - 1, e, e + 1)
                   if 0 < c < want.size})
    out = torch.empty(want.size, dtype=torch.complex64, device="cuda")
    pos = 0
    for c in cuts + [want.size]:
        while pos < c:
            step = 1 if pos + 1 in cuts or pos in cuts else c - pos
            p, _ = tx.exec(out[pos:pos + step])
            pos += p
    torch.cuda.synchronize()
    _same(out.cpu().numpy(), want)


def test_4096_frames_in_one_exec():
    rng = np.random.default_rng(4)
    lengths = [int(n) for n in rng.integers(0, 117, 4096)]
    pays = _pays(rng, lengths)
    tx = ZigbeeTransmitter(100)
    tx.push(*pays)
    got = _run(tx, [1 << 31])
    want, wb, _ = _oracle(pays, 100)
    _same(got, want)
    b = tx.bursts()
    assert b.size == 4096 and [(int(x["index"]), int(x["len"])) for x in b] == wb


def test_pushes_between_execs_and_reset():
    rng = np.random.default_rng(5)
    groups = [_pays(rng, rng.integers(0, 117, k)) for k in (3, 1, 0, 7, 2)]
    flat = [p for g in groups for p in g]
    want, wb, _ = _oracle(flat, 500)
    tx = ZigbeeTransmitter(500)
    out = torch.empty(want.size, dtype=torch.complex64, device="cuda")
    pos = 0
    for g in groups:
        tx.push(*g)
        step = max(1, tx.pending() // 2 + 3)             # half of what is queued: frames are cut mid-stream
        p, f = tx.exec(out[pos:pos + step])
        assert not f
        pos += p
    while tx.pending():
        pos += tx.exec(out[pos:pos + 12345])[0]
    torch.cuda.synchronize()
    _same(out.cpu().numpy(), want)
    assert [(int(b["index"]), int(b["len"])) for b in tx.bursts()] == wb
    tx.reset()                                            # the created state: sequence number 0
    assert tx.pending() == 0 and tx.bursts().size == 0
    assert tx.exec(out) == (0, False)
    tx.push(*flat)
    _same(_run(tx, [99_999]), want)


def test_finish_rule_and_handlers():
    tx = ZigbeeTransmitter(10)
    out = torch.empty(1 << 16, dtype=torch.complex64, device="cuda")
    assert tx.exec(out) == (0, False)
    tx.finish()
    assert tx.exec(out) == (0, True)                      # finished with nothing queued
    tx.push(b"abc")
    n = zigbee.frame_len(3, 10)
    assert tx.pending() == n
    assert tx.exec(out[:n - 1]) == (n - 1, False)         # the tail pad is still to come
    assert tx.exec(out[n - 1:]) == (1, True)
    assert tx.push(b"x" * 117, b"y" * 200) == 2 and tx.pending() == 0


def test_payload_types():
    tx = ZigbeeTransmitter(0)
    with pytest.raises(TypeError):
        tx.push("FutureSDR 0")
    with pytest.raises(TypeError):
        tx.push(5)
    assert tx.pending() == 0
    tx.push(bytearray(b"ab"), memoryview(b"cd"), np.frombuffer(b"ef", np.uint8))
    want, _, _ = _oracle([b"ab", b"cd", b"ef"], 0)
    _same(_run(tx, [1 << 20]), want)


class _Slice:
    """A slice stand-in for exec: a raw device pointer and an item count."""

    def __init__(self, ptr, n):
        self.ptr, self.n = ptr, n

    def data_ptr(self):
        return self.ptr

    def numel(self):
        return self.n


def test_refusals_and_cleanup():
    ctx = fb.default_context()
    base = ctx.bytes_held
    h = C.c_void_p()
    assert lib.b2s_zigbee_tx_create(ctx.handle, 1 << 32, C.byref(h)) == _lib.EINVAL and h.value is None
    assert lib.b2s_zigbee_tx_create(None, 0, C.byref(h)) == _lib.EINVAL
    assert lib.b2s_zigbee_tx_create(ctx.handle, 0, None) == _lib.EINVAL
    with pytest.raises(fb.B200SdrError):
        ZigbeeTransmitter(1 << 32)
    d, p, f, v = C.c_size_t(0), C.c_size_t(0), C.c_int32(0), C.c_uint64(0)
    lens = (C.c_size_t * 1)(3)
    assert lib.b2s_zigbee_tx_push(None, b"abc", lens, 1, C.byref(d)) == _lib.EINVAL
    assert lib.b2s_zigbee_tx_exec(None, None, 0, C.byref(p), C.byref(f)) == _lib.EINVAL
    assert lib.b2s_zigbee_tx_pending(None, C.byref(v)) == _lib.EINVAL
    assert lib.b2s_zigbee_tx_finish(None) == _lib.EINVAL
    assert lib.b2s_zigbee_tx_reset(None) == _lib.EINVAL
    assert lib.b2s_zigbee_tx_drain_bursts(None, None, 0, C.byref(d)) == _lib.EINVAL
    tx = ZigbeeTransmitter(7)
    assert lib.b2s_zigbee_tx_push(tx._h, None, lens, 1, C.byref(d)) == _lib.EINVAL     # 3 bytes from NULL
    assert lib.b2s_zigbee_tx_push(tx._h, b"abc", lens, 1, None) == _lib.EINVAL
    assert tx.pending() == 0
    tx.push(b"abc")
    out = torch.empty(tx.pending() + 1, dtype=torch.complex64, device="cuda")
    with pytest.raises(fb.B200SdrError):                  # an output slice 4 bytes off the 8-byte grid
        tx.exec(_Slice(out.data_ptr() + 4, 16))
    assert lib.b2s_zigbee_tx_exec(tx._h, None, 16, C.byref(p), C.byref(f)) == _lib.EINVAL
    _same(_run(tx, [1 << 20]), _oracle([b"abc"], 7)[0])   # nothing was produced by the refused calls
    big = ZigbeeTransmitter()
    big.push(*[b"z" * 116] * 64)
    o2 = torch.empty(big.pending(), dtype=torch.complex64, device="cuda")
    big.exec(o2)
    big.close()                                           # waits for the exec, then frees
    tx.close()
    torch.cuda.synchronize()
    assert ctx.bytes_held == base


def test_transmitter_graph_into_vector_and_file_sinks(tmp_path):
    rng = np.random.default_rng(6)
    pays = _pays(rng, [10, 116, 0, 60])
    fg = Flowgraph()
    tx = zigbee.transmitter(fg, pad=3000)
    vs = VectorSink(np.complex64, chunk_items=1 << 15)
    fs = FileSink(tmp_path / "zigbee.cf32", np.complex64, chunk_items=1 << 15)
    fg.connect(tx, vs)
    fg.connect(tx, fs)
    tx.push(*pays[:2])
    tx.push(*pays[2:])
    tx.finish()
    fg.run(buffer_items=1 << 16)
    want, wb, _ = _oracle(pays, 3000)
    got = vs.items()
    _same(got, want)
    assert np.array_equal(np.fromfile(tmp_path / "zigbee.cf32", np.complex64).view(np.uint32), got.view(np.uint32))
    assert [(int(b["index"]), int(b["len"])) for b in tx.bursts()] == wb


def _replayed(sinks, b):
    """The receiver oracle from the device's phase stream (its atan2 is not libm's): DC blocker, clock recovery and
    decoder bit for bit; returns the device's frames."""
    phase, dc, mm = (sinks[k].items() for k in ("phase", "dc", "mm"))
    assert np.array_equal(dc.view(np.uint32), zo.DcBlock(zigbee.DC_ALPHA).work(phase).view(np.uint32))
    want_mm, _, err = zo.mm_replay(MM, dc)
    assert err is None
    assert np.array_equal(mm.view(np.uint32), want_mm.view(np.uint32))
    got = b["decoder"].frames()
    want = zo.decode_replay(zigbee.DECODER_THRESHOLD, mm)
    assert [(int(g["index"]), bytes(g["bytes"][:g["len"]].tolist())) for g in got] == want
    return got


def test_transceiver_loop_decodes_every_frame():
    """trx.rs on the device: payloads -> ZigbeeTransmitter -> QuadDemod, DC blocker, ClockRecoveryMm, Decoder."""
    rng = np.random.default_rng(7)
    pays = _pays(rng, rng.integers(0, 117, 20))
    fg = Flowgraph()
    tx = zigbee.transmitter(fg)
    b = zigbee.front_end(fg, tx)
    sinks = {k: VectorSink(np.float32) for k in ("phase", "dc", "mm")}
    for k, v in sinks.items():
        fg.connect(b[k], v)
    tx.push(*pays)
    tx.finish()
    fg.run(buffer_items=1 << 17)
    got = _replayed(sinks, b)
    assert [bytes(g["bytes"][:g["len"]].tolist()) for g in got] == [zo.mac_frame(p, s)[5:] for s, p in enumerate(pays)]
    assert got["crc_ok"].all()


def test_transceiver_loop_through_a_channel():
    """The transmitter's samples through 12 dB SNR, a 20 kHz carrier offset and a +-50 ppm sample-rate offset into the
    front end: every frame still decodes with a good FCS."""
    rng = np.random.default_rng(8)
    pays = _pays(rng, rng.integers(1, 117, 20))
    tx = ZigbeeTransmitter(5000)
    tx.push(*pays)
    x = _run(tx, [1 << 24]).astype(np.complex128)
    sent = [zo.mac_frame(p, s)[5:] for s, p in enumerate(pays)]
    for ppm in (50, -50):
        t = np.arange(int(x.size / (1 + ppm * 1e-6))) * (1 + ppm * 1e-6)
        y = np.interp(t, np.arange(x.size), x.real) + 1j * np.interp(t, np.arange(x.size), x.imag)
        y = y * np.exp(1j * (2 * np.pi * 20e3 / 4e6 * np.arange(y.size) + rng.uniform(0, 2 * np.pi)))
        sigma = np.sqrt(0.5 * 10 ** (-12 / 10))
        y = (y + sigma * (rng.standard_normal(y.size) + 1j * rng.standard_normal(y.size))).astype(np.complex64)
        fg = Flowgraph()
        src = VectorSource(y)
        fg.add(src)
        b = zigbee.front_end(fg, src)
        sinks = {k: VectorSink(np.float32) for k in ("phase", "dc", "mm")}
        for k, v in sinks.items():
            fg.connect(b[k], v)
        fg.run(buffer_items=1 << 17)
        got = _replayed(sinks, b)
        ok = {bytes(g["bytes"][:g["len"]].tolist()) for g in got if g["crc_ok"]}
        assert all(f in ok for f in sent), (ppm, sum(f in ok for f in sent))
