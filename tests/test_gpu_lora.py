"""The LoRa transmitter on the device (csrc/lora.cu) against the C oracle of encoder.rs / modulator.rs
(tests/lora_oracle.c): symbols bit for bit, samples within 1 f32 ulp of libm's and of float32(cos / sin(float64(S))),
the stream bit-identical under every slicing, the handlers' rules and the transmit graph."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import futuresdr_b200 as fb
from futuresdr_b200 import _lib, blocks as B, lora
from futuresdr_b200.edges import FileSink, Flowgraph, VectorSink

import lora_oracle as lo

pytestmark = pytest.mark.gpu

CONFIGS = list(itertools.product(range(5, 13), range(1, 5), (False, True), (False, True), (False, True)))
LENGTHS = [0, 1, 2, 3, 4, 5, 7, 16, 63, 100, 254, 255]


def _payload(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def _tx(sf=7, cr=1, crc=True, ldro=False, implicit=False, os_=4, sync=(8, 16), pre=8, pad=0):
    return B.LoraTransmitter(sf, cr, crc, ldro, implicit, os_, sync, pre, pad)


def _oracle_stream(frames, sf, cr, crc, ldro, implicit, os_, sync, pre, pad):
    outs, phs = [], []
    for p in frames:
        o, ph = lo.modulate(lo.encode(p, sf, cr, crc, ldro, implicit), sf, os_, sync, pre, pad)
        outs.append(o)
        phs.append(ph)
    return np.concatenate(outs), np.concatenate(phs)


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


def test_symbols_equal_the_oracle_for_every_configuration(rng):
    for sf, cr, crc, implicit, ldro in CONFIGS:
        pays = [_payload(rng, n) for n in LENGTHS if not (crc and n < 2)]
        got = lora.encode(pays, sf, cr, crc, ldro, implicit)
        torch.cuda.synchronize()
        for p, g in zip(pays, got):
            want = lo.encode(p, sf, cr, crc, ldro, implicit)
            assert np.array_equal(g.cpu().numpy().view(np.uint16), want), (sf, cr, crc, implicit, ldro, len(p))


def test_encoder_refuses_what_the_reference_panics_on():
    d = torch.zeros(600, dtype=torch.uint8, device="cuda")
    s = torch.zeros(4096, dtype=torch.int16, device="cuda")
    for lens, crc in (([256], False), ([16, 256], False), ([1], True), ([0], True)):
        arr = (C.c_size_t * len(lens))(*lens)
        n = C.c_size_t(99)
        rc = _lib.lib.b2s_lora_encode(fb.default_context().handle, 7, 1, int(crc), 0, 0, C.c_void_p(d.data_ptr()), arr,
                                      len(lens), C.c_void_p(s.data_ptr()), s.numel(), C.byref(n))
        assert rc == _lib.EINVAL and n.value == 0
    tx = _tx(crc=True)
    with pytest.raises(_lib.B200SdrError):
        tx.push(b"ok frame", b"x")                    # the second payload is refused: nothing is queued
    with pytest.raises(_lib.B200SdrError):
        tx.push(bytes(256))
    assert tx.pending() == 0
    for implicit in (False, True):                    # an empty payload without CRC is a frame in both header modes
        t = _tx(crc=False, implicit=implicit)
        t.push(b"")
        assert t.pending() == lo.frame_len(7, 4, 8, 0, len(lo.encode(b"", 7, 1, False, False, implicit)))
        got = _run(t, [1 << 20])
        want, _ = _oracle_stream([b""], 7, 1, False, False, implicit, 4, (8, 16), 8, 0)
        assert lo.ulp_diff(got, want) <= 1


def test_samples_within_one_ulp_over_the_grid(rng):
    identical = total = 0
    max_s = 0.0
    for i, (sf, os_) in enumerate(itertools.product(range(5, 13), (1, 4, 8))):
        _, cr, crc, implicit, ldro = CONFIGS[(i * 37) % len(CONFIGS)]
        n = [0, 3, 16, 255][i % 4] if not crc else [2, 3, 16, 255][i % 4]
        if sf == 12 and os_ == 8:
            n = min(n, 16)
        pad = 10000 if i % 2 else 0
        sync = (8 % (1 << sf), 16 % (1 << sf))
        p = _payload(rng, n)
        tx = _tx(sf, cr, crc, ldro, implicit, os_, sync, lora.preamble_len(sf), pad)
        tx.push(p)
        got = _run(tx, [1 << 26])
        want, ph = _oracle_stream([p], sf, cr, crc, ldro, implicit, os_, sync, lora.preamble_len(sf), pad)
        assert got.size == want.size
        assert lo.ulp_diff(got, want) <= 1, (sf, os_, cr, crc, implicit, ldro, n, pad)
        assert lo.ulp_diff(got, lo.f64_samples(ph)) <= 1
        identical += int(np.sum(got.view(np.uint64) == want.view(np.uint64)))
        total += got.size
        max_s = max(max_s, float(np.max(np.abs(ph))))
        tx.close()
    print(f"bit-identical to libm cosf / sinf: {identical / total:.6f} of {total} samples; largest |S| {max_s:.1f}")


def _small_tx_and_frames(rng, n=5):
    frames = [_payload(rng, int(k)) for k in rng.integers(2, 12, n)]
    tx = _tx(5, 4, True, False, False, 1, (8, 16), 12, 3)
    tx.push(*frames)
    return tx, frames


def test_every_slicing_gives_the_same_stream(rng):
    tx, frames = _small_tx_and_frames(rng)
    ref = _run(tx, [1 << 20])
    want, _ = _oracle_stream(frames, 5, 4, True, False, False, 1, (8, 16), 12, 3)
    assert lo.ulp_diff(ref, want) <= 1
    lens = [int(b["len"]) for b in tx.bursts()]
    bounds = np.cumsum(lens)
    caps_sets = [[1], [lens[0], lens[1], 1, lens[2] - 1], [int(bounds[-1])], [7, 0, 13], [lens[0] - 1, 2]]
    caps_sets.append([int(c) for c in rng.integers(0, 3000, 50)])
    for caps in caps_sets:
        t2 = _tx(5, 4, True, False, False, 1, (8, 16), 12, 3)
        t2.push(*frames)
        got = _run(t2, caps)
        assert np.array_equal(got.view(np.uint64), ref.view(np.uint64)), caps
    t3 = _tx(5, 4, True, False, False, 1, (8, 16), 12, 3)
    t3.push(*frames)
    e = torch.empty(0, dtype=torch.complex64, device="cuda")
    assert t3.exec(e) == (0, False)
    assert np.array_equal(_run(t3, [1 << 20]).view(np.uint64), ref.view(np.uint64))


def test_4096_frames_of_random_lengths_in_one_push(rng):
    frames = [_payload(rng, int(k)) for k in rng.integers(0, 65, 4096)]
    tx = _tx(7, 2, False, False, False, 1, (8, 16), 8, 0)
    tx.push(*frames)
    got = _run(tx, [3_000_017, 1 << 30])
    want, ph = _oracle_stream(frames, 7, 2, False, False, False, 1, (8, 16), 8, 0)
    assert got.size == want.size
    assert lo.ulp_diff(got, want) <= 1
    assert lo.ulp_diff(got, lo.f64_samples(ph)) <= 1
    b = tx.bursts()
    assert b.size == 4096 and int(b["index"][0]) == 0 and int(b["len"].sum()) == got.size


def test_one_sf12_os8_frame_of_255_bytes(rng):
    p = _payload(rng, 255)
    tx = _tx(12, 1, True, True, False, 8, (8, 16), 8, 0)
    tx.push(p)
    got = _run(tx, [(1 << 22) + 5])
    want, ph = _oracle_stream([p], 12, 1, True, True, False, 8, (8, 16), 8, 0)
    assert got.size == want.size > 8_000_000
    assert lo.ulp_diff(got, want) <= 1
    assert lo.ulp_diff(got, lo.f64_samples(ph)) <= 1
    print(f"SF12 OS8 255 B: {got.size} samples, largest |S| {float(np.max(np.abs(ph))):.1f}")


def test_set_sync_word_applies_to_frames_not_yet_started(rng):
    frames = [_payload(rng, 4) for _ in range(3)]
    tx = _tx(7, 1, True, False, False, 1, (8, 16), 8, 0)
    tx.push(*frames)
    L = [lo.frame_len(7, 1, 8, 0, len(lo.encode(f, 7, 1, True, False, False))) for f in frames]
    out = torch.empty(sum(L), dtype=torch.complex64, device="cuda")
    p0, _ = tx.exec(out[:L[0] + 10])                 # frame 1 has started: it keeps (8, 16)
    tx.set_sync_word(0x34)                           # SynchWord::Public -> (24, 32)
    with pytest.raises(_lib.B200SdrError):
        tx.set_sync_word(bytes([200, 1]))            # 200 >= 2^7: refused, (24, 32) stays
    with pytest.raises(ValueError):
        tx.set_sync_word(300)
    p1, _ = tx.exec(out[p0:])
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    w0, _ = _oracle_stream(frames[:2], 7, 1, True, False, False, 1, (8, 16), 8, 0)
    w1, _ = _oracle_stream(frames[2:], 7, 1, True, False, False, 1, (24, 32), 8, 0)
    assert lo.ulp_diff(got, np.concatenate([w0, w1])) <= 1
    assert lo.ulp_diff(got[L[0] + L[1]:], _oracle_stream(frames[2:], 7, 1, True, False, False, 1, (8, 16), 8,
                                                         0)[0]) > 1
    tx2 = _tx(7, 1, True, False, False, 1, (8, 16), 8, 0)
    tx2.set_sync_word(bytes([0x08, 0x16]))           # expanded symbols as given
    tx2.push(frames[0])
    assert lo.ulp_diff(_run(tx2, [1 << 20]), _oracle_stream(frames[:1], 7, 1, True, False, False, 1, (8, 0x16), 8,
                                                            0)[0]) <= 1


def test_create_refusals():
    for kw in ({"sf": 5, "sync": (24, 32)}, {"os_": 0}, {"sf": 12, "os_": 512}, {"sf": 4}, {"cr": 5}):
        with pytest.raises(_lib.B200SdrError) as e:
            _tx(**kw)
        assert e.value.code == _lib.EINVAL
    with pytest.raises(ValueError):
        lora.transmitter(Flowgraph(), sf=lora.SpreadingFactor.SF5, sync_word=lora.SynchWord.PUBLIC)
    _tx(sf=12, os_=256)                              # 2^20 samples per symbol is the largest accepted


def test_finish_reset_and_destroy_in_flight(rng):
    tx = _tx()
    tx.push(_payload(rng, 8))
    total = tx.pending()
    out = torch.empty(total, dtype=torch.complex64, device="cuda")
    assert tx.exec(out[:100]) == (100, False)
    tx.finish()
    assert tx.exec(out[100:200]) == (100, False)
    assert tx.exec(out[200:]) == (total - 200, True)
    assert tx.exec(out[:0]) == (0, True)
    tx.push(_payload(rng, 8))                        # frames queued after finish still go out first
    assert tx.pending() == total and tx.exec(out[:10]) == (10, False)
    tx.reset()
    assert tx.pending() == 0 and tx.exec(out) == (0, False) and tx.bursts().size == 0
    p = _payload(rng, 8)
    tx.push(p)
    got = _run(tx, [1 << 20])
    assert lo.ulp_diff(got, _oracle_stream([p], 7, 1, True, False, False, 4, (8, 16), 8, 0)[0]) <= 1
    t2 = _tx(12, 1, True, True, False, 8)
    t2.push(*[_payload(rng, 255) for _ in range(4)])
    big = torch.empty(t2.pending(), dtype=torch.complex64, device="cuda")
    t2.exec(big)
    t2.close()                                       # waits for the exec, then frees
    torch.cuda.synchronize()


def test_transmitter_graph_into_vector_and_file_sinks(rng, tmp_path):
    frames = [_payload(rng, 16) for _ in range(6)]
    fg = Flowgraph()
    tx = lora.transmitter(fg, sf=lora.SpreadingFactor.SF7, os_factor=4, sync_word=lora.SynchWord.PRIVATE)
    vs = VectorSink(np.complex64, chunk_items=1 << 15)
    fs = FileSink(tmp_path / "lora.cf32", np.complex64, chunk_items=1 << 15)
    fg.connect(tx, vs)
    fg.connect(tx, fs)
    for f in frames:
        tx.push(f)
    tx.finish()
    fg.run(buffer_items=1 << 16)
    sw = lora.SynchWord(value=0x12).expand()
    want, _ = _oracle_stream(frames, 7, 1, True, False, False, 4, sw, 8, 0)
    got = vs.items()
    assert got.size == want.size and lo.ulp_diff(got, want) <= 1
    assert np.array_equal(np.fromfile(tmp_path / "lora.cf32", np.complex64).view(np.uint64), got.view(np.uint64))
    b = tx.bursts()
    assert list(b["len"]) == [lo.frame_len(7, 4, 8, 0, len(lo.encode(f, 7, 1, True, False, False))) for f in frames]
