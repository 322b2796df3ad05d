"""The keyfob receive chain on the GPU against the C oracle (tests/keyfob_oracle.c): Apply(SliceF32U8) bit for bit
against numpy, Apply(DcBlockF32) at alpha 0.0001 against the reference's running-average closure, KeyfobDecoder
(csrc/keyfob.cu) code for code on random, pulse-train, string, dense and noise-derived streams, sliced every way, up
to 64 Mi items per exec and past 2^32 stream positions, list growth and draining, reset, refusals and cleanup; and the
front end (main.rs:39-79) on OOK codes from a numpy transmitter through noise and a carrier offset."""
import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

import futuresdr_b200 as fb
from futuresdr_b200 import _lib, keyfob
from futuresdr_b200._lib import B200SdrError, lib
from futuresdr_b200.blocks import KEYFOB_CODE, Apply, ApplyOp, KeyfobDecoder, _ptr
from futuresdr_b200.edges import Flowgraph, VectorSink, VectorSource

import keyfob_oracle as ko

pytestmark = pytest.mark.gpu


def _cuts(n, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "one":
        return []
    if kind == "ragged":
        return np.cumsum(rng.integers(1, max(2, n // 7), 12)).tolist()
    return list(range(1, min(n, 3000)))                 # single-item steps, then the rest


# ---- SliceF32U8 --------------------------------------------------------------------------------------------------
def _special(n, seed):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(n) * 10.0 ** rng.integers(-40, 30, n)).astype(np.float32)
    sp = np.array([0.0, -0.0, np.nan, -np.nan, np.inf, -np.inf, 1e-45, -1e-45, 1e-40, -1e-40,
                   np.finfo(np.float32).tiny, -np.finfo(np.float32).tiny], np.float32)
    if n:
        k = rng.integers(0, n, min(n, 64))
        x[k] = sp[rng.integers(0, sp.size, k.size)]
    return x


@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, 7, 17, 1000, 4099, 100_003])
@pytest.mark.parametrize("in_off,out_off", [(0, 0), (1, 0), (0, 1), (2, 3), (3, 2), (1, 1)])
def test_slicer_bit_exact_unaligned(n, in_off, out_off):
    x = _special(n, n + 7 * in_off + out_off)
    xd = torch.zeros(n + 8, device="cuda")
    xd[in_off:in_off + n] = torch.from_numpy(x).cuda()
    o = torch.full((n + 8,), 7, dtype=torch.uint8, device="cuda")
    blk = Apply(ApplyOp.SliceF32U8)
    assert blk.apply(xd[in_off:in_off + n], o[out_off:out_off + n]) == n
    got = o.cpu().numpy()
    assert np.array_equal(got[out_off:out_off + n], (x > 0).astype(np.uint8))
    assert np.array_equal(got[out_off:out_off + n], ko.slice_u8(x))
    assert (got[:out_off] == 7).all() and (got[out_off + n:] == 7).all()


def test_slicer_64mi_repeated_execs_and_refusals():
    n = 64 << 20
    x = torch.randn(n, device="cuda")
    x[::1001] = float("nan")
    x[::997] = -0.0
    o = torch.empty(n + 3, dtype=torch.uint8, device="cuda")
    blk = Apply(ApplyOp.SliceF32U8)
    for a, b in [(0, 5), (5, 1 << 20), (1 << 20, n // 2 + 3), (n // 2 + 3, n)]:
        assert blk.apply(x[a:b], o[3 + a:3 + b]) == b - a
    assert torch.equal(o[3:], (x > 0).to(torch.uint8))
    c, p = C.c_size_t(0), C.c_size_t(0)
    assert lib.b2s_apply_exec(blk._h, C.c_void_p(x.data_ptr() + 2), 10, _ptr(o), 10, C.byref(c), C.byref(p)) == \
        _lib.EINVAL
    assert lib.b2s_apply_exec(blk._h, _ptr(x), 16, C.c_void_p(x.data_ptr() + 8), 16, C.byref(c), C.byref(p)) == \
        _lib.EINVAL
    blk.close()


# ---- DcBlockF32 as the keyfob's running average -----------------------------------------------------------------
@pytest.mark.parametrize("cuts", [[], [1, 2, 5000, 5001, 77_777]])
def test_dc_block_is_the_keyfob_average(cuts):
    rng = np.random.default_rng(5)
    x = (np.abs(rng.standard_normal(200_000)) ** 2 + (np.arange(200_000) % 300 < 150)).astype(np.float32)
    blk = Apply(ApplyOp.DcBlockF32, keyfob.DC_ALPHA)
    d = torch.from_numpy(x).cuda()
    out = torch.empty_like(d)
    edges = [0] + cuts + [x.size]
    for a, b in zip(edges[:-1], edges[1:]):
        if b > a:
            blk.apply(d[a:b], out[a:b])
    y = out.cpu().numpy()
    assert np.array_equal(y.view(np.uint32), ko.Avg(0.0001).work(x).view(np.uint32))


# ---- KeyfobDecoder -----------------------------------------------------------------------------------------------
def _dev(x, cuts=(), blk=None):
    blk = blk or KeyfobDecoder()
    d = torch.from_numpy(np.ascontiguousarray(x, np.uint8)).cuda()
    edges = [0] + [c for c in cuts if 0 < c < x.size] + [x.size]
    for a, b in zip(edges[:-1], edges[1:]):
        assert blk.exec(d[a:b]) == b - a
    return blk, blk.codes()


def _check(x, cuts=(), want=None):
    blk, got = _dev(x, cuts)
    want = ko.decode(x, cuts) if want is None else want
    assert [ko.code_tuple(g) for g in got] == want, (got.size, len(want))
    return got


def _pulses(widths, start=0):
    level, out = start, []
    for w in widths:
        out.append(np.full(int(w), level, np.uint8))
        level ^= 1
    return np.concatenate(out) if out else np.zeros(0, np.uint8)


@pytest.mark.parametrize("n", [0, 1, 15, 16, 17, 4095, 4096, 4097, 100_003, 1 << 20])
def test_decoder_random_0_to_3(n):
    rng = np.random.default_rng(n)
    x = rng.integers(0, 4, n).astype(np.uint8)
    _check(x, [n // 3, n // 2 + 1])


def _strings(rng):
    cases = ["10101111" + "11010101", "10101111" + "11100011", "10101111" + "10111001", "10101111", "1010111",
             "0000" + "10101111" + "0110", "1010101111" + "01", "1010111110101111" + "11010101", "", "1",
             "10101111" * 3 + "1110001", "0110" * 20 + "10101111" + "1" * 300 + "11100011"]
    return [ko.levels_for(s, rng, lead=int(rng.integers(162, 900)), start_level=int(rng.integers(0, 2)))
            for s in cases]


@pytest.mark.parametrize("kind", ["one", "ragged", "steps"])
def test_decoder_strings_labels_any_slicing(kind):
    rng = np.random.default_rng(11)
    x = np.concatenate(_strings(rng) * 3)
    want = ko.py_decode(x)
    assert len(want) >= 20 and {c[2] for c in want} == {0, 1, 2, 3}
    assert any(c[1] > 256 for c in want)
    _check(x, _cuts(x.size, kind, 3), want)


def test_decoder_range_edges():
    rng = np.random.default_rng(12)
    widths = rng.choice([62, 63, 83, 84, 130, 131, 161, 162, 5, 300], 200_000)
    x = _pulses(widths)
    want = ko.py_decode(x[:3_000_000])
    assert want == ko.decode(x[:3_000_000])
    _check(x, [4096 * 7 + 3, 1 << 20])
    # 2..255 are ignored, whatever their place
    y = x.copy()
    y[rng.integers(0, y.size, y.size // 50)] = rng.integers(2, 256, y.size // 50).astype(np.uint8)
    _check(y, [12345])


def test_decoder_dense_valid_pulses_and_noise_slicer_streams():
    x = np.resize(_pulses([63, 63]), 64 << 20).astype(np.uint8)      # the densest stream: every edge appends or sets
    _check(x, [777, 30_000_001])
    rng = np.random.default_rng(13)
    z = rng.standard_normal(1 << 22).astype(np.float32)
    lp = np.convolve(z, keyfob.lowpass_taps(), "valid").astype(np.float32)
    _check(ko.slice_u8(lp), [4096, 1 << 20])
    slow = np.convolve(z, np.ones(70, np.float32) / 70, "valid").astype(np.float32)
    _check(ko.slice_u8(slow), [3, 4099])


def test_decoder_64mi_codes_across_tiles_and_execs():
    rng = np.random.default_rng(14)
    parts = []
    while sum(p.size for p in parts) < (64 << 20):
        bits = "".join(rng.choice(["0", "1"], int(rng.integers(0, 40)))) + "10101111" + \
            "".join(rng.choice(["0", "1"], int(rng.integers(0, 300)))) + rng.choice(["11010101", "11100011", ""])
        parts.append(ko.levels_for(bits, rng, lead=int(rng.integers(162, 5000)), start_level=int(rng.integers(0, 2))))
    x = np.concatenate(parts)[:64 << 20]
    want = ko.decode(x)
    assert len(want) > 1000
    _check(x, [], want)
    _check(x, np.cumsum(rng.integers(1, 3_000_000, 40)).tolist(), want)


def test_decoder_positions_past_2_pow_32():
    blk = KeyfobDecoder()
    z = torch.zeros(1 << 30, dtype=torch.uint8, device="cuda")
    for _ in range(4):
        blk.exec(z)
    x = ko.levels_for("10101111" + "11100011", np.random.default_rng(15), lead=500)
    blk.exec(z[:123])
    _, got = _dev(x, blk=blk)
    want = ko.decode(np.concatenate([np.zeros(123, np.uint8), x]))
    off = 4 << 30
    assert [ko.code_tuple(g) for g in got] == [(i + off, nb, lb, bi) for i, nb, lb, bi in want]
    assert len(want) == 1 and want[0][0] + off > 2 ** 32


def test_decoder_list_growth_drain_reset_and_cleanup():
    ctx = fb.default_context()
    base = ctx.bytes_held
    rng = np.random.default_rng(16)
    one = ko.levels_for("10101111" + "11010101", rng, lead=200)
    x = np.tile(one, 3000)
    want = ko.decode(x)
    assert len(want) == 3000
    blk = KeyfobDecoder()
    d = torch.from_numpy(x).cuda()
    for k in range(10):                                 # undrained: the list grows
        blk.exec(d[k * x.size // 10:(k + 1) * x.size // 10])
    buf = np.zeros(7, KEYFOB_CODE)
    n, got = C.c_size_t(0), []
    while True:                                         # drain with a small cap
        assert lib.b2s_keyfob_drain_codes(blk._h, buf.ctypes.data_as(C.c_void_p), buf.size, C.byref(n)) == 0
        got += [ko.code_tuple(g) for g in buf[:n.value]]
        if n.value < buf.size:
            break
    assert got == want
    blk.reset()
    _, again = _dev(x[:50 * one.size], blk=blk)
    assert [ko.code_tuple(g) for g in again] == want[:50]
    h = C.c_void_p()
    assert lib.b2s_keyfob_create(None, C.byref(h)) == _lib.EINVAL
    assert lib.b2s_keyfob_exec(blk._h, None, 10, C.byref(C.c_size_t())) == _lib.EINVAL
    assert lib.b2s_keyfob_exec(None, _ptr(d), 10, C.byref(C.c_size_t())) == _lib.EINVAL
    assert lib.b2s_keyfob_exec(blk._h, _ptr(d), 10, None) == _lib.EINVAL
    assert lib.b2s_keyfob_drain_codes(blk._h, None, 5, C.byref(n)) == _lib.EINVAL
    assert lib.b2s_keyfob_reset(None) == _lib.EINVAL
    blk.exec(d)                                         # destroyed with codes undrained
    blk.close()
    del d
    assert ctx.bytes_held == base


def _golden():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "keyfob_known_answers.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", _golden()["decoder"], ids=lambda c: c["name"])
def test_known_answers_on_device(case):
    x = np.array([int(c) for c in case["items"]], np.uint8)
    _, got = _dev(x, case.get("cuts", []))
    assert [[int(g["index"]), keyfob.code_string(g)] for g in got] == case["codes"]


# ---- the receive front end ---------------------------------------------------------------------------------------
SNR_DB = 10                                  # the CPU restatement of the chain recovers every code from 6 dB


def _transmit(rng, codes, snr_db, cfo):
    """OOK at 4 Msps: each 250 kHz slicer item is 16 samples, carrier on while the level is 1; periods at the middle of
    their ranges (73 and 146 items).  A warm-up of short
    bursts lets the running average settle; each code is preceded by a gap (its first edge flushes) and followed by two
    40-item periods (their edges flush the code)."""
    warm = np.tile(np.repeat(np.array([1, 0], np.uint8), 10), 2000)
    lv = [warm]
    for c in codes:
        # the code without levels_for's closing 20-item period, then two 40-item periods: a flush the FIR keeps
        y = ko.levels_for(c, rng, lead=int(rng.integers(400, 1500)), short=(73, 73), long=(146, 146))[:-25]
        lv += [y, np.full(40, y[-1] ^ 1, np.uint8), np.full(40, y[-1], np.uint8)]
    lv = np.concatenate(lv + [np.zeros(600, np.uint8)])
    s = np.repeat(lv.astype(np.float64), 16)
    t = np.arange(s.size)
    x = s * np.exp(1j * (2 * np.pi * cfo / 4e6 * t + rng.uniform(0, 2 * np.pi)))
    sigma = np.sqrt(0.5 * 10 ** (-snr_db / 10))
    x = x + sigma * (rng.standard_normal(x.size) + 1j * rng.standard_normal(x.size))
    return x.astype(np.complex64)


def test_front_end_ook_codes():
    rng = np.random.default_rng(17)
    labels = ["11010101", "11100011", "10111001", "00110011"]
    codes = ["".join(rng.choice(["0", "1"], int(rng.integers(0, 12)))) + "10101111" +
             "".join(rng.choice(["0", "1"], 16)) + labels[k % 4] for k in range(12)]
    x = _transmit(rng, codes, SNR_DB, cfo=20e3)
    fg = Flowgraph()
    src = VectorSource(x, chunk_items=1 << 16)
    fg.add(src)
    b = keyfob.front_end(fg, src)
    lp_sink, sl_sink = VectorSink(np.float32), VectorSink(np.uint8)
    fg.connect(b["low_pass"], lp_sink)
    fg.connect(b["slice"], sl_sink)
    fg.run(buffer_items=1 << 17)
    lp, sl = lp_sink.items(), sl_sink.items()
    got = b["decoder"].codes()
    # from the FIR's output on, the device chain equals the oracle's
    assert np.array_equal(sl, ko.slice_u8(lp))
    want = ko.decode(sl)
    assert [ko.code_tuple(g) for g in got] == want
    sent = [c[c.index("10101111"):] + keyfob.LABELS[{"11010101": 1, "11100011": 2, "10111001": 3}.get(c[-8:], 0)]
            for c in codes]
    assert [keyfob.code_string(g) for g in got] == sent
