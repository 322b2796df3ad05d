"""The ZigBee receive chain on the GPU, bit for bit against the C oracle (tests/zigbee_oracle.c): Apply(DcBlockF32),
ClockRecoveryMm and ZigbeeDecoder (csrc/apply.cu, csrc/zigbee.cu) at sizes from 0 to 64 Mi, in one exec, ragged and
single-item execs, output-capacity-limited calls, non-finite inputs, a step longer than the shared ring, reset, the
refusals and handle cleanup, the hand-worked cases of tests/golden/zigbee_known_answers.json; and the
front end (rx.rs:66-92) on O-QPSK frames from a numpy transmitter (modulator.rs, iq_delay.rs) through a channel with
noise, a carrier offset and a sample-rate offset."""
import ctypes as C
import json
import os
import tempfile

import numpy as np
import pytest
import torch

import futuresdr_b200 as fb
from futuresdr_b200 import _lib, zigbee
from futuresdr_b200._lib import B200SdrError, lib
from futuresdr_b200.blocks import Apply, ApplyOp, ClockRecoveryMm, ZigbeeDecoder, _ptr
from futuresdr_b200.edges import FileSource, Flowgraph, VectorSink

import zigbee_oracle as zo

pytestmark = pytest.mark.gpu

MM = (2.0, 0.000225, 0.5, 0.03, 0.0002)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _same(a, b):
    """bit for bit, except that any NaN equals any NaN (the device's NaN is not libm's)"""
    assert a.shape == b.shape, (a.shape, b.shape)
    na, nb = np.isnan(a), np.isnan(b)
    bad = np.flatnonzero((na != nb) | (~na & ~nb & (_bits(a) != _bits(b))))
    assert bad.size == 0, (bad[:5], a[bad[:5]], b[bad[:5]])


def _cuts(n, kind, seed=0):
    rng = np.random.default_rng(seed)
    if kind == "one":
        return []
    if kind == "ragged":
        return np.cumsum(rng.integers(1, max(2, n // 7), 12)).tolist()
    return list(range(1, min(n, 300)))                  # single-item steps


def _phase_like(n, seed):
    rng = np.random.default_rng(seed)
    return (np.sin(np.arange(n) * 0.7) * 1.2 + 0.3 * rng.standard_normal(n)).astype(np.float32)


# ---- DcBlockF32 --------------------------------------------------------------------------------------------------
def _dc_device(x, cuts, alpha=0.00016, blk=None):
    blk = blk or Apply(ApplyOp.DcBlockF32, alpha)
    d = torch.from_numpy(x).cuda()
    out = torch.full((x.size,), float("nan"), device="cuda")
    edges = [0] + [c for c in cuts if 0 < c < x.size] + [x.size]
    for a, b in zip(edges[:-1], edges[1:]):
        if b > a:
            assert blk.apply(d[a:b], out[a:b]) == b - a
    return blk, out.cpu().numpy()


@pytest.mark.parametrize("kind", ["one", "ragged", "steps"])
@pytest.mark.parametrize("n", [0, 1, 2, 31, 2047, 2048, 2049, 3 * 2048 + 5, 100_003])
def test_dc_block_sizes_and_slicing(n, kind):
    x = _phase_like(n, n)
    _, y = _dc_device(x, _cuts(n, kind, n))
    _same(y, zo.DcBlock(0.00016).work(x))


def test_dc_block_64mi_non_finite_and_reset():
    n = 64 << 20
    x = _phase_like(n, 3)
    blk, y = _dc_device(x, [n // 3, n // 2 + 7])
    _same(y, zo.DcBlock(0.00016).work(x))
    blk.reset()
    x2 = _phase_like(100_000, 4)
    x2[[10, 500, 9000]] = [np.inf, -np.inf, np.nan]
    _, y2 = _dc_device(x2, [5000], blk=blk)
    _same(y2, zo.DcBlock(0.00016).work(x2))
    for alpha in (0.5, 1.0, -0.25):
        _, y3 = _dc_device(x2[:20000], [333], alpha)
        _same(y3, zo.DcBlock(alpha).work(x2[:20000]))


def test_dc_block_refusals():
    ctx = fb.default_context()
    h = C.c_void_p()
    for a in (float("nan"), float("inf"), -float("inf")):
        assert lib.b2s_apply_create(ctx.handle, _lib.OP_DC_BLOCK_F32, a, C.byref(h)) == _lib.EINVAL
        assert h.value is None
    blk = Apply(ApplyOp.DcBlockF32, 0.1)
    x = torch.zeros(1000, device="cuda")
    with pytest.raises(B200SdrError):
        blk.apply(x[:600], x[400:])                      # overlap
    c, p = C.c_size_t(0), C.c_size_t(0)
    assert lib.b2s_apply_exec(blk._h, C.c_void_p(x.data_ptr() + 2), 10, C.c_void_p(x.data_ptr() + 2000), 10,
                              C.byref(c), C.byref(p)) == _lib.EINVAL
    assert lib.b2s_apply_exec(blk._h, None, 10, C.c_void_p(x.data_ptr()), 10, C.byref(c), C.byref(p)) == _lib.EINVAL
    blk.close()


# ---- ClockRecoveryMm ---------------------------------------------------------------------------------------------
def _mm_device(x, cuts, params=MM, n_out=None, blk=None):
    """Calls on growing slices, as zo.mm_replay makes them -> (outputs, consumed, index of the call that raised)."""
    blk = blk or ClockRecoveryMm(*params)
    d = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    cuts = [c for c in cuts if c < x.size] + [x.size]
    pos, outs = 0, []
    for k, cut in enumerate(cuts):
        cut = max(cut, pos)
        while True:
            cap = (cut - pos + 8) if n_out is None else n_out
            o = torch.full((max(cap, 1),), float("nan"), device="cuda")
            c, p = C.c_size_t(0), C.c_size_t(0)
            rc = lib.b2s_mmclock_exec(blk._h, C.c_void_p(d.data_ptr() + 4 * pos), cut - pos,
                                      C.c_void_p(o.data_ptr()), cap, C.byref(c), C.byref(p))
            assert rc in (_lib.OK, _lib.ESTATE), rc
            pos += c.value
            outs.append(o[:p.value].cpu().numpy())
            if rc == _lib.ESTATE:
                return np.concatenate(outs), pos, k
            if n_out is None or p.value < n_out or c.value == 0:
                break
    return np.concatenate(outs), pos, None


def _mm_check(x, cuts, params=MM, n_out=None):
    got = _mm_device(x, cuts, params, n_out)
    want = zo.mm_replay(params, x, cuts, n_out)
    _same(got[0], want[0])
    assert got[1:] == want[1:], (got[1:], want[1:])
    return got


@pytest.mark.parametrize("kind", ["one", "ragged", "steps"])
@pytest.mark.parametrize("n", [0, 1, 3, 4, 5, 1023, 1025, 8192 + 3, 3 * 8192 + 17, 100_001])
def test_mm_sizes_and_slicing(n, kind):
    x = _phase_like(n, 7 + n)
    out, pos, err = _mm_check(x, _cuts(n, kind, n))
    assert err is None and (n < 4 or out.size > 0)


def test_mm_64mi():
    n = 64 << 20
    x = _phase_like(n, 8)
    out, pos, _ = _mm_check(x, [n // 3])
    assert pos >= n - 4 and abs(out.size - n // 2) < n // 100


@pytest.mark.parametrize("n_out", [1, 7, 1024, 1025, 5000])
def test_mm_output_capacity(n_out):
    x = _phase_like(30_000, 9)
    _mm_check(x, [10_000, 20_001], n_out=n_out)


@pytest.mark.parametrize("params", [(2.0, 0.01, 0.2, 0.2, 0.05), (1.0, 0.0, 0.99, 0.0, 0.0), (3.7, 0.001, 0.0, 0.1, 0.3),
                                    (0.5, 0.0002, 0.5, 0.6, 0.0)])
def test_mm_other_parameters(params):
    x = _phase_like(40_000, 10)
    _mm_check(x, [12_345], params)


def test_mm_nan_latch_and_out_of_slice_steps():
    x = _phase_like(20_000, 11)
    x[5000] = np.nan
    out, pos, err = _mm_check(x, [3000, 9000], n_out=4096)
    assert err is None and np.isnan(out[-1])
    y = _phase_like(20_000, 12)
    y[7000] = 1e9                                        # far above |mm_val| ~ 1: a step of ~3e7 items
    _, _, err = _mm_check(y, [6000, 15000])
    assert err is not None
    z = _phase_like(10_000, 13)
    z[4000] = np.inf
    _mm_check(z, [])
    w = _phase_like(10_000, 14)
    w[[100, 200]] = [-np.inf, np.nan]
    _mm_check(w, [150], n_out=777)


def test_mm_reset_refusals_and_cleanup():
    ctx = fb.default_context()
    base = ctx.bytes_held
    h = C.c_void_p()
    bad = [(float("nan"), 0.1, 0.5, 0.1, 0.1), (2.0, float("inf"), 0.5, 0.1, 0.1), (2.0, 0.1, 0.5, 0.1, -0.1),
           (2.0, 0.1, 0.5, 0.1, float("nan")), (-2.0, 0.1, 0.5, 0.1, 0.1), (0.0, 0.1, 0.5, 0.0, 0.1)]
    for p in bad:
        assert lib.b2s_mmclock_create(ctx.handle, *p, C.byref(h)) == _lib.EINVAL, p
        assert h.value is None
    blk = ClockRecoveryMm(*MM)
    assert blk.look_ahead == 3
    x = _phase_like(50_000, 15)
    a = _mm_device(x, [777], blk=blk)
    blk.reset()
    b = _mm_device(x, [777], blk=blk)
    _same(a[0], b[0])
    t = torch.zeros(1000, device="cuda")
    c, p = C.c_size_t(0), C.c_size_t(0)
    for args in ((C.c_void_p(t.data_ptr() + 2), 100, C.c_void_p(t.data_ptr() + 2000), 100),
                 (None, 100, C.c_void_p(t.data_ptr()), 100),
                 (C.c_void_p(t.data_ptr()), 600, C.c_void_p(t.data_ptr() + 400), 600)):
        assert lib.b2s_mmclock_exec(blk._h, *args, C.byref(c), C.byref(p)) == _lib.EINVAL
    assert blk.exec(t[:3], t[500:600]) == (0, 0)         # within the look-ahead: the loop does not run
    blk.close()
    assert ctx.bytes_held == base


# ---- ZigbeeDecoder -----------------------------------------------------------------------------------------------
def _frame_chips(rng, n_frames, gap=(0, 3000), lens=(1, 110)):
    parts, frames = [], []
    for s in range(n_frames):
        parts.append(rng.integers(0, 2, int(rng.integers(*gap))).astype(np.uint8))
        f = zo.mac_frame(rng.integers(0, 256, int(rng.integers(*lens))).astype(np.uint8).tobytes(), s)
        frames.append(f[5:])
        parts.append(zo.chips_of(f))
    parts.append(rng.integers(0, 2, 500).astype(np.uint8))
    chips = np.concatenate(parts)
    soft = np.where(chips > 0, 1.0, -1.0) * rng.uniform(0.1, 1.0, chips.size)
    return soft.astype(np.float32), frames


def _dec_device(x, cuts, thr=6, blk=None):
    blk = blk or ZigbeeDecoder(thr)
    d = torch.from_numpy(x).cuda()
    edges = [0] + sorted(c for c in set(cuts) if 0 < c < x.size) + [x.size]
    for a, b in zip(edges[:-1], edges[1:]):
        assert blk.exec(d[a:b]) == b - a
    return blk, blk.frames()


def _dec_check(x, cuts, thr=6):
    blk, got = _dec_device(x, cuts, thr)
    want = zo.decode_replay(thr, x, cuts)
    assert got.size == len(want), (got.size, len(want))
    for g, (i, by) in zip(got, want):
        assert int(g["index"]) == i
        assert int(g["len"]) == len(by) and bytes(g["bytes"][:len(by)].tolist()) == by
        assert not g["bytes"][len(by):].any()
        assert bool(g["crc_ok"]) == zo.crc_ok(by)
    return blk, got


@pytest.mark.parametrize("kind", ["one", "ragged", "steps"])
def test_decoder_frames_any_slicing(kind):
    rng = np.random.default_rng(20)
    x, frames = _frame_chips(rng, 40)
    _, got = _dec_check(x, _cuts(x.size, kind, 21))
    assert [bytes(g["bytes"][:g["len"]].tolist()) for g in got] == frames
    assert got["crc_ok"].all()


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 1000, 1 << 20])
@pytest.mark.parametrize("thr", [0, 6, 12, 33])
def test_decoder_noise(n, thr):
    rng = np.random.default_rng(n + thr)
    x = rng.standard_normal(n).astype(np.float32)
    _dec_check(x, [n // 3, n // 2 + 1], thr)


def test_decoder_dense_preamble_and_64mi():
    pre = zo.chips_of(bytes(4))[:256]
    x = np.where(np.tile(pre, 1 << 12) > 0, 1.0, -1.0).astype(np.float32)     # all preamble
    _dec_check(x, [12345, 500_000])
    rng = np.random.default_rng(22)
    f, _ = _frame_chips(rng, 200, gap=(0, 40_000))
    n = 64 << 20
    big = np.resize(f, n).astype(np.float32)
    big[::97] = -big[::97]                                # some chip errors
    big[rng.integers(0, n, 50)] = np.nan
    _, got = _dec_check(big, [n // 3])
    assert got.size > 1000


def test_decoder_list_growth_drain_reset_and_cleanup():
    ctx = fb.default_context()
    base = ctx.bytes_held
    blk = ZigbeeDecoder(6)
    z = -torch.ones(1 << 20, device="cuda")
    blk.exec(z)
    torch.cuda.synchronize()
    first = ctx.bytes_held - base
    for _ in range(300):
        blk.exec(z)
    torch.cuda.synchronize()
    assert ctx.bytes_held - base <= 4 * first, (first, ctx.bytes_held - base)
    assert blk.frames().size == 0
    rng = np.random.default_rng(23)
    x, frames = _frame_chips(rng, 10)
    blk.reset()
    _, a = _dec_device(x, [5000], blk=blk)
    blk.reset()
    _, b = _dec_device(x, [7000], blk=blk)
    assert np.array_equal(a, b) and a.size == len(frames)
    h = C.c_void_p()
    assert lib.b2s_zigbee_exec(blk._h, C.c_void_p(z.data_ptr() + 2), 10, C.byref(C.c_size_t())) == _lib.EINVAL
    assert lib.b2s_zigbee_exec(blk._h, None, 10, C.byref(C.c_size_t())) == _lib.EINVAL
    assert lib.b2s_zigbee_create(None, 6, C.byref(h)) == _lib.EINVAL
    blk.close()
    assert ctx.bytes_held == base


# ---- the receive front end ---------------------------------------------------------------------------------------
_S0, _S8 = "11011001110000110101001000101110", "10001100100101100000011101111011"   # IEEE 802.15.4 symbols 0 and 8


def _std_chips(i):
    base = _S0 if i < 8 else _S8
    k = (i % 8) * 4                                     # symbols 1-7 / 9-15: cyclic shifts by 4 chips
    s = base[-k:] + base[:-k] if k else base
    return np.array([int(c) for c in s])


def _modulate(frame):
    """modulator.rs: per nibble (low first) 16 complex chips (even chips on I, odd on Q), each 4 samples of the
    half-sine SHAPE; then iq_delay.rs: Q two samples late."""
    shape = np.array([0.0, np.sqrt(0.5), 1.0, np.sqrt(0.5)])
    out = []
    for b in frame:
        for nib in (b & 0xF, b >> 4):
            c = 2 * _std_chips(nib) - 1
            out.append(np.repeat(c[0::2] + 1j * c[1::2], 4) * np.tile(shape, 16))
    x = np.concatenate(out)
    return np.concatenate([x.real, [0, 0]]) + 1j * np.concatenate([[0, 0], x.imag])


def _channel(rng, payloads, snr_db, ppm, cfo):
    parts = [np.zeros(2000)]
    for s, p in enumerate(payloads):
        parts += [_modulate(zo.mac_frame(p, s)), np.zeros(int(rng.integers(500, 5000)))]
    x = np.concatenate(parts)
    t = np.arange(int(x.size / (1 + ppm * 1e-6))) * (1 + ppm * 1e-6)          # sample-rate offset
    x = np.interp(t, np.arange(x.size), x.real) + 1j * np.interp(t, np.arange(x.size), x.imag)
    x = x * np.exp(1j * (2 * np.pi * cfo / 4e6 * np.arange(x.size) + rng.uniform(0, 2 * np.pi)))
    sigma = np.sqrt(0.5 * 10 ** (-snr_db / 10))
    x = x + sigma * (rng.standard_normal(x.size) + 1j * rng.standard_normal(x.size))
    return x.astype(np.complex64)


@pytest.mark.parametrize("snr_db,ppm", [(30, 50), (30, -50), (12, 0), (3, 20)])
def test_front_end_oqpsk_frames(snr_db, ppm):
    rng = np.random.default_rng(snr_db * 100 + ppm)
    payloads = [rng.integers(0, 256, int(rng.integers(1, 110))).astype(np.uint8).tobytes() for _ in range(25)]
    x = _channel(rng, payloads, snr_db, ppm, cfo=20e3)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "iq.cf32")
        x.tofile(path)
        fg = Flowgraph()
        src = FileSource(path, np.complex64, chunk_items=1 << 15)
        fg.add(src)
        b = zigbee.front_end(fg, src)
        sinks = {k: VectorSink(np.float32) for k in ("phase", "dc", "mm")}
        for k, v in sinks.items():
            fg.connect(b[k], v)
        fg.run(buffer_items=1 << 17)
    phase, dc, mm = (sinks[k].items() for k in ("phase", "dc", "mm"))
    got = b["decoder"].frames()
    # replay from the device's phase stream (its atan2 is not libm's): DC blocker, clock recovery, decoder
    _same(dc, zo.DcBlock(zigbee.DC_ALPHA).work(phase))
    want_mm, _, err = zo.mm_replay(MM, dc)
    assert err is None
    _same(mm, want_mm)
    want = zo.decode_replay(6, mm)
    assert [int(g["index"]) for g in got] == [i for i, _ in want]
    assert [bytes(g["bytes"][:g["len"]].tolist()) for g in got] == [by for _, by in want]
    ok = {bytes(g["bytes"][:g["len"]].tolist()) for g in got if g["crc_ok"]}
    sent = [zo.mac_frame(p, s)[5:] for s, p in enumerate(payloads)]
    if snr_db >= 12:
        assert all(f in ok for f in sent), sum(f in ok for f in sent)


def _largest_step(params, x):
    """The longest single advance of ii in the oracle's loop over x (one output per call)."""
    m, pos, big = zo.Mm(*params), 0, 0
    while True:
        c, o, e = m.work(x[pos:], 1)
        if e or o.size == 0:
            return big
        big, pos = max(big, c), pos + c


@pytest.mark.parametrize("cuts", [[], [4000, 30_000, 45_000]])
def test_mm_step_longer_than_the_ring(cuts):
    """A step past the 8192-item shared ring that stays inside the slice: the next phase reloads from the new ii."""
    x = _phase_like(60_000, 16)
    x[5000:5002] = 5e5
    assert 8192 < _largest_step(MM, x) < 50_000
    out, pos, err = _mm_check(x, cuts)
    assert err is None and pos >= x.size - 3


def _golden():
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "zigbee_known_answers.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("case", _golden()["decoder"], ids=lambda c: c["name"])
def test_known_answers_decoder_on_device(case):
    x = np.array([1.0 if ch == "1" else -1.0 for ch in case["chips"]], np.float32)
    _, got = _dec_device(x, case.get("cuts", []), case["threshold"])
    assert [(int(g["index"]), bytes(g["bytes"][:g["len"]].tolist()).hex()) for g in got] == \
        [(i, h) for i, h in case["frames"]]


@pytest.mark.parametrize("case", _golden()["mm"], ids=lambda c: c["name"])
def test_known_answers_mm_on_device(case):
    x = torch.tensor([float(v) for v in case["input"]], dtype=torch.float32, device="cuda")
    blk = ClockRecoveryMm(*case["params"])
    o = torch.full((case["n_out"],), float("nan"), device="cuda")
    c, p = C.c_size_t(0), C.c_size_t(0)
    rc = lib.b2s_mmclock_exec(blk._h, _ptr(x), x.numel(), _ptr(o), o.numel(), C.byref(c), C.byref(p))
    assert rc == (_lib.ESTATE if case["err"] else _lib.OK)
    assert c.value == case["consumed"]
    _same(o[:p.value].cpu().numpy(), np.array(case["outputs_bits"], np.uint32).view(np.float32))
    blk.close()
