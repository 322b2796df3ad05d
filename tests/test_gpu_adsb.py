"""AdsbDemod (csrc/adsb.cu) on the GPU, bit for bit against the C oracle (tests/adsb_oracle.c): random streams at
controlled trigger densities (none, sparse, half, every position) and sizes around 64, 544 and the 4096-position
tile, one exec, ragged execs and single-item steps, non-finite inputs, reset, forward_failed_crc, the refusals and
handle cleanup, and the ADS-B receive front end (listen_adsb.rs:85-120) on synthesised PPM frames."""
import ctypes as C

import numpy as np
import pytest
import torch

import futuresdr_b200 as fb
from futuresdr_b200 import _lib, adsb
from futuresdr_b200._lib import lib
from futuresdr_b200.blocks import AdsbDemod
from futuresdr_b200.edges import Flowgraph, VectorSink, VectorSource

import adsb_oracle as orc

pytestmark = pytest.mark.gpu

# frames of test_front_end_synthesised_frames that the reference receiver decodes one sample early (see there)
PINNED_EARLY = {2_200_000: ["8D40621D58C386435CC412692AD6", "8D88890FAA0CE614A75C839D4A90",
                            "8B69D8233BB4261F2939574CCDF0"]}
DF17 = ["8D4840D6202CC371C32CE0576098", "8D40621D58C382D690C8AC2863A7", "8D40621D58C386435CC412692AD6"]


def _stream(n, density, seed, thr=10.0):
    """samples, nf, corr with P(corr > thr * nf) = density."""
    rng = np.random.default_rng(seed)
    s = rng.exponential(1.0, n).astype(np.float32)
    nf = rng.uniform(0.25, 2.0, n).astype(np.float32)
    hit = rng.random(n) < density
    f = np.where(hit, rng.uniform(1.01, 4.0, n), rng.uniform(0.0, 0.99, n)).astype(np.float32)
    corr = (np.float32(thr) * nf * f).astype(np.float32)
    return s, nf, corr


def _device(thr, s, nf, corr, cuts=(), fwd=True, blk=None):
    """Execs on growing slices: before exec k every input holds cuts[k] items, then a final exec on everything."""
    blk = blk or AdsbDemod(thr, fwd)
    d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (s, nf, corr)]
    n, pos = min(a.numel() for a in d), 0
    for cut in cuts:
        if cut >= n or cut < pos:
            continue
        c, done = blk.exec(*(a[pos:cut] for a in d), finished=False)
        assert not done
        pos += c
    c, done = blk.exec(*(a[pos:n] for a in d), finished=True)
    assert done
    return blk, blk.detections(), blk.packets()


def _check(thr, s, nf, corr, dets, pks, fwd=True, cuts=None):
    tags, packets, _ = orc.replay(thr, s, nf, corr, cuts)
    idx = np.array([t[0] for t in tags], np.uint64)
    val = np.array([t[1] for t in tags], np.float32)
    assert dets.size == len(tags), (dets.size, len(tags))
    assert np.array_equal(dets["index"], idx)
    g, w = dets["value"].copy(), val
    assert np.array_equal(np.isnan(g), np.isnan(w))
    ok = ~np.isnan(w)
    assert np.array_equal(g[ok].view(np.uint32), w[ok].view(np.uint32))
    want = [p for p in packets if fwd or p[2]]
    assert pks.size == len(want), (pks.size, len(want))
    for got, (gi, gv, crc, by) in zip(pks, want):
        assert int(got["preamble_index"]) == gi
        assert (np.isnan(got["preamble_correlation"]) and np.isnan(gv)) or \
            np.float32(got["preamble_correlation"]).view(np.uint32) == np.float32(gv).view(np.uint32)
        assert bool(got["crc_passed"]) == crc
        assert bytes(got["bytes"].tolist()) == by
    return len(tags), len(want)


@pytest.mark.parametrize("density", [0.0, 0.002, 0.5, 1.0])
@pytest.mark.parametrize("n", [0, 1, 63, 64, 65, 96, 543, 544, 545, 1000, 4095 + 64, 4096 + 64, 4097 + 64,
                               3 * 4096 + 95, 100_003])
def test_density_and_size_one_exec(n, density):
    s, nf, corr = _stream(n, density, n * 7 + int(density * 1000))
    _, dets, pks = _device(10.0, s, nf, corr)
    _check(10.0, s, nf, corr, dets, pks)


@pytest.mark.parametrize("density", [0.002, 1.0])
def test_large_stream(density):
    n = (64 << 20) if density < 0.5 else (4 << 20)
    s, nf, corr = _stream(n, density, 99)
    _, dets, pks = _device(10.0, s, nf, corr, cuts=[n // 3, n // 2 + 12345])
    nt, _ = _check(10.0, s, nf, corr, dets, pks, cuts=[n // 3])
    assert nt > 0


@pytest.mark.parametrize("density", [0.01, 0.5, 1.0])
def test_ragged_and_single_step_execs(density):
    n = 20_000
    s, nf, corr = _stream(n, density, 5)
    rng = np.random.default_rng(6)
    ragged = np.cumsum(rng.integers(1, 3000, 40)).tolist()
    steps = list(range(500, 700)) + list(range(4100, 4300)) + [9000 + k for k in range(0, 200, 3)]
    for cuts in (ragged, steps, [64, 544, 545, 1088, 4160, 4161, 8256]):
        _, dets, pks = _device(10.0, s, nf, corr, cuts=cuts)
        _check(10.0, s, nf, corr, dets, pks)


def test_non_finite_inputs():
    n = 30_000
    s, nf, corr = _stream(n, 0.05, 11)
    rng = np.random.default_rng(12)
    for a in (s, nf, corr):
        k = rng.integers(0, n, 600)
        a[k[:200]] = np.nan
        a[k[200:400]] = np.inf
        a[k[400:]] = -np.inf
    nf[rng.integers(0, n, 300)] = 0.0
    corr[rng.integers(0, n, 100)] = 0.0
    _, dets, pks = _device(10.0, s, nf, corr, cuts=[7000, 15000])
    _check(10.0, s, nf, corr, dets, pks)


def test_forward_failed_crc_and_reset():
    s, nf, corr = _stream(50_000, 0.02, 21)
    blk, dets, pks = _device(10.0, s, nf, corr, fwd=False)
    _check(10.0, s, nf, corr, dets, pks, fwd=False)
    blk.reset()
    _, dets2, pks2 = _device(10.0, s, nf, corr, blk=blk)
    assert np.array_equal(dets2, dets) and np.array_equal(pks2, pks)
    blk2, dets3, pks3 = _device(10.0, s, nf, corr, fwd=True)
    _check(10.0, s, nf, corr, dets3, pks3, fwd=True)
    assert pks3.size >= pks.size
    blk.close()
    blk2.close()


def test_refusals_and_cleanup():
    ctx = fb.default_context()
    base = ctx.bytes_held
    h = C.c_void_p()
    for thr in (float("nan"), float("inf"), -1.0):
        assert lib.b2s_adsb_create(ctx.handle, thr, 0, C.byref(h)) == _lib.EINVAL
        assert h.value is None
    blk = AdsbDemod(10.0)
    x = torch.zeros(2000, device="cuda")
    c, dn = C.c_size_t(0), C.c_int32(0)
    bad = C.c_void_p(x.data_ptr() + 2)
    assert lib.b2s_adsb_exec(blk._h, bad, 1000, C.c_void_p(x.data_ptr()), 1000, C.c_void_p(x.data_ptr()), 1000, 0,
                             C.byref(c), C.byref(dn)) == _lib.EINVAL
    assert lib.b2s_adsb_exec(blk._h, None, 1000, C.c_void_p(x.data_ptr()), 1000, C.c_void_p(x.data_ptr()), 1000, 0,
                             C.byref(c), C.byref(dn)) == _lib.EINVAL
    assert blk.exec(x, x, x) == (2000 - 544, False)
    torch.cuda.synchronize()
    blk.close()
    assert ctx.bytes_held == base


# ---- the receive front end on synthesised frames ----------------------------------------------------------------
def _crc_frame(rng):
    bits = np.concatenate([[1, 0, 0, 0, 1], rng.integers(0, 2, 83)]).astype(np.uint8)     # DF17 + payload
    data = orc.bits_to_bytes(np.concatenate([bits, np.zeros(24, np.uint8)]))
    crc = orc.crc24_table(np.unpackbits(np.frombuffer(data, np.uint8)))
    return data[:11].hex().upper() + f"{crc:06X}"


def _ppm(frames, fs, rng, amp=1.0, noise=0.02):
    """PPM at 1 Mbit/s: preamble pulses in half-symbols 0, 2, 7, 9, then bit 1 = high first half.  Returns the
    complex baseband at rate fs and each frame's start time in microseconds.

    Frames start on the 0.5 us half-symbol grid.  At 2 MS/s a frame that started between two samples would have
    every pulse split over two samples at half height, and its corr / nf peak (7.5 measured through this front end)
    would stay below the reference's threshold of 10.  At 2.2 MS/s the grid puts frames at every sub-sample phase."""
    starts, t = [], 40.0
    for _ in frames:
        starts.append(t)
        t += 120.0 + 0.5 * rng.integers(160, 400)
    k = 10                                                       # envelope at 10 fs, integrated down to fs
    n = int((t + 60.0) * 1e-6 * fs)
    tt = np.arange(n * k) / (fs * k) * 1e6                       # microseconds
    env = np.zeros(n * k)
    for h, t0 in zip(frames, starts):
        half = np.zeros(240, bool)
        half[[0, 2, 7, 9]] = True
        for j, b in enumerate(orc.hex_to_bits(h)):
            half[16 + 2 * j + (0 if b else 1)] = True
        hs = np.floor((tt - t0) * 2).astype(np.int64)            # half-symbol index (0.5 us each)
        inside = (hs >= 0) & (hs < 240)
        env[inside] = np.where(half[hs[inside]], amp, env[inside])
    env = env.reshape(n, k).mean(axis=1)
    x = env * np.exp(1j * rng.uniform(0, 2 * np.pi)) + noise * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    return x.astype(np.complex64), starts


@pytest.mark.parametrize("fs", [2_000_000, 2_200_000, 4_000_000])
def test_front_end_synthesised_frames(fs):
    rng = np.random.default_rng(fs // 1000)
    frames = DF17 + [_crc_frame(rng) for _ in range(12)]
    x, starts = _ppm(frames, fs, rng)
    fg = Flowgraph()
    src = VectorSource(x, chunk_items=1 << 16)
    fg.add(src)
    b = adsb.front_end(fg, src, fs, threshold=10.0, forward_failed_crc=True)
    sinks = {k: VectorSink(np.float32) for k in ("mag2", "nf", "corr")}
    for k, v in sinks.items():
        fg.connect(b[k], v)
    fg.run(buffer_items=1 << 18)
    s, nf, corr = (sinks[k].items() for k in ("mag2", "nf", "corr"))
    demod = b["demod"]
    dets, pks = demod.detections(), demod.packets()
    _check(10.0, s, nf, corr, dets, pks, fwd=True)
    got = {bytes(p["bytes"].tolist()).hex().upper(): p for p in pks}
    expect = [t0 * 4.0 for t0 in starts]                        # microseconds -> 4 MHz samples
    # At 2.2 MS/s three frames (start phases of 0.3-0.4 input sample) come out with their correlation peak one 4 MHz
    # sample early, and the bits read from there fail the CRC.  That is the reference receiver's result on these
    # streams: _check above reproduces it through the oracle.  They are pinned here as detected but CRC-failing.
    early = PINNED_EARLY.get(fs, [])
    missing = [h for h in frames if h not in got or not int(got[h]["crc_passed"])]
    assert missing == early, missing                             # every other frame, exact bytes, CRC passing
    found = [int(got[h]["preamble_index"]) for h in frames if h not in early]
    expect = [e for h, e in zip(frames, expect) if h not in early]
    failed = [p for p in pks if not int(p["crc_passed"])]
    assert len(failed) == len(early)
    for p, h in zip(failed, early):                              # ... and the pinned ones were found, one sample early
        assert abs(int(p["preamble_index"]) - (starts[frames.index(h)] * 4.0 - 1) - (found[0] - expect[0])) <= 0.5
    off = found[0] - expect[0]
    assert abs(off) < 64, off                                    # the resampler's delay
    for f, e in zip(found, expect):
        assert abs(f - e - off) <= 2, (f, e, off)


def test_lists_grow_with_detections_not_with_positions():
    """An undrained block on an empty channel: the device lists stay at their first size instead of growing by the
    worst case (one detection per 31 positions) on every exec."""
    ctx = fb.default_context()
    base = ctx.bytes_held
    blk = AdsbDemod(10.0)
    n = 1 << 20
    z = torch.zeros(n, device="cuda")
    nf = torch.ones(n, device="cuda")
    blk.exec(z, nf, z)
    torch.cuda.synchronize()
    first = ctx.bytes_held - base
    for _ in range(300):
        blk.exec(z, nf, z)
    torch.cuda.synchronize()
    assert ctx.bytes_held - base <= 4 * first, (first, ctx.bytes_held - base)   # at most two doublings in flight
    assert blk.detections().size == 0 and blk.packets().size == 0
    blk.close()
    assert ctx.bytes_held == base
